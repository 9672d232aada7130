// The center loss of Wen et al. (learn_center_loss.py:17-41) and its backward pass, in one launch without float
// atomics.  The grid is split in two parts that read only z, the centroids and the labels:
//
//   row part    one warp per sample b: d = z_b - c_{y_b}, loss_b = 1/2 sum d^2, dz_b = scale * d (overwritten)
//   class part  one warp per class k: dc_k = -scale * sum_{b: y_b = k} (z_b - c_k), the samples collected with ballots
//               and summed in increasing row order; 0 for a class without a sample
//
// Replaces the 'center_dist' / 'center_loss' layers + the 'cls_centroids' Embedding and their TF autodiff; Keras 2.2
// densifies the Embedding's IndexedSlices gradient into exactly this per-class sum.  Rows whose label lies outside
// [0, C) are padding: loss 0, dz 0, and no part in dc.
#include "common.cuh"

namespace se {

constexpr int CL_WARPS = 4;
constexpr int CL_CHUNK = 128;           // columns a warp covers per pass: four per lane

// Columns of chunk c0 that lane `lane` owns.  vec: four consecutive columns (one float4 when all four lie inside D);
// otherwise columns c0 + lane + 32 j, so that a warp's scalar loads stay coalesced.
__device__ __forceinline__ int cl_col(bool vec, int c0, int lane, int j) { return vec ? c0 + 4 * lane + j : c0 + lane + 32 * j; }

__device__ __forceinline__ void cl_load4(const float* __restrict__ p, bool vec, int c0, int lane, int D, float v[4]) {
  if (vec && c0 + 4 * lane + 3 < D) {
    const float4 q = *reinterpret_cast<const float4*>(p + c0 + 4 * lane);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    return;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = cl_col(vec, c0, lane, j);
    v[j] = c < D ? p[c] : 0.f;
  }
}

__device__ __forceinline__ void cl_store4(float* __restrict__ p, bool vec, int c0, int lane, int D, const float v[4]) {
  if (vec && c0 + 4 * lane + 3 < D) {
    *reinterpret_cast<float4*>(p + c0 + 4 * lane) = make_float4(v[0], v[1], v[2], v[3]);
    return;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = cl_col(vec, c0, lane, j);
    if (c < D) p[c] = v[j];
  }
}

__global__ void __launch_bounds__(CL_WARPS * 32)
center_loss_kernel(const float* __restrict__ z, int ldz, const int* __restrict__ labels, const float* __restrict__ cent,
                   int ldc, int B, int C, int D, float scale, float* __restrict__ loss, float* __restrict__ d_z,
                   float* __restrict__ d_cent, int row_ctas, bool vec) {
  pdl_grid_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if ((int)blockIdx.x < row_ctas) {
    // ---- row part
    const int b = blockIdx.x * CL_WARPS + warp;
    if (b >= B) return;
    const int lab = labels[b];
    const bool real = lab >= 0 && lab < C;
    const float* zr = z + (long long)b * ldz;
    const float* cr = cent + (long long)(real ? lab : 0) * ldc;
    float* dzr = d_z ? d_z + (long long)b * ldz : nullptr;
    float sq = 0.f;
    for (int c0 = 0; c0 < D; c0 += CL_CHUNK) {
      float d[4] = {0.f, 0.f, 0.f, 0.f};
      if (real) {
        float zv[4], cv[4];
        cl_load4(zr, vec, c0, lane, D, zv);
        cl_load4(cr, vec, c0, lane, D, cv);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          d[j] = zv[j] - cv[j];
          sq = fmaf(d[j], d[j], sq);            // columns past D load 0 on both sides: d = 0
        }
      }
      if (dzr) {
#pragma unroll
        for (int j = 0; j < 4; ++j) d[j] *= scale;
        cl_store4(dzr, vec, c0, lane, D, d);
      }
    }
    sq = warp_sum(sq);
    if (loss && lane == 0) loss[b] = 0.5f * sq;
    return;
  }
  // ---- class part
  const int k = (blockIdx.x - row_ctas) * CL_WARPS + warp;
  if (k >= C) return;
  const float* ck = cent + (long long)k * ldc;
  float* dck = d_cent + (long long)k * ldc;
  for (int c0 = 0; c0 < D; c0 += CL_CHUNK) {
    float cv[4], acc[4] = {0.f, 0.f, 0.f, 0.f};
    cl_load4(ck, vec, c0, lane, D, cv);
    for (int i0 = 0; i0 < B; i0 += 32) {
      const int i = i0 + lane;
      unsigned mine = __ballot_sync(0xffffffffu, i < B && labels[i] == k);
      while (mine) {                            // this class's rows of the 32, lowest first
        const int b = i0 + __ffs(mine) - 1;
        mine &= mine - 1;
        float zv[4];
        cl_load4(z + (long long)b * ldz, vec, c0, lane, D, zv);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] += zv[j] - cv[j];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] *= -scale;
    cl_store4(dck, vec, c0, lane, D, acc);
  }
}

}  // namespace se

using namespace se;

extern "C" int se_center_loss_fwd_bwd(const float* z, int ldz, const int32_t* labels, const float* cent, int ldc, int B,
                                      int C, int D, float scale, float* loss, float* d_z, float* d_cent, void* stream) {
  SE_REQUIRE(z && labels && cent, "null pointer");
  SE_REQUIRE(B > 0 && C > 0 && D > 0, "need B, C and D >= 1");
  SE_REQUIRE(ldz >= D && ldc >= D, "need ldz >= D and ldc >= D");
  const int row_ctas = (loss || d_z) ? ceil_div(B, CL_WARPS) : 0;
  const int cls_ctas = d_cent ? ceil_div(C, CL_WARPS) : 0;
  if (row_ctas + cls_ctas == 0) return SE_OK;
  // 128-bit accesses when every row of every operand starts on a 16-byte boundary
  const uintptr_t a = reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(cent) |
                      reinterpret_cast<uintptr_t>(d_z) | reinterpret_cast<uintptr_t>(d_cent);
  const bool vec = (a & 15) == 0 && (ldz & 3) == 0 && (ldc & 3) == 0;
  launch(center_loss_kernel, dim3(row_ctas + cls_ctas), dim3(CL_WARPS * 32), 0, as_stream(stream), z, ldz,
         (const int*)labels, cent, ldc, B, C, D, scale, loss, d_z, d_cent, row_ctas, vec);
  return check_launch("center_loss_kernel");
}
