// All-pairs distance matrix of evaluate_retrieval.py:56-63.
//   normalize: F /= ||F|| (line 58) ; pdist = -F F^T (line 59)
//   else     : sq = sum F^2 (line 61) ; pdist = sq[:,None] + sq[None,:] - 2 F F^T (line 62)
// Algorithmic traffic 4*N*D bytes read + 4*N^2 bytes written => HBM-write bound by construction
// (SURVEY.md section 8d); the contraction must therefore be cheap enough to hide behind the
// output stream.  Two arithmetic modes share the prep kernel below:
//   SE_MODE_F32  : fp32 FFMA tiles (this file) -- exact-fp32 parity mode
//   SE_MODE_TF32 : wgmma split-fp16 x3 (pairwise_tc.cu) -- tensor-pipe fast mode
#include "common.cuh"

namespace se {

// workspace layout (floats): [0,N) squared norms of the (optionally normalised) rows,
// [N,2N) row norms (1 when normalize=0), then (TF32 mode) the split operands.
__global__ void __launch_bounds__(256)
pairwise_prep_kernel(const float* __restrict__ F, int ldF, int N, int D, int normalize, float* __restrict__ sq,
                     float* __restrict__ invn) {
  pdl_grid_sync();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N) return;
  const float* r = F + (long long)warp * ldF;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) { float v = r[i]; s = fmaf(v, v, s); }
  s = warp_sum(s);
  float inv = 1.f;
  if (normalize) {
    inv = sqrtf(s);                   // np.linalg.norm; rows are DIVIDED by it (line 58)
    float s2 = 0.f;
    for (int i = lane; i < D; i += 32) { float v = r[i] / inv; s2 = fmaf(v, v, s2); }
    s = warp_sum(s2);
  }
  if (lane == 0) { sq[warp] = s; invn[warp] = inv; }
}

template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
pairwise_f32_kernel(const float* __restrict__ F, int ldF, int N, int D, int row0, int rows, int pmode,
                    const float* __restrict__ sq, const float* __restrict__ invn, float* __restrict__ out,
                    long long ldout) {
  pdl_grid_sync();
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int CG = BN / TN;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tn = tid % CG, tm = tid / CG;
  const int i0 = row0 + blockIdx.y * BM;  // query rows
  const int j0 = blockIdx.x * BN;         // database columns
  const int iend = row0 + rows;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < D; k0 += BK) {
    for (int idx = tid; idx < BM * BK; idx += NT) {
      int r = idx / BK, k = idx % BK;
      float v = 0.f;
      if (i0 + r < iend && k0 + k < D) v = F[(long long)(i0 + r) * ldF + k0 + k] / invn[i0 + r];
      As[k][r] = v;
    }
    for (int idx = tid; idx < BN * BK; idx += NT) {
      int r = idx / BK, k = idx % BK;
      float v = 0.f;
      if (j0 + r < N && k0 + k < D) v = F[(long long)(j0 + r) * ldF + k0 + k] / invn[j0 + r];
      Bs[k][r] = v;
    }
    __syncthreads();
    tile_fma<BM, BN, TM, TN>(As, Bs, tm, tn, acc);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int gi = i0 + tm * TM + i;
    if (gi >= iend) continue;
    float a = sq[gi];
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int gj = j0 + tn * TN + j;
      if (gj >= N) continue;
      float c = acc[i][j];
      float v = (pmode == SE_PDIST_NEGDOT) ? -c : (a + sq[gj]) - 2.f * c;
      out[(long long)(gi - row0) * ldout + gj] = v;
    }
  }
}

int pairwise_tc(const float* F, int ldF, int N, int D, int row0, int rows, int pmode, int normalize, float* out,
                long long ldout, float* ws, cudaStream_t st);  // pairwise_tc.cu
long long pairwise_tc_workspace_floats(int N, int D);
long long pairwise_topk_extra_bytes(int N, int D, int rows);
int pairwise_tc_topk(const float* F, int ldF, int N, int D, int row0, int rows, int pmode, int k, int* out_idx, float* out_val,
                     int ldo, float* ws, int* status, cudaStream_t st);

}  // namespace se

using namespace se;

extern "C" int64_t se_pairwise_workspace_bytes(int N, int D, int mode) {
  long long f = 2LL * N;
  if (mode != SE_MODE_F32) f += pairwise_tc_workspace_floats(N, D);
  return (f + 64) * (long long)sizeof(float);
}

extern "C" int se_pairwise_dist(const float* F, int ldF, int N, int D, int row0, int rows, int pdist_mode,
                                int normalize, float* out, int64_t ldout, void* workspace, int mode, void* stream) {
  SE_REQUIRE(F && out && workspace, "null pointer");
  SE_REQUIRE(N > 0 && D > 0 && ldF >= D && row0 >= 0 && rows > 0 && row0 + rows <= N && ldout >= N, "bad shape");
  SE_REQUIRE(pdist_mode == SE_PDIST_SQEUCLID || pdist_mode == SE_PDIST_NEGDOT, "unknown pairwise mode");
  cudaStream_t st = as_stream(stream);
  float* ws = reinterpret_cast<float*>(workspace);
  float* sq = ws;
  float* invn = ws + N;
  launch(pairwise_prep_kernel, dim3(ceil_div(N, 8)), dim3(256), 0, st, F, ldF, N, D, normalize, sq, invn);
  int rc = check_launch("pairwise_prep_kernel");
  if (rc) return rc;
  if (mode != SE_MODE_F32) {   // SE_MODE_TF32 and SE_MODE_TF32X3: the tensor path is the error-compensated split-fp16 kernel
    rc = pairwise_tc(F, ldF, N, D, row0, rows, pdist_mode, normalize, out, ldout, ws, st);
    if (rc != SE_ERR_UNSUPPORTED) return rc;   // shapes the tensor path does not cover use the fp32 tiles
  }
  constexpr int BM = 64, BN = 64;
  dim3 grid(ceil_div(N, BN), ceil_div(rows, BM));
  launch(pairwise_f32_kernel<BM, BN, 4, 4>, dim3(grid), dim3(256), 0, st, F, ldF, N, D, row0, rows, pdist_mode, sq, invn, out, ldout);
  return check_launch("pairwise_f32_kernel");
}

extern "C" int64_t se_pairwise_topk_workspace_bytes(int N, int D, int rows) {
  return se_pairwise_workspace_bytes(N, D, SE_MODE_TF32X3) + pairwise_topk_extra_bytes(N, D, rows) + 8192;
}

extern "C" int se_pairwise_topk(const float* F, int ldF, int N, int D, int row0, int rows, int pdist_mode, int normalize, int k,
                                int32_t* out_idx, float* out_val, int ldo, void* workspace, int32_t* status, void* stream) {
  SE_REQUIRE(F && out_idx && workspace && status, "null pointer");
  SE_REQUIRE(N > 0 && D > 0 && ldF >= D && row0 >= 0 && rows > 0 && row0 + rows <= N && k > 0 && ldo >= k, "bad shape");
  SE_REQUIRE(pdist_mode == SE_PDIST_SQEUCLID || pdist_mode == SE_PDIST_NEGDOT, "unknown pairwise mode");
  cudaStream_t st = as_stream(stream);
  float* ws = reinterpret_cast<float*>(workspace);
  launch(pairwise_prep_kernel, dim3(ceil_div(N, 8)), dim3(256), 0, st, F, ldF, N, D, normalize, ws, ws + N);
  int rc = check_launch("pairwise_prep_kernel");
  if (rc) return rc;
  return pairwise_tc_topk(F, ldF, N, D, row0, rows, pdist_mode, k, out_idx, out_val, ldo, ws, status, st);
}
