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

// rows [row0, row0+rows) of the queries F against the N database items X (X == F for the all-pairs matrix)
template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
pairwise_f32_kernel(const float* __restrict__ F, int ldF, const float* __restrict__ X, int ldX, int N, int D, int row0,
                    int rows, int pmode, const float* __restrict__ sq, const float* __restrict__ invn,
                    const float* __restrict__ sq_x, const float* __restrict__ invn_x, float* __restrict__ out,
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
      if (j0 + r < N && k0 + k < D) v = X[(long long)(j0 + r) * ldX + k0 + k] / invn_x[j0 + r];
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
      float v = (pmode == SE_PDIST_NEGDOT) ? -c : (a + sq_x[gj]) - 2.f * c;
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
int pairwise_tc_cross(const float* Q, int ldQ, int Nq, const float* X, int ldX, int Nd, int D, int row0, int rows, int pmode,
                      float* out, long long ldout, float* ws_q, float* ws_x, cudaStream_t st);
long long cross_topk_extra_bytes(int Nd, int D, int rows);
int pairwise_tc_cross_topk(const float* Q, int ldQ, int Nq, const float* X, int ldX, int Nd, int D, int row0, int rows,
                           int pmode, int k, int* out_idx, float* out_val, int ldo, float* ws_q, float* ws_x, void* extra,
                           int* status, cudaStream_t st);

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
  launch(pairwise_f32_kernel<BM, BN, 4, 4>, dim3(grid), dim3(256), 0, st, F, ldF, F, ldF, N, D, row0, rows, pdist_mode, sq, invn,
         sq, invn, out, ldout);
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

// Two feature sets share one workspace: the queries' region (the all-pairs layout for Nq items), then the database's
// region (the same layout for Nd items) at the next 256-byte boundary, then (se_cross_topk) the fused path's own part.
static int64_t cross_region_bytes(int N, int D, int mode) { return (se_pairwise_workspace_bytes(N, D, mode) + 255) & ~255LL; }
static float* cross_ws_x(void* ws, int Nq, int D, int mode) {
  return reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + cross_region_bytes(Nq, D, mode));
}

extern "C" int64_t se_cross_workspace_bytes(int Nq, int Nd, int D, int mode) {
  return cross_region_bytes(Nq, D, mode) + cross_region_bytes(Nd, D, mode);
}

// row norms (and, with normalize, the normalised squared norms) of both sets into their regions
static int cross_prep(const float* Q, int ldQ, int Nq, const float* X, int ldX, int Nd, int D, int normalize, float* wq,
                      float* wx, cudaStream_t st) {
  launch(pairwise_prep_kernel, dim3(ceil_div(Nq, 8)), dim3(256), 0, st, Q, ldQ, Nq, D, normalize, wq, wq + Nq);
  int rc = check_launch("pairwise_prep_kernel");
  if (rc) return rc;
  launch(pairwise_prep_kernel, dim3(ceil_div(Nd, 8)), dim3(256), 0, st, X, ldX, Nd, D, normalize, wx, wx + Nd);
  return check_launch("pairwise_prep_kernel");
}

extern "C" int se_cross_dist(const float* Q, int ldQ, int Nq, const float* X, int ldX, int Nd, int D, int row0, int rows,
                             int pdist_mode, int normalize, float* out, int64_t ldout, void* workspace, int mode, void* stream) {
  SE_REQUIRE(Q && X && out && workspace, "null pointer");
  SE_REQUIRE(Nq > 0 && Nd > 0 && D > 0 && ldQ >= D && ldX >= D && rows > 0 && ldout >= Nd, "bad shape");
  SE_REQUIRE(row0 >= 0 && (int64_t)row0 + rows <= Nq, "query rows outside [0, Nq)");
  SE_REQUIRE(pdist_mode == SE_PDIST_SQEUCLID || pdist_mode == SE_PDIST_NEGDOT, "unknown pairwise mode");
  cudaStream_t st = as_stream(stream);
  float* wq = reinterpret_cast<float*>(workspace);
  float* wx = cross_ws_x(workspace, Nq, D, mode);
  int rc = cross_prep(Q, ldQ, Nq, X, ldX, Nd, D, normalize, wq, wx, st);
  if (rc) return rc;
  if (mode != SE_MODE_F32) {
    rc = pairwise_tc_cross(Q, ldQ, Nq, X, ldX, Nd, D, row0, rows, pdist_mode, out, ldout, wq, wx, st);
    if (rc != SE_ERR_UNSUPPORTED) return rc;   // D > 128 (or unaligned output rows): the fp32 tiles
  }
  constexpr int BM = 64, BN = 64;
  dim3 grid(ceil_div(Nd, BN), ceil_div(rows, BM));
  launch(pairwise_f32_kernel<BM, BN, 4, 4>, dim3(grid), dim3(256), 0, st, Q, ldQ, X, ldX, Nd, D, row0, rows, pdist_mode, wq,
         wq + Nq, wx, wx + Nd, out, ldout);
  return check_launch("pairwise_f32_kernel");
}

extern "C" int64_t se_cross_topk_workspace_bytes(int Nq, int Nd, int D, int rows) {
  return se_cross_workspace_bytes(Nq, Nd, D, SE_MODE_TF32X3) + cross_topk_extra_bytes(Nd, D, rows) + 8192;
}

extern "C" int se_cross_topk(const float* Q, int ldQ, int Nq, const float* X, int ldX, int Nd, int D, int row0, int rows,
                             int pdist_mode, int normalize, int k, int32_t* out_idx, float* out_val, int ldo, void* workspace,
                             int32_t* status, void* stream) {
  SE_REQUIRE(Q && X && out_idx && workspace && status, "null pointer");
  SE_REQUIRE(Nq > 0 && Nd > 0 && D > 0 && ldQ >= D && ldX >= D && rows > 0 && k > 0 && ldo >= k, "bad shape");
  SE_REQUIRE(row0 >= 0 && (int64_t)row0 + rows <= Nq, "query rows outside [0, Nq)");
  SE_REQUIRE(pdist_mode == SE_PDIST_SQEUCLID || pdist_mode == SE_PDIST_NEGDOT, "unknown pairwise mode");
  if (D > 128 || k > 1024 || k > Nd) {
    set_error("se_cross_topk: D = %d, k = %d, Nd = %d outside the fused path (D <= 128, k <= min(1024, Nd))", D, k, Nd);
    return SE_ERR_UNSUPPORTED;
  }
  cudaStream_t st = as_stream(stream);
  float* wq = reinterpret_cast<float*>(workspace);
  float* wx = cross_ws_x(workspace, Nq, D, SE_MODE_TF32X3);
  void* extra = reinterpret_cast<uint8_t*>(workspace) + se_cross_workspace_bytes(Nq, Nd, D, SE_MODE_TF32X3);
  int rc = cross_prep(Q, ldQ, Nq, X, ldX, Nd, D, normalize, wq, wx, st);
  if (rc) return rc;
  return pairwise_tc_cross_topk(Q, ldQ, Nq, X, ldX, Nd, D, row0, rows, pdist_mode, k, out_idx, out_val, ldo, wq, wx, extra,
                                status, st);
}
