// Shared helpers of the se_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <utility>

#include "../../include/se_b200.h"

namespace se {

void set_error(const char* fmt, ...);
int bn_bwd(const float* x, const float* y, const float* dout, int64_t rows, int C, const float* gamma, const float* save_mean,
           const float* save_invstd, int relu, int relu_in, float* dx, float beta_dx, float* dres, float beta_res, float* dgamma,
           float* dbeta, double* scratch, int early, void* stream);
void count_launch(int n = 1);
int sm_count();
// weight gradients without atomics (conv_wgrad_tc.cu): split-K partial sums go to slices of a workspace of the library
// (one per device and stream) and wgrad_reduce adds the slices into dW / dbias in slice order, so the result is the same
// on every run.  Slice k holds [T = kh*kw*Cin*Cout] dW partials at ws + k*T; the bias partials follow all slices,
// [splits][Cout].  wgrad_workspace sets *ws = nullptr when `floats` do not fit (or the stream first appears inside a graph
// capture): the kernels then add their partial sums into dW / dbias with atomics ("direct mode").
int wgrad_workspace(long long floats, cudaStream_t st, float** ws);
long long wgrad_fit_splits(long long want, long long T, int Cout);   // split count whose slices fit (want if none fit)
int wgrad_reduce(const float* ws, int splits, long long T, int Cout, float* dw, float* dbias, cudaStream_t st);

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return SE_ERR_CUDA;
  }
  count_launch();
  return SE_OK;
}

#define SE_REQUIRE(cond, msg)                                \
  do {                                                       \
    if (!(cond)) {                                           \
      se::set_error("%s: requirement failed: %s", __func__, msg); \
      return SE_ERR_ARG;                                     \
    }                                                        \
  } while (0)

// Programmatic dependent launch (PDL).  Every kernel of this library is launched with the
// programmatic-stream-serialization attribute and starts with pdl_grid_sync(): the dependent grid may become resident
// (barrier init, descriptor prefetch) while the preceding grid drains, and it blocks in
// griddepcontrol.wait -- which returns only when ALL prerequisite grids have completed and flushed their writes --
// before it touches global memory.  Invariant that keeps this safe at any chain depth: no kernel reads or writes
// global memory before its griddepcontrol.wait.  SE_NO_PDL=1 turns the attribute off (kernels then serialise fully).
// One documented exception: bn_bwd_reg_kernel with its `early` hint READS (never writes) x, y and the saved statistics
// before the wait.  That is safe only because those tensors were produced by the forward pass and the backward plan
// starts with a cudaMemsetAsync of the gradient buffer -- a full stream dependency that drains every forward kernel;
// Engine._build_plans asserts that memset when it sets the hint (removing it would turn the prefetch into a race).
bool pdl_enabled();
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_grid_sync() { pdl_trigger(); pdl_wait(); }

template <typename... KArgs, typename... Args>
inline void launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);   // errors surface through check_launch()
}

// Kernels with a grid-wide barrier (bn.cu): SE_BN_COOP=1 launches them with the cooperative attribute -- the runtime then
// guarantees that all CTAs are co-resident (or fails the launch) instead of relying on "grid <= #SMs and nothing else
// holds the SMs".  Cooperative launches cannot be programmatic dependents, so the PDL attribute is dropped for them.
bool coop_enabled();
template <typename... KArgs, typename... Args>
inline void launch_grid_barrier(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  if (!coop_enabled()) { launch(kern, grid, block, smem, st, std::forward<Args>(args)...); return; }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeCooperative;
  attr.val.cooperative = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

template <typename T>
__host__ __device__ inline T ceil_div(T a, T b) { return (a + b - 1) / b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// 128-bit streaming load/store (read-once / write-once data: keep L1 for reused tiles)
__device__ __forceinline__ float4 ldg_nc_f4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

constexpr int BK = 16;

// One BK-deep rank update of the TMxTN register tile from the smem tiles.
template <int BM, int BN, int TM, int TN>
__device__ __forceinline__ void tile_fma(const float (*As)[BM + 4], const float (*Bs)[BN + 4], int tm, int tn,
                                         float (&acc)[TM][TN]) {
#pragma unroll
  for (int k = 0; k < BK; ++k) {
    float a[TM], b[TN];
#pragma unroll
    for (int i = 0; i < TM; ++i) a[i] = As[k][tm * TM + i];
#pragma unroll
    for (int j = 0; j < TN; ++j) b[j] = Bs[k][tn * TN + j];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
  }
}


}  // namespace se
