// Per-row ranking of the distance matrix: the k nearest database items of every query, ascending, ties by index
// -- the prefix of `np.argsort(pdist, axis=-1)` (evaluate_retrieval.py:67) that `hierarchical_precision(..., clip_ahp)`
// actually reads (class_hierarchy.py:242-244,273,283: the first kmax+1 ranks).  SURVEY.md §8(f) rank 1.
//
// One CTA per row, the row staged ONCE in shared memory as order-preserving uint32 keys (n <= 52 000 floats = 203 KB):
//   1. radix select of the k-th smallest key, 11 + 11 + 10 bits, three shared-memory histogram passes;
//   2. ordered compaction: thread t owns a contiguous index range, block scans give every selected element its slot, so
//      among equal keys the smallest indices win (stable-argsort semantics);
//   3. bitonic sort of the <= 1024 selected (key << 32 | index) words;
//   4. keys back to floats, indices and values out.
// HBM traffic = the row once (4n bytes) + 8k bytes out: the kernel is bound by the shared-memory passes, not by HBM
// (measured 11.9 ms for the top 251 of 50 000 x 50 000, 13 % of the read roof).  Tried and rejected: digits cut from
// (key - row minimum) below the highest bit of the row's range, to spread the histogram atomics -- the extra min/max and
// subtraction passes cost more than the contention they remove (13.5 ms).
#include <stdlib.h>

#include "common.cuh"

namespace se {

constexpr int TK_THREADS = 512;
constexpr int TK_MAXK = 1024;

__device__ __forceinline__ uint32_t f2key(float f) {
  if (f == 0.f) f = 0.f;                                  // -0.0 ties with +0.0 as in numpy
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);      // ascending floats <-> ascending unsigned keys (-0 < +0)
}
__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// exclusive scan of one int per thread over the CTA (512 threads); `total` gets the sum.  scratch: >= 17 ints
__device__ __forceinline__ int block_exscan(int v, int* scratch, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int n = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += n; }
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = (lane < TK_THREADS / 32) ? scratch[lane] : 0;
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int n = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += n; }
    if (lane < TK_THREADS / 32) scratch[lane] = winc - w;
    if (lane == 31) scratch[16] = winc;
  }
  __syncthreads();
  const int res = scratch[warp] + inc - v;
  *total = scratch[16];
  __syncthreads();
  return res;
}

// one radix-select pass: histogram of digit (key >> shift) & (bins-1) over keys whose higher bits equal `prefix`
// (prefix_shift = number of low bits below the prefix; 32 -> no prefix), then the bin holding the `want`-th smallest.
__device__ __forceinline__ void select_pass(const uint32_t* keys, int n, int* hist, int* scratch, int bins, int shift,
                                            uint32_t prefix, int prefix_shift, int* want, uint32_t* digit_out) {
  for (int i = threadIdx.x; i < bins; i += TK_THREADS) hist[i] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += TK_THREADS) {
    const uint32_t key = keys[i];
    if (prefix_shift >= 32 || (key >> prefix_shift) == prefix) atomicAdd(&hist[(key >> shift) & (bins - 1)], 1);
  }
  __syncthreads();
  // each thread owns bins / 512 consecutive bins (4 or 2)
  const int per = bins / TK_THREADS;
  int local = 0;
  for (int j = 0; j < per; ++j) local += hist[threadIdx.x * per + j];
  int total;
  const int before = block_exscan(local, scratch, &total);
  const int w = *want;                                   // same value in every thread
  if (w > before && w <= before + local) {               // the crossing is inside this thread's bins
    int acc = before;
    for (int j = 0; j < per; ++j) {
      const int c = hist[threadIdx.x * per + j];
      if (w <= acc + c) { scratch[20] = threadIdx.x * per + j; scratch[21] = w - acc; break; }
      acc += c;
    }
  }
  __syncthreads();
  *digit_out = (uint32_t)scratch[20];
  *want = scratch[21];
  __syncthreads();
}

__global__ void __launch_bounds__(TK_THREADS, 1)
row_topk_kernel(const float* __restrict__ dist, long long ld, int rows, int n, int k, float* __restrict__ out_val,
                int* __restrict__ out_idx, int ldo) {
  pdl_grid_sync();
  extern __shared__ __align__(16) uint32_t tsm[];
  uint32_t* keys = tsm;                                            // [n]
  int* hist = reinterpret_cast<int*>(keys + ((n + 3) & ~3));       // [2048]
  int* scratch = hist + 2048;                                      // [32]
  unsigned long long* sel = reinterpret_cast<unsigned long long*>(scratch + 32);   // [P], P = pow2 >= k
  int P = 1;
  while (P < k) P <<= 1;
  const int tid = threadIdx.x;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const float* src = dist + (long long)row * ld;
    __syncthreads();
    if ((ld & 3) == 0 && (reinterpret_cast<uintptr_t>(dist) & 15) == 0) {
      const int n4 = n >> 2;
      for (int i = tid; i < n4; i += TK_THREADS) {
        const float4 v = ldg_nc_f4(src + 4 * i);
        keys[4 * i] = f2key(v.x); keys[4 * i + 1] = f2key(v.y); keys[4 * i + 2] = f2key(v.z); keys[4 * i + 3] = f2key(v.w);
      }
      for (int i = 4 * n4 + tid; i < n; i += TK_THREADS) keys[i] = f2key(src[i]);
    } else {
      for (int i = tid; i < n; i += TK_THREADS) keys[i] = f2key(src[i]);
    }
    __syncthreads();
    // ---- 1. threshold = k-th smallest key
    int want = k;
    uint32_t d1, d2, d3;
    select_pass(keys, n, hist, scratch, 2048, 21, 0u, 32, &want, &d1);
    select_pass(keys, n, hist, scratch, 2048, 10, d1, 21, &want, &d2);
    const uint32_t p2 = (d1 << 11) | d2;
    select_pass(keys, n, hist, scratch, 1024, 0, p2, 10, &want, &d3);
    const uint32_t T = (p2 << 10) | d3;
    const int need_eq = want;                      // how many keys equal to T are taken (smallest indices first)
    // ---- 2. ordered compaction
    const int chunk = (n + TK_THREADS - 1) / TK_THREADS;
    const int i0 = min(n, tid * chunk), i1 = min(n, i0 + chunk);
    int nl = 0, ne = 0;
    for (int i = i0; i < i1; ++i) { const uint32_t key = keys[i]; nl += key < T; ne += key == T; }
    int tot_l, tot_e;
    int off_l = block_exscan(nl, scratch, &tot_l);
    int off_e = block_exscan(ne, scratch, &tot_e);
    for (int i = tid; i < P; i += TK_THREADS) sel[i] = ~0ull;      // padding sorts to the end
    __syncthreads();
    for (int i = i0; i < i1; ++i) {
      const uint32_t key = keys[i];
      if (key < T) sel[off_l++] = ((unsigned long long)key << 32) | (unsigned)i;
      else if (key == T) { if (off_e < need_eq) sel[tot_l + off_e] = ((unsigned long long)key << 32) | (unsigned)i; ++off_e; }
    }
    __syncthreads();
    // ---- 3. bitonic sort of P 64-bit words
    for (int size = 2; size <= P; size <<= 1) {
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int t = tid; t < (P >> 1); t += TK_THREADS) {
          const int lo = ((t / stride) * (stride << 1)) + (t % stride), hi = lo + stride;
          const bool up = ((lo & size) == 0);
          const unsigned long long a = sel[lo], b = sel[hi];
          if ((a > b) == up) { sel[lo] = b; sel[hi] = a; }
        }
        __syncthreads();
      }
    }
    // ---- 4. output
    for (int i = tid; i < k; i += TK_THREADS) {
      const unsigned long long w = sel[i];
      out_idx[(long long)row * ldo + i] = (int)(w & 0xFFFFFFFFu);
      if (out_val) out_val[(long long)row * ldo + i] = key2f((uint32_t)(w >> 32));
    }
  }
}

int init_row_topk() {
  if (cudaFuncSetAttribute(row_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess) {
    set_error("init_row_topk: cannot raise the shared-memory limit");
    return SE_ERR_CUDA;
  }
  return SE_OK;
}

}  // namespace se

using namespace se;

extern "C" int se_row_topk(const float* dist, int64_t ld, int rows, int n, int k, float* out_val, int32_t* out_idx,
                           int ldo, void* stream) {
  SE_REQUIRE(dist && out_idx && rows > 0 && n > 0 && k > 0, "bad arguments");
  SE_REQUIRE(k <= n && ldo >= k && ld >= n, "k, ldo or ld out of range");
  if (k > TK_MAXK) { set_error("se_row_topk: k = %d exceeds %d", k, TK_MAXK); return SE_ERR_UNSUPPORTED; }
  int P = 1;
  while (P < k) P <<= 1;
  const size_t smem = (size_t)((n + 3) & ~3) * 4 + 2048 * 4 + 32 * 4 + (size_t)P * 8;
  if (smem > 227 * 1024) {
    set_error("se_row_topk: a row of %d values does not fit in shared memory (max ~52000)", n);
    return SE_ERR_UNSUPPORTED;
  }
  const int rc = ensure_setup();
  if (rc) return rc;
  const int grid = min(rows, sm_count());
  launch(row_topk_kernel, dim3(grid), dim3(TK_THREADS), smem, as_stream(stream), dist, (long long)ld, rows, n, k, out_val, out_idx, ldo);
  return check_launch("row_topk_kernel");
}
