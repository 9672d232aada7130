// Full-length per-row ranking of the distance matrix: `np.argsort(pdist, axis=-1)` (evaluate_retrieval.py:67) with the
// order defined by the build (ascending distance, ties by ascending index = np.argsort(kind='stable'); -0.0 == +0.0).
// Needed by the metrics that read the whole list: classical AP and the unclipped AHP (class_hierarchy.py:303-316).
//
// One CTA per row sorts 64-bit words (order-preserving key << 32 | column index) with a bitonic network whose
// sub-networks of <= 4096 words run in shared memory:
//   1. every chunk of 4096 words is loaded from the distance row (padding = 0xFFFF..), sorted completely in shared
//      memory (78 compare-exchange steps) and written to the row's scratch buffer in global memory (L2 resident);
//   2. for every larger merge level, the steps with a stride >= 4096 are passes over the scratch buffer, the remaining
//      12 steps of each chunk run in shared memory again.
// N = 50 000 (padded to 65 536): 4 levels above the chunk size -> 10 global passes + 5 shared-memory rounds per row.
// No atomics, no data-dependent control flow: the result is deterministic and identical to a stable argsort.
#include "common.cuh"

namespace se {

constexpr int AS_THREADS = 1024;
constexpr int AS_CHUNK = 4096;                 // words per shared-memory sub-sort (32 KB)

// compare-exchange steps j = j_hi, j_hi/2, ..., 1 of merge level k on a chunk held in shared memory.
// `base` = global index of the chunk's first word (direction of a pair depends on the global index)
__device__ __forceinline__ void smem_steps(unsigned long long* s, int base, int k, int j_hi) {
  for (int j = j_hi; j >= 1; j >>= 1) {
    for (int t = threadIdx.x; t < AS_CHUNK / 2; t += AS_THREADS) {
      const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));      // lower index of the pair
      const int p = i | j;
      const bool up = (((base + i) & k) == 0);                  // ascending block?
      const unsigned long long a = s[i], b = s[p];
      if ((a > b) == up) { s[i] = b; s[p] = a; }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(AS_THREADS)
row_argsort_kernel(const float* __restrict__ dist, long long ld, int n, int npad, unsigned long long* __restrict__ scratch,
                   int* __restrict__ out_idx, long long ldo) {
  pdl_grid_sync();
  __shared__ unsigned long long s[AS_CHUNK];
  const float* row = dist + (long long)blockIdx.x * ld;
  unsigned long long* w = scratch + (long long)blockIdx.x * npad;
  const int nchunks = npad / AS_CHUNK;
  // ---- 1. chunk sorts (levels k = 2 .. AS_CHUNK), directions as in the full network
  for (int c = 0; c < nchunks; ++c) {
    const int base = c * AS_CHUNK;
    for (int t = threadIdx.x; t < AS_CHUNK; t += AS_THREADS) {
      const int i = base + t;
      s[t] = i < n ? (((unsigned long long)as_key(row[i]) << 32) | (unsigned)i) : ~0ull;
    }
    __syncthreads();
    for (int k = 2; k <= AS_CHUNK; k <<= 1) smem_steps(s, base, k, k >> 1);
    for (int t = threadIdx.x; t < AS_CHUNK; t += AS_THREADS) w[base + t] = s[t];
    __syncthreads();
  }
  // ---- 2. merge levels above the chunk size
  for (int k = 2 * AS_CHUNK; k <= npad; k <<= 1) {
    for (int j = k >> 1; j >= AS_CHUNK; j >>= 1) {
      for (int t = threadIdx.x; t < npad / 2; t += AS_THREADS) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int p = i | j;
        const bool up = ((i & k) == 0);
        const unsigned long long a = w[i], b = w[p];
        if ((a > b) == up) { w[i] = b; w[p] = a; }
      }
      __syncthreads();                         // global writes of this CTA -> visible to its own threads
    }
    for (int c = 0; c < nchunks; ++c) {
      const int base = c * AS_CHUNK;
      for (int t = threadIdx.x; t < AS_CHUNK; t += AS_THREADS) s[t] = w[base + t];
      __syncthreads();
      smem_steps(s, base, k, AS_CHUNK >> 1);
      if (k == npad) {                         // last level: the chunk is final -> indices out
        for (int t = threadIdx.x; t < AS_CHUNK; t += AS_THREADS)
          if (base + t < n) out_idx[(long long)blockIdx.x * ldo + base + t] = (int)(unsigned)(s[t] & 0xFFFFFFFFull);
      } else {
        for (int t = threadIdx.x; t < AS_CHUNK; t += AS_THREADS) w[base + t] = s[t];
      }
      __syncthreads();
    }
  }
  if (npad == AS_CHUNK) {                      // a single chunk: already sorted by step 1
    for (int t = threadIdx.x; t < n; t += AS_THREADS) out_idx[(long long)blockIdx.x * ldo + t] = (int)(unsigned)(w[t] & 0xFFFFFFFFull);
  }
}

}  // namespace se

using namespace se;

static int as_npad(int n) {
  int p = AS_CHUNK;
  while (p < n) p <<= 1;
  return p;
}

extern "C" int64_t se_row_argsort_workspace_bytes(int rows, int n) {
  if (rows <= 0 || n <= 0) return 0;
  return (int64_t)rows * as_npad(n) * 8;
}

extern "C" int se_row_argsort(const float* dist, int64_t ld, int rows, int n, int32_t* out_idx, int64_t ldo, void* workspace,
                              void* stream) {
  SE_REQUIRE(dist && out_idx && workspace && rows > 0 && n > 0 && ld >= n && ldo >= n, "bad arguments");
  SE_REQUIRE(n <= (1 << 24), "rows longer than 2^24 entries are not supported");
  launch(row_argsort_kernel, dim3(rows), dim3(AS_THREADS), 0, as_stream(stream), dist, (long long)ld, n, as_npad(n),
         reinterpret_cast<unsigned long long*>(workspace), out_idx, (long long)ldo);
  return check_launch("row_argsort_kernel");
}
