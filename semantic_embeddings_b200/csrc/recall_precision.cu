// Where a query's relevant items land in its ranking (plot_recall_precision.py:59-77 of the reference needs nothing else):
// for query q = q0 + i of a distance block, the 1-based positions of the other members of q's class in the ranking of
// row i with q removed -- ascending distance, ties by ascending index, -0.0 == +0.0, i.e. the order of se_row_argsort --
// without ordering the other items.
//
// One CTA per query row.  The members' (distance, index) words are staged in shared memory in chunks of RP_CHUNK and
// sorted there.  One sweep over the row binary-searches every other item into the chunk and counts it in a histogram of
// insertion slots; a chunk member lands in its own slot, so the inclusive scan of the histogram is each member's
// position.  A second, short sweep over the members alone gives each one's rank among the members (the output order).
// Items behind the chunk's last member are not counted (nothing reads that slot), which also keeps the bulk of a row
// away from a single shared-memory counter.  Integer atomics only: reruns give the same output.
#include "common.cuh"

namespace se {

constexpr int RP_THREADS = 256;
constexpr int RP_CHUNK = 2048;                 // members per shared-memory chunk (16 KB of words)
constexpr int RP_UNROLL = 4;                   // independent binary searches in flight per thread

// Class index: CTA c < C writes offsets[c] = #labels in [0, c) and the items of class c in ascending index order to
// members[offsets[c] ...]; CTA C writes offsets[C] = #labels in [0, C), which equals N only when every label is valid.
__global__ void __launch_bounds__(RP_THREADS)
class_index_kernel(const int32_t* __restrict__ labels, int N, int C, int32_t* __restrict__ offsets,
                   int32_t* __restrict__ members) {
  pdl_grid_sync();
  __shared__ int warp_tot[RP_THREADS / 32];
  __shared__ int total;
  const int c = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int below = 0;
  for (int i = threadIdx.x; i < N; i += RP_THREADS) {
    const int y = labels[i];
    below += (y >= 0 && y < c);
  }
  below = __reduce_add_sync(0xffffffffu, below);
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  if (lane == 0) atomicAdd(&total, below);
  __syncthreads();
  const int base = total;
  if (threadIdx.x == 0) offsets[c] = base;
  if (c == C) return;
  int written = 0;
  for (int i0 = 0; i0 < N; i0 += RP_THREADS) {           // order-preserving compaction, one tile of labels at a time
    const int i = i0 + threadIdx.x;
    const bool hit = i < N && labels[i] == c;
    const unsigned ballot = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) warp_tot[warp] = __popc(ballot);
    __syncthreads();
    int before = written;
    for (int w = 0; w < warp; ++w) before += warp_tot[w];
    if (hit) members[base + before + __popc(ballot & ((1u << lane) - 1u))] = i;
    for (int w = 0; w < RP_THREADS / 32; ++w) written += warp_tot[w];
    __syncthreads();
  }
}

// In-place inclusive scan of a[0, m), m <= RP_CHUNK: RP_CHUNK / RP_THREADS consecutive entries per thread.
__device__ __forceinline__ void block_inclusive_scan(int* a, int m, int* warp_tot) {
  constexpr int PER = RP_CHUNK / RP_THREADS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, t0 = threadIdx.x * PER;
  int v[PER], s = 0;
#pragma unroll
  for (int u = 0; u < PER; ++u) {
    v[u] = t0 + u < m ? a[t0 + u] : 0;
    s += v[u];
  }
  int incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  int run = incl - s;
  for (int w = 0; w < warp; ++w) run += warp_tot[w];
#pragma unroll
  for (int u = 0; u < PER; ++u) {
    run += v[u];
    if (t0 + u < m) a[t0 + u] = run;
  }
  __syncthreads();
}

// the item's (distance, index) word: ascending words = ranking order
__device__ __forceinline__ unsigned long long rank_word(const float* row, int j) {
  return ((unsigned long long)as_key(row[j]) << 32) | (unsigned)j;
}

// number of words of the sorted chunk s[0, P) (P a power of two, padded with ~0) below x
__device__ __forceinline__ int slot_of(const unsigned long long* s, int P, unsigned long long x) {
  int pos = 0;
  for (int step = P >> 1; step > 0; step >>= 1)
    if (s[pos + step - 1] < x) pos += step;
  return pos + (s[pos] < x);
}

__global__ void __launch_bounds__(RP_THREADS, 4)    // 4 CTAs per SM: 128 KB of shared memory, 56 registers, no spills
relevant_positions_kernel(const float* __restrict__ dist, long long ld, int rows, int n, int q0,
                          const int32_t* __restrict__ query_labels, const int32_t* __restrict__ labels, int C,
                          const int32_t* __restrict__ offsets, const int32_t* __restrict__ members,
                          const int64_t* __restrict__ out_offsets, int32_t* __restrict__ out) {
  pdl_grid_sync();
  __shared__ unsigned long long s[RP_CHUNK];
  __shared__ int pos[RP_CHUNK];                // slot histogram -> positions
  __shared__ int rnk[RP_CHUNK];                // member histogram -> ranks among the members
  __shared__ int warp_tot[RP_THREADS / 32];
  // with query_labels (se_relevant_positions_q) the query is no database item: q = -1 removes nothing
  const int i = blockIdx.x, q = query_labels ? -1 : q0 + i;
  const int c = query_labels ? query_labels[i] : labels[q];
  if (c < 0 || c >= C) return;                 // se_class_index has rejected such labels
  const float* row = dist + (long long)i * ld;
  const int32_t* mem = members + offsets[c];
  const int nrel = offsets[c + 1] - offsets[c] - (q >= 0 ? 1 : 0);
  int32_t* o = out + out_offsets[i];
  int qpos = q >= 0 ? 0 : nrel;                // q's place in its class list (ascending indices)
  for (int lo = 0, hi = q >= 0 ? nrel : -1; lo <= hi;) {
    const int mid = (lo + hi) >> 1;
    if (mem[mid] < q) lo = mid + 1; else if (mem[mid] > q) hi = mid - 1; else { qpos = mid; break; }
  }
  for (int c0 = 0; c0 < nrel; c0 += RP_CHUNK) {
    const int m = min(RP_CHUNK, nrel - c0);
    int P = 1;
    while (P < m) P <<= 1;
    for (int t = threadIdx.x; t < P; t += RP_THREADS) {
      if (t < m) {
        const int u = c0 + t;
        s[t] = rank_word(row, mem[u + (u >= qpos)]);
        pos[t] = 0;
        rnk[t] = 0;
      } else {
        s[t] = ~0ull;
      }
    }
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1) {         // bitonic sort of the chunk
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int t = threadIdx.x; t < P / 2; t += RP_THREADS) {
          const int a = ((t & ~(j - 1)) << 1) | (t & (j - 1)), b = a | j;
          const bool up = (a & k) == 0;
          const unsigned long long x = s[a], y = s[b];
          if ((x > y) == up) { s[a] = y; s[b] = x; }
        }
        __syncthreads();
      }
    }
    // sweep the row: slot of every item j != q (q and the tail get ~0, which lands in slot m and is not counted)
    int first = 0;                             // items in slot 0, counted in a register
    for (int j0 = 0; j0 < n; j0 += RP_UNROLL * RP_THREADS) {
      unsigned long long x[RP_UNROLL];
      int sl[RP_UNROLL];
#pragma unroll
      for (int u = 0; u < RP_UNROLL; ++u) {
        const int j = j0 + u * RP_THREADS + threadIdx.x;
        x[u] = (j < n && j != q) ? rank_word(row, j) : ~0ull;
        sl[u] = 0;
      }
      for (int step = P >> 1; step > 0; step >>= 1) {
#pragma unroll
        for (int u = 0; u < RP_UNROLL; ++u)
          if (s[sl[u] + step - 1] < x[u]) sl[u] += step;
      }
#pragma unroll
      for (int u = 0; u < RP_UNROLL; ++u) {
        sl[u] += s[sl[u]] < x[u];
        if (sl[u] == 0) ++first;
        else if (sl[u] < m) atomicAdd(&pos[sl[u]], 1);
      }
    }
    // every member (q excluded) into the chunk: ranks among the members
    for (int u = threadIdx.x; u < nrel; u += RP_THREADS) {
      const int sl = slot_of(s, P, rank_word(row, mem[u + (u >= qpos)]));
      if (sl < m) atomicAdd(&rnk[sl], 1);
    }
    first = __reduce_add_sync(0xffffffffu, first);
    if ((threadIdx.x & 31) == 0 && first) atomicAdd(&pos[0], first);
    __syncthreads();
    block_inclusive_scan(pos, m, warp_tot);
    block_inclusive_scan(rnk, m, warp_tot);
    for (int t = threadIdx.x; t < m; t += RP_THREADS) o[rnk[t] - 1] = pos[t];
    __syncthreads();
  }
}

}  // namespace se

using namespace se;

extern "C" int se_class_index(const int32_t* labels, int N, int C, int32_t* offsets, int32_t* members, void* stream) {
  SE_REQUIRE(labels && offsets && members, "null pointer");
  SE_REQUIRE(N > 0 && C > 0, "bad sizes");
  cudaStream_t st = as_stream(stream);
  launch(class_index_kernel, dim3(C + 1), dim3(RP_THREADS), 0, st, labels, N, C, offsets, members);
  int rc = check_launch("class_index_kernel");
  if (rc != SE_OK) return rc;
  int32_t valid = -1;
  cudaError_t e = cudaMemcpyAsync(&valid, offsets + C, sizeof(valid), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    set_error("se_class_index: %s", cudaGetErrorString(e));
    return SE_ERR_CUDA;
  }
  SE_REQUIRE(valid == N, "labels outside [0, C)");
  return SE_OK;
}

extern "C" int se_relevant_positions(const float* dist, int64_t ld, int rows, int n, int q0, const int32_t* labels, int C,
                                     const int32_t* offsets, const int32_t* members, const int64_t* out_offsets,
                                     int32_t* out, void* stream) {
  SE_REQUIRE(dist && labels && offsets && members && out_offsets && out, "null pointer");
  SE_REQUIRE(rows >= 0 && n >= 0 && q0 >= 0 && C > 0 && ld >= n, "bad sizes");
  SE_REQUIRE((int64_t)q0 + rows <= n, "query rows outside the database");
  if (rows == 0) return SE_OK;
  launch(relevant_positions_kernel, dim3(rows), dim3(RP_THREADS), 0, as_stream(stream), dist, (long long)ld, rows, n, q0,
         (const int32_t*)nullptr, labels, C, offsets, members, out_offsets, out);
  return check_launch("relevant_positions_kernel");
}

extern "C" int se_relevant_positions_q(const float* dist, int64_t ld, int rows, int n, const int32_t* query_labels,
                                       const int32_t* labels, int C, const int32_t* offsets, const int32_t* members,
                                       const int64_t* out_offsets, int32_t* out, void* stream) {
  SE_REQUIRE(dist && query_labels && labels && offsets && members && out_offsets && out, "null pointer");
  SE_REQUIRE(rows >= 0 && n >= 0 && C > 0 && ld >= n, "bad sizes");
  if (rows == 0) return SE_OK;
  launch(relevant_positions_kernel, dim3(rows), dim3(RP_THREADS), 0, as_stream(stream), dist, (long long)ld, rows, n, 0,
         query_labels, labels, C, offsets, members, out_offsets, out);
  return check_launch("relevant_positions_kernel");
}
