// All-pairs distance (evaluate_retrieval.py:56-63) on the tensor cores -- SE_MODE_TF32 / SE_MODE_TF32X3 path.
//
// Arithmetic: "split-fp16 x3".  After a global power-of-two scaling that brings max|f| <= 1, every fp32
// feature value f is split into h = fp16(f) and l = fp16(f - h) (11 + 11 significand bits, the low part
// may be subnormal: absolute error <= 2^-25).  The fp32 product sum is recovered from three fp16 tensor-core
// products accumulated in ONE fp32 accumulator:  F F^T ~= Fh Fh^T + Fh Fl^T + Fl Fh^T  (missing l*l term
// <= 2^-24).  fp16 wgmma moves 2 bytes per element and runs at twice the TF32 rate, which is what keeps the
// contraction hidden behind the fp32 output stream (4 bytes per pair -- the HBM roofline of this kernel).
//
// Two feature sets (se_cross_dist, se_cross_topk): the queries are A and the database is B, and each set gets its own
// power-of-two scaling 2^-e_q, 2^-e_x (the sets may differ in magnitude by orders); the epilogue undoes 2^(e_q + e_x),
// which is the 4^e of the all-pairs matrix when both sets are the same.
//
// Structure (one persistent CTA per SM, 384 threads, warp-specialised):
//   warpgroup 0 : one thread issues the TMA loads -- the A row block (128 rows, h and l, all K) stays RESIDENT while
//                 the CTA sweeps the column tiles; B tiles (128 rows) stream through a 2-stage ring, one 64-wide K
//                 block per stage
//   warpgroups 1, 2 : each owns 64 rows of the 128 x 128 tile: m64n128k16 wgmma into registers, then the accumulator
//                 goes through shared memory so that one thread holds one row of 32 columns at a time for the
//                 epilogue (norms / sign, then a coalesced streaming store, or the ranking passes of the fused top-k)
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc.cuh"

namespace se {

using namespace tc;

constexpr int PW_BM = 128, PW_BN = 128, PW_KB = 64;     // K block = 64 halfs = 128 bytes (SWIZZLE_128B row)
constexpr int PW_MAXKB = 2;                              // resident A: at most 2 K blocks (D <= 128)
constexpr int PW_STAGES = 2;
constexpr int PW_A_BYTES = PW_BM * 128;                  // one K block of A (h or l): 16 KB
constexpr int PW_B_BYTES = PW_BN * 128;                  // one K block of B (h or l): 16 KB
constexpr int PW_PITCH = PW_BN + 8;                      // accumulator staging row pitch (floats)
constexpr int PW_THREADS = 384;
constexpr int PW_SMEM = 2 * PW_MAXKB * PW_A_BYTES + PW_STAGES * 2 * PW_B_BYTES + PW_BM * PW_PITCH * 4 + 1024 /*align*/ + 256;

struct PwParams {
  int N, row0, rows, pmode, tiles_m, tiles_n, kblocks, ksteps_total;
  long long ldout;
  float* out;
  const float* sq;       // squared norms of the (normalised) query rows, [N]
  const float* sq_b;     // squared norms of the column items (== sq for the all-pairs matrix; a sample's norms otherwise)
  const float* scal;     // scal[1] = 2^(e_q + e_x): undoes the power-of-two input scaling
  // fused ranking (se_pairwise_topk).  EPI == 2, sample pass: every (row, 64-column half tile with >= 8 columns) adds the
  // j-th smallest of its distances to tau_sum[row] -- the mean of those order statistics is the row's candidate threshold.  EPI == 1,
  // sweep: entries below the threshold become (value, column) candidates in the region of the writing (row, column
  // half, part of the row block) -- a thread owns its row for the CTA's whole stretch of the row block, so the fill
  // count lives in a register and no atomics are needed.  Part = the CTA's place among the CTAs that share the row block
  // (regions: half * nparts + part).
  float* tau_sum;        // [rows]   EPI 2: accumulates; EPI 1: threshold = tau_sum[row] * tau_scale
  float tau_scale;       // 1 / (number of half tiles of the sample pass with >= 8 columns)
  int* cnt;              // [rows, 2 * nparts] candidates per region (may exceed capr: the finishing kernel reports it)
  float* cand_val;       // [rows, 2 * nparts, capr]
  int* cand_idx;         // [rows, 2 * nparts, capr]
  int capr, ncols;       // ncols: number of valid columns
  int nparts;            // EPI 1: the most CTAs that share one row block
  int jsel;              // EPI 2: which order statistic (0-based, < 8) of a half tile feeds the threshold
};

// ---- prep: fp32 features -> scaled fp16 (h, l) matrices with row pitch KW
__global__ void __launch_bounds__(256)
pairwise_absmax_kernel(const float* __restrict__ F, int ldF, int N, int D, const float* __restrict__ norms,
                       unsigned* __restrict__ absmax_bits) {
  pdl_grid_sync();
  float m = 0.f;
  const long long total = (long long)N * D;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    int r = (int)(e / D), k = (int)(e % D);
    m = fmaxf(m, fabsf(F[(long long)r * ldF + k] / norms[r]));
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0 && m > 0.f && m < 3.0e38f) atomicMax(absmax_bits, __float_as_uint(m));
}

__global__ void __launch_bounds__(256)
pairwise_split_kernel(const float* __restrict__ F, int ldF, int N, int D, int KW, const float* __restrict__ norms,
                      const float* scal, const float* scal_other, float* scale_out, __half* __restrict__ Fh,
                      __half* __restrict__ Fl) {
  pdl_grid_sync();
  // scal[0] / scal_other[0] hold the bit patterns of max|f| of this set / of the other operand's set (0 if all zero);
  // scale_out (may be NULL) receives 2^(e + e_other), the factor the epilogue multiplies the dot products by
  auto exponent = [](const float* sc) {
    const float amax = __uint_as_float(reinterpret_cast<const unsigned*>(sc)[0]);
    int e = 0;
    if (amax > 0.f) frexpf(amax, &e);          // amax = m * 2^e, m in [0.5, 1)  =>  amax * 2^-e < 1
    return e;
  };
  const int e = exponent(scal);
  const float s = ldexpf(1.f, -e);
  if (scale_out && blockIdx.x == 0 && threadIdx.x == 0) *scale_out = ldexpf(1.f, e + exponent(scal_other));
  const long long total = (long long)N * KW;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    int r = (int)(idx / KW), k = (int)(idx % KW);
    float v = 0.f;
    if (k < D) v = (F[(long long)r * ldF + k] / norms[r]) * s;
    __half h = __float2half_rn(v);
    __half l = __float2half_rn(v - __half2float(h));
    Fh[idx] = h;
    Fl[idx] = l;
  }
}

// ---- main kernel
// map_h / map_l: split operands of the query rows (A); map_bh / map_bl: of the column items (B; the same arrays for the
// all-pairs matrix).  EPI 0: distances to p.out; EPI 1: thresholded candidates; EPI 2: threshold sample (fused ranking).
template <int EPI>
__global__ void __launch_bounds__(PW_THREADS, 1)
pairwise_tc_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_l,
                   const __grid_constant__ CUtensorMap map_bh, const __grid_constant__ CUtensorMap map_bl, PwParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = smem;                                            // [h|l][kb] x 16 KB
  uint8_t* sB = sA + 2 * PW_MAXKB * PW_A_BYTES;                  // [stage][h|l] x 16 KB
  float* sAcc = reinterpret_cast<float*>(sB + PW_STAGES * 2 * PW_B_BYTES);   // [128 rows][PW_PITCH]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sAcc + PW_BM * PW_PITCH);
  uint64_t* full = bars;                 // [PW_STAGES]
  uint64_t* empty = bars + PW_STAGES;    // [PW_STAGES]
  uint64_t* a_full = bars + 2 * PW_STAGES;
  uint64_t* a_empty = a_full + 1;

  const int tid = threadIdx.x;
  const int total_tiles = p.tiles_m * p.tiles_n;
  const int per_cta = (total_tiles + gridDim.x - 1) / gridDim.x;
  const int t_begin = blockIdx.x * per_cta;
  const int t_end = min(total_tiles, t_begin + per_cta);

  if (tid == 0) {
    prefetch_tmap(&map_h); prefetch_tmap(&map_l); prefetch_tmap(&map_bh); prefetch_tmap(&map_bl);
    for (int s = 0; s < PW_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_init(a_full, 1); mbar_init(a_empty, 8);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                               // nothing above touches global memory (see common.cuh)

  if (tid < 128) {
    // ===================== TMA producer
    if (tid == 0) {
      int stage = 0, phase = 0, cur_tm = -1, a_phase = 0;
      // the split operands (2 x 11 MB at N = 50 000) are re-read by every CTA for every row block: keep them in L2 while
      // the output streams through
      const uint64_t keep = l2_policy_evict_last();
      for (int t = t_begin; t < t_end; ++t) {
        const int tm = t / p.tiles_n, tn = t % p.tiles_n;
        if (tm != cur_tm) {
          if (cur_tm >= 0) { mbar_wait(a_empty, a_phase); a_phase ^= 1; }   // MMAs reading the old A have retired
          mbar_expect_tx(a_full, 2 * p.kblocks * PW_A_BYTES);
          for (int kb = 0; kb < p.kblocks; ++kb) {
            tma_load_2d_hint(sA + (0 * PW_MAXKB + kb) * PW_A_BYTES, &map_h, a_full, kb * PW_KB, p.row0 + tm * PW_BM, keep);
            tma_load_2d_hint(sA + (1 * PW_MAXKB + kb) * PW_A_BYTES, &map_l, a_full, kb * PW_KB, p.row0 + tm * PW_BM, keep);
          }
          cur_tm = tm;
        }
        for (int kb = 0; kb < p.kblocks; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], 2 * PW_B_BYTES);
          tma_load_2d_hint(sB + (stage * 2 + 0) * PW_B_BYTES, &map_bh, &full[stage], kb * PW_KB, tn * PW_BN, keep);
          tma_load_2d_hint(sB + (stage * 2 + 1) * PW_B_BYTES, &map_bl, &full[stage], kb * PW_KB, tn * PW_BN, keep);
          if (++stage == PW_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers
  const int wg = (tid >> 7) - 1, tid_wg = tid & 127, lane = tid & 31, wq = tid_wg >> 5;
  const int half = wq >> 1;                               // which 64-column half of the tile this warp's epilogue covers
  const int r_local = wg * 64 + (wq & 1) * 32 + lane;     // the row this thread owns in the epilogue
  float* myrow = sAcc + r_local * PW_PITCH;
  const float s2 = p.scal[1];
  int stage = 0, phase = 0, cur_tm = -1, a_phase = 0;
  int e_tm = -1, e_pos = 0, e_region = 0;                 // EPI 1: row block / fill count / region of this thread's candidates
  for (int t = t_begin; t < t_end; ++t) {
    const int tm = t / p.tiles_n, tn = t % p.tiles_n;
    if (tm != cur_tm) { mbar_wait(a_full, a_phase); a_phase ^= 1; cur_tm = tm; }
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int ks_done = 0;
    for (int kb = 0; kb < p.kblocks; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t ah = smem_u32(sA + (0 * PW_MAXKB + kb) * PW_A_BYTES) + wg * 64 * 128;
      const uint32_t al = smem_u32(sA + (1 * PW_MAXKB + kb) * PW_A_BYTES) + wg * 64 * 128;
      const uint32_t bh = smem_u32(sB + (stage * 2 + 0) * PW_B_BYTES);
      const uint32_t bl = smem_u32(sB + (stage * 2 + 1) * PW_B_BYTES);
      const int nks = min(PW_KB / 16, p.ksteps_total - ks_done);
      wgmma_fence();
      for (int ks = 0; ks < nks; ++ks) {
        const uint32_t off = ks * 32;                 // 16 halfs = 32 bytes inside the 128-byte swizzled row
        const uint64_t dah = wgmma_desc(ah + off, 128), dal = wgmma_desc(al + off, 128);
        const uint64_t dbh = wgmma_desc(bh + off, 128), dbl = wgmma_desc(bl + off, 128);
        wgmma_f16_n128(acc, dah, dbh, (ks_done + ks) > 0 ? 1 : 0);
        wgmma_f16_n128(acc, dal, dbh, 1);
        wgmma_f16_n128(acc, dah, dbl, 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      ks_done += nks;
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);      // frees the B stage
      if (++stage == PW_STAGES) { stage = 0; phase ^= 1; }
    }
    const bool last_of_row = (t + 1 == t_end) || ((t + 1) / p.tiles_n != tm);
    if (last_of_row && lane == 0) mbar_arrive(a_empty);
    // accumulator -> shared memory (this warpgroup's 64 rows), then one row per thread
#pragma unroll
    for (int i = 0; i < 64; i += 2)
      *reinterpret_cast<float2*>(sAcc + (wg * 64 + fragment_row(i, tid_wg)) * PW_PITCH + fragment_col(i, tid_wg)) =
          make_float2(acc[i], acc[i + 1]);
    named_bar_sync(1 + wg, 128);

    const int gi = p.row0 + tm * PW_BM + r_local;
    const float a_sq = p.sq[gi];                      // (rows past N read workspace padding; never stored)
    const int lrow = tm * PW_BM + r_local;            // row inside this call's row range
    const bool row_ok = lrow < p.rows;
    float tau = 0.f;
    if (EPI == 1) {
      tau = row_ok ? p.tau_sum[lrow] * p.tau_scale : 0.f;
      if (tm != e_tm) {                                // a new row block: flush the previous block's fill count
        if (e_tm >= 0 && e_tm * PW_BM + r_local < p.rows) p.cnt[(long long)(e_tm * PW_BM + r_local) * 2 * p.nparts + e_region] = e_pos;
        e_tm = tm; e_pos = 0;
        e_region = half * p.nparts + (blockIdx.x - (tm * p.tiles_n) / per_cta);
      }
    }
    float ms[8];                                       // EPI 2: the eight smallest distances of this half tile, ascending
#pragma unroll
    for (int i = 0; i < 8; ++i) ms[i] = 3.0e38f;
    for (int c = 0; c < 2; ++c) {
      const int col = half * (PW_BN / 2) + c * 32;
      const int j0 = tn * PW_BN + col;
      float4 o[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 v = *reinterpret_cast<const float4*>(myrow + col + 4 * q);
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.sq_b + j0) + q);
        const float c0 = v.x * s2, c1 = v.y * s2, c2 = v.z * s2, c3 = v.w * s2;
        if (p.pmode == SE_PDIST_NEGDOT) o[q] = make_float4(-c0, -c1, -c2, -c3);
        else o[q] = make_float4((a_sq + b.x) - 2.f * c0, (a_sq + b.y) - 2.f * c1, (a_sq + b.z) - 2.f * c2, (a_sq + b.w) - 2.f * c3);
      }
      if (EPI == 1) {
        // branch-free pass mask (bit i = column j0 + i is a candidate), then the few set bits are handled one by one
        unsigned mask = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          mask |= (o[q].x < tau ? 1u : 0u) << (4 * q) | (o[q].y < tau ? 1u : 0u) << (4 * q + 1) |
                  (o[q].z < tau ? 1u : 0u) << (4 * q + 2) | (o[q].w < tau ? 1u : 0u) << (4 * q + 3);
        }
        const int nvalid = p.ncols - j0;                   // columns of this block inside the matrix
        if (nvalid < 32) mask &= nvalid > 0 ? ((1u << nvalid) - 1u) : 0u;
        if (!row_ok) mask = 0;
        if (mask) {
#pragma unroll
          for (int q = 0; q < 8; ++q) *reinterpret_cast<float4*>(myrow + col + 4 * q) = o[q];     // own row only
          float* cv = p.cand_val + ((long long)lrow * 2 * p.nparts + e_region) * p.capr;
          int* ci = p.cand_idx + ((long long)lrow * 2 * p.nparts + e_region) * p.capr;
          while (mask) {
            const int i = __ffs(mask) - 1;
            mask &= mask - 1;
            if (e_pos < p.capr) { cv[e_pos] = myrow[col + i]; ci[e_pos] = j0 + i; }
            ++e_pos;
          }
        }
        continue;
      }
      if (EPI == 2) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float vv[4] = {o[q].x, o[q].y, o[q].z, o[q].w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float x = (j0 + 4 * q + e < p.ncols) ? vv[e] : 3.0e38f;
#pragma unroll
            for (int i = 0; i < 8; ++i) { const float lo = fminf(ms[i], x); x = fmaxf(ms[i], x); ms[i] = lo; }
          }
        }
        if (c == 1 && row_ok && p.ncols - (tn * PW_BN + half * (PW_BN / 2)) >= 8) {   // half tiles with >= 8 columns
          float sel = ms[0];
#pragma unroll
          for (int i = 1; i < 8; ++i) if (i == p.jsel) sel = ms[i];
          atomicAdd(&p.tau_sum[lrow], sel);
        }
        continue;
      }
      // EPI 0: back into this thread's row, then the warp stores its 32 rows x 32 columns with coalesced 128-byte rows
#pragma unroll
      for (int q = 0; q < 8; ++q) *reinterpret_cast<float4*>(myrow + col + 4 * q) = o[q];
      __syncwarp();
      const int rbase = r_local - lane;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = rbase + 4 * i + (lane >> 3), cc = col + 4 * (lane & 7);
        const int orow = tm * PW_BM + rr, ocol = tn * PW_BN + cc;
        if (orow >= p.rows || ocol >= p.ncols) continue;
        const float4 v = *reinterpret_cast<const float4*>(sAcc + rr * PW_PITCH + cc);
        float* dst = p.out + (long long)orow * p.ldout + ocol;
        if (ocol + 4 <= p.ncols) {
          __stcs(reinterpret_cast<float4*>(dst), v);
        } else {
          const float e[4] = {v.x, v.y, v.z, v.w};
          for (int k = 0; k < p.ncols - ocol; ++k) __stcs(dst + k, e[k]);
        }
      }
      __syncwarp();
    }
    named_bar_sync(1 + wg, 128);                      // the staging rows are free for the next tile
  }
  if (EPI == 1 && e_tm >= 0 && e_tm * PW_BM + r_local < p.rows) p.cnt[(long long)(e_tm * PW_BM + r_local) * 2 * p.nparts + e_region] = e_pos;
}

// ---- host side
int init_pairwise_tc() {
  if (cudaFuncSetAttribute(pairwise_tc_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM) != cudaSuccess ||
      cudaFuncSetAttribute(pairwise_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM) != cudaSuccess ||
      cudaFuncSetAttribute(pairwise_tc_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM) != cudaSuccess) {
    set_error("pairwise_tc: cannot reserve %d bytes of shared memory", PW_SMEM);
    return SE_ERR_CUDA;
  }
  return SE_OK;
}

long long pairwise_tc_workspace_floats(int N, int D) {
  const long long KW = ceil_div(D, 16) * 16;
  // [pad to 64 floats] scalars (64) + Fh + Fl (halfs, N x KW each, + one spare tile of rows for clipped reads)
  return 64 + 64 + (long long)N * KW + 1024;
}

// ---- host side: operand preparation (shared by the matrix and the fused-ranking entry points) and the launch
struct PwLayout {
  float* sq; float* norms; float* scal; __half* Fh; __half* Fl; int KW, kblocks;
};

// one feature set's region of the workspace: [sq N][norms N] | 256-aligned: scalars (256 bytes), Fh, Fl
static int pw_carve(float* ws, int N, int D, PwLayout* L) {
  L->KW = ceil_div(D, 16) * 16;
  L->kblocks = ceil_div(L->KW, PW_KB);
  if (L->kblocks > PW_MAXKB) return SE_ERR_UNSUPPORTED;                    // D > 128: fp32 tiles
  L->sq = ws;
  L->norms = ws + N;
  uintptr_t base = (reinterpret_cast<uintptr_t>(ws + 2LL * N) + 255) & ~(uintptr_t)255;
  L->scal = reinterpret_cast<float*>(base);
  L->Fh = reinterpret_cast<__half*>(base + 256);
  L->Fl = L->Fh + (long long)N * L->KW;
  return SE_OK;
}

static int pw_absmax(const float* F, int ldF, int N, int D, const PwLayout& L, cudaStream_t st) {
  if (cudaMemsetAsync(L.scal, 0, 256, st) != cudaSuccess) { set_error("pairwise_tc: memset failed"); return SE_ERR_CUDA; }
  long long w1 = ceil_div<long long>((long long)N * D, 256), cap = (long long)sm_count() * 8;
  int g1 = (int)(w1 < cap ? w1 : cap);
  launch(pairwise_absmax_kernel, dim3(g1), dim3(256), 0, st, F, ldF, N, D, L.norms, reinterpret_cast<unsigned*>(L.scal));
  return check_launch("pairwise_absmax_kernel");
}

// scal_other: the other operand's scalars (its max|f| at [0]); scale_out: where 2^(e + e_other) goes (NULL: nowhere)
static int pw_split(const float* F, int ldF, int N, int D, const PwLayout& L, const float* scal_other, float* scale_out,
                    cudaStream_t st) {
  long long w2 = ceil_div<long long>((long long)N * L.KW, 256), cap = (long long)sm_count() * 8;
  int g2 = (int)(w2 < cap ? w2 : cap);
  launch(pairwise_split_kernel, dim3(g2), dim3(256), 0, st, F, ldF, N, D, L.KW, L.norms, (const float*)L.scal, scal_other,
         scale_out, L.Fh, L.Fl);
  return check_launch("pairwise_split_kernel");
}

static int pw_prepare(const float* F, int ldF, int N, int D, float* ws, cudaStream_t st, PwLayout* L) {
  int rc = pw_carve(ws, N, D, L);
  if (!rc) rc = pw_absmax(F, ldF, N, D, *L, st);
  if (!rc) rc = pw_split(F, ldF, N, D, *L, L->scal, L->scal + 1, st);
  return rc;
}

// two feature sets: queries Q (A, region ws_q) and database X (B, region ws_x), each scaled by its own power of two
static int cw_prepare(const float* Q, int ldQ, int Nq, const float* X, int ldX, int Nd, int D, float* ws_q, float* ws_x,
                      cudaStream_t st, PwLayout* A, PwLayout* B) {
  int rc = pw_carve(ws_q, Nq, D, A);
  if (!rc) rc = pw_carve(ws_x, Nd, D, B);
  if (!rc) rc = pw_absmax(Q, ldQ, Nq, D, *A, st);
  if (!rc) rc = pw_absmax(X, ldX, Nd, D, *B, st);
  if (!rc) rc = pw_split(Q, ldQ, Nq, D, *A, B->scal, A->scal + 1, st);
  if (!rc) rc = pw_split(X, ldX, Nd, D, *B, A->scal, nullptr, st);
  return rc;
}

struct PwEpi {
  int kind; float* tau_sum; float tau_scale; int* cnt; float* cand_val; int* cand_idx; int capr; int jsel;
  int grid, nparts;      // kind 1: the sweep's grid and the most CTAs sharing a row block (pt_sweep_shape)
};

// rows [row0, row0+rows) of the N query items against `ncols` column items given by (Bh, Bl, sq_b)
static int pw_launch(const PwLayout& L, int N, int row0, int rows, const __half* Bh, const __half* Bl, const float* sq_b,
                     int ncols, int pmode, float* out, long long ldout, const PwEpi* e1, cudaStream_t st) {
  if (!e1 && ((ldout % 4) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0)) return SE_ERR_UNSUPPORTED;  // 16-byte stores
  CUtensorMap mh, ml, mbh, mbl;
  {
    uint64_t dims[2] = {(uint64_t)L.KW, (uint64_t)N};
    uint64_t strides[1] = {(uint64_t)L.KW * 2};
    uint32_t box[2] = {PW_KB, 128};
    if (!make_tmap(&mh, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, L.Fh, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B) ||
        !make_tmap(&ml, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, L.Fl, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return SE_ERR_CUDA;
    uint64_t bdims[2] = {(uint64_t)L.KW, (uint64_t)ncols};
    if (!make_tmap(&mbh, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(Bh), bdims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B) ||
        !make_tmap(&mbl, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(Bl), bdims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return SE_ERR_CUDA;
  }
  PwParams p;
  p.N = N; p.row0 = row0; p.rows = rows; p.pmode = pmode;
  p.tiles_m = ceil_div(rows, PW_BM); p.tiles_n = ceil_div(ncols, PW_BN);
  p.kblocks = L.kblocks; p.ksteps_total = L.KW / 16;
  p.out = out; p.ldout = ldout;
  p.sq = L.sq; p.sq_b = sq_b; p.scal = L.scal; p.ncols = ncols;
  p.tau_sum = nullptr; p.tau_scale = 0.f; p.cnt = nullptr; p.cand_val = nullptr; p.cand_idx = nullptr; p.capr = 0; p.jsel = 1;
  p.nparts = 2;
  if (e1) { p.jsel = e1->jsel; p.tau_sum = e1->tau_sum; p.tau_scale = e1->tau_scale; p.cnt = e1->cnt; p.cand_val = e1->cand_val; p.cand_idx = e1->cand_idx; p.capr = e1->capr; }
  int rc0 = ensure_setup();
  if (rc0) return rc0;
  int grid = min(sm_count(), p.tiles_m * p.tiles_n);
  if (e1 && e1->kind == 1) { grid = e1->grid; p.nparts = e1->nparts; }   // candidate sweep: regions per (row, half, part)
  if (e1 && e1->kind == 1) launch(pairwise_tc_kernel<1>, dim3(grid), dim3(PW_THREADS), PW_SMEM, st, mh, ml, mbh, mbl, p);
  else if (e1) launch(pairwise_tc_kernel<2>, dim3(grid), dim3(PW_THREADS), PW_SMEM, st, mh, ml, mbh, mbl, p);
  else launch(pairwise_tc_kernel<0>, dim3(grid), dim3(PW_THREADS), PW_SMEM, st, mh, ml, mbh, mbl, p);
  return check_launch("pairwise_tc_kernel");
}

int pairwise_tc(const float* F, int ldF, int N, int D, int row0, int rows, int pmode, int normalize, float* out,
                long long ldout, float* ws, cudaStream_t st) {
  PwLayout L;
  int rc = pw_prepare(F, ldF, N, D, ws, st, &L);
  if (rc) return rc;
  return pw_launch(L, N, row0, rows, L.Fh, L.Fl, L.sq, N, pmode, out, ldout, nullptr, st);
}

int pairwise_tc_cross(const float* Q, int ldQ, int Nq, const float* X, int ldX, int Nd, int D, int row0, int rows, int pmode,
                      float* out, long long ldout, float* ws_q, float* ws_x, cudaStream_t st) {
  PwLayout A, B;
  int rc = cw_prepare(Q, ldQ, Nq, X, ldX, Nd, D, ws_q, ws_x, st, &A, &B);
  if (rc) return rc;
  return pw_launch(A, Nq, row0, rows, B.Fh, B.Fl, B.sq, Nd, pmode, out, ldout, nullptr, st);
}

// ---------------------------------------------------------------------------------------- fused distance + top-k
// SURVEY.md section 8(f) rank 1: the k nearest items of every query WITHOUT the rows x N distance matrix in HBM.
//   1. sample pass (EPI 2): distances to a strided sample of S <= 4096 column items; every (row, 64-column half tile)
//      contributes the j-th smallest of its distances (j = 2..8 by k / N), and their mean -- roughly the j/65 quantile of
//      the row -- is the row's candidate threshold (~3 k of the N entries);
//   2. sweep (EPI 1): the tensor-core kernel over all N columns keeps the entries below the threshold as (value, column)
//      candidates in per-(row, column half, part) regions -- no atomics, nothing else is written;
//   3. one CTA per row sorts its candidates as (key, column) words and writes the first k.
// The values are the ones the matrix kernel would have stored (same arithmetic), so the result equals se_row_topk on the
// written matrix -- provided every row found at least k candidates and no region overflowed, which status[0] reports
// (0 = exact; otherwise the caller falls back to the matrix path).  The threshold is a statistical estimate; exactness
// never depends on it, only the fallback rate does.
// The all-pairs sweep gives a row block to at most two CTAs.  Against a separate database (se_cross_topk) a few query
// blocks would then leave most SMs idle, so that sweep spreads the tiles of all row blocks evenly over every SM: a row
// block is split into column ranges, each CTA keeps its own regions (smaller ones when there are many parts), and the
// finishing sort merges them.
// Thresholds of a large database: the half-tile statistic resolves no quantile below 2/65 of the row, i.e. ~N/32
// candidates, too many for the sort beyond ~65 000 items.  Above PT_NEST_S items (two sets only) the threshold of a row
// is instead the exact k2-th smallest distance to a strided sample of PT_NEST_S database items, with k2 chosen so that
// ~3k of the row's entries are expected below it -- found by this same fused path run on the sample.
constexpr int PT_SAMPLE = 4096, PT_CAPR = 1024, PT_CAP = 4 * PT_CAPR, PT_THREADS = 512, PT_MIN_CAPR = 256;
constexpr int PT_NEST_S = 65536, PT_NEST_MAXK = 1024;

__global__ void __launch_bounds__(256)
pairwise_sample_kernel(const __half* __restrict__ Fh, const __half* __restrict__ Fl, const float* __restrict__ sq, int KW,
                       int S, int stride, __half* __restrict__ Sh, __half* __restrict__ Sl, float* __restrict__ sq_s) {
  pdl_grid_sync();
  const long long total = (long long)S * KW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / KW), k = (int)(i % KW);
    const long long src = (long long)r * stride * KW + k;
    Sh[i] = Fh[src];
    Sl[i] = Fl[src];
    if (k == 0) sq_s[r] = sq[(long long)r * stride];
  }
}

__device__ __forceinline__ uint32_t pt_key(float f) {
  if (f == 0.f) f = 0.f;
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float pt_unkey(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

// one CTA per row: the candidates of its nreg regions (capr entries each) are merged and sorted in shared memory
__global__ void __launch_bounds__(PT_THREADS)
pairwise_topk_finish_kernel(const int* __restrict__ cnt, const float* __restrict__ cand_val, const int* __restrict__ cand_idx,
                            int nreg, int capr, int k, int* __restrict__ out_idx, float* __restrict__ out_val, int ldo,
                            int* __restrict__ status) {
  pdl_grid_sync();
  __shared__ unsigned long long s[PT_CAP];
  __shared__ int s_total, s_bad;
  const int row = blockIdx.x;
  const int* rc = cnt + (long long)row * nreg;
  if (threadIdx.x == 0) { s_total = 0; s_bad = 0; }
  __syncthreads();
  int part = 0, over = 0;
  for (int r = threadIdx.x; r < nreg; r += PT_THREADS) { const int c = rc[r]; part += min(c, capr); over |= c > capr; }
  part = __reduce_add_sync(0xffffffffu, part);
  over = __reduce_or_sync(0xffffffffu, over);
  if ((threadIdx.x & 31) == 0) { atomicAdd(&s_total, part); if (over) s_bad = 1; }
  __syncthreads();
  const int c = s_total;
  if (s_bad || c < k || c > PT_CAP) { if (threadIdx.x == 0) atomicOr(status, 1); return; }
  int npad = 1;
  while (npad < c) npad <<= 1;
  // regions in order; every region's entries are copied by the whole CTA
  for (int r = 0, off = 0; r < nreg; ++r) {
    const int m = min(rc[r], capr);
    const long long src = ((long long)row * nreg + r) * capr;
    for (int i = threadIdx.x; i < m; i += PT_THREADS)
      s[off + i] = ((unsigned long long)pt_key(cand_val[src + i]) << 32) | (unsigned)cand_idx[src + i];
    off += m;
  }
  for (int i = c + threadIdx.x; i < npad; i += PT_THREADS) s[i] = ~0ull;
  __syncthreads();
  for (int kk = 2; kk <= npad; kk <<= 1) {
    for (int j = kk >> 1; j >= 1; j >>= 1) {
      for (int t = threadIdx.x; t < npad / 2; t += PT_THREADS) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int q = i | j;
        const bool up = ((i & kk) == 0);
        const unsigned long long a = s[i], b = s[q];
        if ((a > b) == up) { s[i] = b; s[q] = a; }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < k; i += PT_THREADS) {
    out_idx[(long long)row * ldo + i] = (int)(unsigned)(s[i] & 0xFFFFFFFFull);
    if (out_val) out_val[(long long)row * ldo + i] = pt_unkey((uint32_t)(s[i] >> 32));
  }
}

// the sweep's grid and regions.  All-pairs (split = false): at most one CTA per row block starts inside it, so nparts = 2
// (the fixed layout of se_pairwise_topk).  Two sets (split = true): every SM, and nparts = the most CTAs that share a
// row block; regions shrink (down to PT_MIN_CAPR) so that a row's regions hold about twice the sort's capacity.
struct PtShape { int grid, nparts, capr; };
static PtShape pt_sweep_shape(int rows, int ncols, bool split) {
  const int tiles_m = ceil_div(rows, PW_BM), tiles_n = ceil_div(ncols, PW_BN);
  PtShape sh;
  sh.grid = min(sm_count(), tiles_m * tiles_n);
  if (!split) { sh.grid = max(1, min(sh.grid, tiles_m)); sh.nparts = 2; sh.capr = PT_CAPR; return sh; }
  const int per = ceil_div(tiles_m * tiles_n, sh.grid);
  sh.nparts = 2;
  for (int tm = 0; tm < tiles_m; ++tm) {
    const int first = tm * tiles_n / per, last = ((tm + 1) * tiles_n - 1) / per;
    sh.nparts = max(sh.nparts, last - first + 1);
  }
  sh.capr = min(PT_CAPR, max(PT_MIN_CAPR, ceil_div(PT_CAP, sh.nparts) / 32 * 32));
  return sh;
}

// extra workspace of the fused path, carved behind the matrix path's (all regions 256-byte aligned)
struct PtWs {
  __half* Sh; __half* Sl; float* sq_s; float* tau_sum; int* cnt; float* cv; int* ci; long long bytes;
  int S;
};
static PtWs pt_carve(void* base, int N, int KW, int rows, const PtShape& sh) {
  PtWs w;
  w.S = min(N, PT_SAMPLE);
  const long long nreg = 2LL * sh.nparts;
  uintptr_t p0 = (reinterpret_cast<uintptr_t>(base) + 255) & ~(uintptr_t)255, p = p0;
  auto take = [&](long long bytes) { uintptr_t r = p; p += (bytes + 255) & ~255LL; return r; };
  w.Sh = reinterpret_cast<__half*>(take((long long)(w.S + 256) * KW * 2));     // + one spare tile of rows for clipped reads
  w.Sl = reinterpret_cast<__half*>(take((long long)(w.S + 256) * KW * 2));
  w.sq_s = reinterpret_cast<float*>(take((long long)(w.S + 512) * 4));
  w.tau_sum = reinterpret_cast<float*>(take((long long)rows * 4));
  w.cnt = reinterpret_cast<int*>(take((long long)rows * nreg * 4));
  w.cv = reinterpret_cast<float*>(take((long long)rows * nreg * sh.capr * 4));
  w.ci = reinterpret_cast<int*>(take((long long)rows * nreg * sh.capr * 4));
  w.bytes = (long long)(p - p0) + 256;
  return w;
}

long long pairwise_topk_extra_bytes(int N, int D, int rows) {
  return pt_carve(nullptr, N, ceil_div(D, 16) * 16, rows, pt_sweep_shape(rows, N, false)).bytes;
}

// the nested threshold pass's workspace behind the sweep's: the sample's split operands and norms, the k2 first ranks of
// every row against it, a status word, then the nested call's own PtWs
struct PtNest { __half* Sh; __half* Sl; float* sq; int* idx; float* val; int* status; void* extra; long long bytes; };
static PtNest pt_nest_carve(void* base, int KW, int rows) {
  PtNest n;
  uintptr_t p0 = (reinterpret_cast<uintptr_t>(base) + 255) & ~(uintptr_t)255, p = p0;
  auto take = [&](long long bytes) { uintptr_t r = p; p += (bytes + 255) & ~255LL; return r; };
  n.Sh = reinterpret_cast<__half*>(take((long long)(PT_NEST_S + 256) * KW * 2));
  n.Sl = reinterpret_cast<__half*>(take((long long)(PT_NEST_S + 256) * KW * 2));
  n.sq = reinterpret_cast<float*>(take((long long)(PT_NEST_S + 512) * 4));
  n.idx = reinterpret_cast<int*>(take((long long)rows * PT_NEST_MAXK * 4));
  n.val = reinterpret_cast<float*>(take((long long)rows * PT_NEST_MAXK * 4));
  n.status = reinterpret_cast<int*>(take(256));
  n.extra = reinterpret_cast<void*>(p);
  n.bytes = (long long)(p - p0) + 256 + pt_carve(nullptr, PT_NEST_S, KW, rows, pt_sweep_shape(rows, PT_NEST_S, true)).bytes;
  return n;
}

long long cross_topk_extra_bytes(int Nd, int D, int rows) {
  const int KW = ceil_div(D, 16) * 16;
  const PtWs w = pt_carve(nullptr, Nd, KW, rows, pt_sweep_shape(rows, Nd, true));
  return w.bytes + (Nd > PT_NEST_S ? pt_nest_carve(nullptr, KW, rows).bytes : 0);
}

// row r's threshold = the k2-th smallest sample distance; a failed nested pass fails the call
__global__ void __launch_bounds__(256)
pairwise_nest_threshold_kernel(const float* __restrict__ val, int k2, int rows, const int* __restrict__ nest_status,
                               float* __restrict__ tau, int* __restrict__ status) {
  pdl_grid_sync();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) tau[r] = val[(long long)r * k2 + k2 - 1];
  if (r == 0 && *nest_status) atomicOr(status, 2);
}

// sample pass, sweep and finishing sort of rows [row0, row0+rows) of the A operand against the ncols items of B;
// `extra` is the fused path's own workspace
static int pt_run(const PwLayout& A, int Na, const PwLayout& B, int ncols, bool split, int row0, int rows, int pmode, int k,
                  int* out_idx, float* out_val, int ldo, void* extra, int* status, cudaStream_t st) {
  const PtShape sh = pt_sweep_shape(rows, ncols, split);
  const PtWs w = pt_carve(extra, ncols, A.KW, rows, sh);
  const int S = w.S, stride = ncols / S;
  if (cudaMemsetAsync(w.cnt, 0, (size_t)rows * 2 * sh.nparts * 4, st) != cudaSuccess || cudaMemsetAsync(status, 0, 4, st) != cudaSuccess ||
      cudaMemsetAsync(w.sq_s, 0, (size_t)(S + 512) * 4, st) != cudaSuccess ||
      cudaMemsetAsync(w.tau_sum, 0, (size_t)rows * 4, st) != cudaSuccess) {
    set_error("pairwise_topk: memset failed");
    return SE_ERR_CUDA;
  }
  int rc;
  if (split && ncols > PT_NEST_S) {
    PtNest n = pt_nest_carve(reinterpret_cast<uint8_t*>(extra) + w.bytes, A.KW, rows);
    launch(pairwise_sample_kernel, dim3(min(sm_count() * 4, ceil_div(PT_NEST_S * A.KW, 256))), dim3(256), 0, st, B.Fh, B.Fl, B.sq,
           B.KW, PT_NEST_S, ncols / PT_NEST_S, n.Sh, n.Sl, n.sq);
    rc = check_launch("pairwise_sample_kernel");
    if (rc) return rc;
    PwLayout Bs = B;
    Bs.Fh = n.Sh; Bs.Fl = n.Sl; Bs.sq = n.sq;
    const long long k2l = ceil_div<long long>(3LL * k * PT_NEST_S, ncols);
    const int k2 = (int)(k2l < 1 ? 1 : (k2l > PT_NEST_MAXK ? PT_NEST_MAXK : k2l));
    rc = pt_run(A, Na, Bs, PT_NEST_S, true, row0, rows, pmode, k2, n.idx, n.val, k2, n.extra, n.status, st);
    if (rc) return rc;
    launch(pairwise_nest_threshold_kernel, dim3(ceil_div(rows, 256)), dim3(256), 0, st, (const float*)n.val, k2, rows,
           (const int*)n.status, w.tau_sum, status);
    rc = check_launch("pairwise_nest_threshold_kernel");
    if (rc) return rc;
    PwEpi e1 = {1, w.tau_sum, 1.f, w.cnt, w.cv, w.ci, sh.capr, 0, sh.grid, sh.nparts};
    rc = pw_launch(A, Na, row0, rows, B.Fh, B.Fl, B.sq, ncols, pmode, nullptr, 0, &e1, st);
    if (rc) return rc;
    launch(pairwise_topk_finish_kernel, dim3(rows), dim3(PT_THREADS), 0, st, w.cnt, w.cv, w.ci, 2 * sh.nparts, sh.capr, k,
           out_idx, out_val, ldo, status);
    return check_launch("pairwise_topk_finish_kernel");
  }
  launch(pairwise_sample_kernel, dim3(min(sm_count() * 4, ceil_div(S * A.KW, 256))), dim3(256), 0, st, B.Fh, B.Fl, B.sq, B.KW, S,
         stride, w.Sh, w.Sl, w.sq_s);
  rc = check_launch("pairwise_sample_kernel");
  if (rc) return rc;
  // thresholds: mean over the sample's half tiles (64 distances each) of the j-th smallest distance, j chosen so that
  // ~3k of the row's N entries are expected below it (j / 65 of the row).  j > 8 is not tracked: such shapes (k large
  // against N) simply find fewer than k candidates, report status != 0 and take the matrix path.
  int j = (int)((3LL * k * (PW_BN / 2 + 1) + ncols / 2) / ncols);
  j = max(2, min(8, j));
  PwEpi e2 = {2, w.tau_sum, 0.f, nullptr, nullptr, nullptr, 0, j - 1, 0, 0};
  rc = pw_launch(A, Na, row0, rows, w.Sh, w.Sl, w.sq_s, S, pmode, nullptr, 0, &e2, st);
  if (rc) return rc;
  // the mean over the half tiles that fed the thresholds: those with >= 8 sample columns (a ragged last one may have fewer)
  const int halves = S / (PW_BN / 2) + (S % (PW_BN / 2) >= 8 ? 1 : 0);
  PwEpi e1 = {1, w.tau_sum, 1.f / (float)halves, w.cnt, w.cv, w.ci, sh.capr, 0, sh.grid, sh.nparts};
  rc = pw_launch(A, Na, row0, rows, B.Fh, B.Fl, B.sq, ncols, pmode, nullptr, 0, &e1, st);
  if (rc) return rc;
  launch(pairwise_topk_finish_kernel, dim3(rows), dim3(PT_THREADS), 0, st, w.cnt, w.cv, w.ci, 2 * sh.nparts, sh.capr, k, out_idx,
         out_val, ldo, status);
  return check_launch("pairwise_topk_finish_kernel");
}

int pairwise_tc_topk(const float* F, int ldF, int N, int D, int row0, int rows, int pmode, int k, int* out_idx, float* out_val,
                     int ldo, float* ws, int* status, cudaStream_t st) {
  if (k < 1 || k > 1024 || k > N) return SE_ERR_UNSUPPORTED;
  PwLayout L;
  int rc = pw_prepare(F, ldF, N, D, ws, st, &L);
  if (rc) return rc;
  return pt_run(L, N, L, N, false, row0, rows, pmode, k, out_idx, out_val, ldo, L.Fl + (long long)N * L.KW + 2048, status, st);
}

int pairwise_tc_cross_topk(const float* Q, int ldQ, int Nq, const float* X, int ldX, int Nd, int D, int row0, int rows,
                           int pmode, int k, int* out_idx, float* out_val, int ldo, float* ws_q, float* ws_x, void* extra,
                           int* status, cudaStream_t st) {
  if (k < 1 || k > 1024 || k > Nd) return SE_ERR_UNSUPPORTED;
  PwLayout A, B;
  int rc = cw_prepare(Q, ldQ, Nq, X, ldX, Nd, D, ws_q, ws_x, st, &A, &B);
  if (rc) return rc;
  return pt_run(A, Nq, B, Nd, true, row0, rows, pmode, k, out_idx, out_val, ldo, extra, status, st);
}

}  // namespace se
