// Hierarchical precision of retrieval rankings on the GPU (SURVEY.md §8(f) rank 2):
// ClassHierarchy.hierarchical_precision(..., ks, compute_ahp=K, ignore_qids=True) of the reference
// (class_hierarchy.py:211-316) evaluated on the first K+1 ranks of every query -- exactly the entries the reference
// reads in that mode (`ret[:kmax+1]`, :273,:283) -- from class-similarity look-up tables instead of dictionary lookups.
//
//   per query q with class L = labels[q], for rank j = 0..K:   w_j = wup[L, labels[r_j]],  l_j = 1 - lcs_height[L, labels[r_j]]
//   remove the query itself (first position p with r_p == q, :289-297): the similarity lists lose entry p, the ideal
//   cumulative gains lose entry p and every later entry drops by 1.0 (the query's own similarity)
//   P@k   = sum_{j<k} w'_j / best'_{k-1}                                  (:300-302)
//   AHP@K = trapz_{j<K}( cumsum(w')_j / best'_j, dx = 1/K )               (:308-309)
// `best` (per class, ranking independent: cumsum of the descending class similarities of the whole database, :268,:280)
// is prepared by the caller.  float64 throughout, as the reference (numpy) computes it.
// One warp per query: strided gathers, warp-scan prefix sums with a running carry.
#include "common.cuh"

namespace se {

constexpr int HP_MAXK = 8;          // cut-off points per call

__global__ void __launch_bounds__(128)
hier_precision_kernel(const int* __restrict__ ranks, int ldr, int Q, int K1, int q0, const int* __restrict__ labels, int C,
                      const double* __restrict__ wup, const double* __restrict__ lcsh, const double* __restrict__ best_wup,
                      const double* __restrict__ best_lcs, int nks, int k0, int k1, int k2, int k3, int k4, int k5, int k6, int k7,
                      int clip, double* __restrict__ out) {
  pdl_grid_sync();
  const int ks[HP_MAXK] = {k0, k1, k2, k3, k4, k5, k6, k7};
  const int lane = threadIdx.x & 31;
  const int qi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (qi >= Q) return;
  const int q = q0 + qi;
  const int* r = ranks + (long long)qi * ldr;
  const int L = labels[q];
  const double* wrow = wup + (long long)L * C;
  const double* lrow = lcsh + (long long)L * C;
  const double* bw = best_wup + (long long)L * K1;
  const double* bl = best_lcs + (long long)L * K1;
  // position of the query inside its own list (first occurrence), K1 if absent
  int p = K1;
  for (int j = lane; j < K1; j += 32) if (r[j] == q) p = min(p, j);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) p = min(p, __shfl_xor_sync(0xffffffffu, p, o));
  const int n_eff = (p < K1) ? K1 - 1 : K1;            // entries after the removal
  const int M = 2 * (nks + (clip > 0 ? 1 : 0));
  double* o_q = out + (long long)qi * M;
  double carry_w = 0.0, carry_l = 0.0, ahp_w = 0.0, ahp_l = 0.0, y0_w = 0.0, y0_l = 0.0, yl_w = 0.0, yl_l = 0.0;
  for (int base = 0; base < n_eff; base += 32) {
    const int j = base + lane;                          // index in the list WITHOUT the query
    double w = 0.0, l = 0.0, cbw = 1.0, cbl = 1.0;
    if (j < n_eff) {
      const int src = (j < p) ? j : j + 1;              // index in the original list
      const int lab = labels[r[src]];
      w = wrow[lab];
      l = 1.0 - lrow[lab];
      if (j < p) { cbw = bw[j]; cbl = bl[j]; }
      else { cbw = bw[j + 1] - 1.0; cbl = bl[j + 1] - 1.0; }
    }
    // inclusive scan across the warp
    double sw = w, sl = l;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double tw = __shfl_up_sync(0xffffffffu, sw, o), tl = __shfl_up_sync(0xffffffffu, sl, o);
      if (lane >= o) { sw += tw; sl += tl; }
    }
    sw += carry_w;
    sl += carry_l;
    if (j < n_eff) {
      for (int t = 0; t < nks; ++t)
        if (j == ks[t] - 1) { o_q[2 * t] = sw / cbw; o_q[2 * t + 1] = sl / cbl; }
      if (clip > 0 && j < clip) {
        const double yw = sw / cbw, yl = sl / cbl;
        ahp_w += yw;
        ahp_l += yl;
        if (j == 0) { y0_w = yw; y0_l = yl; }
        if (j == clip - 1) { yl_w = yw; yl_l = yl; }
      }
    }
    carry_w = __shfl_sync(0xffffffffu, sw, 31);
    carry_l = __shfl_sync(0xffffffffu, sl, 31);
  }
  if (clip > 0) {
    // trapezoid rule over j = 0..clip-1 with dx = 1/clip: (sum y - (y_0 + y_last)/2) / clip
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ahp_w += __shfl_xor_sync(0xffffffffu, ahp_w, o); ahp_l += __shfl_xor_sync(0xffffffffu, ahp_l, o);
      y0_w += __shfl_xor_sync(0xffffffffu, y0_w, o); y0_l += __shfl_xor_sync(0xffffffffu, y0_l, o);
      yl_w += __shfl_xor_sync(0xffffffffu, yl_w, o); yl_l += __shfl_xor_sync(0xffffffffu, yl_l, o);
    }
    if (lane == 0) {
      o_q[2 * nks] = (ahp_w - 0.5 * (y0_w + yl_w)) / (double)clip;
      o_q[2 * nks + 1] = (ahp_l - 0.5 * (y0_l + yl_l)) / (double)clip;
    }
  }
}

// The same metrics from rankings of any length, with the whole P@k curve, the unclipped AHP and classical AP
// (what evaluate_retrieval.py:195 asks for: ks = 1..plot_max, compute_ahp = clip or True, compute_ap = True):
//   curve[q, t, k-1] = P@k for k = 1..kcurve, t = 0 WUP / 1 LCS_HEIGHT                        (class_hierarchy.py:300-302)
//   ahp[q, t]        = trapz(cumsum(sim) / best, dx = 1/len) over the first `clip` entries, or over ALL n_ret - 1 entries
//                      of the list without the query when clip < 0                           (:303-309)
//   ap[q]            = average_precision_score(same class?, -rank) = mean over the same-class items of
//                      (same-class items up to and including this rank) / rank, query removed     (:310-314)
// With query_labels (se_hier_metrics_q, ignore_qids=False) the query's class is query_labels[qi] and nothing is removed:
// the queries need not be database items.
// One warp per query walks the list in blocks of 32 ranks with warp scans (float64 for the gains, integers for the hits).
__global__ void __launch_bounds__(128)
hier_metrics_kernel(const int* __restrict__ ranks, long long ldr, int Q, int n_ret, int q0, const int* __restrict__ query_labels,
                    const int* __restrict__ labels, int C, const double* __restrict__ wup, const double* __restrict__ lcsh,
                    const double* __restrict__ best_wup, const double* __restrict__ best_lcs, int kcurve, int clip,
                    double* __restrict__ curve, double* __restrict__ ahp, double* __restrict__ ap) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const int qi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (qi >= Q) return;
  const int q = query_labels ? -1 : q0 + qi;           // -1: no database item is the query
  const int* r = ranks + (long long)qi * ldr;
  const int L = query_labels ? query_labels[qi] : labels[q];
  const double* wrow = wup + (long long)L * C;
  const double* lrow = lcsh + (long long)L * C;
  const double* bw = best_wup + (long long)L * n_ret;
  const double* bl = best_lcs + (long long)L * n_ret;
  int p = n_ret;                                       // position of the query in its own list (first occurrence)
  if (q >= 0)
    for (int j = lane; j < n_ret; j += 32) if (r[j] == q) p = min(p, j);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) p = min(p, __shfl_xor_sync(0xffffffffu, p, o));
  const int n_eff = (p < n_ret) ? n_ret - 1 : n_ret;
  const int n_ahp = clip < 0 ? n_eff : min(clip, n_eff);
  // how far the walk has to go: the curve, the AHP range, or everything (AP)
  const int n_walk = ap ? n_eff : max(min(kcurve, n_eff), n_ahp);
  double carry_w = 0.0, carry_l = 0.0, sum_w = 0.0, sum_l = 0.0, y0_w = 0.0, y0_l = 0.0, ye_w = 0.0, ye_l = 0.0, ap_sum = 0.0;
  int carry_hits = 0;
  for (int base = 0; base < n_walk; base += 32) {
    const int j = base + lane;
    double w = 0.0, l = 0.0, cbw = 1.0, cbl = 1.0;
    int rel = 0;
    if (j < n_walk) {
      const int src = (j < p) ? j : j + 1;
      const int lab = labels[r[src]];
      w = wrow[lab];
      l = 1.0 - lrow[lab];
      rel = (lab == L);
      if (j < p) { cbw = bw[j]; cbl = bl[j]; }
      else { cbw = bw[j + 1] - 1.0; cbl = bl[j + 1] - 1.0; }
    }
    double sw = w, sl = l;
    int hits = rel;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double tw = __shfl_up_sync(0xffffffffu, sw, o), tl = __shfl_up_sync(0xffffffffu, sl, o);
      const int th = __shfl_up_sync(0xffffffffu, hits, o);
      if (lane >= o) { sw += tw; sl += tl; hits += th; }
    }
    sw += carry_w; sl += carry_l; hits += carry_hits;
    if (j < n_walk) {
      const double yw = sw / cbw, yl = sl / cbl;
      if (j < kcurve) {
        curve[((long long)qi * 2 + 0) * kcurve + j] = yw;
        curve[((long long)qi * 2 + 1) * kcurve + j] = yl;
      }
      if (j < n_ahp) {
        sum_w += yw; sum_l += yl;
        if (j == 0) { y0_w = yw; y0_l = yl; }
        if (j == n_ahp - 1) { ye_w = yw; ye_l = yl; }
      }
      if (rel) ap_sum += (double)hits / (double)(j + 1);
    }
    carry_w = __shfl_sync(0xffffffffu, sw, 31);
    carry_l = __shfl_sync(0xffffffffu, sl, 31);
    carry_hits = __shfl_sync(0xffffffffu, hits, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum_w += __shfl_xor_sync(0xffffffffu, sum_w, o); sum_l += __shfl_xor_sync(0xffffffffu, sum_l, o);
    y0_w += __shfl_xor_sync(0xffffffffu, y0_w, o); y0_l += __shfl_xor_sync(0xffffffffu, y0_l, o);
    ye_w += __shfl_xor_sync(0xffffffffu, ye_w, o); ye_l += __shfl_xor_sync(0xffffffffu, ye_l, o);
    ap_sum += __shfl_xor_sync(0xffffffffu, ap_sum, o);
  }
  if (lane == 0) {
    if (ahp && n_ahp > 0) {
      // np.trapz(y, dx = 1/len): (sum y - (y_0 + y_last)/2) / len; the clipped form divides by `clip` (class_hierarchy.py:308)
      const double len = clip > 0 ? (double)clip : (double)n_ahp;
      ahp[2 * (long long)qi] = (sum_w - 0.5 * (y0_w + ye_w)) / len;
      ahp[2 * (long long)qi + 1] = (sum_l - 0.5 * (y0_l + ye_l)) / len;
    }
    if (ap) ap[qi] = carry_hits > 0 ? ap_sum / (double)carry_hits : 0.0;
  }
}

}  // namespace se

using namespace se;

extern "C" int se_hier_metrics(const int32_t* ranks, int64_t ldr, int Q, int n_ret, int q0, const int32_t* labels, int C,
                               const double* wup_lut, const double* lcs_height_lut, const double* best_wup,
                               const double* best_lcs, int kcurve, int clip, double* curve, double* ahp, double* ap,
                               void* stream) {
  SE_REQUIRE(ranks && labels && wup_lut && lcs_height_lut && best_wup && best_lcs, "null pointer");
  SE_REQUIRE(Q > 0 && n_ret > 1 && ldr >= n_ret && C > 0 && kcurve >= 0 && kcurve <= n_ret - 1, "bad sizes");
  SE_REQUIRE(kcurve == 0 || curve, "curve output missing");
  SE_REQUIRE(clip <= n_ret - 1, "clip (compute_ahp) needs clip + 1 retrieved ranks");
  SE_REQUIRE(clip == 0 || ahp, "ahp output missing");
  const int warps = 4;
  launch(hier_metrics_kernel, dim3(ceil_div(Q, warps)), dim3(32 * warps), 0, as_stream(stream), ranks, (long long)ldr, Q, n_ret, q0,
         (const int*)nullptr, labels, C, wup_lut, lcs_height_lut, best_wup, best_lcs, kcurve, clip, curve, clip != 0 ? ahp : nullptr,
         ap);
  return check_launch("hier_metrics_kernel");
}

extern "C" int se_hier_metrics_q(const int32_t* ranks, int64_t ldr, int Q, int n_ret, const int32_t* query_labels,
                                 const int32_t* labels, int C, const double* wup_lut, const double* lcs_height_lut,
                                 const double* best_wup, const double* best_lcs, int kcurve, int clip, double* curve, double* ahp,
                                 double* ap, void* stream) {
  SE_REQUIRE(ranks && query_labels && labels && wup_lut && lcs_height_lut && best_wup && best_lcs, "null pointer");
  SE_REQUIRE(Q > 0 && n_ret > 0 && ldr >= n_ret && C > 0 && kcurve >= 0 && kcurve <= n_ret, "bad sizes");
  SE_REQUIRE(kcurve == 0 || curve, "curve output missing");
  SE_REQUIRE(clip <= n_ret, "clip (compute_ahp) needs clip retrieved ranks");
  SE_REQUIRE(clip == 0 || ahp, "ahp output missing");
  const int warps = 4;
  launch(hier_metrics_kernel, dim3(ceil_div(Q, warps)), dim3(32 * warps), 0, as_stream(stream), ranks, (long long)ldr, Q, n_ret, 0,
         query_labels, labels, C, wup_lut, lcs_height_lut, best_wup, best_lcs, kcurve, clip, curve, clip != 0 ? ahp : nullptr, ap);
  return check_launch("hier_metrics_kernel");
}

extern "C" int se_hier_precision(const int32_t* ranks, int ldr, int Q, int K1, int q0, const int32_t* labels, int C,
                                 const double* wup_lut, const double* lcs_height_lut, const double* best_wup,
                                 const double* best_lcs, const int32_t* ks, int nks, int clip, double* out, void* stream) {
  SE_REQUIRE(ranks && labels && wup_lut && lcs_height_lut && best_wup && best_lcs && out && ks, "null pointer");
  SE_REQUIRE(Q > 0 && K1 > 1 && ldr >= K1 && C > 0 && nks >= 0 && nks <= HP_MAXK, "bad sizes");
  int kk[HP_MAXK] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int t = 0; t < nks; ++t) {
    SE_REQUIRE(ks[t] >= 1 && ks[t] <= K1 - 1, "a cut-off point needs k + 1 retrieved ranks (the query itself is removed)");
    kk[t] = ks[t];
  }
  SE_REQUIRE(clip >= 0 && clip <= K1 - 1, "clip (compute_ahp) needs clip + 1 retrieved ranks");
  const int warps = 4;
  launch(hier_precision_kernel, dim3(ceil_div(Q, warps)), dim3(32 * warps), 0, as_stream(stream), ranks, ldr, Q, K1, q0, labels, C,
         wup_lut, lcs_height_lut, best_wup, best_lcs, nks, kk[0], kk[1], kk[2], kk[3], kk[4], kk[5], kk[6], kk[7], clip, out);
  return check_launch("hier_precision_kernel");
}
