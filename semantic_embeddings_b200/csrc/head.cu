// The embedding head as ONE fused kernel (north-star item): L2-normalise, gather t = E[label],
// 1 - <t,x> (or squared distance) loss, nearest-class accuracy over the whole class matrix, and the
// backward pass -- one warp per sample row, warp-shuffle reductions, 128-bit coalesced loads.
//
// Replaces these graph ops of the reference:
//   utils.l2norm              utils.py:125-127      x = z * rsqrt(max(sum z^2, 1e-12))
//   transform_inputs          learn_image_embeddings.py:48-50   (host gather E[y], now in-kernel)
//   utils.inv_correlation     utils.py:44-46        1 - sum_d t*x
//   utils.squared_distance    utils.py:34-36        sum_d (x-t)^2
//   utils.nn_accuracy         utils.py:57-100       |max_c <x,E_c> - <x,t>| < 1e-6  (k<=1)
//   + TF autodiff of the above (learn_image_embeddings.py:238)
// and Activation('softmax') + categorical_crossentropy of the classifier branch
// (learn_image_embeddings.py:44,230-231), and the DeViSE hinge ranking loss
//   utils.devise_ranking_loss utils.py:103-122   sum_c relu(m - <t,z> + <z,E_c>) - m   (learn_devise.py)
#include <float.h>

#include "common.cuh"

namespace se {

constexpr int HEAD_WARPS = 4;
constexpr int HEAD_WARPS_SPLIT = 8;     // warps of a CTA that share one row's class loop (embed_head_kernel, split mode)

template <bool VEC>
__device__ __forceinline__ float warp_dot(const float* __restrict__ a_smem, const float* __restrict__ b_gmem, int D,
                                          int lane) {
  float s = 0.f;
  if (VEC) {
    for (int i = lane; i < (D >> 2); i += 32) {
      float4 b = *reinterpret_cast<const float4*>(b_gmem + 4 * i);
      float4 a = *reinterpret_cast<const float4*>(a_smem + 4 * i);
      s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); s = fmaf(a.z, b.z, s); s = fmaf(a.w, b.w, s);
    }
  } else {
    for (int i = lane; i < D; i += 32) s = fmaf(a_smem[i], b_gmem[i], s);
  }
  return warp_sum(s);
}

template <bool VEC>
__global__ void __launch_bounds__(HEAD_WARPS_SPLIT * 32)
embed_head_kernel(const float* __restrict__ z, int ldz, const int* __restrict__ labels, const float* __restrict__ E,
                  int ldE, int B, int D, int C, int loss_kind, float loss_scale, const float* __restrict__ extra_dx,
                  float* __restrict__ x_out, float* __restrict__ loss, float* __restrict__ acc, float* __restrict__ dz,
                  float* __restrict__ rank_out, int es_classes, int split, float margin) {
  // split == 0: one row per warp.  split == 1 (large class matrices read from global memory): one row per CTA -- every
  // warp holds the row, the warps share the class loop of the accuracy metric, warp 0 writes the row's outputs.
  pdl_grid_sync();
  extern __shared__ __align__(16) float smem[];
  __shared__ float s_red[HEAD_WARPS_SPLIT][4];
  __shared__ float s_hinge[HEAD_WARPS_SPLIT];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nw = blockDim.x >> 5;
  const int Dp = (D + 3) & ~3;
  float* xs = smem + warp * Dp;  // this warp's row (wrapped output x)
  // class matrix staged in shared memory (row pitch D+1: conflict-free when every lane walks its own class row);
  // es_classes == 0 -> the matrix does not fit, the accuracy loop reads it from global memory
  float* Es = smem + HEAD_WARPS * Dp;
  const bool want_acc = acc || rank_out;
  // the ranking loss' pass over the classes (its loss and its gradient both need it)
  const bool want_rank = loss_kind == SE_LOSS_DEVISE_RANK && (loss || dz);
  if (es_classes > 0 && (want_acc || want_rank)) {
    for (int c = warp; c < C; c += HEAD_WARPS)
      for (int i = lane; i < D; i += 32) Es[c * (D + 1) + i] = E[(long long)c * ldE + i];
    __syncthreads();
  }
  const int row = split ? blockIdx.x : blockIdx.x * HEAD_WARPS + warp;
  if (row >= B) return;                          // (uniform over the CTA when split)
  const bool lead = !split || warp == 0;         // this warp writes the row's outputs
  const int c_first = split ? warp * 32 + lane : lane, c_step = split ? 32 * nw : 32;
  const float* zr = z + (long long)row * ldz;

  // ---- load z, sum of squares
  float ss = 0.f;
  if (VEC) {
    for (int i = lane; i < (D >> 2); i += 32) {
      float4 v = ldg_nc_f4(zr + 4 * i);
      *reinterpret_cast<float4*>(xs + 4 * i) = v;
      ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
  } else {
    for (int i = lane; i < D; i += 32) { float v = zr[i]; xs[i] = v; ss += v * v; }
  }
  ss = warp_sum(ss);
  float inv = 1.f;
  bool clamped = false;
  if (loss_kind == SE_LOSS_INV_CORR) {
    clamped = !(ss >= 1e-12f);
    inv = rsqrtf(fmaxf(ss, 1e-12f));
    __syncwarp();
    for (int i = lane; i < D; i += 32) xs[i] *= inv;
  } else if (loss_kind == SE_LOSS_SOFTMAX_CORR) {
    // Activation('softmax') wrapper (learn_image_embeddings.py:129-130): x = exp(z - max z) / sum
    __syncwarp();
    float m = -FLT_MAX;
    for (int i = lane; i < D; i += 32) m = fmaxf(m, xs[i]);
    m = warp_max(m);
    float se = 0.f;
    for (int i = lane; i < D; i += 32) { const float e = expf(xs[i] - m); xs[i] = e; se += e; }
    se = warp_sum(se);
    const float is = 1.f / se;
    for (int i = lane; i < D; i += 32) xs[i] *= is;
  }
  __syncwarp();
  if (x_out && lead) {
    float* xo = x_out + (long long)row * ldz;
    if (VEC) {
      for (int i = lane; i < (D >> 2); i += 32)
        *reinterpret_cast<float4*>(xo + 4 * i) = *reinterpret_cast<const float4*>(xs + 4 * i);
    } else {
      for (int i = lane; i < D; i += 32) xo[i] = xs[i];
    }
  }

  // ---- loss against the target row
  const int lab = labels[row];
  const float* t = E + (long long)lab * ldE;
  float true_sim = warp_dot<VEC>(xs, t, D, lane);
  float xnorm2 = (loss_kind == SE_LOSS_INV_CORR) ? ss * inv * inv : ss;
  float l;
  float true_dist = 0.f;
  if (loss_kind == SE_LOSS_MSE) {
    float s = 0.f;
    for (int i = lane; i < D; i += 32) { float d = xs[i] - t[i]; s = fmaf(d, d, s); }
    true_dist = warp_sum(s);
    l = true_dist;
  } else {
    l = 1.f - true_sim;
  }
  if (loss && lane == 0 && lead && loss_kind != SE_LOSS_DEVISE_RANK) loss[row] = l;

  // ---- accuracy: nearest class over the whole class matrix (utils.py:73-93)
  if (loss_kind == SE_LOSS_SOFTMAX_CORR) {
    // metric 'accuracy' of the softmax wrapper (learn_image_embeddings.py:166) = Keras categorical_accuracy:
    // argmax x == argmax t (lowest index on ties); rank = number of outputs strictly above the one at argmax t
    if (want_acc) {
      float bt = -FLT_MAX, bx = -FLT_MAX;
      int at = 0, ax = 0;
      for (int i = lane; i < D; i += 32) {
        if (t[i] > bt) { bt = t[i]; at = i; }
        if (xs[i] > bx) { bx = xs[i]; ax = i; }
      }
      for (int o = 16; o > 0; o >>= 1) {
        float ot = __shfl_xor_sync(0xffffffffu, bt, o), ox = __shfl_xor_sync(0xffffffffu, bx, o);
        int oat = __shfl_xor_sync(0xffffffffu, at, o), oax = __shfl_xor_sync(0xffffffffu, ax, o);
        if (ot > bt || (ot == bt && oat < at)) { bt = ot; at = oat; }
        if (ox > bx || (ox == bx && oax < ax)) { bx = ox; ax = oax; }
      }
      const float xt = xs[at];
      float above = 0.f;
      for (int i = lane; i < D; i += 32) above += (xs[i] > xt) ? 1.f : 0.f;
      above = warp_sum(above);
      if (lane == 0) { if (acc) acc[row] = (ax == at) ? 1.f : 0.f; if (rank_out) rank_out[row] = above; }
    }
  } else if (want_acc) {
    // one class per lane and step, no shuffles inside the loop.  The class matrix comes from shared memory when it fits
    // (2 shared loads per FMA), else every lane streams its own row of E from global memory: a lane's 128-byte line
    // serves its next 32 steps from L1, and 32 rows are in flight per warp (a warp-per-class loop with a shuffle
    // reduction per class was latency-bound: 1.6 ms for 32 rows x 555 classes x 555 dimensions)
    const float* Eb = es_classes > 0 ? Es : E;
    const long long ep = es_classes > 0 ? (long long)(D + 1) : (long long)ldE;
    float best = (loss_kind == SE_LOSS_MSE) ? FLT_MAX : -FLT_MAX;
    float mine = -FLT_MAX;                          // this row's own class, from the same summation order as `best`
    for (int c = c_first; c < C; c += c_step) {
      const float* e = Eb + c * ep;
      float sim = 0.f, en = 0.f;
#pragma unroll 8
      for (int i = 0; i < D; ++i) { const float b = e[i]; sim = fmaf(xs[i], b, sim); en = fmaf(b, b, en); }
      if (loss_kind == SE_LOSS_MSE) { const float dist = xnorm2 + en - 2.f * sim; best = fminf(best, dist); if (c == lab) mine = -dist; }
      else { best = fmaxf(best, sim); if (c == lab) mine = sim; }
    }
    best = (loss_kind == SE_LOSS_MSE) ? -warp_max(-best) : warp_max(best);
    mine = warp_max(mine);
    if (split) {                                  // combine the warps' shares of the class loop
      if (lane == 0) { s_red[warp][0] = (loss_kind == SE_LOSS_MSE) ? -best : best; s_red[warp][1] = mine; }
      __syncthreads();
      float bb = -FLT_MAX, mm = -FLT_MAX;
      for (int w2 = 0; w2 < nw; ++w2) { bb = fmaxf(bb, s_red[w2][0]); mm = fmaxf(mm, s_red[w2][1]); }
      best = (loss_kind == SE_LOSS_MSE) ? -bb : bb;
      mine = mm;
    }
    // the true class' score comes from the SAME expression as the other classes' (in exact arithmetic it equals
    // utils.py:80,91's separately computed true_dist / true_sim; in fp32 the two differ by more than the 1e-6 threshold
    // for distances of O(10), which would make the metric a coin flip)
    const float ref = (loss_kind == SE_LOSS_MSE) ? -mine : mine;
    if (acc && lane == 0 && lead) acc[row] = (fabsf(best - ref) < 1e-6f) ? 1.f : 0.f;
    if (rank_out) {
      // top-k form of the metric (utils.py:85,95: any of the k best values within 1e-6 of the true one) for every k at
      // once: with G = classes better than the true value by >= 1e-6 and T = classes within 1e-6 of it, the k best
      // contain a member of T iff G < k (and T is not empty) -> rank = G, or C when T is empty
      float gcnt = 0.f, tcnt = 0.f;
      for (int c = c_first; c < C; c += c_step) {
        const float* e = Eb + c * ep;
        float sim = 0.f, en = 0.f;
#pragma unroll 8
        for (int i = 0; i < D; ++i) { const float b = e[i]; sim = fmaf(xs[i], b, sim); en = fmaf(b, b, en); }
        const float v = (loss_kind == SE_LOSS_MSE) ? -(xnorm2 + en - 2.f * sim) : sim;      // larger = better
        if (fabsf(v - mine) < 1e-6f) tcnt += 1.f; else if (v > mine) gcnt += 1.f;
      }
      gcnt = warp_sum(gcnt); tcnt = warp_sum(tcnt);
      if (split) {
        if (lane == 0) { s_red[warp][2] = gcnt; s_red[warp][3] = tcnt; }
        __syncthreads();
        gcnt = 0.f; tcnt = 0.f;
        for (int w2 = 0; w2 < nw; ++w2) { gcnt += s_red[w2][2]; tcnt += s_red[w2][3]; }
      }
      if (lane == 0 && lead) rank_out[row] = tcnt > 0.f ? gcnt : (float)C;
    }
  }

  // ---- DeViSE hinge ranking loss (utils.py:116-120): h_c = (m - <t,z>) + <z,E_c>; loss = sum_c relu(h_c) - m;
  // dL/dz = scale * sum_{h_c > 0} (E_c - t) = scale * (sum_{c in A} E_c - |A| t).  One class per lane and step (the
  // scores come from the same expression as the accuracy loop's); the active set A goes to a shared-memory bit mask
  // (bit c%32 of word c/32), and the gradient sums the active rows in class order -- a fixed order per row.
  if (want_rank) {
    const float* Eb = es_classes > 0 ? Es : E;
    const long long ep = es_classes > 0 ? (long long)(D + 1) : (long long)ldE;
    const int mw = (C + 31) >> 5;
    unsigned* act = reinterpret_cast<unsigned*>(smem + nw * Dp + es_classes * (D + 1)) + (split ? 0 : warp * mw);
    const float base = margin - true_sim;
    float hsum = 0.f;
    for (int cb = c_first - lane; cb < C; cb += c_step) {    // uniform over the warp: one 32-class word per step
      const int c = cb + lane;
      bool on = false;
      if (c < C) {
        const float* e = Eb + c * ep;
        float sim = 0.f;
#pragma unroll 8
        for (int i = 0; i < D; ++i) sim = fmaf(xs[i], e[i], sim);
        const float h = base + sim;
        on = h > 0.f;                     // relu'(0) = 0: a hinge of exactly zero is not active
        if (on) hsum += h;
      }
      const unsigned bits = __ballot_sync(0xffffffffu, on);
      if (lane == 0) act[cb >> 5] = bits;
    }
    hsum = warp_sum(hsum);
    if (split) {
      if (lane == 0) s_hinge[warp] = hsum;
      __syncthreads();                    // (also publishes every warp's words of the mask)
      hsum = 0.f;
      for (int w2 = 0; w2 < nw; ++w2) hsum += s_hinge[w2];
    } else {
      __syncwarp();
    }
    if (loss && lane == 0 && lead) loss[row] = hsum - margin;
    if (dz) {
      int na = 0;
      for (int w = 0; w < mw; ++w) na += __popc(act[w]);
      const float fa = (float)na;
      float* dzr = dz + (long long)row * ldz;
      const float* ex = extra_dx ? extra_dx + (long long)row * ldz : nullptr;
      // split: the warps share the dimensions of the row
      for (int i = split ? warp * 32 + lane : lane; i < D; i += split ? 32 * nw : 32) {
        float s = 0.f;
        for (int w = 0; w < mw; ++w) {
          unsigned bits = act[w];
          while (bits) {
            const int b = __ffs(bits) - 1;
            bits &= bits - 1;
            s += Eb[(long long)(w * 32 + b) * ep + i];
          }
        }
        dzr[i] = loss_scale * (s - fa * t[i]) + (ex ? ex[i] : 0.f);
      }
    }
  }

  // ---- backward
  if (dz && lead && loss_kind != SE_LOSS_DEVISE_RANK) {
    float* dzr = dz + (long long)row * ldz;
    const float* ex = extra_dx ? extra_dx + (long long)row * ldz : nullptr;
    if (loss_kind == SE_LOSS_INV_CORR) {
      // g = dL/dx = -scale*t + extra ; dz = inv * (g - x <x,g>)   (only inv*g when the clamp is active)
      float xg = 0.f;
      for (int i = lane; i < D; i += 32) {
        float g = -loss_scale * t[i] + (ex ? ex[i] : 0.f);
        xg = fmaf(xs[i], g, xg);
      }
      xg = warp_sum(xg);
      if (clamped) xg = 0.f;
      for (int i = lane; i < D; i += 32) {
        float g = -loss_scale * t[i] + (ex ? ex[i] : 0.f);
        dzr[i] = inv * (g - xs[i] * xg);
      }
    } else if (loss_kind == SE_LOSS_SOFTMAX_CORR) {
      // g = dL/dx = -scale*t + extra ; softmax Jacobian: dz_j = x_j * (g_j - <x,g>)
      float xg = 0.f;
      for (int i = lane; i < D; i += 32) {
        float g = -loss_scale * t[i] + (ex ? ex[i] : 0.f);
        xg = fmaf(xs[i], g, xg);
      }
      xg = warp_sum(xg);
      for (int i = lane; i < D; i += 32) {
        float g = -loss_scale * t[i] + (ex ? ex[i] : 0.f);
        dzr[i] = xs[i] * (g - xg);
      }
    } else if (loss_kind == SE_LOSS_UNNORM_CORR) {
      for (int i = lane; i < D; i += 32) dzr[i] = -loss_scale * t[i] + (ex ? ex[i] : 0.f);
    } else {
      for (int i = lane; i < D; i += 32) dzr[i] = 2.f * loss_scale * (xs[i] - t[i]) + (ex ? ex[i] : 0.f);
    }
  }
}

// softmax + Keras categorical_crossentropy(prob) + arg-max accuracy + backward; one warp per row.
// SMOOTH = false: one-hot targets.  SMOOTH = true: the label-smoothed targets of learn_classifier.py:17-22, t_hi on the
// label and t_lo on every other class (the float32 values of the reference's float32 target array); every class then
// contributes to the loss and, through its clip mask, to the gradient.
template <bool SMOOTH>
__global__ void __launch_bounds__(HEAD_WARPS * 32)
softmax_xent_kernel(const float* __restrict__ logits, int ld, const int* __restrict__ labels, int B, int C, float scale,
                    float* __restrict__ prob, float* __restrict__ loss, float* __restrict__ acc,
                    float* __restrict__ dlogits, float* __restrict__ rank_out, float t_hi, float t_lo) {
  pdl_grid_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * HEAD_WARPS + warp;
  if (row >= B) return;
  const float* lr = logits + (long long)row * ld;
  float m = -FLT_MAX;
  int arg = 0;
  for (int i = lane; i < C; i += 32) { float v = lr[i]; if (v > m) { m = v; arg = i; } }
  // warp arg-max with lowest-index tie-break (np.argmax semantics)
  for (int o = 16; o > 0; o >>= 1) {
    float om = __shfl_xor_sync(0xffffffffu, m, o);
    int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (om > m || (om == m && oa < arg)) { m = om; arg = oa; }
  }
  float s = 0.f;
  for (int i = lane; i < C; i += 32) s += expf(lr[i] - m);
  s = warp_sum(s);
  const float invs = 1.f / s;
  const int lab = labels[row];
  // Keras: p /= sum(p); p = clip(p, 1e-7, 1-1e-7); loss = -sum_c t_c log p_c.  The clip passes the gradient where
  // lo <= p <= hi (tf.clip_by_value).  (p is exp(z - m) / s: the renormalisation is a no-op up to rounding and does not
  // change the gradient.)
  const float lo = 1e-7f, hi = 1.f - 1e-7f;
  // argmax(y_true), the class Keras' accuracy metrics compare against: the label, unless smoothing gives the label the
  // smaller target (ls > (C-1)/C) -- then the lowest other index
  const int tgt = (!SMOOTH || t_hi >= t_lo) ? lab : (lab == 0 ? 1 : 0);
  float row_loss;
  bool live = true;   // one-hot: the label's clip mask
  float tl = 1.f;     // smoothed: T = sum_c live_c t_c
  if constexpr (!SMOOTH) {
    const float py = expf(lr[lab] - m) * invs;
    const float pyc = fminf(fmaxf(py, lo), hi);
    row_loss = -logf(pyc);
    live = (py >= lo) && (py <= hi);
  } else {
    float l = 0.f, t_live = 0.f;
    for (int i = lane; i < C; i += 32) {
      const float p = expf(lr[i] - m) * invs;
      const float t = (i == lab) ? t_hi : t_lo;
      l = fmaf(t, logf(fminf(fmaxf(p, lo), hi)), l);
      if (p >= lo && p <= hi) t_live += t;
    }
    row_loss = -warp_sum(l);
    tl = warp_sum(t_live);
  }
  if (lane == 0) {
    if (loss) loss[row] = row_loss;
    if (acc) acc[row] = (arg == tgt) ? 1.f : 0.f;
  }
  if (rank_out) {   // utils.top_k_acc (utils.py:49-54) = in_top_k: classes with a strictly larger probability than the target's
    const float ll = lr[tgt];
    float above = 0.f;
    for (int i = lane; i < C; i += 32) above += (lr[i] > ll) ? 1.f : 0.f;
    above = warp_sum(above);
    if (lane == 0) rank_out[row] = above;
  }
  for (int i = lane; i < C; i += 32) {
    float p = expf(lr[i] - m) * invs;
    if (prob) prob[(long long)row * ld + i] = p;
    if (dlogits) {
      if constexpr (!SMOOTH) {
        dlogits[(long long)row * ld + i] = live ? scale * (p - (i == lab ? 1.f : 0.f)) : 0.f;
      } else {
        // dz_j = scale * (p_j T - live_j t_j); with one-hot targets this is the branch above
        const float t = (i == lab) ? t_hi : t_lo;
        dlogits[(long long)row * ld + i] = scale * (p * tl - ((p >= lo && p <= hi) ? t : 0.f));
      }
    }
  }
}

}  // namespace se

using namespace se;

extern "C" int se_embed_head_fwd_bwd(const float* z, int ldz, const int32_t* labels, const float* E, int ldE, int B,
                                     int D, int C, int loss_kind, float loss_scale, const float* extra_dx, float* x_out,
                                     float* loss, float* acc, float* dz, void* stream) {
  return se_embed_head_fwd_bwd_ex(z, ldz, labels, E, ldE, B, D, C, loss_kind, loss_scale, extra_dx, x_out, loss, acc, dz,
                                  nullptr, stream);
}

static int embed_head(const float* z, int ldz, const int32_t* labels, const float* E, int ldE, int B, int D, int C,
                      int loss_kind, float loss_scale, const float* extra_dx, float* x_out, float* loss, float* acc,
                      float* dz, float* rank_out, float margin, void* stream) {
  SE_REQUIRE(z && labels && E && B > 0 && D > 0 && C > 0, "bad arguments");
  SE_REQUIRE(ldz >= D && ldE >= D, "leading dimension smaller than D");
  SE_REQUIRE(loss_kind != SE_LOSS_SOFTMAX_CORR || C >= 1, "bad arguments");
  const int Dp = (D + 3) & ~3;
  size_t smem = (size_t)HEAD_WARPS * Dp * sizeof(float);
  SE_REQUIRE(smem <= 48 * 1024, "D too large for the fused head (max 3072)");
  int nwarps = HEAD_WARPS, split = 0;
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  bool vec = (D % 4 == 0) && (ldz % 4 == 0) && (ldE % 4 == 0) && al16(z) && al16(E) && (!x_out || al16(x_out));
  int grid = ceil_div(B, HEAD_WARPS);
  int es_classes = 0;
  const size_t es_bytes = (size_t)C * (D + 1) * sizeof(float);
  // the ranking loss reads the class matrix for its hinge terms and keeps a bit mask of the active classes per row
  const bool rank = loss_kind == SE_LOSS_DEVISE_RANK && (loss || dz);
  const size_t mask_row = rank ? (size_t)((C + 31) / 32) * sizeof(unsigned) : 0;
  const bool need_E = (acc || rank_out || rank) && loss_kind != SE_LOSS_SOFTMAX_CORR;
  if (need_E && smem + es_bytes + HEAD_WARPS * mask_row <= 48 * 1024) {
    es_classes = C; smem += es_bytes + HEAD_WARPS * mask_row;
  } else if (need_E && (size_t)HEAD_WARPS_SPLIT * Dp * sizeof(float) + mask_row <= 48 * 1024) {
    // the class matrix stays in global memory: the loop over it is latency-bound per warp, so a row gets a whole CTA
    split = 1; nwarps = HEAD_WARPS_SPLIT; grid = B; smem = (size_t)HEAD_WARPS_SPLIT * Dp * sizeof(float) + mask_row;
  } else {
    smem += HEAD_WARPS * mask_row;
  }
  SE_REQUIRE(smem <= 48 * 1024, "too many classes for the ranking loss' active-set mask");
  if (vec)
    launch(embed_head_kernel<true>, dim3(grid), dim3(nwarps * 32), smem, as_stream(stream), z, ldz, labels, E, ldE, B, D, C, loss_kind,
           loss_scale, extra_dx, x_out, loss, acc, dz, rank_out, es_classes, split, margin);
  else
    launch(embed_head_kernel<false>, dim3(grid), dim3(nwarps * 32), smem, as_stream(stream), z, ldz, labels, E, ldE, B, D, C, loss_kind,
           loss_scale, extra_dx, x_out, loss, acc, dz, rank_out, es_classes, split, margin);
  return check_launch("embed_head_kernel");
}

extern "C" int se_embed_head_fwd_bwd_ex(const float* z, int ldz, const int32_t* labels, const float* E, int ldE, int B,
                                        int D, int C, int loss_kind, float loss_scale, const float* extra_dx, float* x_out,
                                        float* loss, float* acc, float* dz, float* rank_out, void* stream) {
  SE_REQUIRE(loss_kind >= 0 && loss_kind <= 3, "unknown loss kind");
  return embed_head(z, ldz, labels, E, ldE, B, D, C, loss_kind, loss_scale, extra_dx, x_out, loss, acc, dz, rank_out, 0.f,
                    stream);
}

extern "C" int se_devise_rank_fwd_bwd(const float* z, int ldz, const int32_t* labels, const float* E, int ldE, int B, int D,
                                      int C, int loss_kind, float loss_scale, const float* extra_dx, float* x_out, float* loss,
                                      float* acc, float* dz, float* rank_out, float margin, void* stream) {
  SE_REQUIRE(loss_kind == SE_LOSS_DEVISE_RANK, "se_devise_rank_fwd_bwd computes SE_LOSS_DEVISE_RANK only");
  return embed_head(z, ldz, labels, E, ldE, B, D, C, SE_LOSS_DEVISE_RANK, loss_scale, extra_dx, x_out, loss, acc, dz,
                    rank_out, margin, stream);
}

extern "C" int se_softmax_xent_fwd_bwd(const float* logits, int ld, const int32_t* labels, int B, int C, float scale,
                                       float* prob, float* loss, float* acc, float* dlogits, void* stream) {
  return se_softmax_xent_fwd_bwd_ex(logits, ld, labels, B, C, scale, prob, loss, acc, dlogits, nullptr, stream);
}

extern "C" int se_softmax_xent_fwd_bwd_ex(const float* logits, int ld, const int32_t* labels, int B, int C, float scale,
                                          float* prob, float* loss, float* acc, float* dlogits, float* rank_out, void* stream) {
  SE_REQUIRE(logits && labels && B > 0 && C > 0 && ld >= C, "bad arguments");
  launch(softmax_xent_kernel<false>, dim3(ceil_div(B, HEAD_WARPS)), dim3(HEAD_WARPS * 32), 0, as_stream(stream), logits, ld, labels, B,
         C, scale, prob, loss, acc, dlogits, rank_out, 1.f, 0.f);
  return check_launch("softmax_xent_kernel");
}

extern "C" int se_softmax_xent_smooth_fwd_bwd(const float* logits, int ld, const int32_t* labels, int B, int C,
                                              float smoothing, float scale, float* prob, float* loss, float* acc,
                                              float* dlogits, float* rank_out, void* stream) {
  // learn_classifier.py:20 smooths only for 0 < ls < 1; any other value keeps the one-hot targets
  if (!(smoothing > 0.f && smoothing < 1.f))
    return se_softmax_xent_fwd_bwd_ex(logits, ld, labels, B, C, scale, prob, loss, acc, dlogits, rank_out, stream);
  SE_REQUIRE(logits && labels && B > 0 && C > 1 && ld >= C, "bad arguments (label smoothing needs C >= 2)");
  // Y * (1 - ls) + (1 - Y) * (ls / (C - 1)) on a float32 Y: the factors are formed in double and rounded once
  const float t_hi = (float)(1.0 - (double)smoothing);
  const float t_lo = (float)((double)smoothing / (double)(C - 1));
  launch(softmax_xent_kernel<true>, dim3(ceil_div(B, HEAD_WARPS)), dim3(HEAD_WARPS * 32), 0, as_stream(stream), logits, ld, labels, B,
         C, scale, prob, loss, acc, dlogits, rank_out, t_hi, t_lo);
  return check_launch("softmax_xent_kernel");
}
