// One-vs-rest linear SVM (squared hinge loss, L2 penalty, regularised intercept): the LinearSVC fit of the reference's
// evaluate_classification_accuracy.py:39-41, solved for all classes at once by the trust-region Newton method with
// conjugate-gradient inner steps (Lin, Weng & Keerthi 2008; liblinear's primal solver for L2R_L2LOSS_SVC).  For class c,
// with y_i = +1 on its rows and -1 elsewhere and x~ = [x, 1]:
//   f_c(w~)  = 1/2 |w~|^2 + C sum_i max(0, 1 - y_i w~.x~_i)^2
//   grad f_c = w~ - 2C sum_{i in I} (1 - y_i s_i) y_i x~_i          I = {i : y_i s_i < 1}, s = X w + b
//   H_c v    = v + 2C sum_{i in I} x~_i (x~_i . v)
// Both row sums are the dense-layer kernels: S = X W + b is se_dense_fwd, X^T R with its column sums is the dW / dbias
// of se_dense_bwd (SE_MODE_TF32X3).  The kernels here are the parts between those GEMMs: the hinge pass (residuals and
// per-class objective partials), the masked Hessian pass and the per-class CG / trust-region updates.  Every class owns
// one column of the [D+1, Cp] state matrices; a CTA owns 32 whole columns, so its row sums are private and in a fixed
// order.  No float atomics anywhere, and the weight gradient is only run where it adds its split-K slices in a fixed
// order: reruns give the same bits.
//
// se_scale_features: the feature normalisation of evaluate_classification_accuracy.py:33-38 with numpy's float32 results
// bit for bit (row norms summed in numpy's pairwise order, true division), and the negation of score matrices that lets
// se_row_topk (ascending) rank in descending order.
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace se {

bool conv_wgrad_tc_fixed_order(const se_conv_desc* d, cudaStream_t st);   // conv_wgrad_tc.cu

namespace {

constexpr int SV_COLS = 32;                 // classes per CTA of the per-class kernels (one per lane)
constexpr int SV_THREADS = 1024;            // 32 warps stride the rows of the state matrices
constexpr int SV_WARPS = SV_THREADS / 32;
constexpr int HB_ROWS = 64;                 // rows per CTA of the hinge pass
constexpr int HB_THREADS = 256;

struct SvmClass {
  double f, fnew, gnorm0, gnorm, eps, delta;
  double rtr, cgtol, gs, sr, snorm2, wtn2;
  int active, in_cg, accepted, iters, cg_iters, first_step, pad0, pad1;
};

struct SvmDims {
  int N, Np, Dp, P, C, Cp, nrb, max_cg;
  float penalty;
};

// fixed-order sum over the 32 warps of one value per (warp, lane): result valid in warp 0
__device__ __forceinline__ double cta_col_sum(double v, double (*red)[SV_COLS], int w, int l) {
  __syncthreads();
  red[w][l] = v;
  __syncthreads();
  double s = 0.0;
  if (w == 0) {
    for (int k = 0; k < SV_WARPS; ++k) s += red[k][l];
  }
  return s;
}

__global__ void __launch_bounds__(256) svm_pack_kernel(const float* __restrict__ x, long long ldx, int N, int D, int Np, int Dp,
                                                        float* __restrict__ xp) {
  pdl_grid_sync();
  const long long n = (long long)Np * Dp;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / Dp;
    const int j = (int)(e - i * Dp);
    xp[e] = (i < N && j < D) ? x[i * ldx + j] : 0.f;
  }
}

// counts[c] = rows with label c; bad = 1 when a label lies outside [0, C).  Integer atomics: exact in any order.
__global__ void __launch_bounds__(256) svm_count_kernel(const int32_t* __restrict__ labels, int N, int C, int* counts, int* bad) {
  pdl_grid_sync();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    const int y = labels[i];
    if (y < 0 || y >= C) atomicOr(bad, 1);
    else atomicAdd(&counts[y], 1);
  }
}

__global__ void __launch_bounds__(256) svm_init_kernel(SvmClass* st, const int* counts, SvmDims dm, float tol) {
  pdl_grid_sync();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= dm.Cp) return;
  SvmClass s = {};
  if (c < dm.C) {
    const int pos = counts[c], neg = dm.N - pos;
    s.eps = (double)tol * (double)max(min(pos, neg), 1) / (double)dm.N;   // liblinear's primal tolerance
    s.active = 1;
    s.first_step = 1;
  }
  st[c] = s;
}

// One pass over rows [64 b, 64 b + 64) of a score matrix S [Np, Cp].
//   partial[b, c] = sum_i max(0, 1 - y_ic s_ic)^2 over the CTA's rows (rows in order: warp stride 8, then warps in order)
//   R (when given) = -2C (1 - y s) y on active rows, 0 elsewhere -- the residual whose X^T R + column sums is grad - w~
//   S_new (when given): classes accepted by the last trust-region step take their column from S_new into S first.
__global__ void __launch_bounds__(HB_THREADS) svm_hinge_kernel(float* __restrict__ S, const float* __restrict__ S_new,
                                                               const SvmClass* __restrict__ st, const int32_t* __restrict__ labels,
                                                               SvmDims dm, float* __restrict__ R, double* __restrict__ partial) {
  pdl_grid_sync();
  __shared__ double red[HB_THREADS / 32][32];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const int r0 = blockIdx.x * HB_ROWS;
  for (int c0 = 0; c0 < dm.Cp; c0 += 32) {
    const int c = c0 + l;
    const bool take = S_new && c < dm.Cp && st[c].accepted;
    double acc = 0.0;
    for (int i = r0 + w; i < min(r0 + HB_ROWS, dm.Np); i += HB_THREADS / 32) {
      if (c >= dm.Cp) break;
      const long long o = (long long)i * dm.Cp + c;
      float s = S[o];
      if (take) { s = S_new[o]; S[o] = s; }
      float r = 0.f;
      if (i < dm.N && c < dm.C) {
        const float y = labels[i] == c ? 1.f : -1.f;
        const float m = 1.f - y * s;
        if (m > 0.f) {
          acc += (double)m * (double)m;
          r = -2.f * dm.penalty * m * y;
        }
      }
      if (R) R[o] = r;
    }
    if (partial) {
      __syncthreads();
      red[w][l] = acc;
      __syncthreads();
      if (w == 0 && c < dm.Cp) {
        double s = 0.0;
        for (int k = 0; k < HB_THREADS / 32; ++k) s += red[k][l];
        partial[(long long)blockIdx.x * dm.Cp + c] = s;
      }
    }
  }
}

// T = X V + v_b  ->  2C T on active rows of the current point (the masked Hessian pass), 0 elsewhere (in place)
__global__ void __launch_bounds__(256) svm_hess_mask_kernel(float* __restrict__ T, const float* __restrict__ S,
                                                            const int32_t* __restrict__ labels, SvmDims dm) {
  pdl_grid_sync();
  const long long n = (long long)dm.Np * dm.Cp;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / dm.Cp;
    const int c = (int)(e - i * dm.Cp);
    float v = 0.f;
    if (i < dm.N && c < dm.C) {
      const float y = labels[i] == c ? 1.f : -1.f;
      if (1.f - y * S[e] > 0.f) v = 2.f * dm.penalty * T[e];
    }
    T[e] = v;
  }
}

// Per-class kernels: lane l of every warp works on class c = 32 blockIdx.x + l, warp w on rows w, w + 32, ... of the
// [P, Cp] state matrices (P = Dp + 1 rows: the weights, then the intercept).

// After a gradient GEMM (XtR = X^T R, intercept row = column sums of R): g = w~ + XtR for classes whose point moved (or
// all on the first call, which also sets f, |grad f(0)| and the trust radius), the stopping rule, and the start of the
// next CG solve for every class still active: s = 0, r = -g, d = r.
__global__ void __launch_bounds__(SV_THREADS) svm_newton_kernel(const float* __restrict__ W, const float* __restrict__ XtR,
                                                                float* __restrict__ G, float* __restrict__ Sv,
                                                                float* __restrict__ Rv, float* __restrict__ Dv, SvmClass* st,
                                                                const double* __restrict__ partial, SvmDims dm, int max_iter,
                                                                int* counters) {
  pdl_grid_sync();
  __shared__ double red[SV_WARPS][SV_COLS];
  __shared__ int s_active[SV_COLS];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, c = blockIdx.x * SV_COLS + l;
  const bool valid = c < dm.Cp;
  SvmClass cs = valid ? st[c] : SvmClass{};
  const bool first = cs.first_step != 0;
  // a class that took a step and then stopped on its reductions still gets the gradient of its final point (gnorm)
  const bool moved = (cs.active && first) || cs.accepted;
  double g2 = 0.0, loss = 0.0;
  if (moved) {
    for (int r = w; r < dm.P; r += SV_WARPS) {
      const long long o = (long long)r * dm.Cp + c;
      const float g = W[o] + XtR[o];
      G[o] = g;
      g2 += (double)g * g;
    }
    if (first)
      for (int b = w; b < dm.nrb; b += SV_WARPS) loss += partial[(long long)b * dm.Cp + c];
  }
  g2 = cta_col_sum(g2, red, w, l);
  loss = cta_col_sum(loss, red, w, l);
  if (w == 0) {
    if (moved) {
      cs.gnorm = sqrt(g2);
      if (first) {
        cs.f = (double)dm.penalty * loss;          // w~ = 0
        cs.gnorm0 = cs.gnorm;
        cs.delta = cs.gnorm;
      }
      if (cs.gnorm <= cs.eps * cs.gnorm0) cs.active = 0;
    }
    if (cs.active && cs.iters >= max_iter) cs.active = 0;
    cs.accepted = 0;
    cs.in_cg = cs.active;
    cs.cg_iters = 0;
    if (cs.active) {
      cs.rtr = cs.gnorm * cs.gnorm;
      cs.cgtol = 0.1 * cs.gnorm;
      cs.in_cg = sqrt(cs.rtr) > cs.cgtol;
    }
    s_active[l] = cs.active;
    if (valid) {
      st[c] = cs;
      if (cs.active) atomicAdd(&counters[0], 1);
      if (cs.in_cg) atomicAdd(&counters[1], 1);
    }
  }
  __syncthreads();
  if (valid && s_active[l]) {
    for (int r = w; r < dm.P; r += SV_WARPS) {
      const long long o = (long long)r * dm.Cp + c;
      const float g = G[o];
      Sv[o] = 0.f;
      Rv[o] = -g;
      Dv[o] = -g;
    }
  }
}

// One CG step of every class still in its CG loop (tron.cpp trcg), after the Hessian GEMM: Hd = d + XtR.
//   alpha = r.r / d.Hd; if |s + alpha d| > delta, step to the trust-region boundary along d and leave the loop;
//   s += alpha d; r -= alpha Hd; beta = r'.r' / r.r; d = r + beta d; leave when |r| <= 0.1 |g|.
__global__ void __launch_bounds__(SV_THREADS) svm_cg_kernel(const float* __restrict__ XtR, float* __restrict__ Sv,
                                                            float* __restrict__ Rv, float* __restrict__ Dv, SvmClass* st, SvmDims dm,
                                                            int* counters) {
  pdl_grid_sync();
  __shared__ double red[SV_WARPS][SV_COLS];
  __shared__ float s_alpha[SV_COLS], s_beta[SV_COLS];
  __shared__ int s_more[SV_COLS];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, c = blockIdx.x * SV_COLS + l;
  const bool valid = c < dm.Cp;
  SvmClass cs = valid ? st[c] : SvmClass{};
  const bool go = cs.in_cg != 0;
  double dhd = 0.0, sd = 0.0, ss = 0.0, dd = 0.0;
  if (go) {
    for (int r = w; r < dm.P; r += SV_WARPS) {
      const long long o = (long long)r * dm.Cp + c;
      const float d = Dv[o], s = Sv[o], hd = d + XtR[o];
      dhd += (double)d * hd;
      sd += (double)s * d;
      ss += (double)s * s;
      dd += (double)d * d;
    }
  }
  dhd = cta_col_sum(dhd, red, w, l);
  sd = cta_col_sum(sd, red, w, l);
  ss = cta_col_sum(ss, red, w, l);
  dd = cta_col_sum(dd, red, w, l);
  int boundary = 0;
  if (w == 0) {
    double alpha = 0.0;
    if (go) {
      alpha = cs.rtr / dhd;
      const double sn2 = ss + 2.0 * alpha * sd + alpha * alpha * dd;
      if (sqrt(sn2) > cs.delta) {
        const double dsq = cs.delta * cs.delta, rad = sqrt(sd * sd + dd * (dsq - ss));
        alpha = sd >= 0.0 ? (dsq - ss) / (sd + rad) : (rad - sd) / dd;
        boundary = 1;
      }
    }
    s_alpha[l] = (float)alpha;
    s_more[l] = boundary;            // reused below: 1 = leaves the loop at the boundary
  }
  __syncthreads();
  const float alpha = s_alpha[l];
  double rr = 0.0;
  if (go) {
    for (int r = w; r < dm.P; r += SV_WARPS) {
      const long long o = (long long)r * dm.Cp + c;
      const float d = Dv[o], hd = d + XtR[o];
      Sv[o] = Sv[o] + alpha * d;
      const float rv = Rv[o] - alpha * hd;
      Rv[o] = rv;
      rr += (double)rv * rv;
    }
  }
  rr = cta_col_sum(rr, red, w, l);
  if (w == 0) {
    int more = 0;
    float beta = 0.f;
    if (go) {
      cs.cg_iters += 1;
      if (!s_more[l]) {
        beta = (float)(rr / cs.rtr);
        cs.rtr = rr;
        more = sqrt(rr) > cs.cgtol && cs.cg_iters < dm.max_cg;
      }
      cs.in_cg = more;
      st[c] = cs;
      if (more) atomicAdd(&counters[1], 1);
    }
    s_beta[l] = beta;
    s_more[l] = more;
  }
  __syncthreads();
  if (go && s_more[l]) {
    const float beta = s_beta[l];
    for (int r = w; r < dm.P; r += SV_WARPS) {
      const long long o = (long long)r * dm.Cp + c;
      Dv[o] = Rv[o] + beta * Dv[o];
    }
  }
}

// Trial point of every active class: wt = w + s, and the dot products of the trust-region test (g.s, s.r, |s|^2, |wt|^2).
// Other classes keep wt = w.
__global__ void __launch_bounds__(SV_THREADS) svm_trial_kernel(const float* __restrict__ W, const float* __restrict__ G,
                                                               const float* __restrict__ Sv, const float* __restrict__ Rv,
                                                               float* __restrict__ Wt, SvmClass* st, SvmDims dm) {
  pdl_grid_sync();
  __shared__ double red[SV_WARPS][SV_COLS];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, c = blockIdx.x * SV_COLS + l;
  const bool valid = c < dm.Cp;
  const bool go = valid && st[c].active;
  double gs = 0.0, sr = 0.0, s2 = 0.0, t2 = 0.0;
  if (valid) {
    for (int r = w; r < dm.P; r += SV_WARPS) {
      const long long o = (long long)r * dm.Cp + c;
      if (go) {
        const float s = Sv[o], wt = W[o] + s;
        Wt[o] = wt;
        gs += (double)G[o] * s;
        sr += (double)s * Rv[o];
        s2 += (double)s * s;
        t2 += (double)wt * wt;
      } else {
        Wt[o] = W[o];
      }
    }
  }
  gs = cta_col_sum(gs, red, w, l);
  sr = cta_col_sum(sr, red, w, l);
  s2 = cta_col_sum(s2, red, w, l);
  t2 = cta_col_sum(t2, red, w, l);
  if (w == 0 && go) {
    st[c].gs = gs;
    st[c].sr = sr;
    st[c].snorm2 = s2;
    st[c].wtn2 = t2;
  }
}

// Trust-region test of the trial point (tron.cpp): f(wt) from the hinge partials, actual against predicted reduction,
// the new radius, and w = wt when the step is taken.  A class also stops when its reductions vanish.
__global__ void __launch_bounds__(SV_THREADS) svm_tr_kernel(const float* __restrict__ Wt, float* __restrict__ W, SvmClass* st,
                                                            const double* __restrict__ partial, SvmDims dm) {
  pdl_grid_sync();
  __shared__ double red[SV_WARPS][SV_COLS];
  __shared__ int s_take[SV_COLS];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, c = blockIdx.x * SV_COLS + l;
  const bool valid = c < dm.Cp;
  SvmClass cs = valid ? st[c] : SvmClass{};
  const bool go = cs.active != 0;
  double loss = 0.0;
  if (go)
    for (int b = w; b < dm.nrb; b += SV_WARPS) loss += partial[(long long)b * dm.Cp + c];
  loss = cta_col_sum(loss, red, w, l);
  if (w == 0) {
    int take = 0;
    if (go) {
      constexpr double eta0 = 1e-4, eta1 = 0.25, eta2 = 0.75, sigma1 = 0.25, sigma2 = 0.5, sigma3 = 4.0;
      const double fnew = 0.5 * cs.wtn2 + (double)dm.penalty * loss;
      const double prered = -0.5 * (cs.gs - cs.sr), actred = cs.f - fnew, snorm = sqrt(cs.snorm2);
      if (cs.iters == 0) cs.delta = fmin(cs.delta, snorm);
      const double q = fnew - cs.f - cs.gs;
      const double alpha = q <= 0.0 ? sigma3 : fmax(sigma1, -0.5 * (cs.gs / q));
      if (actred < eta0 * prered) cs.delta = fmin(fmax(alpha, sigma1) * snorm, sigma2 * cs.delta);
      else if (actred < eta1 * prered) cs.delta = fmax(sigma1 * cs.delta, fmin(alpha * snorm, sigma2 * cs.delta));
      else if (actred < eta2 * prered) cs.delta = fmax(sigma1 * cs.delta, fmin(alpha * snorm, sigma3 * cs.delta));
      else cs.delta = fmax(cs.delta, fmin(alpha * snorm, sigma3 * cs.delta));
      if (actred > eta0 * prered) {
        take = 1;
        cs.iters += 1;
        cs.f = fnew;
      }
      if (cs.f < -1.0e32) cs.active = 0;
      else if (fabs(actred) <= 0.0 && prered <= 0.0) cs.active = 0;
      else if (fabs(actred) <= 1.0e-12 * fabs(cs.f) && fabs(prered) <= 1.0e-12 * fabs(cs.f)) cs.active = 0;
      cs.accepted = take;
      cs.first_step = 0;
      st[c] = cs;
    }
    s_take[l] = take;
  }
  __syncthreads();
  if (valid && s_take[l])
    for (int r = w; r < dm.P; r += SV_WARPS) {
      const long long o = (long long)r * dm.Cp + c;
      W[o] = Wt[o];
    }
}

__global__ void __launch_bounds__(256) svm_out_kernel(const float* __restrict__ Wv, const SvmClass* __restrict__ st, SvmDims dm,
                                                      int D, float* __restrict__ W, float* __restrict__ b,
                                                      int32_t* __restrict__ iters, float* __restrict__ gnorm) {
  pdl_grid_sync();
  const long long n = (long long)D * dm.C;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n + dm.C; e += (long long)gridDim.x * blockDim.x) {
    if (e < n) {
      const long long j = e / dm.C;
      const int c = (int)(e - j * dm.C);
      W[e] = Wv[j * dm.Cp + c];
    } else {
      const int c = (int)(e - n);
      if (b) b[c] = Wv[(long long)dm.Dp * dm.Cp + c];
      if (iters) iters[c] = st[c].iters;
      if (gnorm) gnorm[c] = st[c].gnorm0 > 0.0 ? (float)(st[c].gnorm / st[c].gnorm0) : 0.f;
    }
  }
}

// ---------------------------------------------------------------------------------------- feature scaling
// numpy's pairwise summation of float32 (pairwise_sum_FLOAT) over x_j * x_j, as np.linalg.norm(X, axis=-1) computes it:
// ranges of <= 128 elements are summed with eight accumulators, longer ones are cut in two halves at a multiple of 8 and
// the halves' sums added.  The recursion runs on an explicit stack (depth <= 24 for any int length).
__device__ __forceinline__ float np_block_sq(const float* a, int n) {
  if (n < 8) {
    float r = 0.f;
    for (int i = 0; i < n; ++i) r = __fadd_rn(r, __fmul_rn(a[i], a[i]));
    return r;
  }
  float r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = __fmul_rn(a[j], a[j]);
  int i = 8;
  for (; i < n - (n % 8); i += 8)
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], __fmul_rn(a[i + j], a[i + j]));
  float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])), __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __fadd_rn(res, __fmul_rn(a[i], a[i]));
  return res;
}

__device__ float np_pairwise_sq(const float* a, int n0) {
  int off[32], len[32], stage[32];
  float left[32];
  int sp = 0;
  off[0] = 0;
  len[0] = n0;
  float ret = 0.f;
  bool have = false;                       // ret holds the sum of frame sp
  for (;;) {
    if (!have) {
      const int n = len[sp];
      if (n <= 128) { ret = np_block_sq(a + off[sp], n); have = true; continue; }
      const int n2 = n / 2 - (n / 2) % 8;
      stage[sp] = 1;
      off[sp + 1] = off[sp];
      len[sp + 1] = n2;
      ++sp;
      continue;
    }
    if (sp == 0) return ret;
    --sp;
    if (stage[sp] == 1) {                  // left half done: keep it, sum the right half
      left[sp] = ret;
      stage[sp] = 2;
      const int n = len[sp], n2 = n / 2 - (n / 2) % 8;
      off[sp + 1] = off[sp] + n2;
      len[sp + 1] = n - n2;
      ++sp;
      have = false;
    } else {
      ret = __fadd_rn(left[sp], ret);
    }
  }
}

__global__ void __launch_bounds__(128) scale_rows_l2_kernel(const float* x, long long ldx, int rows, int D, float* y, long long ldy) {
  pdl_grid_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  const float* xr = x + i * ldx;
  const float nrm = __fsqrt_rn(np_pairwise_sq(xr, D));
  float* yr = y + i * ldy;
  for (int j = 0; j < D; ++j) yr[j] = __fdiv_rn(xr[j], nrm);
}

// colmax[j] = max_i |x_ij| (non-negative floats order like their bit patterns: an integer max is exact in any order)
__global__ void __launch_bounds__(256) scale_col_maxabs_kernel(const float* __restrict__ x, long long ldx, int rows, int D,
                                                               unsigned int* __restrict__ colmax) {
  pdl_grid_sync();
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  if (j >= D) return;
  float m = 0.f;
  for (int i = blockIdx.y * 8 + (threadIdx.x >> 5); i < rows; i += gridDim.y * 8) m = fmaxf(m, fabsf(x[(long long)i * ldx + j]));
  atomicMax(&colmax[j], __float_as_uint(m));
}

__global__ void __launch_bounds__(256) scale_cols_kernel(const float* x, long long ldx, int rows, int D, const float* __restrict__ colmax,
                                                         float scale, float* y, long long ldy) {
  pdl_grid_sync();
  const long long n = (long long)rows * D;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / D;
    const int j = (int)(e - i * D);
    const float v = x[i * ldx + j];
    y[i * ldy + j] = colmax ? __fdiv_rn(v, fmaxf(1e-8f, colmax[j])) : __fmul_rn(scale, v);
  }
}

inline long long align_up(long long v, long long a) { return (v + a - 1) / a * a; }

struct SvmLayout {
  SvmDims dm;
  long long off_xp, off_scur, off_strial, off_r, off_vec[7], off_partial, off_state, off_counts, off_ctr, total;
};

SvmLayout svm_layout(int N, int D, int C) {
  SvmLayout L = {};
  SvmDims& d = L.dm;
  d.N = N;
  d.Np = std::max(N, 32);                             // the tensor-core weight gradient wants >= 32 rows
  d.Dp = (int)align_up(D, 4);                    // float4 rows of X
  d.P = d.Dp + 1;
  d.C = C;
  d.Cp = (int)align_up(C, 16);                   // output-channel tiles of the weight gradient
  d.nrb = (d.Np + HB_ROWS - 1) / HB_ROWS;
  d.max_cg = 2 * d.P;
  long long o = 0;
  auto take = [&](long long bytes) { const long long at = o; o = align_up(o + bytes, 256); return at; };
  L.off_xp = take((long long)d.Np * d.Dp * 4);
  L.off_scur = take((long long)d.Np * d.Cp * 4);
  L.off_strial = take((long long)d.Np * d.Cp * 4);
  L.off_r = take((long long)d.Np * d.Cp * 4);
  for (int k = 0; k < 7; ++k) L.off_vec[k] = take((long long)d.P * d.Cp * 4);
  L.off_partial = take((long long)d.nrb * d.Cp * 8);
  L.off_state = take((long long)d.Cp * sizeof(SvmClass));
  L.off_counts = take((long long)d.Cp * 4 + 4);
  L.off_ctr = take(16);
  L.total = o;
  return L;
}

int grid_for(long long n, int threads) { return (int)std::min<long long>(std::max<long long>(1, (n + threads - 1) / threads), 8LL * sm_count()); }

}  // namespace
}  // namespace se

using namespace se;

extern "C" int64_t se_linear_svm_workspace_bytes(int N, int D, int C) {
  if (N <= 0 || D <= 0 || C <= 0) return 0;
  return svm_layout(N, D, C).total;
}

extern "C" int se_linear_svm_fit(const float* X, int64_t ldx, int N, int D, const int32_t* labels, int C, float penalty, float tol,
                                 int max_iter, float* W, float* b, int32_t* iters, float* gnorm, void* workspace, void* stream) {
  SE_REQUIRE(X && labels && W && workspace, "null pointer");
  SE_REQUIRE(N > 0 && D > 0 && C > 0 && ldx >= D, "N, D, C > 0 and ldx >= D");
  SE_REQUIRE(penalty > 0.f && tol > 0.f && max_iter > 0, "penalty > 0, tol > 0, max_iter > 0");
  SE_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256-byte aligned");
  const SvmLayout L = svm_layout(N, D, C);
  SvmDims dm = L.dm;
  dm.penalty = penalty;
  SE_REQUIRE((long long)dm.Np * dm.Cp < (1LL << 31) && (long long)dm.Np * dm.Dp < (1LL << 31), "N x D and N x C must stay below 2^31");
  cudaStream_t st = as_stream(stream);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) {
    se::set_error("se_linear_svm_fit: the solver synchronises with its stream and cannot be captured");
    return SE_ERR_ARG;
  }
  // the gradient / Hessian sums X^T R must add their split-K slices in a fixed order (no float atomics)
  se_conv_desc gd = {dm.Np, 1, 1, dm.Dp, dm.Cp, 1, 1, 1, 0, 0, 1, 1};
  if (!conv_wgrad_tc_fixed_order(&gd, st)) {
    se::set_error("se_linear_svm_fit: (D+1) x C = %d x %d does not fit the fixed-order weight-gradient workspace", dm.Dp, dm.Cp);
    return SE_ERR_UNSUPPORTED;
  }
  char* ws = static_cast<char*>(workspace);
  float* xp = reinterpret_cast<float*>(ws + L.off_xp);
  float* s_cur = reinterpret_cast<float*>(ws + L.off_scur);
  float* s_trial = reinterpret_cast<float*>(ws + L.off_strial);
  float* R = reinterpret_cast<float*>(ws + L.off_r);
  float* Wv = reinterpret_cast<float*>(ws + L.off_vec[0]);
  float* Wt = reinterpret_cast<float*>(ws + L.off_vec[1]);
  float* G = reinterpret_cast<float*>(ws + L.off_vec[2]);
  float* Sv = reinterpret_cast<float*>(ws + L.off_vec[3]);
  float* Rv = reinterpret_cast<float*>(ws + L.off_vec[4]);
  float* Dv = reinterpret_cast<float*>(ws + L.off_vec[5]);
  float* XtR = reinterpret_cast<float*>(ws + L.off_vec[6]);
  double* partial = reinterpret_cast<double*>(ws + L.off_partial);
  SvmClass* state = reinterpret_cast<SvmClass*>(ws + L.off_state);
  int* counts = reinterpret_cast<int*>(ws + L.off_counts);
  int* bad = counts + dm.Cp;
  int* ctr = reinterpret_cast<int*>(ws + L.off_ctr);
  const long long vec_bytes = (long long)dm.P * dm.Cp * 4;
  const long long wdw = (long long)dm.Dp * dm.Cp;               // intercept row offset
  const int cls_blocks = (dm.Cp + SV_COLS - 1) / SV_COLS;
  int rc = SE_OK;
#define SV_CHECK(call)           \
  do {                           \
    if ((rc = (call)) != SE_OK) return rc; \
  } while (0)
#define SV_CUDA(call, what)                                                   \
  do {                                                                        \
    cudaError_t e_ = (call);                                                  \
    if (e_ != cudaSuccess) { se::set_error("%s: %s", what, cudaGetErrorString(e_)); return SE_ERR_CUDA; } \
  } while (0)

  // gradient sums: XtR = X^T R (rows < Dp), column sums of R (intercept row)
  auto xt_r = [&](const float* Rm) -> int {
    if (cudaMemsetAsync(XtR, 0, vec_bytes, st) != cudaSuccess) { se::set_error("se_linear_svm_fit: memset"); return SE_ERR_CUDA; }
    return se_dense_bwd(xp, nullptr, Rm, nullptr, 0.f, XtR, XtR + wdw, dm.Np, dm.Dp, dm.Cp, SE_MODE_TF32X3, stream);
  };
  auto read_counters = [&](int* host) -> int {
    SV_CUDA(cudaMemcpyAsync(host, ctr, 2 * sizeof(int), cudaMemcpyDeviceToHost, st), "se_linear_svm_fit: counters");
    SV_CUDA(cudaStreamSynchronize(st), "se_linear_svm_fit");
    return SE_OK;
  };

  SV_CUDA(cudaMemsetAsync(counts, 0, (size_t)dm.Cp * 4 + 4, st), "se_linear_svm_fit: memset");
  for (int k = 0; k < 7; ++k) SV_CUDA(cudaMemsetAsync(ws + L.off_vec[k], 0, vec_bytes, st), "se_linear_svm_fit: memset");
  SV_CUDA(cudaMemsetAsync(s_cur, 0, (size_t)dm.Np * dm.Cp * 4, st), "se_linear_svm_fit: memset");
  launch(svm_pack_kernel, dim3(grid_for((long long)dm.Np * dm.Dp, 256)), dim3(256), 0, st, X, (long long)ldx, N, D, dm.Np, dm.Dp, xp);
  SV_CHECK(check_launch("svm_pack_kernel"));
  launch(svm_count_kernel, dim3(grid_for(N, 256)), dim3(256), 0, st, labels, N, C, counts, bad);
  SV_CHECK(check_launch("svm_count_kernel"));
  int host_bad = 0;
  SV_CUDA(cudaMemcpyAsync(&host_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st), "se_linear_svm_fit: labels");
  SV_CUDA(cudaStreamSynchronize(st), "se_linear_svm_fit");
  if (host_bad) { se::set_error("se_linear_svm_fit: a label lies outside [0, C)"); return SE_ERR_ARG; }
  launch(svm_init_kernel, dim3((dm.Cp + 255) / 256), dim3(256), 0, st, state, (const int*)counts, dm, tol);
  SV_CHECK(check_launch("svm_init_kernel"));

  // w~ = 0: S = 0, f = C N, the first gradient
  launch(svm_hinge_kernel, dim3(dm.nrb), dim3(HB_THREADS), 0, st, s_cur, (const float*)nullptr, (const SvmClass*)state, labels, dm, R,
         partial);
  SV_CHECK(check_launch("svm_hinge_kernel"));
  SV_CHECK(xt_r(R));
  int host[2] = {0, 0};
  for (;;) {
    SV_CUDA(cudaMemsetAsync(ctr, 0, 16, st), "se_linear_svm_fit: memset");
    launch(svm_newton_kernel, dim3(cls_blocks), dim3(SV_THREADS), 0, st, (const float*)Wv, (const float*)XtR, G, Sv, Rv, Dv, state,
           (const double*)partial, dm, max_iter, ctr);
    SV_CHECK(check_launch("svm_newton_kernel"));
    SV_CHECK(read_counters(host));
    if (host[0] == 0) break;
    // conjugate gradient on H s = -g inside the trust region, one Hessian product per step for all classes
    while (host[1] > 0) {
      SV_CHECK(se_dense_fwd(xp, Dv, Dv + wdw, R, dm.Np, dm.Dp, dm.Cp, 0, nullptr, SE_MODE_TF32X3, stream));
      launch(svm_hess_mask_kernel, dim3(grid_for((long long)dm.Np * dm.Cp, 256)), dim3(256), 0, st, R, (const float*)s_cur, labels, dm);
      SV_CHECK(check_launch("svm_hess_mask_kernel"));
      SV_CHECK(xt_r(R));
      SV_CUDA(cudaMemsetAsync(ctr, 0, 16, st), "se_linear_svm_fit: memset");
      launch(svm_cg_kernel, dim3(cls_blocks), dim3(SV_THREADS), 0, st, (const float*)XtR, Sv, Rv, Dv, state, dm, ctr);
      SV_CHECK(check_launch("svm_cg_kernel"));
      SV_CHECK(read_counters(host));
    }
    // trial point, its objective, the trust-region test; the gradient at the classes' new points
    launch(svm_trial_kernel, dim3(cls_blocks), dim3(SV_THREADS), 0, st, (const float*)Wv, (const float*)G, (const float*)Sv,
           (const float*)Rv, Wt, state, dm);
    SV_CHECK(check_launch("svm_trial_kernel"));
    SV_CHECK(se_dense_fwd(xp, Wt, Wt + wdw, s_trial, dm.Np, dm.Dp, dm.Cp, 0, nullptr, SE_MODE_TF32X3, stream));
    launch(svm_hinge_kernel, dim3(dm.nrb), dim3(HB_THREADS), 0, st, s_trial, (const float*)nullptr, (const SvmClass*)state, labels, dm,
           (float*)nullptr, partial);
    SV_CHECK(check_launch("svm_hinge_kernel"));
    launch(svm_tr_kernel, dim3(cls_blocks), dim3(SV_THREADS), 0, st, (const float*)Wt, Wv, state, (const double*)partial, dm);
    SV_CHECK(check_launch("svm_tr_kernel"));
    launch(svm_hinge_kernel, dim3(dm.nrb), dim3(HB_THREADS), 0, st, s_cur, (const float*)s_trial, (const SvmClass*)state, labels, dm,
           R, (double*)nullptr);
    SV_CHECK(check_launch("svm_hinge_kernel"));
    SV_CHECK(xt_r(R));
  }
  launch(svm_out_kernel, dim3(grid_for((long long)D * C + C, 256)), dim3(256), 0, st, (const float*)Wv, (const SvmClass*)state, dm, D,
         W, b, iters, gnorm);
  SV_CHECK(check_launch("svm_out_kernel"));
  SV_CUDA(cudaStreamSynchronize(st), "se_linear_svm_fit");
#undef SV_CHECK
#undef SV_CUDA
  return SE_OK;
}

extern "C" int se_scale_features(const float* x, int64_t ldx, int rows, int D, int op, float* colmax, float scale, float* y,
                                 int64_t ldy, void* stream) {
  SE_REQUIRE(x && rows > 0 && D > 0 && ldx >= D, "x, rows > 0, D > 0, ldx >= D");
  cudaStream_t st = as_stream(stream);
  switch (op) {
    case SE_SCALE_ROW_L2:
      SE_REQUIRE(y && ldy >= D, "y, ldy >= D");
      launch(scale_rows_l2_kernel, dim3((rows + 127) / 128), dim3(128), 0, st, x, (long long)ldx, rows, D, y, (long long)ldy);
      return check_launch("scale_rows_l2_kernel");
    case SE_SCALE_COL_MAXABS: {
      SE_REQUIRE(colmax, "colmax");
      if (cudaMemsetAsync(colmax, 0, (size_t)D * 4, st) != cudaSuccess) { se::set_error("se_scale_features: memset"); return SE_ERR_CUDA; }
      const int gy = std::min((rows + 63) / 64, 1024);
      launch(scale_col_maxabs_kernel, dim3((D + 31) / 32, gy), dim3(256), 0, st, x, (long long)ldx, rows, D,
             reinterpret_cast<unsigned int*>(colmax));
      return check_launch("scale_col_maxabs_kernel");
    }
    case SE_SCALE_COL_DIV:
    case SE_SCALE_MUL:
      SE_REQUIRE(y && ldy >= D && (op == SE_SCALE_MUL || colmax), "y, ldy >= D, colmax for SE_SCALE_COL_DIV");
      launch(scale_cols_kernel, dim3(grid_for((long long)rows * D, 256)), dim3(256), 0, st, x, (long long)ldx, rows, D,
             (const float*)(op == SE_SCALE_COL_DIV ? colmax : nullptr), scale, y, (long long)ldy);
      return check_launch("scale_cols_kernel");
    default:
      se::set_error("se_scale_features: op must be SE_SCALE_ROW_L2, SE_SCALE_COL_MAXABS, SE_SCALE_COL_DIV or SE_SCALE_MUL");
      return SE_ERR_ARG;
  }
}
