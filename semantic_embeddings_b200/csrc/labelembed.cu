// The loss of the label embedding network (Sun et al.; learn_labelembedding.py:21-56) and its backward pass, in two
// launches without float atomics:
//
//   labelembed_row_kernel     one warp per sample: the softmaxes of out1, out2, out2 / tau and of the sample's row of the
//                             label-embedding table, Keras' clipped sparse cross-entropies, argmax(out1) (accuracy) and
//                             argmax(out2) (the mask), the gradients with respect to out1 and out2, and -- into the
//                             workspace -- the per-row terms and the direction of the table's gradient
//   labelembed_finish_kernel  the batch reduction the loss depends on: F = B_eff / (sum mask + 1e-8), the per-sample loss,
//                             and one CTA per class row of the table's gradient, which sums its samples in row order
//
// Replaces labelembed_loss (learn_labelembedding.py:21-37) + TF autodiff, with out2's input and q2, s, mask behind
// stop_gradient.  Rows whose label lies outside [0, C) (label < 0: padding) take no part in anything.
#include <float.h>
#include <limits.h>

#include "common.cuh"

namespace se {

constexpr int LE_WARPS = 4;
constexpr int LE_FIN_THREADS = 128;
constexpr int LE_MAX_B = 8192;          // the finish kernel keeps one row index per sample in shared memory

// first maximum over the warp (np.argmax / tf.argmax: lowest index on ties)
__device__ __forceinline__ void warp_argmax(float& m, int& a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const int oa = __shfl_xor_sync(0xffffffffu, a, o);
    if (om > m || (om == m && oa < a)) { m = om; a = oa; }
  }
}

// Workspace: [B] float4 {mask, CE(q2, softmax(tar)), beta L_o1_y + (1-beta) L_o1_emb + L_o2_y, L_re} |
//            [B][gp] float  softmax(tar) * sum q2 - q2   (only when the table's gradient is wanted) |
//            [B] int        label if mask else -1
__host__ __device__ inline int le_pitch(int C) { return (C + 3) & ~3; }

__global__ void __launch_bounds__(LE_WARPS * 32)
labelembed_row_kernel(const float* __restrict__ out1, const float* __restrict__ out2, int ld, const int* __restrict__ labels,
                      const float* __restrict__ emb, int ldE, int B, int C, float tau, float alpha, float beta, float scale,
                      float* __restrict__ acc, float* __restrict__ d_out1, float* __restrict__ d_out2,
                      float4* __restrict__ terms, float* __restrict__ g_rows, int* __restrict__ key) {
  pdl_grid_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * LE_WARPS + warp;
  if (row >= B) return;
  const long long ro = (long long)row * ld;
  const int lab = labels[row];
  if (lab < 0 || lab >= C) {                     // padding
    for (int i = lane; i < C; i += 32) {
      if (d_out1) d_out1[ro + i] = 0.f;
      if (d_out2) d_out2[ro + i] = 0.f;
    }
    if (lane == 0) {
      terms[row] = make_float4(0.f, 0.f, 0.f, 0.f);
      key[row] = -1;
      if (acc) acc[row] = 0.f;
    }
    return;
  }
  const float* a = out1 + ro;
  const float* b = out2 + ro;
  const float* t = emb + (long long)lab * ldE;

  // ---- maxima (and the arg-max of out1 / out2)
  float m1 = -FLT_MAX, m2 = -FLT_MAX, mt = -FLT_MAX;
  int a1 = INT_MAX, a2 = INT_MAX;
  for (int i = lane; i < C; i += 32) {
    const float v1 = a[i], v2 = b[i];
    if (v1 > m1) { m1 = v1; a1 = i; }
    if (v2 > m2) { m2 = v2; a2 = i; }
    mt = fmaxf(mt, t[i]);
  }
  warp_argmax(m1, a1);
  warp_argmax(m2, a2);
  mt = warp_max(mt);
  const float m2t = m2 / tau;                    // max(out2 / tau): the division is monotone

  // ---- softmax denominators of out1, out2, out2 / tau and tar
  float s1 = 0.f, s2 = 0.f, sq = 0.f, st = 0.f;
  for (int i = lane; i < C; i += 32) {
    s1 += expf(a[i] - m1);
    s2 += expf(b[i] - m2);
    sq += expf(b[i] / tau - m2t);
    st += expf(t[i] - mt);
  }
  s1 = warp_sum(s1); s2 = warp_sum(s2); sq = warp_sum(sq); st = warp_sum(st);
  const float i1 = 1.f / s1, i2 = 1.f / s2, iq = 1.f / sq, it = 1.f / st;
  const float lse1 = logf(s1), lset = logf(st);

  // ---- Keras sparse_categorical_crossentropy on probabilities: c = clip(p, 1e-7, 1 - 1e-7),
  //      loss = -log c_y + log sum_j c_j (TF's sparse softmax cross-entropy on log c); tf.clip_by_value passes the
  //      gradient where lo <= p <= hi
  const float lo = 1e-7f, hi = 1.f - 1e-7f;
  float c1s = 0.f, c2s = 0.f, l1p = 0.f, l2p = 0.f, ssum = 0.f, qsum = 0.f, ce1 = 0.f, cet = 0.f;
  for (int i = lane; i < C; i += 32) {
    const float p1 = expf(a[i] - m1) * i1, p2 = expf(b[i] - m2) * i2;
    const float q = expf(b[i] / tau - m2t) * iq, s = expf(t[i] - mt) * it;
    c1s += fminf(fmaxf(p1, lo), hi);
    c2s += fminf(fmaxf(p2, lo), hi);
    if (p1 >= lo && p1 <= hi) l1p += p1;
    if (p2 >= lo && p2 <= hi) l2p += p2;
    ssum += s;
    qsum += q;
    ce1 = fmaf(s, (a[i] - m1) - lse1, ce1);      // sum_j s_j log_softmax(out1)_j
    cet = fmaf(q, (t[i] - mt) - lset, cet);      // sum_j q2_j log_softmax(tar)_j
  }
  c1s = warp_sum(c1s); c2s = warp_sum(c2s); l1p = warp_sum(l1p); l2p = warp_sum(l2p);
  ssum = warp_sum(ssum); qsum = warp_sum(qsum); ce1 = warp_sum(ce1); cet = warp_sum(cet);

  const float p1y = expf(a[lab] - m1) * i1, p2y = expf(b[lab] - m2) * i2;
  const bool live1 = p1y >= lo && p1y <= hi, live2 = p2y >= lo && p2y <= hi;
  const float L1 = -logf(fminf(fmaxf(p1y, lo), hi)) + logf(c1s);
  const float L2 = -logf(fminf(fmaxf(p2y, lo), hi)) + logf(c2s);
  const float bm = 1.f - beta;
  const float partial = beta * L1 + bm * (-ce1) + L2;
  const float Lre = fmaxf(p2y - alpha, 0.f);
  const bool re_on = p2y > alpha;                // TF's relu gradient is 0 at 0
  const bool mask = a2 == lab;
  if (lane == 0) {
    terms[row] = make_float4(mask ? 1.f : 0.f, -cet, partial, Lre);
    key[row] = mask ? lab : -1;
    if (acc) acc[row] = (a1 == lab) ? 1.f : 0.f;
  }

  // ---- gradients.  Sparse CE through the clip and the softmax:
  //      dL/dz_k = p_k (live_k / S + r - P / S) - [k = y] r,  S = sum_j c_j, P = sum_j live_j p_j, r = live_y
  const float r1 = live1 ? 1.f : 0.f, r2 = live2 ? 1.f : 0.f;
  const float ic1 = 1.f / c1s, ic2 = 1.f / c2s;
  const float A1 = r1 - l1p * ic1, A2 = r2 - l2p * ic2;
  float* g = g_rows ? g_rows + (long long)row * le_pitch(C) : nullptr;
  for (int i = lane; i < C; i += 32) {
    const float p1 = expf(a[i] - m1) * i1, p2 = expf(b[i] - m2) * i2;
    const float q = expf(b[i] / tau - m2t) * iq, s = expf(t[i] - mt) * it;
    const bool y = i == lab;
    if (d_out1) {
      const float dl1 = p1 * (((p1 >= lo && p1 <= hi) ? ic1 : 0.f) + A1) - (y ? r1 : 0.f);
      d_out1[ro + i] = scale * (beta * dl1 + bm * (p1 * ssum - s));
    }
    if (d_out2) {
      const float dl2 = p2 * (((p2 >= lo && p2 <= hi) ? ic2 : 0.f) + A2) - (y ? r2 : 0.f);
      const float dre = re_on ? p2y * ((y ? 1.f : 0.f) - p2) : 0.f;
      d_out2[ro + i] = scale * (dl2 + dre);
    }
    if (g) g[i] = s * qsum - q;                  // d CE(q2, softmax(tar)) / d tar
  }
}

__global__ void __launch_bounds__(LE_FIN_THREADS)
labelembed_finish_kernel(const int* __restrict__ labels, int B, int C, float scale, const float4* __restrict__ terms,
                         const float* __restrict__ g_rows, const int* __restrict__ key, float* __restrict__ loss,
                         float* __restrict__ d_emb, int ldE) {
  pdl_grid_sync();
  extern __shared__ int s_rows[];               // the masked samples of this CTA's class, in increasing order
  __shared__ int s_n[3];
  const int tid = threadIdx.x, lane = tid & 31;
  const int c = blockIdx.x;
  if (tid < 32) {
    // every CTA walks all rows in the same order with integer counts: the same F everywhere
    int nb = 0, nm = 0, nc = 0;
    for (int i0 = 0; i0 < B; i0 += 32) {
      const int i = i0 + lane;
      const int l = i < B ? labels[i] : -1, k = i < B ? key[i] : -1;
      nb += __popc(__ballot_sync(0xffffffffu, l >= 0 && l < C));
      nm += __popc(__ballot_sync(0xffffffffu, k >= 0));
      if (d_emb) {
        const unsigned mine = __ballot_sync(0xffffffffu, k == c);
        if (k == c) s_rows[nc + __popc(mine & ((1u << lane) - 1u))] = i;
        nc += __popc(mine);
      }
    }
    if (lane == 0) { s_n[0] = nb; s_n[1] = nm; s_n[2] = nc; }
  }
  __syncthreads();
  // learn_labelembedding.py:34, in float32: cast(batch size) / (sum(mask) + 1e-8) over the real rows
  const float F = (float)s_n[0] / ((float)s_n[1] + 1e-8f);
  if (loss) {
    for (int i = blockIdx.x * blockDim.x + tid; i < B; i += gridDim.x * blockDim.x) {
      const float4 r = terms[i];
      loss[i] = (r.z + (r.y * r.x) * F) + r.w;  // ((beta L1 + (1-beta) L_emb + L2) + L_emb_o2) + L_re
    }
  }
  if (d_emb && c < C) {
    const int n = s_n[2];
    const int gp = le_pitch(C);
    const float sf = scale * F;
    for (int j = tid; j < C; j += blockDim.x) {
      float s = 0.f;
      for (int k = 0; k < n; ++k) s += g_rows[(long long)s_rows[k] * gp + j];
      d_emb[(long long)c * ldE + j] = sf * s;
    }
  }
}

static size_t le_terms_bytes(int B) { return (size_t)B * sizeof(float4); }
static size_t le_grad_bytes(int B, int C) { return (size_t)B * le_pitch(C) * sizeof(float); }

}  // namespace se

using namespace se;

extern "C" int64_t se_labelembed_workspace_bytes(int B, int C) {
  if (B <= 0 || C <= 0) return SE_ERR_ARG;
  return (int64_t)((le_terms_bytes(B) + le_grad_bytes(B, C) + (size_t)B * sizeof(int) + 15) & ~(size_t)15);
}

extern "C" int se_labelembed_fwd_bwd(const float* out1, const float* out2, int ld, const int32_t* labels, const float* emb,
                                     int ldE, int B, int C, float tau, float alpha, float beta, float scale, float* loss,
                                     float* acc, float* d_out1, float* d_out2, float* d_emb, void* work, void* stream) {
  SE_REQUIRE(out1 && out2 && labels && emb && work, "null pointer");
  SE_REQUIRE(B > 0 && B <= LE_MAX_B, "batch size outside 1..8192");
  SE_REQUIRE(C >= 2 && ld >= C && ldE >= C, "need C >= 2, ld >= C and ldE >= C");
  SE_REQUIRE(tau > 0.f && tau <= FLT_MAX, "the temperature must be positive and finite");
  SE_REQUIRE((reinterpret_cast<uintptr_t>(work) & 15) == 0, "the workspace must be 16-byte aligned");
  char* w = static_cast<char*>(work);
  float4* terms = reinterpret_cast<float4*>(w);
  float* g_rows = reinterpret_cast<float*>(w + le_terms_bytes(B));
  int* key = reinterpret_cast<int*>(w + le_terms_bytes(B) + le_grad_bytes(B, C));
  cudaStream_t st = as_stream(stream);
  launch(labelembed_row_kernel, dim3(ceil_div(B, LE_WARPS)), dim3(LE_WARPS * 32), 0, st, out1, out2, ld, labels, emb, ldE,
         B, C, tau, alpha, beta, scale, acc, d_out1, d_out2, terms, d_emb ? g_rows : nullptr, key);
  int rc = check_launch("labelembed_row_kernel");
  if (rc != SE_OK || !(loss || d_emb)) return rc;
  const int grid = d_emb ? C : ceil_div(B, LE_FIN_THREADS);
  launch(labelembed_finish_kernel, dim3(grid), dim3(LE_FIN_THREADS), d_emb ? (size_t)B * sizeof(int) : 0, st, labels, B, C,
         scale, (const float4*)terms, (const float*)g_rows, (const int*)key, loss, d_emb, ldE);
  return check_launch("labelembed_finish_kernel");
}
