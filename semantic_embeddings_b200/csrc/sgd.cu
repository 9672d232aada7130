// keras.optimizers.SGD(lr, momentum=0.9, decay, nesterov, clipnorm) + regularizers.l2 as two
// multi-tensor passes over ONE flat fp32 buffer (learn_image_embeddings.py:229-236;
// models/cifar_resnet.py:152; models/plainnet.py:8; learn_image_embeddings.py:44).
// HBM-bound: pass 1 reads p,g and writes g; pass 2 reads p,g,v and writes p,v -- 128-bit accesses.
#include "common.cuh"

namespace se {

constexpr int MAX_SEGS = 8;
struct Segs {
  long long begin[MAX_SEGS], end[MAX_SEGS];
  float l2[MAX_SEGS];
  int n;
};

__device__ __forceinline__ float seg_l2(const Segs& s, long long i) {
  float l = 0.f;
#pragma unroll
  for (int k = 0; k < MAX_SEGS; ++k)
    if (k < s.n && i >= s.begin[k] && i < s.end[k]) l = s.l2[k];
  return l;
}

// g += 2*lambda*p ; out[0] += sum g^2 ; out[1] += sum lambda*p^2
__global__ void __launch_bounds__(256)
sgd_prepare_kernel(const float* __restrict__ p, float* __restrict__ g, long long n, Segs segs, double* __restrict__ out) {
  pdl_grid_sync();
  double sq = 0.0, reg = 0.0;
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 gv = *reinterpret_cast<const float4*>(g + 4 * i);
    float gg[4] = {gv.x, gv.y, gv.z, gv.w};
    float l[4];
    bool any = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) { l[j] = seg_l2(segs, 4 * i + j); any |= (l[j] != 0.f); }
    if (any) {
      float4 pv = *reinterpret_cast<const float4*>(p + 4 * i);
      float pp[4] = {pv.x, pv.y, pv.z, pv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        gg[j] = fmaf(2.f * l[j], pp[j], gg[j]);
        reg += (double)(l[j] * pp[j] * pp[j]);
      }
      *reinterpret_cast<float4*>(g + 4 * i) = make_float4(gg[0], gg[1], gg[2], gg[3]);
    }
    float s = gg[0] * gg[0] + gg[1] * gg[1] + gg[2] * gg[2] + gg[3] * gg[3];
    sq += (double)s;
  }
  // tail
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float l = seg_l2(segs, i);
    float gg = g[i];
    if (l != 0.f) { float pp = p[i]; gg = fmaf(2.f * l, pp, gg); reg += (double)(l * pp * pp); g[i] = gg; }
    sq += (double)gg * gg;
  }
  sq = warp_sum(sq);
  reg = warp_sum(reg);
  __shared__ double s_sq[8], s_reg[8];
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s_sq[warp] = sq; s_reg[warp] = reg; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0;
    for (int k = 0; k < 8; ++k) { a += s_sq[k]; b += s_reg[k]; }
    atomicAdd(&out[0], a);
    atomicAdd(&out[1], b);
  }
}

__global__ void __launch_bounds__(256)
sgd_apply_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ v, long long n, float lr,
                 const float* __restrict__ lr_dev, float momentum, int nesterov, float clipnorm,
                 const double* __restrict__ out) {
  pdl_grid_sync();
  if (lr_dev) lr = *lr_dev;   // graph-captured steps read the schedule's learning rate from device memory
  float scale = 1.f;
  if (clipnorm > 0.f) {
    float norm = (float)sqrt(out[0]);
    if (norm >= clipnorm) scale = clipnorm / norm;   // K.switch(norm >= c, g*c/norm, g)
  }
  const float step = lr * scale;
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 gv = *reinterpret_cast<const float4*>(g + 4 * i);
    float4 vv = *reinterpret_cast<const float4*>(v + 4 * i);
    float4 pv = *reinterpret_cast<const float4*>(p + 4 * i);
    float gg[4] = {gv.x, gv.y, gv.z, gv.w}, ve[4] = {vv.x, vv.y, vv.z, vv.w}, pp[4] = {pv.x, pv.y, pv.z, pv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float nv = momentum * ve[j] - step * gg[j];
      ve[j] = nv;
      pp[j] += nesterov ? (momentum * nv - step * gg[j]) : nv;
    }
    *reinterpret_cast<float4*>(v + 4 * i) = make_float4(ve[0], ve[1], ve[2], ve[3]);
    *reinterpret_cast<float4*>(p + 4 * i) = make_float4(pp[0], pp[1], pp[2], pp[3]);
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float nv = momentum * v[i] - step * g[i];
    v[i] = nv;
    p[i] += nesterov ? (momentum * nv - step * g[i]) : nv;
  }
}

// keras.optimizers.Adagrad (Keras 2.2): a += g^2; p -= lr_t g / (sqrt(a) + eps), no momentum; g is the gradient after
// sgd_prepare_kernel (L2 terms added, global norm in out[0]) and the optional clip.  Reads p, g, a and writes p, a.
__global__ void __launch_bounds__(256)
adagrad_apply_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ a, long long n,
                     const float* lr_dev, float eps, float clipnorm, const double* __restrict__ out) {
  pdl_grid_sync();
  // lr_dev is written by the schedule kernel just before: no __restrict__, so that the load is not hoisted above the
  // grid dependency wait as a read-only one
  const float lr = *lr_dev;
  float scale = 1.f;
  if (clipnorm > 0.f) {
    float norm = (float)sqrt(out[0]);
    if (norm >= clipnorm) scale = clipnorm / norm;
  }
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 gv = *reinterpret_cast<const float4*>(g + 4 * i);
    float4 av = *reinterpret_cast<const float4*>(a + 4 * i);
    float4 pv = *reinterpret_cast<const float4*>(p + 4 * i);
    float gg[4] = {gv.x, gv.y, gv.z, gv.w}, ac[4] = {av.x, av.y, av.z, av.w}, pp[4] = {pv.x, pv.y, pv.z, pv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gs = scale * gg[j];
      ac[j] = fmaf(gs, gs, ac[j]);
      pp[j] -= lr * gs / (sqrtf(ac[j]) + eps);
    }
    *reinterpret_cast<float4*>(a + 4 * i) = make_float4(ac[0], ac[1], ac[2], ac[3]);
    *reinterpret_cast<float4*>(p + 4 * i) = make_float4(pp[0], pp[1], pp[2], pp[3]);
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gs = scale * g[i];
    const float na = fmaf(gs, gs, a[i]);
    a[i] = na;
    p[i] -= lr * gs / (sqrtf(na) + eps);
  }
}

static int flat_grid(long long n) {
  long long g = ceil_div<long long>(ceil_div<long long>(n, 4), 256);
  return (int)max(1LL, min(g, (long long)sm_count() * 4));
}

}  // namespace se

using namespace se;

extern "C" int se_sgd_prepare(const float* p, float* g, int64_t n, const se_l2_segment* segs, int nsegs, double* out,
                              void* stream) {
  SE_REQUIRE(p && g && out && n > 0, "bad arguments");
  SE_REQUIRE(nsegs >= 0 && nsegs <= MAX_SEGS, "at most 8 L2 segments");
  Segs s;
  s.n = nsegs;
  for (int k = 0; k < MAX_SEGS; ++k) {
    s.begin[k] = k < nsegs ? segs[k].begin : 0;
    s.end[k] = k < nsegs ? segs[k].end : 0;
    s.l2[k] = k < nsegs ? segs[k].l2 : 0.f;
  }
  launch(sgd_prepare_kernel, dim3(flat_grid(n)), dim3(256), 0, as_stream(stream), p, g, n, s, out);
  return check_launch("sgd_prepare_kernel");
}

// Keras SGD(decay): lr_t = lr / (1 + decay * iterations), iterations counted by the optimizer (learn_image_embeddings.py:
// 224-236 derives `decay` from --max_decay).  state = {lr (set by the schedule), decay, iterations, lr_t (output)}.
__global__ void sgd_schedule_kernel(float* __restrict__ state) {
  pdl_grid_sync();
  if (threadIdx.x == 0) {
    state[3] = state[0] / (1.f + state[1] * state[2]);
    state[2] += 1.f;
  }
}

extern "C" int se_sgd_schedule(float* lr_state, void* stream) {
  SE_REQUIRE(lr_state != nullptr, "bad arguments");
  launch(sgd_schedule_kernel, dim3(1), dim3(32), 0, as_stream(stream), lr_state);
  return check_launch("sgd_schedule_kernel");
}

extern "C" int se_sgd_apply(float* p, const float* g, float* v, int64_t n, float lr, float momentum, int nesterov,
                            float clipnorm, const double* out, void* stream) {
  SE_REQUIRE(p && g && v && out && n > 0, "bad arguments");
  launch(sgd_apply_kernel, dim3(flat_grid(n)), dim3(256), 0, as_stream(stream), p, g, v, n, lr, nullptr, momentum, nesterov, clipnorm, out);
  return check_launch("sgd_apply_kernel");
}

extern "C" int se_sgd_apply_devlr(float* p, const float* g, float* v, int64_t n, const float* lr_dev, float momentum,
                                  int nesterov, float clipnorm, const double* out, void* stream) {
  SE_REQUIRE(p && g && v && out && lr_dev && n > 0, "bad arguments");
  launch(sgd_apply_kernel, dim3(flat_grid(n)), dim3(256), 0, as_stream(stream), p, g, v, n, 0.f, lr_dev, momentum, nesterov, clipnorm, out);
  return check_launch("sgd_apply_kernel");
}

extern "C" int se_sgd_step(float* p, float* g, float* v, int64_t n, const se_l2_segment* segs, int nsegs, float lr,
                           float momentum, int nesterov, float clipnorm, double* out, void* stream) {
  int rc = se_sgd_prepare(p, g, n, segs, nsegs, out, stream);
  if (rc) return rc;
  return se_sgd_apply(p, g, v, n, lr, momentum, nesterov, clipnorm, out, stream);
}

extern "C" int se_adagrad_apply_devlr(float* p, const float* g, float* a, int64_t n, const float* lr_dev, float epsilon,
                                      float clipnorm, const double* out, void* stream) {
  SE_REQUIRE(p && g && a && out && lr_dev && n > 0, "bad arguments");
  launch(adagrad_apply_kernel, dim3(flat_grid(n)), dim3(256), 0, as_stream(stream), p, g, a, n, lr_dev, epsilon, clipnorm, out);
  return check_launch("adagrad_apply_kernel");
}
