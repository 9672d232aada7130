// BatchNormalization (training + inference) fused with the ReLU / residual-add / pooled+padded
// shortcut that follows it in the reference graphs (models/cifar_resnet.py:100-124,220;
// models/plainnet.py:53,68,71; models/wide_residual_network.py:14-92; learn_image_embeddings.py:42-43).
// HBM-bound elementwise + per-channel reductions: 128-bit coalesced accesses along the channel
// axis, float64 cross-CTA accumulation of the statistics.  Backward is ONE launch when a CTA's slab fits in registers
// (bn_bwd_reg_kernel: grid barrier on the two sums, prefetch of the forward-pass inputs before the programmatic grid
// dependency resolves) or in shared memory (bn_bwd_fused_kernel), else reduce + apply kernels.
#include <stdlib.h>

#include "common.cuh"

namespace se {

// ---------------------------------------------------------------------------------------- statistics
// x [rows, C] -> stats[c] += sum x, stats[C+c] += sum x^2.  Thread layout: C4 = C/4 float4 lanes
// along channels, the rest of the block strides over rows.
__global__ void __launch_bounds__(256)
bn_stats_kernel(const float* __restrict__ x, long long rows, int C, double* __restrict__ stats, int rows_per_cta) {
  pdl_grid_sync();
  extern __shared__ double sred[];  // [2*C]
  const int tid = threadIdx.x;
  for (int i = tid; i < 2 * C; i += blockDim.x) sred[i] = 0.0;
  __syncthreads();
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = min(rows, r0 + rows_per_cta);
  if ((C & 3) == 0) {
    const int C4 = C >> 2;
    const int lanes = min(C4, (int)blockDim.x);
    const int rstep = blockDim.x / lanes;
    const int cq0 = tid % lanes, rr = tid / lanes;
    if (rr < rstep) {
      for (int cq = cq0; cq < C4; cq += lanes) {
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = make_float4(0.f, 0.f, 0.f, 0.f);
        double ds[4] = {0, 0, 0, 0}, dq[4] = {0, 0, 0, 0};
        int cnt = 0;
        for (long long r = r0 + rr; r < r1; r += rstep) {
          float4 v = *reinterpret_cast<const float4*>(x + r * C + 4 * cq);
          s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
          q.x += v.x * v.x; q.y += v.y * v.y; q.z += v.z * v.z; q.w += v.w * v.w;
          if (++cnt == 64) {  // flush the short fp32 partials into float64
            ds[0] += s.x; ds[1] += s.y; ds[2] += s.z; ds[3] += s.w;
            dq[0] += q.x; dq[1] += q.y; dq[2] += q.z; dq[3] += q.w;
            s = make_float4(0.f, 0.f, 0.f, 0.f); q = s; cnt = 0;
          }
        }
        ds[0] += s.x; ds[1] += s.y; ds[2] += s.z; ds[3] += s.w;
        dq[0] += q.x; dq[1] += q.y; dq[2] += q.z; dq[3] += q.w;
        // lanes of a warp that share this channel quad (lanes apart by `lanes`, when lanes divides 32) combine first
        const bool pow2 = (lanes & (lanes - 1)) == 0 && lanes < 32 && (C4 <= lanes);
        if (pow2) {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            for (int o = lanes; o < 32; o <<= 1) {
              ds[j] += __shfl_xor_sync(0xffffffffu, ds[j], o);
              dq[j] += __shfl_xor_sync(0xffffffffu, dq[j], o);
            }
        }
        if (!pow2 || (tid & 31) < lanes) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            atomicAdd(&sred[4 * cq + j], ds[j]);
            atomicAdd(&sred[C + 4 * cq + j], dq[j]);
          }
        }
      }
    }
  } else {
    for (int c = tid; c < C; c += blockDim.x) {
      double s = 0, q = 0;
      for (long long r = r0; r < r1; ++r) { float v = x[r * C + c]; s += v; q += (double)v * v; }
      sred[c] += s; sred[C + c] += q;
    }
  }
  __syncthreads();
  for (int i = tid; i < 2 * C; i += blockDim.x) atomicAdd(&stats[i], sred[i]);
}

// ---------------------------------------------------------------------------------------- forward
struct Res {
  const float* ptr; int C, pad_lo, pool, H, W;
};

__device__ __forceinline__ float res_value(const Res& r, long long row, int c) {
  // residual contribution for output element (row, c) of a (N,H,W,Cout) tensor
  int cr = c - r.pad_lo;
  if (cr < 0 || cr >= r.C) return 0.f;
  if (r.pool == 1) return r.ptr[row * r.C + cr];
  int w = (int)(row % r.W);
  long long t = row / r.W;
  int h = (int)(t % r.H);
  long long n = t / r.H;
  const float* b = r.ptr + ((n * (2 * r.H) + 2 * h) * (2 * r.W) + 2 * w) * (long long)r.C + cr;
  long long rs = (long long)(2 * r.W) * r.C;
  return 0.25f * (b[0] + b[r.C] + b[rs] + b[rs + r.C]);
}

// Each CTA first derives scale/shift for all channels (from the float64 sums in training mode, from the
// moving statistics in inference mode), CTA 0 also writes the saved statistics + moving averages.
template <bool TRAIN>
__global__ void __launch_bounds__(256)
bn_fwd_kernel(const float* __restrict__ x, long long rows, int C, const double* __restrict__ stats,
              const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum,
              float* __restrict__ moving_mean, float* __restrict__ moving_var, float* __restrict__ save_mean,
              float* __restrict__ save_invstd, Res res, int relu, float* __restrict__ y) {
  pdl_grid_sync();
  extern __shared__ float sc[];  // scale[C], shift[C]
  float* scale = sc;
  float* shift = sc + C;
  const long long total = rows * C;
  const bool vec4 = (C & 3) == 0;
  const long long total4 = total >> 2;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const bool plain_res = res.ptr && res.pool == 1 && res.pad_lo == 0 && res.C == C;
  // the first batch of loads is issued BEFORE the per-channel coefficients are derived: the float64 moment arithmetic
  // and the block barrier below then overlap the memory latency instead of preceding it
  float4 vq[4], rq[4];
  const long long i_first = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (vec4) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long i = i_first + u * stride;
      if (i < total4) {
        vq[u] = *reinterpret_cast<const float4*>(x + (i << 2));
        if (plain_res) rq[u] = *reinterpret_cast<const float4*>(res.ptr + (i << 2));
      }
    }
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float mean, invstd;
    if (TRAIN) {
      // float64 moments and inverse standard deviation (a 1-ulp change of invstd flips ReLU masks of near-zero
      // activations against the float64 oracle); 1/rows once instead of two divisions
      const double inv_rows = 1.0 / (double)rows;
      double m = stats[c] * inv_rows;
      double var = stats[C + c] * inv_rows - m * m;
      if (var < 0) var = 0;
      mean = (float)m;
      invstd = (float)(1.0 / sqrt(var + (double)eps));
      if (blockIdx.x == 0) {
        save_mean[c] = mean;
        save_invstd[c] = invstd;
        if (moving_mean) {
          double n = (double)rows;
          double uvar = var * (n / (n - (1.0 + (double)eps)));
          moving_mean[c] = moving_mean[c] * momentum + mean * (1.f - momentum);
          moving_var[c] = moving_var[c] * momentum + (float)uvar * (1.f - momentum);
        }
      }
    } else {
      mean = moving_mean[c];
      invstd = rsqrtf(moving_var[c] + eps);
    }
    float g = gamma[c];
    scale[c] = g * invstd;
    shift[c] = beta[c] - mean * g * invstd;
  }
  __syncthreads();
  if (vec4) {
    // channel quad of this thread: fixed when the grid stride is a multiple of C/4 (every power-of-two width), so the
    // per-element 64-bit modulo / division -- which made this kernel instruction-bound -- is done once, in 32 bits
    const int C4 = C >> 2;
    const bool fixed_c = (stride % C4) == 0;
    const int c_fixed = (int)(i_first % C4) * 4;
    for (long long i0 = i_first; i0 < total4; i0 += 4 * stride) {
      if (i0 != i_first) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const long long i = i0 + u * stride;
          if (i < total4) {
            vq[u] = *reinterpret_cast<const float4*>(x + (i << 2));
            if (plain_res) rq[u] = *reinterpret_cast<const float4*>(res.ptr + (i << 2));
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long i = i0 + u * stride;
        if (i >= total4) continue;
        const long long e = i << 2;
        const int c = fixed_c ? c_fixed : (int)(e % C);
        float o[4] = {vq[u].x, vq[u].y, vq[u].z, vq[u].w};
        const float r4[4] = {rq[u].x, rq[u].y, rq[u].z, rq[u].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float t = o[j] * scale[c + j] + shift[c + j];
          if (plain_res) t += r4[j];
          else if (res.ptr) t += res_value(res, e / C, c + j);
          if (relu) t = fmaxf(t, 0.f);
          o[j] = t;
        }
        *reinterpret_cast<float4*>(y + e) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  } else {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
      int c = (int)(e % C);
      long long row = e / C;
      float t = x[e] * scale[c] + shift[c];
      if (res.ptr) t += res_value(res, row, c);
      if (relu) t = fmaxf(t, 0.f);
      y[e] = t;
    }
  }
}

// ---------------------------------------------------------------------------------------- backward
// pass 1: scratch[c] += sum g, scratch[C+c] += sum g*xhat with g = dout * (y > 0 if relu)
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dout,
                     long long rows, int C, const float* __restrict__ save_mean, const float* __restrict__ save_invstd,
                     int relu, double* __restrict__ scratch, int rows_per_cta) {
  pdl_grid_sync();
  extern __shared__ double sred[];
  const int tid = threadIdx.x;
  for (int i = tid; i < 2 * C; i += blockDim.x) sred[i] = 0.0;
  __syncthreads();
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = min(rows, r0 + rows_per_cta);
  if ((C & 3) == 0) {
    const int C4 = C >> 2;
    const int lanes = min(C4, (int)blockDim.x);
    const int rstep = blockDim.x / lanes;
    const int cq0 = tid % lanes, rr = tid / lanes;
    if (rr < rstep) {
      for (int cq = cq0; cq < C4; cq += lanes) {
        float mu[4], is[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { mu[j] = save_mean[4 * cq + j]; is[j] = save_invstd[4 * cq + j]; }
        float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
        double ds[4] = {0, 0, 0, 0}, dq[4] = {0, 0, 0, 0};
        int cnt = 0;
        for (long long r = r0 + rr; r < r1; r += rstep) {
          long long e = r * C + 4 * cq;
          float4 xv = *reinterpret_cast<const float4*>(x + e);
          float4 gv = *reinterpret_cast<const float4*>(dout + e);
          float g[4] = {gv.x, gv.y, gv.z, gv.w};
          float xx[4] = {xv.x, xv.y, xv.z, xv.w};
          if (relu) {
            float4 yv = *reinterpret_cast<const float4*>(y + e);
            if (!(yv.x > 0.f)) g[0] = 0.f;
            if (!(yv.y > 0.f)) g[1] = 0.f;
            if (!(yv.z > 0.f)) g[2] = 0.f;
            if (!(yv.w > 0.f)) g[3] = 0.f;
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) { s[j] += g[j]; q[j] += g[j] * (xx[j] - mu[j]) * is[j]; }
          if (++cnt == 64) {
#pragma unroll
            for (int j = 0; j < 4; ++j) { ds[j] += s[j]; dq[j] += q[j]; s[j] = 0.f; q[j] = 0.f; }
            cnt = 0;
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) { ds[j] += s[j]; dq[j] += q[j]; }
        const bool pow2 = (lanes & (lanes - 1)) == 0 && lanes < 32 && (C4 <= lanes);
        if (pow2) {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            for (int o = lanes; o < 32; o <<= 1) {
              ds[j] += __shfl_xor_sync(0xffffffffu, ds[j], o);
              dq[j] += __shfl_xor_sync(0xffffffffu, dq[j], o);
            }
        }
        if (!pow2 || (tid & 31) < lanes) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            atomicAdd(&sred[4 * cq + j], ds[j]);
            atomicAdd(&sred[C + 4 * cq + j], dq[j]);
          }
        }
      }
    }
  } else {
    for (int c = tid; c < C; c += blockDim.x) {
      double s = 0, q = 0;
      float mu = save_mean[c], is = save_invstd[c];
      for (long long r = r0; r < r1; ++r) {
        float g = dout[r * C + c];
        if (relu && !(y[r * C + c] > 0.f)) g = 0.f;
        s += g; q += (double)g * (x[r * C + c] - mu) * is;
      }
      sred[c] += s; sred[C + c] += q;
    }
  }
  __syncthreads();
  for (int i = tid; i < 2 * C; i += blockDim.x) atomicAdd(&scratch[i], sred[i]);
}

// pass 2: dx, dres, and (CTA 0) dgamma / dbeta
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dout,
                    long long rows, int C, const float* __restrict__ gamma, const float* __restrict__ save_mean,
                    const float* __restrict__ save_invstd, int relu, int relu_in, float* __restrict__ dx, float beta_dx,
                    float* __restrict__ dres, float beta_res, float* __restrict__ dgamma, float* __restrict__ dbeta,
                    const double* __restrict__ scratch) {
  pdl_grid_sync();
  extern __shared__ float sc[];  // a[C], b[C], m[C], k[C]:  dx = a*g + b + k*x   (k = -a*... folded)
  float* ca = sc;
  float* cb = sc + C;
  float* cm = sc + 2 * C;
  float* ck = sc + 3 * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double sg = scratch[c], sgx = scratch[C + c];
    float invstd = save_invstd[c], mean = save_mean[c], g = gamma[c];
    float a = g * invstd;
    // dx = a * (gr - sg/n - xhat * sgx/n),  xhat = (x-mean)*invstd
    ca[c] = a;
    cb[c] = (float)(-(double)a * sg / (double)rows);
    ck[c] = (float)(-(double)a * sgx / (double)rows) * invstd;
    cm[c] = mean;
    if (blockIdx.x == 0) {
      if (dgamma) dgamma[c] += (float)sgx;
      if (dbeta) dbeta[c] += (float)sg;
    }
  }
  __syncthreads();
  const long long total = rows * C;
  if ((C & 3) == 0) {
    const long long total4 = total >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
      long long e = i << 2;
      int c = (int)(e % C);
      float4 xv = *reinterpret_cast<const float4*>(x + e);
      float4 gv = *reinterpret_cast<const float4*>(dout + e);
      float g[4] = {gv.x, gv.y, gv.z, gv.w};
      float xx[4] = {xv.x, xv.y, xv.z, xv.w};
      if (relu) {
        float4 yv = *reinterpret_cast<const float4*>(y + e);
        if (!(yv.x > 0.f)) g[0] = 0.f;
        if (!(yv.y > 0.f)) g[1] = 0.f;
        if (!(yv.z > 0.f)) g[2] = 0.f;
        if (!(yv.w > 0.f)) g[3] = 0.f;
      }
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float d = ca[c + j] * g[j] + cb[c + j] + ck[c + j] * (xx[j] - cm[c + j]);
        if (relu_in && !(xx[j] > 0.f)) d = 0.f;
        o[j] = d;
      }
      if (beta_dx != 0.f) {
        float4 old = *reinterpret_cast<const float4*>(dx + e);
        o[0] += beta_dx * old.x; o[1] += beta_dx * old.y; o[2] += beta_dx * old.z; o[3] += beta_dx * old.w;
      }
      *reinterpret_cast<float4*>(dx + e) = make_float4(o[0], o[1], o[2], o[3]);
      if (dres) {
        if (beta_res != 0.f) {
          float4 old = *reinterpret_cast<const float4*>(dres + e);
          g[0] += beta_res * old.x; g[1] += beta_res * old.y; g[2] += beta_res * old.z; g[3] += beta_res * old.w;
        }
        *reinterpret_cast<float4*>(dres + e) = make_float4(g[0], g[1], g[2], g[3]);
      }
    }
  } else {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
      int c = (int)(e % C);
      float g = dout[e];
      if (relu && !(y[e] > 0.f)) g = 0.f;
      float xv = x[e];
      float d = ca[c] * g + cb[c] + ck[c] * (xv - cm[c]);
      if (relu_in && !(xv > 0.f)) d = 0.f;
      if (beta_dx != 0.f) d += beta_dx * dx[e];
      dx[e] = d;
      if (dres) dres[e] = (beta_res != 0.f ? beta_res * dres[e] : 0.f) + g;
    }
  }
}

// Register-slab variant of the fused backward below: the CTA's slab of x and g = dout*(y>0) stays in REGISTERS
// (up to BNR float4 of each per thread) between the reduction and the apply phase, so the kernel needs almost no shared
// memory -- it can share an SM with the weight-gradient kernel that se_run_ops runs on its side stream -- and skips the
// shared-memory round trip of the slab.  Requires blockDim % (C/4) == 0 (a thread always sees the same channel quad).
// scratch: float64 [2C] sums + [1] arrival counter, caller zeroes.  grid <= #SMs (all CTAs co-resident).
constexpr int BNR = 8;
constexpr int BNR_MAXC = 128;   // channel limit of the register-slab kernel (16 warps x 2C floats of partial sums)
// debug: SE_BN_TRACE_PTR = device address of 8 int64: clock64 stamps of CTA 0 / thread 0 at the phase boundaries
#define BN_STAMP(k) do { if (trace && blockIdx.x == 0 && threadIdx.x == 0) trace[k] = clock64(); } while (0)
__global__ void __maxnreg__(112)
bn_bwd_reg_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dout, long long rows,
                  int C, const float* __restrict__ gamma, const float* __restrict__ save_mean,
                  const float* __restrict__ save_invstd, int relu, int relu_in, float* __restrict__ dx, float beta_dx,
                  float* __restrict__ dres, float beta_res, float* __restrict__ dgamma, float* __restrict__ dbeta,
                  double* __restrict__ scratch, int rows_per_cta, int early, long long* trace) {
  BN_STAMP(0);
  // early != 0: x, y and the saved statistics were written many launches ago (the forward pass), so they are fetched
  // BEFORE the grid dependency resolves -- two thirds of this kernel's input traffic overlaps the tail of the kernel
  // that produces dout.  (The engine sets it only when the producing launch is far enough back; common.cuh.)
  pdl_trigger();
  if (!early) pdl_wait();
  __shared__ float part[16 * 2 * BNR_MAXC];        // [warp][2C] partial sums (plain stores: no shared-memory atomics)
  const double inv_rows = 1.0 / (double)rows;      // the one float64 division, hidden behind the loads
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = min(rows, r0 + rows_per_cta);
  const int nrows = (int)max(0LL, r1 - r0);
  const int n4 = nrows * C / 4;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int C4 = C >> 2;
  const int cq = tid % C4;
  const float4* gx = reinterpret_cast<const float4*>(x + r0 * C);
  const float4* gd = reinterpret_cast<const float4*>(dout + r0 * C);
  const float4* gy = reinterpret_cast<const float4*>(y + r0 * C);
  const float4 mu = make_float4(save_mean[4 * cq], save_mean[4 * cq + 1], save_mean[4 * cq + 2], save_mean[4 * cq + 3]);
  const float4 is = make_float4(save_invstd[4 * cq], save_invstd[4 * cq + 1], save_invstd[4 * cq + 2], save_invstd[4 * cq + 3]);
  const float4 gm = make_float4(gamma[4 * cq], gamma[4 * cq + 1], gamma[4 * cq + 2], gamma[4 * cq + 3]);

  // ---- phase 1: everything this thread will need, in flight at once
  float4 xv[BNR], gv[BNR];
  unsigned keep[BNR];                               // ReLU mask of the four channels (bit j: y_j > 0)
#pragma unroll
  for (int u = 0; u < BNR; ++u) {
    const int i = tid + u * nt;
    keep[u] = 0xFu;
    if (i < n4) {
      xv[u] = ldg_nc_f4(reinterpret_cast<const float*>(gx + i));
      if (relu) {
        const float4 yv = ldg_nc_f4(reinterpret_cast<const float*>(gy + i));
        keep[u] = (yv.x > 0.f ? 1u : 0u) | (yv.y > 0.f ? 2u : 0u) | (yv.z > 0.f ? 4u : 0u) | (yv.w > 0.f ? 8u : 0u);
      }
    }
  }
  BN_STAMP(1);
  if (early) pdl_wait();                            // dout comes from the preceding launch
  BN_STAMP(2);
#pragma unroll
  for (int u = 0; u < BNR; ++u) {
    const int i = tid + u * nt;
    if (i < n4) gv[u] = ldg_nc_f4(reinterpret_cast<const float*>(gd + i));
  }
#pragma unroll
  for (int u = 0; u < BNR; ++u) {
    if (!(keep[u] & 1u)) gv[u].x = 0.f;
    if (!(keep[u] & 2u)) gv[u].y = 0.f;
    if (!(keep[u] & 4u)) gv[u].z = 0.f;
    if (!(keep[u] & 8u)) gv[u].w = 0.f;
  }
  float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
#pragma unroll
  for (int u = 0; u < BNR; ++u) {
    const int i = tid + u * nt;
    if (i < n4) {
      s[0] += gv[u].x; s[1] += gv[u].y; s[2] += gv[u].z; s[3] += gv[u].w;
      q[0] += gv[u].x * (xv[u].x - mu.x) * is.x; q[1] += gv[u].y * (xv[u].y - mu.y) * is.y;
      q[2] += gv[u].z * (xv[u].z - mu.z) * is.z; q[3] += gv[u].w * (xv[u].w - mu.w) * is.w;
    }
  }
  // lanes that share the quad (C4 divides 32) combine with shuffles; one lane per quad and warp then owns a slot of
  // `part` (plain stores), and 2C threads add the 16 warp partials in float64 into the global sums.  (Shared-memory
  // float64 atomics under 16-way contention were the longest phase of this kernel: 2.6-3.4 us.)
  const int warp = tid >> 5, lane = tid & 31;
  if (C4 < 32) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      for (int o = C4; o < 32; o <<= 1) {
        s[j] += __shfl_xor_sync(0xffffffffu, s[j], o);
        q[j] += __shfl_xor_sync(0xffffffffu, q[j], o);
      }
  }
  BN_STAMP(3);
  // C4 <= 32: lanes 0..C4-1 hold the quad totals of the warp.  C4 > 32 (C = 256, 512): consecutive warps cover
  // different quads (quad = tid % C4), each (warp, quad) pair still has exactly one writer; slots of quads a warp
  // does not touch stay zero.
  if (C4 > 32) for (int i = tid; i < 16 * 2 * C; i += nt) part[i] = 0.f;
  if (C4 > 32) __syncthreads();
  if (lane < C4 || C4 > 32) {
    float* pw = part + warp * 2 * C;
#pragma unroll
    for (int j = 0; j < 4; ++j) { pw[4 * cq + j] = s[j]; pw[C + 4 * cq + j] = q[j]; }
  }
  __syncthreads();
  for (int i = tid; i < 2 * C; i += nt) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < 16; ++w) v += (double)part[w * 2 * C + i];
    atomicAdd(&scratch[i], v);
  }

  // ---- grid barrier (arrival counter in scratch[2C], zeroed by the caller once per step).  The block barrier orders
  // the atomics of all threads before thread 0's fence (cumulativity), so one thread fences for the CTA.
  __syncthreads();
  BN_STAMP(4);
  unsigned long long* counter = reinterpret_cast<unsigned long long*>(scratch + 2 * C);
  if (tid == 0) {
    __threadfence();
    atomicAdd(counter, 1ULL);
    while (*reinterpret_cast<volatile unsigned long long*>(counter) < (unsigned long long)gridDim.x) { }
    __threadfence();
  }
  __syncthreads();
  BN_STAMP(5);

  // ---- phase 2: the global sums come into shared memory with ONE L2 read per value and CTA; every thread then
  // derives the coefficients of its four channels itself.  Parameter gradients: fire-and-forget reductions by CTA 0.
  __shared__ double ssum[2 * BNR_MAXC];
  for (int i = tid; i < 2 * C; i += nt) {
    const double v = __ldcg(&scratch[i]);
    ssum[i] = v;
    if (blockIdx.x == 0) {
      if (i < C) { if (dbeta) atomicAdd(&dbeta[i], (float)v); }
      else if (dgamma) atomicAdd(&dgamma[i - C], (float)v);
    }
  }
  __syncthreads();
  float ca_[4], cb_[4], ck_[4];
  {
    const float gmv[4] = {gm.x, gm.y, gm.z, gm.w}, isv[4] = {is.x, is.y, is.z, is.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double sgm = ssum[4 * cq + j], sgx = ssum[C + 4 * cq + j];
      const float a = gmv[j] * isv[j];
      ca_[j] = a;
      cb_[j] = (float)(-(double)a * sgm * inv_rows);
      ck_[j] = (float)(-(double)a * sgx * inv_rows) * isv[j];
    }
  }
  BN_STAMP(6);
  const float4 ca = make_float4(ca_[0], ca_[1], ca_[2], ca_[3]);
  const float4 cb = make_float4(cb_[0], cb_[1], cb_[2], cb_[3]);
  const float4 ck = make_float4(ck_[0], ck_[1], ck_[2], ck_[3]);
  float4* odx = reinterpret_cast<float4*>(dx + r0 * C);
  float4* odr = dres ? reinterpret_cast<float4*>(dres + r0 * C) : nullptr;
#pragma unroll
  for (int u = 0; u < BNR; ++u) {
    const int i = tid + u * nt;
    if (i >= n4) continue;
    float4 o;
    o.x = ca.x * gv[u].x + cb.x + ck.x * (xv[u].x - mu.x);
    o.y = ca.y * gv[u].y + cb.y + ck.y * (xv[u].y - mu.y);
    o.z = ca.z * gv[u].z + cb.z + ck.z * (xv[u].z - mu.z);
    o.w = ca.w * gv[u].w + cb.w + ck.w * (xv[u].w - mu.w);
    if (relu_in) {
      if (!(xv[u].x > 0.f)) o.x = 0.f;
      if (!(xv[u].y > 0.f)) o.y = 0.f;
      if (!(xv[u].z > 0.f)) o.z = 0.f;
      if (!(xv[u].w > 0.f)) o.w = 0.f;
    }
    if (beta_dx != 0.f) {
      const float4 old = odx[i];
      o.x += beta_dx * old.x; o.y += beta_dx * old.y; o.z += beta_dx * old.z; o.w += beta_dx * old.w;
    }
    odx[i] = o;
    if (odr) {
      float4 r = gv[u];
      if (beta_res != 0.f) {
        const float4 old = odr[i];
        r.x += beta_res * old.x; r.y += beta_res * old.y; r.z += beta_res * old.z; r.w += beta_res * old.w;
      }
      odr[i] = r;
    }
  }
  BN_STAMP(7);
}

// Fused backward: ONE launch, every input read once.  Each CTA keeps its slab of x and g = dout*(y>0) in shared
// memory, adds its partial sums into `scratch`, waits at a grid-wide barrier (all CTAs are co-resident: grid <= #SMs,
// one CTA per SM), then finishes dx / dres from shared memory.  5 tensor passes instead of 8, one launch instead of two.
// scratch: float64 [2C] sums + [1] arrival counter, caller zeroes.
__global__ void __launch_bounds__(512, 1)
bn_bwd_fused_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dout, long long rows,
                    int C, const float* __restrict__ gamma, const float* __restrict__ save_mean,
                    const float* __restrict__ save_invstd, int relu, int relu_in, float* __restrict__ dx, float beta_dx,
                    float* __restrict__ dres, float beta_res, float* __restrict__ dgamma, float* __restrict__ dbeta,
                    double* __restrict__ scratch, int rows_per_cta) {
  pdl_grid_sync();
  extern __shared__ __align__(16) unsigned char fsm[];
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = min(rows, r0 + rows_per_cta);
  const int nrows = (int)max(0LL, r1 - r0);
  const int n4 = nrows * C / 4;                       // C % 4 == 0 (checked by the launcher)
  float4* sx = reinterpret_cast<float4*>(fsm);
  float4* sg = sx + rows_per_cta * C / 4;
  double* sred = reinterpret_cast<double*>(sg + rows_per_cta * C / 4);      // [2C]
  float* coef = reinterpret_cast<float*>(sred + 2 * C);                    // a, b, k, mean: [4C]
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int i = tid; i < 2 * C; i += nt) sred[i] = 0.0;
  __syncthreads();

  // ---- phase 1: load, mask, partial sums.  Thread t always touches channel quad (t*... ) % C4 == fixed when nt % C4 == 0
  const int C4 = C >> 2;
  const float4* gx = reinterpret_cast<const float4*>(x + r0 * C);
  const float4* gd = reinterpret_cast<const float4*>(dout + r0 * C);
  const float4* gy = reinterpret_cast<const float4*>(y + r0 * C);
  const bool fixed_quad = (nt % C4) == 0;
  float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
  int cq_fixed = tid % C4;
  float mu[4], is[4];
  if (fixed_quad) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { mu[j] = save_mean[4 * cq_fixed + j]; is[j] = save_invstd[4 * cq_fixed + j]; }
  }
  for (int i0 = tid; i0 < n4; i0 += 4 * nt) {
    // four independent rows in flight per thread (the slab loop is latency-bound otherwise)
    float4 xq[4], gq[4], yq[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = i0 + u * nt;
      if (i < n4) {
        xq[u] = gx[i];
        gq[u] = gd[i];
        if (relu) yq[u] = gy[i];
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = i0 + u * nt;
      if (i >= n4) continue;
      float4 xv = xq[u], gv = gq[u];
      if (relu) {
        float4 yv = yq[u];
        if (!(yv.x > 0.f)) gv.x = 0.f;
        if (!(yv.y > 0.f)) gv.y = 0.f;
        if (!(yv.z > 0.f)) gv.z = 0.f;
        if (!(yv.w > 0.f)) gv.w = 0.f;
      }
      sx[i] = xv;
      sg[i] = gv;
      if (fixed_quad) {
        s[0] += gv.x; s[1] += gv.y; s[2] += gv.z; s[3] += gv.w;
        q[0] += gv.x * (xv.x - mu[0]) * is[0]; q[1] += gv.y * (xv.y - mu[1]) * is[1];
        q[2] += gv.z * (xv.z - mu[2]) * is[2]; q[3] += gv.w * (xv.w - mu[3]) * is[3];
      } else {
        const int cq = i % C4;
        const float g4[4] = {gv.x, gv.y, gv.z, gv.w}, x4[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float m = save_mean[4 * cq + j], iv = save_invstd[4 * cq + j];
          atomicAdd(&sred[4 * cq + j], (double)g4[j]);
          atomicAdd(&sred[C + 4 * cq + j], (double)(g4[j] * (x4[j] - m) * iv));
        }
      }
    }
  }
  if (fixed_quad) {
    // lanes that share the quad (when C4 divides 32) combine with shuffles; then one shared-memory atomic per warp
    double ds[4], dq[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { ds[j] = s[j]; dq[j] = q[j]; }
    const bool pow2 = (C4 & (C4 - 1)) == 0 && C4 < 32;
    if (pow2) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        for (int o = C4; o < 32; o <<= 1) {
          ds[j] += __shfl_xor_sync(0xffffffffu, ds[j], o);
          dq[j] += __shfl_xor_sync(0xffffffffu, dq[j], o);
        }
    }
    if (!pow2 || (tid & 31) < C4) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        atomicAdd(&sred[4 * cq_fixed + j], ds[j]);
        atomicAdd(&sred[C + 4 * cq_fixed + j], dq[j]);
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < 2 * C; i += nt) atomicAdd(&scratch[i], sred[i]);

  // ---- grid barrier (arrival counter in scratch[2C], zeroed by the caller once per step)
  __threadfence();
  __syncthreads();
  unsigned long long* counter = reinterpret_cast<unsigned long long*>(scratch + 2 * C);
  if (tid == 0) {
    atomicAdd(counter, 1ULL);
    while (*reinterpret_cast<volatile unsigned long long*>(counter) < (unsigned long long)gridDim.x) { __nanosleep(64); }
    __threadfence();
  }
  __syncthreads();

  // ---- phase 2: coefficients from the global sums, dx / dres from shared memory
  for (int c = tid; c < C; c += nt) {
    double sgm = __ldcg(&scratch[c]), sgx = __ldcg(&scratch[C + c]);
    float invstd = save_invstd[c], g = gamma[c];
    float a = g * invstd;
    coef[c] = a;
    const double inv_rows = 1.0 / (double)rows;
    coef[C + c] = (float)(-(double)a * sgm * inv_rows);
    coef[2 * C + c] = (float)(-(double)a * sgx * inv_rows) * invstd;
    coef[3 * C + c] = save_mean[c];
    if (blockIdx.x == 0) {
      if (dgamma) dgamma[c] += (float)sgx;
      if (dbeta) dbeta[c] += (float)sgm;
    }
  }
  __syncthreads();
  float4* odx = reinterpret_cast<float4*>(dx + r0 * C);
  float4* odr = dres ? reinterpret_cast<float4*>(dres + r0 * C) : nullptr;
  for (int i = tid; i < n4; i += nt) {
    const int c = fixed_quad ? cq_fixed * 4 : (i % C4) * 4;
    float4 xv = sx[i], gv = sg[i];
    float xx[4] = {xv.x, xv.y, xv.z, xv.w}, gg[4] = {gv.x, gv.y, gv.z, gv.w}, o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float d = coef[c + j] * gg[j] + coef[C + c + j] + coef[2 * C + c + j] * (xx[j] - coef[3 * C + c + j]);
      if (relu_in && !(xx[j] > 0.f)) d = 0.f;
      o[j] = d;
    }
    if (beta_dx != 0.f) {
      float4 old = odx[i];
      o[0] += beta_dx * old.x; o[1] += beta_dx * old.y; o[2] += beta_dx * old.z; o[3] += beta_dx * old.w;
    }
    odx[i] = make_float4(o[0], o[1], o[2], o[3]);
    if (odr) {
      if (beta_res != 0.f) {
        float4 old = odr[i];
        gv.x += beta_res * old.x; gv.y += beta_res * old.y; gv.z += beta_res * old.z; gv.w += beta_res * old.w;
      }
      odr[i] = gv;
    }
  }
}

// dsrc[n, 2h+i, 2w+j, c] = beta*dsrc + scale * g[n,h,w,c+pad_lo]   (pool==2: scale .25; pool==1: scale 1)
__global__ void __launch_bounds__(256)
shortcut_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ y, int relu, int N, int H, int W, int C,
                    Res res, float* __restrict__ dsrc, float beta) {
  pdl_grid_sync();
  const int SH = H * res.pool, SW = W * res.pool;
  const long long total = (long long)N * SH * SW * res.C;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    int c = (int)(e % res.C);
    long long t = e / res.C;
    int sw = (int)(t % SW); t /= SW;
    int sh = (int)(t % SH);
    long long n = t / SH;
    long long o = ((n * H + sh / res.pool) * W + sw / res.pool) * C + c + res.pad_lo;
    float g = dout[o];
    if (relu && !(y[o] > 0.f)) g = 0.f;
    if (res.pool == 2) g *= 0.25f;
    dsrc[e] = (beta != 0.f ? beta * dsrc[e] : 0.f) + g;
  }
}

static Res to_res(const se_residual* r) {
  Res o;
  if (r && r->ptr) { o.ptr = r->ptr; o.C = r->C; o.pad_lo = r->pad_lo; o.pool = r->pool; o.H = r->H; o.W = r->W; }
  else { o.ptr = nullptr; o.C = 0; o.pad_lo = 0; o.pool = 1; o.H = 0; o.W = 0; }
  return o;
}

static int ew_grid(long long work_items) {
  long long g = ceil_div<long long>(work_items, 256);
  long long cap = (long long)sm_count() * 8;
  return (int)max(1LL, min(g, cap));
}

// rows per CTA for the reduction kernels: enough CTAs to fill the machine, at least 32 rows each
static int red_rows_per_cta(long long rows, int* grid) {
  long long target = (long long)sm_count() * 2;
  long long per = max(32LL, ceil_div<long long>(rows, target));
  *grid = (int)ceil_div<long long>(rows, per);
  return (int)per;
}

// The backward implementation of (rows, C) on a device with `sms` SMs (SE_BN_BWD_* in se_b200.h): the one decision that
// bn_bwd launches and se_bn_bwd_path reports.  Host arithmetic only.  The slab paths also get their rows per CTA, grid
// and dynamic shared memory.
static constexpr size_t BNF_MAX_SMEM = 200 * 1024;   // shared-memory slab: dynamic shared memory limit per CTA
static int bn_bwd_plan(long long rows, int C, int sms, long long* per_cta, int* grid, size_t* smem) {
  if ((C & 3) != 0) return SE_BN_BWD_SCALAR;
  // one slab of rows per CTA, a multiple of 4 rows, at most one CTA per SM (the grid barrier needs them co-resident)
  long long per_l = ceil_div<long long>(rows, sms);
  per_l = (per_l + 3) / 4 * 4;
  const int gridf = (int)ceil_div<long long>(rows, per_l);
  const size_t bytes = (size_t)per_l * C * 8 + 2 * C * sizeof(double) + 4 * C * sizeof(float) + 16;
  if (per_cta) *per_cta = per_l;
  if (grid) *grid = gridf;
  if (smem) *smem = bytes;
  const int C4 = C >> 2;
  if (gridf <= sms && C <= BNR_MAXC && (512 % C4) == 0 && per_l * C4 <= (long long)BNR * 512)
    return SE_BN_BWD_SLAB_REG;
  if (bytes <= BNF_MAX_SMEM && gridf <= sms)
    return (512 % C4) == 0 ? SE_BN_BWD_SLAB_QUAD : SE_BN_BWD_SLAB_ATOMIC;   // bn_bwd_fused_kernel's fixed_quad (512 threads)
  return SE_BN_BWD_VEC;
}

int init_bn_bwd() {
  if (cudaFuncSetAttribute(bn_bwd_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BNF_MAX_SMEM) != cudaSuccess) {
    set_error("init_bn_bwd: cannot raise the shared-memory limit");
    return SE_ERR_CUDA;
  }
  return SE_OK;
}

}  // namespace se

using namespace se;

extern "C" int se_bn_stats(const float* x, int64_t rows, int C, double* stats, void* stream) {
  SE_REQUIRE(x && stats && rows > 0 && C > 0, "bad arguments");
  int grid;
  int per = red_rows_per_cta(rows, &grid);
  launch(bn_stats_kernel, dim3(grid), dim3(256), 2 * C * sizeof(double), as_stream(stream), x, rows, C, stats, per);
  return check_launch("bn_stats_kernel");
}

extern "C" int se_bn_fwd_train(const float* x, int64_t rows, int C, const double* stats, const float* gamma,
                               const float* beta, float eps, float momentum, float* moving_mean, float* moving_var,
                               float* save_mean, float* save_invstd, const se_residual* res, int relu, float* y,
                               void* stream) {
  SE_REQUIRE(x && y && stats && gamma && beta && save_mean && save_invstd && rows > 0 && C > 0, "bad arguments");
  Res r = to_res(res);
  long long items = ((C & 3) == 0) ? rows * C / 4 : rows * C;
  launch(bn_fwd_kernel<true>, dim3(ew_grid(ceil_div<long long>(items, 4))), dim3(256), 2 * C * sizeof(float), as_stream(stream), 
      x, rows, C, stats, gamma, beta, eps, momentum, moving_mean, moving_var, save_mean, save_invstd, r, relu, y);
  return check_launch("bn_fwd_kernel<train>");
}

extern "C" int se_bn_fwd_infer(const float* x, int64_t rows, int C, const float* gamma, const float* beta,
                               const float* moving_mean, const float* moving_var, float eps, const se_residual* res,
                               int relu, float* y, void* stream) {
  SE_REQUIRE(x && y && gamma && beta && moving_mean && moving_var && rows > 0 && C > 0, "bad arguments");
  Res r = to_res(res);
  long long items = ((C & 3) == 0) ? rows * C / 4 : rows * C;
  launch(bn_fwd_kernel<false>, dim3(ew_grid(ceil_div<long long>(items, 4))), dim3(256), 2 * C * sizeof(float), as_stream(stream), 
      x, rows, C, nullptr, gamma, beta, eps, 0.f, const_cast<float*>(moving_mean), const_cast<float*>(moving_var),
      nullptr, nullptr, r, relu, y);
  return check_launch("bn_fwd_kernel<infer>");
}

extern "C" int se_bn_bwd(const float* x, const float* y, const float* dout, int64_t rows, int C, const float* gamma,
                         const float* save_mean, const float* save_invstd, int relu, int relu_in, float* dx,
                         float beta_dx, float* dres, float beta_res, float* dgamma, float* dbeta, double* scratch,
                         void* stream) {
  return se::bn_bwd(x, y, dout, rows, C, gamma, save_mean, save_invstd, relu, relu_in, dx, beta_dx, dres, beta_res, dgamma, dbeta,
                    scratch, 0, stream);
}

// `early`: plan-runner hint (se_run_ops): x / y / saved statistics date from the forward pass, prefetch them before the
// programmatic grid dependency resolves.  The public entry point never sets it.
int se::bn_bwd(const float* x, const float* y, const float* dout, int64_t rows, int C, const float* gamma,
               const float* save_mean, const float* save_invstd, int relu, int relu_in, float* dx, float beta_dx, float* dres,
               float beta_res, float* dgamma, float* dbeta, double* scratch, int early, void* stream) {
  SE_REQUIRE(x && dout && dx && gamma && save_mean && save_invstd && scratch && rows > 0 && C > 0, "bad arguments");
  SE_REQUIRE(!relu || y, "relu backward needs y");
  long long per_l = 0;
  int gridf = 0;
  size_t smem = 0;
  const int path = bn_bwd_plan(rows, C, sm_count(), &per_l, &gridf, &smem);
  static const char* bn_trace_env = getenv("SE_BN_TRACE_PTR");
  long long* bn_trace = bn_trace_env ? reinterpret_cast<long long*>(strtoull(bn_trace_env, nullptr, 0)) : nullptr;
  if (path == SE_BN_BWD_SLAB_REG) {
    launch_grid_barrier(bn_bwd_reg_kernel, dim3(gridf), dim3(512), 0, as_stream(stream), x, y ? y : x, dout, rows, C, gamma, save_mean, save_invstd,
           relu, relu_in, dx, beta_dx, dres, beta_res, dgamma, dbeta, scratch, (int)per_l, early ? 1 : 0, bn_trace);
    return check_launch("bn_bwd_reg_kernel");
  }
  if (path == SE_BN_BWD_SLAB_QUAD || path == SE_BN_BWD_SLAB_ATOMIC) {
    // fused single-launch path: every CTA's slab of x and g fits in shared memory (one CTA per SM)
    const int rc = ensure_setup();
    if (rc) return rc;
    // at least 116 KB per CTA would be needed to force one CTA per SM; co-residency only needs grid <= #SMs
    launch_grid_barrier(bn_bwd_fused_kernel, dim3(gridf), dim3(512), smem, as_stream(stream), x, y, dout, rows, C, gamma, save_mean, save_invstd, relu,
                                                                  relu_in, dx, beta_dx, dres, beta_res, dgamma, dbeta,
                                                                  scratch, (int)per_l);
    return check_launch("bn_bwd_fused_kernel");
  }
  int grid;
  int per = red_rows_per_cta(rows, &grid);
  launch(bn_bwd_reduce_kernel, dim3(grid), dim3(256), 2 * C * sizeof(double), as_stream(stream), x, y, dout, rows, C, save_mean,
                                                                                   save_invstd, relu, scratch, per);
  int rc = check_launch("bn_bwd_reduce_kernel");
  if (rc) return rc;
  long long items = ((C & 3) == 0) ? rows * C / 4 : rows * C;
  launch(bn_bwd_apply_kernel, dim3(ew_grid(items)), dim3(256), 4 * C * sizeof(float), as_stream(stream), 
      x, y, dout, rows, C, gamma, save_mean, save_invstd, relu, relu_in, dx, beta_dx, dres, beta_res, dgamma, dbeta,
      scratch);
  return check_launch("bn_bwd_apply_kernel");
}

extern "C" int se_bn_bwd_path(int64_t rows, int C, int sms) {
  SE_REQUIRE(rows > 0 && C > 0, "bad arguments");
  return bn_bwd_plan(rows, C, sms > 0 ? sms : sm_count(), nullptr, nullptr, nullptr);
}

extern "C" int se_shortcut_bwd(const float* dout, const float* y, int relu, int N, int H, int W, int C,
                               const se_residual* res, float* dsrc, float beta, void* stream) {
  SE_REQUIRE(dout && res && dsrc && (!relu || y), "bad arguments");
  SE_REQUIRE(res->pool == 1 || res->pool == 2, "pool must be 1 or 2");
  Res r = to_res(res);
  r.ptr = dsrc;  // only the geometry is used
  long long total = (long long)N * H * r.pool * W * r.pool * r.C;
  launch(shortcut_bwd_kernel, dim3(ew_grid(total)), dim3(256), 0, as_stream(stream), dout, y, relu, N, H, W, C, r, dsrc, beta);
  return check_launch("shortcut_bwd_kernel");
}
