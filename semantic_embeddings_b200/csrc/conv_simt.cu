// fp32 FFMA convolution kernels ("parity mode", SE_MODE_F32) -- implicit GEMM over NHWC / HWIO.
//
// These are the exact-fp32 counterpart of the tensor-core path (conv_tc.cu) and the fallback for the
// shapes that path does not cover (Cin=3 stem, stride-2 layers, 7x7, dense layers).  They stand for
// the Conv2D / Dense ops of the reference graph (models/cifar_resnet.py:96-105,218,233;
// models/plainnet.py:52,67,70,76; models/wide_residual_network.py:9-53,96) and their autodiff
// gradients (learn_image_embeddings.py:238).
//
//   forward : Y[m, co]   = sum_{tap,ci} X[pix(m,tap), ci] * W[tap, ci, co]      M = N*Ho*Wo
//   dgrad   : dX[m, ci]  = sum_{tap,co} dY[opix(m,tap), co] * W[tap, ci, co]    M = N*H*W
//   wgrad   : dW[tap,ci,co] = sum_m X[pix(m,tap), ci] * dY[m, co]               reduction over pixels
#include <algorithm>

#include "common.cuh"
#include "conv_plan.cuh"

namespace se {

struct ConvP {
  int N, H, W, Cin, Cout, kh, kw, stride, pad_t, pad_l, Ho, Wo;
};

static ConvP to_p(const se_conv_desc* d) {
  ConvP p;
  p.N = d->N; p.H = d->H; p.W = d->W; p.Cin = d->Cin; p.Cout = d->Cout; p.kh = d->kh; p.kw = d->kw;
  p.stride = d->stride; p.pad_t = d->pad_t; p.pad_l = d->pad_l; p.Ho = d->Ho; p.Wo = d->Wo;
  return p;
}

constexpr size_t WGRAD3X3_MAX_SMEM = 160 * 1024;

// ---------------------------------------------------------------------------------------- forward
template <int BM, int BN, int TM, int TN, bool VEC>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
conv_fwd_kernel(ConvP p, const float* __restrict__ x, const float* __restrict__ w,
                const float* __restrict__ bias, const float* __restrict__ residual, float* __restrict__ y,
                int relu, double* __restrict__ stats) {
  pdl_grid_sync();
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int CG = BN / TN;  // threads along the channel dimension
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  __shared__ long long row_off[BM];
  __shared__ int row_h0[BM], row_w0[BM];
  __shared__ double s_sum[BN], s_sq[BN];

  const int tid = threadIdx.x;
  const int tn = tid % CG, tm = tid / CG;
  const long long M = (long long)p.N * p.Ho * p.Wo;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  for (int r = tid; r < BM; r += NT) {
    long long m = m0 + r;
    if (m < M) {
      int ow = (int)(m % p.Wo);
      long long t = m / p.Wo;
      int oh = (int)(t % p.Ho);
      int n = (int)(t / p.Ho);
      int h0 = oh * p.stride - p.pad_t, w0 = ow * p.stride - p.pad_l;
      row_h0[r] = h0;
      row_w0[r] = w0;
      row_off[r] = (((long long)n * p.H + h0) * p.W + w0) * p.Cin;
    } else {
      row_h0[r] = -(1 << 28);
      row_w0[r] = -(1 << 28);
      row_off[r] = 0;
    }
  }
  if (tid < BN) { s_sum[tid] = 0.0; s_sq[tid] = 0.0; }
  __syncthreads();

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int taps = p.kh * p.kw;
  for (int tap = 0; tap < taps; ++tap) {
    const int fr = tap / p.kw, fs = tap % p.kw;
    const long long tap_off = ((long long)fr * p.W + fs) * p.Cin;
    for (int ci0 = 0; ci0 < p.Cin; ci0 += BK) {
      if (VEC) {
        for (int idx = tid; idx < BM * (BK / 4); idx += NT) {
          int row = idx / (BK / 4), kq = idx % (BK / 4);
          int ih = row_h0[row] + fr, iw = row_w0[row] + fs;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ih >= 0 && ih < p.H && iw >= 0 && iw < p.W && ci0 + 4 * kq < p.Cin)
            v = *reinterpret_cast<const float4*>(x + row_off[row] + tap_off + ci0 + 4 * kq);
          As[4 * kq + 0][row] = v.x; As[4 * kq + 1][row] = v.y;
          As[4 * kq + 2][row] = v.z; As[4 * kq + 3][row] = v.w;
        }
        for (int idx = tid; idx < BK * (BN / 4); idx += NT) {
          int k = idx / (BN / 4), nq = idx % (BN / 4);
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ci0 + k < p.Cin && n0 + 4 * nq < p.Cout)
            v = *reinterpret_cast<const float4*>(w + ((long long)tap * p.Cin + ci0 + k) * p.Cout + n0 + 4 * nq);
          *reinterpret_cast<float4*>(&Bs[k][4 * nq]) = v;
        }
      } else {
        for (int idx = tid; idx < BM * BK; idx += NT) {
          int row = idx / BK, k = idx % BK;
          int ih = row_h0[row] + fr, iw = row_w0[row] + fs;
          float v = 0.f;
          if (ih >= 0 && ih < p.H && iw >= 0 && iw < p.W && ci0 + k < p.Cin)
            v = x[row_off[row] + tap_off + ci0 + k];
          As[k][row] = v;
        }
        for (int idx = tid; idx < BK * BN; idx += NT) {
          int k = idx / BN, n = idx % BN;
          float v = 0.f;
          if (ci0 + k < p.Cin && n0 + n < p.Cout) v = w[((long long)tap * p.Cin + ci0 + k) * p.Cout + n0 + n];
          Bs[k][n] = v;
        }
      }
      __syncthreads();
      tile_fma<BM, BN, TM, TN>(As, Bs, tm, tn, acc);
      __syncthreads();
    }
  }

  // epilogue: bias, residual, relu, store, BatchNorm statistics of the stored values
  float csum[TN], csq[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) { csum[j] = 0.f; csq[j] = 0.f; }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    long long m = m0 + tm * TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int co = n0 + tn * TN + j;
      if (co >= p.Cout) continue;
      float v = acc[i][j];
      if (bias) v += bias[co];
      if (residual) v += residual[m * p.Cout + co];
      if (relu) v = fmaxf(v, 0.f);
      y[m * p.Cout + co] = v;
      csum[j] += v;
      csq[j] += v * v;
    }
  }
  if (stats) {
    // lanes that share `tn` own the same channels: reduce them with shuffles first (CG divides 32)
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      float a = csum[j], b = csq[j];
      for (int o = CG; o < 32; o <<= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
      }
      if ((tid & 31) < CG) {
        atomicAdd(&s_sum[tn * TN + j], (double)a);
        atomicAdd(&s_sq[tn * TN + j], (double)b);
      }
    }
    __syncthreads();
    if (tid < BN && n0 + tid < p.Cout) {
      atomicAdd(&stats[n0 + tid], s_sum[tid]);
      atomicAdd(&stats[p.Cout + n0 + tid], s_sq[tid]);
    }
  }
}

// ---------------------------------------------------------------------------------------- dgrad
template <int BM, int BN, int TM, int TN, bool VEC>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
conv_dgrad_kernel(ConvP p, const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx,
                  float beta, int par) {
  // par != 0 (stride 2, even H and W): GEMM rows are ordered (parity class, n, h/2, w/2) so that a CTA only holds
  // input pixels of one (h & 1, w & 1) class -- for which only the filter taps of matching parity contribute.  The
  // other taps (3/4 of the 3x3 window on average) are skipped instead of being multiplied by zeros.
  pdl_grid_sync();
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int CG = BN / TN;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  __shared__ int row_n[BM], row_h[BM], row_w[BM];

  const int tid = threadIdx.x;
  const int tn = tid % CG, tm = tid / CG;
  const long long M = (long long)p.N * p.H * p.W;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;  // input-channel tile

  const long long Q = (long long)p.N * (p.H / 2) * (p.W / 2);      // pixels per parity class (par only)
  const int cls = par ? (int)(m0 / Q) : 0;                        // uniform in the CTA: Q % BM == 0 (checked by the host)
  for (int r = tid; r < BM; r += NT) {
    long long m = m0 + r;
    if (m < M) {
      if (par) {
        long long rem = m - (long long)cls * Q;
        const int W2 = p.W / 2, H2 = p.H / 2;
        row_w[r] = 2 * (int)(rem % W2) + (cls & 1);
        long long t = rem / W2;
        row_h[r] = 2 * (int)(t % H2) + (cls >> 1);
        row_n[r] = (int)(t / H2);
      } else {
        row_w[r] = (int)(m % p.W);
        long long t = m / p.W;
        row_h[r] = (int)(t % p.H);
        row_n[r] = (int)(t / p.H);
      }
    } else {
      row_n[r] = -1; row_h[r] = 0; row_w[r] = 0;
    }
  }
  __syncthreads();

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int taps = p.kh * p.kw;
  for (int tap = 0; tap < taps; ++tap) {
    const int fr = tap / p.kw, fs = tap % p.kw;
    if (par && ((((cls >> 1) + p.pad_t - fr) & 1) || (((cls & 1) + p.pad_l - fs) & 1))) continue;   // tap of the other parity
    for (int co0 = 0; co0 < p.Cout; co0 += BK) {
      // A[m, k=co] = dy[n, (ih+pad_t-fr)/s, (iw+pad_l-fs)/s, co] when divisible and in range
      if (VEC) {
        for (int idx = tid; idx < BM * (BK / 4); idx += NT) {
          int row = idx / (BK / 4), kq = idx % (BK / 4);
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          int n = row_n[row];
          int th = row_h[row] + p.pad_t - fr, tw = row_w[row] + p.pad_l - fs;
          if (n >= 0 && th >= 0 && tw >= 0 && (th % p.stride) == 0 && (tw % p.stride) == 0 && co0 + 4 * kq < p.Cout) {
            int oh = th / p.stride, ow = tw / p.stride;
            if (oh < p.Ho && ow < p.Wo)
              v = *reinterpret_cast<const float4*>(dy + (((long long)n * p.Ho + oh) * p.Wo + ow) * p.Cout + co0 + 4 * kq);
          }
          As[4 * kq + 0][row] = v.x; As[4 * kq + 1][row] = v.y;
          As[4 * kq + 2][row] = v.z; As[4 * kq + 3][row] = v.w;
        }
        // B[k=co, n=ci] = w[tap, ci, co]
        for (int idx = tid; idx < BN * (BK / 4); idx += NT) {
          int n = idx / (BK / 4), kq = idx % (BK / 4);
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (n0 + n < p.Cin && co0 + 4 * kq < p.Cout)
            v = *reinterpret_cast<const float4*>(w + ((long long)tap * p.Cin + n0 + n) * p.Cout + co0 + 4 * kq);
          Bs[4 * kq + 0][n] = v.x; Bs[4 * kq + 1][n] = v.y;
          Bs[4 * kq + 2][n] = v.z; Bs[4 * kq + 3][n] = v.w;
        }
      } else {
        for (int idx = tid; idx < BM * BK; idx += NT) {
          int row = idx / BK, k = idx % BK;
          float v = 0.f;
          int n = row_n[row];
          int th = row_h[row] + p.pad_t - fr, tw = row_w[row] + p.pad_l - fs;
          if (n >= 0 && th >= 0 && tw >= 0 && (th % p.stride) == 0 && (tw % p.stride) == 0 && co0 + k < p.Cout) {
            int oh = th / p.stride, ow = tw / p.stride;
            if (oh < p.Ho && ow < p.Wo) v = dy[(((long long)n * p.Ho + oh) * p.Wo + ow) * p.Cout + co0 + k];
          }
          As[k][row] = v;
        }
        for (int idx = tid; idx < BN * BK; idx += NT) {
          int n = idx / BK, k = idx % BK;
          float v = 0.f;
          if (n0 + n < p.Cin && co0 + k < p.Cout) v = w[((long long)tap * p.Cin + n0 + n) * p.Cout + co0 + k];
          Bs[k][n] = v;
        }
      }
      __syncthreads();
      tile_fma<BM, BN, TM, TN>(As, Bs, tm, tn, acc);
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    long long m = m0 + tm * TM + i;
    if (m >= M) continue;
    const int rr = tm * TM + i;
    const long long pix = par ? ((long long)row_n[rr] * p.H + row_h[rr]) * p.W + row_w[rr] : m;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int ci = n0 + tn * TN + j;
      if (ci >= p.Cin) continue;
      float v = acc[i][j];
      if (beta != 0.f) v += beta * dx[pix * p.Cin + ci];
      dx[pix * p.Cin + ci] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------- wgrad (generic)
// M' = kh*kw*Cin (flattened kk), N' = Cout, reduction over output pixels split across blockIdx.z.
template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
conv_wgrad_kernel(ConvP p, const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw,
                  float* __restrict__ dbias, long long pix_per_split, int direct) {
  pdl_grid_sync();
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int CG = BN / TN;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  __shared__ long long pix_off[BK];
  __shared__ int pix_h0[BK], pix_w0[BK];
  __shared__ int kk_tap_off[BM], kk_r[BM], kk_s[BM];

  const int tid = threadIdx.x;
  const int tn = tid % CG, tm = tid / CG;
  const int KK = p.kh * p.kw * p.Cin;
  const long long T = (long long)KK * p.Cout;   // dw / dbias: workspace slices, one per split (wgrad_reduce), or direct
  const int m0 = blockIdx.x * BM;  // kk tile
  const int n0 = blockIdx.y * BN;  // cout tile
  const long long P = (long long)p.N * p.Ho * p.Wo;
  const long long pbeg = (long long)blockIdx.z * pix_per_split;
  const long long pend = min(P, pbeg + pix_per_split);

  for (int r = tid; r < BM; r += NT) {
    int kk = m0 + r;
    if (kk < KK) {
      int tap = kk / p.Cin, ci = kk % p.Cin;
      int fr = tap / p.kw, fs = tap % p.kw;
      kk_r[r] = fr; kk_s[r] = fs;
      kk_tap_off[r] = (fr * p.W + fs) * p.Cin + ci;
    } else {
      kk_r[r] = 1 << 28; kk_s[r] = 1 << 28; kk_tap_off[r] = 0;
    }
  }
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  float bsum = 0.f;
  const bool do_bias = (dbias != nullptr) && blockIdx.x == 0 && tid < BN;

  for (long long pc = pbeg; pc < pend; pc += BK) {
    __syncthreads();
    if (tid < BK) {
      long long m = pc + tid;
      if (m < pend) {
        int ow = (int)(m % p.Wo);
        long long t = m / p.Wo;
        int oh = (int)(t % p.Ho);
        int n = (int)(t / p.Ho);
        int h0 = oh * p.stride - p.pad_t, w0 = ow * p.stride - p.pad_l;
        pix_h0[tid] = h0; pix_w0[tid] = w0;
        pix_off[tid] = (((long long)n * p.H + h0) * p.W + w0) * p.Cin;
      } else {
        pix_h0[tid] = -(1 << 28); pix_w0[tid] = -(1 << 28); pix_off[tid] = 0;
      }
    }
    __syncthreads();
    for (int idx = tid; idx < BK * BM; idx += NT) {
      int k = idx / BM, mm = idx % BM;
      int ih = pix_h0[k] + kk_r[mm], iw = pix_w0[k] + kk_s[mm];
      float v = 0.f;
      if (ih >= 0 && ih < p.H && iw >= 0 && iw < p.W) v = x[pix_off[k] + kk_tap_off[mm]];
      As[k][mm] = v;
    }
    for (int idx = tid; idx < BK * BN; idx += NT) {
      int k = idx / BN, n = idx % BN;
      float v = 0.f;
      if (pc + k < pend && n0 + n < p.Cout) v = dy[(pc + k) * p.Cout + n0 + n];
      Bs[k][n] = v;
    }
    __syncthreads();
    tile_fma<BM, BN, TM, TN>(As, Bs, tm, tn, acc);
    if (do_bias) {
#pragma unroll
      for (int k = 0; k < BK; ++k) bsum += Bs[k][tid];
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int kk = m0 + tm * TM + i;
    if (kk >= KK) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int co = n0 + tn * TN + j;
      if (co >= p.Cout) continue;
      if (direct) atomicAdd(&dw[(long long)kk * p.Cout + co], acc[i][j]);
      else dw[blockIdx.z * T + (long long)kk * p.Cout + co] = acc[i][j];
    }
  }
  if (do_bias && n0 + tid < p.Cout) {
    if (direct) atomicAdd(&dbias[n0 + tid], bsum);
    else dbias[(long long)blockIdx.z * p.Cout + n0 + tid] = bsum;
  }
}

// ---------------------------------------------------------------------------------------- wgrad 3x3 stride 1 'same'
// One CTA walks over (image, row-band) tiles with the 9 x 2 x 2 partial sums of its (ci, co) pairs in registers:
// per pixel a thread reads 3x2 new x values and 2 dy values from shared memory for 36 FMAs (sliding 3x3 window,
// 2x2 register block).  NCI x NCO threads cover the channel tile; when that is fewer than 256 (16-channel layers)
// the remaining threads form RG "row groups" that take alternate rows of the band and are reduced through shared
// memory at the end, so that all 256 threads have work.  The result is added into dW once per CTA.
template <int NCI, int NCO>
__global__ void __launch_bounds__(256)
conv_wgrad3x3_kernel(ConvP p, const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw,
                     float* __restrict__ dbias, int TH, int tiles_per_img, int num_tiles, int direct) {
  pdl_grid_sync();
  constexpr int CI_T = 2, CO_T = 2;
  constexpr int CIT = NCI * CI_T, COT = NCO * CO_T;
  constexpr int PAIRS = NCI * NCO, RG = 256 / PAIRS;
  extern __shared__ __align__(16) float smem[];
  const int W = p.W, H = p.H;
  float* xs = smem;                                   // [(TH+2)][(W+2)][CIT]
  float* ds = smem + (TH + 2) * (W + 2) * CIT;        // [TH][W][COT]
  const int tid = threadIdx.x;
  const int pair = tid % PAIRS, rg = tid / PAIRS;
  const int tco = pair % NCO, tci = pair / NCO;
  const int ci0 = blockIdx.y * CIT, co0 = blockIdx.z * COT;

  float acc[3][3][CI_T][CO_T];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int s = 0; s < 3; ++s)
#pragma unroll
      for (int a = 0; a < CI_T; ++a)
#pragma unroll
        for (int b = 0; b < CO_T; ++b) acc[r][s][a][b] = 0.f;
  float bacc[CO_T];
#pragma unroll
  for (int b = 0; b < CO_T; ++b) bacc[b] = 0.f;

  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int n = tile / tiles_per_img;
    const int h0 = (tile % tiles_per_img) * TH;
    const int th = min(TH, H - h0);
    __syncthreads();
    // x halo band: rows h0-1 .. h0+th, cols -1 .. W, zero outside the image ('same' padding)
    const int xq = CIT / 4;
    for (int idx = tid; idx < (th + 2) * (W + 2) * xq; idx += 256) {
      int q = idx % xq;
      int t = idx / xq;
      int cw = t % (W + 2), rh = t / (W + 2);
      int ih = h0 + rh - 1, iw = cw - 1;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ih >= 0 && ih < H && iw >= 0 && iw < W)
        v = *reinterpret_cast<const float4*>(x + (((long long)n * H + ih) * W + iw) * p.Cin + ci0 + 4 * q);
      *reinterpret_cast<float4*>(xs + (rh * (W + 2) + cw) * CIT + 4 * q) = v;
    }
    const int dq = COT / 4;
    for (int idx = tid; idx < th * W * dq; idx += 256) {
      int q = idx % dq;
      int t = idx / dq;
      float4 v = *reinterpret_cast<const float4*>(dy + (((long long)n * H + h0) * W + t) * p.Cout + co0 + 4 * q);
      *reinterpret_cast<float4*>(ds + t * COT + 4 * q) = v;
    }
    __syncthreads();
    for (int h = rg; h < th; h += RG) {
      float win[3][2][CI_T];  // previous two columns of the three halo rows
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int a = 0; a < CI_T; ++a) {
          win[r][0][a] = xs[((h + r) * (W + 2) + 0) * CIT + tci + NCI * a];
          win[r][1][a] = xs[((h + r) * (W + 2) + 1) * CIT + tci + NCI * a];
        }
      for (int wcol = 0; wcol < W; ++wcol) {
        float d[CO_T];
#pragma unroll
        for (int b = 0; b < CO_T; ++b) d[b] = ds[(h * W + wcol) * COT + tco + NCO * b];
        if (tci == 0) {
#pragma unroll
          for (int b = 0; b < CO_T; ++b) bacc[b] += d[b];
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          float xc[CI_T];
#pragma unroll
          for (int a = 0; a < CI_T; ++a) xc[a] = xs[((h + r) * (W + 2) + wcol + 2) * CIT + tci + NCI * a];
#pragma unroll
          for (int a = 0; a < CI_T; ++a)
#pragma unroll
            for (int b = 0; b < CO_T; ++b) {
              acc[r][0][a][b] = fmaf(win[r][0][a], d[b], acc[r][0][a][b]);
              acc[r][1][a][b] = fmaf(win[r][1][a], d[b], acc[r][1][a][b]);
              acc[r][2][a][b] = fmaf(xc[a], d[b], acc[r][2][a][b]);
            }
#pragma unroll
          for (int a = 0; a < CI_T; ++a) { win[r][0][a] = win[r][1][a]; win[r][1][a] = xc[a]; }
        }
      }
    }
  }
  if (RG > 1) {
    // combine the row groups: red[rg][(r,s,a,b)][pair] in shared memory (reuses the tile buffers)
    __syncthreads();
    float* red = smem;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s = 0; s < 3; ++s)
#pragma unroll
        for (int a = 0; a < CI_T; ++a)
#pragma unroll
          for (int b = 0; b < CO_T; ++b)
            red[(rg * 36 + ((r * 3 + s) * CI_T + a) * CO_T + b) * PAIRS + pair] = acc[r][s][a][b];
    float* redb = smem + RG * 36 * PAIRS;
    if (tci == 0) {
#pragma unroll
      for (int b = 0; b < CO_T; ++b) redb[(rg * CO_T + b) * NCO + tco] = bacc[b];
    }
    __syncthreads();
    if (rg == 0) {
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int s = 0; s < 3; ++s)
#pragma unroll
          for (int a = 0; a < CI_T; ++a)
#pragma unroll
            for (int b = 0; b < CO_T; ++b) {
              float v = 0.f;
#pragma unroll
              for (int g = 0; g < RG; ++g) v += red[(g * 36 + ((r * 3 + s) * CI_T + a) * CO_T + b) * PAIRS + pair];
              acc[r][s][a][b] = v;
            }
      if (tci == 0) {
#pragma unroll
        for (int b = 0; b < CO_T; ++b) {
          float v = 0.f;
#pragma unroll
          for (int g = 0; g < RG; ++g) v += redb[(g * CO_T + b) * NCO + tco];
          bacc[b] = v;
        }
      }
    }
  }
  if (rg == 0) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s = 0; s < 3; ++s)
#pragma unroll
        for (int a = 0; a < CI_T; ++a)
#pragma unroll
          for (int b = 0; b < CO_T; ++b) {
            int ci = ci0 + tci + NCI * a, co = co0 + tco + NCO * b;
            const long long o = ((long long)(r * 3 + s) * p.Cin + ci) * p.Cout + co;
            if (direct) atomicAdd(&dw[o], acc[r][s][a][b]);
            else dw[blockIdx.x * 9LL * p.Cin * p.Cout + o] = acc[r][s][a][b];
          }
    if (dbias != nullptr && tci == 0 && blockIdx.y == 0) {   // dw / dbias: workspace slices, one per CTA column (wgrad_reduce)
#pragma unroll
      for (int b = 0; b < CO_T; ++b) {
        if (direct) atomicAdd(&dbias[co0 + tco + NCO * b], bacc[b]);
        else dbias[(long long)blockIdx.x * p.Cout + co0 + tco + NCO * b] = bacc[b];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------- launchers
int init_conv_simt() {
  cudaError_t e = cudaSuccess;
  auto set = [&](auto kern) {
    if (e == cudaSuccess) e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WGRAD3X3_MAX_SMEM);
  };
  set(conv_wgrad3x3_kernel<16, 16>); set(conv_wgrad3x3_kernel<8, 16>); set(conv_wgrad3x3_kernel<16, 8>); set(conv_wgrad3x3_kernel<8, 8>);
  if (e != cudaSuccess) { set_error("init_conv_simt: %s", cudaGetErrorString(e)); return SE_ERR_CUDA; }
  return SE_OK;
}

// Forward of the RGB stem (3x3 / stride 1 / 'same', Cin <= 4, Cout == 16; models/cifar_resnet.py:218 `conv0`): one thread
// per output pixel keeps all 16 output channels in registers; the 8-row input tile (with its zero halo), the filter
// and the bias sit in shared memory.  The tiled-GEMM kernel above spends a 16-deep K step on K = 27 and measured
// 54 us; this is bound by its 432 FMAs per pixel.  BatchNorm statistics: warp butterfly -> per-warp slots -> one
// float64 atomic per channel and CTA.
__global__ void __launch_bounds__(256)
conv_fwd_stem_kernel(ConvP p, const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                     float* __restrict__ y, int relu, double* __restrict__ stats, int TH) {
  pdl_grid_sync();
  extern __shared__ __align__(16) float fsm[];
  constexpr int CO = 16;
  const int Wp = p.W + 2, KK = 9 * p.Cin;
  float* ws = fsm;                                   // [KK][16]
  float* bs = ws + KK * CO;                          // [16]
  float* xs = bs + CO;                               // [(TH+2)][Wp][Cin]
  float* sst = xs + (((TH + 2) * Wp * p.Cin + 3) & ~3);   // [8 warps][32]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tiles_per_img = p.H / TH;
  const int n = blockIdx.x / tiles_per_img, h0 = (blockIdx.x - n * tiles_per_img) * TH;
  for (int i = tid; i < KK * CO; i += blockDim.x) ws[i] = w[i];
  if (tid < CO) bs[tid] = bias ? bias[tid] : 0.f;
  for (int i = tid; i < (TH + 2) * Wp * p.Cin; i += blockDim.x) {
    const int ci = i % p.Cin, q = i / p.Cin, ww = q % Wp - 1, hh = h0 + q / Wp - 1;
    xs[i] = (hh >= 0 && hh < p.H && ww >= 0 && ww < p.W) ? x[(((long long)n * p.H + hh) * p.W + ww) * p.Cin + ci] : 0.f;
  }
  if (stats) for (int i = tid; i < 8 * 32; i += blockDim.x) sst[i] = 0.f;
  __syncthreads();
  const int npx = TH * p.W;
  for (int px = tid; px < npx; px += blockDim.x) {   // npx is a multiple of 32: warps stay whole
    const int hl = px / p.W, wl = px - hl * p.W;
    float o[CO];
#pragma unroll
    for (int c = 0; c < CO; ++c) o[c] = bs[c];
    for (int tap = 0; tap < 9; ++tap) {
      const float* xp = xs + ((hl + tap / 3) * Wp + wl + tap % 3) * p.Cin;
      for (int ci = 0; ci < p.Cin; ++ci) {
        const float xv = xp[ci];
        const float4* wr = reinterpret_cast<const float4*>(ws + (tap * p.Cin + ci) * CO);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 wv = wr[q];
          o[4 * q] = fmaf(xv, wv.x, o[4 * q]); o[4 * q + 1] = fmaf(xv, wv.y, o[4 * q + 1]);
          o[4 * q + 2] = fmaf(xv, wv.z, o[4 * q + 2]); o[4 * q + 3] = fmaf(xv, wv.w, o[4 * q + 3]);
        }
      }
    }
    if (relu) {
#pragma unroll
      for (int c = 0; c < CO; ++c) o[c] = fmaxf(o[c], 0.f);
    }
    float4* dst = reinterpret_cast<float4*>(y + (((long long)n * p.H + h0 + hl) * p.W + wl) * CO);
#pragma unroll
    for (int q = 0; q < 4; ++q) dst[q] = make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
    if (stats) {
      // column sums over the warp's 32 pixels: after 5 xor-shuffle rounds every lane holds the totals
#pragma unroll
      for (int c = 0; c < CO; ++c) {
        float sv = o[c], qv = o[c] * o[c];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) { sv += __shfl_xor_sync(0xffffffffu, sv, off); qv += __shfl_xor_sync(0xffffffffu, qv, off); }
        if (lane == c) { sst[warp * 32 + c] += sv; sst[warp * 32 + CO + c] += qv; }
      }
    }
  }
  if (stats) {
    __syncthreads();
    if (tid < 2 * CO) {
      double v = 0.0;
      for (int wv = 0; wv < (int)(blockDim.x >> 5); ++wv) v += (double)sst[wv * 32 + tid];
      atomicAdd(&stats[tid], v);
    }
  }
}

// Dense layer on a skinny batch (the 2048 -> 555 'embedding' layer of config 4 at 32 rows: utils.py:242): the generic
// tile kernel has 9 CTAs walking K = 2048 serially (0.42 ms).  Here a CTA owns 8 output columns and splits K over 32
// thread groups (each thread 4 consecutive k per step: one 16-byte load of x per row, four of w), 32 rows of fp32
// accumulators per thread, one shared-memory reduction at the end.  y = x W + b [relu].
constexpr int DS_COLS = 8, DS_KL = 32, DS_ROWS = 32;
__global__ void __launch_bounds__(DS_COLS * DS_KL)
dense_small_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                       float* __restrict__ y, int B, int Cin, int Cout, int relu) {
  pdl_grid_sync();
  __shared__ float red[DS_KL][DS_ROWS][DS_COLS + 1];
  const int c = threadIdx.x % DS_COLS, kl = threadIdx.x / DS_COLS;
  const int col = blockIdx.x * DS_COLS + c;
  const bool col_ok = col < Cout;
  for (int r0 = 0; r0 < B; r0 += DS_ROWS) {
    float acc[DS_ROWS];
#pragma unroll
    for (int b = 0; b < DS_ROWS; ++b) acc[b] = 0.f;
    for (int k = kl * 4; k < Cin; k += DS_KL * 4) {
      float wv[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) wv[j] = col_ok ? __ldg(w + (long long)(k + j) * Cout + col) : 0.f;
#pragma unroll
      for (int b = 0; b < DS_ROWS; ++b) {
        if (r0 + b < B) {
          const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (long long)(r0 + b) * Cin + k));
          acc[b] = fmaf(xv.x, wv[0], acc[b]); acc[b] = fmaf(xv.y, wv[1], acc[b]);
          acc[b] = fmaf(xv.z, wv[2], acc[b]); acc[b] = fmaf(xv.w, wv[3], acc[b]);
        }
      }
    }
    __syncthreads();                                   // (the previous row chunk's reduction has been read)
#pragma unroll
    for (int b = 0; b < DS_ROWS; ++b) red[kl][b][c] = acc[b];
    __syncthreads();
    for (int o = threadIdx.x; o < DS_ROWS * DS_COLS; o += DS_COLS * DS_KL) {
      const int b = o / DS_COLS, cc = o % DS_COLS, oc = blockIdx.x * DS_COLS + cc;
      if (r0 + b < B && oc < Cout) {
        float s = 0.f;
#pragma unroll 8
        for (int g = 0; g < DS_KL; ++g) s += red[g][b][cc];
        if (bias) s += bias[oc];
        if (relu) s = fmaxf(s, 0.f);
        y[(long long)(r0 + b) * Cout + oc] = s;
      }
    }
  }
}

// Weight gradient of a 3x3 / stride 1 / 'same' convolution with very few input channels (the RGB stem,
// models/cifar_resnet.py:218 `conv0`): the 27 x Cout outputs are far too small for the tiled GEMM above (64x64 tiles
// at 1/6 occupancy, 293-way split-K: 123 us).  Here one thread owns (k = (tap, ci) or the bias row, 4 output channels)
// for one of PG pixel groups of a 8-row tile staged in shared memory: 2 shared loads per 4 FMAs, a shared-memory
// combine of the pixel groups, then one partial per output and CTA.  Persistent over the tiles.
__global__ void __launch_bounds__(512)
conv_wgrad_stem_kernel(ConvP p, const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw,
                       float* __restrict__ dbias, int TH, int PG, int num_tiles, int direct) {
  pdl_grid_sync();
  extern __shared__ __align__(16) float ssm[];
  const int Wp = p.W + 2;
  const int KK = 9 * p.Cin;                       // rows of dW; row KK is the bias (x == 1)
  const int CQ = p.Cout >> 2;
  const int per_pg = (KK + 1) * CQ;               // threads of one pixel group
  float* xs = ssm;                                // [(TH+2)][Wp][Cin], zero halo
  float* dys = xs + (((TH + 2) * Wp * p.Cin + 3) & ~3);   // [TH*W][Cout]
  float* red = dys + TH * p.W * p.Cout;           // [PG-1][per_pg][4]
  const int tid = threadIdx.x;
  const bool worker = tid < PG * per_pg;
  const int pg = tid / per_pg, rem = tid - pg * per_pg;
  const int k = rem / CQ, cq = rem - k * CQ;
  int xoff = 0;                                   // offset of this thread's (tap, ci) inside the padded x tile
  if (k < KK) { const int tap = k / p.Cin, ci = k - tap * p.Cin; xoff = ((tap / 3) * Wp + (tap % 3)) * p.Cin + ci; }
  const int tiles_per_img = p.H / TH;
  const int px = TH * p.W, px_pg = px / PG;
  const int lw = 31 - __clz(p.W);
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int n = t / tiles_per_img, h0 = (t - n * tiles_per_img) * TH;
    __syncthreads();                              // previous tile fully consumed
    for (int i = tid; i < (TH + 2) * Wp * p.Cin; i += blockDim.x) {
      const int ci = i % p.Cin, q = i / p.Cin, w = q % Wp - 1, h = h0 + q / Wp - 1;
      xs[i] = (h >= 0 && h < p.H && w >= 0 && w < p.W) ? x[(((long long)n * p.H + h) * p.W + w) * p.Cin + ci] : 0.f;
    }
    const float4* gsrc = reinterpret_cast<const float4*>(dy + ((long long)n * p.H + h0) * p.W * p.Cout);
    for (int i = tid; i < px * p.Cout / 4; i += blockDim.x) reinterpret_cast<float4*>(dys)[i] = gsrc[i];
    __syncthreads();
    if (worker) {
      const int p0 = pg * px_pg;
#pragma unroll 4
      for (int j = 0; j < px_pg; ++j) {
        const int pp = p0 + j, h = pp >> lw, w = pp & (p.W - 1);          // W is a power of two
        const float xv = (k < KK) ? xs[(h * Wp + w) * p.Cin + xoff] : 1.f;
        const float4 g = *reinterpret_cast<const float4*>(dys + pp * p.Cout + 4 * cq);
        a0 = fmaf(xv, g.x, a0); a1 = fmaf(xv, g.y, a1); a2 = fmaf(xv, g.z, a2); a3 = fmaf(xv, g.w, a3);
      }
    }
  }
  __syncthreads();
  if (worker && pg > 0) *reinterpret_cast<float4*>(red + ((pg - 1) * per_pg + rem) * 4) = make_float4(a0, a1, a2, a3);
  __syncthreads();
  if (worker && pg == 0) {
    for (int g = 1; g < PG; ++g) {
      const float4 o = *reinterpret_cast<const float4*>(red + ((g - 1) * per_pg + rem) * 4);
      a0 += o.x; a1 += o.y; a2 += o.z; a3 += o.w;
    }
    // dw / dbias: workspace slices, one per CTA (wgrad_reduce), or direct
    const long long sl = direct ? 0 : blockIdx.x;
    float* dst = (k < KK) ? dw + sl * KK * p.Cout + (long long)k * p.Cout + 4 * cq : (dbias ? dbias + sl * p.Cout + 4 * cq : nullptr);
    if (dst && direct) { atomicAdd(dst, a0); atomicAdd(dst + 1, a1); atomicAdd(dst + 2, a2); atomicAdd(dst + 3, a3); }
    else if (dst) *reinterpret_cast<float4*>(dst) = make_float4(a0, a1, a2, a3);
  }
}

// ---------------------------------------------------------------------------------------- host side
constexpr long long WGRAD_LONG_PX = 1LL << 18, WGRAD_SPLIT_PX = 2048;   // see the split count below

static int stem_rows(int H) { return (H % 8 == 0) ? 8 : ((H % 4 == 0) ? 4 : 1); }

// The fp32 kernel of a call that no tensor-core family takes, and its launch configuration (conv_plan)
void simt_config(const se_conv_desc* d, int dir, const ConvCall& c, ConvPlan* pl) {
  SimtParams& f = pl->fp;
  const bool same3x3 = d->kh == 3 && d->kw == 3 && d->stride == 1 && d->pad_t == 1 && d->pad_l == 1 && d->Ho == d->H &&
                       d->Wo == d->W;
  pl->block = dim3(256);
  if (dir == 0) {
    pl->fused_stats = c.stats;                      // every fp32 forward kernel sums them in its epilogue
    if (d->kh == 1 && d->kw == 1 && d->H == 1 && d->W == 1 && d->Ho == 1 && d->Wo == 1 && d->N <= 64 && d->Cin >= 512 &&
        d->Cin % 4 == 0 && !c.residual && !c.stats && c.x_aligned) {
      pl->grid = dim3(ceil_div(d->Cout, DS_COLS));
      pl->block = dim3(DS_COLS * DS_KL);
      pl->family = CONV_FP32_DENSE_SMALL;
      return;
    }
    if (same3x3 && d->Cin <= 4 && !c.residual && d->Cout == 16 && d->W % 32 == 0 && d->W <= 64 && c.y_aligned) {
      f.TH = stem_rows(d->H);
      const size_t smem = ((size_t)9 * d->Cin * 16 + 16 + (((f.TH + 2) * (d->W + 2) * d->Cin + 3) & ~3) + 8 * 32) * sizeof(float);
      if (smem <= 48 * 1024) {
        pl->grid = dim3(d->N * (d->H / f.TH));
        pl->smem = smem;
        pl->family = CONV_FP32_FWD_STEM;
        return;
      }
    }
  }
  if (dir < 2) {
    // conv_fwd_kernel / conv_dgrad_kernel: the tile by the GEMM's N channels (forward Cout, data gradient Cin)
    const int Nc = dir == 0 ? d->Cout : d->Cin;
    f.bn = Nc <= 16 ? 16 : Nc <= 32 ? 32 : 64;
    const int BM = f.bn == 64 ? 64 : 128;
    const long long M = dir == 0 ? (long long)d->N * d->Ho * d->Wo : (long long)d->N * d->H * d->W;
    f.vec = dir == 0 ? d->Cin % 4 == 0 && d->Cout % 4 == 0 : d->Cout % 4 == 0;
    f.par = dir == 1 && d->stride == 2 && d->H % 2 == 0 && d->W % 2 == 0 &&
            ((long long)d->N * (d->H / 2) * (d->W / 2)) % BM == 0;
    pl->grid = dim3((unsigned)ceil_div<long long>(M, BM), (unsigned)ceil_div(Nc, f.bn));
    pl->family = CONV_FP32_TILES;
    return;
  }
  const long long T = (long long)d->kh * d->kw * d->Cin * d->Cout;
  if (same3x3 && d->Cin <= 4 && (d->Cout & 3) == 0 && d->Cout <= 64 && (d->W & (d->W - 1)) == 0 && d->W <= 64 &&
      c.dy_aligned) {
    f.TH = stem_rows(d->H);
    const int per_pg = (9 * d->Cin + 1) * (d->Cout >> 2);
    f.PG = 1;
    while (2 * f.PG * per_pg <= 512 && (f.TH * d->W) % (2 * f.PG) == 0) f.PG *= 2;
    const size_t smem = ((size_t)(((f.TH + 2) * (d->W + 2) * d->Cin + 3) & ~3) + (size_t)f.TH * d->W * d->Cout +
                         (size_t)max(f.PG - 1, 1) * per_pg * 4) * sizeof(float);
    if (per_pg <= 512 && smem <= 48 * 1024) {
      f.num_tiles = d->N * (d->H / f.TH);
      pl->splits = wgrad_fit_splits(min(f.num_tiles, 2 * c.sms), T, d->Cout);   // one slice per CTA
      pl->grid = dim3((unsigned)pl->splits);
      pl->block = dim3(ceil_div(f.PG * per_pg, 32) * 32);
      pl->smem = smem;
      pl->family = CONV_FP32_WGRAD_STEM;
      return;
    }
  }
  if (same3x3 && d->Cin % 16 == 0 && d->Cout % 16 == 0) {
    f.nci = d->Cin % 32 == 0 ? 16 : 8;
    f.nco = d->Cout % 32 == 0 ? 16 : 8;
    const int CIT = 2 * f.nci, COT = 2 * f.nco, RG = 256 / (f.nci * f.nco);
    f.TH = min(max(1, 128 / d->W), d->H);
    const size_t tile_bytes = ((size_t)(f.TH + 2) * (d->W + 2) * CIT + (size_t)f.TH * d->W * COT) * sizeof(float);
    const size_t red_bytes = RG > 1 ? ((size_t)RG * 36 * f.nci * f.nco + (size_t)RG * 2 * f.nco) * sizeof(float) : 0;
    const size_t smem = max(tile_bytes, red_bytes);
    if (smem <= WGRAD3X3_MAX_SMEM) {
      f.tiles_per_img = ceil_div(d->H, f.TH);
      f.num_tiles = d->N * f.tiles_per_img;
      const int cy = d->Cin / CIT, cz = d->Cout / COT;
      pl->splits = wgrad_fit_splits(min(f.num_tiles, max(1, (2 * c.sms) / (cy * cz))), T, d->Cout);   // one per CTA column
      pl->grid = dim3((unsigned)pl->splits, cy, cz);
      pl->smem = smem;
      pl->family = CONV_FP32_WGRAD_3X3;
      return;
    }
  }
  // conv_wgrad_kernel<64, 64, 4, 4>
  const int KK = d->kh * d->kw * d->Cin;
  const long long P = (long long)d->N * d->Ho * d->Wo;
  const int gx = ceil_div(KK, 64), gy = ceil_div(d->Cout, 64);
  // split the pixel reduction so that the grid fills the machine about twice
  long long want = max(1LL, (long long)(2 * c.sms) / ((long long)gx * gy));
  long long splits = min(want, ceil_div<long long>(P, 4 * BK));
  // and on long reductions each split sums at most WGRAD_SPLIT_PX pixels in fp32 when the workspace holds the slices:
  // ResNet-50's stem at 448 px sums 1.6 M pixels (B = 32), which 88 splits of 18 000 took to 2.6e-6 of the largest dW
  // (8e-7 in splits of 2048)
  if (P >= WGRAD_LONG_PX) splits = max(splits, ceil_div<long long>(P, WGRAD_SPLIT_PX));
  splits = max(1LL, wgrad_fit_splits(splits, T, d->Cout));
  f.per = ceil_div<long long>(ceil_div<long long>(P, splits), BK) * BK;
  pl->splits = ceil_div<long long>(P, f.per);
  pl->split_px = f.per;
  pl->grid = dim3((unsigned)gx, (unsigned)gy, (unsigned)pl->splits);
  pl->family = CONV_FP32_WGRAD;
}

template <int BM, int BN, int TM, int TN>
static void fwd_go(const ConvPlan& pl, const ConvP& p, const float* x, const float* w, const float* bias,
                   const float* residual, float* y, int relu, double* stats, cudaStream_t st) {
  if (pl.fp.vec) launch(conv_fwd_kernel<BM, BN, TM, TN, true>, pl.grid, pl.block, 0, st, p, x, w, bias, residual, y, relu, stats);
  else launch(conv_fwd_kernel<BM, BN, TM, TN, false>, pl.grid, pl.block, 0, st, p, x, w, bias, residual, y, relu, stats);
}

int conv_fwd_simt(const ConvPlan& pl, const se_conv_desc* d, const float* x, const float* w, const float* bias,
                  const float* residual, float* y, int relu, double* stats, cudaStream_t st) {
  const ConvP p = to_p(d);
  switch (pl.family) {
    case CONV_FP32_DENSE_SMALL:
      launch(dense_small_fwd_kernel, pl.grid, pl.block, 0, st, x, w, bias, y, p.N, p.Cin, p.Cout, relu);
      return check_launch("dense_small_fwd_kernel");
    case CONV_FP32_FWD_STEM:
      launch(conv_fwd_stem_kernel, pl.grid, pl.block, pl.smem, st, p, x, w, bias, y, relu, stats, pl.fp.TH);
      return check_launch("conv_fwd_stem_kernel");
    default:
      if (pl.fp.bn == 16) fwd_go<128, 16, 4, 2>(pl, p, x, w, bias, residual, y, relu, stats, st);
      else if (pl.fp.bn == 32) fwd_go<128, 32, 4, 4>(pl, p, x, w, bias, residual, y, relu, stats, st);
      else fwd_go<64, 64, 4, 4>(pl, p, x, w, bias, residual, y, relu, stats, st);
      return check_launch("conv_fwd_kernel");
  }
}

template <int BM, int BN, int TM, int TN>
static void dgrad_go(const ConvPlan& pl, const ConvP& p, const float* dy, const float* w, float* dx, float beta, cudaStream_t st) {
  if (pl.fp.vec) launch(conv_dgrad_kernel<BM, BN, TM, TN, true>, pl.grid, pl.block, 0, st, p, dy, w, dx, beta, pl.fp.par);
  else launch(conv_dgrad_kernel<BM, BN, TM, TN, false>, pl.grid, pl.block, 0, st, p, dy, w, dx, beta, pl.fp.par);
}

int conv_dgrad_simt(const ConvPlan& pl, const se_conv_desc* d, const float* dy, const float* w, float* dx, float beta,
                    cudaStream_t st) {
  const ConvP p = to_p(d);
  if (pl.fp.bn == 16) dgrad_go<128, 16, 4, 2>(pl, p, dy, w, dx, beta, st);
  else if (pl.fp.bn == 32) dgrad_go<128, 32, 4, 4>(pl, p, dy, w, dx, beta, st);
  else dgrad_go<64, 64, 4, 4>(pl, p, dy, w, dx, beta, st);
  return check_launch("conv_dgrad_kernel");
}

int conv_wgrad_simt(const ConvPlan& pl, const se_conv_desc* d, const float* x, const float* dy, const WgOut& o,
                    cudaStream_t st) {
  const ConvP p = to_p(d);
  const SimtParams& f = pl.fp;
  const int direct = o.ws ? 0 : 1;
  switch (pl.family) {
    case CONV_FP32_WGRAD_STEM:
      launch(conv_wgrad_stem_kernel, pl.grid, pl.block, pl.smem, st, p, x, dy, o.dw, o.dbias, f.TH, f.PG, f.num_tiles, direct);
      return check_launch("conv_wgrad_stem_kernel");
    case CONV_FP32_WGRAD_3X3: {
      auto kern = f.nci == 16 ? (f.nco == 16 ? conv_wgrad3x3_kernel<16, 16> : conv_wgrad3x3_kernel<16, 8>)
                              : (f.nco == 16 ? conv_wgrad3x3_kernel<8, 16> : conv_wgrad3x3_kernel<8, 8>);
      launch(kern, pl.grid, pl.block, pl.smem, st, p, x, dy, o.dw, o.dbias, f.TH, f.tiles_per_img, f.num_tiles, direct);
      return check_launch("conv_wgrad3x3_kernel");
    }
    default:
      launch(conv_wgrad_kernel<64, 64, 4, 4>, pl.grid, pl.block, 0, st, p, x, dy, o.dw, o.dbias, f.per, direct);
      return check_launch("conv_wgrad_kernel");
  }
}

}  // namespace se
