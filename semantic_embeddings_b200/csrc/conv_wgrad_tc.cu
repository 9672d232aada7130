// Tensor-core (wgmma, TF32) weight gradient of the convolutions the forward kernels take (conv_tc.cu): 3x3 / stride 1
// / 'same', 1x1 / stride 1 and 2, and the wide 3x3 / stride 2 layers of wide_residual_network.py:20-31:
//   dW[r, s, ci, co] += sum_pixels X[pixel * stride + (r, s) - pad, ci] * dY[pixel, co]      (autodiff of Conv2D, reference
//   models/cifar_resnet.py:96-105 etc. under learn_image_embeddings.py:238)          dbias[co] += sum_pixels dY[pixel, co]
//
// The reduction dimension is the PIXEL axis, in which both NHWC tensors are strided; TF32 wgmma reads only K-major
// operands, so each warpgroup loads a chunk of 32 pixels of X (64 input channels, shifted by the filter tap and
// zero outside the image) and of dY (BN output channels) into registers and writes them TRANSPOSED into shared memory
// as [channel][32 pixels] rows of 128 bytes in the 128-byte swizzle layout; the next chunk's global loads are in flight
// while the MMAs of the current one run.  M = 64 input channels, N = BN output channels, K = 8 pixels per instruction.
// X3 (error-compensated, see conv_tc.cu): the transposing stores write hi and lo parts into two tiles each, and
// dW = X_hi*dY_hi + X_hi*dY_lo + X_lo*dY_hi.
// grid = (pixel ranges, 64-channel input blocks x filter taps, output-channel tiles); the two warpgroups of a CTA take
// alternate chunks of its range (split-K).  Every warpgroup stores its partial sums into its own slice of a library
// workspace, and a second kernel adds the slices into dW / dbias in a fixed order: the result is the same on every run
// (float atomics would add the slices in whatever order they arrive).
#include <stdlib.h>

#include <algorithm>
#include <mutex>

#include "common.cuh"
#include "conv_plan.cuh"
#include "tc.cuh"

namespace se {

using namespace tc;

constexpr int WG_PX = 32;              // pixels per chunk: one 128-byte swizzle row per channel
constexpr int WG_MT = 64;              // rows of dW ((filter tap, input channel) pairs) per warpgroup tile
constexpr int WG_THREADS = 256;

// Workspaces of the split-K partial sums: one per (device, stream), 32 MB each, allocated outside graph captures (se_init
// prepares the one of se_run_ops' side stream).  A request that does not fit, or a stream that first appears inside a
// capture, runs in direct mode instead: the partial sums go into dW with float atomics (correct, not bit-reproducible).
constexpr long long WG_WS_FLOATS = 8LL << 20;
struct WgWorkspace { int dev; cudaStream_t st; float* ptr; };
constexpr int WG_MAX_WS = 32;
static WgWorkspace g_wg_ws[WG_MAX_WS];
static int g_wg_nws = 0;
static std::mutex g_wg_mu;

template <int BN>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t a, uint64_t b, int acc) {
  if constexpr (BN == 16) wgmma_tf32_n16(d, a, b, acc);
  else if constexpr (BN == 32) wgmma_tf32_n32(d, a, b, acc);
  else if constexpr (BN == 64) wgmma_tf32_n64(d, a, b, acc);
  else wgmma_tf32_n128(d, a, b, acc);
}

// one channel quadruple of one pixel -> four transposed rows of a [channel][32 pixels] tile (X3: hi and lo tiles)
template <int X3>
__device__ __forceinline__ void put_t(uint8_t* hi, uint8_t* lo, int c4, int px, float4 v) {
  const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t o = swizzle_offset(4 * c4 + j, px >> 2, 128) + (px & 3) * 4;
    if (X3) {
      *reinterpret_cast<float*>(hi + o) = tf32_hi(e[j]);
      *reinterpret_cast<float*>(lo + o) = tf32_lo(e[j]);
    } else {
      *reinterpret_cast<float*>(hi + o) = e[j];
    }
  }
}

template <int BN, int X3, int NP>
__global__ void __launch_bounds__(WG_THREADS, 1)
conv_wgrad_tc_kernel(const float* __restrict__ x, const float* __restrict__ dy, WgTcParams p) {
  pdl_grid_sync();
  constexpr int XQ = WG_PX * WG_MT / 4 / 128;        // float4 loads of X per thread and chunk (4)
  constexpr int YQ = WG_PX * BN / 4 / 128;           // of dY (1..8)
  constexpr int X_BYTES = WG_MT * 128, Y_BYTES = BN * 128;
  constexpr int WG_BYTES = (X_BYTES + Y_BYTES) * (X3 ? 2 : 1);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  uint8_t* sx = smem + wg * WG_BYTES;
  uint8_t* sy = sx + X_BYTES;
  uint8_t* sxl = sy + Y_BYTES;
  uint8_t* syl = sxl + X_BYTES;

  // rows m0.. of dW are (filter tap, input channel) pairs: narrow layers fill the 64-row tile with several taps
  const int m0 = blockIdx.y * WG_MT, co0 = blockIdx.z * BN;
  const bool do_bias = blockIdx.y == 0;
  const long long split = 2LL * blockIdx.x + wg, T = (long long)p.KK * p.Cout;
  // this thread's four rows (a channel quadruple of one tap: Cin % 4 == 0) and pixel slots (XQ / YQ of them) in a chunk
  const int xc4 = t % (WG_MT / 4), xp0 = t / (WG_MT / 4);
  const int yc4 = t % (BN / 4), yp0 = t / (BN / 4);
  const int kk = m0 + 4 * xc4;
  const bool xc_ok = kk < p.KK;
  const int tap = kk / p.Cin, ci = kk - tap * p.Cin;
  const int r = tap / p.kw, s = tap - r * p.kw;
  const int hw = p.Ho * p.Wo;
  const int c_begin = blockIdx.x * p.per_cta, c_end = min(p.chunks, c_begin + p.per_cta);

  float4 xv[XQ], yv[YQ];
  auto load = [&](int chunk) {
#pragma unroll
    for (int q = 0; q < XQ; ++q) {
      const int g = chunk * WG_PX + xp0 + q * (128 / (WG_MT / 4));
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (g < p.npx && xc_ok) {
        const int n = g / hw, rem = g - n * hw, ho = rem / p.Wo, wo = rem - ho * p.Wo;
        const int hi = ho * p.stride + r - p.pad_t, wi = wo * p.stride + s - p.pad_l;
        if (hi >= 0 && hi < p.H && wi >= 0 && wi < p.W)
          v = __ldg(reinterpret_cast<const float4*>(x + (((long long)n * p.H + hi) * p.W + wi) * p.Cin + ci));
      }
      xv[q] = v;
    }
#pragma unroll
    for (int q = 0; q < YQ; ++q) {
      const int g = chunk * WG_PX + yp0 + q * (128 / (BN / 4));
      yv[q] = g < p.npx ? __ldg(reinterpret_cast<const float4*>(dy + (long long)g * p.Cout + co0) + yc4)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };

  // X3: each chunk's MMAs go into NP fresh register tiles (of 32 / NP pixels each) that are then added into `acc`.  The
  // tensor core keeps fewer bits of a sum than an fp32 add: long reductions (NP = 4, see the host side) start a fresh
  // tile every 8 pixels and add the small terms first
  constexpr int KPP = (WG_PX / 8) / NP;
  float acc[BN / 2], part[NP][BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  float4 bsum = make_float4(0.f, 0.f, 0.f, 0.f);
  int c = c_begin + wg;
  if (c < c_end) load(c);
  int first = 1;
  for (; c < c_end; c += 2) {
#pragma unroll
    for (int q = 0; q < XQ; ++q) put_t<X3>(sx, sxl, xc4, xp0 + q * (128 / (WG_MT / 4)), xv[q]);
#pragma unroll
    for (int q = 0; q < YQ; ++q) {
      put_t<X3>(sy, syl, yc4, yp0 + q * (128 / (BN / 4)), yv[q]);
      if (do_bias) { bsum.x += yv[q].x; bsum.y += yv[q].y; bsum.z += yv[q].z; bsum.w += yv[q].w; }
    }
    fence_proxy_async();                    // generic-proxy writes -> visible to the tensor core
    named_bar_sync(1 + wg, 128);
    if (c + 2 < c_end) load(c + 2);         // next chunk's loads overlap this chunk's MMAs
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < WG_PX / 8; ++ks) {
      const uint64_t da = wgmma_desc(smem_u32(sx) + ks * 32, 128), db = wgmma_desc(smem_u32(sy) + ks * 32, 128);
      if (X3) {
        float (&pt)[BN / 2] = part[ks / KPP];
        if (NP > 1) {
          wgmma_tf32<BN>(pt, da, wgmma_desc(smem_u32(syl) + ks * 32, 128), ks % KPP > 0);
          wgmma_tf32<BN>(pt, wgmma_desc(smem_u32(sxl) + ks * 32, 128), db, 1);
          wgmma_tf32<BN>(pt, da, db, 1);
        } else {
          wgmma_tf32<BN>(pt, da, db, ks > 0);
          wgmma_tf32<BN>(pt, da, wgmma_desc(smem_u32(syl) + ks * 32, 128), 1);
          wgmma_tf32<BN>(pt, wgmma_desc(smem_u32(sxl) + ks * 32, 128), db, 1);
        }
      } else {
        wgmma_tf32<BN>(acc, da, db, first == 0 || ks > 0);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (X3) {
#pragma unroll
      for (int j = 0; j < NP; ++j)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += part[j][i];
    }
    named_bar_sync(1 + wg, 128);            // every warp's MMAs have read the tiles before they are rewritten
    first = 0;
  }
  // this warpgroup's slice (zeros when it had no chunk): every element of the slices is written exactly once
  float* dwt = p.ws ? p.ws + split * T : p.dw;
#pragma unroll
  for (int i = 0; i < BN / 2; i += 2) {
    const int row = m0 + fragment_row(i, t), co = co0 + fragment_col(i, t);
    if (row >= p.KK) continue;
    float2* o = reinterpret_cast<float2*>(dwt + (long long)row * p.Cout + co);
    if (p.ws) *o = make_float2(acc[i], acc[i + 1]);
    else atomicAdd(o, make_float2(acc[i], acc[i + 1]));
  }
  if (do_bias) {
    // the threads of one channel quadruple add their sums in thread order (the tiles are free: the loop ended on a barrier)
    float4* sb = reinterpret_cast<float4*>(sx);
    sb[t] = bsum;
    named_bar_sync(1 + wg, 128);
    if (t < BN / 4) {
      float4 v = sb[t];
      for (int k = t + BN / 4; k < 128; k += BN / 4) { v.x += sb[k].x; v.y += sb[k].y; v.z += sb[k].z; v.w += sb[k].w; }
      if (p.ws) reinterpret_cast<float4*>(p.ws + 2LL * gridDim.x * T + split * p.Cout + co0)[t] = v;
      else if (p.dbias) atomicAdd(reinterpret_cast<float4*>(p.dbias + co0) + t, v);
    }
  }
}

// dW[i] += sum over the slices in slice order; dbias likewise (when given)
__global__ void __launch_bounds__(256)
conv_wgrad_reduce_kernel(const float* __restrict__ ws, int splits, long long T, int Cout, float* __restrict__ dw,
                         float* __restrict__ dbias) {
  pdl_grid_sync();
  const long long n = T + (dbias ? Cout : 0);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const bool b = i >= T;
    const float* src = b ? ws + (long long)splits * T + (i - T) : ws + i;
    const long long stride = b ? Cout : T;
    float v = 0.f;
    for (int k = 0; k < splits; ++k) v += src[k * stride];
    if (b) dbias[i - T] += v;
    else dw[i] += v;
  }
}

// ---------------------------------------------------------------------------------------- host side
template <int BN>
static bool set_smem_limit() {
  return cudaFuncSetAttribute(conv_wgrad_tc_kernel<BN, 0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) == cudaSuccess &&
         cudaFuncSetAttribute(conv_wgrad_tc_kernel<BN, 1, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) == cudaSuccess &&
         cudaFuncSetAttribute(conv_wgrad_tc_kernel<BN, 1, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) == cudaSuccess;
}

int init_conv_wgrad_tc() {
  if (!set_smem_limit<16>() || !set_smem_limit<32>() || !set_smem_limit<64>() || !set_smem_limit<128>()) {
    set_error("init_conv_wgrad_tc: cannot raise the shared-memory limit");
    return SE_ERR_CUDA;
  }
  return SE_OK;
}

int wgrad_workspace(long long floats, cudaStream_t st, float** ws) {
  *ws = nullptr;
  if (floats > WG_WS_FLOATS) return SE_OK;                      // direct mode
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    set_error("wgrad_workspace: no usable CUDA device");
    return SE_ERR_CUDA;
  }
  std::lock_guard<std::mutex> lock(g_wg_mu);
  for (int i = 0; i < g_wg_nws; ++i)
    if (g_wg_ws[i].dev == dev && g_wg_ws[i].st == st) { *ws = g_wg_ws[i].ptr; return SE_OK; }
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (g_wg_nws == WG_MAX_WS || cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone)
    return SE_OK;                                               // direct mode: no allocation inside a capture
  float* ptr = nullptr;
  if (cudaMalloc(&ptr, WG_WS_FLOATS * sizeof(float)) != cudaSuccess) {
    set_error("wgrad_workspace: cannot allocate the %lld-byte weight-gradient workspace", WG_WS_FLOATS * 4);
    return SE_ERR_CUDA;
  }
  g_wg_ws[g_wg_nws++] = {dev, st, ptr};
  *ws = ptr;
  return SE_OK;
}

int wgrad_workspace_prepare(cudaStream_t st) {
  float* ws = nullptr;
  return wgrad_workspace(1, st, &ws);
}

long long wgrad_fit_splits(long long want, long long T, int Cout) {
  const long long fit = WG_WS_FLOATS / (T + Cout);
  return fit >= 1 ? std::min(want, fit) : want;               // not even one slice fits: direct mode, any split count
}

int wgrad_reduce(const float* ws, int splits, long long T, int Cout, float* dw, float* dbias, cudaStream_t st) {
  const long long n = T + (dbias ? Cout : 0);
  const long long blocks = std::min(ceil_div<long long>(n, 256), 4LL * sm_count());
  launch(conv_wgrad_reduce_kernel, dim3((unsigned)blocks), dim3(256), 0, st, ws, splits, T, Cout, dw, dbias);
  return check_launch("conv_wgrad_reduce_kernel");
}

// 1x1 convolutions (stride 1 or 2, no padding): two thirds of the layers of keras.applications.ResNet50 (reference
// utils.py:237) and the shortcut projections of wide_residual_network.py:28
static bool conv1x1_wgrad_tc_ok(const se_conv_desc* d) {
  if (d->kh != 1 || d->kw != 1 || d->pad_t != 0 || d->pad_l != 0) return false;
  if (d->stride == 2) {
    if (d->Ho != (d->H + 1) / 2 || d->Wo != (d->W + 1) / 2 || d->Wo > 32) return false;
  } else if (d->stride != 1 || d->Ho != d->H || d->Wo != d->W) {
    return false;
  }
  return d->Cin % 4 == 0 && d->Cout % 16 == 0 && (long long)d->N * d->H * d->W >= 32 &&
         (long long)d->N * d->H * d->W <= 0x7fffffffLL;
}

// 3x3 / stride 2 / no leading padding (the down-sampling layers of wide_residual_network.py:20-31 on even image sizes:
// 'same' puts the one padding row / column AFTER the image).  Worth it for wide layers only; the 16..64-channel layers
// of the CIFAR ResNets stay on the fp32 kernel.  conv_tc.cu runs their data gradient as nine strided 1x1 GEMMs.
bool conv3x3s2_tc_ok(const se_conv_desc* d) {
  return d->kh == 3 && d->kw == 3 && d->stride == 2 && d->pad_t == 0 && d->pad_l == 0 && d->H % 2 == 0 && d->W % 2 == 0 &&
         d->Ho == d->H / 2 && d->Wo == d->W / 2 && d->Wo <= 32 && d->Wo >= 2 && d->Ho >= 2 && d->Cin >= 128 && d->Cout >= 128 &&
         d->Cin % 16 == 0 && d->Cout % 32 == 0;
}

static bool conv3x3_wgrad_tc_ok(const se_conv_desc* d) {
  return d->kh == 3 && d->kw == 3 && d->stride == 1 && d->pad_t == 1 && d->pad_l == 1 && d->Ho == d->H && d->Wo == d->W &&
         d->Cin % 16 == 0 && d->Cout % 16 == 0 && d->W >= 4 && d->W <= 64;
}

// Error-compensated sums over at least this many pixels take four partial tiles per chunk (NP = 4).  Measured on an H100
// on ResNet-50's res2a_branch2a at 448 px (B = 32, 394 272 pixels, in front of a BatchNorm: dY sums to zero per channel,
// X >= 0): 3.6e-5 of the largest dW with one tile and the big term first, 2.9e-5 small terms first, 5.7e-6 with four
// tiles and small terms first (2.0e-5 big term first), against 7e-7 for the float64 sum of the split operands.  Four
// tiles cost 2-6 % on such layers, and up to 20 % on the short reductions of the CIFAR networks, which keep the one tile
// and the arithmetic they had.
constexpr long long WG_LONG_PX = 1LL << 18;

// The launch configuration of conv_wgrad_tc_kernel (conv_plan): false for the shapes it does not take
bool wgrad_config(const se_conv_desc* d, int x3, int sms, ConvPlan* pl) {
  if (!conv1x1_wgrad_tc_ok(d) && !conv3x3s2_tc_ok(d) && !conv3x3_wgrad_tc_ok(d)) return false;
  const long long npx = (long long)d->N * d->Ho * d->Wo, KK = (long long)d->kh * d->kw * d->Cin;
  if (npx > 0x7fffffffLL - 64 || KK > 0x7fffffffLL) return false;
  int BN = x3 ? 64 : 128;                   // error-compensated mode: a second accumulator tile, see the kernel
  while (d->Cout % BN != 0) BN >>= 1;
  const int gy = (int)ceil_div<long long>(KK, WG_MT), gz = d->Cout / BN;
  if (gy > 65535 || gz > 65535) return false;
  WgTcParams& p = pl->wg;
  p.N = d->N; p.H = d->H; p.W = d->W; p.Cin = d->Cin; p.Cout = d->Cout; p.Ho = d->Ho; p.Wo = d->Wo;
  p.kw = d->kw; p.stride = d->stride; p.pad_t = d->pad_t; p.pad_l = d->pad_l;
  p.KK = (int)KK;
  p.npx = (int)npx;
  p.chunks = (int)ceil_div<long long>(npx, WG_PX);
  // about eight CTAs per SM over all row / column tiles, each with at least 4 chunks: a warpgroup's chunks are
  // latency-bound round trips (load, transpose, MMA), so the pixel range is cut finely
  long long gx = ceil_div<long long>(8LL * sms, (long long)gy * gz);
  gx = std::max(1LL, std::min(gx, ceil_div<long long>(p.chunks, 4)));
  gx = std::max(1LL, wgrad_fit_splits(2 * gx, KK * d->Cout, d->Cout) / 2);      // the slices fit the workspace
  p.per_cta = (int)ceil_div<long long>(p.chunks, gx);
  p.per_cta += p.per_cta & 1;
  gx = ceil_div<long long>(p.chunks, p.per_cta);
  pl->grid = dim3((unsigned)gx, (unsigned)gy, (unsigned)gz);
  pl->wg_bn = BN;
  pl->wg_np = x3 && npx >= WG_LONG_PX ? 4 : 1;
  pl->smem = 1024 + 2 * (size_t)(WG_MT * 128 + BN * 128) * (x3 ? 2 : 1);
  return true;
}

// se_linear_svm_fit: does the tensor-core kernel take this shape on stream `st` and add its split-K slices in a fixed
// order, i.e. does at least one pair of slices fit a workspace that exists or can be allocated now?
bool conv_wgrad_tc_fixed_order(const se_conv_desc* d, cudaStream_t st) {
  ConvPlan pl;
  if (conv_plan(d, 2, SE_MODE_TF32X3, ConvCall(), &pl) != CONV_TC_WGRAD) return false;
  const long long T = (long long)d->kh * d->kw * d->Cin * d->Cout;
  float* ws = nullptr;
  return wgrad_workspace(2 * (T + d->Cout), st, &ws) == SE_OK && ws != nullptr;
}

template <int BN>
static void wgrad_go(const ConvPlan& pl, cudaStream_t st, const float* x, const float* dy, const WgTcParams& p) {
  if (pl.wg_np == 4) launch(conv_wgrad_tc_kernel<BN, 1, 4>, pl.grid, dim3(WG_THREADS), pl.smem, st, x, dy, p);
  else if (pl.x3) launch(conv_wgrad_tc_kernel<BN, 1, 1>, pl.grid, dim3(WG_THREADS), pl.smem, st, x, dy, p);
  else launch(conv_wgrad_tc_kernel<BN, 0, 1>, pl.grid, dim3(WG_THREADS), pl.smem, st, x, dy, p);
}

int conv_wgrad_tc(const ConvPlan& pl, const float* x, const float* dy, float* dw, float* dbias, cudaStream_t st) {
  static bool inited = false;
  if (!inited) { int rc0 = init_conv_wgrad_tc(); if (rc0) return rc0; inited = true; }
  WgTcParams p = pl.wg;
  p.dw = dw; p.dbias = dbias;
  const long long T = (long long)p.KK * p.Cout, splits = 2LL * pl.grid.x;
  int rc = wgrad_workspace(splits * (T + p.Cout), st, &p.ws);
  if (rc) return rc;
  switch (pl.wg_bn) {
    case 16: wgrad_go<16>(pl, st, x, dy, p); break;
    case 32: wgrad_go<32>(pl, st, x, dy, p); break;
    case 64: wgrad_go<64>(pl, st, x, dy, p); break;
    default: wgrad_go<128>(pl, st, x, dy, p); break;
  }
  rc = check_launch("conv_wgrad_tc_kernel");
  if (rc || !p.ws) return rc;
  return wgrad_reduce(p.ws, (int)splits, T, p.Cout, dw, dbias, st);
}

}  // namespace se
