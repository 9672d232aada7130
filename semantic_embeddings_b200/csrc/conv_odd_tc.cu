// Tensor-core (mma.sync m16n8k8, TF32) 3x3 / stride 1 / 'same' convolutions for channel counts that are not multiples
// of 8: the block convolutions of PyramidNet (models/cifar_pyramidnet.py:89-96), whose widths are 16 + 5k.  Forward,
// data gradient and weight gradient, each an implicit GEMM over dense NHWC tensors with their true channel counts.
//
//   forward / dgrad   y[m, n] = sum_k A[m, k] * B[n, k],   m = output pixel (flat N*H*W list), k = (filter tap, channel)
//                     flattened, K = 9 * Kc.  A[m, (tap, c)] = the input pixel shifted by the tap, zero outside the image
//                     (the 'same' padding).  B[n, (tap, c)] = w_t[tap][co][ci] (forward) or w[8 - tap][ci][co] (dgrad):
//                     both are [tap][n][k] with the GEMM K channels contiguous, so one loader serves both.
//   weight gradient   dW[(tap, ci), co] = sum_px X[px + tap shift, ci] * dY[px, co]: M = 9 * Cin, N = Cout, K = pixels,
//                     split over pixel ranges into the library's split-K workspace (fixed-order reduction), atomics in
//                     direct mode.
//
// Operand staging.  The pixel stride of these tensors is C * 4 bytes, not a multiple of 16, so neither TMA boxes nor
// vector loads apply; every operand element is gathered with a 4-byte cp.async that zero-fills out-of-image taps, the
// padding of K to the 16-wide k tile and the columns past N.  K is flattened over (tap, channel) so the only padding is
// the tail of 9 * Kc (189 -> 192 for 21 channels), not one tail per tap.  mma.sync tiles N in steps of 8 per warp; the
// N tile (32 or 64) is chosen per layer to waste the fewest columns, and the stores are masked.
//
// X3 (SE_MODE_TF32X3, see conv_tc.cu): A_hi*B_hi + A_hi*B_lo + A_lo*B_hi, A split in registers; B_lo is the
// se_split_filters copy (forward / dgrad) or split in registers (weight gradient, where B is dY).  Each k tile's MMAs go
// into a fresh register tile that is then added into the accumulator, as in conv_tc_kernel.
//
// BatchNorm statistics are not fused: se_conv2d_fwd_aux runs se_bn_stats after the forward launch (ConvPlan::fused_stats).
#include <algorithm>

#include "common.cuh"
#include "conv_plan.cuh"
#include "tc.cuh"

namespace se {

using tc::smem_u32;

constexpr int OD_BM = 128;          // GEMM rows per CTA (8 warps: 4 along M x 2 along N, 32 rows each)
constexpr int OD_BK = 16;           // k per pipeline stage
constexpr int OD_LD = OD_BK + 4;    // smem row pitch in floats: fragment loads of 8 rows x 4 k hit 32 distinct banks
constexpr int OD_THREADS = 256;

__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool ok) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(ok ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t hi_bits(uint32_t v) { return v & 0xFFFFE000u; }
__device__ __forceinline__ uint32_t lo_bits(uint32_t v) {
  return __float_as_uint(__uint_as_float(v) - __uint_as_float(v & 0xFFFFE000u));
}

// The MMAs of one k tile: acc[mt][nt] += A[32 rows of warp wm][16] * B[BN/2 columns of warp wn][16]^T.
// BLO: B's low parts come from `bl` (the se_split_filters copy); otherwise X3 splits B in registers.
template <int BN, int X3, bool BLO>
__device__ __forceinline__ void od_mma_tile(float (&acc)[2][BN / 16][4], const float (*a)[OD_LD], const float (*b)[OD_LD],
                                            const float (*bl)[OD_LD], int wm, int wn, int lane) {
  constexpr int NT = BN / 16;
  const int g = lane >> 2, t = lane & 3;
  float part[2][NT][4];
  if (X3) {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) part[mt][nt][i] = 0.f;
  }
#pragma unroll
  for (int ks = 0; ks < OD_BK; ks += 8) {
    uint32_t af[2][4], bf[NT][2];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int r = wm * 32 + mt * 16 + g;
      af[mt][0] = __float_as_uint(a[r][ks + t]);
      af[mt][1] = __float_as_uint(a[r + 8][ks + t]);
      af[mt][2] = __float_as_uint(a[r][ks + t + 4]);
      af[mt][3] = __float_as_uint(a[r + 8][ks + t + 4]);
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int n = wn * (BN / 2) + nt * 8 + g;
      bf[nt][0] = __float_as_uint(b[n][ks + t]);
      bf[nt][1] = __float_as_uint(b[n][ks + t + 4]);
    }
    if (X3) {
      uint32_t al[2][4], bh[NT][2], blo[NT][2];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int i = 0; i < 4; ++i) { al[mt][i] = lo_bits(af[mt][i]); af[mt][i] = hi_bits(af[mt][i]); }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int n = wn * (BN / 2) + nt * 8 + g;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          // the tensor core reads the TF32 truncation of an fp32 word: B as stored is B_hi
          bh[nt][j] = BLO ? bf[nt][j] : hi_bits(bf[nt][j]);
          blo[nt][j] = BLO ? __float_as_uint(bl[n][ks + t + 4 * j]) : lo_bits(bf[nt][j]);
        }
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          mma_tf32(part[mt][nt], af[mt], bh[nt][0], bh[nt][1]);
          mma_tf32(part[mt][nt], af[mt], blo[nt][0], blo[nt][1]);
          mma_tf32(part[mt][nt], al[mt], bh[nt][0], bh[nt][1]);
        }
    } else {
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_tf32(acc[mt][nt], af[mt], bf[nt][0], bf[nt][1]);
    }
  }
  if (X3) {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[mt][nt][i] += part[mt][nt][i];
  }
}

// ------------------------------------------------------------------------------------------------ forward / dgrad
// grid = (ceil(N*H*W / 128), ceil(Nc / BN)); out = beta * out + (A (*) B + bias + residual), ReLU
template <int BN, int X3>
__global__ void __launch_bounds__(OD_THREADS)
conv_odd_tc_kernel(const float* __restrict__ act, const float* __restrict__ bmat, const float* __restrict__ bmat_lo,
                   OddTcParams p) {
  constexpr int S = X3 ? 2 : 3;       // pipeline stages (static shared memory <= 48 KB)
  __shared__ __align__(16) float sa[S][OD_BM][OD_LD];
  __shared__ __align__(16) float sb[S][BN][OD_LD];
  __shared__ __align__(16) float sbl[X3 ? S : 1][BN][OD_LD];
  pdl_grid_sync();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp & 3, wn = warp >> 2;
  const int m0 = blockIdx.x * OD_BM, n0 = blockIdx.y * BN;
  const int Kc = p.Kc, Nc = p.Nc, Ktot = 9 * Kc;
  const int kk = tid & 15, rsub = tid >> 4;          // this thread's k column and first row of every loaded tile
  // the 8 output pixels whose A rows this thread loads: rows rsub + 16 i
  int py[8], px[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + rsub + 16 * i;
    const int rem = m % (p.H * p.W);
    py[i] = m < p.npx ? rem / p.W : -4;              // -4: no pixel (every tap fails the bounds check)
    px[i] = rem % p.W;
  }
  const long long tap_stride = (long long)Nc * Kc;
  auto load = [&](int kt, int slot) {
    const int k = kt * OD_BK + kk;
    const bool kok = k < Ktot;
    const int tap = kok ? k / Kc : 0, c = k - tap * Kc;
    const int dy = tap / 3 - 1, dx = tap % 3 - 1;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int yy = py[i] + dy, xx = px[i] + dx;
      const bool ok = kok && yy >= 0 && yy < p.H && xx >= 0 && xx < p.W;
      const long long src = ((long long)(m0 + rsub + 16 * i) + dy * p.W + dx) * Kc + c;
      cp_async4(&sa[slot][rsub + 16 * i][kk], ok ? act + src : act, ok);
    }
    const long long boff = (long long)(p.flip ? 8 - tap : tap) * tap_stride + c;
#pragma unroll
    for (int j = 0; j < BN / 16; ++j) {
      const int n = n0 + rsub + 16 * j;
      const bool ok = kok && n < Nc;
      cp_async4(&sb[slot][rsub + 16 * j][kk], ok ? bmat + boff + (long long)n * Kc : bmat, ok);
      if (X3) cp_async4(&sbl[X3 ? slot : 0][rsub + 16 * j][kk], ok ? bmat_lo + boff + (long long)n * Kc : bmat_lo, ok);
    }
  };

  float acc[2][BN / 16][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < BN / 16; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
  const int nk = ceil_div(Ktot, OD_BK);
#pragma unroll
  for (int s = 0; s < S - 1; ++s) {
    if (s < nk) load(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<S - 2>();
    __syncthreads();                         // stage kt landed for every thread; stage kt - 1 is no longer read
    if (kt + S - 1 < nk) load(kt + S - 1, (kt + S - 1) % S);
    cp_async_commit();
    const int slot = kt % S;
    od_mma_tile<BN, X3, true>(acc, sa[slot], sb[slot], sbl[X3 ? slot : 0], wm, wn, lane);
  }

  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + wm * 32 + mt * 16 + g + 8 * h;
      if (m >= p.npx) continue;
      float* orow = p.out + (long long)m * Nc;
      const float* rrow = p.residual ? p.residual + (long long)m * Nc : nullptr;
#pragma unroll
      for (int nt = 0; nt < BN / 16; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int n = n0 + wn * (BN / 2) + nt * 8 + 2 * t + j;
          if (n >= Nc) continue;
          float v = acc[mt][nt][2 * h + j];
          if (p.bias) v += __ldg(p.bias + n);
          if (rrow) v += __ldg(rrow + n);
          if (p.relu) v = fmaxf(v, 0.f);
          if (p.beta != 0.f) v += p.beta * orow[n];
          orow[n] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------ weight gradient
// grid = (ceil(9*Cin / 128), ceil(Cout / BN), splits); split z sums pixels [z * per_split, (z + 1) * per_split)
template <int BN, int X3>
__global__ void __launch_bounds__(OD_THREADS)
conv_odd_wgrad_tc_kernel(const float* __restrict__ x, const float* __restrict__ dyp, OddWgParams p) {
  constexpr int S = 3;
  __shared__ __align__(16) float sa[S][OD_BM][OD_LD];
  __shared__ __align__(16) float sb[S][BN][OD_LD];
  pdl_grid_sync();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp & 3, wn = warp >> 2;
  const int m0 = blockIdx.x * OD_BM, n0 = blockIdx.y * BN, z = blockIdx.z;
  const int Cin = p.Cin, Cout = p.Cout, KK = 9 * Cin;
  const int hw = p.H * p.W;
  const int px_begin = z * p.per_split, px_end = min(p.npx, px_begin + p.per_split);
  // A: this thread's dW row (filter tap, input channel) and its pixel columns (tid >> 7) + 2 i
  const int arow = tid & 127, acol = tid >> 7;
  const int kr = m0 + arow;
  const bool rok = kr < KK;
  const int tap = rok ? kr / Cin : 0, ci = kr - tap * Cin;
  const int sdy = tap / 3 - 1, sdx = tap % 3 - 1;
  // B: this thread's output channel and its pixel columns
  const int bcol = tid % BN, bk0 = tid / BN;
  const int co = n0 + bcol;
  const bool cok = co < Cout;
  const bool do_bias = blockIdx.x == 0;
  auto load = [&](int kt, int slot) {
    const int k0 = px_begin + kt * OD_BK;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int pxl = k0 + acol + 2 * i;
      const int rem = pxl % hw, y = rem / p.W + sdy, xx = rem % p.W + sdx;
      const bool ok = rok && pxl < px_end && y >= 0 && y < p.H && xx >= 0 && xx < p.W;
      const long long src = ((long long)pxl + sdy * p.W + sdx) * Cin + ci;
      cp_async4(&sa[slot][arow][acol + 2 * i], ok ? x + src : x, ok);
    }
#pragma unroll
    for (int j = 0; j < BN * OD_BK / OD_THREADS; ++j) {
      const int kc = bk0 + j * (OD_THREADS / BN);
      const int pxl = k0 + kc;
      const bool ok = cok && pxl < px_end;
      cp_async4(&sb[slot][bcol][kc], ok ? dyp + (long long)pxl * Cout + co : dyp, ok);
    }
  };

  float acc[2][BN / 16][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < BN / 16; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
  double bsum = 0.0;                  // dbias: a sum over the whole pixel range of the split, kept in float64
  const int nk = px_end > px_begin ? ceil_div(px_end - px_begin, OD_BK) : 0;
#pragma unroll
  for (int s = 0; s < S - 1; ++s) {
    if (s < nk) load(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<S - 2>();
    __syncthreads();
    if (kt + S - 1 < nk) load(kt + S - 1, (kt + S - 1) % S);
    cp_async_commit();
    const int slot = kt % S;
    if (do_bias && tid < BN) {
#pragma unroll
      for (int k = 0; k < OD_BK; ++k) bsum += sb[slot][tid][k];
    }
    od_mma_tile<BN, X3, false>(acc, sa[slot], sb[slot], nullptr, wm, wn, lane);
  }

  const long long T = (long long)KK * Cout;
  float* dwt = p.ws ? p.ws + z * T : p.dw;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + wm * 32 + mt * 16 + g + 8 * h;
      if (row >= KK) continue;
#pragma unroll
      for (int nt = 0; nt < BN / 16; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int n = n0 + wn * (BN / 2) + nt * 8 + 2 * t + j;
          if (n >= Cout) continue;
          float* o = dwt + (long long)row * Cout + n;
          if (p.ws) *o = acc[mt][nt][2 * h + j];
          else atomicAdd(o, acc[mt][nt][2 * h + j]);
        }
    }
  if (do_bias && tid < BN && n0 + tid < Cout) {
    if (p.ws) p.ws[(long long)gridDim.z * T + (long long)z * Cout + n0 + tid] = (float)bsum;
    else if (p.dbias) atomicAdd(p.dbias + n0 + tid, (float)bsum);
  }
}

// ---------------------------------------------------------------------------------------- host side
// The shapes of this family (conv_plan, after every other tensor-core family has declined): 3x3 / stride 1 / 'same' on
// images 8..32 pixels wide (PyramidNet's 32-, 16- and 8-wide stages), both channel counts >= 16 and at least one of them
// not a multiple of 8.  Every channel count in the recorded plan table (tests/golden/conv_paths.npz) is 3, 4 or a
// multiple of 8, so no layer of the other networks moves: the 24- and 48-channel layers stay where they are.
bool conv_odd_tc_ok(const se_conv_desc* d) {
  return d->kh == 3 && d->kw == 3 && d->stride == 1 && d->pad_t == 1 && d->pad_l == 1 && d->Ho == d->H && d->Wo == d->W &&
         d->W >= 8 && d->W <= 32 && d->Cin >= 16 && d->Cout >= 16 && (d->Cin % 8 != 0 || d->Cout % 8 != 0) &&
         (long long)d->N * d->H * d->W <= 0x7fffffffLL - OD_BM;
}

// N tile: the one of 32 / 64 that leaves the fewest padded columns (64 on a tie)
static int odd_bn(int Nc) { return ceil_div(Nc, 64) * 64 <= ceil_div(Nc, 32) * 32 ? 64 : 32; }

bool odd_config(const se_conv_desc* d, int dir, int sms, ConvPlan* pl) {
  const long long npx = (long long)d->N * d->H * d->W;
  if (dir < 2) {
    OddTcParams& p = pl->od;
    p.H = d->H; p.W = d->W; p.npx = (int)npx;
    p.Kc = dir == 0 ? d->Cin : d->Cout; p.Nc = dir == 0 ? d->Cout : d->Cin;
    p.flip = dir;
    pl->od_bn = odd_bn(p.Nc);
    const long long gx = ceil_div<long long>(npx, OD_BM);
    if (gx > 0x7fffffffLL) return false;
    pl->grid = dim3((unsigned)gx, (unsigned)ceil_div(p.Nc, pl->od_bn));
    return true;
  }
  OddWgParams& p = pl->owg;
  p.H = d->H; p.W = d->W; p.Cin = d->Cin; p.Cout = d->Cout; p.npx = (int)npx;
  pl->od_bn = odd_bn(d->Cout);
  const long long KK = 9LL * d->Cin, T = KK * d->Cout;
  const long long tiles = ceil_div<long long>(KK, OD_BM) * ceil_div(d->Cout, pl->od_bn);
  if (ceil_div<long long>(KK, OD_BM) > 65535) return false;
  // about four CTAs per SM over all tiles, each split at least 8 k tiles long, within the workspace
  long long splits = ceil_div<long long>(4LL * (sms > 0 ? sms : 132), tiles);
  splits = std::max(1LL, std::min(splits, ceil_div<long long>(npx, 8 * OD_BK)));
  splits = std::min(std::max(1LL, wgrad_fit_splits(splits, T, d->Cout)), 65535LL);
  p.per_split = (int)(ceil_div<long long>(ceil_div<long long>(npx, splits), OD_BK) * OD_BK);
  splits = ceil_div<long long>(npx, p.per_split);
  pl->grid = dim3((unsigned)ceil_div<long long>(KK, OD_BM), (unsigned)ceil_div(d->Cout, pl->od_bn), (unsigned)splits);
  pl->splits = splits;
  pl->split_px = p.per_split;
  return true;
}

template <int BN>
static void odd_go(const ConvPlan& pl, cudaStream_t st, const float* a, const float* b, const float* bl, const OddTcParams& p) {
  if (pl.x3) launch(conv_odd_tc_kernel<BN, 1>, pl.grid, dim3(OD_THREADS), 0, st, a, b, bl, p);
  else launch(conv_odd_tc_kernel<BN, 0>, pl.grid, dim3(OD_THREADS), 0, st, a, b, bl, p);
}

static int odd_launch(const ConvPlan& pl, OddTcParams p, const float* a, const float* b, const float* bl, cudaStream_t st) {
  if (pl.od_bn == 64) odd_go<64>(pl, st, a, b, bl, p);
  else odd_go<32>(pl, st, a, b, bl, p);
  return check_launch("conv_odd_tc_kernel");
}

int conv_fwd_odd_tc(const ConvPlan& pl, const float* x, const float* w_t, const float* w_t_lo, const float* bias,
                    const float* residual, float* y, int relu, cudaStream_t st) {
  OddTcParams p = pl.od;
  p.bias = bias; p.residual = residual; p.out = y; p.relu = relu; p.beta = 0.f;
  return odd_launch(pl, p, x, w_t, pl.x3 ? w_t_lo : w_t, st);
}

int conv_dgrad_odd_tc(const ConvPlan& pl, const float* dy, const float* w, const float* w_lo, float* dx, float beta,
                      cudaStream_t st) {
  OddTcParams p = pl.od;
  p.bias = nullptr; p.residual = nullptr; p.out = dx; p.relu = 0; p.beta = beta;
  return odd_launch(pl, p, dy, w, pl.x3 ? w_lo : w, st);
}

int conv_wgrad_odd_tc(const ConvPlan& pl, const float* x, const float* dy, const WgOut& o, cudaStream_t st) {
  OddWgParams p = pl.owg;
  p.ws = o.ws; p.dw = o.dw; p.dbias = o.dbias;
  if (pl.od_bn == 64) {
    if (pl.x3) launch(conv_odd_wgrad_tc_kernel<64, 1>, pl.grid, dim3(OD_THREADS), 0, st, x, dy, p);
    else launch(conv_odd_wgrad_tc_kernel<64, 0>, pl.grid, dim3(OD_THREADS), 0, st, x, dy, p);
  } else {
    if (pl.x3) launch(conv_odd_wgrad_tc_kernel<32, 1>, pl.grid, dim3(OD_THREADS), 0, st, x, dy, p);
    else launch(conv_odd_wgrad_tc_kernel<32, 0>, pl.grid, dim3(OD_THREADS), 0, st, x, dy, p);
  }
  return check_launch("conv_odd_wgrad_tc_kernel");
}

}  // namespace se
