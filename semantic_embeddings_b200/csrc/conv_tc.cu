// Tensor-core (wgmma, TF32) implicit-GEMM convolution for 3x3 / stride 1 / 'same' layers -- the bulk of every
// reference architecture (models/cifar_resnet.py:96-105, models/wide_residual_network.py:20-53,
// models/plainnet.py:52,70) -- and for the 1x1 layers (stride 1 and 2) of keras.applications.ResNet50 (utils.py:237) and
// of the wide-ResNet shortcuts (wide_residual_network.py:28): forward and data gradient.  fp32 NHWC activations are read
// as TF32 operands straight from HBM/L2 (no conversion pass), fp32 accumulation in registers.
//
//   GEMM view   y[m, n] = sum_{tap, k} A_tap[m, k] * B_tap[n, k]
//     m : 128 output pixels of one tile = a (Wb x Hb x Nb) box of the NHWC tensor (powers of two; pixels past the
//         image are zero-filled on load and skipped on store)
//     A_tap : the same box shifted by the filter tap (r - 1, s - 1); TMA zero-fills what lies outside the image, which
//             is the 'same' padding -- no im2col buffer, no index arithmetic on the load path
//     forward : k = input channel,  n = output channel, B = transposed kernel copy [tap][co][ci]
//     dgrad   : k = output channel, n = input channel,  B = the HWIO kernel itself [8 - tap][ci][co]
//               (dX = conv(dY, W rotated by 180 degrees and transposed))
//   1x1 / stride 1 layers are the same GEMM over the flat pixel list (tiles of 128 consecutive pixels), 1x1 / stride 2
//   layers address the input (forward) or the output (backward data) through the sub-sampled view x[:, ::2, ::2, :].
//
// Warp-specialised (384 threads): warp 0 issues the TMA loads of a ring of stages, the two consumer warpgroups
// (threads 128..383) each own 64 rows of the tile and issue m64nBNk8 wgmma on them; the epilogue (bias / residual /
// ReLU / BatchNorm sums, or the accumulate of the data gradient) runs on the accumulator registers.
//
// Stages.  A stage is one (filter tap, channel block) pair, in that order (tap-major).  3x3 layers whose channels fit
// ("resident box", ConvTcParams::res): TMA loads the (Wb + 2) x (Hb + 2) x Nb pixels around the tile -- every channel
// block, once per tile -- and the stages carry only B; tap (r, s) reads the box r * (Wb + 2) + s rows further on, so
// every input pixel is loaded once per tile instead of 9 times.  Other layers (1x1, wide 3x3) load A with each stage,
// as the box shifted by the tap.  Both read A into registers per thread (wgmma with A from registers), so a tap's rows
// need not be whole swizzle groups, and both issue the same MMAs in the same order.
//
// X3 = error-compensated arithmetic ("3xTF32"): every fp32 operand is the sum of hi = its mantissa truncated to 10
// bits and lo = x - hi, and the product is accumulated as A_hi*B_hi + A_hi*B_lo + A_lo*B_hi in the same fp32
// accumulator (the dropped A_lo*B_lo and the truncation of lo are ~2^-21 relative: fp32-level results from
// tensor-core tiles).  Weights: lo is a second B tile written once per step by se_split_filters.  Activations: each
// consumer thread splits its A fragments in registers and feeds both halves to wgmma from registers; nothing in shared
// memory is rewritten.
#include <stdlib.h>

#include "common.cuh"
#include "tc.cuh"

namespace se {

using namespace tc;

constexpr int CT_BM = 128;
constexpr int CT_THREADS = 384;        // warpgroup 0: TMA producer (one thread), warpgroups 1 and 2: MMA + epilogue
constexpr int CT_MAX_STAGES = 6;
constexpr int CT_SMEM_LIMIT = 227 * 1024;

struct ConvTcParams {
  int N, H, W;              // extent of the grid the pixel tiles cover (images, rows, pixels)
  int Kc, Nc, BN;           // GEMM K channels (A tensor channels), GEMM N channels, output channels per tile
  int Wb, Hb, Nb;           // pixel box, Wb*Hb*Nb == 128
  int tw, th;               // tiles along a row / along the rows of an image
  int cblk, kblocks;        // channels per pipeline stage (16 or 32), Kc / cblk
  int taps, pad, flip;      // filter size (3 or 1), 'same' padding rows (1 or 0), 1: dgrad (tap order reversed for B)
  int res;                  // 1: resident box (A loaded once per tile, stages hold B only), 0: per-tap stages
  int ring_off;             // bytes of shared memory before the stage ring (the resident box)
  int stages, stage_bytes, b_bytes;   // stage = [A of one tap (per-tap only)] B [B_lo (X3)]
  int a_bytes, a_tx;        // one A tile (per-tap stage / channel block of the resident box): slot size, TMA bytes
  long long o_sn, o_sh, o_sw;   // output (and residual) element strides of an image, a row, a pixel
  int ovh, ovw;             // rows / pixels of the output view that exist (a strided view may be one short)
  int relu;
  float beta;               // dgrad: out = beta*out + D
  const float* bias;
  const float* residual;
  float* out;
  double* stats;
};

template <int BN>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t a, uint64_t b, int acc) {
  if constexpr (BN == 16) wgmma_tf32_n16(d, a, b, acc);
  else if constexpr (BN == 32) wgmma_tf32_n32(d, a, b, acc);
  else if constexpr (BN == 64) wgmma_tf32_n64(d, a, b, acc);
  else wgmma_tf32_n128(d, a, b, acc);
}

template <int BN>
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t b, int acc) {
  if constexpr (BN == 16) wgmma_tf32_rs_n16(d, a, b, acc);
  else if constexpr (BN == 32) wgmma_tf32_rs_n32(d, a, b, acc);
  else if constexpr (BN == 64) wgmma_tf32_rs_n64(d, a, b, acc);
  else wgmma_tf32_rs_n128(d, a, b, acc);
}

// The A words of k-steps 0..nks-1 for this thread's two rows: a[ks] = (row0, 8ks + t), (row1, 8ks + t),
// (row0, 8ks + 4 + t), (row1, 8ks + 4 + t) -- the register fragment of wgmma_tf32_rs_n*.  Rows are numbered in the
// tile `base` (a stage, or one channel block of the resident box); channel 8ks + 4c + t of a row lies in its 16-byte
// chunk 2ks + c, which the TMA swizzle moves to chunk (2ks + c) ^ (row & 7) for 128-byte rows and
// (2ks + c) ^ ((row >> 1) & 3) for 64-byte rows (tile bases are 1024-byte aligned).
//   Bank conflicts: one load instruction of a warp reads word t of one logical chunk from the rows of 8 consecutive
//   output pixels g = 0..7.  Where these are 8 consecutive rows of the tile (every tile of the per-tap staging; the
//   resident box when Wb >= 8), the load is conflict-free for both widths: 128-byte rows each span all 32 banks and
//   their XOR terms row & 7 are 8 different values -> 8 chunks x 4 words = 32 banks; 64-byte rows alternate between
//   the two bank halves, and the four rows of a half have four different XOR terms (row >> 1) & 3 -> 32 banks.  Only
//   4-pixel-wide boxes (two image rows per 8 pixels) can meet 2-way conflicts.
__device__ __forceinline__ void load_a(uint32_t (&a)[4][4], const uint8_t* base, int row0, int row1, int nks, int row_bytes,
                                       int t) {
  const uint8_t* p0 = base + row0 * row_bytes + 4 * t;
  const uint8_t* p1 = base + row1 * row_bytes + 4 * t;
  const int sw0 = row_bytes == 128 ? row0 & 7 : (row0 >> 1) & 3;
  const int sw1 = row_bytes == 128 ? row1 & 7 : (row1 >> 1) & 3;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    if (ks < nks) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = 2 * ks + (i >> 1);
        a[ks][i] = *reinterpret_cast<const uint32_t*>((i & 1) ? p1 + ((c ^ sw1) << 4) : p0 + ((c ^ sw0) << 4));
      }
    }
  }
}

template <int BN, int X3>
__global__ void __launch_bounds__(CT_THREADS, (X3 && BN == 16) ? 2 : 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
               const __grid_constant__ CUtensorMap map_bl, ConvTcParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring = smem + p.ring_off;
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)p.stages * p.stage_bytes);
  uint64_t* empty = full + CT_MAX_STAGES;
  uint64_t* abar = empty + CT_MAX_STAGES;                                // resident box loaded
  float* s_stats = reinterpret_cast<float*>(abar + 1);                   // [8 consumer warps][2][BN]

  const int tid = threadIdx.x;
  const int tm = blockIdx.x, tn = blockIdx.y;
  const int tw_i = tm % p.tw, rest = tm / p.tw;
  const int w0 = tw_i * p.Wb, h0 = (rest % p.th) * p.Hb, n0 = (rest / p.th) * p.Nb;
  const int row_bytes = p.cblk * 4;
  const int nk = p.taps * p.taps * p.kblocks;

  if (tid == 0) {
    prefetch_tmap(&map_a); prefetch_tmap(&map_b);
    if (X3) prefetch_tmap(&map_bl);
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_init(abar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                               // nothing above touches global memory (see common.cuh)

  if (tid < 128) {
    // ===================== TMA producer
    if (tid == 0) {
      if (p.res) {
        // the resident box: every channel block of the (Wb + 2) x (Hb + 2) x Nb pixels around the tile, once
        mbar_expect_tx(abar, p.kblocks * p.a_tx);
        for (int kb = 0; kb < p.kblocks; ++kb)
          tma_load_4d(smem + (size_t)kb * p.a_bytes, &map_a, abar, kb * p.cblk, w0 - 1, h0 - 1, n0);
      }
      int stage = 0, phase = 0;
      const uint32_t tx = (p.res ? 0 : p.a_tx) + p.b_bytes * (X3 ? 2 : 1);
      for (int it = 0; it < nk; ++it) {
        const int tap = it / p.kblocks, kb = it - tap * p.kblocks;
        const int r = tap / p.taps, s = tap - r * p.taps;
        const int btap = p.flip ? p.taps * p.taps - 1 - tap : tap;
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_expect_tx(&full[stage], tx);
        uint8_t* sb = ring + (size_t)stage * p.stage_bytes;
        if (!p.res) {
          tma_load_4d(sb, &map_a, &full[stage], kb * p.cblk, w0 + s - p.pad, h0 + r - p.pad, n0);
          sb += p.a_bytes;
        }
        tma_load_2d(sb, &map_b, &full[stage], kb * p.cblk, btap * p.Nc + tn * BN);
        if (X3) tma_load_2d(sb + p.b_bytes, &map_bl, &full[stage], kb * p.cblk, btap * p.Nc + tn * BN);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns rows 64*wg .. 64*wg+63 of the tile
  const int wg = (tid >> 7) - 1, tid_wg = tid & 127, lane = tid & 31;
  const int nks = p.cblk / 8;
  // the tile rows of this thread's two A rows (output pixels m and m + 8): in a per-tap stage the pixel index itself,
  // in the resident box the pixel's row for filter tap (0, 0); tap (r, s) is r * (Wb + 2) + s rows further on
  int arow[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = wg * 64 + fragment_row(2 * h, tid_wg);
    const int wb = m % p.Wb, hb = (m / p.Wb) % p.Hb, nb = m / (p.Wb * p.Hb);
    arow[h] = p.res ? (nb * (p.Hb + 2) + hb) * (p.Wb + 2) + wb : m;
  }
  // X3: each stage's MMAs start a fresh register tile `part` that is then added into `acc` -- the tensor core's own
  // accumulation loses low bits with every instruction, which over the 3 x 9 x Kc / 8 MMAs of a wide layer exceeds the
  // fp32-level error budget of this mode
  float acc[BN / 2], part[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  if (p.res) mbar_wait(abar, 0);
  int stage = 0, phase = 0;
  for (int it = 0; it < nk; ++it) {
    const int tap = it / p.kblocks, kb = it - tap * p.kblocks;
    const int r = tap / p.taps, s = tap - r * p.taps;
    mbar_wait(&full[stage], phase);
    const uint8_t* sst = ring + (size_t)stage * p.stage_bytes;
    const uint8_t* abase = p.res ? smem + (size_t)kb * p.a_bytes : sst;
    const int aoff = p.res ? r * (p.Wb + 2) + s : 0;
    const uint32_t b0 = smem_u32(p.res ? sst : sst + p.a_bytes), bl0 = b0 + p.b_bytes;
    uint32_t a[4][4];
    load_a(a, abase, arow[0] + aoff, arow[1] + aoff, nks, row_bytes, lane & 3);
    if (X3) {
      // A is split here: hi = the TF32 truncation, lo = x - hi (exact in fp32).  B is fed as TMA delivered it: the
      // tensor core reads the TF32 truncation of each fp32 word (test_tf32_operands_are_truncated_by_the_tensor_core),
      // i.e. B_hi of w, and of the low parts w - trunc(w) that se_split_filters wrote
      uint32_t lo[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (ks >= nks) break;
          const uint32_t hi = a[ks][i] & 0xFFFFE000u;
          lo[ks][i] = __float_as_uint(__uint_as_float(a[ks][i]) - __uint_as_float(hi));
          a[ks][i] = hi;
        }
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        if (ks < nks) {
          const uint64_t db = wgmma_desc(b0 + ks * 32, row_bytes);
          wgmma_tf32_rs<BN>(part, a[ks], db, ks != 0);
          wgmma_tf32_rs<BN>(part, a[ks], wgmma_desc(bl0 + ks * 32, row_bytes), 1);
          wgmma_tf32_rs<BN>(part, lo[ks], db, 1);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
    } else {
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        if (ks < nks) wgmma_tf32_rs<BN>(acc, a[ks], wgmma_desc(b0 + ks * 32, row_bytes), (it | ks) != 0);
      wgmma_commit();
      wgmma_wait<0>();
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);
    if (++stage == p.stages) { stage = 0; phase ^= 1; }
  }

  // ===================== epilogue on the registers: the two rows of this thread, BN/8 column pairs each
  long long off[2];
  bool valid[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = wg * 64 + fragment_row(2 * h, tid_wg);
    const int wb = m % p.Wb, hb = (m / p.Wb) % p.Hb, nb = m / (p.Wb * p.Hb);
    const int n = n0 + nb, y = h0 + hb, x = w0 + wb;
    valid[h] = n < p.N && y < p.H && x < p.W && y < p.ovh && x < p.ovw;
    off[h] = valid[h] ? n * p.o_sn + y * p.o_sh + x * p.o_sw : 0;
  }
  float csum[BN / 4], csq[BN / 4];
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = tn * BN + 8 * j + 2 * (lane & 3);
    float2 b = make_float2(0.f, 0.f);
    if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
    float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float2 v = make_float2(acc[4 * j + 2 * h] + b.x, acc[4 * j + 2 * h + 1] + b.y);
      if (valid[h]) {
        float2* o = reinterpret_cast<float2*>(p.out + off[h] + col);
        if (p.residual) {
          const float2 e = __ldg(reinterpret_cast<const float2*>(p.residual + off[h] + col));
          v.x += e.x; v.y += e.y;
        }
        if (p.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
        if (p.beta != 0.f) { const float2 prev = *o; v.x += p.beta * prev.x; v.y += p.beta * prev.y; }
        *o = v;
        s0 += v.x; s1 += v.y; q0 += v.x * v.x; q1 += v.y * v.y;
      }
    }
    csum[2 * j] = s0; csum[2 * j + 1] = s1; csq[2 * j] = q0; csq[2 * j + 1] = q1;
  }
  if (p.stats) {
    // column sums over the 8 row groups of the warp (lanes with the same lane & 3), then over the 8 warps in warp order;
    // the per-CTA sums are added across CTAs with float64 atomics (arrival order, float64 rounding)
#pragma unroll
    for (int j = 0; j < BN / 4; ++j) {
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        csum[j] += __shfl_xor_sync(0xffffffffu, csum[j], o);
        csq[j] += __shfl_xor_sync(0xffffffffu, csq[j], o);
      }
    }
    float* sw = s_stats + ((tid - 128) >> 5) * 2 * BN;
    if (lane < 4) {
#pragma unroll
      for (int j = 0; j < BN / 4; ++j) {
        const int c = 8 * (j >> 1) + 2 * lane + (j & 1);
        sw[c] = csum[j];
        sw[BN + c] = csq[j];
      }
    }
    named_bar_sync(2, 256);
    for (int i = tid - 128; i < 2 * BN; i += 256) {
      double v = 0.0;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += (double)s_stats[w * 2 * BN + i];
      if (v != 0.0) atomicAdd(&p.stats[(i >= BN ? p.Nc : 0) + tn * BN + (i % BN)], v);
    }
  }
}

// [tap][ci][co] (HWIO) -> [tap][co][ci] for every listed conv kernel of a flat parameter buffer, in one launch
struct TrEntry { long long off; int taps, cin, cout; };
constexpr int TR_MAX = 160;
struct TrTable { TrEntry e[TR_MAX]; int n; };

// PL / PTL (both or neither): the low parts w - tf32_trunc(w) in the HWIO and the transposed order (error-compensated
// mode: B_lo operands of the backward-data and the forward kernel)
__global__ void __launch_bounds__(256)
transpose_filters_kernel(const float* __restrict__ P, float* __restrict__ PT, float* __restrict__ PL, float* __restrict__ PTL,
                         const __grid_constant__ TrTable tab) {
  pdl_grid_sync();
  for (int li = blockIdx.y; li < tab.n; li += gridDim.y) {
    const TrEntry e = tab.e[li];
    const long long total = (long long)e.taps * e.cin * e.cout;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
      // i indexes the destination [tap][co][ci]
      int ci = (int)(i % e.cin);
      long long t2 = i / e.cin;
      int co = (int)(t2 % e.cout);
      int tap = (int)(t2 / e.cout);
      const long long src = e.off + ((long long)tap * e.cin + ci) * e.cout + co;
      const float v = P[src];
      PT[e.off + i] = v;
      if (PTL) { const float l = tf32_lo(v); PTL[e.off + i] = l; PL[src] = l; }
    }
  }
}

// ---------------------------------------------------------------------------------------- host side
static int pow2_ge(int v) { int q = 1; while (q < v) q <<= 1; return q; }

// image sizes the 3x3 tiles take: rows of 4..56 pixels (every layer of the reference networks at their input sizes)
static bool geometry_ok(int W) { return W >= 4 && W <= 56; }

static bool tc_shape_ok(const se_conv_desc* d, int Kc, int Nc) {
  if (d->kh != 3 || d->kw != 3 || d->stride != 1 || d->pad_t != 1 || d->pad_l != 1 || d->Ho != d->H || d->Wo != d->W)
    return false;
  if (Kc % 16 != 0 || Nc % 16 != 0) return false;
  if (Kc > 16 && Kc % 32 != 0) return false;
  return geometry_ok(d->W);
}

// 1x1 / stride 1 / no padding: a GEMM over the flat pixel list, any image size
static bool tc_shape_ok_1x1(const se_conv_desc* d, int Kc, int Nc) {
  if (d->kh != 1 || d->kw != 1 || d->stride != 1 || d->pad_t != 0 || d->pad_l != 0 || d->Ho != d->H || d->Wo != d->W)
    return false;
  if (Kc % 16 != 0 || Nc % 16 != 0) return false;
  if (Kc > 16 && Kc % 32 != 0) return false;
  return (long long)d->N * d->H * d->W >= CT_BM;
}

// 1x1 / stride 2 / no padding (the first convolution and the projection shortcut of a ResNet-50 stage, the shortcuts of
// wide_residual_network.py:28): the GEMM of the 1x1 case over the (Ho, Wo) grid, the input (forward) or the output
// (backward data) addressed through a tensor map of the sub-sampled VIEW x[:, ::2, ::2, :] (pixel and row strides
// doubled) -- no gather pass.
static bool tc_shape_ok_1x1_s2(const se_conv_desc* d, int Kc, int Nc) {
  if (d->kh != 1 || d->kw != 1 || d->stride != 2 || d->pad_t != 0 || d->pad_l != 0 || d->Ho != (d->H + 1) / 2 ||
      d->Wo != (d->W + 1) / 2)
    return false;
  if (Kc % 16 != 0 || Nc % 16 != 0) return false;
  if (Kc > 16 && Kc % 32 != 0) return false;
  return d->Wo <= 32 && geometry_ok(d->Wo);
}

// output channels per tile: the widest wgmma N that divides the channel count (<= 128; <= 64 in the error-compensated
// mode, whose second accumulator tile would not fit the registers at 128)
static int pick_bn(int Nc, int x3) {
  for (int bn = x3 ? 64 : 128; bn >= 16; bn >>= 1)
    if (Nc % bn == 0) return bn;
  return 0;
}

template <int BN>
static void conv_tc_go(int x3, dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& ma, const CUtensorMap& mb,
                       const CUtensorMap& mbl, const ConvTcParams& p) {
  if constexpr (BN <= 64)       // pick_bn: <= 64 channels per tile in the error-compensated mode
    if (x3) return launch(conv_tc_kernel<BN, 1>, grid, dim3(CT_THREADS), smem, st, ma, mb, mbl, p);
  launch(conv_tc_kernel<BN, 0>, grid, dim3(CT_THREADS), smem, st, ma, mb, mbl, p);
}

static int conv_tc_launch(const se_conv_desc* d, const float* a_tensor, int Kc, const float* bmat, int Nc, int flip,
                          const float* bias, const float* residual, float* out, int relu, float beta, double* stats,
                          cudaStream_t st, const float* bmat_lo = nullptr, int taps = 3, int s2 = 0, int x3_plan = -1,
                          int out_view_w = 0, int out_view_h = 0) {
  // out_view_w / out_view_h (s2 backward data only, 0 = Wo x Ho): extent of the sub-sampled output view that starts at
  // `out` -- a caller that passes dx + (r*W + s)*Cin writes dx[:, r::2, s::2, :], whose last column / row may not exist:
  // one tap of a 3x3 / stride 2 data gradient, conv_dgrad_tc below
  // x3_plan >= 0: plan only (se_conv2d_path) -- the shape / shared-memory decisions below for arithmetic mode x3_plan,
  // no pointers touched, nothing launched: SE_OK when this kernel would take the layer
  // s2 (1x1 / stride 2): tiles over the (Ho, Wo) grid; forward reads the sub-sampled view of a_tensor, backward data
  // (flip) writes the sub-sampled view of out (after zeroing it: the other three quarters of dx are zero)
  ConvTcParams p;
  const int gW = s2 ? d->Wo : d->W, gH = s2 ? d->Ho : d->H;      // the grid the pixel tiles cover
  const int x3 = x3_plan >= 0 ? x3_plan : (bmat_lo ? 1 : 0);   // error-compensated mode: bmat_lo = the low parts of bmat (se_split_filters)
  const long long total_px = (long long)d->N * gH * gW;
  const bool flat = taps == 1 && !s2;
  p.taps = taps; p.pad = taps == 3 ? 1 : 0; p.flip = flip;
  p.N = d->N; p.H = gH; p.W = gW; p.Kc = Kc; p.Nc = Nc;
  if (flat) {
    // a 128-pixel tile is a run of the flat [N*H*W][C] matrix: the kernel sees one "image" of 1 x total_px pixels
    if (total_px > 0x7fffffffLL) return SE_ERR_UNSUPPORTED;
    p.N = 1; p.H = 1; p.W = (int)total_px; p.Wb = CT_BM; p.Hb = 1; p.Nb = 1;
  } else {
    p.Wb = min(pow2_ge(gW), CT_BM);
    p.Hb = min(CT_BM / p.Wb, pow2_ge(gH));
    p.Nb = CT_BM / (p.Wb * p.Hb);
  }
  p.tw = ceil_div(p.W, p.Wb); p.th = ceil_div(p.H, p.Hb);
  const long long tiles_m = (long long)p.tw * p.th * ceil_div(p.N, p.Nb);
  p.BN = pick_bn(Nc, x3);
  if (p.BN == 0 || tiles_m > 0x7fffffffLL || Nc / p.BN > 65535) return SE_ERR_UNSUPPORTED;
  p.cblk = Kc >= 32 ? 32 : 16;
  p.kblocks = Kc / p.cblk;
  // The order in which the products reach the accumulator -- filter tap, then channel block, then k-step -- is the
  // same for both stagings; only where A comes from differs.  The resident box (every channel block of the
  // (Wb + 2) x (Hb + 2) x Nb pixels around the tile, loaded once) is taken whenever it leaves room for a two-stage ring
  // of B tiles; wider 3x3 layers, and the 1x1 layers, stage A once per (tap, channel block).
  p.b_bytes = p.BN * p.cblk * 4;
  const int smem_fixed = 1024 + (2 * CT_MAX_STAGES + 1) * 8 + 16 * p.BN * 4;   // alignment slack, barriers, statistics
  p.res = 0;
  if (taps == 3) {
    p.a_tx = (p.Wb + 2) * (p.Hb + 2) * p.Nb * p.cblk * 4;
    p.a_bytes = (p.a_tx + 1023) & ~1023;                    // 1024-byte aligned: the swizzle pattern starts over
    p.stage_bytes = p.b_bytes * (1 + x3);
    p.res = (CT_SMEM_LIMIT - smem_fixed - p.kblocks * p.a_bytes) / p.stage_bytes >= 2;
  }
  if (!p.res) {
    p.a_tx = p.a_bytes = CT_BM * p.cblk * 4;
    p.stage_bytes = p.a_bytes + p.b_bytes * (1 + x3);
  }
  p.ring_off = p.res ? p.kblocks * p.a_bytes : 0;
  p.stages = min(CT_MAX_STAGES, (CT_SMEM_LIMIT - smem_fixed - p.ring_off) / p.stage_bytes);
  if (p.stages < 2) return SE_ERR_UNSUPPORTED;
  // a CTA runs one tile: a ring longer than the tile's stages would only hold shared memory that other CTAs can use
  p.stages = min(p.stages, taps * taps * p.kblocks);
  p.relu = relu; p.beta = beta;
  p.bias = bias; p.residual = residual; p.out = out; p.stats = stats;
  if (stats && (size_t)16 * Nc * sizeof(float) > 24 * 1024) return SE_ERR_UNSUPPORTED;   // wide layers: separate statistics pass
  if (beta != 0.f && (beta != 1.f || residual || relu)) return SE_ERR_UNSUPPORTED;
  const size_t smem = (size_t)p.ring_off + (size_t)p.stages * p.stage_bytes + smem_fixed;
  if (smem > CT_SMEM_LIMIT) return SE_ERR_UNSUPPORTED;
  if (x3_plan >= 0) return SE_OK;
  // output (and residual) addressing: NHWC over the tile grid, or the strided view dx[:, ::2, ::2, :] (s2 backward data)
  p.o_sw = Nc; p.o_sh = (long long)p.W * Nc; p.o_sn = (long long)p.H * p.W * Nc;
  p.ovw = p.W; p.ovh = p.H;
  if (s2 && flip) {
    p.o_sw = 2LL * Nc; p.o_sh = 2LL * d->W * Nc; p.o_sn = (long long)d->H * d->W * Nc;
    if (out_view_w) p.ovw = out_view_w;
    if (out_view_h) p.ovh = out_view_h;
  }
  CUtensorMap ma, mb, mbl;
  {
    uint64_t dims[4] = {(uint64_t)Kc, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.N};
    uint64_t strides[3] = {(uint64_t)Kc * 4, (uint64_t)p.W * Kc * 4, (uint64_t)p.H * p.W * Kc * 4};
    if (s2 && !flip) {      // forward: x[:, ::2, ::2, :]
      strides[0] = (uint64_t)2 * Kc * 4; strides[1] = (uint64_t)2 * d->W * Kc * 4; strides[2] = (uint64_t)d->H * d->W * Kc * 4;
    }
    uint32_t box[4] = {(uint32_t)p.cblk, (uint32_t)(p.Wb + 2 * p.res), (uint32_t)(p.Hb + 2 * p.res), (uint32_t)p.Nb};
    CUtensorMapSwizzle sw = p.cblk == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    if (!make_tmap(&ma, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(a_tensor), dims, strides, box, sw)) return SE_ERR_CUDA;
    uint64_t bdims[2] = {(uint64_t)Kc, (uint64_t)taps * taps * Nc};
    uint64_t bstrides[1] = {(uint64_t)Kc * 4};
    uint32_t bbox[2] = {(uint32_t)p.cblk, (uint32_t)p.BN};
    if (!make_tmap(&mb, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(bmat), bdims, bstrides, bbox, sw)) return SE_ERR_CUDA;
    mbl = mb;
    if (x3 && !make_tmap(&mbl, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(bmat_lo), bdims, bstrides, bbox, sw))
      return SE_ERR_CUDA;
  }
  if (s2 && flip && beta == 0.f &&
      cudaMemsetAsync(out, 0, (size_t)d->N * d->H * d->W * Nc * sizeof(float), st) != cudaSuccess) {
    set_error("conv_tc: cudaMemsetAsync failed");
    return SE_ERR_CUDA;
  }
  const dim3 grid((unsigned)tiles_m, (unsigned)(Nc / p.BN));
  switch (p.BN) {
    case 16: conv_tc_go<16>(x3, grid, smem, st, ma, mb, mbl, p); break;
    case 32: conv_tc_go<32>(x3, grid, smem, st, ma, mb, mbl, p); break;
    case 64: conv_tc_go<64>(x3, grid, smem, st, ma, mb, mbl, p); break;
    default: conv_tc_go<128>(x3, grid, smem, st, ma, mb, mbl, p); break;
  }
  return check_launch("conv_tc_kernel");
}

template <int BN>
static bool set_smem_limit() {
  if constexpr (BN <= 64)
    if (cudaFuncSetAttribute(conv_tc_kernel<BN, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM_LIMIT) != cudaSuccess)
      return false;
  return cudaFuncSetAttribute(conv_tc_kernel<BN, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM_LIMIT) == cudaSuccess;
}

int init_conv_tc() {
  if (!set_smem_limit<16>() || !set_smem_limit<32>() || !set_smem_limit<64>() || !set_smem_limit<128>()) {
    set_error("init_conv_tc: cannot raise the shared-memory limit");
    return SE_ERR_CUDA;
  }
  return SE_OK;
}

static bool g_tc_inited = false;
static int ensure_init() {
  if (!g_tc_inited) { int rc = init_conv_tc(); if (rc) return rc; g_tc_inited = true; }
  return SE_OK;
}

// forward needs the transposed kernel copy w_t = [tap][co][ci]; without it the caller falls back to the fp32 kernels
// w_t_lo != null selects the error-compensated arithmetic (w_t_lo = low parts of w_t, se_split_filters)
int conv_fwd_tc(const se_conv_desc* d, const float* x, const float* w_t, const float* w_t_lo, const float* bias,
                const float* residual, float* y, int relu, double* stats, cudaStream_t st) {
  if (!w_t) return SE_ERR_UNSUPPORTED;
  const bool k2 = tc_shape_ok_1x1_s2(d, d->Cin, d->Cout);
  const bool k1 = k2 || tc_shape_ok_1x1(d, d->Cin, d->Cout);
  if (!k1 && !tc_shape_ok(d, d->Cin, d->Cout)) return SE_ERR_UNSUPPORTED;
  int rc = ensure_init();
  if (rc) return rc;
  return conv_tc_launch(d, x, d->Cin, w_t, d->Cout, 0, bias, residual, y, relu, 0.f, stats, st, w_t_lo, k1 ? 1 : 3, k2);
}

bool conv3x3s2_tc_ok(const se_conv_desc* d);      // conv_wgrad_tc.cu

// 3x3 / stride 2 / no leading padding, wide layers (see conv3x3s2_tc_ok): nine 1x1 / stride 2 data gradients, one per
// filter tap, each added into its own sub-sampled view of dx:   dx[:, r::2, s::2, :] += dY W[r, s]^T
static int conv_dgrad_tc_3x3s2(const se_conv_desc* d, const float* dy, const float* w, const float* w_lo, float* dx, float beta,
                               cudaStream_t st) {
  if (beta != 0.f && beta != 1.f) return SE_ERR_UNSUPPORTED;
  int rc = ensure_init();
  if (rc) return rc;
  se_conv_desc d1 = *d;
  d1.kh = 1; d1.kw = 1;
  if (!tc_shape_ok_1x1_s2(&d1, d->Cout, d->Cin)) return SE_ERR_UNSUPPORTED;
  if (beta == 0.f && cudaMemsetAsync(dx, 0, (size_t)d->N * d->H * d->W * d->Cin * sizeof(float), st) != cudaSuccess) {
    set_error("conv_dgrad_tc: cudaMemsetAsync failed");
    return SE_ERR_CUDA;
  }
  for (int r = 0; r < 3; ++r)
    for (int s = 0; s < 3; ++s) {
      const long long woff = (long long)(r * 3 + s) * d->Cin * d->Cout;
      rc = conv_tc_launch(&d1, dy, d->Cout, w + woff, d->Cin, 1, nullptr, nullptr, dx + ((long long)r * d->W + s) * d->Cin, 0, 1.f,
                          nullptr, st, w_lo ? w_lo + woff : nullptr, 1, 1, -1, d->Wo - (s == 2), d->Ho - (r == 2));
      if (rc != SE_OK) return rc;
    }
  return SE_OK;
}

int conv_dgrad_tc(const se_conv_desc* d, const float* dy, const float* w, const float* w_lo, float* dx, float beta,
                  cudaStream_t st) {
  if (conv3x3s2_tc_ok(d)) return conv_dgrad_tc_3x3s2(d, dy, w, w_lo, dx, beta, st);
  const bool k2 = tc_shape_ok_1x1_s2(d, d->Cout, d->Cin);
  const bool k1 = k2 || tc_shape_ok_1x1(d, d->Cout, d->Cin);
  if (!k1 && !tc_shape_ok(d, d->Cout, d->Cin)) return SE_ERR_UNSUPPORTED;
  int rc = ensure_init();
  if (rc) return rc;
  return conv_tc_launch(d, dy, d->Cout, w, d->Cin, 1, nullptr, nullptr, dx, 0, beta, nullptr, st, w_lo, k1 ? 1 : 3, k2);
}

// se_conv2d_path: would the tensor-core kernel of this file take the layer?  (dir 0 forward, 1 backward data; x3 = 0 / 1)
bool conv_tc_would_run(const se_conv_desc* d, int dir, int x3) {
  if (dir == 1 && conv3x3s2_tc_ok(d)) {
    se_conv_desc d1 = *d;
    d1.kh = 1; d1.kw = 1;
    return conv_tc_would_run(&d1, 1, x3);
  }
  const int Kc = dir == 0 ? d->Cin : d->Cout, Nc = dir == 0 ? d->Cout : d->Cin;
  const bool k2 = tc_shape_ok_1x1_s2(d, Kc, Nc);
  const bool k1 = k2 || tc_shape_ok_1x1(d, Kc, Nc);
  if (!k1 && !tc_shape_ok(d, Kc, Nc)) return false;
  return conv_tc_launch(d, nullptr, Kc, nullptr, Nc, dir, nullptr, nullptr, nullptr, 0, 0.f, nullptr, nullptr, nullptr, k1 ? 1 : 3,
                        k2, x3) == SE_OK;
}

int transpose_filters(const float* P, float* PT, float* PL, float* PTL, const long long* table, int n, cudaStream_t st) {
  for (int base = 0; base < n; base += TR_MAX) {
    TrTable tab;
    tab.n = min(TR_MAX, n - base);
    long long maxtot = 1;
    for (int i = 0; i < tab.n; ++i) {
      const long long* e = table + 4 * (base + i);
      tab.e[i].off = e[0]; tab.e[i].taps = (int)e[1]; tab.e[i].cin = (int)e[2]; tab.e[i].cout = (int)e[3];
      maxtot = max(maxtot, e[1] * e[2] * e[3]);
    }
    long long gx = ceil_div<long long>(maxtot, 256);
    dim3 grid((unsigned)(gx < 64 ? gx : 64), (unsigned)tab.n);
    launch(transpose_filters_kernel, dim3(grid), dim3(256), 0, st, P, PT, PL, PTL, tab);
    int rc = check_launch("transpose_filters_kernel");
    if (rc) return rc;
  }
  return SE_OK;
}

// bit 0 conv fwd, bit 1 conv dgrad, bit 2 conv wgrad, bit 3 pairwise: which tensor-core kernels are compiled in
int tc_capabilities() { return 1 | 2 | 4 | 8; }

}  // namespace se
