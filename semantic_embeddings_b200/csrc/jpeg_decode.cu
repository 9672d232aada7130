// Batched JPEG decoding on the device, bit-identical to libjpeg-turbo's default decode as Pillow runs it (load_img):
// Huffman decoding, DC prediction, dequantisation, jpeg_idct_islow, fancy upsampling and YCbCr -> RGB, all in the
// integer arithmetic libjpeg uses.  The host (jpeg_parse.cu) has checked every header, built the Huffman lookup tables
// and removed the byte stuffing and restart markers; this file never sees a stream that parser rejected.
//
// 1. entropy_kernel, one CTA per image: Huffman decoding in parallel within the image, after Weissenberger & Schmidt
//    ("Massively parallel Huffman decoding on GPUs", ICPP 2018; JPEG decoding, 2021).  Each restart interval is cut
//    into subsequences of SE_JPEG_SUBSEQ_BYTES; a decoder state is (bit position, block within the MCU, zig-zag index)
//    at a code boundary.  Each thread owns a contiguous run of subsequences and
//      a. decodes its run speculatively: its first subsequence from (its first bit, block 0, index 0) -- the true
//         state when the subsequence opens a restart interval -- the next ones from where the previous one stopped;
//      b. synchronises: when the state the predecessor's run ended in differs from the one the thread started from,
//         it decodes again from that state, subsequence after subsequence, until it reaches an entry state it had
//         already used (from there on, its earlier decode was the true one: the decode is a function of the state).
//         Repeated until no thread changes anything; Huffman codes resynchronise after a few codes, so a pass or
//         two suffices, and in the worst case every run is decoded once per pass ahead of it;
//      c. takes an exclusive scan of the blocks completed and of the DC differences summed per component in each
//         subsequence (minus the prefix at the interval's start: DC predictions restart at every interval), and
//      d. decodes once more from the synchronised entry states, writing each coefficient at its block's place in
//         the component planes (DC = prediction + difference, in 32-bit wrapping arithmetic, stored as int16 as
//         libjpeg's JCOEF).  A run longer than the block writes coefficient 63, as libjpeg's natural-order table does.
//    An interval that yields fewer blocks than it should (the data ended, or a code matched no table) sets the
//    image's status to SE_JPEG_DEV_CORRUPT; Pillow would decode such a file with a warning and the caller re-decodes it
//    on the host.
// 2. idct_kernel: jidctint.c jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2, DESCALE rounding, 64-bit intermediates
//    like its JLONG) on the dequantised block, columns then rows, output through libjpeg's sample_range_limit table
//    indexed with RANGE_MASK (1023), built the way jdmaster.c prepare_range_limit_table builds it.  8 threads per block.
//    A dequantised coefficient outside int16 sets SE_JPEG_DEV_CORRUPT (libjpeg-turbo's SIMD and C paths differ there).
// 3. color_kernel, one thread per output pixel: jdsample.c's h2v1 / h1v2 / h2v2 fancy upsampling of the chroma planes
//    (the triangle filters with their alternating rounding biases, first / last columns special-cased, the rows above
//    the first and below the last (downsampled_height) row replicated as jdmainct.c's context rows are, plain
//    replication when the chroma width is <= 2 as jinit_upsampler chooses), then jdcolor.c ycc_rgb_convert
//    (SCALEBITS 16, ONE_HALF rounding, range limit).  One component: R = G = B = Y, as convert('RGB') does.
#include <algorithm>

#include "common.cuh"

namespace se {

namespace {

constexpr int kEntropyThreads = 512;
constexpr uint64_t kDead = ~0ull;          // a decoder that ran out of data or met a code no table matches
constexpr int kIdctBlocks = 32;            // DCT blocks per CTA of idct_kernel (8 threads each)

__constant__ int kNaturalDev[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Block geometry of a frame (libjpeg's jdinput.c initial_setup / per_scan_setup)
struct Geo {
  int nc, bpm, W, H, mcus_x;
  int h[3], v[3];
  int dw[3], dh[3];                // downsampled_width / downsampled_height
  int bw[3], bh[3];                // blocks per row / column of each component plane
  long long boff[3];               // first block of each component in the image's block arrays
  long long nblocks;
  int blk_comp[10], blk_dx[10], blk_dy[10];   // the blocks of an MCU
};

__host__ __device__ inline void geometry(const se_jpeg_info& f, Geo& g) {
  g.nc = f.ncomp;
  g.W = f.width;
  g.H = f.height;
  g.mcus_x = f.mcus_x;
  g.bpm = 0;
  long long off = 0;
  for (int c = 0; c < 3; ++c) {
    if (c >= f.ncomp) {
      g.boff[c] = off;
      g.h[c] = g.v[c] = 1;
      g.dw[c] = g.dh[c] = g.bw[c] = g.bh[c] = 0;
      continue;
    }
    g.h[c] = f.h[c];
    g.v[c] = f.v[c];
    g.dw[c] = (f.width * f.h[c] + f.hmax - 1) / f.hmax;
    g.dh[c] = (f.height * f.v[c] + f.vmax - 1) / f.vmax;
    if (f.ncomp == 1) {
      g.bw[c] = (g.dw[c] + 7) / 8;
      g.bh[c] = (g.dh[c] + 7) / 8;
      g.blk_comp[0] = 0;
      g.blk_dx[0] = g.blk_dy[0] = 0;
      g.bpm = 1;
    } else {
      g.bw[c] = f.mcus_x * f.h[c];
      g.bh[c] = f.mcus_y * f.v[c];
      for (int y = 0; y < f.v[c]; ++y)
        for (int x = 0; x < f.h[c]; ++x) {
          g.blk_comp[g.bpm] = c;
          g.blk_dx[g.bpm] = x;
          g.blk_dy[g.bpm] = y;
          ++g.bpm;
        }
    }
    g.boff[c] = off;
    off += (long long)g.bw[c] * g.bh[c];
  }
  g.nblocks = off;
}

__host__ __device__ inline long long align256(long long v) { return (v + 255) & ~255LL; }
__host__ __device__ inline long long align16(long long v) { return (v + 15) & ~15LL; }

// The workspace of one image: coefficients (int16), samples (uint8), and per subsequence the entry and exit states,
// the statistics (blocks completed, DC difference sums of 3 components) and their exclusive prefix.
struct Layout {
  long long coef, samp, entry, exit, stats, prefix, total;
};
__host__ __device__ inline Layout layout(const Geo& g, int nsub) {
  Layout L;
  L.coef = 0;
  L.samp = L.coef + align256(g.nblocks * 64 * 2);
  L.entry = L.samp + align256(g.nblocks * 64);
  L.exit = L.entry + align256((long long)nsub * 8);
  L.stats = L.exit + align256((long long)nsub * 8);
  L.prefix = L.stats + align256((long long)nsub * 16);
  L.total = L.prefix + align256((long long)(nsub + 1) * 16);
  return L;
}

// jdmaster.c prepare_range_limit_table for 8-bit samples, at srl[0 .. 5 * 256 + 128): sample_range_limit = srl + 256
// (x < 0 -> 0, 0..255 -> x, 256.. -> 255), the IDCT's table at sample_range_limit + 128, indexed with x & 1023.
__device__ void build_range_limit(unsigned char* srl) {
  for (int i = threadIdx.x; i < 5 * 256 + 128; i += blockDim.x) {
    int v;
    if (i < 256) v = 0;                          // limit[x] = 0 for x < 0
    else if (i < 512) v = i - 256;               // limit[x] = x
    else if (i < 256 + 128 + 512) v = 255;       // rest of the first half of the post-IDCT table
    else if (i < 256 + 128 + 1024 - 128) v = 0;  // second half: zeros ...
    else v = i - (256 + 128 + 1024 - 128);       // ... then the copy of limit[0 .. 127]
    srl[i] = (unsigned char)v;
  }
}

__device__ __forceinline__ uint32_t peek32(const uint8_t* __restrict__ d, uint32_t pos) {
  const uint8_t* p = d + (pos >> 3);
  const uint64_t v = ((uint64_t)p[0] << 32) | ((uint64_t)p[1] << 24) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 8) |
                     (uint64_t)p[4];
  return (uint32_t)(v >> (8 - (pos & 7)));
}

__device__ __forceinline__ uint64_t mk_state(uint32_t pos, int b, int k) {
  return ((uint64_t)pos << 16) | ((uint64_t)b << 8) | (uint64_t)k;
}

struct EntropyShared {
  se_jpeg_huff dc[3], ac[3];
  Geo geo;
};

struct Writer {
  int16_t* coef;
  long long gbase;                 // global index of the interval's first block
  uint32_t g, gmax;                // block within the interval, blocks of the interval
  uint32_t pred[3];                // DC predictions
};

__device__ __forceinline__ int16_t* block_ptr(const Geo& g, int16_t* coef, long long gi) {
  if (g.nc == 1) return coef + gi * 64;
  const long long mcu = gi / g.bpm;
  const int b = (int)(gi - mcu * g.bpm);
  const int c = g.blk_comp[b];
  const long long my = mcu / g.mcus_x, mx = mcu - my * g.mcus_x;
  const long long bx = mx * g.h[c] + g.blk_dx[b], by = my * g.v[c] + g.blk_dy[b];
  return coef + (g.boff[c] + by * g.bw[c] + bx) * 64;
}

// Decodes from state `st` while the position is below `end` (codes may run on up to `limit`, the interval's end).
// stat: blocks completed, DC difference sums per component.  WRITE: also stores the coefficients through w.
template <bool WRITE>
__device__ uint64_t run(uint64_t st, uint32_t end, uint32_t limit, const uint8_t* __restrict__ d, const EntropyShared& S,
                        uint32_t* stat, Writer* w) {
  if (st == kDead) return kDead;
  uint32_t pos = (uint32_t)(st >> 16);
  int b = (int)((st >> 8) & 0xFF), k = (int)(st & 0xFF);
  int16_t* blk = nullptr;
  if (WRITE) {
    if (w->g >= w->gmax) return st;
    blk = block_ptr(S.geo, w->coef, w->gbase + w->g);
  }
  const int bpm = S.geo.bpm;
  while (pos < end) {
    const int c = S.geo.blk_comp[b];
    const se_jpeg_huff& t = k == 0 ? S.dc[c] : S.ac[c];
    const uint32_t bits = peek32(d, pos);
    int l, sym;
    const int e = t.lookup[bits >> 23];
    if (e) {
      l = e >> 8;
      sym = e & 0xFF;
    } else {
      l = 10;
      int code = (int)(bits >> 22);
      while (code > t.maxcode[l]) {
        if (++l > 16) return kDead;
        code = (int)(bits >> (32 - l));
      }
      sym = t.huffval[(code + t.valoffset[l]) & 0xFF];
    }
    const int s = k == 0 ? sym : (sym & 15);
    if ((uint64_t)pos + (uint64_t)(l + s) > limit) return kDead;
    int val = 0;
    if (s) {
      const uint32_t x = (bits << l) >> (32 - s);
      val = x < (1u << (s - 1)) ? (int)x - (1 << s) + 1 : (int)x;   // HUFF_EXTEND
    }
    pos += l + s;
    if (k == 0) {
      stat[1 + c] += (uint32_t)val;
      if (WRITE) {
        w->pred[c] += (uint32_t)val;
        blk[0] = (int16_t)(uint16_t)w->pred[c];
      }
      k = 1;
    } else {
      const int r = sym >> 4;
      if (s == 0) {
        k = r == 15 ? k + 16 : 64;                 // ZRL / EOB
      } else {
        k += r;
        if (WRITE) blk[kNaturalDev[k > 63 ? 63 : k]] = (int16_t)val;
        k += 1;
      }
    }
    if (k >= 64) {
      k = 0;
      b = b + 1 == bpm ? 0 : b + 1;
      stat[0] += 1;
      if (WRITE) {
        if (++w->g >= w->gmax) return mk_state(pos, b, k);
        blk = block_ptr(S.geo, w->coef, w->gbase + w->g);
      }
    }
  }
  return mk_state(pos, b, k);
}

struct Sub {
  uint32_t begin, end, limit;
};
__device__ __forceinline__ Sub sub_bits(const uint32_t* int_start, const uint32_t* sub_first, int i, int j) {
  Sub s;
  s.limit = int_start[i + 1] * 8u;
  s.begin = int_start[i] * 8u + (uint32_t)(j - (int)sub_first[i]) * (SE_JPEG_SUBSEQ_BYTES * 8u);
  s.end = min(s.begin + SE_JPEG_SUBSEQ_BYTES * 8u, s.limit);
  return s;
}

__global__ void __launch_bounds__(kEntropyThreads)
entropy_kernel(const uint8_t* __restrict__ in, const se_jpeg_job* __restrict__ jobs, uint8_t* __restrict__ ws,
               int32_t* __restrict__ status) {
  __shared__ EntropyShared S;
  __shared__ uint32_t scan[4][kEntropyThreads];
  __shared__ int err;
  const int tid = threadIdx.x, T = kEntropyThreads;
  // launched without programmatic dependent launch: see se_jpeg_decode_batch

  const se_jpeg_job job = jobs[blockIdx.x];
  const se_jpeg_info* f = (const se_jpeg_info*)(in + job.info_offset);
  const int nc = f->ncomp;
  {
    const int words = (int)(sizeof(se_jpeg_huff) / 4);
    for (int i = tid; i < 2 * nc * words; i += T) {
      const int c = i / (2 * words), r = i - c * 2 * words, ac = r >= words, o = ac ? r - words : r;
      const se_jpeg_huff* src = ac ? &f->ac[f->ta[c]] : &f->dc[f->td[c]];
      ((uint32_t*)(ac ? &S.ac[c] : &S.dc[c]))[o] = ((const uint32_t*)src)[o];
    }
  }
  if (tid == 0) {
    geometry(*f, S.geo);
    err = 0;
  }
  __syncthreads();
  const int nint = f->n_intervals, nsub = f->n_subseq;
  const long long ri = f->restart_interval;
  const uint8_t* packed = in + job.packed_offset;
  const uint32_t* int_start = (const uint32_t*)packed;
  const uint32_t* sub_first = int_start + nint + 1;
  const uint8_t* data = packed + align16(8LL * (nint + 1));
  const Layout L = layout(S.geo, nsub);
  uint8_t* base = ws + job.ws_offset;
  int16_t* coef = (int16_t*)(base + L.coef);
  uint64_t* entry = (uint64_t*)(base + L.entry);
  uint64_t* exitst = (uint64_t*)(base + L.exit);
  uint4* stats = (uint4*)(base + L.stats);
  uint4* prefix = (uint4*)(base + L.prefix);
  const long long per_int = ri ? ri * S.geo.bpm : S.geo.nblocks;
  auto expected = [&](int i) -> long long {
    return i + 1 < nint ? per_int : S.geo.nblocks - (long long)(nint - 1) * per_int;
  };

  const int q = (nsub + T - 1) / T;
  const int j0 = min(tid * q, nsub), j1 = min(j0 + q, nsub);
  int i0 = 0;                                            // interval of j0: the last i with sub_first[i] <= j0
  if (j0 < j1) {
    int lo = 0, hi = nint - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if ((int)sub_first[mid] <= j0) lo = mid;
      else hi = mid - 1;
    }
    i0 = lo;
  }

  // a. speculative decode of the run
  {
    int i = i0;
    uint64_t prev = kDead;
    for (int j = j0; j < j1; ++j) {
      while ((int)sub_first[i + 1] <= j) ++i;
      const Sub s = sub_bits(int_start, sub_first, i, j);
      const uint64_t e = (j == (int)sub_first[i] || j == j0) ? mk_state(s.begin, 0, 0) : prev;
      uint32_t st[4] = {0, 0, 0, 0};
      prev = run<false>(e, s.end, s.limit, data, S, st, nullptr);
      entry[j] = e;
      exitst[j] = prev;
      stats[j] = make_uint4(st[0], st[1], st[2], st[3]);
    }
  }
  __syncthreads();

  // b. synchronisation
  const bool opens = j0 < j1 && j0 == (int)sub_first[i0];
  for (;;) {
    bool need = false;
    uint64_t e = 0;
    if (j0 < j1 && !opens) {
      e = exitst[j0 - 1];
      need = e != entry[j0];
    }
    __syncthreads();
    if (need) {
      int i = i0;
      for (int j = j0; j < j1; ++j) {
        while ((int)sub_first[i + 1] <= j) ++i;
        if (j > j0) {
          if (j == (int)sub_first[i]) break;
          e = exitst[j - 1];
          if (e == entry[j]) break;
        }
        const Sub s = sub_bits(int_start, sub_first, i, j);
        uint32_t st[4] = {0, 0, 0, 0};
        entry[j] = e;
        exitst[j] = run<false>(e, s.end, s.limit, data, S, st, nullptr);
        stats[j] = make_uint4(st[0], st[1], st[2], st[3]);
      }
    }
    if (!__syncthreads_or(need)) break;
  }

  // c. exclusive scan of the statistics
  uint32_t loc[4] = {0, 0, 0, 0};
  for (int j = j0; j < j1; ++j) {
    const uint4 s = stats[j];
    loc[0] += s.x;
    loc[1] += s.y;
    loc[2] += s.z;
    loc[3] += s.w;
  }
  for (int c = 0; c < 4; ++c) scan[c][tid] = loc[c];
  __syncthreads();
  for (int off = 1; off < T; off <<= 1) {
    uint32_t add[4];
    for (int c = 0; c < 4; ++c) add[c] = tid >= off ? scan[c][tid - off] : 0u;
    __syncthreads();
    for (int c = 0; c < 4; ++c) scan[c][tid] += add[c];
    __syncthreads();
  }
  {
    uint4 run_p = tid ? make_uint4(scan[0][tid - 1], scan[1][tid - 1], scan[2][tid - 1], scan[3][tid - 1])
                      : make_uint4(0, 0, 0, 0);
    for (int j = j0; j < j1; ++j) {
      prefix[j] = run_p;
      const uint4 s = stats[j];
      run_p.x += s.x;
      run_p.y += s.y;
      run_p.z += s.z;
      run_p.w += s.w;
    }
    if (tid == T - 1) prefix[nsub] = make_uint4(scan[0][T - 1], scan[1][T - 1], scan[2][T - 1], scan[3][T - 1]);
  }
  __syncthreads();

  // every interval must yield its blocks
  for (int i = tid; i < nint; i += T) {
    const uint32_t got = prefix[sub_first[i + 1]].x - prefix[sub_first[i]].x;
    if ((long long)got < expected(i)) atomicOr(&err, 1);
  }
  __syncthreads();
  if (tid == 0) status[blockIdx.x] = err ? SE_JPEG_DEV_CORRUPT : SE_JPEG_OK;
  if (err) return;

  // d. write the coefficients
  int i = i0;
  for (int j = j0; j < j1; ++j) {
    while ((int)sub_first[i + 1] <= j) ++i;
    const uint4 pf = prefix[sub_first[i]], p = prefix[j];
    Writer w;
    w.coef = coef;
    w.gbase = (long long)i * per_int;
    w.g = p.x - pf.x;
    w.gmax = (uint32_t)expected(i);
    w.pred[0] = p.y - pf.y;
    w.pred[1] = p.z - pf.z;
    w.pred[2] = p.w - pf.w;
    const Sub s = sub_bits(int_start, sub_first, i, j);
    uint32_t st[4] = {0, 0, 0, 0};
    run<true>(entry[j], s.end, s.limit, data, S, st, &w);
  }
}

// jidctint.c: the 1-D LL&M transform shared by both passes (inputs already dequantised / from the workspace), 64-bit
// like JLONG; outputs before DESCALE in libjpeg's order.
__device__ __forceinline__ void idct8(const long long* x, long long* o) {
  long long z2 = x[2], z3 = x[6];
  long long z1 = (z2 + z3) * 4433;                           // FIX_0_541196100
  long long tmp2 = z1 + z3 * -15137;                         // FIX_1_847759065
  long long tmp3 = z1 + z2 * 6270;                           // FIX_0_765366865
  z2 = x[0];
  z3 = x[4];
  long long tmp0 = (z2 + z3) * 8192;                         // LEFT_SHIFT(.., CONST_BITS)
  long long tmp1 = (z2 - z3) * 8192;
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = x[7];
  tmp1 = x[5];
  tmp2 = x[3];
  tmp3 = x[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * 9633;                     // FIX_1_175875602
  tmp0 *= 2446;                                              // FIX_0_298631336
  tmp1 *= 16819;                                             // FIX_2_053119869
  tmp2 *= 25172;                                             // FIX_3_072711026
  tmp3 *= 12299;                                             // FIX_1_501321110
  z1 *= -7373;                                               // FIX_0_899976223
  z2 *= -20995;                                              // FIX_2_562915447
  z3 *= -16069;                                              // FIX_1_961570560
  z4 *= -3196;                                               // FIX_0_390180644
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  o[0] = tmp10 + tmp3;
  o[7] = tmp10 - tmp3;
  o[1] = tmp11 + tmp2;
  o[6] = tmp11 - tmp2;
  o[2] = tmp12 + tmp1;
  o[5] = tmp12 - tmp1;
  o[3] = tmp13 + tmp0;
  o[4] = tmp13 - tmp0;
}

__device__ __forceinline__ long long descale(long long x, int n) { return (x + (1LL << (n - 1))) >> n; }

__global__ void __launch_bounds__(kIdctBlocks * 8)
idct_kernel(const uint8_t* __restrict__ in, const se_jpeg_job* __restrict__ jobs, uint8_t* __restrict__ ws,
            int32_t* __restrict__ status) {
  __shared__ unsigned char srl[5 * 256 + 128];
  __shared__ int wsp[kIdctBlocks][64];
  __shared__ Geo geo;
  build_range_limit(srl);
  const se_jpeg_job job = jobs[blockIdx.y];
  const se_jpeg_info* f = (const se_jpeg_info*)(in + job.info_offset);
  if (threadIdx.x == 0) geometry(*f, geo);
  __syncthreads();
  const unsigned char* range = srl + 256 + 128;
  const Layout L = layout(geo, f->n_subseq);
  const int lb = threadIdx.x >> 3, t = threadIdx.x & 7;
  const long long gb = (long long)blockIdx.x * kIdctBlocks + lb;
  const bool active = gb < geo.nblocks;
  int c = 0;
  if (geo.nc == 3) c = gb >= geo.boff[2] ? 2 : (gb >= geo.boff[1] ? 1 : 0);
  const int16_t* cf = (const int16_t*)(ws + job.ws_offset + L.coef) + gb * 64;
  const uint16_t* qt = f->qt[f->tq[c]];
  long long x[8], o[8];
  if (active) {                                              // pass 1: column t
    bool wide = false;
    for (int r = 0; r < 8; ++r) {
      x[r] = (long long)cf[r * 8 + t] * (long long)qt[r * 8 + t];
      wide |= x[r] < -32768 || x[r] > 32767;
    }
    // libjpeg-turbo's SIMD IDCT dequantises with 16-bit multiplies (the low half of the product), its C IDCT with the
    // full product: a product outside int16 (never met in real images) has no single libjpeg answer to reproduce, so
    // the image goes back to the host decoder.  Every writer stores the same value: no ordering is needed.
    if (wide) status[blockIdx.y] = SE_JPEG_DEV_CORRUPT;
    idct8(x, o);
    for (int r = 0; r < 8; ++r) wsp[lb][r * 8 + t] = (int)descale(o[r], 11);   // CONST_BITS - PASS1_BITS
  }
  __syncwarp();
  if (active) {                                              // pass 2: row t
    for (int cc = 0; cc < 8; ++cc) x[cc] = (long long)wsp[lb][t * 8 + cc];
    idct8(x, o);
    unsigned char px[8];
    for (int cc = 0; cc < 8; ++cc) px[cc] = range[(int)descale(o[cc], 18) & 1023];   // CONST_BITS + PASS1_BITS + 3
    const long long lbc = gb - geo.boff[c];
    const long long by = lbc / geo.bw[c], bx = lbc - by * geo.bw[c];
    uint8_t* dst = ws + job.ws_offset + L.samp + geo.boff[c] * 64 + (by * 8 + t) * (long long)(geo.bw[c] * 8) + bx * 8;
    uint2 pk;
    pk.x = px[0] | (px[1] << 8) | (px[2] << 16) | ((uint32_t)px[3] << 24);
    pk.y = px[4] | (px[5] << 8) | (px[6] << 16) | ((uint32_t)px[7] << 24);
    *(uint2*)dst = pk;
  }
}

// jdsample.c fancy upsampling of a chroma plane at output pixel (x, y); luma factors (hf, vf) in {1, 2}
__device__ __forceinline__ int upsample(const uint8_t* __restrict__ p, int stride, int dw, int dh, int hf, int vf, int x,
                                        int y) {
  if (hf == 1 && vf == 1) return p[(long long)y * stride + x];
  if (hf == 2 && vf == 1) {                                  // h2v1_fancy_upsample
    const uint8_t* row = p + (long long)y * stride;
    const int cx = x >> 1;
    if (dw <= 2) return row[cx];
    const int v3 = 3 * row[cx];
    if ((x & 1) == 0) return cx == 0 ? row[0] : (v3 + row[cx - 1] + 1) >> 2;
    return cx == dw - 1 ? row[cx] : (v3 + row[cx + 1] + 2) >> 2;
  }
  const int r = y >> 1;
  const int rn = (y & 1) ? min(r + 1, dh - 1) : max(r - 1, 0);      // context rows: first / last row replicated
  const uint8_t* near = p + (long long)r * stride;
  const uint8_t* far = p + (long long)rn * stride;
  if (hf == 1) return (3 * near[x] + far[x] + ((y & 1) ? 2 : 1)) >> 2;   // h1v2_fancy_upsample
  const int cx = x >> 1;                                     // h2v2_fancy_upsample
  if (dw <= 2) return near[cx];                              // h2v2_upsample: replication
  const int cs = 3 * near[cx] + far[cx];
  if ((x & 1) == 0) {
    const int ls = cx == 0 ? cs : 3 * near[cx - 1] + far[cx - 1];
    return (3 * cs + ls + 8) >> 4;
  }
  const int rs = cx == dw - 1 ? cs : 3 * near[cx + 1] + far[cx + 1];
  return (3 * cs + rs + 7) >> 4;
}

__global__ void __launch_bounds__(256)
color_kernel(const uint8_t* __restrict__ in, const se_jpeg_job* __restrict__ jobs, const uint8_t* __restrict__ ws,
             uint8_t* __restrict__ out) {
  __shared__ unsigned char srl[5 * 256 + 128];
  __shared__ Geo geo;
  build_range_limit(srl);
  const se_jpeg_job job = jobs[blockIdx.y];
  const se_jpeg_info* f = (const se_jpeg_info*)(in + job.info_offset);
  if (threadIdx.x == 0) geometry(*f, geo);
  __syncthreads();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)geo.W * geo.H) return;
  const int y = (int)(pix / geo.W), x = (int)(pix - (long long)y * geo.W);
  const Layout L = layout(geo, f->n_subseq);
  const uint8_t* samp = ws + job.ws_offset + L.samp;
  const unsigned char* limit = srl + 256;                    // sample_range_limit
  const int Y = samp[(long long)y * geo.bw[0] * 8 + x];
  uint8_t* o = out + job.out_offset + pix * 3;
  if (geo.nc == 1) {
    o[0] = o[1] = o[2] = (uint8_t)Y;
    return;
  }
  const int hf = geo.h[0], vf = geo.v[0];
  const int cb = upsample(samp + geo.boff[1] * 64, geo.bw[1] * 8, geo.dw[1], geo.dh[1], hf, vf, x, y) - 128;
  const int cr = upsample(samp + geo.boff[2] * 64, geo.bw[2] * 8, geo.dw[2], geo.dh[2], hf, vf, x, y) - 128;
  // jdcolor.c build_ycc_rgb_table: FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802,
  // FIX(0.34414) = 22554, ONE_HALF = 1 << 15
  const int cr_r = (91881 * cr + 32768) >> 16;
  const int cb_b = (116130 * cb + 32768) >> 16;
  const int g = (-46802 * cr + (-22554 * cb + 32768)) >> 16;
  o[0] = limit[Y + cr_r];
  o[1] = limit[Y + g];
  o[2] = limit[Y + cb_b];
}

}  // namespace

}  // namespace se

using namespace se;

extern "C" int64_t se_jpeg_workspace_bytes(const se_jpeg_info* info, se_jpeg_job* job, int B) {
  SE_REQUIRE(info && job && B > 0, "null pointer or empty batch");
  long long total = 0;
  for (int i = 0; i < B; ++i) {
    SE_REQUIRE(info[i].status == SE_JPEG_OK && info[i].n_subseq > 0 && info[i].n_intervals > 0,
               "image not supported by the device decoder");
    Geo g;
    geometry(info[i], g);
    job[i].ws_offset = total;
    total += layout(g, info[i].n_subseq).total;
  }
  return total;
}

extern "C" int se_jpeg_decode_batch(const unsigned char* in, const se_jpeg_info* info_host, const se_jpeg_job* job_host,
                                    const se_jpeg_job* job_dev, int B, unsigned char* out, int32_t* status,
                                    void* workspace, int64_t workspace_bytes, void* stream) {
  SE_REQUIRE(in && info_host && job_host && job_dev && out && status && workspace && B > 0, "null pointer or empty batch");
  long long total = 0, max_blocks = 0, max_pix = 0;
  for (int i = 0; i < B; ++i) {
    const se_jpeg_info& f = info_host[i];
    SE_REQUIRE(f.status == SE_JPEG_OK && f.n_subseq > 0 && f.n_intervals > 0, "image not supported by the device decoder");
    SE_REQUIRE(job_host[i].info_offset % 8 == 0 && job_host[i].packed_offset % 16 == 0 && job_host[i].out_offset >= 0,
               "misaligned job offsets");
    Geo g;
    geometry(f, g);
    SE_REQUIRE(job_host[i].ws_offset == total, "job ws_offset differs from se_jpeg_workspace_bytes");
    total += layout(g, f.n_subseq).total;
    max_blocks = std::max(max_blocks, g.nblocks);
    max_pix = std::max(max_pix, (long long)f.width * f.height);
  }
  SE_REQUIRE(workspace_bytes >= total, "workspace smaller than se_jpeg_workspace_bytes");
  cudaStream_t st = as_stream(stream);
  cudaMemsetAsync(workspace, 0, (size_t)total, st);          // coefficients a block does not code are zero
  uint8_t* ws = (uint8_t*)workspace;
  // Plain stream launches, not programmatic dependent ones (the library's default, common.cuh): entropy_kernel runs
  // long on one CTA per image, and an early-launched idct_kernel grid would park thousands of waiting CTAs on every SM
  // for that whole time, keeping the training kernels of other streams off the GPU.
  entropy_kernel<<<B, kEntropyThreads, 0, st>>>((const uint8_t*)in, job_dev, ws, status);
  int rc = check_launch("entropy_kernel");
  if (rc) return rc;
  idct_kernel<<<dim3((unsigned)ceil_div(max_blocks, (long long)kIdctBlocks), B), kIdctBlocks * 8, 0, st>>>(
      (const uint8_t*)in, job_dev, ws, status);
  rc = check_launch("idct_kernel");
  if (rc) return rc;
  color_kernel<<<dim3((unsigned)ceil_div(max_pix, 256LL), B), 256, 0, st>>>((const uint8_t*)in, job_dev,
                                                                             (const uint8_t*)ws, out);
  return check_launch("color_kernel");
}
