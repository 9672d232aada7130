// Batched input pipeline of the reference's file datasets on the device:
//   FileDatasetGenerator.compose_batch (datasets/common.py:380-432) over _load_image (:435-472) and _transform
//   (:475-542) for NABirds / CUB (datasets/nab.py, datasets/__init__.py:101-117) -- per image
//     PIL resize(BILINEAR) to the target shorter side (:460-470)  ->  float32, (x - mean) / std (:514-516)
//     ->  RGB -> BGR for '-caffe' (:519-520)  ->  horizontal flip (:523-524)  ->  random erasing (:530-540)
//     ->  crop (:414-425)  ->  np.stack (:432).
// JPEG / PNG decoding stays on host threads; the decoded uint8 RGB images of a batch arrive packed in one buffer and
// this file writes the float32 NHWC input tensor of the network in ONE launch.  Only the crop window of the resized
// image is ever resampled.
//
// Resampling restates Pillow's libImaging/Resample.c (ImagingResampleInner, precompute_coeffs, normalize_coeffs_8bpc,
// ImagingResampleHorizontal_8bpc / Vertical_8bpc) for the bilinear filter on 8-bit images:
//   scale = in / out, filterscale = max(scale, 1), support = filterscale (bilinear support 1)
//   output index i: center = (i + 0.5) * scale, window [int(center - support + 0.5), int(center + support + 0.5))
//   clipped to [0, in), weight of tap t = 1 - |(t - center + 0.5) / filterscale| (0 outside), weights divided by their
//   sum, then quantised to 22 fractional bits with rounding half away from zero;
//   a horizontal pass on uint8 rows, then a vertical pass on its uint8 result, each (2^21 + sum px * w) >> 22 clamped
//   to 0..255.
// The coefficients are computed in double with explicitly rounded operations (__dmul_rn / __dadd_rn / __ddiv_rn): a
// contracted multiply-add would move the last bit of a weight and, through the 22-bit quantisation, a pixel.  A pass
// whose scale is exactly 1 has weights (1, 0) and is the identity, as Pillow's skipped pass is.
//
// One CTA owns R consecutive output rows of one image.  The source rows their vertical windows span are visited in
// chunks of S rows: the CTA resamples a chunk horizontally into a shared-memory band (crop columns only), then every
// thread adds the chunk's vertical taps into its own int32 accumulators in shared memory.  Integer sums are exact, so the
// chunking does not change a bit.  HBM-bound: 12 bytes written per output pixel, each source byte read about once
// (neighbouring CTAs share up to 2 * support rows, mostly through L2).
#include <algorithm>
#include <math.h>

#include "common.cuh"

namespace se {

namespace {

constexpr int kThreads = 256;
constexpr int kRows = 8;                 // output rows per CTA
constexpr int kPrecision = 22;           // Resample.c PRECISION_BITS = 32 - 8 - 2
constexpr int kSmemBudget = 200 * 1024;  // dynamic shared memory per CTA at most (crops up to 1024 wide)

struct Window {
  int min, len;
};

// precompute_coeffs for one output index (bilinear filter, box = whole image) + normalize_coeffs_8bpc.
// Writes `len` quantised weights to k (when k != nullptr) and returns the clipped window.
__host__ __device__ inline int ksize_of(int in, int out) {
  const double scale = (double)in / (double)out;
  const double fs = scale < 1.0 ? 1.0 : scale;
  return (int)ceil(fs) * 2 + 1;
}

__device__ Window coeffs(int in, int out, int i, int* k) {
  const double scale = __ddiv_rn((double)in, (double)out);
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = fs;                                  // bilinear support 1.0 * filterscale
  const double center = __dmul_rn(__dadd_rn((double)i, 0.5), scale);
  const double ss = __ddiv_rn(1.0, fs);
  int xmin = (int)__dadd_rn(__dadd_rn(center, -support), 0.5);
  if (xmin < 0) xmin = 0;
  int xmax = (int)__dadd_rn(__dadd_rn(center, support), 0.5);
  if (xmax > in) xmax = in;
  const int len = xmax - xmin;
  double w[64];                                               // only used when len <= 64 (see se_resample_crop_batch)
  double ww = 0.0;
  for (int t = 0; t < len; ++t) {
    double a = __dmul_rn(__dadd_rn(__dadd_rn((double)(t + xmin), -center), 0.5), ss);
    a = fabs(a);
    const double v = a < 1.0 ? __dadd_rn(1.0, -a) : 0.0;
    if (len <= 64) w[t] = v;
    ww = __dadd_rn(ww, v);
  }
  if (k) {
    for (int t = 0; t < len; ++t) {
      double v = w[t];
      if (ww != 0.0) v = __ddiv_rn(v, ww);
      // normalize_coeffs_8bpc: (int)(0.5 + v * 2^22) for v >= 0 (bilinear weights are never negative)
      k[t] = (int)__dadd_rn(0.5, __dmul_rn(v, (double)(1 << kPrecision)));
    }
  }
  return Window{xmin, len};
}

// The erase noise documented in include/se_b200.h (SE_RESAMPLE_MAX_RESIZED keeps y and x below 2^20).
__device__ __forceinline__ double erase_noise(unsigned long long seed, int b, int y, int x, int c) {
  unsigned long long z = (((((unsigned long long)b << 20) | (unsigned)y) << 20 | (unsigned)x) << 2 | (unsigned)c) + 1ull;
  z = seed + z * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return __dmul_rn((double)(z >> 11) * 0x1.0p-53, 255.0);
}

__device__ __forceinline__ int clip8(int v) {
  v >>= kPrecision;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

__global__ void __launch_bounds__(kThreads)
resample_crop_kernel(const unsigned char* __restrict__ src, const se_resample_desc* __restrict__ descs, int ch, int cw,
                     int KH, int KV, int S, float m0, float m1, float m2, float s0, float s1, float s2, int bgr,
                     unsigned long long seed, float* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem[];
  int* acc = (int*)smem;                                      // [kRows][cw][3]
  int* kh = acc + kRows * cw * 3;                             // [cw][KH]
  int* kv = kh + cw * KH;                                     // [kRows][KV]
  int* xwin = kv + kRows * KV;                                // [cw][2]
  int* ywin = xwin + cw * 2;                                  // [kRows][2]
  unsigned char* band = (unsigned char*)(ywin + kRows * 2);   // [S][cw][3]

  pdl_grid_sync();
  const int b = blockIdx.y;
  const int oy0 = blockIdx.x * kRows;
  const int rows = min(kRows, ch - oy0);
  const se_resample_desc d = descs[b];
  const unsigned char* img = src + d.src_offset;

  for (int ox = threadIdx.x; ox < cw; ox += kThreads) {
    const int rx = d.flip ? d.rw - 1 - d.cx - ox : d.cx + ox;  // the crop is taken from the flipped image
    const Window w = coeffs(d.src_w, d.rw, rx, kh + ox * KH);
    xwin[2 * ox] = w.min;
    xwin[2 * ox + 1] = w.len;
  }
  for (int r = threadIdx.x; r < rows; r += kThreads) {
    const Window w = coeffs(d.src_h, d.rh, d.cy + oy0 + r, kv + r * KV);
    ywin[2 * r] = w.min;
    ywin[2 * r + 1] = w.len;
  }
  const int half = 1 << (kPrecision - 1);
  for (int i = threadIdx.x; i < rows * cw * 3; i += kThreads) acc[i] = half;
  __syncthreads();

  const int y_lo = ywin[0];
  const int y_hi = ywin[2 * (rows - 1)] + ywin[2 * (rows - 1) + 1];  // windows move monotonically with the row
  for (int c0 = y_lo; c0 < y_hi; c0 += S) {
    const int n = min(S, y_hi - c0);
    // horizontal pass of source rows [c0, c0 + n), crop columns only
    for (int i = threadIdx.x; i < n * cw; i += kThreads) {
      const int yy = i / cw, ox = i - yy * cw;
      const int xmin = xwin[2 * ox], len = xwin[2 * ox + 1];
      const int* k = kh + ox * KH;
      const unsigned char* p = img + ((long long)(c0 + yy) * d.src_w + xmin) * 3;
      int a0 = half, a1 = half, a2 = half;
      for (int t = 0; t < len; ++t) {
        const int w = k[t];
        a0 += (int)p[3 * t] * w;
        a1 += (int)p[3 * t + 1] * w;
        a2 += (int)p[3 * t + 2] * w;
      }
      unsigned char* q = band + (long long)i * 3;
      q[0] = (unsigned char)clip8(a0);
      q[1] = (unsigned char)clip8(a1);
      q[2] = (unsigned char)clip8(a2);
    }
    __syncthreads();
    // vertical taps of this chunk into each output pixel's accumulators
    for (int i = threadIdx.x; i < rows * cw; i += kThreads) {
      const int r = i / cw, ox = i - r * cw;
      const int ymin = ywin[2 * r], ylen = ywin[2 * r + 1];
      const int t0 = max(ymin, c0), t1 = min(ymin + ylen, c0 + n);
      if (t0 >= t1) continue;
      const int* k = kv + r * KV - ymin;
      int a0 = 0, a1 = 0, a2 = 0;
      for (int y = t0; y < t1; ++y) {
        const unsigned char* q = band + ((long long)(y - c0) * cw + ox) * 3;
        const int w = k[y];
        a0 += (int)q[0] * w;
        a1 += (int)q[1] * w;
        a2 += (int)q[2] * w;
      }
      acc[3 * i] += a0;
      acc[3 * i + 1] += a1;
      acc[3 * i + 2] += a2;
    }
    __syncthreads();
  }

  // standardise, BGR, erase, store (the erase rectangle is in the coordinates of the flipped resized image)
  const float mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
  for (int i = threadIdx.x; i < rows * cw; i += kThreads) {
    const int r = i / cw, ox = i - r * cw;
    const int oy = oy0 + r;
    const int Y = d.cy + oy, X = d.cx + ox;
    const bool erased = d.eh > 0 && Y >= d.ey && Y < d.ey + d.eh && X >= d.ex && X < d.ex + d.ew;
    float* o = out + (((long long)b * ch + oy) * cw + ox) * 3;
    for (int c = 0; c < 3; ++c) {
      float v;
      if (erased) {
        // (U(0, 255) - mean) / std in float64, stored as float32; mean / std in RGB order even after the BGR swap
        const double u = erase_noise(seed, d.noise_id, Y, X, c);
        v = (float)__ddiv_rn(__dadd_rn(u, -(double)mean[c]), (double)stdv[c]);
      } else {
        const int sc = bgr ? 2 - c : c;
        const float x = (float)clip8(acc[3 * i + sc]);
        v = __fdiv_rn(__fsub_rn(x, mean[sc]), stdv[sc]);
      }
      o[c] = v;
    }
  }
}

}  // namespace

// plan() asks for at most kSmemBudget bytes
int init_resample_crop() {
  if (cudaFuncSetAttribute(resample_crop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBudget) != cudaSuccess) {
    set_error("init_resample_crop: cannot raise the shared-memory limit");
    return SE_ERR_CUDA;
  }
  return SE_OK;
}

}  // namespace se

using namespace se;

// Launch plan of a batch: validates the descriptors and returns the dynamic shared memory of a CTA (or SE_ERR_ARG); KH / KV
// are the largest tap counts, S the source rows of a band chunk (enough for a CTA's whole span when it fits).
static int plan(const se_resample_desc* desc, int B, int ch, int cw, int* KH, int* KV, int* S) {
  SE_REQUIRE(desc && B > 0 && ch > 0 && cw > 0 && ch <= SE_RESAMPLE_MAX_CROP && cw <= SE_RESAMPLE_MAX_CROP,
             "bad batch or crop size");
  int kh = 1, kv = 1;
  double fs = 1.0;
  for (int i = 0; i < B; ++i) {
    const se_resample_desc& d = desc[i];
    SE_REQUIRE(d.src_h > 0 && d.src_w > 0 && d.src_h <= SE_RESAMPLE_MAX_SIDE && d.src_w <= SE_RESAMPLE_MAX_SIDE,
               "source side outside [1, SE_RESAMPLE_MAX_SIDE]");
    SE_REQUIRE(d.rh >= ch && d.rw >= cw && d.rh <= SE_RESAMPLE_MAX_RESIZED && d.rw <= SE_RESAMPLE_MAX_RESIZED,
               "resized image smaller than the crop (reflect padding is not implemented) or larger than "
               "SE_RESAMPLE_MAX_RESIZED");
    SE_REQUIRE(d.cy >= 0 && d.cx >= 0 && d.cy + ch <= d.rh && d.cx + cw <= d.rw, "crop outside the resized image");
    SE_REQUIRE(d.flip == 0 || d.flip == 1, "flip must be 0 or 1");
    SE_REQUIRE(d.eh == 0 || (d.eh > 0 && d.ew > 0 && d.ey >= 0 && d.ex >= 0 && d.ey + d.eh <= d.rh && d.ex + d.ew <= d.rw),
               "erase rectangle outside the resized image");
    SE_REQUIRE(d.src_offset >= 0, "negative source offset");
    SE_REQUIRE(d.noise_id >= 0 && d.noise_id < (1 << 20), "noise_id outside [0, 2^20)");
    kh = std::max(kh, ksize_of(d.src_w, d.rw));
    kv = std::max(kv, ksize_of(d.src_h, d.rh));
    fs = std::max(fs, (double)d.src_h / d.rh);
  }
  // the per-thread weight scratch of coeffs() holds 64 taps
  SE_REQUIRE(kh <= 64 && kv <= 64, "downscale factor above 31 (source side / resized side)");
  const long long fixed = 4LL * (kRows * cw * 3 + cw * kh + kRows * kv + cw * 2 + kRows * 2);
  const long long row = 3LL * cw;
  SE_REQUIRE(fixed + row <= kSmemBudget, "crop too wide for the shared-memory band");
  const long long span = (long long)ceil((kRows + 1) * fs) + 2 * (long long)ceil(fs) + 2;   // source rows of a CTA
  const long long s = std::min(span, (kSmemBudget - fixed) / row);
  *KH = kh;
  *KV = kv;
  *S = (int)s;
  return (int)(fixed + s * row);
}

extern "C" int se_resample_crop_batch(const unsigned char* src, const se_resample_desc* desc_host,
                                      const se_resample_desc* desc_dev, int B, int crop_h, int crop_w, const float* mean,
                                      const float* std, int bgr, uint64_t seed, float* out, void* stream) {
  SE_REQUIRE(src && desc_host && desc_dev && mean && std && out, "null pointer");
  SE_REQUIRE(bgr == 0 || bgr == 1, "bgr must be 0 or 1");
  int KH, KV, S;
  const int smem = plan(desc_host, B, crop_h, crop_w, &KH, &KV, &S);
  if (smem < 0) return smem;
  const int rc = ensure_setup();
  if (rc) return rc;
  const dim3 grid((crop_h + kRows - 1) / kRows, B);
  launch(resample_crop_kernel, grid, dim3(kThreads), (size_t)smem, as_stream(stream), src, desc_dev, crop_h, crop_w, KH, KV,
         S, mean[0], mean[1], mean[2], std[0], std[1], std[2], bgr, (unsigned long long)seed, out);
  return check_launch("resample_crop_kernel");
}
