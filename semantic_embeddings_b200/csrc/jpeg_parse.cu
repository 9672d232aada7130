// JPEG header parser and scan packer of the device decoder (host code; see include/se_b200.h and jpeg_decode.cu).
//
// se_jpeg_parse walks the markers of one file the way libjpeg reads a baseline / extended-sequential Huffman file and
// decides whether jpeg_decode.cu reproduces libjpeg-turbo's output for it.  Every read is checked against the file size.
// Anything libjpeg would reject, warn about or decode through another path is reported as unsupported, with a reason:
// such files go to the host decoder (Pillow), so the device decoder only ever sees streams whose decode is determined
// by the tables and the entropy-coded data alone.
//
// se_jpeg_pack copies the entropy-coded segment without its byte stuffing (0xFF 0x00 -> 0xFF, fill bytes 0xFF before a
// stuffed zero dropped, as libjpeg's bit reader does) and without its RSTn markers, and records where each restart
// interval starts: each interval starts on a byte boundary with zero DC predictions, so it is decoded independently.
#include <stddef.h>
#include <string.h>

#include "common.cuh"

namespace {

// zig-zag position -> natural (row-major) position
const int kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                          41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                          30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

inline int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// Expands the counts / symbols of a DHT table into lookup form (the canonical code assignment of JPEG Annex C).
// Returns false for a table libjpeg's jpeg_make_d_derived_tbl rejects: more than 256 symbols, an all-ones code (or
// codes that overflow their length), or a DC symbol above 15.  Since no code is all ones, the 1-bits that pad the end
// of an interval never complete a code.
bool build_huff(const uint8_t* counts, const uint8_t* vals, int nsym, bool dc, se_jpeg_huff* t) {
  memset(t, 0, sizeof(*t));
  if (nsym > 256) return false;
  memcpy(t->huffval, vals, nsym);
  if (dc)
    for (int i = 0; i < nsym; ++i)
      if (vals[i] > 15) return false;
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    const int n = counts[l - 1];
    if (n == 0) {
      t->maxcode[l] = -1;
    } else {
      t->valoffset[l] = k - code;
      for (int i = 0; i < n; ++i, ++code, ++k) {
        if (l <= 9) {
          const int lo = code << (9 - l), hi = (code + 1) << (9 - l);
          for (int e = lo; e < hi; ++e) t->lookup[e] = (uint16_t)((l << 8) | vals[k]);
        }
      }
      t->maxcode[l] = code - 1;
    }
    if (code >= (1 << l)) return false;  // no code may be all ones (or overflow its length)
    code <<= 1;
  }
  t->maxcode[0] = -1;
  t->maxcode[17] = 0x7fffffff;
  return true;
}

inline int64_t align16(int64_t v) { return (v + 15) & ~(int64_t)15; }

// Blocks of one restart interval and the interval count (interleaved scan: MCUs; one component: its blocks)
inline int64_t total_mcus(const se_jpeg_info& f) { return (int64_t)f.mcus_x * f.mcus_y; }

int parse(const uint8_t* d, int64_t n, se_jpeg_info* f) {
  if (n < 2 || d[0] != 0xFF || d[1] != 0xD8) return SE_JPEG_NOT_JPEG;
  int64_t p = 2;
  bool have_sof = false, have_dc[4] = {}, have_ac[4] = {};
  f->restart_interval = 0;
  for (;;) {
    // a marker: 0xFF, fill bytes 0xFF, the code
    if (p >= n) return SE_JPEG_TRUNCATED;
    if (d[p] != 0xFF) return SE_JPEG_MALFORMED;        // libjpeg skips such garbage with a warning
    while (p < n && d[p] == 0xFF) ++p;
    if (p >= n) return SE_JPEG_TRUNCATED;
    const int m = d[p++];
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01 || m == 0x00) return SE_JPEG_MALFORMED;
    if (p + 2 > n) return SE_JPEG_TRUNCATED;
    const int len = be16(d + p);
    if (len < 2) return SE_JPEG_MALFORMED;
    if (p + len > n) return SE_JPEG_TRUNCATED;
    const uint8_t* s = d + p + 2;
    const int sl = len - 2;
    const int64_t next = p + len;
    if (m == 0xE0) {                                    // APP0: JFIF (jdmarker.c examine_app0: 14 bytes or more)
      if (sl >= 14 && s[0] == 'J' && s[1] == 'F' && s[2] == 'I' && s[3] == 'F' && s[4] == 0) f->saw_jfif = 1;
    } else if (m == 0xEE) {                             // APP14: Adobe (examine_app14: 12 bytes or more)
      if (sl >= 12 && s[0] == 'A' && s[1] == 'd' && s[2] == 'o' && s[3] == 'b' && s[4] == 'e') {
        f->saw_adobe = 1;
        f->adobe_transform = s[11];
      }
    } else if ((m >= 0xE1 && m <= 0xEF) || m == 0xFE) {  // other APPn, COM
    } else if (m == 0xDB) {                             // DQT
      int q = 0;
      while (q < sl) {
        const int pq = s[q] >> 4, tq = s[q] & 15;
        if (pq > 1 || tq > 3) return SE_JPEG_MALFORMED;
        const int sz = pq ? 128 : 64;
        if (q + 1 + sz > sl) return SE_JPEG_MALFORMED;
        for (int i = 0; i < 64; ++i) {
          const int val = pq ? be16(s + q + 1 + 2 * i) : s[q + 1 + i];
          // libjpeg-turbo keeps quantisation values in 16-bit signed multiplies: above 32767 (which its own writer
          // never emits) its SIMD and C paths dequantise differently
          if (val > 32767) return SE_JPEG_MALFORMED;
          f->qt[tq][kNatural[i]] = (uint16_t)val;
        }
        f->qt_mask |= 1 << tq;
        q += 1 + sz;
      }
    } else if (m == 0xC4) {                             // DHT
      int q = 0;
      while (q < sl) {
        if (q + 17 > sl) return SE_JPEG_MALFORMED;
        const int tc = s[q] >> 4, th = s[q] & 15;
        if (tc > 1 || th > 3) return SE_JPEG_MALFORMED;
        int nsym = 0;
        for (int i = 0; i < 16; ++i) nsym += s[q + 1 + i];
        if (nsym > 256 || q + 17 + nsym > sl) return SE_JPEG_MALFORMED;
        if (!build_huff(s + q + 1, s + q + 17, nsym, tc == 0, tc ? &f->ac[th] : &f->dc[th])) return SE_JPEG_MALFORMED;
        (tc ? have_ac : have_dc)[th] = true;
        q += 17 + nsym;
      }
    } else if (m == 0xDD) {                             // DRI
      if (sl != 2) return SE_JPEG_MALFORMED;
      f->restart_interval = be16(s);
    } else if (m == 0xC0 || m == 0xC1) {                // SOF0 / SOF1
      if (have_sof) return SE_JPEG_MALFORMED;
      have_sof = true;
      if (sl < 6) return SE_JPEG_MALFORMED;
      if (s[0] != 8) return SE_JPEG_PRECISION;
      f->height = be16(s + 1);
      f->width = be16(s + 3);
      const int nc = s[5];
      if (nc <= 0 || sl != 6 + 3 * nc) return SE_JPEG_MALFORMED;
      if (nc != 1 && nc != 3) return SE_JPEG_COMPONENTS;
      f->ncomp = nc;
      for (int c = 0; c < nc; ++c) {
        f->comp_id[c] = s[6 + 3 * c];
        f->h[c] = s[7 + 3 * c] >> 4;
        f->v[c] = s[7 + 3 * c] & 15;
        f->tq[c] = s[8 + 3 * c];
        if (f->h[c] < 1 || f->h[c] > 4 || f->v[c] < 1 || f->v[c] > 4 || f->tq[c] > 3) return SE_JPEG_MALFORMED;
      }
    } else if (m == 0xC2 || m == 0xC6) {
      return SE_JPEG_PROGRESSIVE;
    } else if (m == 0xC3 || m == 0xC5 || m == 0xC7) {
      return SE_JPEG_OTHER_PROCESS;
    } else if ((m >= 0xC9 && m <= 0xCB) || (m >= 0xCD && m <= 0xCF) || m == 0xCC) {
      return SE_JPEG_ARITHMETIC;
    } else if (m == 0xDC) {
      return SE_JPEG_SIZE;                              // DNL: the height is given after the scan
    } else if (m == 0xDA) {                             // SOS
      if (!have_sof) return SE_JPEG_MALFORMED;
      if (sl < 1) return SE_JPEG_MALFORMED;
      const int ns = s[0];
      if (sl != 4 + 2 * ns || ns < 1) return SE_JPEG_MALFORMED;
      if (ns != f->ncomp) return SE_JPEG_MULTISCAN;
      for (int c = 0; c < ns; ++c) {
        if (s[1 + 2 * c] != f->comp_id[c]) return SE_JPEG_MULTISCAN;   // components in frame order
        f->td[c] = s[2 + 2 * c] >> 4;
        f->ta[c] = s[2 + 2 * c] & 15;
        if (f->td[c] > 3 || f->ta[c] > 3 || !have_dc[f->td[c]] || !have_ac[f->ta[c]]) return SE_JPEG_MALFORMED;
        if (!(f->qt_mask >> f->tq[c] & 1)) return SE_JPEG_MALFORMED;
      }
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return SE_JPEG_MALFORMED;
      p = next;
      break;
    } else {
      return SE_JPEG_MALFORMED;                         // DHP, EXP, JPGn, reserved
    }
    p = next;
  }

  // colour space (jdapimin.c default_decompress_parms) and sampling
  if (f->ncomp == 3) {
    bool ycc;
    if (f->saw_jfif) ycc = true;
    else if (f->saw_adobe) ycc = f->adobe_transform == 1;   // 0: RGB; other values: libjpeg warns
    else ycc = !(f->comp_id[0] == 'R' && f->comp_id[1] == 'G' && f->comp_id[2] == 'B');
    if (!ycc) return SE_JPEG_COLORSPACE;
    for (int c = 1; c < 3; ++c)
      if (f->h[c] != 1 || f->v[c] != 1) return SE_JPEG_SAMPLING;
    if (f->h[0] > 2 || f->v[0] > 2) return SE_JPEG_SAMPLING;
  }
  if (f->width <= 0 || f->height <= 0 || f->width > SE_RESAMPLE_MAX_SIDE || f->height > SE_RESAMPLE_MAX_SIDE)
    return SE_JPEG_SIZE;
  f->hmax = f->vmax = 1;
  for (int c = 0; c < f->ncomp; ++c) {
    f->hmax = f->h[c] > f->hmax ? f->h[c] : f->hmax;
    f->vmax = f->v[c] > f->vmax ? f->v[c] : f->vmax;
  }
  if (f->ncomp == 1) {                                  // non-interleaved: one block per MCU over the component
    f->mcus_x = (f->width + 7) / 8;
    f->mcus_y = (f->height + 7) / 8;
  } else {
    f->mcus_x = (f->width + 8 * f->hmax - 1) / (8 * f->hmax);
    f->mcus_y = (f->height + 8 * f->vmax - 1) / (8 * f->vmax);
  }
  const int64_t mcus = total_mcus(*f);
  const int64_t nint = f->restart_interval ? (mcus + f->restart_interval - 1) / f->restart_interval : 1;

  // the entropy-coded segment: stuffed bytes, RSTn in sequence, then a marker that ends it
  f->scan_begin = p;
  int64_t seen = 0, len = 0, data = 0, nsub = 0;
  for (;;) {
    const uint8_t* q = (const uint8_t*)memchr(d + p, 0xFF, (size_t)(n - p));
    if (!q) return SE_JPEG_TRUNCATED;
    const int64_t at = q - d;
    len += at - p;
    int64_t r = at + 1;
    while (r < n && d[r] == 0xFF) ++r;
    if (r >= n) return SE_JPEG_TRUNCATED;
    const int m = d[r];
    if (m == 0x00) {
      len += 1;
      p = r + 1;
      continue;
    }
    if (m >= 0xD0 && m <= 0xD7) {
      if (f->restart_interval == 0 || m != 0xD0 + (seen & 7) || seen + 1 >= nint) return SE_JPEG_RESTART;
      ++seen;
      data += len;
      nsub += len > 0 ? (len + SE_JPEG_SUBSEQ_BYTES - 1) / SE_JPEG_SUBSEQ_BYTES : 1;
      len = 0;
      p = r + 1;
      continue;
    }
    f->scan_end = at;
    p = r + 1;
    // what follows the scan: tables, APPn / COM, then EOI; another SOS is a second scan
    int mk = m;
    for (;;) {
      if (mk == 0xD9) break;
      if (mk == 0xDA) return SE_JPEG_MULTISCAN;
      if (mk == 0xDC) return SE_JPEG_SIZE;
      if (!((mk >= 0xE0 && mk <= 0xEF) || mk == 0xFE || mk == 0xDB || mk == 0xC4 || mk == 0xDD)) return SE_JPEG_MALFORMED;
      if (p + 2 > n) return SE_JPEG_TRUNCATED;
      const int l2 = be16(d + p);
      if (l2 < 2) return SE_JPEG_MALFORMED;
      if (p + l2 > n) return SE_JPEG_TRUNCATED;
      p += l2;
      if (p >= n) return SE_JPEG_TRUNCATED;
      if (d[p] != 0xFF) return SE_JPEG_MALFORMED;
      while (p < n && d[p] == 0xFF) ++p;
      if (p >= n) return SE_JPEG_TRUNCATED;
      mk = d[p++];
    }
    break;
  }
  if (seen + 1 != nint) return SE_JPEG_RESTART;
  data += len;
  nsub += len > 0 ? (len + SE_JPEG_SUBSEQ_BYTES - 1) / SE_JPEG_SUBSEQ_BYTES : 1;
  if (data >= (1LL << 28) || nsub >= (1LL << 30)) return SE_JPEG_SIZE;   // bit positions stay below 2^31
  f->n_intervals = (int32_t)nint;
  f->n_subseq = (int32_t)nsub;
  f->data_bytes = data;
  f->packed_bytes = align16(8 * (nint + 1)) + align16(data) + 16;
  return SE_JPEG_OK;
}

}  // namespace

extern "C" int se_jpeg_parse(const uint8_t* data, int64_t n, se_jpeg_info* out) {
  SE_REQUIRE(data && out && n >= 0, "null pointer or negative size");
  memset(out, 0, sizeof(*out));
  out->status = parse(data, n, out);
  return out->status;
}

extern "C" int64_t se_jpeg_pack(const uint8_t* data, int64_t n, const se_jpeg_info* f, uint8_t* out, int64_t cap) {
  SE_REQUIRE(data && f && out, "null pointer");
  SE_REQUIRE(f->status == SE_JPEG_OK, "file not supported by the device decoder");
  SE_REQUIRE(cap >= f->packed_bytes && f->scan_end <= n && f->scan_begin <= f->scan_end, "output too small or bad info");
  const int64_t nint = f->n_intervals;
  uint32_t* int_start = (uint32_t*)out;
  uint32_t* sub_first = int_start + nint + 1;
  uint8_t* dst = out + align16(8 * (nint + 1));
  memset(out, 0, (size_t)f->packed_bytes);
  int64_t w = 0, i = 0, nsub = 0, p = f->scan_begin;
  int_start[0] = 0;
  sub_first[0] = 0;
  auto close = [&]() {
    const int64_t len = w - int_start[i];
    nsub += len > 0 ? (len + SE_JPEG_SUBSEQ_BYTES - 1) / SE_JPEG_SUBSEQ_BYTES : 1;
    ++i;
    int_start[i] = (uint32_t)w;
    sub_first[i] = (uint32_t)nsub;
  };
  const int64_t end = f->scan_end;
  while (p < end) {
    const uint8_t* q = (const uint8_t*)memchr(data + p, 0xFF, (size_t)(end - p));
    const int64_t at = q ? q - data : end;
    SE_REQUIRE(w + (at - p) <= f->data_bytes, "scan differs from the parsed one");
    memcpy(dst + w, data + p, (size_t)(at - p));
    w += at - p;
    if (!q) break;
    int64_t r = at + 1;
    while (r < end && data[r] == 0xFF) ++r;
    SE_REQUIRE(r < end, "scan differs from the parsed one");
    if (data[r] == 0x00) {
      SE_REQUIRE(w < f->data_bytes, "scan differs from the parsed one");
      dst[w++] = 0xFF;
    } else {
      SE_REQUIRE(i + 1 < nint, "scan differs from the parsed one");
      close();
    }
    p = r + 1;
  }
  close();
  SE_REQUIRE(i == nint && w == f->data_bytes && nsub == f->n_subseq, "scan differs from the parsed one");
  return f->packed_bytes;
}

extern "C" int se_jpeg_layout(int64_t* out, int cap) {
#define SE_F(T, f) (int64_t) offsetof(T, f)
  const int64_t v[] = {
      (int64_t)sizeof(se_jpeg_info), (int64_t)sizeof(se_jpeg_huff), (int64_t)sizeof(se_jpeg_job),
      SE_F(se_jpeg_info, status), SE_F(se_jpeg_info, width), SE_F(se_jpeg_info, height), SE_F(se_jpeg_info, ncomp),
      SE_F(se_jpeg_info, comp_id), SE_F(se_jpeg_info, h), SE_F(se_jpeg_info, v), SE_F(se_jpeg_info, tq),
      SE_F(se_jpeg_info, td), SE_F(se_jpeg_info, ta), SE_F(se_jpeg_info, hmax), SE_F(se_jpeg_info, vmax),
      SE_F(se_jpeg_info, mcus_x), SE_F(se_jpeg_info, mcus_y), SE_F(se_jpeg_info, restart_interval),
      SE_F(se_jpeg_info, n_intervals), SE_F(se_jpeg_info, n_subseq), SE_F(se_jpeg_info, saw_jfif),
      SE_F(se_jpeg_info, saw_adobe), SE_F(se_jpeg_info, adobe_transform), SE_F(se_jpeg_info, qt_mask),
      SE_F(se_jpeg_info, reserved), SE_F(se_jpeg_info, scan_begin), SE_F(se_jpeg_info, scan_end),
      SE_F(se_jpeg_info, data_bytes), SE_F(se_jpeg_info, packed_bytes), SE_F(se_jpeg_info, qt), SE_F(se_jpeg_info, dc),
      SE_F(se_jpeg_info, ac),
      SE_F(se_jpeg_huff, lookup), SE_F(se_jpeg_huff, maxcode), SE_F(se_jpeg_huff, valoffset), SE_F(se_jpeg_huff, huffval),
      SE_F(se_jpeg_job, info_offset), SE_F(se_jpeg_job, packed_offset), SE_F(se_jpeg_job, out_offset),
      SE_F(se_jpeg_job, ws_offset)};
#undef SE_F
  const int cnt = (int)(sizeof(v) / sizeof(v[0]));
  if (!out) return cnt;
  const int k = cap < cnt ? cap : cnt;
  for (int i = 0; i < k; ++i) out[i] = v[i];
  return k;
}
