// jpeg.cu — baseline JPEG decoding on the device, bit-exact with libjpeg-turbo as Pillow calls it (JDCT_ISLOW, fancy
// upsampling, no draft mode), for the files that decoder takes; every other file gets a fallback reason and stays on the
// host (include/vdk_b200.h lists the set; oracle/jpeg.py restates the arithmetic and is pinned against Pillow).
//
// Host: vdk_jpeg_parse walks the markers of each file, builds the Huffman tables in the form the entropy kernel reads (a 9-bit
// lookahead table plus libjpeg's maxcode / valoffset for longer codes), and walks the scan once: it checks the restart
// markers' sequence and count, records where each restart interval starts, and finds the scan's end.  Device, three
// launches per batch (after one memset of the coefficient stores and the status words):
//   1. jpeg_entropy_kernel: one thread per restart interval (the whole scan without DRI) Huffman-decodes its MCUs into
//      int16 coefficients (natural order, zero-initialised store).  The bit buffer is refilled a byte at a time: FF 00 is
//      un-stuffed, a marker or the interval's end feeds zeros, and reading into those zeros flags the image.
//   2. jpeg_idct_kernel: 8 threads per 8x8 block (columns, then rows through shared memory): dequantise and jidctint.c's
//      islow IDCT in 64-bit arithmetic, range-limited through the masked IDCT table, into uint8 component planes.
//   3. jpeg_color_kernel: one thread per output pixel: jdsample.c's fancy upsampling of the chroma sample it needs, then
//      jdcolor.c's fixed-point YCbCr->RGB, written as packed RGB cropped to the image size.
// Progressive files (vdk_jpeg_parse_progressive, vdk_jpeg_decode_ex) share the coefficient store, IDCT and colour kernels:
// between 1 and 2, jpeg_progressive_kernel runs once per dependency level of their scans (oracle/jpeg_progressive.py).
#include "vdk_host.h"

#include <algorithm>
#include <climits>
#include <cstring>
#include <vector>

namespace vdk {
namespace {

constexpr int kIdctBlocksPerCta = 32;   // 8 threads per block, 256 threads
constexpr int kColorPixelsPerCta = 1024;  // 256 threads x 4 pixels
constexpr int kEntropyThreads = 32;

__constant__ uint8_t kNatural[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
    62, 63};
const uint8_t kNaturalHost[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
    62, 63};

inline size_t up256(size_t x) { return (x + 255) & ~size_t(255); }
__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------------------------------------------------------- host parse
struct RawHuff {
  bool present = false;
  uint8_t counts[16];
  uint8_t vals[256];
};

// jdhuff.c jpeg_make_d_derived_tbl in the kernel's form; false for a table libjpeg refuses
bool build_huff(const RawHuff& r, bool is_dc, vdk_jpeg_huff* t) {
  memset(t, 0, sizeof(*t));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    const int cnt = r.counts[l - 1];
    if (cnt) {
      t->valoffset[l] = k - code;
      for (int j = 0; j < cnt; ++j, ++code, ++k) {
        if (l <= 9)
          for (int e = 0; e < (1 << (9 - l)); ++e) t->lut[(code << (9 - l)) | e] = static_cast<uint16_t>((l << 8) | r.vals[k]);
      }
      t->maxcode[l] = code - 1;
    } else {
      t->maxcode[l] = -1;
    }
    if (code >= (1 << l)) return false;  // no code may be all ones (JERR_BAD_HUFF_TABLE)
    code <<= 1;
  }
  t->maxcode[17] = 0x7fffffff;
  for (int i = 0; i < k; ++i) {
    t->huffval[i] = r.vals[i];
    if (is_dc && r.vals[i] > 15) return false;
  }
  return true;
}

// Pillow's own header reader (JpegImagePlugin.APP and SOF's ICC fix-up) raises on a few short application segments before
// libjpeg runs: a "JFIF" APP0 or "Adobe" APP14 without the 16-bit field at offset 5, an "ICC_PROFILE" APP2 without its
// fragment count at offset 13, and a "Photoshop 3.0" APP13 whose 8BIM resource ends right after its code.  Those files go
// to the host, which raises what Image.open raises.
bool pillow_reads_app(int m, const uint8_t* s, int sl) {
  auto starts = [&](const char* tag, int len) { return sl >= len && memcmp(s, tag, len) == 0; };
  if ((m == 0xE0 && starts("JFIF", 4)) || (m == 0xEE && starts("Adobe", 5))) return sl >= 7;
  if (m == 0xE2 && starts("ICC_PROFILE\0", 12)) return sl >= 14;
  if (m == 0xED && starts("Photoshop 3.0\0", 14)) {
    int64_t off = 14;
    while (off + 4 <= sl && memcmp(s + off, "8BIM", 4) == 0) {
      off += 4;
      if (off + 2 > sl) return true;  // struct.error: Pillow stops reading the block
      off += 2;
      if (off >= sl) return false;    // IndexError: Image.open fails
      off += 1 + s[off];
      off += off & 1;
      if (off + 4 > sl) return true;
      const int64_t size = (int64_t(s[off]) << 24) | (s[off + 1] << 16) | (s[off + 2] << 8) | s[off + 3];
      off += 4 + size;
      off += off & 1;
    }
  }
  return true;
}

// one SOFn segment: 0, or the fallback reason
int read_sof(const uint8_t* s, int sl, int* nf, int* width, int* height, int* cid, int* ch, int* cv, int* ctq) {
  if (sl < 6) return VDK_JPEG_MALFORMED;
  *nf = s[5];
  if (sl != 6 + 3 * *nf) return VDK_JPEG_MALFORMED;
  if (s[0] != 8) return VDK_JPEG_PRECISION;
  *height = (s[1] << 8) | s[2];
  *width = (s[3] << 8) | s[4];
  if (*width == 0 || *height == 0) return VDK_JPEG_MALFORMED;
  if (*width > 65500 || *height > 65500) return VDK_JPEG_TOO_LARGE;  // libjpeg's JPEG_MAX_DIMENSION
  if (*nf != 1 && *nf != 3) return VDK_JPEG_COLOR;
  for (int i = 0; i < *nf; ++i) {
    cid[i] = s[6 + 3 * i];
    ch[i] = s[7 + 3 * i] >> 4;
    cv[i] = s[7 + 3 * i] & 15;
    ctq[i] = s[8 + 3 * i];
    if (ch[i] < 1 || ch[i] > 4 || cv[i] < 1 || cv[i] > 4 || ctq[i] > 3) return VDK_JPEG_MALFORMED;
  }
  return 0;
}

// one DHT segment into the raw tables; false for a malformed segment
bool read_dht(const uint8_t* s, int sl, RawHuff (*huff)[4]) {
  for (int i = 0; i < sl;) {
    if (i + 17 > sl) return false;
    const int tc = s[i] >> 4, th = s[i] & 15;
    int total = 0;
    for (int l = 0; l < 16; ++l) total += s[i + 1 + l];
    if (tc > 1 || th > 3 || total > 256 || i + 17 + total > sl) return false;
    RawHuff& h = huff[tc][th];
    h.present = true;
    memcpy(h.counts, s + i + 1, 16);
    memcpy(h.vals, s + i + 17, total);
    i += 17 + total;
  }
  return true;
}

// one DQT segment into natural-order tables; false for a malformed segment
bool read_dqt(const uint8_t* s, int sl, int16_t (*qt)[64], bool* have_q) {
  for (int i = 0; i < sl;) {
    const int pq = s[i] >> 4, tq = s[i] & 15, size = pq ? 128 : 64;
    if (pq > 1 || tq > 3 || i + 1 + size > sl) return false;
    for (int k = 0; k < 64; ++k) {
      const int v = pq ? (s[i + 1 + 2 * k] << 8) | s[i + 2 + 2 * k] : s[i + 1 + k];
      qt[tq][kNaturalHost[k]] = static_cast<int16_t>(static_cast<uint16_t>(v));
    }
    have_q[tq] = true;
    i += 1 + size;
  }
  return true;
}

// libjpeg's colour-space guess (jdapimin.c default_decompress_parms) and the samplings decoded here: 0 when the frame
// decodes as greyscale or YCbCr with 1x1 chroma and luma 1 or 2 either way
int colour_reason(int nf, const int* cid, const int* ch, const int* cv, bool jfif, bool adobe, int adobe_transform) {
  if (nf != 3) return 0;
  if (!jfif && adobe && adobe_transform != 1) return VDK_JPEG_COLOR;
  if (!jfif && !adobe && cid[0] == 'R' && cid[1] == 'G' && cid[2] == 'B') return VDK_JPEG_COLOR;
  const bool chroma11 = ch[1] == 1 && cv[1] == 1 && ch[2] == 1 && cv[2] == 1;
  const bool luma_ok = (ch[0] == 1 || ch[0] == 2) && (cv[0] == 1 || cv[0] == 2);
  return chroma11 && luma_ok ? 0 : VDK_JPEG_SAMPLING;
}

// the frame fields of a descriptor (sampling 1 x 1 for a single component), shared by both parsers
void fill_frame(vdk_jpeg_desc* out, int width, int height, int nf, const int* ch, const int* cv) {
  const int hmax = nf == 3 ? std::max(ch[0], 1) : 1, vmax = nf == 3 ? std::max(cv[0], 1) : 1;
  out->width = width;
  out->height = height;
  out->ncomp = nf;
  out->hmax = hmax;
  out->vmax = vmax;
  for (int i = 0; i < 3; ++i) {
    out->h[i] = (nf == 3 && i == 0) ? ch[0] : 1;
    out->v[i] = (nf == 3 && i == 0) ? cv[0] : 1;
  }
  out->mcus_x = ceil_div(width, 8 * hmax);
  out->mcus_y = ceil_div(height, 8 * vmax);
}

// Walks entropy-coded data from `pos` to the first marker that is not RSTn, checking the restart markers' sequence and
// recording where each restart interval starts (entries past seg_capacity are not written).  Returns that marker's position
// (d[p] == 0xFF), or minus the fallback reason.
int64_t scan_extent(const uint8_t* d, int64_t n, int64_t pos, int restart, int64_t* segs, int64_t seg_capacity, int64_t seg_first,
                    int* segments) {
  int count = 1, expect = 0;
  if (seg_first < seg_capacity) segs[seg_first] = pos;
  int64_t p = pos;
  for (;;) {
    const void* f = memchr(d + p, 0xFF, static_cast<size_t>(n - p));
    if (!f) return -VDK_JPEG_MALFORMED;
    p = static_cast<const uint8_t*>(f) - d;
    if (p + 1 >= n) return -VDK_JPEG_MALFORMED;
    const int b = d[p + 1];
    if (b == 0x00) { p += 2; continue; }
    if (b == 0xFF) { p += 1; continue; }
    if (b >= 0xD0 && b <= 0xD7) {
      if (!restart || b != 0xD0 + expect) return -VDK_JPEG_RESTART;
      expect = (expect + 1) & 7;
      p += 2;
      if (seg_first + count < seg_capacity) segs[seg_first + count] = p;
      ++count;
      continue;
    }
    *segments = count;
    return p;
  }
}

int parse_one(const uint8_t* d, vdk_jpeg_desc* out, int64_t* segs, int64_t seg_capacity, int64_t seg_first) {
  const int64_t n = out->data_bytes;
  if (n < 3 || d[0] != 0xFF || d[1] != 0xD8 || d[2] != 0xFF) return VDK_JPEG_NOT_JPEG;
  int64_t pos = 2;
  RawHuff huff[2][4];
  int16_t qt[4][64];
  bool have_q[4] = {false, false, false, false};
  bool frame = false, jfif = false, adobe = false;
  int adobe_transform = -1, restart = 0, nf = 0, width = 0, height = 0;
  int cid[4] = {0}, ch[4] = {0}, cv[4] = {0}, ctq[4] = {0};
  for (;;) {
    while (pos < n && d[pos] == 0xFF) ++pos;
    if (pos >= n) return VDK_JPEG_MALFORMED;
    const int m = d[pos++];
    if (m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD9)) return VDK_JPEG_MALFORMED;
    if (pos + 2 > n) return VDK_JPEG_MALFORMED;
    const int len = (d[pos] << 8) | d[pos + 1];
    if (len < 2 || pos + len > n) return VDK_JPEG_MALFORMED;
    const uint8_t* s = d + pos + 2;
    const int sl = len - 2;
    pos += len;
    if (m == 0xC0 || m == 0xC1) {
      if (frame) return VDK_JPEG_MALFORMED;
      if (const int r = read_sof(s, sl, &nf, &width, &height, cid, ch, cv, ctq)) return r;
      frame = true;
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8) {
      return VDK_JPEG_PROCESS;  // progressive, lossless, hierarchical, arithmetic-coded (and its DAC)
    } else if (m == 0xC4) {
      if (!read_dht(s, sl, huff)) return VDK_JPEG_MALFORMED;
    } else if (m == 0xDB) {
      if (!read_dqt(s, sl, qt, have_q)) return VDK_JPEG_MALFORMED;
    } else if (m == 0xDD) {
      if (sl != 2) return VDK_JPEG_MALFORMED;
      restart = (s[0] << 8) | s[1];
    } else if ((m >= 0xE0 && m <= 0xEF) && !pillow_reads_app(m, s, sl)) {
      return VDK_JPEG_MALFORMED;  // Image.open itself refuses the file before libjpeg sees it
    } else if (m == 0xE0) {
      jfif = jfif || (sl >= 14 && memcmp(s, "JFIF\0", 5) == 0);
    } else if (m == 0xE2 && sl >= 4 && memcmp(s, "MPF\0", 4) == 0) {
      return VDK_JPEG_MPO;
    } else if (m == 0xEE) {
      if (sl >= 12 && memcmp(s, "Adobe", 5) == 0) {
        adobe = true;
        adobe_transform = s[11];
      }
    } else if ((m >= 0xE1 && m <= 0xEF) || m == 0xFE) {
      // other application segments and comments
    } else if (m == 0xDA) {
      if (!frame) return VDK_JPEG_MALFORMED;
      if (const int r = colour_reason(nf, cid, ch, cv, jfif, adobe, adobe_transform)) return r;
      if (sl < 1 || sl != 4 + 2 * s[0]) return VDK_JPEG_MALFORMED;
      const int ns = s[0];
      if (ns != nf) return VDK_JPEG_SCAN;
      for (int i = 0; i < ns; ++i)
        if (s[1 + 2 * i] != cid[i]) return VDK_JPEG_SCAN;
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return VDK_JPEG_MALFORMED;
      for (int i = 0; i < ns; ++i) {
        const int td = s[2 + 2 * i] >> 4, ta = s[2 + 2 * i] & 15;
        if (td > 3 || ta > 3 || !have_q[ctq[i]] || !huff[0][td].present || !huff[1][ta].present) return VDK_JPEG_MALFORMED;
        if (!build_huff(huff[0][td], true, &out->dc[i]) || !build_huff(huff[1][ta], false, &out->ac[i])) return VDK_JPEG_MALFORMED;
        memcpy(out->quant[i], qt[ctq[i]], sizeof(out->quant[i]));
      }
      // the entropy-coded data runs to the first marker that is not RSTn, which must be EOI (anything else: another scan)
      const int64_t begin = pos;
      int segments = 0;
      const int64_t p = scan_extent(d, n, pos, restart, segs, seg_capacity, seg_first, &segments);
      if (p < 0) return static_cast<int>(-p);
      if (d[p + 1] != 0xD9) return VDK_JPEG_SCAN;
      fill_frame(out, width, height, nf, ch, cv);
      const int64_t mcus = static_cast<int64_t>(out->mcus_x) * out->mcus_y;
      if (segments != (restart ? (mcus + restart - 1) / restart : 1)) return VDK_JPEG_RESTART;
      out->restart_interval = restart;
      out->n_segments = segments;
      out->scan_begin = begin;
      out->scan_end = p;
      return VDK_JPEG_DEVICE;
    } else {
      return VDK_JPEG_MALFORMED;
    }
  }
}

// A progressive file (SOF2): the same header rules as parse_one for the frame and everything before the first SOS, then every
// scan up to EOI.  Each scan is checked as jdphuff.c's start_pass_phuff_decoder checks it (JERR_BAD_PROGRESSION: the file
// goes to the host, where Pillow raises; JWRN_BOGUS_PROGRESSION: the host too), takes the DHT and DRI in force at its SOS,
// latches the quantisation table of each component at its first scan (jdinput.c latch_quant_tables), and gets its dependency
// level.  At EOI every coefficient of every component must have been sent with Al = 0 (coef_bits all 0): otherwise libjpeg's
// block smoothing may apply, and the file stays on the host.  Scans past scan_capacity are counted, not written.
int parse_progressive_one(const uint8_t* d, vdk_jpeg_desc* out, vdk_jpeg_scan* scans, int64_t scan_capacity,
                          int64_t scan_first, int64_t* segs, int64_t seg_capacity, int64_t seg_first) {
  const int64_t n = out->data_bytes;
  if (n < 3 || d[0] != 0xFF || d[1] != 0xD8 || d[2] != 0xFF) return VDK_JPEG_NOT_JPEG;
  int64_t pos = 2;
  RawHuff huff[2][4];
  int16_t qt[4][64];
  bool have_q[4] = {false, false, false, false}, latched[3] = {false, false, false};
  bool frame = false, jfif = false, adobe = false;
  int adobe_transform = -1, restart = 0, nf = 0, width = 0, height = 0;
  int cid[4] = {0}, ch[4] = {0}, cv[4] = {0}, ctq[4] = {0};
  int coef_bits[3][64];
  for (auto& cb : coef_bits) std::fill(cb, cb + 64, -1);
  struct Done { int comps, ss, se, level; };  // component bit mask, band and level of every scan so far
  std::vector<Done> done;
  int n_segs = 0, n_levels = 0;
  for (;;) {
    while (pos < n && d[pos] == 0xFF) ++pos;
    if (pos >= n) return VDK_JPEG_MALFORMED;
    const int m = d[pos++];
    if (m == 0xD9 && !done.empty()) {
      for (int c = 0; c < nf; ++c)
        for (int k = 0; k < 64; ++k)
          if (coef_bits[c][k] != 0) return VDK_JPEG_SCAN;  // a coefficient unsent or not fully refined
      out->restart_interval = 0;
      out->n_segments = n_segs;
      out->scan_first = scan_first;
      out->n_scans = static_cast<int>(done.size());
      out->n_levels = n_levels;
      out->scan_begin = scans && scan_first < scan_capacity ? scans[scan_first].scan_begin : 0;
      out->scan_end = pos - 2;
      return VDK_JPEG_DEVICE_PROGRESSIVE;
    }
    if (m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD9)) return VDK_JPEG_MALFORMED;
    if (pos + 2 > n) return VDK_JPEG_MALFORMED;
    const int len = (d[pos] << 8) | d[pos + 1];
    if (len < 2 || pos + len > n) return VDK_JPEG_MALFORMED;
    const uint8_t* s = d + pos + 2;
    const int sl = len - 2;
    pos += len;
    if (m == 0xC2) {
      if (frame) return VDK_JPEG_MALFORMED;
      if (const int r = read_sof(s, sl, &nf, &width, &height, cid, ch, cv, ctq)) return r;
      frame = true;
    } else if (m == 0xC0 || m == 0xC1) {
      return VDK_JPEG_MALFORMED;  // a second frame
    } else if (m >= 0xC3 && m <= 0xCF && m != 0xC4 && m != 0xC8) {
      return VDK_JPEG_PROCESS;  // lossless, hierarchical, arithmetic-coded (and its DAC)
    } else if (m == 0xC4) {
      if (!read_dht(s, sl, huff)) return VDK_JPEG_MALFORMED;
    } else if (m == 0xDB) {
      if (!read_dqt(s, sl, qt, have_q)) return VDK_JPEG_MALFORMED;
    } else if (m == 0xDD) {
      if (sl != 2) return VDK_JPEG_MALFORMED;
      restart = (s[0] << 8) | s[1];
    } else if (!done.empty() && ((m >= 0xE0 && m <= 0xEF) || m == 0xFE)) {
      // between scans libjpeg skips application segments and comments; Pillow's header reader has stopped at the first SOS
    } else if ((m >= 0xE0 && m <= 0xEF) && !pillow_reads_app(m, s, sl)) {
      return VDK_JPEG_MALFORMED;  // Image.open itself refuses the file before libjpeg sees it
    } else if (m == 0xE0) {
      jfif = jfif || (sl >= 14 && memcmp(s, "JFIF\0", 5) == 0);
    } else if (m == 0xE2 && sl >= 4 && memcmp(s, "MPF\0", 4) == 0) {
      return VDK_JPEG_MPO;
    } else if (m == 0xEE) {
      if (sl >= 12 && memcmp(s, "Adobe", 5) == 0) {
        adobe = true;
        adobe_transform = s[11];
      }
    } else if ((m >= 0xE1 && m <= 0xEF) || m == 0xFE) {
      // other application segments and comments
    } else if (m == 0xDA) {
      if (!frame) return VDK_JPEG_MALFORMED;
      if (done.empty()) {
        if (const int r = colour_reason(nf, cid, ch, cv, jfif, adobe, adobe_transform)) return r;
        fill_frame(out, width, height, nf, ch, cv);
      }
      if (sl < 1 || sl != 4 + 2 * s[0] || s[0] < 1 || s[0] > 4) return VDK_JPEG_MALFORMED;  // JERR_BAD_LENGTH
      const int ns = s[0];
      int comp[4], mask = 0;
      for (int i = 0; i < ns; ++i) {
        comp[i] = -1;
        for (int c = 0; c < nf; ++c)
          if (cid[c] == s[1 + 2 * i]) comp[i] = c;
        if (comp[i] < 0 || (mask >> comp[i] & 1)) return VDK_JPEG_MALFORMED;  // JERR_BAD_COMPONENT_ID
        if (i && comp[i] < comp[i - 1]) return VDK_JPEG_SCAN;  // MCU blocks in another order than the frame's
        mask |= 1 << comp[i];
      }
      const int ss = s[1 + 2 * ns], se = s[2 + 2 * ns], ah = s[3 + 2 * ns] >> 4, al = s[3 + 2 * ns] & 15;
      const bool dc = ss == 0;
      bool bad = dc ? se != 0 : (ss > se || se > 63 || ns != 1);
      if (ah != 0 && al != ah - 1) bad = true;
      if (al > 13 || bad) return VDK_JPEG_MALFORMED;  // JERR_BAD_PROGRESSION
      for (int i = 0; i < ns; ++i) {
        int* cb = coef_bits[comp[i]];
        if (!dc && cb[0] < 0) return VDK_JPEG_SCAN;  // JWRN_BOGUS_PROGRESSION: AC before any DC
        for (int k = ss; k <= se; ++k) {
          if (ah != std::max(cb[k], 0)) return VDK_JPEG_SCAN;  // JWRN_BOGUS_PROGRESSION
          cb[k] = al;
        }
        if (!latched[comp[i]]) {
          if (!have_q[ctq[comp[i]]]) return VDK_JPEG_MALFORMED;  // JERR_NO_QUANT_TABLE
          memcpy(out->quant[comp[i]], qt[ctq[comp[i]]], sizeof(out->quant[0]));
          latched[comp[i]] = true;
        }
      }
      const int64_t at = scan_first + static_cast<int64_t>(done.size());
      vdk_jpeg_scan* sc = scans && at < scan_capacity ? scans + at : nullptr;
      vdk_jpeg_scan spare;  // checks the tables of a scan that is not written
      if (!sc) sc = &spare;
      for (int i = 0; i < ns; ++i) {
        const int td = s[2 + 2 * i] >> 4, ta = s[2 + 2 * i] & 15;
        if (dc && ah == 0 && (td > 3 || !huff[0][td].present || !build_huff(huff[0][td], true, &sc->tbl[i])))
          return VDK_JPEG_MALFORMED;
        if (!dc && (ta > 3 || !huff[1][ta].present || !build_huff(huff[1][ta], false, &sc->tbl[0]))) return VDK_JPEG_MALFORMED;
      }
      int units_x = out->mcus_x, units_y = out->mcus_y;
      if (ns == 1) {  // one component: its own blocks, not the MCU-padded grid
        units_x = ceil_div(width * out->h[comp[0]], 8 * out->hmax);
        units_y = ceil_div(height * out->v[comp[0]], 8 * out->vmax);
      }
      int segments = 0;
      const int64_t p = scan_extent(d, n, pos, restart, segs, seg_capacity, seg_first + n_segs, &segments);
      if (p < 0) return static_cast<int>(-p);
      const int64_t units = static_cast<int64_t>(units_x) * units_y;
      if (segments != (restart ? (units + restart - 1) / restart : 1)) return VDK_JPEG_RESTART;
      int level = 0;
      for (const Done& e : done)
        if ((e.comps & mask) && e.ss <= se && ss <= e.se) level = std::max(level, e.level + 1);
      n_levels = std::max(n_levels, level + 1);
      sc->scan_begin = pos;
      sc->scan_end = p;
      sc->seg_first = seg_first + n_segs;
      sc->n_segments = segments;
      sc->restart_interval = restart;
      sc->level = level;
      sc->ncomp = ns;
      for (int i = 0; i < 3; ++i) sc->comp[i] = i < ns ? comp[i] : 0;
      sc->ss = ss;
      sc->se = se;
      sc->ah = ah;
      sc->al = al;
      sc->units_x = units_x;
      sc->units_y = units_y;
      done.push_back({mask, ss, se, level});
      n_segs += segments;
      pos = p;
    } else {
      return VDK_JPEG_MALFORMED;
    }
  }
}

__host__ __device__ inline int64_t image_blocks(const vdk_jpeg_desc& d, int c) {
  return static_cast<int64_t>(d.mcus_x) * d.h[c] * d.mcus_y * d.v[c];
}

// ---------------------------------------------------------------------------------------------------------------- kernels
// whether a launch decodes image `d`: baseline images always, progressive ones only in vdk_jpeg_decode_ex
__host__ __device__ inline bool decoded(const vdk_jpeg_desc& d, int progressive) {
  return d.reason == VDK_JPEG_DEVICE || (progressive && d.reason == VDK_JPEG_DEVICE_PROGRESSIVE);
}

// index of the image owning CTA `cta` of a grid laid out by *_cta_base (images without CTAs share the next image's base)
__device__ int owner(const vdk_jpeg_desc* descs, int n, int64_t cta, bool color) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const int64_t b = color ? descs[mid].color_cta_base : descs[mid].idct_cta_base;
    if (b <= cta) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct BitReader {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t buf;
  int bits;  // valid bits at the bottom of buf, oldest first
  int pad;   // zero bytes fed after a marker or the interval's end

  __device__ __forceinline__ void fill() {
    while (bits <= 56) {
      uint32_t b = 0;
      if (p < end) {
        b = __ldg(p);
        if (b == 0xFF) {
          if (p + 1 < end && __ldg(p + 1) == 0) {
            p += 2;
          } else {  // a marker inside the interval: feed zeros from here on
            p = end;
            b = 0;
            ++pad;
          }
        } else {
          ++p;
        }
      } else {
        ++pad;
      }
      buf = (buf << 8) | b;
      bits += 8;
    }
  }
  __device__ __forceinline__ int get(int s) {
    bits -= s;
    return static_cast<int>((buf >> bits) & ((1u << s) - 1));
  }
};

__device__ __forceinline__ int huff_extend(int r, int s) { return r < (1 << (s - 1)) ? r - (1 << s) + 1 : r; }

// jdhuff.c's decode of one symbol; bits >= 32 on entry
__device__ __forceinline__ int huff_decode(BitReader& br, const vdk_jpeg_huff* t, int& err) {
  const uint32_t e = __ldg(&t->lut[(br.buf >> (br.bits - 9)) & 511]);
  if (e) {
    br.bits -= e >> 8;
    return e & 255;
  }
  int l = 10;
  int code = static_cast<int>((br.buf >> (br.bits - 10)) & 1023);
  while (l <= 16 && code > __ldg(&t->maxcode[l])) {
    ++l;
    code = static_cast<int>((br.buf >> (br.bits - l)) & ((1u << l) - 1));
  }
  if (l > 16) {
    err |= VDK_JPEG_BAD_CODE;
    return 0;
  }
  br.bits -= l;
  return __ldg(&t->huffval[code + __ldg(&t->valoffset[l])]);
}

__global__ void __launch_bounds__(kEntropyThreads) jpeg_entropy_kernel(const uint8_t* __restrict__ data,
                                                                       const vdk_jpeg_desc* descs, const int64_t* seg_table,
                                                                       uint8_t* ws, int32_t* status, int progressive) {
  const int img = blockIdx.y;
  const vdk_jpeg_desc& d = descs[img];
  const int seg = blockIdx.x * kEntropyThreads + threadIdx.x;
  if (d.reason != VDK_JPEG_DEVICE) {
    if (seg == 0 && !decoded(d, progressive)) status[img] = VDK_JPEG_BAD_SKIPPED;
    return;
  }
  if (seg >= d.n_segments) return;
  const int64_t* segs = seg_table + d.seg_first;
  const uint8_t* f = data + d.data_offset;
  BitReader br;
  br.p = f + segs[seg];
  br.end = f + (seg + 1 < d.n_segments ? segs[seg + 1] - 2 : d.scan_end);
  br.buf = 0;
  br.bits = 0;
  br.pad = 0;
  const int64_t mcus = static_cast<int64_t>(d.mcus_x) * d.mcus_y;
  const int64_t m0 = d.restart_interval ? static_cast<int64_t>(seg) * d.restart_interval : 0;
  const int64_t m1 = d.restart_interval ? min(mcus, m0 + d.restart_interval) : mcus;
  int16_t* comp[3];
  int bw[3];
  int64_t off = d.ws_coef;
  for (int c = 0; c < d.ncomp; ++c) {
    comp[c] = reinterpret_cast<int16_t*>(ws + off);
    bw[c] = d.mcus_x * d.h[c];
    off += image_blocks(d, c) * 128;
  }
  int pred[3] = {0, 0, 0};
  int err = 0;
  for (int64_t m = m0; m < m1 && !err; ++m) {
    const int my = static_cast<int>(m / d.mcus_x), mx = static_cast<int>(m % d.mcus_x);
    for (int c = 0; c < d.ncomp && !err; ++c) {
      const vdk_jpeg_huff* dc = &d.dc[c];
      const vdk_jpeg_huff* ac = &d.ac[c];
      for (int by = 0; by < d.v[c] && !err; ++by) {
        for (int bx = 0; bx < d.h[c] && !err; ++bx) {
          int16_t* blk = comp[c] + (static_cast<int64_t>(my * d.v[c] + by) * bw[c] + mx * d.h[c] + bx) * 64;
          if (br.bits < 32) br.fill();
          int s = huff_decode(br, dc, err);
          if (s) pred[c] += huff_extend(br.get(s), s);
          blk[0] = static_cast<int16_t>(pred[c]);
          for (int k = 1; k < 64 && !err; ++k) {
            if (br.bits < 32) br.fill();
            const int rs = huff_decode(br, ac, err);
            const int r = rs >> 4;
            s = rs & 15;
            if (s) {
              k += r;
              if (k > 63) { err |= VDK_JPEG_BAD_AC_RUN; break; }
              blk[kNatural[k]] = static_cast<int16_t>(huff_extend(br.get(s), s));
            } else if (r == 15) {
              k += 15;
              if (k > 63) { err |= VDK_JPEG_BAD_AC_RUN; break; }
            } else {
              break;
            }
          }
        }
      }
    }
    if (br.pad * 8 > br.bits) err |= VDK_JPEG_BAD_SHORT;  // decoded bits the stream does not have
  }
  if (!err && (br.bits - br.pad * 8) + 8 * (br.end - br.p) >= 8) err |= VDK_JPEG_BAD_EXTRA;
  if (err) atomicOr(status + img, err);
}

// jdphuff.c's four decoders on one block of a scan; `i` is the component's place in the scan (its DC table and predictor).
// A stream libjpeg decodes with a warning or an error, or into a coefficient outside the band, is flagged (the host decodes
// it), so everything flagged here is either malformed or decoded by libjpeg in a way not restated.
__device__ __forceinline__ void progressive_block(BitReader& br, const vdk_jpeg_scan& sc, int i, int16_t* blk, int64_t& pred,
                                                  int& eobrun, int& err) {
  const int al = sc.al;
  if (br.bits < 32) br.fill();
  if (sc.ss == 0) {
    if (sc.ah == 0) {  // DC first: the predictor is an int (JERR_BAD_DCT_COEF on overflow), stored as (JCOEF)(s << Al)
      const int s = huff_decode(br, &sc.tbl[i], err);
      if (s) pred += huff_extend(br.get(s), s);
      if (pred > INT_MAX || pred < INT_MIN) err |= VDK_JPEG_BAD_CODE;
      blk[0] = static_cast<int16_t>(static_cast<uint32_t>(static_cast<int>(pred)) << al);
    } else if (br.get(1)) {  // DC refine: the next bit of the value
      blk[0] = static_cast<int16_t>(blk[0] | (1 << al));
    }
    return;
  }
  const vdk_jpeg_huff* t = &sc.tbl[0];
  if (sc.ah == 0) {  // AC first
    if (eobrun > 0) {
      --eobrun;
      return;
    }
    for (int k = sc.ss; k <= sc.se; ++k) {
      if (br.bits < 32) br.fill();
      const int rs = huff_decode(br, t, err);
      if (err) return;
      const int r = rs >> 4, s = rs & 15;
      if (s) {
        k += r;
        if (k > sc.se) { err |= VDK_JPEG_BAD_AC_RUN; return; }
        blk[kNatural[k]] = static_cast<int16_t>(static_cast<uint32_t>(huff_extend(br.get(s), s)) << al);
      } else if (r == 15) {
        k += 15;  // ZRL; one past Se just ends the band, as in libjpeg
      } else {
        eobrun = (1 << r) - 1;
        if (r) eobrun += br.get(r);
        break;
      }
    }
    return;
  }
  // AC refine: correction bits for the coefficients already non-zero, new ones of magnitude 1 << Al
  const int p1 = 1 << al, m1 = -p1;
  int k = sc.ss;
  auto correct = [&](int16_t& c) {
    if (br.bits < 32) br.fill();
    if (br.get(1) && (c & p1) == 0) c = static_cast<int16_t>(c >= 0 ? c + p1 : c + m1);
  };
  if (eobrun == 0) {
    for (; k <= sc.se; ++k) {
      if (br.bits < 32) br.fill();
      const int rs = huff_decode(br, t, err);
      if (err) return;
      int r = rs >> 4, s = rs & 15;
      if (s) {
        if (s != 1) { err |= VDK_JPEG_BAD_CODE; return; }  // JWRN_HUFF_BAD_CODE
        s = br.get(1) ? p1 : m1;
      } else if (r != 15) {
        eobrun = 1 << r;
        if (r) eobrun += br.get(r);
        break;
      }
      do {
        int16_t& c = blk[kNatural[k]];
        if (c != 0) {
          correct(c);
        } else if (--r < 0) {
          break;
        }
        ++k;
      } while (k <= sc.se);
      if (s) {
        if (k > sc.se) { err |= VDK_JPEG_BAD_AC_RUN; return; }
        blk[kNatural[k]] = static_cast<int16_t>(s);
      }
    }
  }
  if (eobrun > 0) {
    for (; k <= sc.se; ++k) {
      int16_t& c = blk[kNatural[k]];
      if (c != 0) correct(c);
    }
    --eobrun;
  }
}

// One thread per (image, scan of dependency level `level`, restart interval): blockIdx.y is the image, blockIdx.z the scan's
// rank among the image's scans of that level.  Scans of one level write disjoint coefficients.
__global__ void __launch_bounds__(kEntropyThreads) jpeg_progressive_kernel(const uint8_t* __restrict__ data,
                                                                           const vdk_jpeg_desc* descs,
                                                                           const vdk_jpeg_scan* scans,
                                                                           const int64_t* seg_table, uint8_t* ws,
                                                                           int32_t* status, int level) {
  const int img = blockIdx.y;
  const vdk_jpeg_desc& d = descs[img];
  if (d.reason != VDK_JPEG_DEVICE_PROGRESSIVE || level >= d.n_levels) return;
  const vdk_jpeg_scan* sc = nullptr;
  for (int i = 0, rank = blockIdx.z; i < d.n_scans; ++i) {
    const vdk_jpeg_scan* s = scans + d.scan_first + i;
    if (s->level == level && rank-- == 0) {
      sc = s;
      break;
    }
  }
  const int seg = blockIdx.x * kEntropyThreads + threadIdx.x;
  if (!sc || seg >= sc->n_segments) return;
  const int64_t* segs = seg_table + sc->seg_first;
  const uint8_t* f = data + d.data_offset;
  BitReader br;
  br.p = f + segs[seg];
  br.end = f + (seg + 1 < sc->n_segments ? segs[seg + 1] - 2 : sc->scan_end);
  br.buf = 0;
  br.bits = 0;
  br.pad = 0;
  const int64_t units = static_cast<int64_t>(sc->units_x) * sc->units_y;
  const int64_t u0 = sc->restart_interval ? static_cast<int64_t>(seg) * sc->restart_interval : 0;
  const int64_t u1 = sc->restart_interval ? min(units, u0 + sc->restart_interval) : units;
  int16_t* comp[3];
  int bw[3];
  int64_t off = d.ws_coef;
  for (int c = 0; c < d.ncomp; ++c) {
    comp[c] = reinterpret_cast<int16_t*>(ws + off);
    bw[c] = d.mcus_x * d.h[c];
    off += image_blocks(d, c) * 128;
  }
  int64_t pred[3] = {0, 0, 0};
  int eobrun = 0, err = 0;
  for (int64_t u = u0; u < u1 && !err; ++u) {
    const int uy = static_cast<int>(u / sc->units_x), ux = static_cast<int>(u % sc->units_x);
    if (sc->ncomp == 1) {  // a block of the component's own grid
      const int c = sc->comp[0];
      progressive_block(br, *sc, 0, comp[c] + (static_cast<int64_t>(uy) * bw[c] + ux) * 64, pred[0], eobrun, err);
    } else {  // an MCU of an interleaved DC scan
      for (int i = 0; i < sc->ncomp && !err; ++i) {
        const int c = sc->comp[i];
        for (int by = 0; by < d.v[c] && !err; ++by)
          for (int bx = 0; bx < d.h[c] && !err; ++bx)
            progressive_block(br, *sc, i, comp[c] + (static_cast<int64_t>(uy * d.v[c] + by) * bw[c] + ux * d.h[c] + bx) * 64,
                              pred[i], eobrun, err);
      }
    }
    if (br.pad * 8 > br.bits) err |= VDK_JPEG_BAD_SHORT;  // decoded bits the stream does not have
  }
  if (!err && (br.bits - br.pad * 8) + 8 * (br.end - br.p) >= 8) err |= VDK_JPEG_BAD_EXTRA;
  if (err) atomicOr(status + img, err);
}

constexpr int64_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                  F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

// one jpeg_idct_islow pass over 8 values; results DESCALEd by `shift`
__device__ __forceinline__ void idct_1d(const int64_t* c, int shift, int64_t* out) {
  int64_t z2 = c[2], z3 = c[6];
  int64_t z1 = (z2 + z3) * F0541;
  const int64_t tmp2e = z1 + z3 * -F1847, tmp3e = z1 + z2 * F0765;
  const int64_t tmp0e = (c[0] + c[4]) * 8192, tmp1e = (c[0] - c[4]) * 8192;
  const int64_t t10 = tmp0e + tmp3e, t13 = tmp0e - tmp3e, t11 = tmp1e + tmp2e, t12 = tmp1e - tmp2e;
  int64_t o0 = c[7], o1 = c[5], o2 = c[3], o3 = c[1];
  z1 = o0 + o3;
  z2 = o1 + o2;
  z3 = o0 + o2;
  int64_t z4 = o1 + o3;
  const int64_t z5 = (z3 + z4) * F1175;
  o0 *= F0298;
  o1 *= F2053;
  o2 *= F3072;
  o3 *= F1501;
  z1 *= -F0899;
  z2 *= -F2562;
  z3 = z3 * -F1961 + z5;
  z4 = z4 * -F0390 + z5;
  o0 += z1 + z3;
  o1 += z2 + z4;
  o2 += z2 + z3;
  o3 += z1 + z4;
  const int64_t r = int64_t(1) << (shift - 1);
  out[0] = (t10 + o3 + r) >> shift;
  out[7] = (t10 - o3 + r) >> shift;
  out[1] = (t11 + o2 + r) >> shift;
  out[6] = (t11 - o2 + r) >> shift;
  out[2] = (t12 + o1 + r) >> shift;
  out[5] = (t12 - o1 + r) >> shift;
  out[3] = (t13 + o0 + r) >> shift;
  out[4] = (t13 - o0 + r) >> shift;
}

// libjpeg's IDCT range limit: sample_range_limit + CENTERJSAMPLE indexed by x & RANGE_MASK
__device__ __forceinline__ uint32_t idct_limit(int64_t x) {
  const int t = static_cast<int>(x & 1023);
  return t < 128 ? t + 128 : (t < 512 ? 255 : (t < 896 ? 0 : t - 896));
}

__global__ void __launch_bounds__(256) jpeg_idct_kernel(const vdk_jpeg_desc* descs, int n, uint8_t* ws, int progressive) {
  __shared__ int32_t work[kIdctBlocksPerCta][8][9];
  __shared__ int s_img;
  if (threadIdx.x == 0) s_img = owner(descs, n, blockIdx.x, false);
  __syncthreads();
  const vdk_jpeg_desc& d = descs[s_img];
  if (!decoded(d, progressive)) return;  // laid out, but not decoded by this launch
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  int64_t b = (blockIdx.x - d.idct_cta_base) * kIdctBlocksPerCta + lb;
  int c = 0;
  int64_t coef_off = d.ws_coef, plane_off = d.ws_plane;
  for (; c < d.ncomp && b >= image_blocks(d, c); ++c) {
    b -= image_blocks(d, c);
    coef_off += image_blocks(d, c) * 128;
    plane_off += image_blocks(d, c) * 64;
  }
  const bool active = c < d.ncomp;
  if (active) {  // pass 1: column `lane`
    const int16_t* blk = reinterpret_cast<const int16_t*>(ws + coef_off) + b * 64;
    int64_t col[8], res[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) col[r] = static_cast<int64_t>(blk[r * 8 + lane]) * d.quant[c][r * 8 + lane];
    idct_1d(col, 11, res);
#pragma unroll
    for (int r = 0; r < 8; ++r) work[lb][r][lane] = static_cast<int32_t>(res[r]);
  }
  __syncwarp();
  if (active) {  // pass 2: row `lane`
    int64_t row[8], res[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) row[k] = work[lb][lane][k];
    idct_1d(row, 18, res);
    const int bw = d.mcus_x * d.h[c];
    const int64_t by = b / bw, bx = b % bw;
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      lo |= idct_limit(res[k]) << (8 * k);
      hi |= idct_limit(res[k + 4]) << (8 * k);
    }
    uint8_t* dst = ws + plane_off + (by * 8 + lane) * (static_cast<int64_t>(bw) * 8) + bx * 8;
    *reinterpret_cast<uint2*>(dst) = make_uint2(lo, hi);
  }
}

// jdsample.c: the chroma sample at output pixel (x, y) of a plane of downsampled size dw x dh, factors hf x vf (1 or 2)
__device__ __forceinline__ int upsampled(const uint8_t* pl, int64_t pitch, int dw, int dh, int hf, int vf, int x, int y) {
  if (vf == 1) {
    const uint8_t* row = pl + y * pitch;
    if (hf == 1) return row[x];
    const int i = x >> 1;
    if (dw <= 2) return row[i];  // h2v1_upsample
    if (x & 1) return i == dw - 1 ? row[i] : (3 * row[i] + row[i + 1] + 2) >> 2;
    return i == 0 ? row[0] : (3 * row[i] + row[i - 1] + 1) >> 2;
  }
  const int j = y >> 1, odd = y & 1;
  const int j1 = odd ? min(j + 1, dh - 1) : max(j - 1, 0);  // the nearer of the rows above / below, edges duplicated
  const uint8_t* r0 = pl + j * pitch;
  const uint8_t* r1 = pl + j1 * pitch;
  if (hf == 1) return (3 * r0[x] + r1[x] + 1 + odd) >> 2;  // h1v2_fancy_upsample
  const int i = x >> 1;
  if (dw <= 2) return r0[i];  // h2v2_upsample
  const int cs = 3 * r0[i] + r1[i];
  if (x & 1) return i == dw - 1 ? (cs * 4 + 7) >> 4 : (3 * cs + 3 * r0[i + 1] + r1[i + 1] + 7) >> 4;
  return i == 0 ? (cs * 4 + 8) >> 4 : (3 * cs + 3 * r0[i - 1] + r1[i - 1] + 8) >> 4;
}

__device__ __forceinline__ uint8_t clamp255(int v) { return static_cast<uint8_t>(min(max(v, 0), 255)); }

__global__ void __launch_bounds__(256) jpeg_color_kernel(const vdk_jpeg_desc* descs, int n, const uint8_t* ws, uint8_t* out,
                                                        int progressive) {
  __shared__ int s_img;
  if (threadIdx.x == 0) s_img = owner(descs, n, blockIdx.x, true);
  __syncthreads();
  const vdk_jpeg_desc& d = descs[s_img];
  if (!decoded(d, progressive)) return;
  const int w = d.width, h = d.height;
  const int64_t pix0 = (blockIdx.x - d.color_cta_base) * kColorPixelsPerCta;
  const int64_t pitch0 = static_cast<int64_t>(d.mcus_x) * d.h[0] * 8;
  const uint8_t* p0 = ws + d.ws_plane;
  uint8_t* o = out + d.out_offset;
  if (d.ncomp == 1) {
    for (int k = threadIdx.x; k < kColorPixelsPerCta; k += 256) {
      const int64_t p = pix0 + k;
      if (p >= static_cast<int64_t>(w) * h) break;
      const int y = static_cast<int>(p / w), x = static_cast<int>(p % w);
      const uint8_t g = p0[y * pitch0 + x];
      o[p * 3] = g;
      o[p * 3 + 1] = g;
      o[p * 3 + 2] = g;
    }
    return;
  }
  const int64_t pitch1 = static_cast<int64_t>(d.mcus_x) * 8;
  const uint8_t* p1 = p0 + image_blocks(d, 0) * 64;
  const uint8_t* p2 = p1 + image_blocks(d, 1) * 64;
  const int hf = d.hmax, vf = d.vmax, dw = ceil_div(w, hf), dh = ceil_div(h, vf);
  for (int k = threadIdx.x; k < kColorPixelsPerCta; k += 256) {
    const int64_t p = pix0 + k;
    if (p >= static_cast<int64_t>(w) * h) break;
    const int y = static_cast<int>(p / w), x = static_cast<int>(p % w);
    const int yy = p0[y * pitch0 + x];
    const int cb = upsampled(p1, pitch1, dw, dh, hf, vf, x, y) - 128;
    const int cr = upsampled(p2, pitch1, dw, dh, hf, vf, x, y) - 128;
    // jdcolor.c build_ycc_rgb_table: FIX(1.40200), FIX(1.77200), FIX(0.71414), FIX(0.34414) at SCALEBITS 16
    o[p * 3] = clamp255(yy + ((91881 * cr + 32768) >> 16));
    o[p * 3 + 1] = clamp255(yy + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
    o[p * 3 + 2] = clamp255(yy + ((116130 * cb + 32768) >> 16));
  }
}

}  // namespace
}  // namespace vdk

using namespace vdk;

extern "C" int vdk_jpeg_parse(const uint8_t* packed, vdk_jpeg_desc* descs, int n, int64_t* segs, int64_t seg_capacity) {
  VDK_REQUIRE(packed && descs && n > 0 && seg_capacity >= 0 && (segs || seg_capacity == 0), "vdk_jpeg_parse: bad arguments");
  int64_t seg_first = 0;
  for (int i = 0; i < n; ++i) {
    vdk_jpeg_desc& d = descs[i];
    VDK_REQUIRE(d.data_offset >= 0 && d.data_bytes >= 0, "vdk_jpeg_parse: bad byte range of file %d", i);
    const int64_t off = d.data_offset, bytes = d.data_bytes;
    memset(&d, 0, sizeof(d));
    d.data_offset = off;
    d.data_bytes = bytes;
    d.reason = parse_one(packed + off, &d, segs, seg_capacity, seg_first);
    d.seg_first = seg_first;
    if (d.reason == VDK_JPEG_DEVICE) seg_first += d.n_segments;
  }
  return VDK_OK;
}

extern "C" int vdk_jpeg_parse_progressive(const uint8_t* packed, vdk_jpeg_desc* descs, int n, vdk_jpeg_scan* scans,
                                          int64_t scan_capacity, int64_t* segs, int64_t seg_capacity) {
  VDK_REQUIRE(packed && descs && n > 0 && scan_capacity >= 0 && seg_capacity >= 0 && (scans || scan_capacity == 0) &&
                  (segs || seg_capacity == 0),
              "vdk_jpeg_parse_progressive: bad arguments");
  int64_t seg_first = 0, scan_first = 0;  // after every entry the parsers already wrote
  for (int i = 0; i < n; ++i) {
    const vdk_jpeg_desc& d = descs[i];
    if (d.reason == VDK_JPEG_DEVICE || d.reason == VDK_JPEG_DEVICE_PROGRESSIVE)
      seg_first = std::max(seg_first, d.seg_first + d.n_segments);
    if (d.reason == VDK_JPEG_DEVICE_PROGRESSIVE) scan_first = std::max(scan_first, d.scan_first + d.n_scans);
  }
  for (int i = 0; i < n; ++i) {
    vdk_jpeg_desc& d = descs[i];
    if (d.reason != VDK_JPEG_PROCESS) continue;
    VDK_REQUIRE(d.data_offset >= 0 && d.data_bytes >= 0, "vdk_jpeg_parse_progressive: bad byte range of file %d", i);
    const int64_t off = d.data_offset, bytes = d.data_bytes;
    memset(&d, 0, sizeof(d));
    d.data_offset = off;
    d.data_bytes = bytes;
    d.reason = parse_progressive_one(packed + off, &d, scans, scan_capacity, scan_first, segs, seg_capacity, seg_first);
    d.seg_first = seg_first;
    if (d.reason == VDK_JPEG_DEVICE_PROGRESSIVE) {
      seg_first += d.n_segments;
      scan_first += d.n_scans;
    } else {
      d.n_segments = d.n_scans = d.n_levels = 0;
    }
  }
  return VDK_OK;
}

extern "C" size_t vdk_jpeg_workspace_bytes(vdk_jpeg_desc* descs, int n) {
  if (!descs || n <= 0) return 0;
  size_t off = 0;
  int64_t idct = 0, color = 0;
  for (int pass = 0; pass < 2; ++pass) {  // every coefficient store first (one memset clears them), then planes and RST tables
    for (int i = 0; i < n; ++i) {
      vdk_jpeg_desc& d = descs[i];
      if (pass == 1) {
        d.idct_cta_base = idct;
        d.color_cta_base = color;
      }
      if (!decoded(d, 1)) continue;
      if (d.width <= 0 || d.height <= 0 || (d.ncomp != 1 && d.ncomp != 3) || d.n_segments < 1 || d.out_offset < 0 ||
          (d.out_offset & 255) || (d.reason == VDK_JPEG_DEVICE_PROGRESSIVE && d.n_scans < 1)) {
        set_error("vdk_jpeg_workspace_bytes: descriptor %d is not a parsed device image with a 256-byte aligned out_offset", i);
        return 0;
      }
      int64_t blocks = 0;
      for (int c = 0; c < d.ncomp; ++c) blocks += image_blocks(d, c);
      if (pass == 0) {
        d.ws_coef = off;
        off += up256(blocks * 128);
        continue;
      }
      d.ws_plane = off;
      off += up256(blocks * 64);
      idct += (blocks + kIdctBlocksPerCta - 1) / kIdctBlocksPerCta;
      color += (static_cast<int64_t>(d.width) * d.height + kColorPixelsPerCta - 1) / kColorPixelsPerCta;
    }
  }
  return std::max<size_t>(off, 256);
}

namespace {

// vdk_jpeg_decode and vdk_jpeg_decode_ex: `scans` null decodes the baseline images only
int decode_batch(const uint8_t* data, const vdk_jpeg_desc* descs, const vdk_jpeg_desc* descs_dev, const int64_t* segs_dev,
                 const vdk_jpeg_scan* scans, const vdk_jpeg_scan* scans_dev, int n, uint8_t* out, int32_t* status,
                 void* workspace, size_t workspace_bytes, void* stream) {
  const int progressive = scans != nullptr;
  size_t need = 0, coef_end = 0;
  int64_t idct_ctas = 0, color_ctas = 0, max_segs = 0, images = 0;
  int levels = 0;
  for (int i = 0; i < n; ++i) {
    const vdk_jpeg_desc& d = descs[i];
    if (!decoded(d, 1)) continue;  // progressive images are laid out even when this call skips them
    int64_t blocks = 0;
    for (int c = 0; c < d.ncomp; ++c) blocks += image_blocks(d, c);
    VDK_REQUIRE(d.idct_cta_base == idct_ctas && d.color_cta_base == color_ctas,
                "vdk_jpeg_decode: descriptor %d was not laid out by vdk_jpeg_workspace_bytes", i);
    idct_ctas += (blocks + kIdctBlocksPerCta - 1) / kIdctBlocksPerCta;
    color_ctas += (static_cast<int64_t>(d.width) * d.height + kColorPixelsPerCta - 1) / kColorPixelsPerCta;
    if (!decoded(d, progressive)) continue;
    ++images;
    need = std::max<size_t>(need, d.ws_plane + up256(static_cast<size_t>(blocks) * 64));
    coef_end = std::max<size_t>(coef_end, d.ws_coef + static_cast<size_t>(blocks) * 128);
    if (d.reason == VDK_JPEG_DEVICE) max_segs = std::max<int64_t>(max_segs, d.n_segments);
    else levels = std::max(levels, d.n_levels);
  }
  VDK_REQUIRE(workspace_bytes >= need, "vdk_jpeg_decode: workspace too small (%zu < %zu)", workspace_bytes, need);
  VDK_REQUIRE(n <= 65535, "vdk_jpeg_decode: at most 65535 images per call");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  VDK_CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int32_t) * n, s));
  if (coef_end) VDK_CUDA_OK(cudaMemsetAsync(ws, 0, coef_end, s));  // the entropy kernels write only non-zero coefficients
  const int64_t seg_blocks = std::max<int64_t>(1, (max_segs + kEntropyThreads - 1) / kEntropyThreads);
  jpeg_entropy_kernel<<<dim3(static_cast<unsigned>(seg_blocks), n), kEntropyThreads, 0, s>>>(data, descs_dev, segs_dev, ws,
                                                                                           status, progressive);
  VDK_CUDA_OK(cudaGetLastError());
  for (int level = 0; level < levels; ++level) {  // one launch per dependency level across the batch
    int64_t per_image = 0, segs = 0;
    for (int i = 0; i < n; ++i) {
      const vdk_jpeg_desc& d = descs[i];
      if (d.reason != VDK_JPEG_DEVICE_PROGRESSIVE) continue;
      int64_t k = 0;
      for (int j = 0; j < d.n_scans; ++j) {
        const vdk_jpeg_scan& sc = scans[d.scan_first + j];
        if (sc.level != level) continue;
        ++k;
        segs = std::max<int64_t>(segs, sc.n_segments);
      }
      per_image = std::max(per_image, k);
    }
    VDK_REQUIRE(per_image <= 65535, "vdk_jpeg_decode_ex: more than 65535 scans of one level in an image");
    const unsigned blocks = static_cast<unsigned>((segs + kEntropyThreads - 1) / kEntropyThreads);
    jpeg_progressive_kernel<<<dim3(blocks, n, static_cast<unsigned>(per_image)), kEntropyThreads, 0, s>>>(
        data, descs_dev, scans_dev, segs_dev, ws, status, level);
    VDK_CUDA_OK(cudaGetLastError());
  }
  if (images == 0) return VDK_OK;
  jpeg_idct_kernel<<<static_cast<unsigned>(idct_ctas), 256, 0, s>>>(descs_dev, n, ws, progressive);
  VDK_CUDA_OK(cudaGetLastError());
  jpeg_color_kernel<<<static_cast<unsigned>(color_ctas), 256, 0, s>>>(descs_dev, n, ws, out, progressive);
  VDK_CUDA_OK(cudaGetLastError());
  return VDK_OK;
}

}  // namespace

extern "C" int vdk_jpeg_decode(const uint8_t* data, const vdk_jpeg_desc* descs, const vdk_jpeg_desc* descs_dev,
                               const int64_t* segs_dev, int n, uint8_t* out, int32_t* status, void* workspace,
                               size_t workspace_bytes, void* stream) {
  VDK_REQUIRE(data && descs && descs_dev && segs_dev && n > 0 && out && status && workspace, "vdk_jpeg_decode: bad arguments");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_jpeg_decode: workspace must be 256-byte aligned");
  return decode_batch(data, descs, descs_dev, segs_dev, nullptr, nullptr, n, out, status, workspace, workspace_bytes, stream);
}

extern "C" int vdk_jpeg_decode_ex(const uint8_t* data, const vdk_jpeg_desc* descs, const vdk_jpeg_desc* descs_dev,
                                  const int64_t* segs_dev, const vdk_jpeg_scan* scans, const vdk_jpeg_scan* scans_dev, int n,
                                  uint8_t* out, int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  VDK_REQUIRE(data && descs && descs_dev && segs_dev && scans && scans_dev && n > 0 && out && status && workspace,
              "vdk_jpeg_decode_ex: bad arguments");
  VDK_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "vdk_jpeg_decode_ex: workspace must be 256-byte aligned");
  return decode_batch(data, descs, descs_dev, segs_dev, scans, scans_dev, n, out, status, workspace, workspace_bytes, stream);
}

extern "C" int vdk_jpeg_struct_sizes(size_t* out, int n) {
  const size_t sizes[] = {sizeof(vdk_jpeg_huff), sizeof(vdk_jpeg_desc)};
  const int k = static_cast<int>(sizeof(sizes) / sizeof(sizes[0]));
  for (int i = 0; i < n && i < k; ++i) out[i] = sizes[i];
  return k;
}

extern "C" int vdk_jpeg_progressive_struct_sizes(size_t* out, int n) {
  if (n > 0) out[0] = sizeof(vdk_jpeg_scan);
  return 1;
}
