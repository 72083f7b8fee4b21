// Host half of the JPEG codec: ITU-T T.81 tables, marker layer, Huffman coder / decoder.
// The entropy coder is bit-exact with libjpeg-turbo's jchuff.c for baseline sequential scans.
#include <cstring>

#include "jpeg.h"

namespace uhdr_b200 {

// ---- T.81 Annex K tables (what jpeg_set_defaults installs) ---------------------------------------
static const uint8_t kLumQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                  14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                  18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                  49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
static const uint8_t kChrQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                                  24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
                                  99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                  99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                             12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                             35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                             58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct HuffSpec { uint8_t counts[16]; const uint8_t* symbols; int nsym; };
static const uint8_t kDcSyms[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t kAcLumSyms[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71,
    0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72,
    0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37,
    0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
    0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
    0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3,
    0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
    0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
static const uint8_t kAcChrSyms[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22,
    0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1,
    0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36,
    0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
    0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
    0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a,
    0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
    0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
// index: 0 DC lum, 1 AC lum, 2 DC chr, 3 AC chr
static const HuffSpec kStdHuff[4] = {
    {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, kDcSyms, 12},
    {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d}, kAcLumSyms, 162},
    {{0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}, kDcSyms, 12},
    {{0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}, kAcChrSyms, 162}};

// packed (code << 8 | length) per symbol; shared with huffman.cu through jpeg_std_codebook()
struct Codebook { uint32_t e[256]; };
static Codebook make_codebook(const HuffSpec& s) {
  Codebook cb;
  memset(&cb, 0, sizeof cb);
  uint32_t code = 0;
  int k = 0;
  for (int len = 1; len <= 16; len++) {
    for (int i = 0; i < s.counts[len - 1]; i++, k++) cb.e[s.symbols[k]] = (code++ << 8) | (uint32_t)len;
    code <<= 1;
  }
  return cb;
}
void jpeg_std_codebook(int which, uint32_t out[256]) {
  Codebook cb = make_codebook(kStdHuff[which]);
  memcpy(out, cb.e, sizeof cb.e);
}

void jpeg_quality_tables(int quality, uint16_t lum[64], uint16_t chr[64]) {
  // jcparam.c: jpeg_quality_scaling + jpeg_add_quant_table(force_baseline = TRUE)
  quality = quality <= 0 ? 1 : (quality > 100 ? 100 : quality);
  const long scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
  auto scaled = [scale](int base) {
    long v = (base * scale + 50) / 100;
    return (uint16_t)(v < 1 ? 1 : (v > 255 ? 255 : v));
  };
  for (int i = 0; i < 64; i++) {
    lum[i] = scaled(kLumQ[i]);
    chr[i] = scaled(kChrQ[i]);
  }
}

static int cdiv(int a, int b) { return (a + b - 1) / b; }

void jpeg_frame_finish(JpegFrame* f) {
  f->max_h = f->max_v = 1;
  for (int c = 0; c < f->ncomp; c++) {
    if (f->comp[c].h_samp > f->max_h) f->max_h = f->comp[c].h_samp;
    if (f->comp[c].v_samp > f->max_v) f->max_v = f->comp[c].v_samp;
  }
  for (int c = 0; c < f->ncomp; c++) {
    JpegComp& k = f->comp[c];
    k.width = cdiv(f->width * k.h_samp, f->max_h);
    k.height = cdiv(f->height * k.v_samp, f->max_v);
    k.wblocks = cdiv(f->width * k.h_samp, f->max_h * 8);
    k.hblocks = cdiv(f->height * k.v_samp, f->max_v * 8);
  }
  if (f->ncomp == 1) {
    f->mcus_per_row = f->comp[0].wblocks;
    f->mcu_rows = f->comp[0].hblocks;
  } else {
    f->mcus_per_row = cdiv(f->width, f->max_h * 8);
    f->mcu_rows = cdiv(f->height, f->max_v * 8);
  }
}

bool JpegFrame::has_dummy_blocks() const {
  if (ncomp == 1) return false;
  for (int c = 0; c < ncomp; c++)
    if (mcus_per_row * comp[c].h_samp != comp[c].wblocks || mcu_rows * comp[c].v_samp != comp[c].hblocks)
      return true;
  return false;
}

int jpeg_frame_init(JpegFrame* f, int fmt, int width, int height, int quality) {
  *f = JpegFrame();
  f->width = width;
  f->height = height;
  int hs = 1, vs = 1;
  switch (fmt) {  // sampling table jpegencoderhelper.cpp:26-43
    case F_Y400: f->ncomp = 1; break;
    case F_YUV420: f->ncomp = 3; hs = 2; vs = 2; break;
    case F_YUV422: f->ncomp = 3; hs = 2; break;
    case F_YUV444: case F_RGB888: f->ncomp = 3; break;
    default: return fail(E_INVALID_PARAM, "unrecognized input format %d", fmt);
  }
  for (int c = 0; c < f->ncomp; c++) {
    f->comp[c].h_samp = c == 0 ? hs : 1;
    f->comp[c].v_samp = c == 0 ? vs : 1;
    f->comp[c].tq = c == 0 ? 0 : 1;
  }
  jpeg_quality_tables(quality, f->qt[0], f->qt[1]);
  jpeg_frame_finish(f);
  return E_OK;
}

const char* jpeg_gainmap_comment() {
  // jpegencoderhelper.cpp:205-211 with UHDR_LIB_VERSION_STR 2.0.2 and libjpeg-turbo's default
  // JPEG_LIB_VERSION 62
  return "Source: google libuhdr v2.0.2, Coder: libjpeg v62, Attrib: GainMap Image";
}

// ---- marker layer (jcmarker.c order: SOI, JFIF, [APP2], [COM], DQT.., SOF0, DHT.., SOS) ----------
namespace {
void put_dht(ByteSink& o, int cls_id, const HuffSpec& s) {
  o.u16(0xFFC4);
  o.u16(2 + 1 + 16 + s.nsym);
  o.u8(cls_id);
  o.raw(s.counts, 16);
  o.raw(s.symbols, s.nsym);
}
}  // namespace

// upper bound of what write_headers emits next to the ICC payload and the comment text: SOI 2, JFIF 18, APP2 and
// COM marker headers 8, two DQT 138, SOF0 19, four DHT 432, SOS 14
constexpr size_t kJpegHeadFixedBytes = 640;
size_t jpeg_head_capacity(size_t icc_size, const char* comment) { return kJpegHeadFixedBytes + icc_size + (comment ? strlen(comment) : 0); }

static void write_headers(const JpegFrame& f, const void* icc, size_t icc_size, const char* comment, ByteSink& o) {
  o.u16(0xFFD8);
  static const uint8_t jfif[16] = {0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  o.u16(0xFFE0);
  o.raw(jfif, sizeof jfif);
  if (icc && icc_size) {
    o.u16(0xFFE2);
    o.u16((unsigned)icc_size + 2);
    o.raw(icc, icc_size);
  }
  if (comment) {
    const size_t n = strlen(comment);
    o.u16(0xFFFE);
    o.u16((unsigned)n + 2);
    o.raw(comment, n);
  }
  for (int t = 0; t < (f.ncomp > 1 ? 2 : 1); t++) {
    o.u16(0xFFDB);
    o.u16(67);
    o.u8(t);
    for (int i = 0; i < 64; i++) o.u8(f.qt[t][kZigzag[i]]);
  }
  o.u16(0xFFC0);
  o.u16(8 + 3 * f.ncomp);
  o.u8(8);
  o.u16(f.height);
  o.u16(f.width);
  o.u8(f.ncomp);
  for (int c = 0; c < f.ncomp; c++) {
    o.u8(c + 1);
    o.u8((f.comp[c].h_samp << 4) | f.comp[c].v_samp);
    o.u8(f.comp[c].tq);
  }
  put_dht(o, 0x00, kStdHuff[0]);
  put_dht(o, 0x10, kStdHuff[1]);
  if (f.ncomp > 1) {
    put_dht(o, 0x01, kStdHuff[2]);
    put_dht(o, 0x11, kStdHuff[3]);
  }
  o.u16(0xFFDA);
  o.u16(6 + 2 * f.ncomp);
  o.u8(f.ncomp);
  for (int c = 0; c < f.ncomp; c++) {
    o.u8(c + 1);
    o.u8(c == 0 ? 0x00 : 0x11);
  }
  o.u8(0);
  o.u8(63);
  o.u8(0);
}

// (There is no host entropy coder: every stream is coded by huffman.cu on the device.)

int jpeg_finish_stream(const JpegEncodeJob& job, const void* icc, size_t icc_size, const char* comment,
                       std::vector<uint8_t>* out) {
  if (!job.h_scan_bytes) return fail(E_ERROR, "jpeg_finish_stream called before the device entropy coder ran");
  out->resize(jpeg_head_capacity(icc_size, comment) + job.h_scan_bytes[3] + 2);
  size_t n = 0;
  const int rc = jpeg_finish_stream_into(job, icc, icc_size, comment, out->data(), out->size(), &n);
  if (rc) return rc;
  out->resize(n);
  return E_OK;
}

// device entropy path, caller storage (workspace arena): SOI .. EOI into `out`
int jpeg_finish_stream_into(const JpegEncodeJob& job, const void* icc, size_t icc_size, const char* comment, uint8_t* out,
                            size_t cap, size_t* out_size) {
  if (!job.h_scan_bytes || job.h_scan_bytes[4] || !job.h_scan)
    return fail(E_MEM, "entropy-coded segment exceeds the device scan buffer (%zu bytes)", job.scan_capacity);
  ByteSink o(out, cap);
  write_headers(job.frame, icc, icc_size, comment, o);
  o.raw(job.h_scan, job.h_scan_bytes[3]);
  o.u16(0xFFD9);
  if (!o.ok()) return fail(E_MEM, "JPEG stream of %zu bytes does not fit its %zu-byte buffer", o.size(), cap);
  *out_size = o.size();
  return E_OK;
}

int jpeg_stream_pieces(const JpegEncodeJob& job, const void* icc, size_t icc_size, const char* comment, uint8_t* head,
                       size_t head_cap, size_t* head_len, const uint8_t** scan, size_t* scan_len) {
  if (!job.h_scan_bytes || job.h_scan_bytes[4] || !job.h_scan)
    return fail(E_MEM, "entropy-coded segment exceeds the device scan buffer (%zu bytes)", job.scan_capacity);
  ByteSink o(head, head_cap);
  write_headers(job.frame, icc, icc_size, comment, o);
  if (!o.ok()) return fail(E_ERROR, "JPEG header of %zu bytes exceeds its bound of %zu", o.size(), head_cap);
  *head_len = o.size();
  *scan = job.h_scan;
  *scan_len = job.h_scan_bytes[3];
  return E_OK;
}

// ---- decoder: marker parser (jdmarker.c subset) + Huffman decoder (jdhuff.c semantics) ----------
// jdhuff.c jpeg_make_d_derived_tbl's sanity checks, applied to the tables a scan refers to: the
// code lengths must describe a prefix code, and a DC table may only hold categories 0..15
// (libjpeg: JERR_BAD_HUFF_TABLE, "Bogus Huffman table definition")
static bool huff_table_ok(const uint8_t bits[17], const uint8_t* vals, bool is_dc) {
  long code = 0;
  int total = 0;
  for (int len = 1; len <= 16; len++) {
    code += bits[len];
    total += bits[len];
    if (bits[len] && code >= (1L << len)) return false;   // the all-ones code of a length is reserved
    code <<= 1;
  }
  if (total > 256) return false;
  if (is_dc)
    for (int i = 0; i < total; i++)
      if (vals[i] > 15) return false;
  return true;
}

int jpeg_read_header(const uint8_t* d, size_t n, JpegHeader* h) {
  *h = JpegHeader();
  memset(h->bits, 0, sizeof h->bits);
  if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return fail(E_ERROR, "Not a JPEG file: starts with 0x%02x 0x%02x", n > 0 ? d[0] : 0, n > 1 ? d[1] : 0);
  size_t p = 2;
  bool sof = false;
  while (p + 4 <= n) {
    if (d[p] != 0xFF) return fail(E_ERROR, "corrupt JPEG data: expected a marker at offset %zu", p);
    while (p < n && d[p] == 0xFF) p++;
    if (p >= n) break;
    const uint8_t m = d[p++];
    if (m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;
    if (m == 0xD9) break;
    if (p + 2 > n) break;
    const size_t len = ((size_t)d[p] << 8) | d[p + 1];
    if (len < 2 || p + len > n) return fail(E_ERROR, "corrupt JPEG data: bad marker length at offset %zu", p);
    const uint8_t* s = d + p + 2;
    const size_t sl = len - 2;
    if (m >= 0xE0 && m <= 0xE2) {
      h->markers.push_back({m, p + 2, sl});
      if (m == 0xE0 && sl >= 5 && !memcmp(s, "JFIF", 5)) h->jfif = 1;
    } else if (m == 0xEE && sl >= 12 && !memcmp(s, "Adobe", 5)) {
      h->adobe_transform = s[11];
    } else if (m == 0xDB) {
      for (size_t i = 0; i < sl;) {
        const int prec = s[i] >> 4, id = s[i] & 15;
        i++;
        if (id > 1 || i + (prec ? 128u : 64u) > sl) return fail(E_UNSUPPORTED, "unsupported DQT (id %d)", id);
        for (int k = 0; k < 64; k++) {
          h->frame.qt[id][kZigzag[k]] = prec ? (uint16_t)((s[i] << 8) | s[i + 1]) : s[i];
          i += prec ? 2 : 1;
        }
      }
    } else if (m == 0xC0 || m == 0xC1) {
      if (sl < 6 || s[0] != 8) return fail(E_UNSUPPORTED, "Unsupported JPEG data precision %d", sl ? s[0] : 0);
      JpegFrame& f = h->frame;
      f.height = (s[1] << 8) | s[2];
      f.width = (s[3] << 8) | s[4];
      f.ncomp = s[5];
      if ((f.ncomp != 1 && f.ncomp != 3) || sl < 6 + 3u * f.ncomp) {
        if (f.ncomp != 1 && f.ncomp != 3) { sof = true; p += len; continue; }  // reported by caller
        return fail(E_ERROR, "corrupt SOF marker");
      }
      for (int c = 0; c < f.ncomp; c++) {
        h->comp_id[c] = s[6 + 3 * c];
        f.comp[c].h_samp = s[7 + 3 * c] >> 4;
        f.comp[c].v_samp = s[7 + 3 * c] & 15;
        f.comp[c].tq = s[8 + 3 * c];
        if (f.comp[c].tq > 1) return fail(E_UNSUPPORTED, "quantization table %d not supported", f.comp[c].tq);
      }
      sof = true;
    } else if (m == 0xC2 || m == 0xC3 || (m >= 0xC5 && m <= 0xCF && m != 0xC8 && m != 0xCC)) {
      return fail(E_UNSUPPORTED, "Unsupported JPEG process: SOF type 0x%02x", m);
    } else if (m == 0xC4) {
      for (size_t i = 0; i + 17 <= sl;) {
        const int cls = s[i] >> 4, id = s[i] & 15;
        if (cls > 1 || id > 1) return fail(E_UNSUPPORTED, "Huffman table 0x%02x not supported", s[i]);
        int cnt = 0;
        for (int k = 1; k <= 16; k++) cnt += (h->bits[cls][id][k] = s[i + k]);
        i += 17;
        if (cnt > 256 || i + cnt > sl) return fail(E_ERROR, "corrupt DHT marker");
        memcpy(h->vals[cls][id], s + i, cnt);
        i += cnt;
        h->have_tbl[cls][id] = true;
      }
    } else if (m == 0xDD) {
      if (sl >= 2) h->restart_interval = (s[0] << 8) | s[1];
    } else if (m == 0xDA) {
      JpegFrame& f = h->frame;
      if (!sof) return fail(E_ERROR, "SOS before SOF");
      if (f.ncomp != 1 && f.ncomp != 3) { h->scan_offset = p + len; return E_OK; }
      if (sl < 1 || s[0] != f.ncomp || sl < 1 + 2u * s[0] + 3)
        return fail(E_UNSUPPORTED, "multi-scan JPEG streams are not supported");
      if (f.ncomp == 1) f.comp[0].h_samp = f.comp[0].v_samp = 1;
      jpeg_frame_finish(&f);
      for (int c = 0; c < f.ncomp; c++) {
        if (s[1 + 2 * c] != h->comp_id[c]) return fail(E_UNSUPPORTED, "unexpected component order in SOS");
        h->dc_sel[c] = s[2 + 2 * c] >> 4;
        h->ac_sel[c] = s[2 + 2 * c] & 15;
        if (h->dc_sel[c] > 1 || h->ac_sel[c] > 1 || !h->have_tbl[0][h->dc_sel[c]] || !h->have_tbl[1][h->ac_sel[c]])
          return fail(E_ERROR, "Huffman table was not defined");
        if (!huff_table_ok(h->bits[0][h->dc_sel[c]], h->vals[0][h->dc_sel[c]], true) ||
            !huff_table_ok(h->bits[1][h->ac_sel[c]], h->vals[1][h->ac_sel[c]], false))
          return fail(E_ERROR, "Bogus Huffman table definition");
      }
      // libjpeg derives decoding tables lazily, for the tables a scan selects only: a malformed table
      // nobody refers to is legal input.  Forget such tables here so that no table builder (host or
      // device) ever sees code lengths that do not describe a prefix code.
      for (int cls = 0; cls < 2; cls++)
        for (int id = 0; id < 2; id++)
          if (h->have_tbl[cls][id] && !huff_table_ok(h->bits[cls][id], h->vals[cls][id], cls == 0)) {
            h->have_tbl[cls][id] = false;
            memset(h->bits[cls][id], 0, sizeof h->bits[cls][id]);
          }
      h->scan_offset = p + len;
      return E_OK;
    }
    p += len;
  }
  return fail(E_ERROR, "JPEG datastream contains no image");
}

namespace {
struct DecodeTable {
  uint16_t fast[1 << 10];  // (len << 8) | symbol for codes up to 10 bits, 0 = long code
  int maxcode[18];
  int valptr[17];
  const uint8_t* vals;
  void build(const uint8_t bits[17], const uint8_t* v) {
    memset(fast, 0, sizeof fast);
    vals = v;
    int code = 0, k = 0;
    for (int len = 1; len <= 16; len++) {
      valptr[len] = k - code;
      for (int i = 0; i < bits[len]; i++, k++, code++)
        if (len <= 10 && code < (1 << len) && k < 256)  // guards: never index past `fast` / `v` whatever the lengths say
          for (int r = 0; r < (1 << (10 - len)); r++) fast[(code << (10 - len)) | r] = (uint16_t)((len << 8) | v[k]);
      maxcode[len] = bits[len] ? code - 1 : -1;
      code <<= 1;
    }
    maxcode[17] = 0x7fffffff;
  }
};
struct BitSource {
  const uint8_t* d;
  size_t p, n;
  uint64_t acc = 0;
  int fill = 0;
  bool marker = false;
  void refill() {
    while (fill <= 56) {
      unsigned b = 0;
      if (!marker && p < n) {
        b = d[p];
        if (b == 0xFF) {
          if (p + 1 < n && d[p + 1] == 0) p += 2;
          else { marker = true; b = 0; }
        } else {
          p++;
        }
      }
      acc = (acc << 8) | b;
      fill += 8;
    }
  }
  unsigned peek(int k) { if (fill < k) refill(); return (unsigned)(acc >> (fill - k)) & ((1u << k) - 1u); }
  void drop(int k) { fill -= k; }
  unsigned take(int k) { unsigned v = peek(k); fill -= k; return v; }
};
inline int decode_symbol(BitSource& bs, const DecodeTable& t) {
  const unsigned e = t.fast[bs.peek(10)];
  if (e) { bs.drop(e >> 8); return e & 0xff; }
  const unsigned w = bs.peek(16);
  for (int len = 11; len <= 16; len++) {
    const int code = (int)(w >> (16 - len));
    if (code <= t.maxcode[len]) { bs.drop(len); return t.vals[(code + t.valptr[len]) & 0xff]; }
  }
  bs.drop(16);
  return 0;
}
inline int sign_extend(unsigned v, int nb) { return v < (1u << (nb - 1)) ? (int)v - (1 << nb) + 1 : (int)v; }
}  // namespace

int jpeg_host_decode_coefs(const uint8_t* data, size_t size, const JpegHeader& h, int16_t* coefs[3]) {
  const JpegFrame& f = h.frame;
  DecodeTable dct[2], act[2];
  for (int i = 0; i < 2; i++) {
    if (h.have_tbl[0][i]) dct[i].build(h.bits[0][i], h.vals[0][i]);
    if (h.have_tbl[1][i]) act[i].build(h.bits[1][i], h.vals[1][i]);
  }
  BitSource bs{data, h.scan_offset, size};
  int pred[3] = {0, 0, 0};
  int16_t sink[64];
  long mcu = 0;
  for (int my = 0; my < f.mcu_rows; my++)
    for (int mx = 0; mx < f.mcus_per_row; mx++, mcu++) {
      if (h.restart_interval && mcu && mcu % h.restart_interval == 0) {
        bs.acc = 0; bs.fill = 0; bs.marker = false;
        while (bs.p + 1 < bs.n && !(bs.d[bs.p] == 0xFF && bs.d[bs.p + 1] >= 0xD0 && bs.d[bs.p + 1] <= 0xD7)) bs.p++;
        bs.p += 2;
        pred[0] = pred[1] = pred[2] = 0;
      }
      for (int c = 0; c < f.ncomp; c++) {
        const JpegComp& k = f.comp[c];
        const int mw = f.ncomp == 1 ? 1 : k.h_samp, mh = f.ncomp == 1 ? 1 : k.v_samp;
        const DecodeTable& dt = dct[h.dc_sel[c]];
        const DecodeTable& at = act[h.ac_sel[c]];
        for (int j = 0; j < mh; j++)
          for (int i = 0; i < mw; i++) {
            const int bx = mx * mw + i, by = my * mh + j;
            int16_t* blk = (bx < k.wblocks && by < k.hblocks) ? coefs[c] + ((size_t)by * k.wblocks + bx) * 64 : sink;
            memset(blk, 0, 128);
            const int s = decode_symbol(bs, dt);
            if (s) pred[c] = (int)((unsigned)pred[c] + (unsigned)sign_extend(bs.take(s), s));  // wraps like the int16 it feeds
            blk[0] = (int16_t)pred[c];
            for (int z = 1; z < 64; z++) {
              const int rs = decode_symbol(bs, at);
              const int r = rs >> 4, sz = rs & 15;
              if (sz) {
                z += r;
                if (z > 63) return fail(E_ERROR, "Corrupt JPEG data: bad Huffman code");
                blk[kZigzag[z]] = (int16_t)sign_extend(bs.take(sz), sz);
              } else {
                if (r != 15) break;
                z += 15;
              }
            }
          }
      }
    }
  return E_OK;
}

int jpeg_scaled_geometry(const JpegFrame& f, int k, JpegScaled* g) {
  if (k != 1 && k != 2 && k != 4 && k != 8) return fail(E_INVALID_PARAM, "scale denominator %d, expects 1, 2, 4 or 8", k);
  *g = JpegScaled();
  g->k = k;
  g->width = (f.width + k - 1) / k;
  g->height = (f.height + k - 1) / k;
  const int m = 8 / k;
  for (int c = 0; c < f.ncomp; c++) {
    const JpegComp& p = f.comp[c];
    int s = m;
    while (s < 8 && (f.max_h * m) % (p.h_samp * s * 2) == 0 && (f.max_v * m) % (p.v_samp * s * 2) == 0) s *= 2;
    g->s[c] = s;
    g->w[c] = (int)(((long long)f.width * p.h_samp * s + f.max_h * 8 - 1) / (f.max_h * 8));
    g->h[c] = (int)(((long long)f.height * p.v_samp * s + f.max_v * 8 - 1) / (f.max_v * 8));
  }
  for (int c = f.ncomp; c < 3; c++) g->s[c] = g->s[0];
  return E_OK;
}

bool JpegScaled::full_chroma() const {
  for (int c = 0; c < 3; c++)
    if (w[c] && (w[c] != width || h[c] != height)) return false;
  return true;
}

}  // namespace uhdr_b200
