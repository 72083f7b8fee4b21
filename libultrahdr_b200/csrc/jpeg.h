// Baseline JPEG codec of libuhdr_b200: the CUDA counterpart of JpegEncoderHelper /
// JpegDecoderHelper (lib/src/jpegencoderhelper.cpp, lib/src/jpegdecoderhelper.cpp), which in the
// reference are thin drivers over libjpeg-turbo.  Block arithmetic (colour conversion, level
// shift, islow FDCT/IDCT, quantise/dequantise) runs in CUDA kernels; entropy coding runs on the device
// (huffman.cu; decoding: huffdec.cu, with a host decoder in jpeg_host.cpp for the streams it declines) and the
// marker layer is host code.  Streams are byte-identical to what libjpeg-turbo emits for the reference's settings
// (jpeg_set_defaults + jpeg_set_quality(q, TRUE), JDCT_ISLOW, default Huffman tables, one
// interleaved scan, no restart markers).
#pragma once
#include <cstddef>
#include <cstdint>

#include "bytes.h"
#include "container.h"
#include "engine.h"

namespace uhdr_b200 {

struct JpegComp {
  int h_samp = 1, v_samp = 1, tq = 0;
  int width = 0, height = 0;     // real plane size
  int wblocks = 0, hblocks = 0;  // padded to whole blocks (libjpeg width_in_blocks)
};
struct JpegFrame {
  int ncomp = 0, width = 0, height = 0, max_h = 1, max_v = 1;
  int mcus_per_row = 0, mcu_rows = 0;
  JpegComp comp[3];
  uint16_t qt[2][64];  // natural order
  size_t blocks(int c) const { return (size_t)comp[c].wblocks * comp[c].hblocks; }
  size_t total_blocks() const { size_t n = 0; for (int c = 0; c < ncomp; c++) n += blocks(c); return n; }
  bool has_dummy_blocks() const;  // interleaved MCUs reaching past a component's block grid
};

extern const uint8_t kZigzag[64];  // zigzag position -> natural index
void jpeg_quality_tables(int quality, uint16_t lum[64], uint16_t chr[64]);
int jpeg_frame_init(JpegFrame* f, int fmt, int width, int height, int quality);
void jpeg_frame_finish(JpegFrame* f);

// ---- encoder -----------------------------------------------------------------------------------
struct JpegEncodeJob {
  JpegFrame frame;
  int16_t* d_coefs[3] = {nullptr, nullptr, nullptr};  // device, [block][64] natural order
  // per block {AC code bits << 16 | DC, first 96 bits of the AC bit string} from the forward stage (zigzag launches only)
  uint4* d_meta[3] = {nullptr, nullptr, nullptr};
  // device-side entropy coding products (huffman.cu)
  uint8_t* d_scan = nullptr;      // stuffed entropy-coded segment
  unsigned* d_scan_bytes = nullptr;
  uint8_t* h_scan = nullptr;      // pinned copy
  unsigned* h_scan_bytes = nullptr;  // pinned control words: [3] = bytes, [4] = overflow flag
  size_t scan_capacity = 0;
  bool zigzag = false;            // d_coefs hold zigzag-ordered blocks
  // the head carries the COM marker the reference writes for gain-map images: RGB888 or Y400 input
  // (jpegencoderhelper.cpp:163-211)
  bool gainmap_comment = false;
};

// Enqueue the block stage for `img` (device image): colour conversion (RGB888 only), level
// shift, FDCT, quantise.  Mirrors JpegEncoderHelper::compressImage's input handling
// (jpegencoderhelper.cpp:131-309) including libjpeg's edge rules.
// rows[c] > 0: the block stage reads rows [0, rows[c]) of plane c from memory (the encoder helper's scratch rows),
// not only those up to the plane height
int jpeg_forward_dev(Workspace& ws, const DevImage& img, int quality, JpegEncodeJob* job, bool zigzag = false,
                     const int* rows = nullptr);
// jpeg_forward_dev without the launch: the job's buffers and the block stage's parameters
int jpeg_forward_plan(Workspace& ws, const DevImage& img, int quality, JpegEncodeJob* job, bool zigzag, const int* rows,
                      Fdct8Params* P);
// Enqueue the entropy coder for a zigzag forward stage, and the copy of its control words to pinned memory.
int jpeg_entropy_dev(Workspace& ws, JpegEncodeJob* job);
// Enqueue a JPEG coded on the device: the zigzag block stage, then the entropy coder.  Every geometry, MCUs that reach
// past the block grid included (huffman.cu codes libjpeg's dummy blocks).
int jpeg_encode_dev(Workspace& ws, const DevImage& img, int quality, JpegEncodeJob* job, const int* rows = nullptr);
// The scans of jobs enqueued by jpeg_encode_dev to pinned memory: one host wait for their sizes, then for each job in
// the order given jpeg_scan_check and the copy of its segment, then one host wait for the copies.
int jpeg_entropy_collect(Workspace& ws, JpegEncodeJob* const* jobs, int n);
// E_MEM, with its message, when the job's segment overflowed its device buffer; its control words are on the host
int jpeg_scan_check(const JpegEncodeJob& job);
// Entropy coding of many JPEGs with one launch (k_huff_encode_batch): each job gets the segment jpeg_entropy_dev gives
// it, one chunk size for all of them.  Enqueued on ws.stream() with one copy of every job's control words to pinned
// memory (job->h_scan_bytes).  jpeg_entropy_batch_fetch, once the stream was synchronised: one launch gathers the
// segments into one buffer and one copy brings it to pinned memory (job->h_scan; null for a scan that overflowed).
int jpeg_entropy_batch_dev(Workspace& ws, JpegEncodeJob* const* jobs, int n);
int jpeg_entropy_batch_fetch(Workspace& ws, JpegEncodeJob* const* jobs, int n);
// since process start: [0] k_huff_encode_batch launches, [1] scans they coded
void jpeg_encode_batch_stats(unsigned long long out[2]);
// k_huff_encode plans since process start: [0] resident CTAs per wave, [1..8] launches by blocks per thread,
// [9] launches whose grid exceeded one wave
void jpeg_encode_stats(unsigned long long out[10]);
// The head of a job's JPEG, SOI .. SOS header in jcmarker.c's order (JFIF, `icc` as APP2, the gain-map COM marker when
// job.gainmap_comment, DQT, SOF0, DHT, SOS), into `o`.  At most kJpegHeadBytes + icc_size bytes: SOI 2, JFIF 18, APP2
// and COM marker headers 8, the 72-byte comment, two DQT 138, SOF0 19, four DHT 432, SOS 14.
constexpr size_t kJpegHeadBytes = 720;
void jpeg_write_headers(const JpegEncodeJob& job, const void* icc, size_t icc_size, ByteSink& o);
// The JPEG of a job whose scan is on the host (jpeg_entropy_collect, or jpeg_entropy_batch_fetch and jpeg_scan_check):
// its head written into the workspace's pinned arena, and its entropy-coded segment where the device's copy left it.
// No copy of the segment is made.
int jpeg_stream_pieces(Workspace& ws, const JpegEncodeJob& job, const void* icc, size_t icc_size, JpegPieces* out);

// ---- decoder -----------------------------------------------------------------------------------
struct JpegMarker { uint8_t id; size_t offset, length; };
// APPn markers of a header in stream order; fixed capacity (no heap): the first kMax are kept, which is more than
// any writer emits ahead of SOS (the look-ups below want the first EXIF / ICC / XMP / ISO / MPF marker)
struct JpegMarkerList {
  static constexpr int kMax = 48;
  JpegMarker v[kMax];
  int n = 0;
  void push_back(const JpegMarker& m) { if (n < kMax) v[n++] = m; }
  void clear() { n = 0; }
  const JpegMarker* begin() const { return v; }
  const JpegMarker* end() const { return v + n; }
  size_t size() const { return (size_t)n; }
};
struct JpegHeader {
  JpegFrame frame;
  int comp_id[3] = {0, 0, 0};
  int restart_interval = 0;
  size_t scan_offset = 0;
  JpegMarkerList markers;  // APP0..APP2 in stream order
  uint8_t bits[2][2][17];
  uint8_t vals[2][2][256];
  bool have_tbl[2][2] = {{false, false}, {false, false}};
  int dc_sel[3] = {0, 0, 0}, ac_sel[3] = {0, 0, 0};
  int jfif = 0, adobe_transform = -1;
};
int jpeg_read_header(const uint8_t* data, size_t size, JpegHeader* h);
// entropy-decode into [block][64] natural-order coefficient arrays (host)
int jpeg_host_decode_coefs(const uint8_t* data, size_t size, const JpegHeader& h, int16_t* coefs[3]);
// Reduced-size decoding, libjpeg's scale_num = 1, scale_denom = k (jdmaster.c): the output is ceil(W/k) x ceil(H/k).
// Every component starts at a DCT scaled size of 8/k samples per block side, doubled while that is < 8 and the
// sampling factors allow it (chroma is scaled up by the IDCT, not by an upsampler): a 4:2:0 frame comes out 4:4:4.
// Component c is w[c] x h[c] = ceil(W*h_samp*s / (max_h*8)) x ceil(H*v_samp*s / (max_v*8)).
struct JpegScaled {
  int k = 1, width = 0, height = 0;
  int s[3] = {8, 8, 8}, w[3] = {0, 0, 0}, h[3] = {0, 0, 0};
  bool full_chroma() const;  // every component at the output size (gray, 4:4:4, 4:2:0 at k > 1)
};
// E_INVALID_PARAM for k outside {1, 2, 4, 8}
int jpeg_scaled_geometry(const JpegFrame& f, int k, JpegScaled* g);
// Dequant + IDCT (idct.cu).  Component c of a decode comes out at DCT scaled size s (8 at full size, JpegScaled::s[c]
// at 1/k): hblocks*s rows of wblocks*s samples at its plane's stride, clipped to the stride at s = 8.
// Pinned room in the workspace's arena for n planes of an IDCT launch and their CTA ends
IdctPlane* jpeg_idct_stage(Workspace& ws, int n);
// Adds to p the output of component c of frame f at size s into dst at `stride`; the plane's first output (p->nout = 0)
// also sets its coefficients (device, [block][64] natural order), quantiser and block counts
void jpeg_idct_plane(IdctPlane* p, const JpegFrame& f, int c, const int16_t* coefs, int s, uint8_t* dst, int stride);
// One JPEG of an inverse DCT: g null for the full size, else the geometry of its 1/k decode
struct JpegIdctJob {
  const JpegHeader* h;
  const JpegScaled* g;
  int16_t* d_coefs[3];
  uint8_t* planes[3];
  int strides[3];
};
// Every plane of every job, enqueued on ws.stream(): one copy of the planes to the device, then one k_idct<s> launch per
// size s for all of them
int jpeg_idct_dev(Workspace& ws, const JpegIdctJob* jobs, int n);
// One k_idct<0> launch over planes[0, n) of a jpeg_idct_stage, after one copy to the device: each plane's coefficients
// are read once and written at every size its outputs ask for
int jpeg_idct_multi_dev(Workspace& ws, IdctPlane* planes, int n);
// Entropy decoding (huffdec.cu) of one or many JPEGs: one relaxation over the subsequences of every scan (one host
// check per batch of rounds for all of them), then one writing pass and one DC pass.  A scan the device decoder
// declines (irregular restart markers, no fixed point, inconsistent data), and every scan while the host decoder is
// selected, goes to jpeg_host_decode_coefs by itself; that decoder also produces the reference's error texts.
// Enqueued on ws.stream(), the last copies may still be in flight.  Returns an error only for what fails the whole
// call (CUDA, memory); a corrupt scan gets its code in rc.
struct JpegScanJob {
  const uint8_t* data;
  size_t size;
  const JpegHeader* h;
  int16_t* d_coefs[3];  // out: [block][64] natural order, from the workspace
  int rc;               // out: E_OK, or the error decoding this scan gives (its message in err)
  char err[256];
};
int jpeg_entropy_decode_dev(Workspace& ws, JpegScanJob* scans, int n);
// 0 = default = 2 = device whenever the stream allows (host only for streams the device decoder declines), 1 = host (tests, triage)
// [0] scans decoded on the device, [1] scans handed back to the host decoder, [2] relaxation rounds of the last one
void jpeg_entropy_decoder_stats(unsigned long long out[3]);
void jpeg_set_entropy_decoder(int mode);
int jpeg_get_entropy_decoder();

}  // namespace uhdr_b200
