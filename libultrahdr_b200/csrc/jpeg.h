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
#include <string>
#include <vector>

#include "bytes.h"
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
  // device-side entropy coding products (huffman.cu); null when the host path is used
  uint8_t* d_scan = nullptr;      // stuffed entropy-coded segment
  unsigned* d_scan_bytes = nullptr;
  uint8_t* h_scan = nullptr;      // pinned copy
  unsigned* h_scan_bytes = nullptr;  // pinned control words: [3] = bytes, [4] = overflow flag
  size_t scan_capacity = 0;
  bool zigzag = false;            // d_coefs hold zigzag-ordered blocks
};

// Enqueue the block stage for `img` (device image): colour conversion (RGB888 only), level
// shift, FDCT, quantise.  Mirrors JpegEncoderHelper::compressImage's input handling
// (jpegencoderhelper.cpp:131-309) including libjpeg's edge rules.
int jpeg_forward_dev(Workspace& ws, const DevImage& img, int quality, JpegEncodeJob* job, bool zigzag = false);
// Enqueue entropy coding on the device + async copy of the scan to pinned memory.
int jpeg_entropy_dev(Workspace& ws, JpegEncodeJob* job);
// second phase, once the stream was synchronised and the sizes are on the host
int jpeg_entropy_fetch(Workspace& ws, JpegEncodeJob* job);
// After stream sync: assemble SOI..EOI.  `comment` != nullptr adds the COM marker the reference
// writes for gain-map images (jpegencoderhelper.cpp:205-211).
int jpeg_finish_stream(const JpegEncodeJob& job, const void* icc, size_t icc_size,
                       const char* comment, std::vector<uint8_t>* out);
// The same for the device entropy path into storage the caller owns (no heap): `cap` >= jpeg_head_capacity() +
// the segment's bytes + 2.
size_t jpeg_head_capacity(size_t icc_size, const char* comment);
int jpeg_finish_stream_into(const JpegEncodeJob& job, const void* icc, size_t icc_size, const char* comment, uint8_t* out,
                            size_t cap, size_t* out_size);
// Head (SOI .. SOS header) only, into `head` (capacity jpeg_head_capacity()), and the entropy-coded segment as a
// pointer into the pinned buffer the device wrote it to.  No copy of the segment is made.
int jpeg_stream_pieces(const JpegEncodeJob& job, const void* icc, size_t icc_size, const char* comment, uint8_t* head,
                       size_t head_cap, size_t* head_len, const uint8_t** scan, size_t* scan_len);

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
// Enqueue H2D of coefficients + dequant/IDCT into device planes (stride = wblocks*8).
int jpeg_inverse_dev(Workspace& ws, const JpegHeader& h, int16_t* const h_coefs[3],
                     uint8_t* d_planes[3], int plane_stride[3]);
// Same, coefficients already on the device.
int jpeg_idct_dev(Workspace& ws, const JpegHeader& h, int16_t* const d_coefs[3], uint8_t* d_planes[3], int plane_stride[3]);
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
// Dequant + IDCT at the scaled sizes: components of size 8 through k_idct_dequant, the others through the reduced
// IDCT (one launch per size).  Plane c holds hblocks*s[c] rows of wblocks*s[c] samples at plane_stride[c].
int jpeg_idct_scaled_dev(Workspace& ws, const JpegHeader& h, const JpegScaled& g, int16_t* const d_coefs[3],
                         uint8_t* d_planes[3], int plane_stride[3]);
// Same, coefficients decoded on the host.
int jpeg_inverse_scaled_dev(Workspace& ws, const JpegHeader& h, const JpegScaled& g, int16_t* const h_coefs[3],
                            uint8_t* d_planes[3], int plane_stride[3]);
// Entropy decoding on the device (huffdec.cu): fills d_coefs[c] (allocated from the workspace) with
// [block][64] natural-order coefficients.  Returns kHuffDecFallback when the stream is outside what
// the parallel decoder handles (restart markers, no fixed point, inconsistent data): the caller then
// runs jpeg_host_decode_coefs, which also produces the reference's error texts.
constexpr int kHuffDecFallback = -1000;
int jpeg_entropy_decode_dev(Workspace& ws, const uint8_t* data, size_t size, const JpegHeader& h, int16_t* d_coefs[3]);
// 0 = default = 2 = device whenever the stream allows (host only for streams the device decoder declines), 1 = host (tests, triage)
// [0] scans decoded on the device, [1] scans handed back to the host decoder, [2] relaxation rounds of the last one
void jpeg_entropy_decoder_stats(unsigned long long out[3]);
void jpeg_set_entropy_decoder(int mode);
int jpeg_get_entropy_decoder();

const char* jpeg_gainmap_comment();

}  // namespace uhdr_b200
