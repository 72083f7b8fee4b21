// Codec orchestration: the CUDA counterpart of ultrahdr::JpegR (lib/include/ultrahdr/jpegr.h:52-222).
// encodeJPEGR API-0 / API-1 and decodeJPEGR run their pixel and block stages on the device;
// the marker/container layer is host code.
#pragma once
#include <condition_variable>
#include <cstdio>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "container.h"
#include "effects.h"
#include "engine.h"
#include "jpeg.h"

namespace uhdr_b200 {

struct DecodedInfo {
  int width = 0, height = 0, gm_width = 0, gm_height = 0, gm_channels = 0;
  ByteView exif, icc;   // views into the probed stream (the caller keeps it alive: the C API handle owns a copy)
  size_t base_off = 0, base_len = 0, gainmap_off = 0, gainmap_len = 0;  // the two JPEGs inside the probed stream
  uhdr_gainmap_metadata_t metadata{};
  bool has_metadata = false;
};

// decode_jpeg_dev between its stages (codec.cu): the resolved mode, the scale and the output planes
struct JpegDecodeJob {
  int mode = 0, k = 1;
  JpegScaled g;
  uint8_t* planes[3] = {nullptr, nullptr, nullptr};
  int strides[3] = {0, 0, 0};
};

// One JPEG/R file of a batched call (decode_batch, transcode_batch).  The caller fills the first group of fields;
// rc != E_OK on entry skips the file.
struct BatchFile {
  const uint8_t* data = nullptr;
  size_t size = 0;
  DecodedInfo info;  // probe() of the file
  bool want_map = true;   // the gain-map JPEG is decoded too
  int rc = 0;        // out: the code the single call gives for this file alone, its message in err
  char err[256] = {0};
  // the two JPEGs' decode between its batched stages (JpegRCodec::decode_batch_files)
  JpegHeader ph, gh;
  JpegDecodeJob pj, gj;
  DevImage sdr{}, map{};
  YccToRgbaParams to_rgba{};   // the primary's colour conversion when decode_batch_files defers it
  int map_rc = 0;    // an error of the gain-map JPEG's header stage, returned after the primary image's own
  char map_err[256] = {0};
};

// the file's code and message: it drops out of the rest of the batch
inline void batch_fail(BatchFile& f, int rc, const char* msg) {
  f.rc = rc;
  snprintf(f.err, sizeof f.err, "%s", msg);
}

// One file of JpegRCodec::decode_batch: the decode() outputs
struct DecodeBatchItem : BatchFile {
  uhdr_raw_image_t* dest = nullptr;
  uhdr_raw_image_t* gainmap = nullptr;
  uhdr_gainmap_metadata_t* md_out = nullptr;
};

// One output of JpegRCodec::transcode_batch (a file) or transcode_ladders (a rung): the transcode() settings and output,
// and the two encodes between their batched stages
struct TranscodeBatchItem : BatchFile {
  uhdr_b200_transcode_config_t cfg{};
  uint8_t* out = nullptr;
  size_t cap = 0;
  size_t out_size = 0;  // out: what transcode() sets
  JpegEncodeJob base_jpeg, gm_jpeg;
};

// decode_jpeg_dev's stages (codec.cu): up to the entropy decoding (the header, its checks, the output planes), and after
// the inverse DCT (the colour conversion of mode 1, or the planes' format of mode 0)
int decode_jpeg_begin(Workspace& ws, const uint8_t* data, size_t size, int mode, int k, DevImage* out, JpegHeader* h,
                      JpegDecodeJob* j);
int decode_jpeg_end(Workspace& ws, const JpegHeader* h, const JpegDecodeJob& j, DevImage* out, YccToRgbaParams* to_rgba);
// decode_jpeg_begin's part after the header: the checks and output planes of a decode at 1/k
int decode_jpeg_plan(Workspace& ws, const JpegHeader& h, int mode, int k, DevImage* out, JpegDecodeJob* j);

// the most rungs of one file of transcode_ladders, and the most distinct (base_quality, gainmap_quality) pairs of one of
// its groups: it bounds the host plan of transcode_encode
constexpr int kLadderMaxRungs = 16;

// One file of JpegRCodec::transcode_ladders.  The caller fills the first group of fields; rc != E_OK on entry (the
// file's own argument error) skips the file.
struct LadderFile {
  const uint8_t* data = nullptr;
  DecodedInfo info;  // probe() of the file
  int r0 = 0, nr = 0;   // its rungs: [r0, r0 + nr) of the call's rung array, one file after the other
  int rc = 0;        // the entry points' own: the file's argument error, or what the ladder returns, with its message
  char err[300] = {0};
  // decode_ladders' state: both headers, the scans' indices in the group's entropy decoding (-1: not decoded), and per
  // distinct k of the valid rungs both JPEGs' plans at 1/k and the code transcode() gives at that k once decoded
  JpegHeader ph, gh;
  int ps = -1, gs = -1, nk = 0;
  struct K {
    int k, rc, map_rc;
    char err[256], map_err[256];
    JpegDecodeJob pj, gj;
    DevImage sdr, map;
  } ks[4];
};

// One parked host thread per codec (spawned on first use, kept until the codec dies): runs the gain-map JPEG of a
// decode next to the primary one without creating a thread per call.
class ParkedThread {
 public:
  ~ParkedThread();
  void start(void (*fn)(void*), void* arg);   // fn(arg) on the parked thread
  void wait();                                // until that call has returned
 private:
  void loop();
  std::thread th_;
  std::mutex mu_;
  std::condition_variable cv_;
  void (*fn_)(void*) = nullptr;
  void* arg_ = nullptr;
  bool busy_ = false, quit_ = false;
};

class JpegRCodec {
 public:
  int init() { return ws_.init(); }
  Workspace& ws() { return ws_; }

  // JpegR::encodeJPEGR API-1 (jpegr.cpp:247-291) when sdr_dev != nullptr, API-0 (:179-244)
  // otherwise.  Inputs are device images previously uploaded on ws().stream(), or with `caller_planes` a caller's
  // device planes (any pitch, element alignment, undefined bytes past the width: see block_stage_input).
  int encode(const DevImage& hdr, const DevImage* sdr, const uhdr_b200_gm_config_t& cfg, int base_quality,
             const uint8_t* exif, size_t exif_size, uint8_t* out, size_t cap, size_t* out_size,
             bool caller_planes = false);
  // JpegR::encodeJPEGR API-2 (jpegr.cpp:294-324, sdr != nullptr) / API-3 (:326-386, the compressed SDR is
  // decoded on the device and the map is computed with BT.601 luma): gain map from the intents, its JPEG,
  // appended to the caller's compressed SDR image.  `sdr_jpg_cg`: gamut of the compressed image when it
  // carries no ICC profile.
  int encode_with_compressed_sdr(const DevImage& hdr, const DevImage* sdr, const uint8_t* sdr_jpg, size_t sdr_jpg_size,
                                 int sdr_jpg_cg, const uhdr_b200_gm_config_t& cfg, uint8_t* out, size_t cap, size_t* out_size);
  // API-4 (:388-434): container work only, no device
  static int encode_from_compressed(const uint8_t* base, size_t base_size, int base_cg, const uint8_t* gainmap, size_t gainmap_size,
                                    const uhdr_gainmap_metadata_t& md, uint8_t* out, size_t cap, size_t* out_size);
  // convenience: host descriptors
  int encode_host(const uhdr_raw_image_t& hdr, const uhdr_raw_image_t* sdr, const uhdr_b200_gm_config_t& cfg,
                  int base_quality, const uint8_t* exif, size_t exif_size, uint8_t* out, size_t cap,
                  size_t* out_size);

  // JpegR::getJPEGRInfo (jpegr.cpp:1417-1430): sizes, exif/icc, metadata; no pixel work
  int probe(const uint8_t* data, size_t size, DecodedInfo* info);
  // JpegR::decodeJPEGR (jpegr.cpp:1469-1531).  dest: host descriptor with planes allocated by the
  // caller (fmt/stride set); gainmap_out optional host descriptor (planes allocated, Y400/RGBA8888).
  // `probed`: the result of probe() on the same stream (saves the second scan of the container), or null.
  // With `dev_stream`, dest->planes[0] and gainmap_out->planes[0] are device memory (w / h equal to the decoded
  // images', checked before anything is written): the decoding runs on this codec's streams, the writes into the
  // two planes are ordered after the work enqueued earlier on *dev_stream, and *dev_stream waits for them.  The
  // call returns without waiting for either; settle() (run by the next decode()) waits for the writes.
  // `k` (1, 2, 4, 8): both JPEGs are decoded at 1/k size (jpeg_scaled_geometry) and the gain map is applied to those.
  // `fx` (host outputs at k = 1 only): the editor chain planned for this file's sizes; the output image and the map
  // are gathered through it in HBM, and dest / gainmap_out get the sizes it ends with.  A planned error is returned
  // once everything before it has succeeded, as the reference applies effects after decodeJPEGR.
  int decode(const uint8_t* data, size_t size, int out_ct, int out_fmt, float max_display_boost,
             uhdr_raw_image_t* dest, uhdr_raw_image_t* gainmap_out, uhdr_gainmap_metadata_t* md_out,
             const DecodedInfo* probed = nullptr, const cudaStream_t* dev_stream = nullptr, int k = 1,
             const DecodeEffects* fx = nullptr);
  // The two images decode() hands to applyGainMap, at 1/k: the primary as YCbCr planes (DECODE_TO_YCBCR_CS; Y400,
  // YUV420 / 422 / 444 at k = 1, Y400 / YUV444 above), the map as Y400 or RGBA8888 (DECODE_STREAM), each with the gamut
  // of its ICC profile, and the metadata.  `probed`: probe() of the same stream.  Enqueued on ws().stream(); the planes
  // are this codec's scratch, valid until its next call.
  int decode_images(const uint8_t* data, size_t size, const DecodedInfo& probed, int k, DevImage* sdr, DevImage* map,
                    uhdr_gainmap_metadata_t* md);
  // decode() into device planes (dev_stream, k) of many files, with one entropy decoding and one inverse DCT for all of
  // them (jpeg_entropy_decode_dev, jpeg_idct_dev), then each file's colour conversion / gain-map
  // application into its planes.  Each item gets the bytes and the code decode() gives for it alone; a failing item
  // writes nothing.  Items are taken in groups that fit `group_bytes` of scratch.  The writes are ordered after the
  // work enqueued earlier on `caller`, which waits for them; settle() waits for them on the host.  The return value is
  // an error that ends the whole call (CUDA, memory): the items not finished then are left as they were.
  int decode_batch(DecodeBatchItem* items, int n, int k, int out_ct, float max_display_boost, cudaStream_t caller,
                   size_t group_bytes);
  // Host wait until what an earlier decode() left in flight is done -- its writes into device planes, or the kernels
  // of a failed call: its scratch (device arenas of both workspaces, the pinned gain tables still waiting for their
  // copy) may be reused after this.
  int settle();

  // With gainmap_out->planes[0] == nullptr and lazy_gainmap set, decode() only fills the descriptor's
  // geometry and keeps the map in HBM; fetch_gainmap() copies it out when somebody asks for it
  // (uhdr_get_decoded_gainmap_image).  Valid until the next decode() on this codec.
  void set_lazy_gainmap(bool on) { lazy_gainmap_ = on; }
  int fetch_gainmap(uhdr_raw_image_t* gainmap_out);

  // JpegDecoderHelper::decompressImage equivalent producing a device image
  // `k` > 1: at 1/k size, gray / 4:4:4 / 4:2:0 input only, the planes come out Y400 or YUV444 (jpeg_scaled_geometry)
  int decode_jpeg_dev(const uint8_t* data, size_t size, int mode, DevImage* out, JpegHeader* hdr, int k = 1) {
    return decode_jpeg_dev(ws_, data, size, mode, out, hdr, nullptr, k);
  }
  // uhdr_b200_transcode (transcode.cu): both JPEGs of the file decoded at 1/cfg.k as raw planes, re-encoded at the
  // configured qualities -- the base image optionally 4:2:0 through libjpeg's scanline downsampling -- and assembled
  // as API-4 assembles them, with the file's ICC profiles, metadata and (keep_exif) EXIF.  `probed`: probe() of data.
  int transcode(const uint8_t* data, size_t size, const DecodedInfo& probed, const uhdr_b200_transcode_config_t& cfg,
                uint8_t* out, size_t cap, size_t* out_size);
  // transcode() of many files with one entropy decoding, one inverse DCT, one staging launch, one block-stage launch and
  // one entropy-coding launch per group of items (groups as decode_batch forms them, the encoder's scratch included),
  // and two host waits for the encoder.  Each item gets the bytes, size and code transcode() gives for it alone; a
  // failing item writes nothing.  The return value is an error that ends the whole call (CUDA, memory).
  int transcode_batch(TranscodeBatchItem* items, int n, const uhdr_b200_transcode_config_t& cfg, size_t group_bytes);
  // transcode() of many files, each into up to kLadderMaxRungs outputs with their own cfg (rungs[files[i].r0 + j], data
  // and info set as the file's): per group of files, both JPEGs of every file entropy-decoded once, one k_idct<0> launch
  // for every k of every file, then the batch's encode (transcode_encode) over every rung of the group.  Groups close
  // at `group_bytes` of scratch, 2^29 entropy-coded bytes or kLadderMaxRungs distinct quality pairs.  A rung with
  // rc != E_OK on entry is skipped.  Each rung gets the bytes, size and code transcode() gives for its cfg alone; a
  // failing rung writes nothing.  The return value is an error that ends the whole call (CUDA, memory).
  int transcode_ladders(LadderFile* files, int n, TranscodeBatchItem* rungs, size_t group_bytes);
  ~JpegRCodec();

 private:
  // `to_rgba` (mode 1 only): the colour conversion is not launched; its parameters, all but the destination,
  // are returned there, out->v.p[0] stays null
  int decode_jpeg_dev(Workspace& ws, const uint8_t* data, size_t size, int mode, DevImage* out, JpegHeader* hdr,
                      YccToRgbaParams* to_rgba = nullptr, int k = 1);
  // both JPEGs of a JPEG/R (po / pl, go / gl: their spans in data) on this codec's streams -- the gain map's on the
  // helper thread when both are sizeable, joined into ws_ -- and the gamuts of their ICC profiles; want_map false: the
  // primary only.  sdr_mode / to_rgba: decode_jpeg_dev's mode / to_rgba of the primary; map_mode: the map's mode
  // (2 = DECODE_STREAM, what decodeJPEGR uses, jpegr.cpp:1486).
  int decode_pair(const uint8_t* data, size_t po, size_t pl, size_t go, size_t gl, int sdr_mode, YccToRgbaParams* to_rgba,
                  bool want_map, int k, DevImage* sdr, DevImage* map, JpegHeader* ph, JpegHeader* gh, PhaseTrace& tr,
                  int map_mode = 2);
  int decode_body(const uint8_t* data, size_t size, int out_ct, int out_fmt, float max_display_boost,
                  uhdr_raw_image_t* dest, uhdr_raw_image_t* gainmap_out, uhdr_gainmap_metadata_t* md_out,
                  const DecodedInfo* probed, const cudaStream_t* dev_stream, int k, const DecodeEffects* fx);
  // record where this codec's streams are (both joined into ws_); settle() waits for that point
  int mark_in_flight();
  int write_dev_outputs(const DevImage& sdr, const DevImage& map, const YccToRgbaParams& to_rgba,
                        const uhdr_gainmap_metadata_t& md, int out_ct, float max_display_boost,
                        uhdr_raw_image_t* dest, uhdr_raw_image_t* gainmap_out, cudaStream_t caller);
  // write_dev_outputs' parts: the descriptors' checks, the wait for the caller's stream, the writes
  static int check_dev_outputs(const DevImage& sdr, const DevImage& map, int out_ct, const uhdr_raw_image_t* dest,
                               const uhdr_raw_image_t* gainmap_out);
  int join_caller(cudaStream_t caller);
  int enqueue_dev_writes(const DevImage& sdr, const DevImage& map, const YccToRgbaParams& to_rgba,
                         const uhdr_gainmap_metadata_t& md, int out_ct, float max_display_boost,
                         uhdr_raw_image_t* dest, uhdr_raw_image_t* gainmap_out);
  // Both batched calls' decode of a group (Item: DecodeBatchItem or TranscodeBatchItem), as decode_pair would decode
  // each file at 1/k: the headers, one entropy decoding and one inverse DCT for every scan, the tail stages and the
  // gamuts.  sdr_mode / map_mode: decode_jpeg_dev's modes; defer_rgba: the primary's colour conversion (mode 1) is left
  // in to_rgba.  A file's own error goes to the file, in the order the single call meets it; the return value is an
  // error that ends the call (CUDA, memory).
  template <class Item>
  int decode_batch_files(Item* items, int n, int k, int sdr_mode, bool defer_rgba, int map_mode);
  int decode_batch_group(DecodeBatchItem* items, int n, int k, int out_ct, float max_display_boost, cudaStream_t caller);
  int transcode_batch_group(TranscodeBatchItem* items, int n, const uhdr_b200_transcode_config_t& cfg);
  // transcode_ladders' decode of a group: per file the headers once and per distinct k the plans of both JPEGs, one
  // entropy decoding of every file's scans, per file and k the errors in transcode()'s order, one k_idct<0> over every
  // file's planes; then each rung's decoded pair (sdr, map, ph, gh)
  int decode_ladders(LadderFile* files, int n, TranscodeBatchItem* rungs);
  // Both transcode paths' encode, once every item's pair is decoded: per item its cfg's 4:2:2 check of base_420, one
  // k_stage_batch launch, one k_fdct8_code_batch launch per distinct (base_quality, gainmap_quality) pair (at most
  // kLadderMaxRungs of them), one k_huff_encode_batch, two host waits with k_pack_scans, then per item the scan checks
  // and transcode_finish.  A failing item gets its code; the return value is an error that ends the call.
  int transcode_encode(TranscodeBatchItem* items, int n);
  // transcode_encode's scratch for one item at 1/k: per JPEG the staged planes, the code-word entries and meta, the scan
  static size_t encode_bytes(const DecodedInfo& in, int k);
  // transcode()'s last stage, once both scans are on the host: API-4's checks, the heads, EXIF, the container, the cap
  int transcode_finish(const uint8_t* data, const DecodedInfo& probed, const JpegHeader& ph, const JpegHeader& gh,
                       const JpegEncodeJob& base_jpeg, const JpegEncodeJob& gm_jpeg, const uhdr_b200_transcode_config_t& cfg,
                       uint8_t* out, size_t cap, size_t* out_size);
  static int fail_base_422();
  // scratch of one file of a batched decode at 1/k (w x h, gw x gh: the 1/k sizes; size: the file's bytes)
  static size_t batch_decode_bytes(int w, int h, int gw, int gh, int k, size_t size);
  // The batches' groups: items [g0, g1) as long as their scratch cost(i, &coded) fits `group_bytes` (at least one item)
  // and their entropy-coded bytes stay below 2^29, so that every bit position of a group fits 32 bits, and admit(i,
  // fresh) takes item i into the group being formed (a new one when `fresh`, which it must take).  run(g0, g1) runs
  // each group once the previous one's work is done on the host and the workspace is rewound.
  static bool admit_any(int, bool) { return true; }
  template <class Cost, class Run, class Admit = bool (*)(int, bool)>
  int for_each_group(int n, size_t group_bytes, Cost cost, Run run, Admit admit = admit_any) {
    int rc = E_OK;
    for (int g0 = 0; g0 < n && !rc;) {
      size_t bytes = 0, coded = 0;
      int g1 = g0;
      for (; g1 < n; g1++) {
        size_t c = 0;
        const size_t b = cost(g1, &c);
        if (g1 > g0 && (bytes + b > group_bytes || coded + c >= (1u << 29))) break;
        if (!admit(g1, g1 == g0)) break;
        bytes += b;
        coded += c;
      }
      if (g0 > 0 && (rc = ws_.sync())) break;  // the previous group's pinned staging is rewound below
      ws_.rewind();
      rc = run(g0, g1);
      g0 = g1;
    }
    return rc;
  }
  std::vector<JpegScanJob> batch_scans_;   // grow-only scratch of the batched calls
  std::vector<JpegIdctJob> batch_idct_;
  std::vector<JpegEncodeJob*> batch_enc_;
  Workspace ws_;
  // second stream + arenas: the gain-map JPEG of a decode is processed by a helper thread while the
  // calling thread handles the primary image (both entropy decoders alternate host and device phases)
  std::unique_ptr<Workspace> ws2_;
  ParkedThread helper_;
  cudaEvent_t map_ready_ = nullptr;
  // decode() into device planes: the caller's stream up to the call, and this codec's writes into its planes
  cudaEvent_t caller_ready_ = nullptr, writes_done_ = nullptr;
  bool writes_pending_ = false;
  bool lazy_gainmap_ = false, map_pending_ = false;
  DevImage last_map_{};
};

// JpegEncoderHelper::compressImage (jpegencoderhelper.cpp:101) of a device image, on ws.stream(); returns once the
// stream is in `out`.  `caller_planes`: see block_stage_input.
// rows: from upload_jpeg_input (nullptr: the planes are read up to their height, then the pad row)
int compress_image_dev(Workspace& ws, const DevImage& img, int quality, const void* icc, size_t icc_size,
                       bool caller_planes, uint8_t* out, size_t cap, size_t* out_size, const int* rows = nullptr);
// The input of JpegEncoderHelper::compressImage from HOST planes (uhdr_b200_jpeg_encode, uhdr_b200_jpeg_forward, the
// C++ JpegEncoderHelper): upload_image, then the helper's edge padding of planes whose width is not a multiple of 8
// for the caller's strides (jpegencoderhelper.cpp:246-309).  rows[c] goes to jpeg_forward_dev.
int upload_jpeg_input(Workspace& ws, const uhdr_raw_image_t& src, DevImage* out, int rows[3]);
// upload_jpeg_input's second half: the helper's padding of `img`, a workspace copy of `caller`'s planes made with
// upload_image (kind: where caller's planes are)
int helper_padding(Workspace& ws, const uhdr_raw_image_t& caller, cudaMemcpyKind kind, const DevImage& img, int rows[3]);

// first APPn marker `id` of a header whose payload starts with `sig`, as a view into the stream d
ByteView find_marker(const uint8_t* d, const JpegHeader& h, uint8_t id, const char* sig, size_t sig_len);

// API-4's ICC rules for a primary / gain-map pair (jpegr.cpp:397-428): with md.use_base_cg = 0 the map must carry an ICC
// profile (map_has_icc), and a primary without one (base_icc empty) gets the profile of its gamut base_cg, which must be
// a known one.  *icc / *icc_n: the profile assemble_jpegr is to add, null when the primary keeps its own.
int api4_icc(const ByteView& base_icc, bool map_has_icc, int base_cg, const uhdr_gainmap_metadata_t& md, const uint8_t** icc,
             size_t* icc_n);

// uhdr_enc_set_raw_image's checks of one intent's descriptor (ultrahdr_api.cpp:842-1025): its code, the last error
// set.  The planes are not dereferenced.
int validate_raw_intent(const uhdr_raw_image_t& img, int intent);

// The *_dev entry points' helpers (capi_stages.cu).  dev_codec: the calling thread's codec for the current device,
// settled and rewound.  check_dev_planes: a device descriptor's planes present, strides >= widths, elements aligned;
// check_dev_memory: each plane device memory of the current device.
int dev_codec(JpegRCodec** out);
int check_dev_planes(const uhdr_raw_image_t& img, const char* what);
int check_dev_memory(const uhdr_raw_image_t& img, const char* what);


}  // namespace uhdr_b200
