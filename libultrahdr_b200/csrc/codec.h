// Codec orchestration: the CUDA counterpart of ultrahdr::JpegR (lib/include/ultrahdr/jpegr.h:52-222).
// encodeJPEGR API-0 / API-1 and decodeJPEGR run their pixel and block stages on the device;
// the marker/container layer is host code.
#pragma once
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "container.h"
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
  int decode(const uint8_t* data, size_t size, int out_ct, int out_fmt, float max_display_boost,
             uhdr_raw_image_t* dest, uhdr_raw_image_t* gainmap_out, uhdr_gainmap_metadata_t* md_out,
             const DecodedInfo* probed = nullptr, const cudaStream_t* dev_stream = nullptr, int k = 1);
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
  ~JpegRCodec();

 private:
  // `to_rgba` (mode 1 only): the colour conversion is not launched; its parameters, all but the destination,
  // are returned there, out->v.p[0] stays null
  int decode_jpeg_dev(Workspace& ws, const uint8_t* data, size_t size, int mode, DevImage* out, JpegHeader* hdr,
                      YccToRgbaParams* to_rgba = nullptr, int k = 1);
  int decode_body(const uint8_t* data, size_t size, int out_ct, int out_fmt, float max_display_boost,
                  uhdr_raw_image_t* dest, uhdr_raw_image_t* gainmap_out, uhdr_gainmap_metadata_t* md_out,
                  const DecodedInfo* probed, const cudaStream_t* dev_stream, int k);
  // record where this codec's streams are (both joined into ws_); settle() waits for that point
  int mark_in_flight();
  int write_dev_outputs(const DevImage& sdr, const DevImage& map, const YccToRgbaParams& to_rgba,
                        const uhdr_gainmap_metadata_t& md, int out_ct, float max_display_boost,
                        uhdr_raw_image_t* dest, uhdr_raw_image_t* gainmap_out, cudaStream_t caller);
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
int compress_image_dev(Workspace& ws, const DevImage& img, int quality, const void* icc, size_t icc_size,
                       bool caller_planes, uint8_t* out, size_t cap, size_t* out_size);

// uhdr_enc_set_raw_image's checks of one intent's descriptor (ultrahdr_api.cpp:842-1025): its code, the last error
// set.  The planes are not dereferenced.
int validate_raw_intent(const uhdr_raw_image_t& img, int intent);


}  // namespace uhdr_b200
