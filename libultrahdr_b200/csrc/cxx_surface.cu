// The reference's C++ surface (include/ultrahdr/*.h: ultrahdr::UltraHdr, ultrahdr::JpegR incl. the
// deprecated jr_* overloads, JpegEncoderHelper, JpegDecoderHelper) on top of the CUDA codec.  The
// classes are thin: arguments are validated like in the reference (error texts are its own), the work
// is done by JpegRCodec / the engine stages on the calling thread's workspace (one stream + arenas per
// host thread, created on first use).  Reference bodies: lib/src/jpegr.cpp:179-434 (encode API-0..4),
// :1417-1531 (info / decode), :2224-2890 (deprecated aliases), lib/src/ultrahdr_api.cpp:44-143
// (owning descriptors), lib/src/jpegencoderhelper.cpp:101-129, lib/src/jpegdecoderhelper.cpp:169-210,
// :536-555.
#include <cmath>
#include <cstring>

#include "codec.h"

#pragma GCC visibility push(default)
#include "ultrahdr/jpegr.h"
#pragma GCC visibility pop

using namespace uhdr_b200;

namespace {

uhdr_error_info_t ok() {
  uhdr_error_info_t s;
  memset(&s, 0, sizeof s);
  s.error_code = UHDR_CODEC_OK;
  return s;
}
uhdr_error_info_t from_rc(int rc) {
  if (rc == E_OK) return ok();
  uhdr_error_info_t s;
  memset(&s, 0, sizeof s);
  s.error_code = (uhdr_codec_err_t)rc;
  s.has_detail = 1;
  snprintf(s.detail, sizeof s.detail, "%s", last_error());
  return s;
}
uhdr_error_info_t err(uhdr_codec_err_t code, const char* msg) {
  uhdr_error_info_t s;
  memset(&s, 0, sizeof s);
  s.error_code = code;
  s.has_detail = 1;
  snprintf(s.detail, sizeof s.detail, "%s", msg);
  return s;
}

// one codec (stream + device / pinned arenas) per host thread, rewound at every call
JpegRCodec* tls_codec(int* rc) {
  static thread_local JpegRCodec* c = nullptr;
  *rc = E_OK;
  if (!c) {
    c = new JpegRCodec();
    *rc = c->init();
    if (*rc) {
      delete c;
      c = nullptr;
      return nullptr;
    }
  }
  c->ws().sync();  // an earlier call that failed can have left copies from the pinned arena in flight
  c->ws().rewind();
  return c;
}

inline size_t align_up(size_t v, size_t a) { return a ? (v + a - 1) / a * a : v; }

}  // namespace

#pragma GCC visibility push(default)
namespace ultrahdr {

const int kMinWidth = 8;
const int kMinHeight = 8;
const int kMaxWidth = 8192;   // UHDR_MAX_DIMENSION of the reference's default build
const int kMaxHeight = 8192;

// ---- owning descriptors (ultrahdr_api.cpp:44-143) ------------------------------------------------
uhdr_memory_block::uhdr_memory_block(size_t capacity) {
  m_buffer = std::make_unique<uint8_t[]>(capacity);  // value-initialised: zeros, like the reference's
  m_capacity = capacity;
}

uhdr_raw_image_ext::uhdr_raw_image_ext(uhdr_img_fmt_t fmt_, uhdr_color_gamut_t cg_, uhdr_color_transfer_t ct_,
                                       uhdr_color_range_t range_, unsigned w_, unsigned h_, unsigned align_stride_to) {
  fmt = fmt_; cg = cg_; ct = ct_; range = range_; w = w_; h = h_;
  const size_t aw = align_up(w_, align_stride_to);
  size_t bpp = 1;
  if (fmt_ == UHDR_IMG_FMT_24bppYCbCrP010 || fmt_ == UHDR_IMG_FMT_30bppYCbCr444) bpp = 2;
  else if (fmt_ == UHDR_IMG_FMT_24bppRGB888) bpp = 3;
  else if (fmt_ == UHDR_IMG_FMT_32bppRGBA8888 || fmt_ == UHDR_IMG_FMT_32bppRGBA1010102) bpp = 4;
  else if (fmt_ == UHDR_IMG_FMT_64bppRGBAHalfFloat) bpp = 8;
  const size_t p1 = bpp * aw * h_;
  size_t p2 = 0, p3 = 0;
  if (fmt_ == UHDR_IMG_FMT_24bppYCbCrP010) p2 = 2 * bpp * (aw / 2) * (h_ / 2);
  else if (fmt_ == UHDR_IMG_FMT_30bppYCbCr444 || fmt_ == UHDR_IMG_FMT_24bppYCbCr444) p2 = p3 = bpp * aw * h_;
  else if (fmt_ == UHDR_IMG_FMT_12bppYCbCr420) p2 = p3 = bpp * (aw / 2) * (h_ / 2);
  m_block = std::make_unique<uhdr_memory_block_t>(p1 + p2 + p3);
  uint8_t* data = m_block->m_buffer.get();
  planes[UHDR_PLANE_Y] = data;
  stride[UHDR_PLANE_Y] = (unsigned)aw;
  planes[UHDR_PLANE_U] = planes[UHDR_PLANE_V] = nullptr;
  stride[UHDR_PLANE_U] = stride[UHDR_PLANE_V] = 0;
  if (fmt_ == UHDR_IMG_FMT_24bppYCbCrP010) {
    planes[UHDR_PLANE_UV] = data + p1;
    stride[UHDR_PLANE_UV] = (unsigned)aw;
  } else if (fmt_ == UHDR_IMG_FMT_30bppYCbCr444 || fmt_ == UHDR_IMG_FMT_24bppYCbCr444) {
    planes[UHDR_PLANE_U] = data + p1;
    planes[UHDR_PLANE_V] = data + p1 + p2;
    stride[UHDR_PLANE_U] = stride[UHDR_PLANE_V] = (unsigned)aw;
  } else if (fmt_ == UHDR_IMG_FMT_12bppYCbCr420) {
    planes[UHDR_PLANE_U] = data + p1;
    planes[UHDR_PLANE_V] = data + p1 + p2;
    stride[UHDR_PLANE_U] = stride[UHDR_PLANE_V] = (unsigned)(aw / 2);
  }
}

uhdr_compressed_image_ext::uhdr_compressed_image_ext(uhdr_color_gamut_t cg_, uhdr_color_transfer_t ct_, uhdr_color_range_t range_,
                                                     size_t sz) {
  m_block = std::make_unique<uhdr_memory_block_t>(sz);
  data = m_block->m_buffer.get();
  capacity = sz;
  data_sz = 0;
  cg = cg_; ct = ct_; range = range_;
}

uhdr_error_info_t uhdr_validate_gainmap_metadata_descriptor(uhdr_gainmap_metadata_t* metadata) {
  if (!metadata) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for gainmap metadata descriptor");
  return from_rc(validate_metadata(*metadata));
}

uhdr_color_transfer_t map_legacy_ct_to_ct(ultrahdr_transfer_function ct) {
  switch (ct) {
    case ULTRAHDR_TF_HLG: return UHDR_CT_HLG;
    case ULTRAHDR_TF_PQ: return UHDR_CT_PQ;
    case ULTRAHDR_TF_LINEAR: return UHDR_CT_LINEAR;
    case ULTRAHDR_TF_SRGB: return UHDR_CT_SRGB;
    default: return UHDR_CT_UNSPECIFIED;
  }
}
uhdr_color_gamut_t map_legacy_cg_to_cg(ultrahdr_color_gamut cg) {
  switch (cg) {
    case ULTRAHDR_COLORGAMUT_BT2100: return UHDR_CG_BT_2100;
    case ULTRAHDR_COLORGAMUT_BT709: return UHDR_CG_BT_709;
    case ULTRAHDR_COLORGAMUT_P3: return UHDR_CG_DISPLAY_P3;
    default: return UHDR_CG_UNSPECIFIED;
  }
}
ultrahdr_color_gamut map_cg_to_legacy_cg(uhdr_color_gamut_t cg) {
  switch (cg) {
    case UHDR_CG_BT_2100: return ULTRAHDR_COLORGAMUT_BT2100;
    case UHDR_CG_BT_709: return ULTRAHDR_COLORGAMUT_BT709;
    case UHDR_CG_DISPLAY_P3: return ULTRAHDR_COLORGAMUT_P3;
    default: return ULTRAHDR_COLORGAMUT_UNSPECIFIED;
  }
}

// ---- UltraHdr -------------------------------------------------------------------------------------
UltraHdr::UltraHdr(void* uhdrGLESCtxt, int mapDimensionScaleFactor, int mapCompressQuality, bool useMultiChannelGainMap, float gamma,
                   uhdr_enc_preset_t preset, float minContentBoost, float maxContentBoost, float targetDispPeakBrightness)
    : mUhdrGLESCtxt(uhdrGLESCtxt), mMapDimensionScaleFactor(mapDimensionScaleFactor), mMapCompressQuality(mapCompressQuality),
      mUseMultiChannelGainMap(useMultiChannelGainMap), mGamma(gamma), mEncPreset(preset), mMinContentBoost(minContentBoost),
      mMaxContentBoost(maxContentBoost), mTargetDispPeakBrightness(targetDispPeakBrightness) {}

static uhdr_b200_gm_config_t make_cfg(int scale, int quality, bool multi, float gamma, uhdr_enc_preset_t preset, float mn, float mx,
                                      float nits) {
  uhdr_b200_gm_config_t c;
  c.scale_factor = scale;
  c.quality = quality;
  c.multichannel = multi ? 1 : 0;
  c.gamma = gamma;
  c.preset = preset;
  c.min_content_boost = mn;
  c.max_content_boost = mx;
  c.target_disp_peak_nits = nits;
  c.sdr_is_601 = 0;
  c.use_luminance = 1;
  return c;
}

uhdr_error_info_t UltraHdr::parseGainMapMetadata(uint8_t* iso_data, size_t iso_size, uint8_t* xmp_data, size_t xmp_size,
                                                 uint8_t* exif_data, int exif_size, uhdr_gainmap_metadata_ext_t* uhdr_metadata) {
  if (!uhdr_metadata) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for gainmap metadata descriptor");
  uhdr_gainmap_metadata_t md;
  memset(&md, 0, sizeof md);
  const int rc = parse_gainmap_metadata(iso_data, iso_size, xmp_data, xmp_size, exif_data, exif_size > 0 ? (size_t)exif_size : 0, &md);
  if (rc) return from_rc(rc);
  static_cast<uhdr_gainmap_metadata&>(*uhdr_metadata) = md;
  uhdr_metadata->version = kJpegrVersion;
  return ok();
}

uhdr_error_info_t UltraHdr::toneMap(uhdr_raw_image_t* hdr_intent, uhdr_raw_image_t* sdr_intent) {
  if (!hdr_intent || !sdr_intent) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for image descriptor");
  int rc;
  JpegRCodec* c = tls_codec(&rc);
  if (!c) return from_rc(rc);
  Workspace& ws = c->ws();
  DevImage dh, ds;
  if ((rc = upload_image(ws, *hdr_intent, &dh))) return from_rc(rc);
  if ((rc = alloc_dev_image(ws, sdr_intent->fmt, hdr_intent->w, hdr_intent->h, 64, &ds))) return from_rc(rc);
  if ((rc = tonemap_dev(ws, dh, &ds))) return from_rc(rc);
  sdr_intent->cg = (uhdr_color_gamut_t)ds.cg;
  sdr_intent->ct = (uhdr_color_transfer_t)ds.ct;
  sdr_intent->range = (uhdr_color_range_t)ds.range;
  if ((rc = download_image(ws, ds, sdr_intent))) return from_rc(rc);
  return from_rc(ws.sync());
}

uhdr_error_info_t UltraHdr::generateGainMap(uhdr_raw_image_t* sdr_intent, uhdr_raw_image_t* hdr_intent,
                                            uhdr_gainmap_metadata_ext_t* gainmap_metadata,
                                            std::unique_ptr<uhdr_raw_image_ext_t>& gainmap_img, bool sdr_is_601, bool use_luminance) {
  if (!sdr_intent || !hdr_intent || !gainmap_metadata) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr argument");
  int rc;
  JpegRCodec* c = tls_codec(&rc);
  if (!c) return from_rc(rc);
  Workspace& ws = c->ws();
  uhdr_b200_gm_config_t cfg = make_cfg(mMapDimensionScaleFactor, mMapCompressQuality, mUseMultiChannelGainMap, mGamma, mEncPreset,
                                       mMinContentBoost, mMaxContentBoost, mTargetDispPeakBrightness);
  cfg.sdr_is_601 = sdr_is_601 ? 1 : 0;
  cfg.use_luminance = use_luminance ? 1 : 0;
  DevImage ds, dh;
  if ((rc = upload_image(ws, *sdr_intent, &ds))) return from_rc(rc);
  if ((rc = upload_image(ws, *hdr_intent, &dh))) return from_rc(rc);
  GainmapJob job;
  if ((rc = generate_gainmap_dev(ws, ds, dh, cfg, 64, &job))) return from_rc(rc);
  // jpegr.cpp:714-716: owned by the caller through the unique_ptr, stride aligned to 64
  gainmap_img = std::make_unique<uhdr_raw_image_ext_t>((uhdr_img_fmt_t)job.map.v.fmt, (uhdr_color_gamut_t)job.map.cg,
                                                       (uhdr_color_transfer_t)job.map.ct, (uhdr_color_range_t)job.map.range,
                                                       job.map.v.w, job.map.v.h, 64);
  if ((rc = download_image(ws, job.map, gainmap_img.get()))) return from_rc(rc);
  if ((rc = ws.sync())) return from_rc(rc);
  uhdr_gainmap_metadata_t md;
  finish_gainmap_metadata(job, &md);
  static_cast<uhdr_gainmap_metadata&>(*gainmap_metadata) = md;
  gainmap_metadata->version = kJpegrVersion;
  return ok();
}

uhdr_error_info_t UltraHdr::applyGainMap(uhdr_raw_image_t* sdr_intent, uhdr_raw_image_t* gainmap_img,
                                         uhdr_gainmap_metadata_ext_t* gainmap_metadata, uhdr_color_transfer_t output_ct,
                                         uhdr_img_fmt_t output_format, float max_display_boost, uhdr_raw_image_t* dest) {
  (void)output_format;
  if (!sdr_intent || !gainmap_img || !gainmap_metadata) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr argument");
  if (dest == nullptr || dest->planes[UHDR_PLANE_PACKED] == nullptr)
    return err(UHDR_CODEC_INVALID_PARAM, "apply gainmap method received nullptr for destination image or plane pointer");
  if (gainmap_metadata->version.compare(kJpegrVersion)) {  // jpegr.cpp:1538-1547
    uhdr_error_info_t s = err(UHDR_CODEC_UNSUPPORTED_FEATURE, "");
    snprintf(s.detail, sizeof s.detail, "Unsupported gainmap metadata, version. Expected %s, Got %s", kJpegrVersion,
             gainmap_metadata->version.c_str());
    return s;
  }
  int rc;
  JpegRCodec* c = tls_codec(&rc);
  if (!c) return from_rc(rc);
  Workspace& ws = c->ws();
  DevImage ds, dm, dd;
  if ((rc = upload_image(ws, *sdr_intent, &ds))) return from_rc(rc);
  if ((rc = upload_image(ws, *gainmap_img, &dm))) return from_rc(rc);
  if ((rc = alloc_dev_image(ws, dest->fmt, sdr_intent->w, sdr_intent->h, 64, &dd))) return from_rc(rc);
  if ((rc = apply_gainmap_dev(ws, ds, dm, *gainmap_metadata, output_ct, max_display_boost, &dd))) return from_rc(rc);
  dest->cg = (uhdr_color_gamut_t)dd.cg;
  if ((rc = download_image(ws, dd, dest))) return from_rc(rc);
  return from_rc(ws.sync());
}

uhdr_error_info_t UltraHdr::convertYuv(uhdr_raw_image_t* image, uhdr_color_gamut_t src_encoding, uhdr_color_gamut_t dst_encoding) {
  if (!image) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for image descriptor");
  int rc;
  JpegRCodec* c = tls_codec(&rc);
  if (!c) return from_rc(rc);
  Workspace& ws = c->ws();
  DevImage d;
  if ((rc = upload_image(ws, *image, &d))) return from_rc(rc);
  if ((rc = convert_yuv_dev(ws, &d, src_encoding, dst_encoding))) return from_rc(rc);
  if ((rc = download_image(ws, d, image))) return from_rc(rc);
  return from_rc(ws.sync());
}

// jpegr.cpp:1945-1977: scalar host form (the device kernel applies the same expressions per pixel)
GlobalTonemapOutputs globalTonemap(const std::array<float, 3>& rgb_in, float headroom, bool is_normalized) {
  std::array<float, 3> rgb_hdr;
  for (int i = 0; i < 3; i++) rgb_hdr[i] = is_normalized ? rgb_in[i] * headroom : rgb_in[i];
  const float max_hdr = std::max(std::max(rgb_hdr[0], rgb_hdr[1]), rgb_hdr[2]);
  const float max_sdr = max_hdr * (1.0f + (max_hdr / (headroom * headroom))) / (1.0f + max_hdr);  // ReinhardMap
  std::array<float, 3> rgb_sdr;
  for (int i = 0; i < 3; i++) rgb_sdr[i] = max_hdr > 0.0f ? rgb_hdr[i] * max_sdr / max_hdr : 0.0f;
  GlobalTonemapOutputs o;
  o.rgb_out = rgb_sdr;
  o.y_hdr = max_hdr;
  o.y_sdr = max_sdr;
  return o;
}

// ---- JpegEncoderHelper / JpegDecoderHelper -------------------------------------------------------
uhdr_error_info_t JpegEncoderHelper::compressImage(const uhdr_raw_image_t* img, const int qfactor, const void* iccBuffer,
                                                   const size_t iccSize) {
  if (!img) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for image descriptor");
  int rc;
  JpegRCodec* c = tls_codec(&rc);
  if (!c) return from_rc(rc);
  Workspace& ws = c->ws();
  DevImage d;
  int rows[3];
  if ((rc = upload_jpeg_input(ws, *img, &d, rows))) return from_rc(rc);
  JpegEncodeJob job, *jobs[] = {&job};
  JpegPieces p;
  if ((rc = jpeg_encode_dev(ws, d, qfactor, &job, rows)) || (rc = jpeg_entropy_collect(ws, jobs, 1)) ||
      (rc = jpeg_stream_pieces(ws, job, iccBuffer, iccSize, &p)))
    return from_rc(rc);
  mResult.resize(p.total());
  p.copy_to(mResult.data());
  return ok();
}

uhdr_error_info_t JpegEncoderHelper::compressImage(const uint8_t* planes[3], const unsigned int strides[3], const int width,
                                                   const int height, const uhdr_img_fmt_t format, const int qfactor,
                                                   const void* iccBuffer, const size_t iccSize) {
  uhdr_raw_image_t img;
  memset(&img, 0, sizeof img);
  img.fmt = format;
  img.cg = UHDR_CG_UNSPECIFIED;
  img.ct = UHDR_CT_UNSPECIFIED;
  img.range = UHDR_CR_FULL_RANGE;
  img.w = width;
  img.h = height;
  for (int i = 0; i < 3; i++) {
    img.planes[i] = const_cast<uint8_t*>(planes[i]);
    img.stride[i] = strides[i];
  }
  return compressImage(&img, qfactor, iccBuffer, iccSize);
}

uhdr_compressed_image_t JpegEncoderHelper::getCompressedImage() {
  uhdr_compressed_image_t img;
  img.data = mResult.data();
  img.capacity = img.data_sz = mResult.size();
  img.cg = UHDR_CG_UNSPECIFIED;
  img.ct = UHDR_CT_UNSPECIFIED;
  img.range = UHDR_CR_UNSPECIFIED;
  return img;
}

static void take_marker(const uint8_t* d, const JpegHeader& h, uint8_t id, const char* sig, size_t sig_len, std::vector<uint8_t>* out,
                        long* pos) {
  out->clear();
  if (pos) *pos = -1;
  for (const JpegMarker& m : h.markers)
    if (m.id == id && m.length > sig_len && !memcmp(d + m.offset, sig, sig_len)) {
      out->assign(d + m.offset, d + m.offset + m.length);
      if (pos) *pos = (long)m.offset;
      return;
    }
}

uhdr_error_info_t JpegDecoderHelper::decompressImage(const void* image, size_t length, decode_mode_t mode) {
  if (image == nullptr) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for compressed image data");
  if (length <= 0) return err(UHDR_CODEC_INVALID_PARAM, "received bad compressed image size 0");
  mResultBuffer.clear();
  const uint8_t* d = static_cast<const uint8_t*>(image);
  JpegHeader h;
  int rc = jpeg_read_header(d, length, &h);
  if (rc) return from_rc(rc);
  take_marker(d, h, 0xE1, "http://ns.adobe.com/xap/1.0/", 29, &mXMPBuffer, nullptr);
  take_marker(d, h, 0xE1, "Exif\0\0", 6, &mEXIFBuffer, &mExifPayLoadOffset);
  take_marker(d, h, 0xE2, "ICC_PROFILE", 12, &mICCBuffer, nullptr);
  take_marker(d, h, 0xE2, "urn:iso:std:iso:ts:21496:-1", 28, &mIsoMetadataBuffer, nullptr);
  const JpegFrame& f = h.frame;
  mNumComponents = f.ncomp;
  for (int i = 0; i < f.ncomp && i < kMaxNumComponents; i++) {
    mPlaneWidth[i] = f.comp[i].width;
    mPlaneHeight[i] = f.comp[i].height;
  }
  if (mode == PARSE_STREAM) {
    mOutFormat = UHDR_IMG_FMT_UNSPECIFIED;
    return ok();
  }
  JpegRCodec* c = tls_codec(&rc);
  if (!c) return from_rc(rc);
  DevImage img;
  JpegHeader h2;
  const int m = mode == DECODE_TO_RGB_CS ? 1 : (mode == DECODE_STREAM ? 2 : 0);
  if ((rc = c->decode_jpeg_dev(d, length, m, &img, &h2))) return from_rc(rc);
  mOutFormat = (uhdr_img_fmt_t)img.v.fmt;
  // host layout of the reference's result buffer (jpegdecoderhelper.cpp:363-392): planes back to back,
  // each plane's stride / height rounded up to the maximum sampling factor
  size_t need = 0;
  if (img.v.fmt == F_RGBA8888) {
    mPlaneHStride[0] = f.width;
    mPlaneVStride[0] = f.height;
    need = (size_t)f.width * f.height * 4;
  } else {
    for (int k = 0; k < f.ncomp; k++) {
      mPlaneHStride[k] = (f.comp[k].width + f.max_h - 1) / f.max_h * f.max_h;
      mPlaneVStride[k] = (f.comp[k].height + f.max_v - 1) / f.max_v * f.max_v;
      need += (size_t)mPlaneHStride[k] * mPlaneVStride[k];
    }
  }
  mResultBuffer.assign(need, 0);
  Workspace& ws = c->ws();
  if (img.v.fmt == F_RGBA8888) {
    uhdr_raw_image_t out = getDecompressedImage();
    if ((rc = download_image(ws, img, &out))) return from_rc(rc);
  } else {
    uint8_t* p = mResultBuffer.data();
    for (int k = 0; k < f.ncomp; k++) {
      const size_t wbytes = (mPlaneHStride[k] % 8 == 0) ? mPlaneHStride[k] : (size_t)f.comp[k].width;
      const size_t rows = std::min<size_t>(mPlaneVStride[k], (size_t)f.comp[k].hblocks * 8);
      if (cudaMemcpy2DAsync(p, mPlaneHStride[k], img.v.p[k], img.v.stride[k], wbytes, rows, cudaMemcpyDeviceToHost, ws.stream()) !=
          cudaSuccess)
        return err(UHDR_CODEC_ERROR, "device to host copy of the decoded planes failed");
      p += (size_t)mPlaneHStride[k] * mPlaneVStride[k];
    }
  }
  return from_rc(ws.sync());
}

uhdr_raw_image_t JpegDecoderHelper::getDecompressedImage() {  // jpegdecoderhelper.cpp:536-555
  uhdr_raw_image_t img;
  memset(&img, 0, sizeof img);
  img.fmt = mOutFormat;
  img.cg = UHDR_CG_UNSPECIFIED;
  img.ct = UHDR_CT_UNSPECIFIED;
  img.range = UHDR_CR_FULL_RANGE;
  img.w = mPlaneWidth[0];
  img.h = mPlaneHeight[0];
  uint8_t* data = mResultBuffer.data();
  for (int i = 0; i < 3; i++) {
    if (i < (int)mNumComponents && (mOutFormat != UHDR_IMG_FMT_32bppRGBA8888 || i == 0)) {
      img.planes[i] = data;
      img.stride[i] = mPlaneHStride[i];
      data += (size_t)mPlaneHStride[i] * mPlaneVStride[i];
    } else {
      img.planes[i] = nullptr;
      img.stride[i] = 0;
    }
  }
  return img;
}

// ---- JpegR ---------------------------------------------------------------------------------------
JpegR::JpegR(void* uhdrGLESCtxt, int mapDimensionScaleFactor, int mapCompressQuality, bool useMultiChannelGainMap, float gamma,
             uhdr_enc_preset_t preset, float minContentBoost, float maxContentBoost, float targetDispPeakBrightness)
    : UltraHdr(uhdrGLESCtxt, mapDimensionScaleFactor, mapCompressQuality, useMultiChannelGainMap, gamma, preset, minContentBoost,
               maxContentBoost, targetDispPeakBrightness) {}

#define SURFACE_CFG()                                                                                                              \
  make_cfg(mMapDimensionScaleFactor, mMapCompressQuality, mUseMultiChannelGainMap, mGamma, mEncPreset, mMinContentBoost, \
           mMaxContentBoost, mTargetDispPeakBrightness)

static uhdr_error_info_t encode_raw(const uhdr_b200_gm_config_t& cfg, uhdr_raw_image_t* hdr, uhdr_raw_image_t* sdr,
                                    uhdr_compressed_image_t* dest, int quality, uhdr_mem_block_t* exif) {
  if (!hdr || !dest || !dest->data) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for an image descriptor");
  int rc;
  JpegRCodec* c = tls_codec(&rc);
  if (!c) return from_rc(rc);
  size_t n = 0;
  rc = c->encode_host(*hdr, sdr, cfg, quality, exif ? (const uint8_t*)exif->data : nullptr, exif ? exif->data_sz : 0,
                      (uint8_t*)dest->data, dest->capacity, &n);
  if (rc) return from_rc(rc);
  dest->data_sz = n;
  return ok();
}

uhdr_error_info_t JpegR::encodeJPEGR(uhdr_raw_image_t* hdr_intent, uhdr_compressed_image_t* dest, int quality, uhdr_mem_block_t* exif) {
  return encode_raw(SURFACE_CFG(), hdr_intent, nullptr, dest, quality, exif);
}
uhdr_error_info_t JpegR::encodeJPEGR(uhdr_raw_image_t* hdr_intent, uhdr_raw_image_t* sdr_intent, uhdr_compressed_image_t* dest,
                                     int quality, uhdr_mem_block_t* exif) {
  if (!sdr_intent) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for sdr intent image descriptor");
  return encode_raw(SURFACE_CFG(), hdr_intent, sdr_intent, dest, quality, exif);
}

static uhdr_error_info_t encode_with_jpg(const uhdr_b200_gm_config_t& cfg, uhdr_raw_image_t* hdr, uhdr_raw_image_t* sdr,
                                         uhdr_compressed_image_t* sdr_jpg, uhdr_compressed_image_t* dest) {
  if (!hdr || !sdr_jpg || !sdr_jpg->data || !dest || !dest->data) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for an image descriptor");
  int rc;
  JpegRCodec* c = tls_codec(&rc);
  if (!c) return from_rc(rc);
  Workspace& ws = c->ws();
  DevImage dh, ds;
  if ((rc = upload_image(ws, *hdr, &dh))) return from_rc(rc);
  if (sdr && (rc = upload_image(ws, *sdr, &ds))) return from_rc(rc);
  size_t n = 0;
  rc = c->encode_with_compressed_sdr(dh, sdr ? &ds : nullptr, (const uint8_t*)sdr_jpg->data, sdr_jpg->data_sz, sdr_jpg->cg, cfg,
                                     (uint8_t*)dest->data, dest->capacity, &n);
  if (rc) return from_rc(rc);
  dest->data_sz = n;
  return ok();
}
uhdr_error_info_t JpegR::encodeJPEGR(uhdr_raw_image_t* hdr_intent, uhdr_raw_image_t* sdr_intent,
                                     uhdr_compressed_image_t* sdr_intent_compressed, uhdr_compressed_image_t* dest) {
  if (!sdr_intent) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for sdr intent image descriptor");
  return encode_with_jpg(SURFACE_CFG(), hdr_intent, sdr_intent, sdr_intent_compressed, dest);
}
uhdr_error_info_t JpegR::encodeJPEGR(uhdr_raw_image_t* hdr_intent, uhdr_compressed_image_t* sdr_intent_compressed,
                                     uhdr_compressed_image_t* dest) {
  return encode_with_jpg(SURFACE_CFG(), hdr_intent, nullptr, sdr_intent_compressed, dest);
}
uhdr_error_info_t JpegR::encodeJPEGR(uhdr_compressed_image_t* base_img_compressed, uhdr_compressed_image_t* gainmap_img_compressed,
                                     uhdr_gainmap_metadata_ext_t* metadata, uhdr_compressed_image_t* dest) {
  if (!base_img_compressed || !base_img_compressed->data || !gainmap_img_compressed || !gainmap_img_compressed->data || !metadata ||
      !dest || !dest->data)
    return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for an image descriptor");
  size_t n = 0;
  const int rc = JpegRCodec::encode_from_compressed((const uint8_t*)base_img_compressed->data, base_img_compressed->data_sz,
                                                    base_img_compressed->cg, (const uint8_t*)gainmap_img_compressed->data,
                                                    gainmap_img_compressed->data_sz, *metadata, (uint8_t*)dest->data, dest->capacity, &n);
  if (rc) return from_rc(rc);
  dest->data_sz = n;
  return ok();
}

uhdr_error_info_t JpegR::decodeJPEGR(uhdr_compressed_image_t* uhdr_compressed_img, uhdr_raw_image_t* dest, float max_display_boost,
                                     uhdr_color_transfer_t output_ct, uhdr_img_fmt_t output_format, uhdr_raw_image_t* gainmap_img,
                                     uhdr_gainmap_metadata_t* gainmap_metadata) {
  if (!uhdr_compressed_img || !uhdr_compressed_img->data || !dest || !dest->planes[0])
    return err(UHDR_CODEC_INVALID_PARAM, "received nullptr for an image descriptor");
  int rc;
  JpegRCodec* c = tls_codec(&rc);
  if (!c) return from_rc(rc);
  c->set_lazy_gainmap(false);
  if (gainmap_img && gainmap_img->planes[0]) {  // copy_raw_image (gainmapmath.cpp:1492-1502) refuses a size mismatch
    DecodedInfo info;
    if ((rc = c->probe((const uint8_t*)uhdr_compressed_img->data, uhdr_compressed_img->data_sz, &info))) return from_rc(rc);
    if ((int)gainmap_img->w != info.gm_width || (int)gainmap_img->h != info.gm_height) {
      uhdr_error_info_t s = err(UHDR_CODEC_MEM_ERROR, "");
      snprintf(s.detail, sizeof s.detail, "destination image dimensions %dx%d and source image dimensions %dx%d are not identical for "
               "copy_raw_image", gainmap_img->w, gainmap_img->h, info.gm_width, info.gm_height);
      return s;
    }
  }
  dest->fmt = output_format;
  rc = c->decode((const uint8_t*)uhdr_compressed_img->data, uhdr_compressed_img->data_sz, output_ct, output_format, max_display_boost,
                 dest, gainmap_img, gainmap_metadata);
  return from_rc(rc);
}

static void fill_info(const uint8_t* d, size_t n, const JpegHeader& h, j_info_ptr info) {  // parseJpegInfo :1900-1943
  if (!info) return;
  info->width = h.frame.width;
  info->height = h.frame.height;
  info->numComponents = h.frame.ncomp;
  info->imgData.assign(d, d + n);
  take_marker(d, h, 0xE2, "ICC_PROFILE", 12, &info->iccData, nullptr);
  take_marker(d, h, 0xE1, "Exif\0\0", 6, &info->exifData, nullptr);
  take_marker(d, h, 0xE1, "http://ns.adobe.com/xap/1.0/", 29, &info->xmpData, nullptr);
  take_marker(d, h, 0xE2, "urn:iso:std:iso:ts:21496:-1", 28, &info->isoData, nullptr);
}

uhdr_error_info_t JpegR::getJPEGRInfo(uhdr_compressed_image_t* uhdr_compressed_img, jr_info_ptr uhdr_image_info) {
  if (!uhdr_compressed_img || !uhdr_compressed_img->data || !uhdr_image_info) return err(UHDR_CODEC_INVALID_PARAM, "received nullptr argument");
  const uint8_t* d = (const uint8_t*)uhdr_compressed_img->data;
  size_t po, pl, go, gl;
  int rc = split_jpegr(d, uhdr_compressed_img->data_sz, &po, &pl, &go, &gl);
  if (rc) return from_rc(rc);
  JpegHeader ph, gh;
  if ((rc = jpeg_read_header(d + po, pl, &ph))) return from_rc(rc);
  fill_info(d + po, pl, ph, uhdr_image_info->primaryImgInfo);
  uhdr_image_info->width = ph.frame.width;
  uhdr_image_info->height = ph.frame.height;
  if (uhdr_image_info->gainmapImgInfo) {
    if ((rc = jpeg_read_header(d + go, gl, &gh))) return from_rc(rc);
    fill_info(d + go, gl, gh, uhdr_image_info->gainmapImgInfo);
  }
  return ok();
}

// ---- deprecated aliases (jpegr.cpp:2224-2890) ------------------------------------------------------
status_t JpegR::areInputArgumentsValid(jr_uncompressed_ptr p010, jr_uncompressed_ptr yuv420, ultrahdr_transfer_function hdr_tf,
                                       jr_compressed_ptr dest_ptr) {
  if (p010 == nullptr || p010->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (p010->width % 2 != 0 || p010->height % 2 != 0) return ERROR_JPEGR_UNSUPPORTED_WIDTH_HEIGHT;
  if ((int)p010->width < kMinWidth || (int)p010->height < kMinHeight) return ERROR_JPEGR_UNSUPPORTED_WIDTH_HEIGHT;
  if ((int)p010->width > kMaxWidth || (int)p010->height > kMaxHeight) return ERROR_JPEGR_UNSUPPORTED_WIDTH_HEIGHT;
  if (p010->colorGamut <= ULTRAHDR_COLORGAMUT_UNSPECIFIED || p010->colorGamut > ULTRAHDR_COLORGAMUT_MAX) return ERROR_JPEGR_INVALID_COLORGAMUT;
  if (p010->luma_stride != 0 && p010->luma_stride < p010->width) return ERROR_JPEGR_INVALID_STRIDE;
  if (p010->chroma_data != nullptr && p010->chroma_stride < p010->width) return ERROR_JPEGR_INVALID_STRIDE;
  if (dest_ptr == nullptr || dest_ptr->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (hdr_tf <= ULTRAHDR_TF_UNSPECIFIED || hdr_tf > ULTRAHDR_TF_MAX || hdr_tf == ULTRAHDR_TF_SRGB) return ERROR_JPEGR_INVALID_TRANS_FUNC;
  if (mMapDimensionScaleFactor <= 0 || mMapDimensionScaleFactor > 128) return ERROR_JPEGR_UNSUPPORTED_MAP_SCALE_FACTOR;
  if (mMapCompressQuality < 0 || mMapCompressQuality > 100) return ERROR_JPEGR_INVALID_QUALITY_FACTOR;
  if (!std::isfinite(mGamma) || mGamma <= 0.0f) return ERROR_JPEGR_INVALID_GAMMA;
  if (mEncPreset != UHDR_USAGE_REALTIME && mEncPreset != UHDR_USAGE_BEST_QUALITY) return ERROR_JPEGR_INVALID_ENC_PRESET;
  if (!std::isfinite(mMinContentBoost) || !std::isfinite(mMaxContentBoost) || mMaxContentBoost < mMinContentBoost ||
      mMinContentBoost <= 0.0f)
    return ERROR_JPEGR_INVALID_DISPLAY_BOOST;
  if ((!std::isfinite(mTargetDispPeakBrightness) || mTargetDispPeakBrightness < 203.0f || mTargetDispPeakBrightness > 10000.0f) &&
      mTargetDispPeakBrightness != -1.0f)
    return ERROR_JPEGR_INVALID_TARGET_DISP_PEAK_BRIGHTNESS;
  if (yuv420 == nullptr) return JPEGR_NO_ERROR;
  if (yuv420->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (yuv420->luma_stride != 0 && yuv420->luma_stride < yuv420->width) return ERROR_JPEGR_INVALID_STRIDE;
  if (yuv420->chroma_data != nullptr && yuv420->chroma_stride < yuv420->width / 2) return ERROR_JPEGR_INVALID_STRIDE;
  if (p010->width != yuv420->width || p010->height != yuv420->height) return ERROR_JPEGR_RESOLUTION_MISMATCH;
  if (yuv420->colorGamut <= ULTRAHDR_COLORGAMUT_UNSPECIFIED || yuv420->colorGamut > ULTRAHDR_COLORGAMUT_MAX) return ERROR_JPEGR_INVALID_COLORGAMUT;
  return JPEGR_NO_ERROR;
}
status_t JpegR::areInputArgumentsValid(jr_uncompressed_ptr p010, jr_uncompressed_ptr yuv420, ultrahdr_transfer_function hdr_tf,
                                       jr_compressed_ptr dest_ptr, int quality) {
  if (quality < 0 || quality > 100) return ERROR_JPEGR_INVALID_QUALITY_FACTOR;
  return areInputArgumentsValid(p010, yuv420, hdr_tf, dest_ptr);
}

static uhdr_raw_image_t p010_desc(const jpegr_uncompressed_struct& in, ultrahdr_transfer_function tf) {
  jpegr_uncompressed_struct p = in;
  if (p.luma_stride == 0) p.luma_stride = p.width;
  if (!p.chroma_data) {
    p.chroma_data = reinterpret_cast<uint16_t*>(p.data) + (size_t)p.luma_stride * p.height;
    p.chroma_stride = p.luma_stride;
  }
  uhdr_raw_image_t r;
  memset(&r, 0, sizeof r);
  r.fmt = UHDR_IMG_FMT_24bppYCbCrP010;
  r.cg = map_legacy_cg_to_cg(p.colorGamut);
  r.ct = map_legacy_ct_to_ct(tf);
  r.range = p.colorRange;
  r.w = p.width;
  r.h = p.height;
  r.planes[UHDR_PLANE_Y] = p.data;
  r.stride[UHDR_PLANE_Y] = p.luma_stride;
  r.planes[UHDR_PLANE_UV] = p.chroma_data;
  r.stride[UHDR_PLANE_UV] = p.chroma_stride;
  return r;
}
static uhdr_raw_image_t yuv420_desc(const jpegr_uncompressed_struct& in) {
  jpegr_uncompressed_struct y = in;
  if (y.luma_stride == 0) y.luma_stride = y.width;
  if (!y.chroma_data) {
    y.chroma_data = reinterpret_cast<uint8_t*>(y.data) + (size_t)y.luma_stride * y.height;
    y.chroma_stride = y.luma_stride >> 1;
  }
  uhdr_raw_image_t r;
  memset(&r, 0, sizeof r);
  r.fmt = UHDR_IMG_FMT_12bppYCbCr420;
  r.cg = map_legacy_cg_to_cg(y.colorGamut);
  r.ct = UHDR_CT_SRGB;
  r.range = y.colorRange;
  r.w = y.width;
  r.h = y.height;
  r.planes[UHDR_PLANE_Y] = y.data;
  r.stride[UHDR_PLANE_Y] = y.luma_stride;
  r.planes[UHDR_PLANE_U] = y.chroma_data;
  r.stride[UHDR_PLANE_U] = y.chroma_stride;
  r.planes[UHDR_PLANE_V] = reinterpret_cast<uint8_t*>(y.chroma_data) + ((size_t)y.height * y.chroma_stride) / 2;
  r.stride[UHDR_PLANE_V] = y.chroma_stride;
  return r;
}
static uhdr_compressed_image_t out_desc(jr_compressed_ptr dest) {
  uhdr_compressed_image_t o;
  o.data = dest->data;
  o.data_sz = 0;
  o.capacity = dest->maxLength;
  o.cg = UHDR_CG_UNSPECIFIED;
  o.ct = UHDR_CT_UNSPECIFIED;
  o.range = UHDR_CR_UNSPECIFIED;
  return o;
}
static uhdr_compressed_image_t in_desc(jr_compressed_ptr src) {
  uhdr_compressed_image_t i;
  i.data = src->data;
  i.data_sz = src->length;
  i.capacity = src->maxLength;
  i.cg = map_legacy_cg_to_cg(src->colorGamut);
  i.ct = UHDR_CT_UNSPECIFIED;
  i.range = UHDR_CR_UNSPECIFIED;
  return i;
}
static status_t finish(const uhdr_error_info_t& r, const uhdr_compressed_image_t& o, jr_compressed_ptr dest) {
  if (r.error_code == UHDR_CODEC_OK) {
    dest->colorGamut = map_cg_to_legacy_cg(o.cg);
    dest->length = o.data_sz;
    return JPEGR_NO_ERROR;
  }
  return JPEGR_UNKNOWN_ERROR;
}

status_t JpegR::encodeJPEGR(jr_uncompressed_ptr p010_image_ptr, ultrahdr_transfer_function hdr_tf, jr_compressed_ptr dest, int quality,
                            jr_exif_ptr exif) {
  JPEGR_CHECK(areInputArgumentsValid(p010_image_ptr, nullptr, hdr_tf, dest, quality));
  if (exif != nullptr && exif->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  uhdr_raw_image_t hdr = p010_desc(*p010_image_ptr, hdr_tf);
  uhdr_compressed_image_t o = out_desc(dest);
  uhdr_mem_block_t xb;
  if (exif) { xb.data = exif->data; xb.data_sz = xb.capacity = exif->length; }
  return finish(encodeJPEGR(&hdr, &o, quality, exif ? &xb : nullptr), o, dest);
}
status_t JpegR::encodeJPEGR(jr_uncompressed_ptr p010_image_ptr, jr_uncompressed_ptr yuv420_image_ptr, ultrahdr_transfer_function hdr_tf,
                            jr_compressed_ptr dest, int quality, jr_exif_ptr exif) {
  if (yuv420_image_ptr == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (exif != nullptr && exif->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  JPEGR_CHECK(areInputArgumentsValid(p010_image_ptr, yuv420_image_ptr, hdr_tf, dest, quality))
  uhdr_raw_image_t hdr = p010_desc(*p010_image_ptr, hdr_tf), sdr = yuv420_desc(*yuv420_image_ptr);
  uhdr_compressed_image_t o = out_desc(dest);
  uhdr_mem_block_t xb;
  if (exif) { xb.data = exif->data; xb.data_sz = xb.capacity = exif->length; }
  return finish(encodeJPEGR(&hdr, &sdr, &o, quality, exif ? &xb : nullptr), o, dest);
}
status_t JpegR::encodeJPEGR(jr_uncompressed_ptr p010_image_ptr, jr_uncompressed_ptr yuv420_image_ptr,
                            jr_compressed_ptr yuv420jpg_image_ptr, ultrahdr_transfer_function hdr_tf, jr_compressed_ptr dest) {
  if (yuv420_image_ptr == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (yuv420jpg_image_ptr == nullptr || yuv420jpg_image_ptr->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  JPEGR_CHECK(areInputArgumentsValid(p010_image_ptr, yuv420_image_ptr, hdr_tf, dest))
  uhdr_raw_image_t hdr = p010_desc(*p010_image_ptr, hdr_tf), sdr = yuv420_desc(*yuv420_image_ptr);
  uhdr_compressed_image_t in = in_desc(yuv420jpg_image_ptr), o = out_desc(dest);
  return finish(encodeJPEGR(&hdr, &sdr, &in, &o), o, dest);
}
status_t JpegR::encodeJPEGR(jr_uncompressed_ptr p010_image_ptr, jr_compressed_ptr yuv420jpg_image_ptr, ultrahdr_transfer_function hdr_tf,
                            jr_compressed_ptr dest) {
  if (yuv420jpg_image_ptr == nullptr || yuv420jpg_image_ptr->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  JPEGR_CHECK(areInputArgumentsValid(p010_image_ptr, nullptr, hdr_tf, dest))
  uhdr_raw_image_t hdr = p010_desc(*p010_image_ptr, hdr_tf);
  uhdr_compressed_image_t in = in_desc(yuv420jpg_image_ptr), o = out_desc(dest);
  return finish(encodeJPEGR(&hdr, &in, &o), o, dest);
}
status_t JpegR::encodeJPEGR(jr_compressed_ptr yuv420jpg_image_ptr, jr_compressed_ptr gainmapjpg_image_ptr, ultrahdr_metadata_ptr metadata,
                            jr_compressed_ptr dest) {
  if (yuv420jpg_image_ptr == nullptr || yuv420jpg_image_ptr->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (gainmapjpg_image_ptr == nullptr || gainmapjpg_image_ptr->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (dest == nullptr || dest->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (metadata == nullptr) return ERROR_JPEGR_BAD_PTR;
  uhdr_compressed_image_t in = in_desc(yuv420jpg_image_ptr), gm = in_desc(gainmapjpg_image_ptr), o = out_desc(dest);
  gm.cg = UHDR_CG_UNSPECIFIED;
  uhdr_gainmap_metadata_ext_t meta(metadata->version);
  meta.hdr_capacity_max = metadata->hdrCapacityMax;
  meta.hdr_capacity_min = metadata->hdrCapacityMin;
  std::fill_n(meta.gamma, 3, metadata->gamma);
  std::fill_n(meta.offset_sdr, 3, metadata->offsetSdr);
  std::fill_n(meta.offset_hdr, 3, metadata->offsetHdr);
  std::fill_n(meta.max_content_boost, 3, metadata->maxContentBoost);
  std::fill_n(meta.min_content_boost, 3, metadata->minContentBoost);
  meta.use_base_cg = true;
  return finish(encodeJPEGR(&in, &gm, &meta, &o), o, dest);
}

status_t JpegR::getJPEGRInfo(jr_compressed_ptr jpegr_image_ptr, jr_info_ptr jpegr_image_info_ptr) {
  if (jpegr_image_ptr == nullptr || jpegr_image_ptr->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (jpegr_image_info_ptr == nullptr) return ERROR_JPEGR_BAD_PTR;
  uhdr_compressed_image_t in = in_desc(jpegr_image_ptr);
  return getJPEGRInfo(&in, jpegr_image_info_ptr).error_code == UHDR_CODEC_OK ? JPEGR_NO_ERROR : JPEGR_UNKNOWN_ERROR;
}

status_t JpegR::decodeJPEGR(jr_compressed_ptr jpegr_image_ptr, jr_uncompressed_ptr dest, float max_display_boost, jr_exif_ptr exif,
                            ultrahdr_output_format output_format, jr_uncompressed_ptr gainmap_image_ptr, ultrahdr_metadata_ptr metadata) {
  if (jpegr_image_ptr == nullptr || jpegr_image_ptr->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (dest == nullptr || dest->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (max_display_boost < 1.0f) return ERROR_JPEGR_INVALID_DISPLAY_BOOST;
  if (exif != nullptr && exif->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (gainmap_image_ptr != nullptr && gainmap_image_ptr->data == nullptr) return ERROR_JPEGR_BAD_PTR;
  if (output_format <= ULTRAHDR_OUTPUT_UNSPECIFIED || output_format > ULTRAHDR_OUTPUT_MAX) return ERROR_JPEGR_INVALID_OUTPUT_FORMAT;
  uhdr_color_transfer_t ct = UHDR_CT_SRGB;
  uhdr_img_fmt_t fmt = UHDR_IMG_FMT_32bppRGBA8888;
  if (output_format == ULTRAHDR_OUTPUT_HDR_HLG) { fmt = UHDR_IMG_FMT_32bppRGBA1010102; ct = UHDR_CT_HLG; }
  else if (output_format == ULTRAHDR_OUTPUT_HDR_PQ) { fmt = UHDR_IMG_FMT_32bppRGBA1010102; ct = UHDR_CT_PQ; }
  else if (output_format == ULTRAHDR_OUTPUT_HDR_LINEAR) { fmt = UHDR_IMG_FMT_64bppRGBAHalfFloat; ct = UHDR_CT_LINEAR; }
  uhdr_compressed_image_t in = in_desc(jpegr_image_ptr);
  jpeg_info_struct primary_image, gainmap_image;
  jpegr_info_struct info;
  info.primaryImgInfo = &primary_image;
  info.gainmapImgInfo = &gainmap_image;
  if (getJPEGRInfo(&in, &info).error_code != UHDR_CODEC_OK) return JPEGR_UNKNOWN_ERROR;
  if (exif != nullptr) {
    if (exif->length < primary_image.exifData.size()) return ERROR_JPEGR_BUFFER_TOO_SMALL;
    memcpy(exif->data, primary_image.exifData.data(), primary_image.exifData.size());
    exif->length = primary_image.exifData.size();
  }
  uhdr_raw_image_t out;
  memset(&out, 0, sizeof out);
  out.fmt = fmt;
  out.cg = UHDR_CG_UNSPECIFIED;
  out.ct = UHDR_CT_UNSPECIFIED;
  out.range = UHDR_CR_UNSPECIFIED;
  out.w = info.width;
  out.h = info.height;
  out.planes[UHDR_PLANE_PACKED] = dest->data;
  out.stride[UHDR_PLANE_PACKED] = info.width;
  // (the reference fills the primary descriptor a second time here instead of the gain-map one and then
  // hands an uninitialised descriptor to decodeJPEGR, jpegr.cpp:2841-2856; what it means to do is this)
  uhdr_raw_image_t out_gm;
  memset(&out_gm, 0, sizeof out_gm);
  if (gainmap_image_ptr) {
    out_gm.fmt = gainmap_image.numComponents == 1 ? UHDR_IMG_FMT_8bppYCbCr400 : UHDR_IMG_FMT_32bppRGBA8888;
    out_gm.cg = UHDR_CG_UNSPECIFIED;
    out_gm.ct = UHDR_CT_UNSPECIFIED;
    out_gm.range = UHDR_CR_UNSPECIFIED;
    out_gm.w = gainmap_image.width;
    out_gm.h = gainmap_image.height;
    out_gm.planes[UHDR_PLANE_PACKED] = gainmap_image_ptr->data;
    out_gm.stride[UHDR_PLANE_PACKED] = gainmap_image.width;
  }
  uhdr_gainmap_metadata_ext_t meta;
  const uhdr_error_info_t r = decodeJPEGR(&in, &out, max_display_boost, ct, fmt, gainmap_image_ptr ? &out_gm : nullptr,
                                          metadata ? &meta : nullptr);
  if (r.error_code != UHDR_CODEC_OK) return JPEGR_UNKNOWN_ERROR;
  dest->width = out.w;
  dest->height = out.h;
  dest->colorGamut = map_cg_to_legacy_cg(out.cg);
  dest->colorRange = out.range;
  dest->pixelFormat = out.fmt;
  dest->chroma_data = nullptr;
  if (gainmap_image_ptr) {
    gainmap_image_ptr->width = out_gm.w;
    gainmap_image_ptr->height = out_gm.h;
    gainmap_image_ptr->colorGamut = map_cg_to_legacy_cg(out_gm.cg);
    gainmap_image_ptr->colorRange = out_gm.range;
    gainmap_image_ptr->pixelFormat = out_gm.fmt;
    gainmap_image_ptr->chroma_data = nullptr;
  }
  if (metadata) {
    if (!meta.are_all_channels_identical()) return ERROR_JPEGR_METADATA_ERROR;
    metadata->version = meta.version;  // (the reference's decode leaves it empty)
    metadata->hdrCapacityMax = meta.hdr_capacity_max;
    metadata->hdrCapacityMin = meta.hdr_capacity_min;
    metadata->gamma = meta.gamma[0];
    metadata->offsetSdr = meta.offset_sdr[0];
    metadata->offsetHdr = meta.offset_hdr[0];
    metadata->maxContentBoost = meta.max_content_boost[0];
    metadata->minContentBoost = meta.min_content_boost[0];
  }
  return JPEGR_NO_ERROR;
}

}  // namespace ultrahdr
#pragma GCC visibility pop
