/*
 * ultrahdr/ultrahdrcommon.h -- libuhdr_b200's declaration of the reference's common C++ surface
 * (lib/include/ultrahdr/ultrahdrcommon.h:158-229 owning descriptors, :424-457
 * defaults, :471-546 class UltraHdr, :677 globalTonemap).  Member signatures are the reference's; the
 * bodies live in libuhdr_b200.so and run the CUDA (sm_90a) stages.  There is no CPU fallback: every
 * stage method returns UHDR_CODEC_ERROR with a CUDA message when no device is usable.
 */
#ifndef UHDR_B200_ULTRAHDR_ULTRAHDRCOMMON_H
#define UHDR_B200_ULTRAHDR_ULTRAHDRCOMMON_H

#include <algorithm>
#include <array>
#include <cfloat>
#include <cstdint>
#include <cstdio>
#include <memory>
#include <string>

#include "ultrahdr_api.h"

#define UHDR_ERR_CHECK(x)                                     \
  {                                                           \
    uhdr_error_info_t uhdr_err_check_st = (x);                \
    if (uhdr_err_check_st.error_code != UHDR_CODEC_OK) return uhdr_err_check_st; \
  }

static const uhdr_error_info_t g_no_error = {UHDR_CODEC_OK, 0, ""};

namespace ultrahdr {

/* ref ultrahdrcommon.h:164-165, jpegdecoderhelper.cpp:46-60 */
extern const int kMinWidth, kMinHeight;
extern const int kMaxWidth, kMaxHeight;

/* ref ultrahdrcommon.h:167-175 */
typedef struct uhdr_memory_block {
  explicit uhdr_memory_block(size_t capacity);
  std::unique_ptr<uint8_t[]> m_buffer;
  size_t m_capacity;
} uhdr_memory_block_t;

/* ref ultrahdrcommon.h:177-186, ultrahdr_api.cpp:50-117: owning raw image, planes contiguous, zero
 * initialised, stride aligned to `align_stride_to` pixels */
typedef struct uhdr_raw_image_ext : uhdr_raw_image_t {
  uhdr_raw_image_ext(uhdr_img_fmt_t fmt, uhdr_color_gamut_t cg, uhdr_color_transfer_t ct, uhdr_color_range_t range,
                     unsigned w, unsigned h, unsigned align_stride_to);

 private:
  std::unique_ptr<ultrahdr::uhdr_memory_block> m_block;
} uhdr_raw_image_ext_t;

/* ref ultrahdrcommon.h:188-196 */
typedef struct uhdr_compressed_image_ext : uhdr_compressed_image_t {
  uhdr_compressed_image_ext(uhdr_color_gamut_t cg, uhdr_color_transfer_t ct, uhdr_color_range_t range, size_t sz);

 private:
  std::unique_ptr<ultrahdr::uhdr_memory_block> m_block;
} uhdr_compressed_image_ext_t;

/* ref ultrahdrcommon.h:201-229 */
typedef struct uhdr_gainmap_metadata_ext : uhdr_gainmap_metadata {
  uhdr_gainmap_metadata_ext() {}
  explicit uhdr_gainmap_metadata_ext(std::string ver) : version(ver) {}
  uhdr_gainmap_metadata_ext(uhdr_gainmap_metadata& metadata, std::string ver) : uhdr_gainmap_metadata_ext(ver) {
    static_cast<uhdr_gainmap_metadata&>(*this) = metadata;
  }
  bool are_all_channels_identical() const {
    for (int c = 1; c < 3; c++)
      if (max_content_boost[c] != max_content_boost[0] || min_content_boost[c] != min_content_boost[0] || gamma[c] != gamma[0] ||
          offset_sdr[c] != offset_sdr[0] || offset_hdr[c] != offset_hdr[0])
        return false;
    return true;
  }
  std::string version;
} uhdr_gainmap_metadata_ext_t;

/* ref ultrahdrcommon.h:330, ultrahdr_api.cpp:431-503 */
uhdr_error_info_t uhdr_validate_gainmap_metadata_descriptor(uhdr_gainmap_metadata_t* metadata);

/* ref ultrahdrcommon.h:424-457 */
static const int kMapDimensionScaleFactorDefault = 1;
static const int kMapDimensionScaleFactorAndroidDefault = 4;
static const int kBaseCompressQualityDefault = 95;
static const int kMapCompressQualityDefault = 95;
static const int kMapCompressQualityAndroidDefault = 85;
static const bool kUseMultiChannelGainMapDefault = true;
static const bool kUseMultiChannelGainMapAndroidDefault = false;
static const uhdr_enc_preset_t kEncSpeedPresetDefault = UHDR_USAGE_BEST_QUALITY;
static const uhdr_enc_preset_t kEncSpeedPresetAndroidDefault = UHDR_USAGE_REALTIME;
static const float kGainMapGammaDefault = 1.0f;
static const char* const kJpegrVersion = "1.0";

/* ref ultrahdrcommon.h:471-546.  Descriptors carry HOST pointers, like in the reference; each call
 * uploads, runs the device stage and downloads (the *_dev entry points of uhdr_b200.h skip the copies). */
class UltraHdr {
 public:
  UltraHdr(void* uhdrGLESCtxt = nullptr, int mapDimensionScaleFactor = kMapDimensionScaleFactorAndroidDefault,
           int mapCompressQuality = kMapCompressQualityAndroidDefault,
           bool useMultiChannelGainMap = kUseMultiChannelGainMapAndroidDefault, float gamma = kGainMapGammaDefault,
           uhdr_enc_preset_t preset = kEncSpeedPresetAndroidDefault, float minContentBoost = FLT_MIN,
           float maxContentBoost = FLT_MAX, float targetDispPeakBrightness = -1.0f);

  /* jpegr.cpp:1432-1466: ISO 21496-1 block if present, else hdrgm XMP (exif: Apple headroom fallback) */
  uhdr_error_info_t parseGainMapMetadata(uint8_t* iso_data, size_t iso_size, uint8_t* xmp_data, size_t xmp_size,
                                         uint8_t* exif_data, int exif_size, uhdr_gainmap_metadata_ext_t* uhdr_metadata);
  /* jpegr.cpp:1985-2222 */
  uhdr_error_info_t toneMap(uhdr_raw_image_t* hdr_intent, uhdr_raw_image_t* sdr_intent);
  /* jpegr.cpp:530-1058; allocates gainmap_img like the reference (:714) */
  uhdr_error_info_t generateGainMap(uhdr_raw_image_t* sdr_intent, uhdr_raw_image_t* hdr_intent,
                                    uhdr_gainmap_metadata_ext_t* gainmap_metadata,
                                    std::unique_ptr<uhdr_raw_image_ext_t>& gainmap_img, bool sdr_is_601 = false,
                                    bool use_luminance = true);
  /* jpegr.cpp:1533-1831 */
  uhdr_error_info_t applyGainMap(uhdr_raw_image_t* sdr_intent, uhdr_raw_image_t* gainmap_img,
                                 uhdr_gainmap_metadata_ext_t* gainmap_metadata, uhdr_color_transfer_t output_ct,
                                 uhdr_img_fmt_t output_format, float max_display_boost, uhdr_raw_image_t* dest);
  /* jpegr.cpp:436-518, in place */
  uhdr_error_info_t convertYuv(uhdr_raw_image_t* image, uhdr_color_gamut_t src_encoding, uhdr_color_gamut_t dst_encoding);

 protected:
  void setMapDimensionScaleFactor(int v) { mMapDimensionScaleFactor = v; }
  int getMapDimensionScaleFactor() { return mMapDimensionScaleFactor; }
  void setMapCompressQuality(int v) { mMapCompressQuality = v; }
  int getMapCompressQuality() { return mMapCompressQuality; }
  void setGainMapGamma(float v) { mGamma = v; }
  float getGainMapGamma() { return mGamma; }
  void setUseMultiChannelGainMap(bool v) { mUseMultiChannelGainMap = v; }
  bool isUsingMultiChannelGainMap() { return mUseMultiChannelGainMap; }
  void setGainMapMinMaxContentBoost(float mn, float mx) { mMinContentBoost = mn; mMaxContentBoost = mx; }
  void getGainMapMinMaxContentBoost(float& mn, float& mx) { mn = mMinContentBoost; mx = mMaxContentBoost; }

  void* mUhdrGLESCtxt;              // unused: there is no OpenGL ES path
  int mMapDimensionScaleFactor;
  int mMapCompressQuality;
  bool mUseMultiChannelGainMap;
  float mGamma;
  uhdr_enc_preset_t mEncPreset;
  float mMinContentBoost;
  float mMaxContentBoost;
  float mTargetDispPeakBrightness;
};

/* ref ultrahdrcommon.h:668-677 / jpegr.cpp:1951-1977: host scalar form of the tone-mapping operator
 * the toneMap kernel applies per pixel */
struct GlobalTonemapOutputs {
  std::array<float, 3> rgb_out;
  float y_hdr;
  float y_sdr;
};
GlobalTonemapOutputs globalTonemap(const std::array<float, 3>& rgb_in, float headroom, bool is_normalized);

}  // namespace ultrahdr

#endif
