/*
 * ultrahdr/jpegr.h -- the reference's ultrahdr::JpegR surface
 * (lib/include/ultrahdr/jpegr.h:25-276) implemented by libuhdr_b200.so: constructor,
 * the five encodeJPEGR overloads (API-0 .. API-4), decodeJPEGR, getJPEGRInfo and the seven deprecated
 * jr_* overloads (bodies lib/src/jpegr.cpp:179-434, 1417-1531, 2224-2890).  Pixel and
 * block stages run on the device (sm_90a); a JpegR object is cheap and, like the reference's, not
 * thread safe.
 */
#ifndef UHDR_B200_ULTRAHDR_JPEGR_H
#define UHDR_B200_ULTRAHDR_JPEGR_H

#include <array>
#include <cfloat>
#include <vector>

#include "ultrahdr_api.h"
#include "ultrahdr/jpegdecoderhelper.h"
#include "ultrahdr/jpegencoderhelper.h"
#include "ultrahdr/ultrahdr.h"
#include "ultrahdr/ultrahdrcommon.h"

namespace ultrahdr {

/* ref jpegr.h:25-35 */
struct jpeg_info_struct {
  std::vector<uint8_t> imgData = std::vector<uint8_t>(0);
  std::vector<uint8_t> iccData = std::vector<uint8_t>(0);
  std::vector<uint8_t> exifData = std::vector<uint8_t>(0);
  std::vector<uint8_t> xmpData = std::vector<uint8_t>(0);
  std::vector<uint8_t> isoData = std::vector<uint8_t>(0);
  unsigned int width;
  unsigned int height;
  unsigned int numComponents;
};
/* ref jpegr.h:40-47 */
struct jpegr_info_struct {
  unsigned int width;
  unsigned int height;
  jpeg_info_struct* primaryImgInfo = nullptr;
  jpeg_info_struct* gainmapImgInfo = nullptr;
};
typedef struct jpeg_info_struct* j_info_ptr;
typedef struct jpegr_info_struct* jr_info_ptr;

class JpegR : public UltraHdr {
 public:
  /* ref jpegr.h:54-60 */
  JpegR(void* uhdrGLESCtxt = nullptr, int mapDimensionScaleFactor = kMapDimensionScaleFactorAndroidDefault,
        int mapCompressQuality = kMapCompressQualityAndroidDefault,
        bool useMultiChannelGainMap = kUseMultiChannelGainMapAndroidDefault, float gamma = kGainMapGammaDefault,
        uhdr_enc_preset_t preset = kEncSpeedPresetAndroidDefault, float minContentBoost = FLT_MIN,
        float maxContentBoost = FLT_MAX, float targetDispPeakBrightness = -1.0f);

  /* Encode API-0 (ref :81-82): hdr intent -> tone map -> gain map -> two JPEGs -> JPEG/R */
  uhdr_error_info_t encodeJPEGR(uhdr_raw_image_t* hdr_intent, uhdr_compressed_image_t* dest, int quality, uhdr_mem_block_t* exif);
  /* Encode API-1 (ref :101-102) */
  uhdr_error_info_t encodeJPEGR(uhdr_raw_image_t* hdr_intent, uhdr_raw_image_t* sdr_intent, uhdr_compressed_image_t* dest,
                                int quality, uhdr_mem_block_t* exif);
  /* Encode API-2 (ref :123-125) */
  uhdr_error_info_t encodeJPEGR(uhdr_raw_image_t* hdr_intent, uhdr_raw_image_t* sdr_intent,
                                uhdr_compressed_image_t* sdr_intent_compressed, uhdr_compressed_image_t* dest);
  /* Encode API-3 (ref :143-145) */
  uhdr_error_info_t encodeJPEGR(uhdr_raw_image_t* hdr_intent, uhdr_compressed_image_t* sdr_intent_compressed,
                                uhdr_compressed_image_t* dest);
  /* Encode API-4 (ref :162-165) */
  uhdr_error_info_t encodeJPEGR(uhdr_compressed_image_t* base_img_compressed, uhdr_compressed_image_t* gainmap_img_compressed,
                                uhdr_gainmap_metadata_ext_t* metadata, uhdr_compressed_image_t* dest);
  /* Decode (ref :204-209).  dest->planes[0] (and gainmap_img->planes[0]) are caller memory; the supported
   * (output_ct, output_format) pairs are SRGB/RGBA8888, LINEAR/RGBAHalfFloat, PQ|HLG/RGBA1010102. */
  uhdr_error_info_t decodeJPEGR(uhdr_compressed_image_t* uhdr_compressed_img, uhdr_raw_image_t* dest,
                                float max_display_boost = FLT_MAX, uhdr_color_transfer_t output_ct = UHDR_CT_LINEAR,
                                uhdr_img_fmt_t output_format = UHDR_IMG_FMT_64bppRGBAHalfFloat,
                                uhdr_raw_image_t* gainmap_img = nullptr, uhdr_gainmap_metadata_t* gainmap_metadata = nullptr);
  /* ref :219-220 */
  uhdr_error_info_t getJPEGRInfo(uhdr_compressed_image_t* uhdr_compressed_img, jr_info_ptr uhdr_image_info);

  /* deprecated aliases, ref :226-276 */
  status_t encodeJPEGR(jr_uncompressed_ptr p010_image_ptr, ultrahdr_transfer_function hdr_tf, jr_compressed_ptr dest, int quality,
                       jr_exif_ptr exif);
  status_t encodeJPEGR(jr_uncompressed_ptr p010_image_ptr, jr_uncompressed_ptr yuv420_image_ptr, ultrahdr_transfer_function hdr_tf,
                       jr_compressed_ptr dest, int quality, jr_exif_ptr exif);
  status_t encodeJPEGR(jr_uncompressed_ptr p010_image_ptr, jr_uncompressed_ptr yuv420_image_ptr,
                       jr_compressed_ptr yuv420jpg_image_ptr, ultrahdr_transfer_function hdr_tf, jr_compressed_ptr dest);
  status_t encodeJPEGR(jr_uncompressed_ptr p010_image_ptr, jr_compressed_ptr yuv420jpg_image_ptr,
                       ultrahdr_transfer_function hdr_tf, jr_compressed_ptr dest);
  status_t encodeJPEGR(jr_compressed_ptr yuv420jpg_image_ptr, jr_compressed_ptr gainmapjpg_image_ptr,
                       ultrahdr_metadata_ptr metadata, jr_compressed_ptr dest);
  status_t decodeJPEGR(jr_compressed_ptr jpegr_image_ptr, jr_uncompressed_ptr dest, float max_display_boost = FLT_MAX,
                       jr_exif_ptr exif = nullptr, ultrahdr_output_format output_format = ULTRAHDR_OUTPUT_HDR_LINEAR,
                       jr_uncompressed_ptr gainmap_image_ptr = nullptr, ultrahdr_metadata_ptr metadata = nullptr);
  status_t getJPEGRInfo(jr_compressed_ptr jpegr_image_ptr, jr_info_ptr jpegr_image_info_ptr);

 private:
  /* argument checks of the deprecated entry points, ref jpegr.cpp:2224-2346 */
  status_t areInputArgumentsValid(jr_uncompressed_ptr p010_image_ptr, jr_uncompressed_ptr yuv420_image_ptr,
                                  ultrahdr_transfer_function hdr_tf, jr_compressed_ptr dest_ptr);
  status_t areInputArgumentsValid(jr_uncompressed_ptr p010_image_ptr, jr_uncompressed_ptr yuv420_image_ptr,
                                  ultrahdr_transfer_function hdr_tf, jr_compressed_ptr dest_ptr, int quality);
};

/* ref jpegr.cpp:2349-2390 (declared by the reference in ultrahdrcommon-using translation units) */
uhdr_color_transfer_t map_legacy_ct_to_ct(ultrahdr::ultrahdr_transfer_function ct);
uhdr_color_gamut_t map_legacy_cg_to_cg(ultrahdr::ultrahdr_color_gamut cg);
ultrahdr::ultrahdr_color_gamut map_cg_to_legacy_cg(uhdr_color_gamut_t cg);

}  // namespace ultrahdr

#endif
