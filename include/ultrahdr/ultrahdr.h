/*
 * ultrahdr/ultrahdr.h -- libuhdr_b200's declaration of the reference's LEGACY C++ vocabulary
 * (lib/include/ultrahdr/ultrahdr.h:28-196): status codes, legacy enums and the
 * jr_* descriptors the deprecated JpegR overloads take.  Same names, same values, same field
 * order, so code written against the reference header compiles unchanged; implemented by
 * libuhdr_b200.so (CUDA, sm_90a).
 */
#ifndef UHDR_B200_ULTRAHDR_ULTRAHDR_H
#define UHDR_B200_ULTRAHDR_ULTRAHDR_H

#include <string>

#include "ultrahdr_api.h"

namespace ultrahdr {

#define JPEGR_CHECK(x)                         \
  {                                            \
    ::ultrahdr::status_t jpegr_check_st = (x); \
    if (jpegr_check_st != ::ultrahdr::JPEGR_NO_ERROR) return jpegr_check_st; \
  }

/* ref ultrahdr.h:37-76 */
typedef enum {
  JPEGR_NO_ERROR = 0,
  JPEGR_UNKNOWN_ERROR = -1,
  JPEGR_IO_ERROR_BASE = -10000,
  ERROR_JPEGR_BAD_PTR = JPEGR_IO_ERROR_BASE - 1,
  ERROR_JPEGR_UNSUPPORTED_WIDTH_HEIGHT = JPEGR_IO_ERROR_BASE - 2,
  ERROR_JPEGR_INVALID_COLORGAMUT = JPEGR_IO_ERROR_BASE - 3,
  ERROR_JPEGR_INVALID_STRIDE = JPEGR_IO_ERROR_BASE - 4,
  ERROR_JPEGR_INVALID_TRANS_FUNC = JPEGR_IO_ERROR_BASE - 5,
  ERROR_JPEGR_RESOLUTION_MISMATCH = JPEGR_IO_ERROR_BASE - 6,
  ERROR_JPEGR_INVALID_QUALITY_FACTOR = JPEGR_IO_ERROR_BASE - 7,
  ERROR_JPEGR_INVALID_DISPLAY_BOOST = JPEGR_IO_ERROR_BASE - 8,
  ERROR_JPEGR_INVALID_OUTPUT_FORMAT = JPEGR_IO_ERROR_BASE - 9,
  ERROR_JPEGR_BAD_METADATA = JPEGR_IO_ERROR_BASE - 10,
  ERROR_JPEGR_INVALID_CROPPING_PARAMETERS = JPEGR_IO_ERROR_BASE - 11,
  ERROR_JPEGR_INVALID_GAMMA = JPEGR_IO_ERROR_BASE - 12,
  ERROR_JPEGR_INVALID_ENC_PRESET = JPEGR_IO_ERROR_BASE - 13,
  ERROR_JPEGR_INVALID_TARGET_DISP_PEAK_BRIGHTNESS = JPEGR_IO_ERROR_BASE - 14,
  JPEGR_RUNTIME_ERROR_BASE = -20000,
  ERROR_JPEGR_ENCODE_ERROR = JPEGR_RUNTIME_ERROR_BASE - 1,
  ERROR_JPEGR_DECODE_ERROR = JPEGR_RUNTIME_ERROR_BASE - 2,
  ERROR_JPEGR_GAIN_MAP_IMAGE_NOT_FOUND = JPEGR_RUNTIME_ERROR_BASE - 3,
  ERROR_JPEGR_BUFFER_TOO_SMALL = JPEGR_RUNTIME_ERROR_BASE - 4,
  ERROR_JPEGR_METADATA_ERROR = JPEGR_RUNTIME_ERROR_BASE - 5,
  ERROR_JPEGR_NO_IMAGES_FOUND = JPEGR_RUNTIME_ERROR_BASE - 6,
  ERROR_JPEGR_MULTIPLE_EXIFS_RECEIVED = JPEGR_RUNTIME_ERROR_BASE - 7,
  ERROR_JPEGR_UNSUPPORTED_MAP_SCALE_FACTOR = JPEGR_RUNTIME_ERROR_BASE - 8,
  ERROR_JPEGR_GAIN_MAP_SIZE_ERROR = JPEGR_RUNTIME_ERROR_BASE - 9,
  ERROR_JPEGR_UNSUPPORTED_FEATURE = -30000,
} status_t;

/* ref ultrahdr.h:79-85 */
typedef enum {
  ULTRAHDR_COLORGAMUT_UNSPECIFIED = -1,
  ULTRAHDR_COLORGAMUT_BT709,
  ULTRAHDR_COLORGAMUT_P3,
  ULTRAHDR_COLORGAMUT_BT2100,
  ULTRAHDR_COLORGAMUT_MAX = ULTRAHDR_COLORGAMUT_BT2100,
} ultrahdr_color_gamut;

/* ref ultrahdr.h:89-96 */
typedef enum {
  ULTRAHDR_TF_UNSPECIFIED = -1,
  ULTRAHDR_TF_LINEAR = 0,
  ULTRAHDR_TF_HLG = 1,
  ULTRAHDR_TF_PQ = 2,
  ULTRAHDR_TF_SRGB = 3,
  ULTRAHDR_TF_MAX = ULTRAHDR_TF_SRGB,
} ultrahdr_transfer_function;

/* ref ultrahdr.h:99-106: SDR = RGBA8888, HDR_LINEAR = RGBA half float, HDR_PQ / HDR_HLG = RGBA1010102 */
typedef enum {
  ULTRAHDR_OUTPUT_UNSPECIFIED = -1,
  ULTRAHDR_OUTPUT_SDR,
  ULTRAHDR_OUTPUT_HDR_LINEAR,
  ULTRAHDR_OUTPUT_HDR_PQ,
  ULTRAHDR_OUTPUT_HDR_HLG,
  ULTRAHDR_OUTPUT_MAX = ULTRAHDR_OUTPUT_HDR_HLG,
} ultrahdr_output_format;

/* ref ultrahdr.h:108-131 */
struct ultrahdr_metadata_struct {
  std::string version;
  float maxContentBoost;
  float minContentBoost;
  float gamma;
  float offsetSdr;
  float offsetHdr;
  float hdrCapacityMin;
  float hdrCapacityMax;
};

/* ref ultrahdr.h:136-165: uncompressed image; data = luma (+ chroma right behind it when chroma_data
 * is null), strides in pixels, 0 = tight */
struct jpegr_uncompressed_struct {
  void* data;
  unsigned int width;
  unsigned int height;
  ultrahdr_color_gamut colorGamut;
  void* chroma_data = nullptr;
  unsigned int luma_stride = 0;
  unsigned int chroma_stride = 0;
  uhdr_img_fmt_t pixelFormat = UHDR_IMG_FMT_UNSPECIFIED;
  uhdr_color_range_t colorRange = UHDR_CR_UNSPECIFIED;
};

/* ref ultrahdr.h:170-179 */
struct jpegr_compressed_struct {
  void* data;
  size_t length;
  size_t maxLength;
  ultrahdr_color_gamut colorGamut;
};

/* ref ultrahdr.h:184-189 */
struct jpegr_exif_struct {
  void* data;
  size_t length;
};

typedef struct jpegr_uncompressed_struct* jr_uncompressed_ptr;
typedef struct jpegr_compressed_struct* jr_compressed_ptr;
typedef struct jpegr_exif_struct* jr_exif_ptr;
typedef struct ultrahdr_metadata_struct* ultrahdr_metadata_ptr;

}  // namespace ultrahdr

#endif
