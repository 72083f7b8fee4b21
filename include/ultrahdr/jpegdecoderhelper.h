/*
 * ultrahdr/jpegdecoderhelper.h -- the reference's JpegDecoderHelper surface
 * (lib/include/ultrahdr/jpegdecoderhelper.h:36-162): marker extraction on the host,
 * entropy decoding (self-synchronising parallel decoder, huffdec.cu), dequantiser + islow IDCT, chroma
 * upsampling and colour conversion on the device.  Baseline sequential single-scan streams.
 */
#ifndef UHDR_B200_ULTRAHDR_JPEGDECODERHELPER_H
#define UHDR_B200_ULTRAHDR_JPEGDECODERHELPER_H

#include <cstdint>
#include <vector>

#include "ultrahdr_api.h"

namespace ultrahdr {

/* ref :36-43 */
typedef enum {
  PARSE_STREAM = (1 << 0),         /* header and APPn markers (Exif, Icc, Xmp, Iso) only */
  DECODE_STREAM = (1 << 16),       /* one component -> grayscale, several -> RGB(A) */
  DECODE_TO_YCBCR_CS = (1 << 17),  /* planes as coded, no chroma upsampling */
  DECODE_TO_RGB_CS = (1 << 18),    /* RGBA8888 */
} decode_mode_t;

class JpegDecoderHelper {
 public:
  JpegDecoderHelper() = default;
  ~JpegDecoderHelper() = default;

  /* ref :59-60, :69-71 */
  uhdr_error_info_t decompressImage(const void* image, size_t length, decode_mode_t mode = DECODE_TO_YCBCR_CS);
  uhdr_error_info_t parseImage(const void* image, size_t length) { return decompressImage(image, length, PARSE_STREAM); }

  /* ref :80-152: valid after decompressImage / parseImage */
  uhdr_raw_image_t getDecompressedImage();
  void* getDecompressedImagePtr() { return mResultBuffer.data(); }
  size_t getDecompressedImageSize() { return mResultBuffer.size(); }
  unsigned int getDecompressedImageWidth() { return mPlaneWidth[0]; }
  unsigned int getDecompressedImageHeight() { return mPlaneHeight[0]; }
  unsigned int getNumComponentsInImage() { return mNumComponents; }
  void* getXMPPtr() { return mXMPBuffer.data(); }
  size_t getXMPSize() { return mXMPBuffer.size(); }
  void* getEXIFPtr() { return mEXIFBuffer.data(); }
  size_t getEXIFSize() { return mEXIFBuffer.size(); }
  void* getICCPtr() { return mICCBuffer.data(); }
  size_t getICCSize() { return mICCBuffer.size(); }
  void* getIsoMetadataPtr() { return mIsoMetadataBuffer.data(); }
  size_t getIsoMetadataSize() { return mIsoMetadataBuffer.size(); }
  /* offset of the EXIF payload relative to the start of the stream, -1 if there is none */
  long getEXIFPos() { return mExifPayLoadOffset; }

 private:
  static constexpr int kMaxNumComponents = 3;
  std::vector<uint8_t> mResultBuffer, mXMPBuffer, mEXIFBuffer, mICCBuffer, mIsoMetadataBuffer;
  uhdr_img_fmt_t mOutFormat = UHDR_IMG_FMT_UNSPECIFIED;
  unsigned int mNumComponents = 0;
  unsigned int mPlaneWidth[kMaxNumComponents] = {0, 0, 0};
  unsigned int mPlaneHeight[kMaxNumComponents] = {0, 0, 0};
  unsigned int mPlaneHStride[kMaxNumComponents] = {0, 0, 0};
  unsigned int mPlaneVStride[kMaxNumComponents] = {0, 0, 0};
  long mExifPayLoadOffset = -1;
};

}  // namespace ultrahdr

#endif
