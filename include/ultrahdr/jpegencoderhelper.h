/*
 * ultrahdr/jpegencoderhelper.h -- the reference's JpegEncoderHelper surface
 * (lib/include/ultrahdr/jpegencoderhelper.h:42-112) on the CUDA JPEG block stage:
 * colour conversion / level shift / islow FDCT / quantiser and the baseline Huffman coder run as CUDA
 * kernels (fdct8.cu, huffman.cu); the stream is byte-identical to what libjpeg-turbo writes for the
 * reference's settings.  Not thread safe per object, like the reference's.
 */
#ifndef UHDR_B200_ULTRAHDR_JPEGENCODERHELPER_H
#define UHDR_B200_ULTRAHDR_JPEGENCODERHELPER_H

#include <cstdint>
#include <vector>

#include "ultrahdr_api.h"

namespace ultrahdr {

class JpegEncoderHelper {
 public:
  JpegEncoderHelper() = default;
  ~JpegEncoderHelper() = default;

  /* ref :55-56.  Formats: YCbCr 4:4:4 / 4:2:2 / 4:2:0, Y400, RGB888 (the gain map); gain-map formats get
   * the reference's COM marker (jpegencoderhelper.cpp:205-211). */
  uhdr_error_info_t compressImage(const uhdr_raw_image_t* img, const int qfactor, const void* iccBuffer, const size_t iccSize);
  /* ref :72-74: strides in pixels */
  uhdr_error_info_t compressImage(const uint8_t* planes[3], const unsigned int strides[3], const int width, const int height,
                                  const uhdr_img_fmt_t format, const int qfactor, const void* iccBuffer, const size_t iccSize);
  /* ref :81, :87, :93 */
  uhdr_compressed_image_t getCompressedImage();
  void* getCompressedImagePtr() { return mResult.data(); }
  size_t getCompressedImageSize() { return mResult.size(); }

 private:
  std::vector<uint8_t> mResult;
};

}  // namespace ultrahdr

#endif
