// Host container layer of the JPEG/R file: the byte-shuffling the reference does in
// JpegR::appendGainMap (lib/src/jpegr.cpp:1105-1415), gainmapmetadata.cpp (ISO 21496-1 codec),
// multipictureformat.cpp (MPF) and the image splitter (jpegr.cpp:1833-1900).  Pure CPU, tiny;
// only its observable bytes matter (SURVEY.md section 2 marks it out of the hot path) but the
// drop-in C API needs it to produce/consume real files.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#include "bytes.h"

#include "../../include/ultrahdr_api.h"

namespace uhdr_b200 {

// ISO 21496-1 payload for the gain-map image (gainmapmetadata.cpp:113-193 after
// gainmapMetadataFloatToFraction :349-425). Returns uhdr_codec_err_t.
// Writes into caller storage (no heap): kIsoMetadataMaxBytes always suffices (2+2+1 bytes of versions and flags,
// 4 header fractions of 8 bytes, 3 channels x 5 fractions of 8 bytes).
constexpr size_t kIsoMetadataMaxBytes = 160;
int iso_encode_metadata(const uhdr_gainmap_metadata_t& md, uint8_t* out, size_t cap, size_t* out_size);
// inverse (:195-347); validates like uhdr_validate_gainmap_metadata_descriptor
int iso_decode_metadata(const uint8_t* data, size_t size, uhdr_gainmap_metadata_t* md);
int validate_metadata(const uhdr_gainmap_metadata_t& md);
// hdrgm XMP packet of the gain-map image's APP1 marker (Ultra HDR v1 files and Apple's variant carry
// no ISO 21496-1 block): getMetadataFromXMP, jpegrutils.cpp:646-874, incl. the Apple branch that takes
// the headroom from the XMP element or from the primary image's EXIF maker notes (:506-644).
// `xmp` starts at the "http://ns.adobe.com/xap/1.0/" signature; `exif` may be null.
int xmp_decode_metadata(const uint8_t* xmp, size_t size, const uint8_t* exif, size_t exif_size, uhdr_gainmap_metadata_t* md);
// UltraHdr::parseGainMapMetadata (jpegr.cpp:1432-1466): ISO block if present, else XMP.  `iso` / `xmp`
// are whole marker payloads (signature included) or empty.
int parse_gainmap_metadata(const uint8_t* iso, size_t iso_size, const uint8_t* xmp, size_t xmp_size, const uint8_t* exif,
                           size_t exif_size, uhdr_gainmap_metadata_t* md);

// ICC profile (with "ICC_PROFILE" prefix) the reference writes for (ct, cg); nullptr if unknown
const uint8_t* icc_profile(int ct, int cg, size_t* size);
// IccHelper::readIccColorGamut (icc.cpp:640-748)
int icc_read_gamut(const uint8_t* data, size_t size);

// One JFIF stream handed over in two pieces so that the (large) entropy-coded segment is copied
// exactly once, straight from the pinned buffer the device wrote it to: `head` = SOI .. SOS header
// (what libjpeg writes before the first MCU), `scan` = entropy-coded bytes; EOI is implied.
struct JpegPieces {
  const uint8_t* head;
  size_t head_len;
  const uint8_t* scan;
  size_t scan_len;
  // whole = true: `head` is a complete JPEG file as the caller handed it in (encode API-2/3/4); its bytes
  // from SOS on are copied verbatim, EOI is not implied
  bool whole = false;
  size_t total() const { return head_len + scan_len + (whole ? 0 : 2); }
  // the stream, EOI included, into out[0, total())
  void copy_to(uint8_t* out) const {
    memcpy(out, head, head_len);
    if (scan_len) memcpy(out + head_len, scan, scan_len);
    if (!whole) memcpy(out + head_len + scan_len, "\xFF\xD9", 2);
  }
};

// appendGainMap with UHDR_WRITE_ISO on / UHDR_WRITE_XMP off (the reference's default build).
// icc / icc_size: profile to write when the primary image carries none (API-4, jpegr.cpp:413-431); the
// primary image's own ICC and EXIF markers are carried over (:1173-1217), an `exif` argument next to an
// EXIF marker in the primary image is an error like in the reference.
int assemble_jpegr(const JpegPieces& primary, const JpegPieces& gainmap, const uint8_t* exif, size_t exif_size,
                   const uhdr_gainmap_metadata_t& md, uint8_t* out, size_t cap, size_t* out_size,
                   const uint8_t* icc = nullptr, size_t icc_size = 0);
// number of JPEG images in a buffer as image_io's scanner counts them and the range of the first one
// (uhdr_enc_set_compressed_image keeps the first, ultrahdr_api.cpp:548-584); -1: corrupt
int count_jpeg_images(const uint8_t* data, size_t size, size_t* first_off = nullptr, size_t* first_len = nullptr);

// locate primary image and gain-map image inside a JPEG/R file
int split_jpegr(const uint8_t* data, size_t size, size_t* p_off, size_t* p_len, size_t* g_off,
                size_t* g_len);

}  // namespace uhdr_b200
