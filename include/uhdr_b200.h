/*
 * uhdr_b200.h -- extensions of libuhdr_b200 beyond the reference C API: stage-level entry points
 * (the reference exposes these only as C++ members of ultrahdr::JpegR / UltraHdr), batch encode
 * and the LUT install hook used for the multi-GPU NCCL broadcast.  Plain C ABI: pointers, sizes,
 * PODs; no torch / CUDA types.  Return value: a uhdr_codec_err_t (0 = UHDR_CODEC_OK); on failure
 * uhdr_b200_last_error() returns a thread-local message.
 *
 * All image descriptors carry HOST pointers unless the function name ends in `_dev`.
 * Every entry point needs a CUDA device: there is no CPU fallback.
 */
#ifndef UHDR_B200_H
#define UHDR_B200_H

#include <stdint.h>
#include "ultrahdr_api.h"

typedef struct uhdr_b200_gm_config {
  /* ultrahdr::JpegR constructor arguments, ref lib/include/ultrahdr/jpegr.h:54-62 and
   * lib/include/ultrahdr/ultrahdrcommon.h:450-457 */
  int scale_factor;            /* mapDimensionScaleFactor */
  int quality;                 /* mapCompressQuality */
  int multichannel;            /* useMultiChannelGainMap */
  float gamma;
  int preset;                  /* uhdr_enc_preset_t */
  float min_content_boost;     /* FLT_MIN = unset */
  float max_content_boost;     /* FLT_MAX = unset */
  float target_disp_peak_nits; /* -1 = unset */
  /* UltraHdr::generateGainMap flags, ref lib/include/ultrahdr/ultrahdrcommon.h:496-499 */
  int sdr_is_601;
  int use_luminance;
} uhdr_b200_gm_config_t;

UHDR_EXTERN const char* uhdr_b200_last_error(void);
UHDR_EXTERN int uhdr_b200_device_count(void);
UHDR_EXTERN unsigned long long uhdr_b200_kernel_launches(void);

/* UltraHdr::generateGainMap, ref lib/src/jpegr.cpp:530.  gainmap_out->planes[0] must point to
 * (w/scale)*(h/scale)*(multichannel?3:1) bytes; written tightly packed, descriptor filled in. */
UHDR_EXTERN int uhdr_b200_generate_gainmap(const uhdr_raw_image_t* sdr, const uhdr_raw_image_t* hdr,
                                           const uhdr_b200_gm_config_t* cfg,
                                           uhdr_gainmap_metadata_t* metadata_out,
                                           uhdr_raw_image_t* gainmap_out);
/* UltraHdr::applyGainMap, ref lib/src/jpegr.cpp:1533 */
UHDR_EXTERN int uhdr_b200_apply_gainmap(const uhdr_raw_image_t* sdr, const uhdr_raw_image_t* gainmap,
                                        const uhdr_gainmap_metadata_t* metadata, int output_ct,
                                        int output_fmt, float max_display_boost,
                                        uhdr_raw_image_t* dest);
/* UltraHdr::toneMap, ref lib/src/jpegr.cpp:1985 */
UHDR_EXTERN int uhdr_b200_tonemap(const uhdr_raw_image_t* hdr, uhdr_raw_image_t* sdr);
/* UltraHdr::convertYuv (in place), ref lib/src/jpegr.cpp:436 */
UHDR_EXTERN int uhdr_b200_convert_yuv(uhdr_raw_image_t* image, int src_cg, int dst_cg);

/* The same four stages on DEVICE memory: every plane pointer in the descriptors is a device pointer (strides
 * in pixels, as everywhere), `stream` is the caller's cudaStream_t (passed as void* to keep this header free
 * of CUDA types; NULL = the legacy default stream).  Kernels are enqueued on that stream and the call returns
 * without synchronising -- nothing crosses PCIe -- with one exception: uhdr_b200_generate_gainmap_dev with the
 * two-pass preset (UHDR_USAGE_BEST_QUALITY) drains the stream before returning, because the metadata it hands
 * back is derived from the image-wide min / max.  A maintainer chaining generateGainMap -> compressImage, or
 * decode -> applyGainMap -> display, binds these instead of the host-pointer forms above.  Scratch memory comes
 * from the calling host thread's workspace: keep one stream per host thread, or synchronise between calls.
 * Alignment for the vectorised kernels (else the generic ones run): planes 16-byte aligned, strides multiples
 * of 4 pixels.  dest / gainmap planes must be allocated by the caller: gain map (w/scale)*(h/scale)*(3|1) bytes
 * with stride >= width, apply destination w*h*(8|4) bytes, tone-map destination in the SDR format matching the
 * HDR one (P010 -> YCbCr420, RGBA1010102 / RGBAHalfFloat -> RGBA8888). */
UHDR_EXTERN int uhdr_b200_generate_gainmap_dev(const uhdr_raw_image_t* sdr_dev, const uhdr_raw_image_t* hdr_dev,
                                               const uhdr_b200_gm_config_t* cfg, uhdr_gainmap_metadata_t* metadata_out,
                                               uhdr_raw_image_t* gainmap_dev, void* stream);
UHDR_EXTERN int uhdr_b200_apply_gainmap_dev(const uhdr_raw_image_t* sdr_dev, const uhdr_raw_image_t* gainmap_dev,
                                            const uhdr_gainmap_metadata_t* metadata, int output_ct, float max_display_boost,
                                            uhdr_raw_image_t* dest_dev, void* stream);
UHDR_EXTERN int uhdr_b200_tonemap_dev(const uhdr_raw_image_t* hdr_dev, uhdr_raw_image_t* sdr_dev, void* stream);
UHDR_EXTERN int uhdr_b200_convert_yuv_dev(uhdr_raw_image_t* image_dev, int src_cg, int dst_cg, void* stream);

/* JpegEncoderHelper::compressImage, ref lib/src/jpegencoderhelper.cpp:101.  `is_gainmap_comment`
 * is implied by the format exactly as in the reference (RGB888 / Y400 carry the COM marker).
 * out must hold `cap` bytes.  Planes whose width is not a multiple of 8 are padded the way the helper pads them for
 * the given strides: a stride below the 8-aligned width gives columns of 0 (luma) / 128 (chroma) and rows past the
 * height that repeat the previous iMCU row's; a larger stride reads the caller's bytes up to the aligned width. */
UHDR_EXTERN int uhdr_b200_jpeg_encode(const uhdr_raw_image_t* img, int quality, const void* icc,
                                      size_t icc_size, void* out, size_t cap, size_t* out_size);
/* forward block stage only: quantised coefficients per component, raster block order, natural
 * order inside a block (parity hook for FDCT + quantise). coefs[c] sized wblocks*hblocks*64.  Edge padding as in
 * uhdr_b200_jpeg_encode. */
UHDR_EXTERN int uhdr_b200_jpeg_forward(const uhdr_raw_image_t* img, int quality, int16_t* coefs[3]);
/* JpegDecoderHelper::decompressImage, ref lib/src/jpegdecoderhelper.cpp:169.
 * mode: 0 = DECODE_TO_YCBCR_CS raw planes, 1 = DECODE_TO_RGB_CS (RGBA8888), 2 = DECODE_STREAM.
 * out->planes[0] must point to a buffer of `cap` bytes; planes are laid out back to back like
 * JpegDecoderHelper::getDecompressedImage (:536-552). */
UHDR_EXTERN int uhdr_b200_jpeg_decode(const void* data, size_t size, int mode, uhdr_raw_image_t* out,
                                      size_t cap);

/* The whole-file codec on DEVICE images: decodeJPEGR into device planes, encodeJPEGR from device intents and
 * compressImage of a device image.  The compressed bytes stay in HOST memory.  Contract of all three:
 *  - Device images: every plane pointer of a descriptor is device memory of the current device (checked with
 *    cudaPointerGetAttributes), aligned to its element only (a sample of the planar formats, a pixel of the packed
 *    ones, a byte for RGB888).  Strides are in pixels and may be any value >= the plane width.  Bytes between a
 *    row's width and its stride are never read into a result and never written.  Inputs are never modified.
 *  - Stream order (`stream`: the caller's cudaStream_t, NULL = the legacy default stream): writes into dest_dev /
 *    gainmap_dev happen after all work enqueued earlier on `stream`, and work enqueued on it after the call sees
 *    them without a host synchronise.  Encode inputs are read after the earlier work on `stream`.
 *  - Host blocking: uhdr_b200_decode_dev may return before its pixels are written and does not wait for the work
 *    enqueued on `stream` before it: the JPEG decoding runs on the library's own streams, only the writes into the
 *    caller's planes are ordered onto `stream` (events).  A following call of any of the three on the same host
 *    thread first waits on the host until those writes (or the kernels a failed decode left running) are done,
 *    since they read the scratch memory it reuses: behind a busy stream, back-to-back decodes wait for the work
 *    queued before the previous call.  The two encode calls run on `stream` and return when the file is complete.
 *  - Errors: the codes of the host counterparts on the same input (uhdr_decode; uhdr_enc_set_raw_image plus
 *    uhdr_encode; uhdr_b200_jpeg_encode).  Bad or host pointers, another device's memory, misalignment and wrong
 *    dimensions give UHDR_CODEC_INVALID_PARAM.  A failing call writes nothing into the caller's device buffers.
 *    Without a device: UHDR_CODEC_ERROR with a CUDA message.
 *  - Threads: host threads with their own streams may call concurrently.  State is per host thread and device.
 *
 * uhdr_b200_decode_dev: JpegR::decodeJPEGR (ref lib/src/jpegr.cpp:1469-1531).  data/size: the JPEG/R file.
 * dest_dev: fmt, w, h, stride[0] set by the caller, planes[0] a device pointer.  fmt and out_ct pair exactly as in
 * uhdr_decode: RGBAHalfFloat + LINEAR, RGBA1010102 + HLG | PQ, RGBA8888 + SRGB (base image only).  w / h equal the
 * primary image's (uhdr_dec_probe gives them).  On return dest_dev->cg / ct / range are filled in.
 * gainmap_dev: optional.  w / h equal the map's, stride[0] >= w, the buffer holds h * stride[0] * 4 bytes.  The call
 * sets fmt to Y400 or RGBA8888 and writes the decoded map (what uhdr_get_decoded_gainmap_image returns).
 * metadata_out: optional host struct. */
UHDR_EXTERN int uhdr_b200_decode_dev(const void* data, size_t size, int out_ct, float max_display_boost,
                                     uhdr_raw_image_t* dest_dev, uhdr_raw_image_t* gainmap_dev,
                                     uhdr_gainmap_metadata_t* metadata_out, void* stream);
/* Reduced-size decoding: both JPEGs of the file at 1/k size, k in {1, 2, 4, 8}, the way libjpeg-turbo decodes with
 * scale_num = 1, scale_denom = k -- a reduced inverse DCT per 8x8 block (4x4, 2x2 or 1x1 samples), not a decode
 * followed by a downscale.  The primary image and the gain map each come out ceil(w / k) x ceil(h / k).  Chroma is
 * scaled up by the IDCT, as libjpeg does: a 4:2:0 primary decodes to a 4:4:4 image at 1/k.  For HDR outputs the gain
 * map is then applied as uhdr_decode applies it (applyGainMap on the two decoded images, with the file's metadata,
 * out_ct and max_display_boost); an SRGB output is the primary image as RGBA8888.  k = 1 is the full-size decode.
 * k > 1 supports gray, 4:4:4 and 4:2:0 JPEGs; another sampling (4:2:2, 4:4:0, 4:1:1) gives
 * UHDR_CODEC_UNSUPPORTED_FEATURE, and a k outside {1, 2, 4, 8} UHDR_CODEC_INVALID_PARAM.
 *
 * uhdr_b200_scaled_dims: the sizes the caller allocates for a decode at 1/k -- primary *w x *h, gain map
 * *gm_w x *gm_h.  Reads the container only; needs no device.
 * uhdr_b200_decode_scaled_dev: uhdr_b200_decode_dev at 1/k, with exactly its contract (device planes of any pitch,
 * stream order through events, the next call's host wait, nothing written on failure, the same error codes).
 * dest_dev and gainmap_dev have the sizes uhdr_b200_scaled_dims returns.  A small result is copied to the host by the
 * caller: there is no host-buffer form. */
UHDR_EXTERN int uhdr_b200_scaled_dims(const void* data, size_t size, int k, unsigned* w, unsigned* h, unsigned* gm_w,
                                      unsigned* gm_h);
UHDR_EXTERN int uhdr_b200_decode_scaled_dev(const void* data, size_t size, int k, int out_ct, float max_display_boost,
                                            uhdr_raw_image_t* dest_dev, uhdr_raw_image_t* gainmap_dev,
                                            uhdr_gainmap_metadata_t* metadata_out, void* stream);
/* Batched decoding: uhdr_b200_decode_scaled_dev of n files in one call, with one entropy-decoding pass and one inverse
 * DCT per reduced size over both JPEGs of every file, then each file's colour conversion and gain-map application.
 * For many small outputs (thumbnails, previews) this saves the fixed launches and host waits a single decode costs.
 *  - Same bytes: each item's dest_dev, gainmap_dev and metadata_out get byte for byte what uhdr_b200_decode_scaled_dev
 *    writes for that file with the same k, out_ct and max_display_boost.  dest_dev->fmt is read per item (each must
 *    pair with out_ct), so one batch may mix formats; the sizes are those uhdr_b200_scaled_dims gives.
 *  - Errors per item: status is the code the single call returns for that file (corrupt data, no metadata, 4:2:2 at
 *    k > 1, a bad descriptor).  A failing item gets nothing written into its buffers; the others are unaffected.  The
 *    return value is UHDR_CODEC_OK when every item succeeded, else the first failing item's code, and
 *    uhdr_b200_last_error() names that item's index and gives its message.  An error of the whole call (CUDA, device
 *    memory) is returned and set as the status of every item without an error of its own.
 *  - n < 1, a k outside {1, 2, 4, 8} or a null items give UHDR_CODEC_INVALID_PARAM and decode nothing.
 *  - Stream order, host blocking and threads: uhdr_b200_decode_dev's rules.  The writes are ordered after the work
 *    enqueued earlier on `stream`, later work on it sees them, the call may return before they land, and the next
 *    call on the thread first waits for them.  State is per host thread and device.
 *  - A batch whose scratch would exceed a device-memory budget (4 GiB; the environment variable
 *    UHDR_B200_BATCH_GROUP_BYTES sets another) is decoded in groups, one after the other, with the same results. */
typedef struct uhdr_b200_decode_item {
  const void* data;                      /* one JPEG/R file, host memory */
  size_t size;
  uhdr_raw_image_t* dest_dev;            /* as uhdr_b200_decode_scaled_dev's dest_dev */
  uhdr_raw_image_t* gainmap_dev;         /* optional, as there */
  uhdr_gainmap_metadata_t* metadata_out; /* optional, as there */
  int status;                            /* out: this item's uhdr_codec_err_t */
} uhdr_b200_decode_item_t;
UHDR_EXTERN int uhdr_b200_decode_batch_dev(uhdr_b200_decode_item_t* items, int n, int k, int out_ct, float max_display_boost,
                                           void* stream);
/* uhdr_b200_jpeg_decode of one JPEG at 1/k (stage hook, host buffers).  k = 1 is uhdr_b200_jpeg_decode.  For k > 1,
 * mode 0 gives Y400 or YUV444 planes of ceil(w / k) x ceil(h / k) samples, back to back at stride = width; mode 1
 * gives RGBA8888 at that size. */
UHDR_EXTERN int uhdr_b200_jpeg_decode_scaled(const void* data, size_t size, int mode, int k, uhdr_raw_image_t* out,
                                             size_t cap);
/* A JPEG/R decoded once and kept in device memory, then rendered at any display boost, output transfer and viewport
 * without decoding again: a viewer re-renders as the display's headroom or the visible rectangle changes, a server
 * renders one upload as linear, HLG and PQ.  A render costs one apply kernel (or, for SRGB, one colour conversion)
 * over the rectangle plus a table upload of a few KB.
 *
 * uhdr_b200_image_open_dev: decodes both JPEGs of the file at 1/k (k in {1, 2, 4, 8}, as uhdr_b200_decode_scaled_dev)
 * on the current device, to which the image stays bound.  It keeps the primary image's YCbCr planes, the decoded gain
 * map (resized once, here, when its aspect ratio differs from the primary image's by more than 1 %, as applyGainMap
 * would on every call), the metadata and the gamuts; the entropy decoder's scratch is not kept.  Returns when the
 * image is resident.  Errors: those of uhdr_b200_decode_scaled_dev on the same file (corrupt data, no metadata, a k
 * outside {1, 2, 4, 8}, 4:2:2 / 4:4:0 / 4:1:1 at k > 1); a gray primary image gives UHDR_CODEC_UNSUPPORTED_FEATURE.
 * Without a device: UHDR_CODEC_ERROR with a CUDA message.  *out is NULL after a failure.
 * uhdr_b200_image_info: the 1/k primary image's *w x *h, the decoded gain map's *gm_w x *gm_h (both as
 * uhdr_b200_scaled_dims gives them), the metadata and the device memory the image holds.  Any pointer may be NULL.
 * uhdr_b200_image_render_dev: writes the dest_dev->w x dest_dev->h pixels of the image that start at (x, y) into
 * dest_dev.  The bytes equal that rectangle cut from uhdr_b200_decode_scaled_dev's result for the same k, out_ct,
 * max_display_boost and format (for k = 1 also from uhdr_b200_decode_dev's and uhdr_decode's).  dest_dev follows the
 * decode_dev rules above: fmt / out_ct pair as there, planes[0] device memory of the image's device aligned to a
 * pixel, any stride >= w, the bytes past a row's width untouched; on success cg / ct / range are set as decode_dev sets
 * them.  The rectangle must be non-empty and inside the image.  Stream order: the writes follow the work enqueued
 * earlier on `stream` and are visible to later work on it; the call does not wait on the host, except when all of the
 * image's few per-render table slots are still in use by renders in flight.  Renders may go to different streams.  A
 * failing call writes nothing; bad arguments give UHDR_CODEC_INVALID_PARAM.  An image is not thread-safe (one host
 * thread at a time), distinct images are independent.
 * uhdr_b200_image_release: waits for the image's outstanding renders, then returns its memory to the process-wide
 * cache of released handles (uhdr_b200_trim_cache). */
typedef struct uhdr_b200_image uhdr_b200_image_t;
UHDR_EXTERN int uhdr_b200_image_open_dev(const void* data, size_t size, int k, uhdr_b200_image_t** out);
UHDR_EXTERN int uhdr_b200_image_info(const uhdr_b200_image_t* img, unsigned* w, unsigned* h, unsigned* gm_w,
                                     unsigned* gm_h, uhdr_gainmap_metadata_t* md, size_t* device_bytes);
UHDR_EXTERN int uhdr_b200_image_render_dev(uhdr_b200_image_t* img, int out_ct, float max_display_boost, unsigned x,
                                           unsigned y, uhdr_raw_image_t* dest_dev, void* stream);
UHDR_EXTERN int uhdr_b200_image_release(uhdr_b200_image_t* img);
/* JpegR::encodeJPEGR API-1 (sdr_dev != NULL, ref lib/src/jpegr.cpp:247-291) / API-0 (sdr_dev == NULL, :179-244)
 * from intents in device memory.  The JPEG/R file is written to the HOST buffer out (cap bytes); *out_size
 * receives its length.  The bytes equal uhdr_encode's for the same intents and settings: cfg carries the settings
 * uhdr_encode has (checked with its setters' ranges; FLT_MIN / FLT_MAX / -1 mean unset), and sdr_is_601 /
 * use_luminance are ignored (uhdr_encode's values, 0 / 1, are used). */
UHDR_EXTERN int uhdr_b200_encode_dev(const uhdr_raw_image_t* hdr_dev, const uhdr_raw_image_t* sdr_dev,
                                     const uhdr_b200_gm_config_t* cfg, int base_quality,
                                     const void* exif, size_t exif_size,
                                     void* out, size_t cap, size_t* out_size, void* stream);
/* JpegEncoderHelper::compressImage (ref lib/src/jpegencoderhelper.cpp:101) of a DEVICE image: the formats and
 * bytes of uhdr_b200_jpeg_encode given zero-initialised rows of 64-pixel aligned stride (the layout uhdr_encode
 * compresses from; no byte past a row's width is read); the stream goes to the HOST buffer out. */
UHDR_EXTERN int uhdr_b200_jpeg_encode_dev(const uhdr_raw_image_t* img_dev, int quality, const void* icc,
                                          size_t icc_size, void* out, size_t cap, size_t* out_size, void* stream);

/* Transcoding: a smaller or recompressed JPEG/R made from a JPEG/R, keeping its SDR rendition and its gain map (no
 * decode to HDR pixels, no new tone mapping).  Both JPEGs of the file are decoded at 1/k, as libjpeg-turbo decodes
 * with scale_denom = k (raw YCbCr planes, the 3-channel map too), re-encoded, and put into a new container with the
 * file's metadata.  The output bytes equal this composition of the reference's pieces:
 *  - each JPEG's planes, as JpegDecoderHelper's raw_data_out decode at 1/k gives them (tight strides), re-encoded by
 *    JpegEncoderHelper::compressImage in the format they form (Y400, YUV420, YUV422 or YUV444) at base_quality /
 *    gainmap_quality, with that JPEG's own ICC APP2 payload (none if it has none);
 *  - base_420 = 1 and a 4:4:4 base (a 4:4:4 file, or a 4:2:0 one at k > 1): the base is instead what libjpeg-turbo's
 *    jpeg_write_scanlines writes from the YCbCr planes with 2x2 / 1x1 / 1x1 sampling -- libjpeg's own chroma
 *    downsampling, (a + b + c + d + bias) >> 2 with bias 1, 2, 1, 2, ... along a row, edges replicated.  A base that
 *    is already 4:2:0 is taken as above, a gray base ignores the flag, 4:2:2 gives UHDR_CODEC_UNSUPPORTED_FEATURE;
 *  - keep_exif = 1: the primary image's EXIF block is carried into the new file;
 *  - the container is what API-4 (uhdr_enc_set_compressed_image with the primary image's ICC gamut,
 *    uhdr_enc_set_gainmap_image with the file's metadata, uhdr_encode) writes: ISO 21496-1 metadata, MPF, ICC.
 * Input and output are HOST bytes; the work runs on the calling thread's codec for the current device and the call
 * returns when the file is complete.  Errors: those of the composition (corrupt or progressive data, no metadata,
 * 4:2:2 / 4:4:0 / 4:1:1 at k > 1 as uhdr_b200_decode_scaled_dev, a sampling the encoder does not write, API-4's
 * checks); a k outside {1, 2, 4, 8}, a quality outside 0..100 or a null pointer give UHDR_CODEC_INVALID_PARAM.  A cap
 * that is too small gives UHDR_CODEC_MEM_ERROR with *out_size set to the size needed.  Nothing is written to out on
 * failure.  Without a device: UHDR_CODEC_ERROR with a CUDA message.  New fields go at the end of the struct. */
typedef struct uhdr_b200_transcode_config {
  int k;               /* 1, 2, 4 or 8: both JPEGs reduced as libjpeg-turbo's scale_denom = k does */
  int base_quality;    /* 0..100 */
  int gainmap_quality; /* 0..100 */
  int base_420;        /* 0: the base keeps the sampling its scaled decode produced; 1: the base is written 4:2:0 */
  int keep_exif;       /* 1: the primary image's EXIF block is carried into the new file */
} uhdr_b200_transcode_config_t;
UHDR_EXTERN int uhdr_b200_transcode(const void* data, size_t size, const uhdr_b200_transcode_config_t* cfg, void* out,
                                    size_t cap, size_t* out_size);
/* uhdr_b200_transcode of many files in one call, for thumbnail and preview jobs over many uploads: both JPEGs of every
 * file go through one entropy decoding, one inverse DCT per reduced size, one staging pass, one block stage and one
 * entropy coding, with two host waits for the encoder, instead of a single call's fixed cost per file.
 *  - Each item gets exactly what uhdr_b200_transcode(data, size, cfg, out, cap, &out_size) gives for that file alone:
 *    the same bytes, out_size and status.  One cfg (k, both qualities, base_420, keep_exif) applies to every item.
 *  - A failing item gets the code the single call returns and nothing is written to its out (corrupt or progressive
 *    data, no metadata, 4:2:2 at k > 1 or with base_420, API-4's checks, a short cap: UHDR_CODEC_MEM_ERROR with
 *    out_size set to the size needed).  The others are unaffected.  The return value is UHDR_CODEC_OK when every item
 *    succeeded, else the first failing item's code, and uhdr_b200_last_error() names that item's index and gives its
 *    message.  An error of the whole call (CUDA, device memory) is returned and set as the status of every item without
 *    an error of its own.
 *  - A null items or cfg, n < 1, a k outside {1, 2, 4, 8} or a quality outside 0..100 give UHDR_CODEC_INVALID_PARAM
 *    and transcode nothing.  Without a device: UHDR_CODEC_ERROR with a CUDA message.
 *  - Input and output are HOST bytes; the call returns when every file is complete.  It runs on the calling thread's
 *    codec for the current device, as uhdr_b200_transcode does, and the two may be interleaved on one thread.
 *  - A batch whose scratch would exceed a device-memory budget (4 GiB; the environment variable
 *    UHDR_B200_BATCH_GROUP_BYTES sets another) is transcoded in groups, one after the other, with the same results.
 *  - A repeated batch of the same or a smaller size makes no heap call. */
typedef struct uhdr_b200_transcode_item {
  const void* data;  /* one JPEG/R file, host memory */
  size_t size;
  void* out;         /* host buffer for the new file */
  size_t cap;
  size_t out_size;   /* out: bytes written; with UHDR_CODEC_MEM_ERROR, the size needed */
  int status;        /* out: this item's uhdr_codec_err_t */
} uhdr_b200_transcode_item_t;
UHDR_EXTERN int uhdr_b200_transcode_batch(uhdr_b200_transcode_item_t* items, int n,
                                          const uhdr_b200_transcode_config_t* cfg);
/* uhdr_b200_transcode of ONE file into a ladder of outputs in one call, each rung with its own config (a recompressed
 * full-size copy, a 1/2 preview, 1/4 and 1/8 thumbnails, ...): both JPEGs are entropy-decoded once whatever the number
 * of rungs, one inverse DCT pass writes every reduced size the rungs ask for, and the rungs share one staging pass, one
 * block stage per distinct (base_quality, gainmap_quality) pair and one entropy coding, with two host waits.
 *  - Each rung gets exactly what uhdr_b200_transcode(data, size, &rung.cfg, out, cap, &out_size) gives alone: the
 *    same bytes, out_size and status.  Rungs may repeat a k with other qualities, base_420 or keep_exif, may be
 *    identical, and may come in any order.
 *  - A null data or rungs, or n outside 1..16, give UHDR_CODEC_INVALID_PARAM and touch no rung.
 *  - A rung's own errors are the single call's, in its order of checks: a null out, a k outside {1, 2, 4, 8} or a
 *    quality outside 0..100 (UHDR_CODEC_INVALID_PARAM, before any device work); 4:2:2 / 4:4:0 / 4:1:1 at k > 1 and
 *    base_420 on a 4:2:2 base (UHDR_CODEC_UNSUPPORTED_FEATURE); a cap that is too small (UHDR_CODEC_MEM_ERROR with
 *    out_size set to the size needed).  Errors of the file (a failed probe, corrupt or progressive data, no metadata,
 *    an error of the gain-map JPEG) go to every rung that is still valid, at the point the single call meets them:
 *    when the primary image fails only at some k, the rungs at the other k go on to the map's error or succeed.
 *  - A failing rung writes nothing to its out; the others are unaffected.  The return value is UHDR_CODEC_OK when
 *    every rung succeeded, else the first failing rung's code, and uhdr_b200_last_error() reads "rung <i>: <message>".
 *    An error of the whole call (CUDA, device memory) is returned and set as the status of every rung without an error
 *    of its own.  Without a device: UHDR_CODEC_ERROR with a CUDA message, on the call and on every valid rung.
 *  - Input and output are HOST bytes; the call returns when every output is complete.  It runs on the calling thread's
 *    codec for the current device and may be interleaved on one thread with uhdr_b200_transcode, _batch and the
 *    decode calls.
 *  - A repeated ladder of the same or a smaller shape makes no heap call. */
typedef struct uhdr_b200_transcode_rung {
  uhdr_b200_transcode_config_t cfg;  /* this output's k, base_quality, gainmap_quality, base_420, keep_exif */
  void* out;                         /* host buffer for this output */
  size_t cap;
  size_t out_size;                   /* out: bytes written; with UHDR_CODEC_MEM_ERROR, the size needed */
  int status;                        /* out: this rung's uhdr_codec_err_t */
} uhdr_b200_transcode_rung_t;
UHDR_EXTERN int uhdr_b200_transcode_ladder(const void* data, size_t size, uhdr_b200_transcode_rung_t* rungs, int n);
/* uhdr_b200_transcode_ladder over MANY files in one call, each file with its own ladder (a derivative set for every
 * upload): the files are taken in groups, and per group both JPEGs of every file are entropy-decoded once, one inverse
 * DCT pass writes every reduced size every file's rungs ask for, and all the group's rungs share one staging pass, one
 * block stage per distinct (base_quality, gainmap_quality) pair and one entropy coding, with two host waits.
 *  - Each file gets exactly what uhdr_b200_transcode_ladder(data, size, rungs, n) gives for it alone: that return value
 *    in status, and on every rung the same bytes, out_size and status.  So every rung equals uhdr_b200_transcode with
 *    its cfg alone.  A file's null data or rungs, or n outside 1..16, give UHDR_CODEC_INVALID_PARAM on that file and
 *    touch none of its rungs.  A failing file or rung writes nothing; the others are unaffected.
 *  - A null files or n < 1 give UHDR_CODEC_INVALID_PARAM and touch no file.  Otherwise the return value is
 *    UHDR_CODEC_OK when every file succeeded, else the first failing file's status, and uhdr_b200_last_error() reads
 *    "file <i>: <that ladder's message>" ("file <i>: rung <j>: ..." for an error of a rung).  An error of the whole
 *    call (CUDA, device memory) ends it and is set as the status of every file and rung without an error of its own.
 *    Without a device: UHDR_CODEC_ERROR with a CUDA message on every valid rung, as uhdr_b200_transcode_ladder gives.
 *  - A group closes before its scratch would exceed a device-memory budget (4 GiB; the environment variable
 *    UHDR_B200_BATCH_GROUP_BYTES sets another), 2^29 entropy-coded bytes or 16 distinct quality pairs; a file is never
 *    split, and one that exceeds the budget runs alone.  The results are the same whatever the grouping.
 *  - Input and output are HOST bytes; the call returns when every output is complete.  It runs on the calling thread's
 *    codec for the current device and may be interleaved on one thread with the other transcode and decode calls.
 *  - A repeated call of the same or a smaller shape makes no heap call. */
typedef struct uhdr_b200_transcode_file {
  const void* data;                   /* one JPEG/R file, host memory */
  size_t size;
  uhdr_b200_transcode_rung_t* rungs;  /* this file's outputs, as in uhdr_b200_transcode_ladder */
  int n;                              /* 1..16 */
  int status;                         /* out: what uhdr_b200_transcode_ladder returns for this file alone */
} uhdr_b200_transcode_file_t;
UHDR_EXTERN int uhdr_b200_transcode_ladders(uhdr_b200_transcode_file_t* files, int n);

/* Measurement hooks.  Kernel timing brackets every kernel launch with CUDA events on the
 * launching stream and accumulates per-kernel totals ("name count total_ms min_ms max_ms" lines).
 * uhdr_b200_enc_rearm() makes a finished encoder handle runnable again while keeping the inputs
 * it uploaded at uhdr_enc_set_raw_image() time resident in HBM (streaming re-encode). */
UHDR_EXTERN void uhdr_b200_set_kernel_timing(int on);
UHDR_EXTERN int uhdr_b200_kernel_timing_report(char* buf, size_t cap, int reset);
UHDR_EXTERN int uhdr_b200_enc_rearm(uhdr_codec_private_t* enc);
/* Released handles park their device / pinned arena blocks in a process-wide cache (at most 8 GiB of
 * HBM and 4 GiB of pinned host memory) so that the reference's create / run / release per image pattern
 * does not pay cudaHostAlloc every time.  This returns the cache to the driver; result = bytes freed. */
UHDR_EXTERN size_t uhdr_b200_trim_cache(void);
/* Where JpegDecoderHelper's entropy decoding (libjpeg-turbo jdhuff.c behind jpegdecoderhelper.cpp:397-411)
 * runs: 0 (default) and 2 = on the device for every stream the parallel decoder accepts, whatever its size (the
 * host decoder only takes the streams it declines: restart markers out of sequence or in the wrong number, RST markers
 * without a DRI marker, another marker before EOI, no fixed point, inconsistent data);
 * 1 = host, for tests and triage.  Process-wide; returns the previous setting.  Results are identical either way. */
UHDR_EXTERN int uhdr_b200_set_entropy_decoder(int mode);
/* out[0] = scans entropy-decoded on the device so far, out[1] = scans the device decoder handed back to
 * the host decoder, out[2] = relaxation rounds the last device decode needed */
UHDR_EXTERN void uhdr_b200_entropy_decoder_stats(unsigned long long out[3]);
/* Two-pass generateGainMap with gamma 1 on the fast kernels takes the log2 of the quotient (hdr+eps)/(sdr+eps) only
 * when it maps the quotient to its byte: in fp32 (lg2.approx) wherever the byte provably does not depend on more, in
 * fp64 otherwise.  At map scale 1 a statistics pass finds the extremes of the quotient and a code pass recomputes every
 * quotient and writes its byte; at scales 2 / 4 a float plane carries the quotients to the byte pass.  Other routes
 * (gamma != 1, the generic kernels, UHDR_B200_GAINS_PLANE) do not count here.
 * out[0] = gain values quantised that way since process start, out[1] = how many of them took the fp64 path. */
UHDR_EXTERN void uhdr_b200_generate_stats(unsigned long long out[2]);
/* diagnostic: worst[0] = max over the `count` floats whose bit patterns start at first_bits of
 * |lg2.approx(x) - float(log2(double(x)))| / bound(x), the bound being the one pass 2 relies on (must stay <= 0.5:
 * a factor 2 to spare); host pointer. */
UHDR_EXTERN int uhdr_b200_probe_log2_fast(unsigned first_bits, unsigned count, float* worst);
/* toneMap's fast kernel screens srgbOetf's powf: a 2x2 pixel group first runs with a hardware fp32 approximation and is
 * redone with the exact routine only if one of its six 8-bit codes could depend on the difference.
 * out[0] = groups processed since process start, out[1] = groups redone (current device). */
UHDR_EXTERN void uhdr_b200_tonemap_stats(unsigned long long out[2]);
/* applyGainMap kernel launches since process start, every entry point (host buffers, device pointers, the C++
 * surface, uhdr_decode): out[0] = k_apply_lin1 (scale 1 -> linear half float), out[1] = k_apply_fast (other integer
 * scales up to 16 and the PQ / HLG outputs), out[2] = k_apply_gainmap (every other input), out[3] = gain-map resizes
 * (aspect ratio off by more than 1 %), each followed by one of the other three. */
UHDR_EXTERN void uhdr_b200_apply_stats(unsigned long long out[4]);
/* The encoder's device entropy coder (k_huff_encode) gives each CTA 256 * bpt consecutive blocks of the scan, bpt in
 * 1..8 being the smallest value that makes the whole grid resident at once (8 beyond 8 waves' worth of blocks).  Plans
 * since process start, every entry point: out[0] = resident CTAs per wave the plan assumed (0 before the first
 * encode), out[1..8] = launches with bpt = 1..8, out[9] = launches whose grid exceeded one wave.  Host-side counts. */
UHDR_EXTERN void uhdr_b200_jpeg_encode_stats(unsigned long long out[10]);
/* The batched entropy coder (k_huff_encode_batch, uhdr_b200_transcode_batch: one launch per group of items, bpt chosen by
 * the rule above over all the group's blocks; not counted in uhdr_b200_jpeg_encode_stats).  Since process start:
 * out[0] = launches, out[1] = scans they coded.  Host-side counts. */
UHDR_EXTERN void uhdr_b200_jpeg_encode_batch_stats(unsigned long long out[2]);
/* Per-device kernel state, made once per device on its first use and kept for the life of the process.  Since
 * process start: out[0] = constant tables uploaded to a device (code books, log2 table, zigzag order), out[1] = wave
 * sizes (co-resident CTAs of a kernel) asked of the CUDA runtime.  Host-side counts; needs no device. */
UHDR_EXTERN void uhdr_b200_device_state_stats(unsigned long long out[2]);
/* diagnostic: worst[0] = max |approximate pow(e, 1/2.4) - the exact one| over the `count` floats whose bit patterns
 * start at first_bits (the screen relies on <= 3e-7 for e in (0.0031308, 1]; must measure <= 1.5e-7); host pointer. */
UHDR_EXTERN int uhdr_b200_probe_pow_fast(unsigned first_bits, unsigned count, float* worst);
/* diagnostic: out[i] = float(log2(double(in[i]))) exactly as the gain-map kernels evaluate computeGain's
 * log2 (gainmapmath.cpp:773-782); host pointers. */
UHDR_EXTERN int uhdr_b200_probe_log2(const float* in, float* out, int n);
/* diagnostic: out[i] = powf(in[i], y) as the device evaluates the reference's float std::pow sites */
UHDR_EXTERN int uhdr_b200_probe_powf(const float* in, float y, float* out, int n);

/* LUT blob (OETF / inverse-OETF tables): build on the host with the reference's libm
 * expressions, or install a blob that was broadcast from rank 0 (NCCL) into device memory. */
UHDR_EXTERN size_t uhdr_b200_lut_blob_floats(void);
UHDR_EXTERN int uhdr_b200_build_lut_blob(float* host_out);
UHDR_EXTERN int uhdr_b200_install_lut_blob_dev(const void* device_ptr); /* copies D2D on the current device */
UHDR_EXTERN int uhdr_b200_get_lut_blob(float* host_out);               /* read back what the device holds */

/* Batch API-1 / API-0 encode of independent frames on the current device: `n` frames share one
 * geometry/config; frames are pipelined over `streams` CUDA streams with pinned staging.
 * hdr[i] / sdr[i] host descriptors (sdr == NULL selects API-0); out[i].data must hold
 * out[i].capacity bytes and receives data_sz. */
UHDR_EXTERN int uhdr_b200_encode_batch(int n, const uhdr_raw_image_t* hdr, const uhdr_raw_image_t* sdr,
                                       const uhdr_b200_gm_config_t* cfg, int base_quality,
                                       uhdr_compressed_image_t* out, int streams);

#endif
