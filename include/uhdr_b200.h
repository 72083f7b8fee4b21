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
 * out must hold `cap` bytes. */
UHDR_EXTERN int uhdr_b200_jpeg_encode(const uhdr_raw_image_t* img, int quality, const void* icc,
                                      size_t icc_size, void* out, size_t cap, size_t* out_size);
/* forward block stage only: quantised coefficients per component, raster block order, natural
 * order inside a block (parity hook for FDCT + quantise). coefs[c] sized wblocks*hblocks*64. */
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
/* uhdr_b200_jpeg_decode of one JPEG at 1/k (stage hook, host buffers).  k = 1 is uhdr_b200_jpeg_decode.  For k > 1,
 * mode 0 gives Y400 or YUV444 planes of ceil(w / k) x ceil(h / k) samples, back to back at stride = width; mode 1
 * gives RGBA8888 at that size. */
UHDR_EXTERN int uhdr_b200_jpeg_decode_scaled(const void* data, size_t size, int mode, int k, uhdr_raw_image_t* out,
                                             size_t cap);
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
 * bytes of uhdr_b200_jpeg_encode; the stream goes to the HOST buffer out. */
UHDR_EXTERN int uhdr_b200_jpeg_encode_dev(const uhdr_raw_image_t* img_dev, int quality, const void* icc,
                                          size_t icc_size, void* out, size_t cap, size_t* out_size, void* stream);

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
