// Device-side parameter blocks and launcher prototypes of the gain-map hot path (sm_90a).
// All launchers take DEVICE pointers and a stream; they never synchronise.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace uhdr_b200 {

// uhdr_img_fmt_t values (ultrahdr_api.h)
enum : int { F_P010 = 0, F_YUV420 = 1, F_Y400 = 2, F_RGBA8888 = 3, F_RGBAF16 = 4,
             F_RGBA1010102 = 5, F_YUV444 = 6, F_YUV422 = 7, F_RGB888 = 11, F_YUV444_10 = 12 };
enum : int { CT_LINEAR = 0, CT_HLG = 1, CT_PQ = 2, CT_SRGB = 3 };

struct ImgView {           // device view of a uhdr_raw_image_t
  const void* p[3];
  int stride[3];           // in pixels (elements), like the reference
  int fmt, w, h, full_range;
};

struct GainmapGenParams {  // generateGainMap, lib/src/jpegr.cpp:530-1058
  ImgView hdr, sdr;
  int hdr_ct;
  int map_w, map_h, scale, nch;     // nch = 3 multichannel, 1 single
  float hdr_y2r[4], sdr_y2r[4];     // {cr, cb, gcb, gcr}
  float gamut[9];
  int gamut_on_hdr, gamut_identity; // use_sdr_cg rule, :607-638
  float lum[3];
  int use_luminance;
  float sdr_nits, hdr_nits;         // 203 and hdrSampleToNitsFactor
  const float* luts;                // LUT blob (tables.h)
  // two-pass (BEST_QUALITY)
  float* gains;                     // map_w*map_h*nch floats, tight
  unsigned* minmax;                 // 6 order-preserving keys: min[3], max[3]
  // one-pass (REALTIME) :724-737, encodeGain gainmapmath.cpp:758-771
  float min_boost, max_boost, log2_min, log2_max, gamma;
  // one-pass fast kernels: correctly rounded 1 / double(log2_max - log2_min), or 0 when that range is zero / not finite
  // (then the kernels divide); see encode_gain_norm in gainmap_fast.cu
  double inv_log2_range;
  // two-pass fast kernels at map scale 2 / 4: the float plane receives the quotient (hdr+eps)/(sdr+eps) per value,
  // negated when the pixel is dark (sdr < 2/255), instead of its log2; minmax holds q keys (k_affine_q finishes the job)
  int store_q;
  uint8_t* dst;                     // RGB888 / Y400
  int dst_stride;                   // pixels
};

struct GainmapFinalizeParams {      // clamp / hints, jpegr.cpp:969-986
  unsigned* minmax;                 // in : keys
  float* minmax_f;                  // out: min[3], max[3] as floats after clamping
  int nch;
  float log2_user_max, log2_user_min;
  int has_user_max, has_user_min;
};

struct AffineParams {               // jpegr.cpp:988-1013, affineMapGain gainmapmath.cpp:784-789
  const float* gains;
  const float* minmax_f;
  uint8_t* dst;
  int map_w, map_h, nch, dst_stride;
  float gamma;
};

struct ApplyParams {                // applyGainMap, jpegr.cpp:1533-1831
  ImgView sdr;
  const uint8_t* map;
  int map_w, map_h, map_stride, map_bpp, map_nch;  // bpp 1/3/4 bytes per map pixel, nch 1/3
  int scale_int;                    // integer scale (0 -> use scale_f path)
  float scale_f;
  const float* idw;                 // 4 variants x s*s*4 (device)
  const float* gain_lut;            // 3 x 1024 (device)
  float gamma_inv[3], off_sdr[3], off_hdr[3];
  float y2r[4];                     // BT.601 always (:1723)
  float gamut[9];
  int gamut_on_sdr, gamut_identity; // !use_base_cg -> sdr side
  int out_ct;                       // LINEAR / HLG / PQ
  float out_nits;                   // kHlgMaxNits / kPqMaxNits
  const float* luts;
  void* dst;
  int dst_stride;
  int nan_possible;                 // the gain table is so large that a channel can become inf or NaN
};

struct TonemapParams {              // toneMap, jpegr.cpp:1985-2222
  ImgView hdr;
  int hdr_ct;
  float y2r[4];
  float gamut[9];                   // hdr cg -> P3
  int gamut_identity;
  float headroom;
  int normalized;
  const float* luts;
  uint8_t* dst[3];
  int dst_stride[3];
  int dst_fmt;                      // YUV420 / YUV444 / RGBA8888
};

struct YuvConvParams {              // transformYuv420/444, gainmapmath.cpp:686-748
  const uint8_t* p[3];              // source planes
  int stride[3];
  uint8_t* d[3];                    // destination planes (== p for the reference's in-place form)
  int dstride[3];
  int w, h, fmt;
  float m[9];
};

struct RgbToYccParams {             // convert_raw_input_to_ycbcr, gainmapmath.cpp:1440-1467 (RGBA8888 / RGB888 -> YCbCr 4:4:4)
  const uint8_t* src;
  int src_stride, bpp;              // pixels per row; 4 or 3 bytes per pixel
  uint8_t* dst[3];
  int dst_stride;
  int w, h;
  float k[5];                       // yr, yg, yb, cb, cr
};

struct ResizeMapParams {            // resize_image, editorhelper.cpp:100-146 (gain map to the base image's size)
  const uint8_t* src;
  int src_w, src_h, src_stride, bpp;   // bpp 1 (Y400) / 3 (RGB888) / 4 (RGBA8888)
  uint8_t* dst;
  int dst_w, dst_h, dst_stride;
};

struct Fdct8Plane {                 // one launch covers every plane of an image (fdct8.cu)
  const uint8_t* src;
  int stride;                       // bytes per row for planes, pixels per row for RGB888
  int w, h;                         // RGB: real size (edges replicated); plane: rows (>= h read `fill`)
  int wblocks, hblocks;
  int fill, rgb;
  int tq[3];
  // plane: [0]; RGB888: Y, Cb, Cr.  Natural-order launches: [block][64] coefficients.  Zigzag launches
  // (device entropy coder follows): [block][64] 32-bit code-word entries instead, see fdct8.cu block_code
  int16_t* coefs[3];
  // entropy-coder side information, one uint4 per block (zigzag launches only; may be null):
  //   x       = code bits of the block's AC part (Huffman codes + magnitude bits + ZRLs + EOB) << 16 | DC coefficient
  //   y, z, w = the first 96 bits of the AC part's bit string, MSB first
  uint4* meta[3];
  int hsel[3];                      // Huffman table pair of the component: 0 luminance, 1 chrominance
};
struct Fdct8Params {
  Fdct8Plane plane[3];
  int nplanes, zigzag;
  uint16_t q[2][64];
  unsigned mag[2][64];              // ceil(2^32 / (8*q)), filled by launch_fdct8
  int tile_end[3];                  // cumulative count of 32-block tiles per plane, filled by launch_fdct8
  const uint32_t* acbooks;          // zigzag launches: device pointer, AC code books (code << 8 | length), [0..255] luminance [256..511] chrominance (filled by launch_fdct8)
};

struct IdctPlaneParams {
  const int16_t* coefs;
  uint16_t q[64];
  int wblocks, hblocks;
  uint8_t* dst;
  int dst_stride;                   // >= wblocks*8 unless clipped by dst_w/dst_h
  int dst_w, dst_h;                 // samples beyond are not written
};

// reduced-size IDCT (idct_scaled.cu): the planes of one JPEG whose DCT scaled size is the launch's (4, 2 or 1)
struct IdctScaledParams {
  int nplanes;
  int block_end[3];                 // cumulative block counts: plane i holds blocks [block_end[i-1], block_end[i])
  struct Plane {
    const int16_t* coefs;
    uint16_t q[64];
    int wblocks;
    uint8_t* dst;
    int dst_stride;                 // >= wblocks * size
    int dst_w, dst_h;               // samples beyond are not written
  } plane[3];
};

struct YccToRgbaParams {
  const uint8_t* y; const uint8_t* cb; const uint8_t* cr;
  int src_stride, w, h;
  int hs, vs;                       // chroma subsampling (1,1) (2,1) (2,2)
  int c_stride, cw, ch;             // chroma plane stride and real (downsampled) size
  uint8_t* dst;                     // RGBA8888
  int dst_stride;                   // pixels
};

cudaError_t launch_gainmap_pass1(const GainmapGenParams& p, cudaStream_t s);
cudaError_t launch_gainmap_onepass(const GainmapGenParams& p, cudaStream_t s);
cudaError_t launch_gainmap_init_minmax(unsigned* minmax, cudaStream_t s);
cudaError_t launch_gainmap_finalize(const GainmapFinalizeParams& p, cudaStream_t s);
cudaError_t launch_gainmap_affine(const AffineParams& p, cudaStream_t s);
cudaError_t launch_apply_gainmap(const ApplyParams& p, cudaStream_t s);
// fast path (apply_fast.cu): YUV420 base, integer scale, gamma 1.  gain_u8 = 3x256 composed table
bool apply_fast_eligible(const ApplyParams& p);
cudaError_t launch_apply_fast(const ApplyParams& p, const float* gain_u8, cudaStream_t s);
// fast path (gainmap_fast.cu): P010 + YUV420, scale 1
bool affine_fast_eligible(const AffineParams& p);
// finalize (clamp / hints) + affine in one launch; also writes fin.minmax_f
cudaError_t launch_affine_fast(const AffineParams& p, const GainmapFinalizeParams& fin, cudaStream_t s);
cudaError_t launch_affine_q(const AffineParams& p, const GainmapFinalizeParams& fin, unsigned* exact_count, cudaStream_t s);
cudaError_t launch_init_q_keys(unsigned* minmax, cudaStream_t s);
cudaError_t launch_log2_fast_probe(unsigned first_bits, unsigned count, float* d_worst, cudaStream_t s);
cudaError_t launch_pow_fast_probe(unsigned first_bits, unsigned count, float* d_worst, cudaStream_t s);
void tonemap_screen_stats(unsigned long long out[2]);
bool gainmap_fast_eligible(const GainmapGenParams& p, bool onepass);
cudaError_t launch_gainmap_fast(const GainmapGenParams& p, bool onepass, unsigned* sched, cudaStream_t s);
// two-pass map at scale 1 without a plane, keys set up by launch_init_q_keys: the statistics pass (code = false) leaves
// the extremes of the quotient in p.minmax; the code pass (code = true) recomputes every quotient and writes its byte to
// p.dst, fin.minmax_f and the exact-path count.  sched: a zeroed tile-ticket word per pass.
cudaError_t launch_gainmap_q2(const GainmapGenParams& p, const GainmapFinalizeParams& fin, bool code, unsigned* sched,
                              unsigned* exact_count, cudaStream_t s);
cudaError_t launch_log2_probe(const float* d_in, float* d_out, int n, cudaStream_t s);
cudaError_t launch_powf_probe(const float* d_in, float y, float* d_out, int n, cudaStream_t s);
cudaError_t launch_tonemap(const TonemapParams& p, cudaStream_t s);
bool tonemap_fast_eligible(const TonemapParams& p);
cudaError_t launch_tonemap_fast(const TonemapParams& p, cudaStream_t s);
cudaError_t launch_yuv_convert(const YuvConvParams& p, cudaStream_t s);
bool yuv420_fast_eligible(const YuvConvParams& p);
cudaError_t launch_yuv420_fast(const YuvConvParams& p, cudaStream_t s);
cudaError_t launch_rgb_to_ycc(const RgbToYccParams& p, cudaStream_t s);
cudaError_t launch_resize_map(const ResizeMapParams& p, cudaStream_t s);
cudaError_t launch_fdct8(const Fdct8Params& p, cudaStream_t s);
cudaError_t launch_idct_dequant(const IdctPlaneParams& p, cudaStream_t s);
cudaError_t launch_idct_scaled(const IdctScaledParams& p, int size, cudaStream_t s);
cudaError_t launch_ycc_to_rgba(const YccToRgbaParams& p, cudaStream_t s);

// number of kernel launches issued by this library since load (bench.py's gpu_launches)
unsigned long long launch_count();
void count_launches(unsigned n);  // launches made outside kernels.cu (fast paths, JPEG stages)

}  // namespace uhdr_b200
