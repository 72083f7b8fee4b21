// Hand-written sm_90a kernels for the gain-map hot path.  Compile with -fmad=false: the
// reference CPU path is x86-64 baseline (SSE2, no FMA, lib CMakeLists.txt:290-301), so every
// float expression below must round after each operation, in the reference's operand order.
// Transcendentals are table fetches (tables.h) except where noted.  No tensor cores: this is
// scalar per-pixel work bounded by HBM traffic and instruction issue.
#include "kernels.cuh"

#include <atomic>

#include "powf_glibc.cuh"
#include "tables.h"

namespace uhdr_b200 {

static std::atomic<unsigned long long> g_launches{0};
unsigned long long launch_count() { return g_launches.load(); }
void count_launches(unsigned n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
#define COUNT_LAUNCH() g_launches.fetch_add(1, std::memory_order_relaxed)

struct C3 { float r, g, b; };  // also y,u,v

// ------------------------------------------------------------------------------------------------
// small device helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float clamp01(float v) { return v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v); }
__device__ __forceinline__ float clip_neg(float v) { return v < 0.0f ? 0.0f : v; }

// index = int32(double(x * (N-1)) + 0.5) clamped to [0, N-1]  (gainmapmath.cpp:127,249,272,321,
// 340; gainmapmath.h:485).  Evaluated without fp64: floor(v) + (frac >= .5) is the same integer
// because v - trunc(v) is exact in binary32.
__device__ __forceinline__ int lut_index(float x, float nm1f, int nm1) {
  float v = x * nm1f;
  if (!(v > 0.0f)) return 0;
  int i = __float2int_rz(v);
  float fr = v - (float)i;
  i += (fr >= 0.5f) ? 1 : 0;
  return min(i, nm1);
}
__device__ __forceinline__ float lut1024(const float* __restrict__ t, float x) {
  return __ldg(t + lut_index(x, 1023.0f, 1023));
}
__device__ __forceinline__ float lut4096(const float* __restrict__ t, float x) {
  return __ldg(t + lut_index(x, 4095.0f, 4095));
}
__device__ __forceinline__ float lut65536(const float* __restrict__ t, float x) {
  return __ldg(t + lut_index(x, 65535.0f, 65535));
}

__device__ __forceinline__ C3 yuv_to_rgb(const float* k, C3 e) {  // k = {cr, cb, gcb, gcr}
  C3 o;
  o.r = clamp01(e.r + k[0] * e.b);
  o.g = clamp01(e.r - k[2] * e.g - k[3] * e.b);
  o.b = clamp01(e.r + k[1] * e.g);
  return o;
}
__device__ __forceinline__ C3 mat3(const float* c, C3 e) {
  C3 o;
  o.r = c[0] * e.r + c[1] * e.g + c[2] * e.b;
  o.g = c[3] * e.r + c[4] * e.g + c[5] * e.b;
  o.b = c[6] * e.r + c[7] * e.g + c[8] * e.b;
  return o;
}

// gainmapmath.h:193-216 (Skia half_to_float_fast2)
__device__ __forceinline__ float half_to_float_ref(unsigned h) {
  unsigned e = (h >> 10) & 0x1f, m = h & 0x3ff;
  unsigned o;
  if (e == 0) {
    float f = __uint_as_float((126u << 23) + m) - __uint_as_float(126u << 23);
    o = __float_as_uint(f);
  } else {
    o = m << 13;
    o |= e == 0x1f ? (255u << 23) : ((127 - 15 + e) << 23);
  }
  o |= (h >> 15) << 31;
  return __uint_as_float(o);
}
__device__ __forceinline__ float sanitize1(float v) {  // gainmapmath.h:572-593
  const float kMax = 10000.0f / 203.0f;
  if (isfinite(v)) return v < 0.0f ? 0.0f : (v > kMax ? kMax : v);
  if (isinf(v)) return v > 0 ? kMax : 0.0f;
  return 0.0f;
}
// gainmapmath.h:160-173 (add-half then truncate; denormals by shifting; saturate 0x7FFF)
__device__ __forceinline__ unsigned float_to_half_ref(float f) {
  const unsigned b = __float_as_uint(f) + 0x00001000u;
  const int e = (int)((b & 0x7F800000u) >> 23);
  const unsigned m = b & 0x007FFFFFu;
  unsigned r = (b & 0x80000000u) >> 16;
  if (e > 112) r |= ((((unsigned)(e - 112)) << 10) & 0x7C00u) | (m >> 13);
  if (e < 113 && e > 101) r |= (((0x007FF000u + m) >> (125 - e)) + 1) >> 1;
  if (e > 143) r |= 0x7FFFu;
  return r & 0xFFFFu;
}

// ------------------------------------------------------------------------------------------------
// pixel fetch (gainmapmath.cpp:354-492).  Returns gamma-domain YUV (or RGB for packed formats).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ C3 fetch_pixel(const ImgView& im, int x, int y) {
  C3 c = {0.f, 0.f, 0.f};
  switch (im.fmt) {
    case F_YUV420:
    case F_YUV422:
    case F_YUV444: {
      const int hs = im.fmt == F_YUV444 ? 0 : 1, vs = im.fmt == F_YUV420 ? 1 : 0;
      int yy = __ldg((const uint8_t*)im.p[0] + x + (size_t)y * im.stride[0]);
      int u = __ldg((const uint8_t*)im.p[1] + (x >> hs) + (size_t)(y >> vs) * im.stride[1]);
      int v = __ldg((const uint8_t*)im.p[2] + (x >> hs) + (size_t)(y >> vs) * im.stride[2]);
      c.r = (float)yy * (1 / 255.0f);
      c.g = (float)(u - 128) * (1 / 255.0f);
      c.b = (float)(v - 128) * (1 / 255.0f);
      break;
    }
    case F_Y400:
      c.r = (float)__ldg((const uint8_t*)im.p[0] + x + (size_t)y * im.stride[0]) * (1 / 255.0f);
      break;
    case F_P010:
    case F_YUV444_10: {
      int yy, u, v;
      if (im.fmt == F_P010) {
        const uint16_t* uv = (const uint16_t*)im.p[1] + (size_t)(y >> 1) * im.stride[1] + (x & ~1);
        yy = __ldg((const uint16_t*)im.p[0] + (size_t)y * im.stride[0] + x) >> 6;
        u = __ldg(uv) >> 6;
        v = __ldg(uv + 1) >> 6;
      } else {
        yy = __ldg((const uint16_t*)im.p[0] + (size_t)y * im.stride[0] + x);
        u = __ldg((const uint16_t*)im.p[1] + (size_t)y * im.stride[1] + x);
        v = __ldg((const uint16_t*)im.p[2] + (size_t)y * im.stride[2] + x);
      }
      if (im.full_range) {
        c.r = (float)yy / 1023.0f;
        c.g = (float)u / 1023.0f - 0.5f;
        c.b = (float)v / 1023.0f - 0.5f;
      } else {
        c.r = (float)(yy - 64) * (1 / 876.0f);
        c.g = (float)(u - 64) * (1 / 896.0f) - 0.5f;
        c.b = (float)(v - 64) * (1 / 896.0f) - 0.5f;
      }
      break;
    }
    case F_RGB888: {
      const uint8_t* p = (const uint8_t*)im.p[0] + ((size_t)y * im.stride[0] + x) * 3;
      c.r = (float)__ldg(p) / 255.0f;
      c.g = (float)__ldg(p + 1) / 255.0f;
      c.b = (float)__ldg(p + 2) / 255.0f;
      break;
    }
    case F_RGBA8888: {
      unsigned p = __ldg((const unsigned*)im.p[0] + (size_t)y * im.stride[0] + x);
      c.r = (float)(p & 0xff) / 255.0f;
      c.g = (float)((p >> 8) & 0xff) / 255.0f;
      c.b = (float)((p >> 16) & 0xff) / 255.0f;
      break;
    }
    case F_RGBA1010102: {
      unsigned p = __ldg((const unsigned*)im.p[0] + (size_t)y * im.stride[0] + x);
      c.r = (float)(p & 0x3ff) / 1023.0f;
      c.g = (float)((p >> 10) & 0x3ff) / 1023.0f;
      c.b = (float)((p >> 20) & 0x3ff) / 1023.0f;
      break;
    }
    case F_RGBAF16: {
      uint2 p = __ldg((const uint2*)im.p[0] + (size_t)y * im.stride[0] + x);
      c.r = sanitize1(half_to_float_ref(p.x & 0xffff));
      c.g = sanitize1(half_to_float_ref(p.x >> 16));
      c.b = sanitize1(half_to_float_ref(p.y & 0xffff));
      break;
    }
  }
  return c;
}
__device__ __forceinline__ bool fmt_is_rgb(int f) {  // isPixelFormatRgb gainmapmath.cpp:1274
  return f == F_RGBAF16 || f == F_RGBA8888 || f == F_RGBA1010102;
}
// samplePixels gainmapmath.cpp:494-504
__device__ __forceinline__ C3 sample_pixels(const ImgView& im, int s, int x, int y) {
  if (s == 1) return fetch_pixel(im, x, y);  // (0 + p) / 1.0f == p
  C3 e = {0.f, 0.f, 0.f};
  for (int dy = 0; dy < s; dy++)
    for (int dx = 0; dx < s; dx++) {
      C3 p = fetch_pixel(im, x * s + dx, y * s + dy);
      e.r += p.r;
      e.g += p.g;
      e.b += p.b;
    }
  const float d = (float)(s * s);
  e.r /= d;
  e.g /= d;
  e.b /= d;
  return e;
}

// hdr gamma -> linear (+ HLG OOTF folded into the table), gainmapmath.cpp:1159-1201
__device__ __forceinline__ C3 hdr_linearize(const float* __restrict__ luts, int ct, C3 g) {
  C3 o = g;
  if (ct == CT_HLG) {
    const float* t = luts + kLutHlgInvOotf;
    o.r = lut4096(t, g.r); o.g = lut4096(t, g.g); o.b = lut4096(t, g.b);
  } else if (ct == CT_PQ) {
    const float* t = luts + kLutPqInv;
    o.r = lut4096(t, g.r); o.g = lut4096(t, g.g); o.b = lut4096(t, g.b);
  } else if (ct == CT_SRGB) {
    const float* t = luts + kLutSrgbInv;
    o.r = lut1024(t, g.r); o.g = lut1024(t, g.g); o.b = lut1024(t, g.b);
  }
  return o;
}
__device__ __forceinline__ C3 srgb_linearize(const float* __restrict__ luts, C3 g) {
  const float* t = luts + kLutSrgbInv;
  C3 o;
  o.r = lut1024(t, g.r); o.g = lut1024(t, g.g); o.b = lut1024(t, g.b);
  return o;
}

// order-preserving float <-> uint key for atomicMin/Max
__device__ __forceinline__ unsigned fkey(float f) {
  unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// ------------------------------------------------------------------------------------------------
// generateGainMap: shared per-map-pixel front end (jpegr.cpp:753-786 == :866-898)
// out: sdr / hdr values in nits for nch channels
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void gm_front(const GainmapGenParams& p, int x, int y, float sv[3],
                                         float hv[3]) {
  C3 sg = sample_pixels(p.sdr, p.scale, x, y);
  if (!fmt_is_rgb(p.sdr.fmt)) sg = yuv_to_rgb(p.sdr_y2r, sg);
  C3 sl = srgb_linearize(p.luts, sg);
  if (!p.gamut_on_hdr && !p.gamut_identity) sl = mat3(p.gamut, sl);
  sl.r = clip_neg(sl.r); sl.g = clip_neg(sl.g); sl.b = clip_neg(sl.b);

  C3 hg = sample_pixels(p.hdr, p.scale, x, y);
  if (!fmt_is_rgb(p.hdr.fmt)) hg = yuv_to_rgb(p.hdr_y2r, hg);
  C3 hl = hdr_linearize(p.luts, p.hdr_ct, hg);
  if (p.gamut_on_hdr && !p.gamut_identity) hl = mat3(p.gamut, hl);
  hl.r = clip_neg(hl.r); hl.g = clip_neg(hl.g); hl.b = clip_neg(hl.b);

  if (p.nch == 3) {
    sv[0] = sl.r * p.sdr_nits; sv[1] = sl.g * p.sdr_nits; sv[2] = sl.b * p.sdr_nits;
    hv[0] = hl.r * p.hdr_nits; hv[1] = hl.g * p.hdr_nits; hv[2] = hl.b * p.hdr_nits;
  } else if (p.use_luminance) {
    sv[0] = (p.lum[0] * sl.r + p.lum[1] * sl.g + p.lum[2] * sl.b) * p.sdr_nits;
    hv[0] = (p.lum[0] * hl.r + p.lum[1] * hl.g + p.lum[2] * hl.b) * p.hdr_nits;
  } else {
    sv[0] = fmaxf(sl.r, fmaxf(sl.g, sl.b)) * p.sdr_nits;
    hv[0] = fmaxf(hl.r, fmaxf(hl.g, hl.b)) * p.hdr_nits;
  }
}

// computeGain gainmapmath.cpp:773-782: double log2 of a float quotient, narrowed to float
__device__ __forceinline__ float compute_gain(float sdr, float hdr) {
  float gain = (float)log2((double)((hdr + 1e-7f) / (sdr + 1e-7f)));
  if (sdr < 2.f / 255.0f) gain = fminf(gain, 2.3f);
  return gain;
}

constexpr int kGmPx = 4;  // map pixels per thread (12-byte RGB888 store / 4-byte Y400 store)

__global__ void __launch_bounds__(256) k_gainmap_pass1(const GainmapGenParams p) {
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * kGmPx;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  float mn[3] = {127.0f, 127.0f, 127.0f}, mx[3] = {-128.0f, -128.0f, -128.0f};
  if (y < p.map_h) {
    for (int i = 0; i < kGmPx; i++) {
      const int x = x0 + i;
      if (x >= p.map_w) break;
      float sv[3], hv[3];
      gm_front(p, x, y, sv, hv);
      float* g = p.gains + ((size_t)y * p.map_w + x) * p.nch;
      for (int c = 0; c < p.nch; c++) {
        float v = compute_gain(sv[c], hv[c]);
        g[c] = v;
        mn[c] = fminf(mn[c], v);
        mx[c] = fmaxf(mx[c], v);
      }
    }
  }
  // warp shuffle -> shared -> one atomic per block and channel (min/max are order independent,
  // so the result equals the reference's mutex-merged per-thread extrema, jpegr.cpp:932-938)
  __shared__ unsigned s_mn[3][8], s_mx[3][8];
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  for (int c = 0; c < p.nch; c++) {
    unsigned kmn = fkey(mn[c]), kmx = fkey(mx[c]);
    for (int o = 16; o; o >>= 1) {
      kmn = min(kmn, __shfl_xor_sync(0xffffffffu, kmn, o));
      kmx = max(kmx, __shfl_xor_sync(0xffffffffu, kmx, o));
    }
    if (lane == 0) { s_mn[c][warp] = kmn; s_mx[c][warp] = kmx; }
  }
  __syncthreads();
  if (warp == 0) {
    const int nw = (blockDim.x * blockDim.y) >> 5;
    for (int c = 0; c < p.nch; c++) {
      unsigned kmn = lane < nw ? s_mn[c][lane] : 0xffffffffu;
      unsigned kmx = lane < nw ? s_mx[c][lane] : 0u;
      for (int o = 4; o; o >>= 1) {
        kmn = min(kmn, __shfl_xor_sync(0xffffffffu, kmn, o));
        kmx = max(kmx, __shfl_xor_sync(0xffffffffu, kmx, o));
      }
      if (lane == 0) {
        atomicMin(p.minmax + c, kmn);
        atomicMax(p.minmax + 3 + c, kmx);
      }
    }
  }
}

__global__ void k_gainmap_init_minmax(unsigned* mm) {
  if (threadIdx.x < 3) mm[threadIdx.x] = fkey(127.0f);
  else if (threadIdx.x < 6) mm[threadIdx.x] = fkey(-128.0f);
  else if (threadIdx.x == 8) mm[8] = 0;  // tile-ticket counter of k_gainmap_fast
}

// jpegr.cpp:969-986 on the device so pass 2 can follow without a host round trip
__global__ void k_gainmap_finalize(const GainmapFinalizeParams p) {
  const int c = threadIdx.x;
  if (c >= 3) return;
  float mn = fkey_inv(p.minmax[c < p.nch ? c : 0]);
  float mx = fkey_inv(p.minmax[3 + (c < p.nch ? c : 0)]);
  mn = mn < -14.3f ? -14.3f : (mn > 15.6f ? 15.6f : mn);
  mx = mx < -14.3f ? -14.3f : (mx > 15.6f ? 15.6f : mx);
  if (p.has_user_max) mx = fminf(mx, p.log2_user_max);
  if (p.has_user_min) mn = fmaxf(mn, p.log2_user_min);
  if (fabsf(mx - mn) < 1.1920928955078125e-07f) mx += 0.1f;
  p.minmax_f[c] = mn;
  p.minmax_f[3 + c] = mx;
}

// affineMapGain gainmapmath.cpp:784-789
__device__ __forceinline__ unsigned affine_map(float g, float mn, float mx, float gamma) {
  float m = (g - mn) / (mx - mn);
  if (gamma != 1.0f) m = (float)pow((double)m, (double)gamma);
  m *= 255.0f;
  float t = m + 0.5f;
  t = t < 0.0f ? 0.0f : (t > 255.0f ? 255.0f : t);
  return (unsigned)__float2int_rz(t) & 0xff;  // NaN -> 0 like cvttss2si's low byte
}

__global__ void __launch_bounds__(256) k_gainmap_affine(const AffineParams p) {
  // one thread = 4 consecutive output bytes of one map row
  const int row_bytes = p.map_w * p.nch;
  const int b0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int y = blockIdx.y;
  if (b0 >= row_bytes) return;
  const float* g = p.gains + (size_t)y * row_bytes + b0;
  uint8_t* d = p.dst + (size_t)y * p.dst_stride * p.nch + b0;
  unsigned v[4];
  const int n = min(4, row_bytes - b0);
  for (int i = 0; i < n; i++) {
    const int c = (b0 + i) % p.nch;
    v[i] = affine_map(g[i], p.minmax_f[c], p.minmax_f[3 + c], p.gamma);
  }
  if (n == 4 && ((((size_t)d) & 3) == 0)) {
    *(unsigned*)d = v[0] | (v[1] << 8) | (v[2] << 16) | (v[3] << 24);
  } else {
    for (int i = 0; i < n; i++) d[i] = (uint8_t)v[i];
  }
}

// encodeGain gainmapmath.cpp:758-771
__device__ __forceinline__ unsigned encode_gain(const GainmapGenParams& p, float y_sdr, float y_hdr) {
  float gain = 1.0f;
  if (y_sdr > 0.0f) gain = y_hdr / y_sdr;
  if (gain < p.min_boost) gain = p.min_boost;
  if (gain > p.max_boost) gain = p.max_boost;
  float gn = (float)((log2((double)gain) - (double)p.log2_min) / (double)(p.log2_max - p.log2_min));
  float gg = p.gamma == 1.0f ? gn : powf_glibc(gn, p.gamma);  // powf(x, 1.0f) == x
  return (unsigned)__float2int_rz(gg * 255.0f) & 0xff;
}

__global__ void __launch_bounds__(256) k_gainmap_onepass(const GainmapGenParams p) {
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * kGmPx;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (y >= p.map_h || x0 >= p.map_w) return;
  uint8_t* d = p.dst + ((size_t)y * p.dst_stride + x0) * p.nch;
  for (int i = 0; i < kGmPx; i++) {
    const int x = x0 + i;
    if (x >= p.map_w) break;
    float sv[3], hv[3];
    gm_front(p, x, y, sv, hv);
    for (int c = 0; c < p.nch; c++) d[i * p.nch + c] = (uint8_t)encode_gain(p, sv[c], hv[c]);
  }
}

// ------------------------------------------------------------------------------------------------
// applyGainMap  jpegr.cpp:1714-1811
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float map_u8(const float* __restrict__ luts, unsigned v) {
  return __ldg(luts + kLutU8Div255 + v);  // float(v) / 255.0f, tabulated on the host
}

// sampleMap / sampleMap3Channel with ShepardsIDW tables, gainmapmath.cpp:920-956,1026-1080
__device__ __forceinline__ void sample_map_int(const ApplyParams& p, int x, int y, float g[3]) {
  const int s = p.scale_int;
  const uint8_t* __restrict__ m = p.map;
  if (s == 1) {  // weights are {1,0,0,0}: e1*1 + e2*0 + e3*0 + e4*0 == e1 for finite taps
    const int xl = min(x, p.map_w - 1), yl = min(y, p.map_h - 1);
    const uint8_t* q = m + ((size_t)yl * p.map_stride + xl) * p.map_bpp;
    if (p.map_bpp == 4) {
      unsigned v = __ldg((const unsigned*)q);
      g[0] = map_u8(p.luts, v & 0xff); g[1] = map_u8(p.luts, (v >> 8) & 0xff);
      g[2] = map_u8(p.luts, (v >> 16) & 0xff);
    } else {
      for (int c = 0; c < p.map_nch; c++) g[c] = map_u8(p.luts, __ldg(q + c));
    }
    return;
  }
  int xl = x / s, yl = y / s;
  int xu = min(xl + 1, p.map_w - 1), yu = min(yl + 1, p.map_h - 1);
  xl = min(xl, p.map_w - 1);
  yl = min(yl, p.map_h - 1);
  const int ox = x % s, oy = y % s;
  int variant = 0;
  if (xl == xu && yl == yu) variant = 3;
  else if (xl == xu) variant = 1;
  else if (yl == yu) variant = 2;
  const float* __restrict__ w = p.idw + ((size_t)variant * s * s + (size_t)oy * s + ox) * 4;
  const float w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2), w3 = __ldg(w + 3);
  const size_t i1 = ((size_t)yl * p.map_stride + xl) * p.map_bpp;
  const size_t i2 = ((size_t)yu * p.map_stride + xl) * p.map_bpp;
  const size_t i3 = ((size_t)yl * p.map_stride + xu) * p.map_bpp;
  const size_t i4 = ((size_t)yu * p.map_stride + xu) * p.map_bpp;
  for (int c = 0; c < p.map_nch; c++) {
    float e1 = map_u8(p.luts, __ldg(m + i1 + c)), e2 = map_u8(p.luts, __ldg(m + i2 + c));
    float e3 = map_u8(p.luts, __ldg(m + i3 + c)), e4 = map_u8(p.luts, __ldg(m + i4 + c));
    g[c] = e1 * w0 + e2 * w1 + e3 * w2 + e4 * w3;
  }
}

// non-integer scale: on-the-fly IDW, gainmapmath.cpp:871-918, 958-1024
__device__ __forceinline__ float pyth(float xd, float yd) {
  // sqrt(pow(x,2.0) + pow(y,2.0)) in double: the squares of binary32 values are exact in
  // binary64, IEEE sqrt is correctly rounded on the device
  return (float)sqrt((double)xd * (double)xd + (double)yd * (double)yd);
}
__device__ __forceinline__ void sample_map_float(const ApplyParams& p, int x, int y, float g[3]) {
  const float xm = (float)x / p.scale_f, ym = (float)y / p.scale_f;
  int xl = (int)floorf(xm), yl = (int)floorf(ym);
  int xu = min(xl + 1, p.map_w - 1), yu = min(yl + 1, p.map_h - 1);
  xl = min(xl, p.map_w - 1);
  yl = min(yl, p.map_h - 1);
  const float d1 = pyth(xm - (float)xl, ym - (float)yl), d2 = pyth(xm - (float)xl, ym - (float)yu);
  const float d3 = pyth(xm - (float)xu, ym - (float)yl), d4 = pyth(xm - (float)xu, ym - (float)yu);
  int early = -1;
  float w0 = 0, w1 = 0, w2 = 0, w3 = 0;
  if (d1 == 0.0f) early = 0;
  else if (d2 == 0.0f) early = 1;
  else if (d3 == 0.0f) early = 2;
  else if (d4 == 0.0f) early = p.map_nch == 1 ? 1 : 3;  // :908 returns e2 in the 1-channel code
  else {
    const float a = 1.0f / d1, b = 1.0f / d2, c = 1.0f / d3, d = 1.0f / d4;
    const float tot = a + b + c + d;
    w0 = a / tot; w1 = b / tot; w2 = c / tot; w3 = d / tot;
  }
  const uint8_t* __restrict__ m = p.map;
  const size_t i1 = ((size_t)yl * p.map_stride + xl) * p.map_bpp;
  const size_t i2 = ((size_t)yu * p.map_stride + xl) * p.map_bpp;
  const size_t i3 = ((size_t)yl * p.map_stride + xu) * p.map_bpp;
  const size_t i4 = ((size_t)yu * p.map_stride + xu) * p.map_bpp;
  for (int c = 0; c < p.map_nch; c++) {
    float e1 = map_u8(p.luts, __ldg(m + i1 + c)), e2 = map_u8(p.luts, __ldg(m + i2 + c));
    float e3 = map_u8(p.luts, __ldg(m + i3 + c)), e4 = map_u8(p.luts, __ldg(m + i4 + c));
    g[c] = early < 0 ? e1 * w0 + e2 * w1 + e3 * w2 + e4 * w3
                     : (early == 0 ? e1 : early == 1 ? e2 : early == 2 ? e3 : e4);
  }
}

// GainLUT::getGainFactor gainmapmath.h:483-489
__device__ __forceinline__ float gain_factor(const float* __restrict__ lut, float gain, float ginv) {
  if (ginv != 1.0f) gain = (float)pow((double)gain, (double)ginv);
  return __ldg(lut + lut_index(gain, 1023.0f, 1023));
}

__device__ __forceinline__ void apply_one(const ApplyParams& p, int x, int y, C3 g, unsigned out[2]) {
  // g: gamma-domain sdr pixel as fetched.  isPixelFormatRgb() is false for RGB888, so the
  // reference runs the BT.601 yuv->rgb step on it too (:1719-1724); mirrored here.
  if (!fmt_is_rgb(p.sdr.fmt)) g = yuv_to_rgb(p.y2r, g);
  C3 l = srgb_linearize(p.luts, g);
  if (p.gamut_on_sdr && !p.gamut_identity) l = mat3(p.gamut, l);
  float gn[3];
  if (p.scale_int) sample_map_int(p, x, y, gn);
  else sample_map_float(p, x, y, gn);
  C3 h;
  if (p.map_nch == 1) {  // applyGainLUT(Color, float) gainmapmath.cpp:807-810
    const float f = gain_factor(p.gain_lut, gn[0], p.gamma_inv[0]);
    h.r = ((l.r + p.off_sdr[0]) * f) - p.off_hdr[0];
    h.g = ((l.g + p.off_sdr[0]) * f) - p.off_hdr[0];
    h.b = ((l.b + p.off_sdr[0]) * f) - p.off_hdr[0];
  } else {               // :848-855
    const float fr = gain_factor(p.gain_lut, gn[0], p.gamma_inv[0]);
    const float fg = gain_factor(p.gain_lut + 1024, gn[1], p.gamma_inv[1]);
    const float fb = gain_factor(p.gain_lut + 2048, gn[2], p.gamma_inv[2]);
    h.r = ((l.r + p.off_sdr[0]) * fr) - p.off_hdr[0];
    h.g = ((l.g + p.off_sdr[1]) * fg) - p.off_hdr[1];
    h.b = ((l.b + p.off_sdr[2]) * fb) - p.off_hdr[2];
  }
  if (p.out_ct == CT_LINEAR) {
    if (!p.gamut_on_sdr && !p.gamut_identity) h = mat3(p.gamut, h);
    const float kMax = 10000.0f / 203.0f;
    h.r = h.r < 0.0f ? 0.0f : (h.r > kMax ? kMax : h.r);
    h.g = h.g < 0.0f ? 0.0f : (h.g > kMax ? kMax : h.g);
    h.b = h.b < 0.0f ? 0.0f : (h.b > kMax ? kMax : h.b);
    // a NaN passes the clamp as in the reference (0 * inf or inf - inf once max_content_boost puts +inf
    // into the gain table); the reference's is x86's default NaN 0xFFC00000, the device's 0x7FFFFFFF
    const float kNaN = __uint_as_float(0xFFC00000u);
    if (h.r != h.r) h.r = kNaN;
    if (h.g != h.g) h.g = kNaN;
    if (h.b != h.b) h.b = kNaN;
    out[0] = float_to_half_ref(h.r) | (float_to_half_ref(h.g) << 16);
    out[1] = float_to_half_ref(h.b) | (0x3C00u << 16);
  } else {
    h.r = h.r * 203.0f / p.out_nits;
    h.g = h.g * 203.0f / p.out_nits;
    h.b = h.b * 203.0f / p.out_nits;
    if (!p.gamut_on_sdr && !p.gamut_identity) h = mat3(p.gamut, h);
    h.r = clamp01(h.r); h.g = clamp01(h.g); h.b = clamp01(h.b);
    const float* t;
    if (p.out_ct == CT_HLG) {
      // hlgInverseOotfApprox: float std::pow(x, 1/1.2f) on a continuous argument: glibc's powf,
      // operation for operation (powf_glibc.cuh)
      const float ex = 1.0f / 1.2f;
      h.r = powf_glibc(h.r, ex);
      h.g = powf_glibc(h.g, ex);
      h.b = powf_glibc(h.b, ex);
      t = p.luts + kLutHlgOetf;
    } else {
      t = p.luts + kLutPqOetf;
    }
    const float er = lut65536(t, h.r), eg = lut65536(t, h.g), eb = lut65536(t, h.b);
    // colorToRgba1010102 gainmapmath.cpp:1279-1284
    float a = er * 1023.0f + 0.5f, b = eg * 1023.0f + 0.5f, c = eb * 1023.0f + 0.5f;
    a = a < 0.0f ? 0.0f : (a > 1023.0f ? 1023.0f : a);
    b = b < 0.0f ? 0.0f : (b > 1023.0f ? 1023.0f : b);
    c = c < 0.0f ? 0.0f : (c > 1023.0f ? 1023.0f : c);
    out[0] = (unsigned)__float2int_rz(a) | ((unsigned)__float2int_rz(b) << 10) |
             ((unsigned)__float2int_rz(c) << 20) | (0x3u << 30);
    out[1] = 0;
  }
}

// one thread = 2 horizontally adjacent pixels (shared chroma sample for 4:2:0 / 4:2:2);
// a warp writes 512 contiguous bytes of RGBA-F16 (or 256 of 1010102) per row.  x, y: relative to the region origin
// (p.ox, p.oy), which ORG = false takes as 0, 0: the whole-image kernel.
template <bool ORG>
__global__ void __launch_bounds__(256) k_apply_gainmap(const ApplyParams p) {
  const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= p.sdr.w || y >= p.sdr.h) return;
  const bool two = x + 1 < p.sdr.w;
  const int ax = ORG ? p.ox + x : x, ay = ORG ? p.oy + y : y;
  C3 g0 = fetch_pixel(p.sdr, ax, ay);
  C3 g1 = two ? fetch_pixel(p.sdr, ax + 1, ay) : g0;
  unsigned o0[2], o1[2] = {0, 0};
  apply_one(p, ax, ay, g0, o0);
  if (two) apply_one(p, ax + 1, ay, g1, o1);
  if (p.out_ct == CT_LINEAR) {
    uint2* d = (uint2*)p.dst + (size_t)y * p.dst_stride + x;
    if (two && ((((size_t)d) & 15) == 0)) {
      *(uint4*)d = make_uint4(o0[0], o0[1], o1[0], o1[1]);
    } else {
      d[0] = make_uint2(o0[0], o0[1]);
      if (two) d[1] = make_uint2(o1[0], o1[1]);
    }
  } else {
    unsigned* d = (unsigned*)p.dst + (size_t)y * p.dst_stride + x;
    if (two && ((((size_t)d) & 7) == 0)) {
      *(uint2*)d = make_uint2(o0[0], o1[0]);
    } else {
      d[0] = o0[0];
      if (two) d[1] = o1[0];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// toneMap  jpegr.cpp:2147-2202
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float srgb_oetf_dev(float e) {  // gainmapmath.cpp:139-148
  if (e <= 0.0031308f) return 12.92f * e;
  // float std::pow with a continuous argument: glibc's powf, operation for operation
  return (1.0f + 0.055f) * powf_glibc(e, 1.0f / 2.4f) - 0.055f;
}
__device__ __forceinline__ unsigned scale_to_8bit(float v) {  // :1979-1983 std::round
  int i = __float2int_rz(roundf(v * 255.0f));
  return (unsigned)min(max(i, 0), 255);
}
__device__ __forceinline__ C3 tonemap_px(const TonemapParams& p, int x, int y) {
  C3 g = fetch_pixel(p.hdr, x, y);
  if (!fmt_is_rgb(p.hdr.fmt)) g = yuv_to_rgb(p.y2r, g);
  C3 l = hdr_linearize(p.luts, p.hdr_ct, g);
  // globalTonemap :1951-1977
  C3 h = l;
  if (p.normalized) { h.r = l.r * p.headroom; h.g = l.g * p.headroom; h.b = l.b * p.headroom; }
  float max_hdr = h.r;
  if (h.g > max_hdr) max_hdr = h.g;
  if (h.b > max_hdr) max_hdr = h.b;
  float o = 1.0f + max_hdr / (p.headroom * p.headroom);
  o /= 1.0f + max_hdr;
  const float max_sdr = o * max_hdr;
  C3 s;
  s.r = h.r > 0.0f ? h.r * max_sdr / max_hdr : 0.0f;
  s.g = h.g > 0.0f ? h.g * max_sdr / max_hdr : 0.0f;
  s.b = h.b > 0.0f ? h.b * max_sdr / max_hdr : 0.0f;
  if (!p.gamut_identity) s = mat3(p.gamut, s);
  s.r = clamp01(s.r); s.g = clamp01(s.g); s.b = clamp01(s.b);
  C3 e;
  e.r = srgb_oetf_dev(s.r); e.g = srgb_oetf_dev(s.g); e.b = srgb_oetf_dev(s.b);
  return e;
}
__device__ __forceinline__ C3 p3_rgb_to_yuv(C3 e) {  // gainmapmath.cpp:166-169, then +0.5 chroma
  const float y = 0.299f * e.r + 0.587f * e.g + 0.114f * e.b;
  C3 o;
  o.r = y;
  o.g = (e.b - y) / 1.772f + 0.5f;
  o.b = (e.r - y) / 1.402f + 0.5f;
  return o;
}

__global__ void __launch_bounds__(256) k_tonemap(const TonemapParams p) {
  const int tx = blockIdx.x * blockDim.x + threadIdx.x;
  const int ty = blockIdx.y * blockDim.y + threadIdx.y;
  if (p.dst_fmt == F_YUV420) {  // one thread = one 2x2 quad
    const int x = tx * 2, y = ty * 2;
    if (x >= p.hdr.w || y >= p.hdr.h) return;
    float su = 0.0f, sv = 0.0f;
    unsigned yy[4];
    for (int i = 0; i < 2; i++)
      for (int j = 0; j < 2; j++) {
        C3 yuv = p3_rgb_to_yuv(tonemap_px(p, x + j, y + i));
        yy[i * 2 + j] = scale_to_8bit(yuv.r);
        su += yuv.g;
        sv += yuv.b;
      }
    su /= 4.0f;
    sv /= 4.0f;
    uint8_t* r0 = p.dst[0] + (size_t)y * p.dst_stride[0] + x;
    uint8_t* r1 = r0 + p.dst_stride[0];
    *(uint16_t*)r0 = (uint16_t)(yy[0] | (yy[1] << 8));
    *(uint16_t*)r1 = (uint16_t)(yy[2] | (yy[3] << 8));
    p.dst[1][(size_t)ty * p.dst_stride[1] + tx] = (uint8_t)scale_to_8bit(su);
    p.dst[2][(size_t)ty * p.dst_stride[2] + tx] = (uint8_t)scale_to_8bit(sv);
  } else {
    const int x = tx, y = ty;
    if (x >= p.hdr.w || y >= p.hdr.h) return;
    C3 e = tonemap_px(p, x, y);
    if (p.dst_fmt == F_RGBA8888) {  // putRgba8888Pixel gainmapmath.cpp:538-552
      float v[3] = {e.r * 255.0f + 0.5f, e.g * 255.0f + 0.5f, e.b * 255.0f + 0.5f};
      unsigned px = 255u << 24;
      for (int c = 0; c < 3; c++) {
        float q = v[c] < 0.0f ? 0.0f : (v[c] > 255.0f ? 255.0f : v[c]);
        px |= (unsigned)__float2int_rz(q) << (8 * c);
      }
      ((unsigned*)p.dst[0])[(size_t)y * p.dst_stride[0] + x] = px;
    } else {  // YUV444: putYuv444Pixel :579-596
      C3 yuv = p3_rgb_to_yuv(e);
      float v[3] = {yuv.r * 255.0f + 0.5f, yuv.g * 255.0f + 0.5f, yuv.b * 255.0f + 0.5f};
      for (int c = 0; c < 3; c++) {
        float q = v[c] < 0.0f ? 0.0f : (v[c] > 255.0f ? 255.0f : v[c]);
        p.dst[c][(size_t)y * p.dst_stride[c] + x] = (uint8_t)__float2int_rz(q);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// convertYuv  gainmapmath.cpp:686-748 (in place)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned clip255(float v) {
  v = v < 0.0f ? 0.0f : (v > 255.0f ? 255.0f : v);
  return (unsigned)__float2int_rz(v);
}
__global__ void __launch_bounds__(256) k_yuv_convert(const YuvConvParams p) {
  const int tx = blockIdx.x * blockDim.x + threadIdx.x;
  const int ty = blockIdx.y * blockDim.y + threadIdx.y;
  if (p.fmt == F_YUV420) {
    if (tx >= p.w / 2 || ty >= p.h / 2) return;
    const uint8_t* y0 = p.p[0] + (size_t)(ty * 2) * p.stride[0] + tx * 2;
    const uint8_t* y1 = y0 + p.stride[0];
    const float u = (float)((int)p.p[1][(size_t)ty * p.stride[1] + tx] - 128) * (1 / 255.0f);
    const float v = (float)((int)p.p[2][(size_t)ty * p.stride[2] + tx] - 128) * (1 / 255.0f);
    const unsigned ys[4] = {y0[0], y0[1], y1[0], y1[1]};
    float ny[4], su = 0.f, sv = 0.f;
    for (int k = 0; k < 4; k++) {
      const float yy = (float)ys[k] * (1 / 255.0f);
      ny[k] = yy * p.m[0] + u * p.m[1] + v * p.m[2];
      const float cu = yy * p.m[3] + u * p.m[4] + v * p.m[5];
      const float cv = yy * p.m[6] + u * p.m[7] + v * p.m[8];
      su = k == 0 ? cu : su + cu;
      sv = k == 0 ? cv : sv + cv;
    }
    su /= 4.0f;
    sv /= 4.0f;
    uint8_t* d0 = p.d[0] + (size_t)(ty * 2) * p.dstride[0] + tx * 2;
    uint8_t* d1 = d0 + p.dstride[0];
    d0[0] = (uint8_t)clip255(ny[0] * 255.0f + 0.5f);
    d0[1] = (uint8_t)clip255(ny[1] * 255.0f + 0.5f);
    d1[0] = (uint8_t)clip255(ny[2] * 255.0f + 0.5f);
    d1[1] = (uint8_t)clip255(ny[3] * 255.0f + 0.5f);
    p.d[1][(size_t)ty * p.dstride[1] + tx] = (uint8_t)clip255(su * 255.0f + 128.0f + 0.5f);
    p.d[2][(size_t)ty * p.dstride[2] + tx] = (uint8_t)clip255(sv * 255.0f + 128.0f + 0.5f);
  } else {  // 4:4:4
    if (tx >= p.w || ty >= p.h) return;
    const float yy = (float)p.p[0][(size_t)ty * p.stride[0] + tx] * (1 / 255.0f);
    const float u = (float)((int)p.p[1][(size_t)ty * p.stride[1] + tx] - 128) * (1 / 255.0f);
    const float v = (float)((int)p.p[2][(size_t)ty * p.stride[2] + tx] - 128) * (1 / 255.0f);
    p.d[0][(size_t)ty * p.dstride[0] + tx] = (uint8_t)clip255((yy * p.m[0] + u * p.m[1] + v * p.m[2]) * 255.0f + 0.5f);
    p.d[1][(size_t)ty * p.dstride[1] + tx] = (uint8_t)clip255((yy * p.m[3] + u * p.m[4] + v * p.m[5]) * 255.0f + 128.0f + 0.5f);
    p.d[2][(size_t)ty * p.dstride[2] + tx] = (uint8_t)clip255((yy * p.m[6] + u * p.m[7] + v * p.m[8]) * 255.0f + 128.0f + 0.5f);
  }
}

// ------------------------------------------------------------------------------------------------
// JPEG decoder colour stage: jdcolor.c colour conversion, integer arithmetic, bit-exact (the forward block stage lives in
// fdct8.cu, the inverse DCT in idct.cu).
// ------------------------------------------------------------------------------------------------

// jdcolor.c ycc_rgb_convert with JCS_EXT_RGBA (alpha 0xFF).  ORG: a region with an origin other than 0, 0
template <bool ORG>
__global__ void __launch_bounds__(256) k_ycc_to_rgba(const YccToRgbaParams p) {
  const int rx = blockIdx.x * blockDim.x + threadIdx.x;
  const int ry = blockIdx.y * blockDim.y + threadIdx.y;
  if (rx >= p.w || ry >= p.h) return;
  const int x = ORG ? p.ox + rx : rx, y = ORG ? p.oy + ry : ry;   // absolute: every read below
  const size_t i = (size_t)y * p.src_stride + x;
  const int yy = __ldg(p.y + i);
  int xb, xr;
  if (p.hs == 1) {
    xb = (int)__ldg(p.cb + i) - 128;
    xr = (int)__ldg(p.cr + i) - 128;
  } else {
    // libjpeg-turbo jdsample.c: h2v1 / h2v2 "fancy" (triangle) upsampling, the library default; a
    // component whose downsampled width is <= 2 is replicated instead (jinit_upsampler).  Rows above
    // the first / below the last real row are that row itself (jdmainct.c context rows).
    const int cx = x >> 1;
    const uint8_t* pl[2] = {p.cb, p.cr};
    int o[2];
#pragma unroll
    for (int c = 0; c < 2; c++) {
      const uint8_t* base = pl[c];
      if (p.cw <= 2) {
        o[c] = __ldg(base + (size_t)(y / p.vs) * p.c_stride + cx);
      } else if (p.vs == 1) {
        const uint8_t* in = base + (size_t)y * p.c_stride;
        const int cur = __ldg(in + cx);
        if (x & 1) o[c] = cx == p.cw - 1 ? cur : (cur * 3 + (int)__ldg(in + cx + 1) + 2) >> 2;
        else o[c] = cx == 0 ? cur : (cur * 3 + (int)__ldg(in + cx - 1) + 1) >> 2;
      } else {
        const int r0 = y >> 1;
        const int r1 = (y & 1) ? min(r0 + 1, p.ch - 1) : max(r0 - 1, 0);
        const uint8_t* in0 = base + (size_t)r0 * p.c_stride;
        const uint8_t* in1 = base + (size_t)r1 * p.c_stride;
        const int cur = (int)__ldg(in0 + cx) * 3 + (int)__ldg(in1 + cx);
        if (x & 1) {
          if (cx == p.cw - 1) o[c] = (cur * 4 + 7) >> 4;
          else o[c] = (cur * 3 + (int)__ldg(in0 + cx + 1) * 3 + (int)__ldg(in1 + cx + 1) + 7) >> 4;
        } else {
          if (cx == 0) o[c] = (cur * 4 + 8) >> 4;
          else o[c] = (cur * 3 + (int)__ldg(in0 + cx - 1) * 3 + (int)__ldg(in1 + cx - 1) + 8) >> 4;
        }
      }
    }
    xb = o[0] - 128;
    xr = o[1] - 128;
  }
  const int r = yy + ((91881 * xr + 32768) >> 16);
  const int b = yy + ((116130 * xb + 32768) >> 16);
  const int g = yy + ((-22554 * xb + 32768 - 46802 * xr) >> 16);
  const unsigned px = (unsigned)min(max(r, 0), 255) | ((unsigned)min(max(g, 0), 255) << 8) |
                      ((unsigned)min(max(b, 0), 255) << 16) | 0xFF000000u;
  ((unsigned*)p.dst)[(size_t)ry * p.dst_stride + rx] = px;
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
static inline dim3 grid2(int wx, int hy, dim3 b) {
  return dim3((wx + b.x - 1) / b.x, (hy + b.y - 1) / b.y);
}

cudaError_t launch_gainmap_init_minmax(unsigned* minmax, cudaStream_t s) {
  k_gainmap_init_minmax<<<1, 32, 0, s>>>(minmax);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
cudaError_t launch_gainmap_pass1(const GainmapGenParams& p, cudaStream_t s) {
  dim3 b(32, 8);
  k_gainmap_pass1<<<grid2((p.map_w + kGmPx - 1) / kGmPx, p.map_h, b), b, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
cudaError_t launch_gainmap_onepass(const GainmapGenParams& p, cudaStream_t s) {
  dim3 b(32, 8);
  k_gainmap_onepass<<<grid2((p.map_w + kGmPx - 1) / kGmPx, p.map_h, b), b, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
cudaError_t launch_gainmap_finalize(const GainmapFinalizeParams& p, cudaStream_t s) {
  k_gainmap_finalize<<<1, 32, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
cudaError_t launch_gainmap_affine(const AffineParams& p, cudaStream_t s) {
  const int row_bytes = p.map_w * p.nch;
  dim3 b(256, 1);
  dim3 g((row_bytes / 4 + 1 + 255) / 256, p.map_h);
  k_gainmap_affine<<<g, b, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
cudaError_t launch_apply_gainmap(const ApplyParams& p, cudaStream_t s) {
  dim3 b(32, 8);
  if (p.ox | p.oy) k_apply_gainmap<true><<<grid2((p.sdr.w + 1) / 2, p.sdr.h, b), b, 0, s>>>(p);
  else k_apply_gainmap<false><<<grid2((p.sdr.w + 1) / 2, p.sdr.h, b), b, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
cudaError_t launch_tonemap(const TonemapParams& p, cudaStream_t s) {
  if (tonemap_fast_eligible(p)) return launch_tonemap_fast(p, s);
  dim3 b(32, 8);
  const int f = p.dst_fmt == F_YUV420 ? 2 : 1;
  k_tonemap<<<grid2((p.hdr.w + f - 1) / f, (p.hdr.h + f - 1) / f, b), b, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
// convert_raw_input_to_ycbcr for 8-bit RGB input (gainmapmath.cpp:1440-1467): getPixel (/255.0f), the
// gamut's rgbToYuv, *255 + 0.5 (+128 for chroma), clip, truncate
__global__ void __launch_bounds__(256) k_rgb_to_ycc(const RgbToYccParams p) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= p.w) return;
  const uint8_t* s = p.src + ((size_t)y * p.src_stride + x) * p.bpp;
  float r, g, b;
  if (p.bpp == 4) {
    const unsigned v = __ldg((const unsigned*)s);
    r = (float)(v & 0xff); g = (float)((v >> 8) & 0xff); b = (float)((v >> 16) & 0xff);
  } else {
    r = (float)s[0]; g = (float)s[1]; b = (float)s[2];
  }
  r = r / 255.0f; g = g / 255.0f; b = b / 255.0f;
  const float yg = p.k[0] * r + p.k[1] * g + p.k[2] * b;
  const float u = (b - yg) / p.k[3], v = (r - yg) / p.k[4];
  float yy = yg * 255.0f + 0.5f;
  yy = yy < 0.0f ? 0.0f : (yy > 255.0f ? 255.0f : yy);
  float uu = u * 255.0f + 0.5f + 128.0f, vv = v * 255.0f + 0.5f + 128.0f;
  uu = uu < 0.0f ? 0.0f : (uu > 255.0f ? 255.0f : uu);
  vv = vv < 0.0f ? 0.0f : (vv > 255.0f ? 255.0f : vv);
  const size_t o = (size_t)y * p.dst_stride + x;
  p.dst[0][o] = (uint8_t)__float2int_rz(yy);
  p.dst[1][o] = (uint8_t)__float2int_rz(uu);
  p.dst[2][o] = (uint8_t)__float2int_rz(vv);
}
// resize_image (editorhelper.cpp:100-146): the reference's "bicubic" is a cubic Bernstein blend of the
// four neighbours p0 (x0,y0), p1 (x0+1,y0), p2 (x0,y0+1), p3 (x0+1,y0+1) weighted by the *horizontal*
// fraction only, evaluated in double; pixels go through getPixel / putPixel of the map's format.
__global__ void __launch_bounds__(256) k_resize_map(const ResizeMapParams p) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= p.dst_w) return;
  const double scale_x = (double)p.src_w / p.dst_w, scale_y = (double)p.src_h / p.dst_h;
  const double ori_x = x * scale_x, ori_y = y * scale_y;
  const int p0x = min(max((int)floor(ori_x), 0), p.src_w - 1), p0y = min(max((int)floor(ori_y), 0), p.src_h - 1);
  const int p1x = min(max(p0x + 1, 0), p.src_w - 1), p2y = min(max(p0y + 1, 0), p.src_h - 1);
  const double fx = ori_x - p0x;
  const double w0 = (1 - fx) * (1 - fx) * (1 - fx), w1 = 3 * fx * (1 - fx) * (1 - fx), w2 = 3 * fx * fx * (1 - fx), w3 = fx * fx * fx;
  const int nch = p.bpp == 1 ? 1 : 3;
  unsigned outv[3] = {0, 0, 0};
  for (int c = 0; c < nch; c++) {
    auto px = [&](int xx, int yy) -> float {
      const unsigned b = __ldg(p.src + ((size_t)yy * p.src_stride + xx) * p.bpp + c);
      // getYuv400Pixel multiplies by (1 / 255.0f), getRgb888Pixel / getRgba8888Pixel divide by 255.0f
      return p.bpp == 1 ? (float)b * (1 / 255.0f) : (float)b / 255.0f;
    };
    const double a0 = px(p0x, p0y), a1 = px(p1x, p0y), a2 = px(p0x, p2y), a3 = px(p1x, p2y);
    float v = (float)(w0 * a0 + w1 * a1 + w2 * a2 + w3 * a3);
    v = v * 255.0f;
    v = v + 0.5f;
    v = v < 0.0f ? 0.0f : (v > 255.0f ? 255.0f : v);
    outv[c] = (unsigned)__float2int_rz(v);
  }
  uint8_t* d = p.dst + ((size_t)y * p.dst_stride + x) * p.bpp;
  if (p.bpp == 4) *reinterpret_cast<unsigned*>(d) = outv[0] | (outv[1] << 8) | (outv[2] << 16) | (255u << 24);
  else for (int c = 0; c < nch; c++) d[c] = (uint8_t)outv[c];
}
cudaError_t launch_resize_map(const ResizeMapParams& p, cudaStream_t s) {
  k_resize_map<<<dim3((p.dst_w + 255) / 256, p.dst_h), 256, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
cudaError_t launch_rgb_to_ycc(const RgbToYccParams& p, cudaStream_t s) {
  k_rgb_to_ycc<<<dim3((p.w + 255) / 256, p.h), 256, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
cudaError_t launch_yuv_convert(const YuvConvParams& p, cudaStream_t s) {
  if (yuv420_fast_eligible(p)) {
    COUNT_LAUNCH();
    return launch_yuv420_fast(p, s);
  }
  dim3 b(32, 8);
  const int f = p.fmt == F_YUV420 ? 2 : 1;
  k_yuv_convert<<<grid2(p.w / f, p.h / f, b), b, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}
cudaError_t launch_ycc_to_rgba(const YccToRgbaParams& p, cudaStream_t s) {
  dim3 b(32, 8);
  if (p.ox | p.oy) k_ycc_to_rgba<true><<<grid2(p.w, p.h, b), b, 0, s>>>(p);
  else k_ycc_to_rgba<false><<<grid2(p.w, p.h, b), b, 0, s>>>(p);
  COUNT_LAUNCH();
  return cudaGetLastError();
}

}  // namespace uhdr_b200
