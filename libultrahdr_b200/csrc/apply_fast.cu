// applyGainMap fast path (jpegr.cpp:1714-1811) for the configurations that matter at scale:
// YUV 4:2:0 base image (what JpegDecoderHelper hands over), integer map scale, gamma 1.
// Same arithmetic as k_apply_gainmap (kernels.cu) -- operand order, rounding and tables are
// identical -- but specialised at compile time and restructured for instruction issue, which is
// what bounds this kernel (13.5 B/px of traffic against ~400 instructions/px in the generic one):
//   * one thread = a 4x2 pixel tile: the two chroma samples and their products are computed once,
//     loads are 4/2/2/16 bytes wide, every store instruction writes 16 B per lane (512 B per warp)
//   * all tables in shared memory: sRGB-inverse LUT (4 KB) and, at scale 1, a 3x256 table that
//     maps a gain-map byte straight to its gain factor (mapUintToFloat -> IDW {1,0,0,0} ->
//     GainLUT index -> table value composed on the host with the reference's expressions);
//     other integer scales keep the 3x1024 gain LUT + u8/255 + IDW weights in shared memory
//   * floatToHalf: values are clamped to [0, 10000/203] first; there the reference's bit routine
//     equals one packed hardware conversion per two channels (see pack_half4)
//   * LUT indices come out of the float mantissa (add 2^23 toward zero) instead of the conversion unit
// k_apply_lin1 (scale 1 -> linear half float, the 8K decode configuration) adds: a persistent grid
// with atomic tile tickets, register prefetch of the next tile, fp32 pixel pairs (packed_f32.cuh),
// clamping on the packed half bit patterns and two 128-bit stores per row; k_apply_fast covers the other
// integer scales and the PQ / HLG outputs.
#include <cuda_fp16.h>

#include "kernels.cuh"
#include "packed_f32.cuh"
#include "powf_glibc.cuh"
#include "runtime.h"
#include "tables.h"

namespace uhdr_b200 {

namespace {

constexpr int kRowsPerThread = 8;   // 4 tile rows of 2
constexpr int kBlockX = 64, kBlockY = 4;

// reference floatToHalf (gainmapmath.h:160-173) adds half a half-ulp (0x1000) to the float bits and
// truncates: round-half-up, also in its denormal branch.  For the non-negative values that reach it
// here (clamped to [0, 10000/203]) that equals the hardware's round-to-nearest-even conversion of
// the float with its last mantissa bit forced to 1 -- the forced bit only ever moves an exact tie
// upwards.  Checked exhaustively over all 1.1e9 floats of that interval (DESIGN.md section 4).
__device__ __forceinline__ void pack_half4(float r, float g, float b, unsigned& lo, unsigned& hi) {
  const __half2 rg = __floats2half2_rn(__uint_as_float(__float_as_uint(r) | 1u), __uint_as_float(__float_as_uint(g) | 1u));
  const __half2 ba = __floats2half2_rn(__uint_as_float(__float_as_uint(b) | 1u), 1.0f);
  lo = *reinterpret_cast<const unsigned*>(&rg);
  hi = *reinterpret_cast<const unsigned*>(&ba);
}

// `mask` if x is a NaN, else 0.  A NaN channel occurs with valid metadata: a max_content_boost of FLT_MAX
// puts +inf into the gain table, and then 0 * inf (black base pixel, offset 0) or inf - inf (a gamut row)
// is NaN.  The reference's clamps are comparisons, which keep the NaN, x86 makes it the default NaN
// 0xFFC00000, and floatToHalf of that is 0xFFFF: ORing the mask into a clamped half writes the same.
__device__ __forceinline__ unsigned nan_bits(float x, unsigned mask) { return x != x ? mask : 0u; }

// kMaxH = reference floatToHalf(10000/203) = 0x5228; the alpha half 0x3C00 passes through both bounds.
// The conversion turns NaN and +-inf alike into a NaN half (bits | 1), so NaN is told apart on the floats;
// NANS = false where the host has ruled out inf and NaN (ApplyParams::nan_possible), which saves the selects.
template <bool NANS>
__device__ __forceinline__ void pack_half4_clamped(float r, float g, float b, unsigned& lo, unsigned& hi) {
  pack_half4(r, g, b, lo, hi);
  lo = __vmins2(__vmaxs2(lo, 0u), 0x52285228u);
  hi = __vmins2(__vmaxs2(hi, 0u), 0x52285228u);
  if (NANS) {
    lo |= nan_bits(r, 0xFFFFu) | nan_bits(g, 0xFFFF0000u);
    hi |= nan_bits(b, 0xFFFFu);
  }
}

// Shared-memory tables, byte-offset addressed.
//   srgb2[j] = srgbInvOetfLUT[(j + 1) >> 1], j = floor(2 * x * 1023): the reference index
//   int32(double(x*1023) + 0.5) equals (floor(2v) + 1) >> 1, and floor(4a) & ~3 == 4 * floor(a),
//   so the byte offset of the entry is  int(x * 8184.0f) & ~3  (x*8184 == 8*(x*1023) exactly).
struct FastSmem {
  float srgb2[2048];
  float gain[3 * 1024];  // scale 1: first 3*256 entries hold the byte -> factor tables
  float u8f[256];
};
__device__ __forceinline__ float srgb_fetch(const FastSmem& sm, float x) {  // x in [0, 1]
  // trunc(x * 8184) read out of the mantissa after adding 2^23 toward zero (no conversion unit)
  const int off = __float_as_int(__fadd_rz(x * 8184.0f, 8388608.0f)) & 0x1ffc;
  return *reinterpret_cast<const float*>(reinterpret_cast<const char*>(sm.srgb2) + off);
}
__device__ __forceinline__ int idx1023(float x) {  // x >= 0: int32(double(x*1023) + 0.5)
  return (__float2int_rz(x * 2046.0f) + 1) >> 1;
}

// ORG: a region whose origin (p.ox, p.oy) is not 0, 0 (x, y below are relative to it); false compiles to the
// whole-image kernel
template <int BPP, bool SCALE1, int GAMUT /*0 none 1 sdr side 2 hdr side*/, int OUT /*0 F16 1 PQ 2 HLG*/, bool ORG>
__global__ void __launch_bounds__(kBlockX* kBlockY) k_apply_fast(const ApplyParams p, const float* __restrict__ gain_u8) {
  extern __shared__ float smem_raw[];
  FastSmem& sm = *reinterpret_cast<FastSmem*>(smem_raw);
  float* idw = smem_raw + sizeof(FastSmem) / sizeof(float);
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
  for (int i = tid; i < 2048; i += nt) sm.srgb2[i] = __ldg(p.luts + kLutSrgbInv + ((i + 1) >> 1 > 1023 ? 1023 : (i + 1) >> 1));
  if (SCALE1) {
    for (int i = tid; i < 768; i += nt) sm.gain[i] = __ldg(gain_u8 + i);
  } else {
    for (int i = tid; i < 3072; i += nt) sm.gain[i] = __ldg(p.gain_lut + i);
    for (int i = tid; i < 256; i += nt) sm.u8f[i] = __ldg(p.luts + kLutU8Div255 + i);
    const int n = 16 * p.scale_int * p.scale_int;
    for (int i = tid; i < n; i += nt) idw[i] = __ldg(p.idw + i);
  }
  __syncthreads();
  const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (x >= p.sdr.w) return;
  const int ax = ORG ? p.ox + x : x;   // absolute column of the reads (ox % 4 == 0, oy % 2 == 0)
  const uint8_t* __restrict__ Y = (const uint8_t*)p.sdr.p[0];
  const int ybase = blockIdx.y * (kBlockY * kRowsPerThread) + threadIdx.y * 2;
#pragma unroll 1
  for (int it = 0; it < kRowsPerThread / 2; it++) {
  const int y = ybase + it * (kBlockY * 2);
  if (y >= p.sdr.h) break;
  const int ay = ORG ? p.oy + y : y;
  const unsigned y0 = __ldg((const unsigned*)(Y + (size_t)ay * p.sdr.stride[0] + ax));
  const unsigned y1 = __ldg((const unsigned*)(Y + (size_t)(ay + 1) * p.sdr.stride[0] + ax));
  const size_t coff = (size_t)(ay >> 1) * p.sdr.stride[1] + (ax >> 1);
  const unsigned uu = __ldg((const uint16_t*)((const uint8_t*)p.sdr.p[1] + coff));
  const unsigned vv = __ldg((const uint16_t*)((const uint8_t*)p.sdr.p[2] + (size_t)(ay >> 1) * p.sdr.stride[2] + (ax >> 1)));
  // chroma terms of p3YuvToRgb, shared by the 2x2 pixels under each chroma sample
  float crv[2], gcbu[2], gcrv[2], cbu[2];
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const float u = (float)((int)((uu >> (8 * k)) & 0xff) - 128) * (1 / 255.0f);
    const float v = (float)((int)((vv >> (8 * k)) & 0xff) - 128) * (1 / 255.0f);
    crv[k] = p.y2r[0] * v;
    cbu[k] = p.y2r[1] * u;
    gcbu[k] = p.y2r[2] * u;
    gcrv[k] = p.y2r[3] * v;
  }
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const unsigned yw = r ? y1 : y0;
    const int yy = y + r, ayy = ay + r;
    unsigned out[8];
    // gain-map taps for the 4 pixels of this row
    uint4 m4 = make_uint4(0, 0, 0, 0);
    unsigned m3[3] = {0, 0, 0};
    if (SCALE1) {
      const uint8_t* mrow = p.map + ((size_t)ayy * p.map_stride + ax) * BPP;
      if (BPP == 4) m4 = __ldg((const uint4*)mrow);
      else if (BPP == 3) { m3[0] = __ldg((const unsigned*)mrow); m3[1] = __ldg((const unsigned*)mrow + 1); m3[2] = __ldg((const unsigned*)mrow + 2); }
      else m3[0] = __ldg((const unsigned*)mrow);
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int k = i >> 1;
      const float yf = (float)((yw >> (8 * i)) & 0xff) * (1 / 255.0f);
      // p3YuvToRgb with clampPixelFloat (saturate == clamp for the finite values that occur)
      const float rg = __saturatef(yf + crv[k]);
      const float gg = __saturatef(yf - gcbu[k] - gcrv[k]);
      const float bg = __saturatef(yf + cbu[k]);
      float lr = srgb_fetch(sm, rg), lg = srgb_fetch(sm, gg), lb = srgb_fetch(sm, bg);
      if (GAMUT == 1) {
        const float a = p.gamut[0] * lr + p.gamut[1] * lg + p.gamut[2] * lb;
        const float b = p.gamut[3] * lr + p.gamut[4] * lg + p.gamut[5] * lb;
        const float c = p.gamut[6] * lr + p.gamut[7] * lg + p.gamut[8] * lb;
        lr = a; lg = b; lb = c;
      }
      float fr, fg, fb;
      if (SCALE1) {
        // byte c of the pixel, pre-scaled to a byte offset into its 256-float table
        unsigned o0, o1, o2;
        const char* gt = reinterpret_cast<const char*>(sm.gain);
        if (BPP == 4) {
          const unsigned w = i == 0 ? m4.x : i == 1 ? m4.y : i == 2 ? m4.z : m4.w;
          o0 = (w << 2) & 0x3FCu; o1 = (w >> 6) & 0x3FCu; o2 = (w >> 14) & 0x3FCu;
        } else if (BPP == 3) {
          const unsigned long long lo = m3[0] | ((unsigned long long)m3[1] << 32);
          const unsigned hi = m3[2];
          auto byte_at = [&](int n) -> unsigned { return n < 8 ? (unsigned)((lo >> (8 * n)) & 0xff) : ((hi >> (8 * (n - 8))) & 0xff); };
          o0 = byte_at(3 * i) << 2; o1 = byte_at(3 * i + 1) << 2; o2 = byte_at(3 * i + 2) << 2;
        } else {
          o0 = o1 = o2 = ((m3[0] >> (8 * i)) & 0xff) << 2;
        }
        fr = *reinterpret_cast<const float*>(gt + o0);
        fg = BPP == 1 ? fr : *reinterpret_cast<const float*>(gt + 1024 + o1);
        fb = BPP == 1 ? fr : *reinterpret_cast<const float*>(gt + 2048 + o2);
      } else {
        const int s = p.scale_int;
        const int px = ax + i;
        int xl = px / s, yl = ayy / s;
        const int xu = min(xl + 1, p.map_w - 1), yu = min(yl + 1, p.map_h - 1);
        xl = min(xl, p.map_w - 1);
        yl = min(yl, p.map_h - 1);
        int variant = 0;
        if (xl == xu && yl == yu) variant = 3;
        else if (xl == xu) variant = 1;
        else if (yl == yu) variant = 2;
        const float* w = idw + (variant * s * s + (ayy % s) * s + (px % s)) * 4;
        const float w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3];
        const uint8_t* m = p.map;
        const size_t i1 = ((size_t)yl * p.map_stride + xl) * BPP, i2 = ((size_t)yu * p.map_stride + xl) * BPP;
        const size_t i3 = ((size_t)yl * p.map_stride + xu) * BPP, i4 = ((size_t)yu * p.map_stride + xu) * BPP;
        float g[3];
#pragma unroll
        for (int c = 0; c < (BPP == 1 ? 1 : 3); c++) {
          const float e1 = sm.u8f[__ldg(m + i1 + c)], e2 = sm.u8f[__ldg(m + i2 + c)];
          const float e3 = sm.u8f[__ldg(m + i3 + c)], e4 = sm.u8f[__ldg(m + i4 + c)];
          g[c] = e1 * w0 + e2 * w1 + e3 * w2 + e4 * w3;
        }
        // GainLUT::getGainFactor, gamma 1; gains are >= 0; the weighted sum of taps <= 1 may
        // exceed 1 by an ulp, hence the clamp of the index
        fr = sm.gain[min(idx1023(g[0]), 1023)];
        fg = BPP == 1 ? fr : sm.gain[1024 + min(idx1023(g[1]), 1023)];
        fb = BPP == 1 ? fr : sm.gain[2048 + min(idx1023(g[2]), 1023)];
      }
      const int o1 = BPP == 1 ? 0 : 1, o2 = BPP == 1 ? 0 : 2;
      float hr = ((lr + p.off_sdr[0]) * fr) - p.off_hdr[0];
      float hg = ((lg + p.off_sdr[o1]) * fg) - p.off_hdr[o1];
      float hb = ((lb + p.off_sdr[o2]) * fb) - p.off_hdr[o2];
      if (OUT == 0) {
        if (GAMUT == 2) {
          const float a = p.gamut[0] * hr + p.gamut[1] * hg + p.gamut[2] * hb;
          const float b = p.gamut[3] * hr + p.gamut[4] * hg + p.gamut[5] * hb;
          const float c = p.gamut[6] * hr + p.gamut[7] * hg + p.gamut[8] * hb;
          hr = a; hg = b; hb = c;
        }
        // clampPixelFloatLinear; the min/max form equals it for numbers (no negative zero reaches this
        // point: sums of a positive-leading gamut row, x - x == +0), but drops a NaN, which the reference
        // keeps: a NaN channel is written as the reference's 0xFFFF (nan_bits)
        const unsigned nan_lo = nan_bits(hr, 0xFFFFu) | nan_bits(hg, 0xFFFF0000u), nan_hi = nan_bits(hb, 0xFFFFu);
        const float kMax = 10000.0f / 203.0f;
        hr = fminf(fmaxf(hr, 0.0f), kMax);
        hg = fminf(fmaxf(hg, 0.0f), kMax);
        hb = fminf(fmaxf(hb, 0.0f), kMax);
        pack_half4(hr, hg, hb, out[2 * i], out[2 * i + 1]);
        out[2 * i] |= nan_lo;
        out[2 * i + 1] |= nan_hi;
      } else {
        hr = hr * 203.0f / p.out_nits;
        hg = hg * 203.0f / p.out_nits;
        hb = hb * 203.0f / p.out_nits;
        if (GAMUT == 2) {
          const float a = p.gamut[0] * hr + p.gamut[1] * hg + p.gamut[2] * hb;
          const float b = p.gamut[3] * hr + p.gamut[4] * hg + p.gamut[5] * hb;
          const float c = p.gamut[6] * hr + p.gamut[7] * hg + p.gamut[8] * hb;
          hr = a; hg = b; hb = c;
        }
        hr = hr < 0.0f ? 0.0f : (hr > 1.0f ? 1.0f : hr);
        hg = hg < 0.0f ? 0.0f : (hg > 1.0f ? 1.0f : hg);
        hb = hb < 0.0f ? 0.0f : (hb > 1.0f ? 1.0f : hb);
        const float* t = p.luts + (OUT == 2 ? kLutHlgOetf : kLutPqOetf);
        if (OUT == 2) {
          const float ex = 1.0f / 1.2f;
          hr = powf_glibc(hr, ex);
          hg = powf_glibc(hg, ex);
          hb = powf_glibc(hb, ex);
        }
        float e[3] = {hr, hg, hb};
        unsigned px = 0x3u << 30;
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float v = e[c] * 65535.0f;
          int j = 0;
          if (v > 0.0f) {
            j = __float2int_rz(v);
            j += ((v - (float)j) >= 0.5f) ? 1 : 0;
            j = min(j, 65535);
          }
          float q = __ldg(t + j) * 1023.0f + 0.5f;
          q = q < 0.0f ? 0.0f : (q > 1023.0f ? 1023.0f : q);
          px |= (unsigned)__float2int_rz(q) << (10 * c);
        }
        out[i] = px;
      }
    }
    if (OUT == 0) {
      uint4* d = (uint4*)((uint2*)p.dst + (size_t)yy * p.dst_stride + x);
      d[0] = make_uint4(out[0], out[1], out[2], out[3]);
      d[1] = make_uint4(out[4], out[5], out[6], out[7]);
    } else {
      *(uint4*)((unsigned*)p.dst + (size_t)yy * p.dst_stride + x) = make_uint4(out[0], out[1], out[2], out[3]);
    }
  }
  }
}

// ---- scale 1, linear half-float output: the 8K decode configuration ----------------------------
// Persistent grid (tables staged once per CTA, no wave tail); the two horizontally adjacent pixels
// that share a chroma sample go through the arithmetic as a pair (packed_f32.cuh), each lane
// rounding every step separately like the reference.  nz: the run-time -0 of the pair product.
struct Lin1Smem {
  float srgb2[2048];
  float gain[768];
};
__device__ __forceinline__ float lds_off(const float* base, unsigned byte_off) {
  return *reinterpret_cast<const float*>(reinterpret_cast<const char*>(base) + byte_off);
}

template <int BPP>
struct TileIn {   // what one thread reads for its 4x2 pixels
  unsigned yw[2], uu, vv;
  uint4 m4[2];
  unsigned m3[2][3];
  int x, y;
};

template <int BPP, int GAMUT, bool NANS, bool ORG>
__global__ void __launch_bounds__(kBlockX* kBlockY, 4) k_apply_lin1(const ApplyParams p, const float* __restrict__ gain_u8, const int tiles_x,
                                                                 const int ntiles, const unsigned long long nz,
                                                                 unsigned* __restrict__ sched) {
  __shared__ Lin1Smem sm;
  __shared__ int s_tile[4];
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
  for (int i = tid; i < 2048; i += nt) sm.srgb2[i] = __ldg(p.luts + kLutSrgbInv + ((i + 1) >> 1 > 1023 ? 1023 : (i + 1) >> 1));
  for (int i = tid; i < 768; i += nt) sm.gain[i] = __ldg(gain_u8 + i);
  // tiles are handed out through a counter (zeroed by the caller with the table upload): the CTAs
  // of the single resident wave then finish together instead of leaving SMs idle behind the
  // slowest static share.  The next ticket is fetched while the current tile is being processed.
  int tick = (int)blockIdx.x;   // static striding when no counter is given
  auto next_ticket = [&]() -> int {
    if (sched) return (int)atomicAdd(sched, 1u);
    const int t = tick;
    tick += (int)gridDim.x;
    return t;
  };
  if (tid == 0) {
    s_tile[0] = next_ticket();
    s_tile[1] = next_ticket();
  }
  __syncthreads();
  const uint8_t* __restrict__ Y = (const uint8_t*)p.sdr.p[0];
  const V2 k255 = bc(1 / 255.0f), k8184 = bc(8184.0f);
  const int o1 = BPP == 1 ? 0 : 1, o2 = BPP == 1 ? 0 : 2;
  const V2 osr = bc(p.off_sdr[0]), osg = bc(p.off_sdr[o1]), osb = bc(p.off_sdr[o2]);
  const V2 ohr = bc(p.off_hdr[0]), ohg = bc(p.off_hdr[o1]), ohb = bc(p.off_hdr[o2]);
  auto load_tile = [&](int t, TileIn<BPP>& in) -> bool {
    if (t >= ntiles) return false;
    const int ty = t / tiles_x, tx = t - ty * tiles_x;
    const int x = (tx * kBlockX + threadIdx.x) * 4;
    const int y = ty * (kBlockY * 2) + threadIdx.y * 2;
    if (x >= p.sdr.w || y >= p.sdr.h) return false;
    in.x = x;   // stores: relative to the region
    in.y = y;
    const int ax = ORG ? p.ox + x : x, ay = ORG ? p.oy + y : y;   // reads: absolute
    in.yw[0] = __ldg((const unsigned*)(Y + (size_t)ay * p.sdr.stride[0] + ax));
    in.yw[1] = __ldg((const unsigned*)(Y + (size_t)(ay + 1) * p.sdr.stride[0] + ax));
    in.uu = __ldg((const uint16_t*)((const uint8_t*)p.sdr.p[1] + (size_t)(ay >> 1) * p.sdr.stride[1] + (ax >> 1)));
    in.vv = __ldg((const uint16_t*)((const uint8_t*)p.sdr.p[2] + (size_t)(ay >> 1) * p.sdr.stride[2] + (ax >> 1)));
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const uint8_t* mrow = p.map + ((size_t)(ay + r) * p.map_stride + ax) * BPP;
      if (BPP == 4) in.m4[r] = __ldg((const uint4*)mrow);
      else if (BPP == 3) { in.m3[r][0] = __ldg((const unsigned*)mrow); in.m3[r][1] = __ldg((const unsigned*)mrow + 1); in.m3[r][2] = __ldg((const unsigned*)mrow + 2); }
      else in.m3[r][0] = __ldg((const unsigned*)mrow);
    }
    return true;
  };
  auto compute_tile = [&](const TileIn<BPP>& in) {
    const int x = in.x, y = in.y;
    const unsigned* yw = in.yw;
    const unsigned uu = in.uu, vv = in.vv;
    const uint4* m4 = in.m4;
    const unsigned (*m3)[3] = in.m3;
    // chroma terms of p3YuvToRgb, shared by the 2x2 pixels under each chroma sample
    float crv[2], gcbu[2], gcrv[2], cbu[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const float u = (float)((int)((uu >> (8 * k)) & 0xff) - 128) * (1 / 255.0f);
      const float v = (float)((int)((vv >> (8 * k)) & 0xff) - 128) * (1 / 255.0f);
      crv[k] = p.y2r[0] * v;
      cbu[k] = p.y2r[1] * u;
      gcbu[k] = p.y2r[2] * u;
      gcrv[k] = p.y2r[3] * v;
    }
#pragma unroll
    for (int r = 0; r < 2; r++) {
      unsigned out[8];
#pragma unroll
      for (int k = 0; k < 2; k++) {  // pixel pair (2k, 2k+1)
        const V2 yf = vmul(v2((float)((yw[r] >> (16 * k)) & 0xff), (float)((yw[r] >> (16 * k + 8)) & 0xff)), k255, nz);
        float y0, y1, t0, t1;
        un(yf, y0, y1);
        un(vsub(yf, bc(gcbu[k])), t0, t1);
        // p3YuvToRgb with clampPixelFloat (saturate == clamp for the finite values that occur)
        const V2 rg = v2(__saturatef(y0 + crv[k]), __saturatef(y1 + crv[k]));
        const V2 gg = v2(__saturatef(t0 - gcrv[k]), __saturatef(t1 - gcrv[k]));
        const V2 bg = v2(__saturatef(y0 + cbu[k]), __saturatef(y1 + cbu[k]));
        unsigned ir0, ir1, ig0, ig1, ib0, ib1;
        un(vtrunc_bits(vmul(rg, k8184, nz)), ir0, ir1);
        un(vtrunc_bits(vmul(gg, k8184, nz)), ig0, ig1);
        un(vtrunc_bits(vmul(bg, k8184, nz)), ib0, ib1);
        V2 lr = v2(lds_off(sm.srgb2, ir0 & 0x1ffc), lds_off(sm.srgb2, ir1 & 0x1ffc));
        V2 lg = v2(lds_off(sm.srgb2, ig0 & 0x1ffc), lds_off(sm.srgb2, ig1 & 0x1ffc));
        V2 lb = v2(lds_off(sm.srgb2, ib0 & 0x1ffc), lds_off(sm.srgb2, ib1 & 0x1ffc));
        if (GAMUT == 1) {
          const V2 a = vadd(vadd(vmul(bc(p.gamut[0]), lr, nz), vmul(bc(p.gamut[1]), lg, nz)), vmul(bc(p.gamut[2]), lb, nz));
          const V2 b = vadd(vadd(vmul(bc(p.gamut[3]), lr, nz), vmul(bc(p.gamut[4]), lg, nz)), vmul(bc(p.gamut[5]), lb, nz));
          const V2 c = vadd(vadd(vmul(bc(p.gamut[6]), lr, nz), vmul(bc(p.gamut[7]), lg, nz)), vmul(bc(p.gamut[8]), lb, nz));
          lr = a; lg = b; lb = c;
        }
        // gain factors: byte c of each pixel -> its 256-float table
        unsigned q[2][3];
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int i = 2 * k + e;
          if (BPP == 4) {
            const unsigned w = i == 0 ? m4[r].x : i == 1 ? m4[r].y : i == 2 ? m4[r].z : m4[r].w;
            q[e][0] = (w << 2) & 0x3FCu; q[e][1] = (w >> 6) & 0x3FCu; q[e][2] = (w >> 14) & 0x3FCu;
          } else if (BPP == 3) {
            const unsigned long long lo = m3[r][0] | ((unsigned long long)m3[r][1] << 32);
            const unsigned hi = m3[r][2];
            auto byte_at = [&](int n) -> unsigned { return n < 8 ? (unsigned)((lo >> (8 * n)) & 0xff) : ((hi >> (8 * (n - 8))) & 0xff); };
            q[e][0] = byte_at(3 * i) << 2; q[e][1] = byte_at(3 * i + 1) << 2; q[e][2] = byte_at(3 * i + 2) << 2;
          } else {
            q[e][0] = q[e][1] = q[e][2] = ((m3[r][0] >> (8 * i)) & 0xff) << 2;
          }
        }
        const V2 fr = v2(lds_off(sm.gain, q[0][0]), lds_off(sm.gain, q[1][0]));
        const V2 fg = BPP == 1 ? fr : v2(lds_off(sm.gain + 256, q[0][1]), lds_off(sm.gain + 256, q[1][1]));
        const V2 fb = BPP == 1 ? fr : v2(lds_off(sm.gain + 512, q[0][2]), lds_off(sm.gain + 512, q[1][2]));
        V2 hr = vsub(vmul(vadd(lr, osr), fr, nz), ohr);
        V2 hg = vsub(vmul(vadd(lg, osg), fg, nz), ohg);
        V2 hb = vsub(vmul(vadd(lb, osb), fb, nz), ohb);
        if (GAMUT == 2) {
          const V2 a = vadd(vadd(vmul(bc(p.gamut[0]), hr, nz), vmul(bc(p.gamut[1]), hg, nz)), vmul(bc(p.gamut[2]), hb, nz));
          const V2 b = vadd(vadd(vmul(bc(p.gamut[3]), hr, nz), vmul(bc(p.gamut[4]), hg, nz)), vmul(bc(p.gamut[5]), hb, nz));
          const V2 c = vadd(vadd(vmul(bc(p.gamut[6]), hr, nz), vmul(bc(p.gamut[7]), hg, nz)), vmul(bc(p.gamut[8]), hb, nz));
          hr = a; hg = b; hb = c;
        }
        // clampPixelFloatLinear then floatToHalf, in the other order: the conversion is monotonic, so
        // clamping the half bit patterns (as signed 16-bit integers: negative halves are negative,
        // non-negative ones order like their bits) to [0, half(10000/203)] gives the same result with
        // two packed integer min/max per pixel.  Negative inputs only ever clamp to 0, so forcing
        // their last mantissa bit as well is harmless.
        float r0, r1, g0, g1, b0, b1;
        un(hr, r0, r1); un(hg, g0, g1); un(hb, b0, b1);
        pack_half4_clamped<NANS>(r0, g0, b0, out[4 * k], out[4 * k + 1]);
        pack_half4_clamped<NANS>(r1, g1, b1, out[4 * k + 2], out[4 * k + 3]);
      }
      uint2* d = (uint2*)p.dst + (size_t)(y + r) * p.dst_stride + x;
      ((uint4*)d)[0] = make_uint4(out[0], out[1], out[2], out[3]);
      ((uint4*)d)[1] = make_uint4(out[4], out[5], out[6], out[7]);
    }
  };
  {
    // software pipeline: the loads of the next tile are in flight while this one is computed
    TileIn<BPP> cur;
    int t = s_tile[0];
    bool cv = load_tile(t, cur);
#pragma unroll 1
    for (int it = 0; t < ntiles; it++) {
      const int tn = s_tile[(it + 1) & 3];
      if (tid == 0) s_tile[(it + 2) & 3] = next_ticket();
      TileIn<BPP> nx;
      const bool nv = load_tile(tn, nx);
      if (cv) compute_tile(cur);
      cur = nx;
      cv = nv;
      t = tn;
      __syncthreads();
    }
  }
}

template <int BPP, bool NANS, bool ORG>
cudaError_t launch_lin1(const ApplyParams& p, const float* gain_u8, unsigned* sched, cudaStream_t s) {
  const int tiles_x = (p.sdr.w / 4 + kBlockX - 1) / kBlockX, tiles_y = (p.sdr.h + kBlockY * 2 - 1) / (kBlockY * 2);
  const int ntiles = tiles_x * tiles_y;
  dim3 block(kBlockX, kBlockY);
  const int g = p.gamut_identity ? 0 : (p.gamut_on_sdr ? 1 : 2);
  // persistent grid = exactly the CTAs that are co-resident (a partial second wave would double the time)
  static PerDevice<int> wave[3];
  const void* fn = g == 0 ? (const void*)k_apply_lin1<BPP, 0, NANS, ORG> : g == 1 ? (const void*)k_apply_lin1<BPP, 1, NANS, ORG>
                                                                            : (const void*)k_apply_lin1<BPP, 2, NANS, ORG>;
  int ctas = wave_ctas(wave[g], fn, kBlockX * kBlockY, 0);
  if (!ctas) return cudaErrorUnknown;
  if (ctas > ntiles) ctas = ntiles;
  if (g == 0) k_apply_lin1<BPP, 0, NANS, ORG><<<ctas, block, 0, s>>>(p, gain_u8, tiles_x, ntiles, kNegZero2, sched);
  else if (g == 1) k_apply_lin1<BPP, 1, NANS, ORG><<<ctas, block, 0, s>>>(p, gain_u8, tiles_x, ntiles, kNegZero2, sched);
  else k_apply_lin1<BPP, 2, NANS, ORG><<<ctas, block, 0, s>>>(p, gain_u8, tiles_x, ntiles, kNegZero2, sched);
  return cudaGetLastError();
}
template <int BPP, bool ORG>
cudaError_t launch_lin1(const ApplyParams& p, const float* gain_u8, unsigned* sched, cudaStream_t s) {
  return p.nan_possible ? launch_lin1<BPP, true, ORG>(p, gain_u8, sched, s) : launch_lin1<BPP, false, ORG>(p, gain_u8, sched, s);
}

template <int BPP, bool S1, int G, bool ORG>
cudaError_t launch_out(const ApplyParams& p, const float* gain_u8, dim3 grid, dim3 block, size_t smem, cudaStream_t s) {
  if (p.out_ct == CT_LINEAR) k_apply_fast<BPP, S1, G, 0, ORG><<<grid, block, smem, s>>>(p, gain_u8);
  else if (p.out_ct == CT_PQ) k_apply_fast<BPP, S1, G, 1, ORG><<<grid, block, smem, s>>>(p, gain_u8);
  else k_apply_fast<BPP, S1, G, 2, ORG><<<grid, block, smem, s>>>(p, gain_u8);
  return cudaGetLastError();
}
template <int BPP, bool S1, bool ORG>
cudaError_t launch_gamut(const ApplyParams& p, const float* gain_u8, dim3 grid, dim3 block, size_t smem, cudaStream_t s) {
  const int g = p.gamut_identity ? 0 : (p.gamut_on_sdr ? 1 : 2);
  if (g == 0) return launch_out<BPP, S1, 0, ORG>(p, gain_u8, grid, block, smem, s);
  if (g == 1) return launch_out<BPP, S1, 1, ORG>(p, gain_u8, grid, block, smem, s);
  return launch_out<BPP, S1, 2, ORG>(p, gain_u8, grid, block, smem, s);
}

template <bool ORG>
cudaError_t launch_fast(const ApplyParams& p, const float* gain_u8, cudaStream_t s) {
  dim3 block(kBlockX, kBlockY);
  dim3 grid((p.sdr.w / 4 + kBlockX - 1) / kBlockX, (p.sdr.h + kBlockY * kRowsPerThread - 1) / (kBlockY * kRowsPerThread));
  const bool s1 = p.scale_int == 1;
  if (s1 && p.out_ct == CT_LINEAR) {
    unsigned* sched = reinterpret_cast<unsigned*>(const_cast<float*>(gain_u8) + 768);  // zeroed with the upload
    if (p.map_bpp == 4) return launch_lin1<4, ORG>(p, gain_u8, sched, s);
    if (p.map_bpp == 3) return launch_lin1<3, ORG>(p, gain_u8, sched, s);
    return launch_lin1<1, ORG>(p, gain_u8, sched, s);
  }
  const size_t smem = sizeof(FastSmem) + (s1 ? 0 : sizeof(float) * 16 * p.scale_int * p.scale_int);
  if (p.map_bpp == 4) return s1 ? launch_gamut<4, true, ORG>(p, gain_u8, grid, block, smem, s) : launch_gamut<4, false, ORG>(p, gain_u8, grid, block, smem, s);
  if (p.map_bpp == 3) return s1 ? launch_gamut<3, true, ORG>(p, gain_u8, grid, block, smem, s) : launch_gamut<3, false, ORG>(p, gain_u8, grid, block, smem, s);
  return s1 ? launch_gamut<1, true, ORG>(p, gain_u8, grid, block, smem, s) : launch_gamut<1, false, ORG>(p, gain_u8, grid, block, smem, s);
}

}  // namespace

bool apply_fast_eligible(const ApplyParams& p) {
  if (p.sdr.fmt != F_YUV420 || !p.scale_int) return false;
  if (p.gamma_inv[0] != 1.0f || p.gamma_inv[1] != 1.0f || p.gamma_inv[2] != 1.0f) return false;
  if ((p.sdr.w & 3) || (p.sdr.h & 1)) return false;
  if ((p.ox & 3) || (p.oy & 1)) return false;   // a region keeps the 4x2 tiles on the chroma grid and the loads aligned
  if ((p.sdr.stride[0] & 3) || (p.sdr.stride[1] & 1) || (p.sdr.stride[2] & 1)) return false;
  if (((size_t)p.sdr.p[0] & 3) || ((size_t)p.sdr.p[1] & 1) || ((size_t)p.sdr.p[2] & 1)) return false;
  if (((size_t)p.dst & 15) || (p.dst_stride & 3)) return false;
  if (p.scale_int == 1) {
    if (p.map_w < p.ox + p.sdr.w || p.map_h < p.oy + p.sdr.h) return false;  // no edge clamping in the vector path
    const int row_bytes = p.map_stride * p.map_bpp;
    if ((row_bytes & 3) || ((size_t)p.map & 15) || (p.map_bpp == 4 && (row_bytes & 15))) return false;
  } else if (p.scale_int > 16) {
    return false;  // IDW tables beyond shared-memory budget
  }
  return true;
}

// gain_u8: device pointer to the 3x256 composed table (scale 1 only) followed by 4 zeroed words
// (tile counter of the persistent kernel)
cudaError_t launch_apply_fast(const ApplyParams& p, const float* gain_u8, cudaStream_t s) {
  count_launches(1);
  return (p.ox | p.oy) ? launch_fast<true>(p, gain_u8, s) : launch_fast<false>(p, gain_u8, s);
}

}  // namespace uhdr_b200
