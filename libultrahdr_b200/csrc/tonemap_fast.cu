// toneMap fast path (jpegr.cpp:2147-2202 with globalTonemap :1951-1977) for the API-0 benchmark
// configuration: P010 HDR intent (HLG or PQ) -> YCbCr 4:2:0.  Arithmetic and operand order are
// those of k_tonemap (kernels.cu); what changes:
//   * persistent CTAs striding over 256x8-pixel tiles, the 4096-entry inverse-OETF (+OOTF) table
//     staged once per CTA in shared memory in "doubled" form (index out of the float mantissa)
//   * one thread = a 4x2 pixel tile: 8-byte luma loads, the two chroma samples and their products
//     computed once, 32-bit luma / 16-bit chroma stores
//   * the seven IEEE divisions per pixel without the range-check slow path; the three that share a
//     divisor (max_hdr) and the constant divisors (headroom^2, 1.772, 1.402) reuse one refined
//     reciprocal
// srgbOetf stays glibc's powf restated in fp64 (powf_glibc.cuh): it is what the remaining time is.
#include "kernels.cuh"
#include "packed_f32.cuh"
#include <atomic>

#include "powf_glibc.cuh"
#include "runtime.h"
#include "tables.h"

namespace uhdr_b200 {

namespace {

__device__ unsigned long long g_tm_exact_groups;            // 2x2 groups redone with the exact powf (this device)
std::atomic<unsigned long long> g_tm_groups{0};           // 2x2 groups processed by the fast kernel (process)

__device__ __forceinline__ float srgb_oetf_fast(float e) {  // gainmapmath.cpp:139-148
  if (e <= 0.0031308f) return 12.92f * e;
  return (1.0f + 0.055f) * powf_glibc(e, 1.0f / 2.4f) - 0.055f;
}
__device__ __forceinline__ unsigned scale8(float v) {  // ScaleTo8Bit :1979-1983 (std::round)
  const int i = __float2int_rz(roundf(v * 255.0f));
  return (unsigned)min(max(i, 0), 255);
}
__device__ __forceinline__ float fetch_hdr2(const float* t, float x) {  // x in [0, 1]
  const unsigned off = __float_as_uint(__fadd_rz(x * 32760.0f, 8388608.0f)) & 0x7ffc;
  return *reinterpret_cast<const float*>(reinterpret_cast<const char*>(t) + off);
}

// ---- srgbOetf, screened ------------------------------------------------------------------------------------------
// The three powf per pixel (glibc's, restated in fp64: powf_glibc.cuh) are what this kernel spends its time on, and
// only 8-bit codes leave it.  Every 2x2 group therefore first runs with pow(e, 1/2.4) = ex2.approx(lg2.approx(e) / 2.4),
// whose distance to the exact routine is bounded by kPowAbs for every float e of (0.0031308, 1] (all of them checked
// on the device, tests/test_gpu_stages.py::test_fast_pow_error_bound, with a factor 2 to spare).  The bound is carried
// through the float operations behind it (1.055 p - 0.055; the luma sum; (b - y) / 1.772 and (r - y) / 1.402; the mean
// of four; * 255), giving the thresholds below.  If one of the six codes of the group (4 luma, Cb, Cr) has its
// pre-rounding value within the threshold of a rounding boundary (k + 0.5), the group is redone with the exact powf;
// otherwise exact and approximate values round to the same codes.
constexpr float kPowAbs = 3.0e-7f;   // checked over all inputs by test_fast_pow_error_bound
constexpr float kTmE = 1.055f * kPowAbs + 1.3e-7f;                    // sRGB value: two float roundings on top
constexpr float kTmEy = kTmE + 2.0e-7f;                               // luma: convex combination + its roundings
constexpr float kTmThrY = 255.0f * kTmEy + 1.6e-5f;                   // in code units, with the rounding of * 255
constexpr float kTmThrU = 255.0f * ((kTmE + kTmEy) / 1.772f + 2.0e-7f + 1.3e-7f) + 1.6e-5f;
constexpr float kTmThrV = 255.0f * ((kTmE + kTmEy) / 1.402f + 2.0e-7f + 1.3e-7f) + 1.6e-5f;

__device__ __forceinline__ float pow_1_24_approx(float e) {   // e in (0.0031308, 1]
  float l, r;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(e));   // e and the result are normal: ftz changes nothing, saves the subnormal fix-up
  l *= 1.0f / 2.4f;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(l));
  return r;
}
template <bool EXACT>
__device__ __forceinline__ float srgb_oetf_sel(float e) {  // gainmapmath.cpp:139-148
  if (e <= 0.0031308f) return 12.92f * e;
  return (1.0f + 0.055f) * (EXACT ? powf_glibc(e, 1.0f / 2.4f) : pow_1_24_approx(e)) - 0.055f;
}
// distance of v * 255 from the nearest rounding boundary of scale8 (std::round: k + 0.5) below `thr`?
__device__ __forceinline__ bool near_half(float v, float thr) {
  const float t = v * 255.0f;
  return fabsf((t - floorf(t)) - 0.5f) < thr;
}

// OETF -> YUV -> codes for the 4 pixels of a chroma sample (order: row 0 left, right, row 1 left, right).
// Returns whether any code is within its threshold of a rounding boundary (meaningful when !EXACT).
template <bool EXACT>
__device__ __forceinline__ bool tm_group_codes(const float (&lin)[4][3], const Rcp r_cb, const Rcp r_cr, unsigned (&y8)[4], unsigned& u8, unsigned& v8) {
  float su = 0.0f, sv = 0.0f;
  bool near = false;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const float er = srgb_oetf_sel<EXACT>(lin[i][0]), eg = srgb_oetf_sel<EXACT>(lin[i][1]), eb = srgb_oetf_sel<EXACT>(lin[i][2]);
    // p3RgbToYuv (gainmapmath.cpp:166-169), chroma offset +0.5
    const float yy = 0.299f * er + 0.587f * eg + 0.114f * eb;
    const float uo = div_by(eb - yy, r_cb) + 0.5f, vo = div_by(er - yy, r_cr) + 0.5f;
    y8[i] = scale8(yy);
    if (!EXACT) near |= near_half(yy, kTmThrY);
    su += uo;
    sv += vo;
  }
  su *= 0.25f;  // / 4.0f
  sv *= 0.25f;
  u8 = scale8(su);
  v8 = scale8(sv);
  if (!EXACT) near |= near_half(su, kTmThrU) | near_half(sv, kTmThrV);
  return near;
}

__global__ void k_pow_fast_probe(unsigned first_bits, unsigned count, float* __restrict__ worst) {
  float w = 0.0f;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    const float e = __uint_as_float(first_bits + i);
    w = fmaxf(w, fabsf(pow_1_24_approx(e) - powf_glibc(e, 1.0f / 2.4f)));
  }
  for (int o = 16; o; o >>= 1) w = fmaxf(w, __shfl_xor_sync(0xffffffffu, w, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned*>(worst), __float_as_uint(w));
}

template <bool LIMITED, bool GAMUT>
__global__ void __launch_bounds__(256, 3) k_tonemap_fast(const TonemapParams p, const int tiles_x, const int ntiles, unsigned long long* __restrict__ exact_groups) {
  extern __shared__ float hdr2[];  // hdr2[j] = LUT[(j + 1) >> 1], 8192 entries
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
  const float* src = p.luts + (p.hdr_ct == CT_HLG ? kLutHlgInvOotf : kLutPqInv);
  for (int i = tid; i < 8192; i += nt) hdr2[i] = __ldg(src + min((i + 1) >> 1, 4095));
  __syncthreads();
  const Rcp r_hh = make_rcp(p.headroom * p.headroom), r_cb = make_rcp(1.772f), r_cr = make_rcp(1.402f);
  const uint16_t* HY = (const uint16_t*)p.hdr.p[0];
  const uint16_t* HUV = (const uint16_t*)p.hdr.p[1];
  unsigned n_exact = 0;
#pragma unroll 1
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int ty = t / tiles_x, tx = t - ty * tiles_x;
    const int x = (tx * 64 + threadIdx.x) * 4, y = (ty * 4 + threadIdx.y) * 2;
    if (x >= p.hdr.w || y >= p.hdr.h) continue;
    const uint2 hyw[2] = {__ldg((const uint2*)(HY + (size_t)y * p.hdr.stride[0] + x)),
                          __ldg((const uint2*)(HY + (size_t)(y + 1) * p.hdr.stride[0] + x))};
    const uint2 huv = __ldg((const uint2*)(HUV + (size_t)(y >> 1) * p.hdr.stride[1] + x));
    unsigned oy[2] = {0, 0}, ou = 0, ov = 0;
#pragma unroll
    for (int k = 0; k < 2; k++) {  // chroma sample k covers pixels 2k, 2k+1 of both rows
      const unsigned uvw = k ? huv.y : huv.x;
      const int u10 = (int)((uvw & 0xffff) >> 6), v10 = (int)(uvw >> 22);
      float hu, hv;
      if (LIMITED) {
        hu = (float)(u10 - 64) * (1 / 896.0f) - 0.5f;
        hv = (float)(v10 - 64) * (1 / 896.0f) - 0.5f;
      } else {
        hu = (float)u10 / 1023.0f - 0.5f;
        hv = (float)v10 / 1023.0f - 0.5f;
      }
      const float crv = p.y2r[0] * hv, cbu = p.y2r[1] * hu, gcbu = p.y2r[2] * hu, gcrv = p.y2r[3] * hv;
      float lin[4][3];   // tone-mapped linear sRGB of the 4 pixels under this chroma sample
#pragma unroll
      for (int r = 0; r < 2; r++) {
        const unsigned hw = k ? hyw[r].y : hyw[r].x;
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int y10 = (int)(((hw >> (16 * e)) & 0xffff) >> 6);
          const float yf = LIMITED ? (float)(y10 - 64) * (1 / 876.0f) : (float)y10 / 1023.0f;
          // yuv -> rgb (clamped), inverse OETF (+ OOTF) through the table
          const float lr = fetch_hdr2(hdr2, __saturatef(yf + crv));
          const float lg = fetch_hdr2(hdr2, __saturatef(yf - gcbu - gcrv));
          const float lb = fetch_hdr2(hdr2, __saturatef(yf + cbu));
          // globalTonemap (always "normalized" for HLG / PQ)
          const float hr = lr * p.headroom, hg = lg * p.headroom, hb = lb * p.headroom;
          float max_hdr = hr;
          if (hg > max_hdr) max_hdr = hg;
          if (hb > max_hdr) max_hdr = hb;
          float o = 1.0f + div_by(max_hdr, r_hh);
          o = div_pos(o, 1.0f + max_hdr);
          const float max_sdr = o * max_hdr;
          const Rcp r_mx = make_rcp(max_hdr);
          float sr = hr > 0.0f ? div_by(hr * max_sdr, r_mx) : 0.0f;
          float sg = hg > 0.0f ? div_by(hg * max_sdr, r_mx) : 0.0f;
          float sb = hb > 0.0f ? div_by(hb * max_sdr, r_mx) : 0.0f;
          if (GAMUT) {
            const float a = p.gamut[0] * sr + p.gamut[1] * sg + p.gamut[2] * sb;
            const float b = p.gamut[3] * sr + p.gamut[4] * sg + p.gamut[5] * sb;
            const float c = p.gamut[6] * sr + p.gamut[7] * sg + p.gamut[8] * sb;
            sr = a; sg = b; sb = c;
          }
          lin[2 * r + e][0] = sr < 0.0f ? 0.0f : (sr > 1.0f ? 1.0f : sr);
          lin[2 * r + e][1] = sg < 0.0f ? 0.0f : (sg > 1.0f ? 1.0f : sg);
          lin[2 * r + e][2] = sb < 0.0f ? 0.0f : (sb > 1.0f ? 1.0f : sb);
        }
      }
      unsigned y8[4], u8, v8;
      if (tm_group_codes<false>(lin, r_cb, r_cr, y8, u8, v8)) {   // a code too close to a rounding boundary: exact powf
        tm_group_codes<true>(lin, r_cb, r_cr, y8, u8, v8);
        n_exact++;
      }
      oy[0] |= (y8[0] << (8 * (2 * k))) | (y8[1] << (8 * (2 * k + 1)));
      oy[1] |= (y8[2] << (8 * (2 * k))) | (y8[3] << (8 * (2 * k + 1)));
      ou |= u8 << (8 * k);
      ov |= v8 << (8 * k);
    }
    *(unsigned*)(p.dst[0] + (size_t)y * p.dst_stride[0] + x) = oy[0];
    *(unsigned*)(p.dst[0] + (size_t)(y + 1) * p.dst_stride[0] + x) = oy[1];
    *(uint16_t*)(p.dst[1] + (size_t)(y >> 1) * p.dst_stride[1] + (x >> 1)) = (uint16_t)ou;
    *(uint16_t*)(p.dst[2] + (size_t)(y >> 1) * p.dst_stride[2] + (x >> 1)) = (uint16_t)ov;
  }
  if (n_exact) atomicAdd(exact_groups, (unsigned long long)n_exact);
}

template <bool LIMITED, bool GAMUT>
cudaError_t launch_tm(const TonemapParams& p, int tiles_x, int ntiles, cudaStream_t s) {
  static PerDevice<int> wave;
  const size_t smem = 8192 * sizeof(float);
  auto fn = k_tonemap_fast<LIMITED, GAMUT>;
  const int resident = wave_ctas(wave, (const void*)fn, 256, smem);
  if (!resident) return cudaErrorUnknown;
  const int ctas = resident < ntiles ? resident : ntiles;
  unsigned long long* cnt = nullptr;
  if (cudaGetSymbolAddress((void**)&cnt, g_tm_exact_groups) != cudaSuccess) return cudaErrorUnknown;
  g_tm_groups.fetch_add((unsigned long long)(p.hdr.w / 2) * (p.hdr.h / 2));
  fn<<<ctas, dim3(64, 4), smem, s>>>(p, tiles_x, ntiles, cnt);
  return cudaGetLastError();
}

}  // namespace

bool tonemap_fast_eligible(const TonemapParams& p) {
  if (p.hdr.fmt != F_P010 || p.dst_fmt != F_YUV420 || !p.normalized) return false;
  if (p.hdr_ct != CT_HLG && p.hdr_ct != CT_PQ) return false;
  if ((p.hdr.w & 3) || (p.hdr.h & 1)) return false;
  if ((p.hdr.stride[0] & 3) || (p.hdr.stride[1] & 3) || (p.dst_stride[0] & 3) || (p.dst_stride[1] & 1) || (p.dst_stride[2] & 1)) return false;
  if (((size_t)p.hdr.p[0] & 7) || ((size_t)p.hdr.p[1] & 7) || ((size_t)p.dst[0] & 3) || ((size_t)p.dst[1] & 1) || ((size_t)p.dst[2] & 1)) return false;
  return true;
}

cudaError_t launch_tonemap_fast(const TonemapParams& p, cudaStream_t s) {
  count_launches(1);
  const int tiles_x = (p.hdr.w / 4 + 63) / 64, ntiles = tiles_x * ((p.hdr.h + 7) / 8);
  if (p.hdr.full_range) return p.gamut_identity ? launch_tm<false, false>(p, tiles_x, ntiles, s) : launch_tm<false, true>(p, tiles_x, ntiles, s);
  return p.gamut_identity ? launch_tm<true, false>(p, tiles_x, ntiles, s) : launch_tm<true, true>(p, tiles_x, ntiles, s);
}

// [0] 2x2 groups the fast kernel processed since process start, [1] of those redone with the exact powf (current device)
void tonemap_screen_stats(unsigned long long out[2]) {
  out[0] = g_tm_groups.load();
  out[1] = 0;
  cudaMemcpyFromSymbol(&out[1], g_tm_exact_groups, sizeof(unsigned long long));
}
// worst[0] (device float, zeroed by the caller) = max |ex2(lg2(e) / 2.4) - powf_glibc(e, 1/2.4)| over `count` floats from first_bits
cudaError_t launch_pow_fast_probe(unsigned first_bits, unsigned count, float* d_worst, cudaStream_t s) {
  k_pow_fast_probe<<<132 * 8, 256, 0, s>>>(first_bits, count, d_worst);
  return cudaGetLastError();
}

}  // namespace uhdr_b200
