// Reduced-size inverse DCT of the scaled decoder (libjpeg scale_num = 1, scale_denom = 2 / 4 / 8): dequantise an 8x8
// coefficient block and output 4x4, 2x2 or 1x1 samples, the arithmetic of libjpeg-turbo's jidctred.c
// (jpeg_idct_4x4 / _2x2 / _1x1).  Integer, bit-exact:
//  - 4x4: the even part from inputs 0, 2, 6 and the odd part from 1, 3, 5, 7 of each column, column 4 left out,
//    then the same on the four rows; 2x2: DC and the odd inputs only, columns 2, 4 and 6 left out.  Dequantised with
//    the islow multipliers (the raw quantiser values), CONST_BITS 13, PASS1_BITS 2, 32-bit intermediates as in
//    k_idct_dequant; +128 and a saturating clamp, the semantics of the SIMD forms the library runs.
//  - 1x1: (dc * q0 + 4) >> 3 through the C range-limit table (the library has no SIMD form of it): the value is read
//    modulo 1024 as a signed number, then +128 and clamped.
// One thread per block; one launch covers every plane of a JPEG whose DCT scaled size is S.
#include "kernels.cuh"

namespace uhdr_b200 {

namespace {

constexpr int kCb = 13, kPb = 2;

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

__device__ __forceinline__ void idct4(int d0, int d1, int d2, int d3, int d5, int d6, int d7, int shift, int o[4]) {
  const int t0 = d0 * (1 << (kCb + 1));
  const int t2 = d2 * 15137 + d6 * -6270;                           // FIX(1.847759065), -FIX(0.765366865)
  const int t10 = t0 + t2, t12 = t0 - t2;
  const int a = d7 * -1730 + d5 * 11893 + d3 * -17799 + d1 * 8697;  // -0.211164243 1.451774981 -2.172734803 1.061594337
  const int b = d7 * -4176 + d5 * -4926 + d3 * 7373 + d1 * 20995;   // -0.509795579 -0.601344887 0.899976223 2.562915447
  o[0] = descale(t10 + b, shift);
  o[3] = descale(t10 - b, shift);
  o[1] = descale(t12 + a, shift);
  o[2] = descale(t12 - a, shift);
}

__device__ __forceinline__ void idct2(int d0, int d1, int d3, int d5, int d7, int shift, int o[2]) {
  const int t10 = d0 * (1 << (kCb + 2));
  const int t0 = d7 * -5906 + d5 * 6967 + d3 * -10426 + d1 * 29692;  // -0.720959822 0.850430095 -1.272758580 3.624509785
  o[0] = descale(t10 + t0, shift);
  o[1] = descale(t10 - t0, shift);
}

__device__ __forceinline__ unsigned px(int v) { return (unsigned)min(max(v + 128, 0), 255); }

// dequantised row r of the block (8 coefficients, one 16-byte load)
__device__ __forceinline__ void load_row(const int16_t* blk, const uint16_t* q, int r, int v[8]) {
  const uint4 w4 = __ldg((const uint4*)(blk + r * 8));
  const unsigned w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
  for (int k = 0; k < 8; k++) v[k] = (int)(int16_t)((w[k >> 1] >> ((k & 1) * 16)) & 0xffff) * (int)q[r * 8 + k];
}

template <int S>
__global__ void __launch_bounds__(128) k_idct_scaled(const __grid_constant__ IdctScaledParams p) {
  __shared__ uint16_t sq[3][64];
  for (int i = threadIdx.x; i < p.nplanes * 64; i += blockDim.x) sq[i >> 6][i & 63] = p.plane[i >> 6].q[i & 63];
  __syncthreads();
  const int gb = blockIdx.x * blockDim.x + threadIdx.x;
  if (gb >= p.block_end[p.nplanes - 1]) return;
  const int c = gb < p.block_end[0] ? 0 : gb < p.block_end[1] ? 1 : 2;
  const IdctScaledParams::Plane& pl = p.plane[c];  // __grid_constant__: read in place, no local copy
  const int16_t* coefs = pl.coefs;
  uint8_t* dst = pl.dst;
  const int wblocks = pl.wblocks, stride = pl.dst_stride, dst_w = pl.dst_w, dst_h = pl.dst_h;
  const int local = gb - (c == 0 ? 0 : p.block_end[c - 1]);
  const int by = local / wblocks, bx = local - by * wblocks;
  const int16_t* blk = coefs + (size_t)local * 64;
  const uint16_t* q = sq[c];
  uint8_t* out = dst + (size_t)by * S * stride + bx * S;
  if (S == 1) {
    if (by >= dst_h || bx >= dst_w) return;
    int t = descale((int)__ldg(blk) * (int)q[0], 3) & 1023;
    if (t >= 512) t -= 1024;
    *out = (uint8_t)px(t);
    return;
  }
  int o[4];
  if (S == 4) {
    int v[8][8];
#pragma unroll
    for (int r = 0; r < 8; r++)
      if (r != 4) load_row(blk, q, r, v[r]);
#pragma unroll
    for (int col = 0; col < 8; col++) {  // pass 1: columns (column 4 does not contribute)
      if (col == 4) continue;
      idct4(v[0][col], v[1][col], v[2][col], v[3][col], v[5][col], v[6][col], v[7][col], kCb - kPb + 1, o);
#pragma unroll
      for (int r = 0; r < 4; r++) v[r][col] = o[r];
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {  // pass 2: rows
      idct4(v[r][0], v[r][1], v[r][2], v[r][3], v[r][5], v[r][6], v[r][7], kCb + kPb + 3 + 1, o);
      if (by * 4 + r >= dst_h) break;
      const unsigned word = px(o[0]) | px(o[1]) << 8 | px(o[2]) << 16 | px(o[3]) << 24;
      uint8_t* d = out + (size_t)r * stride;
      if (bx * 4 + 4 <= dst_w && ((size_t)d & 3) == 0) {
        *(unsigned*)d = word;
      } else {
        for (int k = 0; k < 4 && bx * 4 + k < dst_w; k++) d[k] = (uint8_t)(word >> (8 * k));
      }
    }
  } else {  // S == 2
    int v[5][8];  // rows 0, 1, 3, 5, 7
#pragma unroll
    for (int i = 0; i < 5; i++) load_row(blk, q, i == 0 ? 0 : 2 * i - 1, v[i]);
    int ws[2][8];
#pragma unroll
    for (int col = 0; col < 8; col++) {  // pass 1: columns 0, 1, 3, 5, 7
      if (col == 2 || col == 4 || col == 6) continue;
      idct2(v[0][col], v[1][col], v[2][col], v[3][col], v[4][col], kCb - kPb + 2, o);
      ws[0][col] = o[0];
      ws[1][col] = o[1];
    }
#pragma unroll
    for (int r = 0; r < 2; r++) {
      idct2(ws[r][0], ws[r][1], ws[r][3], ws[r][5], ws[r][7], kCb + kPb + 3 + 2, o);
      if (by * 2 + r >= dst_h) break;
      uint8_t* d = out + (size_t)r * stride;
      if (bx * 2 + 2 <= dst_w && ((size_t)d & 1) == 0) {
        *(unsigned short*)d = (unsigned short)(px(o[0]) | px(o[1]) << 8);
      } else {
        for (int k = 0; k < 2 && bx * 2 + k < dst_w; k++) d[k] = (uint8_t)px(o[k]);
      }
    }
  }
}

}  // namespace

cudaError_t launch_idct_scaled(const IdctScaledParams& p, int size, cudaStream_t s) {
  if (p.nplanes < 1 || p.nplanes > 3) return cudaErrorInvalidValue;
  const int blocks = p.block_end[p.nplanes - 1];
  if (blocks <= 0) return cudaSuccess;
  const dim3 g((blocks + 127) / 128), b(128);
  count_launches(1);
  switch (size) {
    case 4: k_idct_scaled<4><<<g, b, 0, s>>>(p); break;
    case 2: k_idct_scaled<2><<<g, b, 0, s>>>(p); break;
    case 1: k_idct_scaled<1><<<g, b, 0, s>>>(p); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace uhdr_b200
