// The inverse DCT of one 8x8 coefficient block, the bodies the IDCT kernels of idct.cu call:
//  - idct_dequant_block: libjpeg-turbo jidctint.c "islow" (LL&M, CONST_BITS 13, PASS1_BITS 2), dequantised with the
//    raw quantiser values, +128 and a saturating clamp (the semantics of the SIMD forms the library runs);
//  - idct_scaled_block<S>, S = 4 / 2 / 1: jidctred.c (jpeg_idct_4x4 / _2x2 / _1x1), described in idct.cu.
// Integer arithmetic, bit-exact.
#pragma once
#include <cstdint>

namespace uhdr_b200 {

#define C_BITS 13
#define P1_BITS 2
#define FX_0_298631336 2446
#define FX_0_390180644 3196
#define FX_0_541196100 4433
#define FX_0_765366865 6270
#define FX_0_899976223 7373
#define FX_1_175875602 9633
#define FX_1_501321110 12299
#define FX_1_847759065 15137
#define FX_1_961570560 16069
#define FX_2_053119869 16819
#define FX_2_562915447 20995
#define FX_3_072711026 25172
#define DESCALE(x, n) (((x) + (1 << ((n)-1))) >> (n))

__device__ __forceinline__ void idct8(int d0, int d1, int d2, int d3, int d4, int d5, int d6, int d7,
                                      int o[8], int shift) {
  int z2 = d2, z3 = d6;
  int z1 = (z2 + z3) * FX_0_541196100;
  int tmp2 = z1 + z3 * (-FX_1_847759065);
  int tmp3 = z1 + z2 * FX_0_765366865;
  int tmp0 = (d0 + d4) << C_BITS;
  int tmp1 = (d0 - d4) << C_BITS;
  int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = d7; tmp1 = d5; tmp2 = d3; tmp3 = d1;
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  int z4 = tmp1 + tmp3;
  int z5 = (z3 + z4) * FX_1_175875602;
  tmp0 *= FX_0_298631336;
  tmp1 *= FX_2_053119869;
  tmp2 *= FX_3_072711026;
  tmp3 *= FX_1_501321110;
  z1 *= -FX_0_899976223;
  z2 *= -FX_2_562915447;
  z3 *= -FX_1_961570560;
  z4 *= -FX_0_390180644;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  o[0] = DESCALE(tmp10 + tmp3, shift);
  o[7] = DESCALE(tmp10 - tmp3, shift);
  o[1] = DESCALE(tmp11 + tmp2, shift);
  o[6] = DESCALE(tmp11 - tmp2, shift);
  o[2] = DESCALE(tmp12 + tmp1, shift);
  o[5] = DESCALE(tmp12 - tmp1, shift);
  o[3] = DESCALE(tmp13 + tmp0, shift);
  o[4] = DESCALE(tmp13 - tmp0, shift);
}

// block (bx, by) of a plane, quantiser in shared memory
__device__ __forceinline__ void idct_dequant_block(const int16_t* coefs, const uint16_t* sq, int wblocks, int bx, int by, uint8_t* dst,
                                                   int dst_stride, int dst_w, int dst_h) {
  const int16_t* in = coefs + ((size_t)by * wblocks + bx) * 64;
  int v[64];
#pragma unroll
  for (int i = 0; i < 64; i += 8) {
    const uint4 q = __ldg((const uint4*)(in + i));
    const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const int c = (int)(int16_t)((w[k >> 1] >> ((k & 1) * 16)) & 0xffff);
      v[i + k] = c * (int)sq[i + k];
    }
  }
  int o[8];
#pragma unroll
  for (int c = 0; c < 8; c++) {  // pass 1: columns
    idct8(v[c], v[8 + c], v[16 + c], v[24 + c], v[32 + c], v[40 + c], v[48 + c], v[56 + c], o,
          C_BITS - P1_BITS);
#pragma unroll
    for (int r = 0; r < 8; r++) v[r * 8 + c] = o[r];
  }
#pragma unroll
  for (int r = 0; r < 8; r++) {  // pass 2: rows, +128, clamp (SIMD saturating pack semantics)
    idct8(v[r * 8], v[r * 8 + 1], v[r * 8 + 2], v[r * 8 + 3], v[r * 8 + 4], v[r * 8 + 5],
          v[r * 8 + 6], v[r * 8 + 7], o, C_BITS + P1_BITS + 3);
    const int y = by * 8 + r;
    if (y >= dst_h) continue;
    unsigned lo = 0, hi = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
      lo |= (unsigned)min(max(o[c] + 128, 0), 255) << (8 * c);
      hi |= (unsigned)min(max(o[4 + c] + 128, 0), 255) << (8 * c);
    }
    uint8_t* d = dst + (size_t)y * dst_stride + bx * 8;
    if (bx * 8 + 8 <= dst_w && ((((size_t)d) & 7) == 0)) {
      *(uint2*)d = make_uint2(lo, hi);
    } else {
      for (int c = 0; c < 8 && bx * 8 + c < dst_w; c++)
        d[c] = (uint8_t)(((c < 4 ? lo : hi) >> (8 * (c & 3))) & 0xff);
    }
  }
}

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

}  // namespace

// block `local` of a plane, quantiser q in shared memory
template <int S>
__device__ __forceinline__ void idct_scaled_block(const int16_t* coefs, const uint16_t* q, int local, int wblocks, uint8_t* dst, int stride,
                                                  int dst_w, int dst_h) {
  const int by = local / wblocks, bx = local - by * wblocks;
  const int16_t* blk = coefs + (size_t)local * 64;
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

}  // namespace uhdr_b200
