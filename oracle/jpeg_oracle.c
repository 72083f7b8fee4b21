/*
 * jpeg_oracle.c -- TEST INFRASTRUCTURE ONLY.  See jpeg_oracle.h for what is restated and how it
 * is pinned.  Plain C99, integer arithmetic only.
 */
#include "jpeg_oracle.h"

#include <stdlib.h>
#include <string.h>

/* ---------------------------------------------------------------------------------------------
 * Tables: ITU-T T.81 Annex K (the defaults jpeg_set_defaults installs, jcparam.c)
 * ------------------------------------------------------------------------------------------ */
static const uint8_t k_std_lum_q[64] = {
    16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
    14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
    18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
static const uint8_t k_std_chr_q[64] = {
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
    99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
    99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};

/* zigzag index -> natural index */
static const uint8_t k_natural_order[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

static const uint8_t k_bits_dc_lum[17] = {0, 0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
static const uint8_t k_val_dc[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t k_bits_dc_chr[17] = {0, 0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
static const uint8_t k_bits_ac_lum[17] = {0, 0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
static const uint8_t k_val_ac_lum[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61,
    0x07, 0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52,
    0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25,
    0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
    0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
    0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
    0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3,
    0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8,
    0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
static const uint8_t k_bits_ac_chr[17] = {0, 0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
static const uint8_t k_val_ac_chr[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61,
    0x71, 0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33,
    0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18,
    0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63,
    0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
    0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
    0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
    0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7,
    0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

/* ---------------------------------------------------------------------------------------------
 * Quality -> tables  (jcparam.c: jpeg_quality_scaling + jpeg_add_quant_table, force_baseline)
 * ------------------------------------------------------------------------------------------ */
void jo_quant_tables(int quality, uint16_t lum[64], uint16_t chr[64]) {
  if (quality <= 0) quality = 1;
  if (quality > 100) quality = 100;
  int scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
  for (int i = 0; i < 64; i++) {
    long t = ((long)k_std_lum_q[i] * scale + 50L) / 100L;
    if (t <= 0) t = 1;
    if (t > 255) t = 255;
    lum[i] = (uint16_t)t;
    t = ((long)k_std_chr_q[i] * scale + 50L) / 100L;
    if (t <= 0) t = 1;
    if (t > 255) t = 255;
    chr[i] = (uint16_t)t;
  }
}

/* ---------------------------------------------------------------------------------------------
 * Colour conversion (jccolor.c / jdcolor.c), SCALEBITS = 16
 * ------------------------------------------------------------------------------------------ */
#define SCALEBITS 16
#define ONE_HALF ((int32_t)1 << (SCALEBITS - 1))
#define FIX(x) ((int32_t)((x) * (1L << SCALEBITS) + 0.5))
#define CBCR_OFFSET ((int32_t)128 << SCALEBITS)

void jo_rgb_to_ycc(int r, int g, int b, uint8_t* y, uint8_t* cb, uint8_t* cr) {
  int32_t yy = FIX(0.29900) * r + FIX(0.58700) * g + FIX(0.11400) * b + ONE_HALF;
  int32_t cbb = (-FIX(0.16874)) * r + (-FIX(0.33126)) * g + FIX(0.50000) * b + CBCR_OFFSET +
                ONE_HALF - 1;
  int32_t crr = FIX(0.50000) * r + CBCR_OFFSET + ONE_HALF - 1 + (-FIX(0.41869)) * g +
                (-FIX(0.08131)) * b;
  *y = (uint8_t)(yy >> SCALEBITS);
  *cb = (uint8_t)(cbb >> SCALEBITS);
  *cr = (uint8_t)(crr >> SCALEBITS);
}

static inline uint8_t clamp_u8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

void jo_ycc_to_rgb(int y, int cb, int cr, uint8_t* r, uint8_t* g, uint8_t* b) {
  int xb = cb - 128, xr = cr - 128;
  /* arithmetic right shifts of possibly negative values, as RIGHT_SHIFT does */
  int cr_r = (int)((FIX(1.40200) * xr + ONE_HALF) >> SCALEBITS);
  int cb_b = (int)((FIX(1.77200) * xb + ONE_HALF) >> SCALEBITS);
  int32_t cr_g = (-FIX(0.71414)) * xr;
  int32_t cb_g = (-FIX(0.34414)) * xb + ONE_HALF;
  *r = clamp_u8(y + cr_r);
  *g = clamp_u8(y + (int)((cb_g + cr_g) >> SCALEBITS));
  *b = clamp_u8(y + cb_b);
}

/* ---------------------------------------------------------------------------------------------
 * islow DCT (jfdctint.c / jidctint.c): Loeffler-Ligtenberg-Moschytz, CONST_BITS 13, PASS1_BITS 2
 * ------------------------------------------------------------------------------------------ */
#define CONST_BITS 13
#define PASS1_BITS 2
#define F_0_298631336 2446
#define F_0_390180644 3196
#define F_0_541196100 4433
#define F_0_765366865 6270
#define F_0_899976223 7373
#define F_1_175875602 9633
#define F_1_501321110 12299
#define F_1_847759065 15137
#define F_1_961570560 16069
#define F_2_053119869 16819
#define F_2_562915447 20995
#define F_3_072711026 25172
#define DESCALE(x, n) (((x) + ((int32_t)1 << ((n)-1))) >> (n))

static void fdct_1d(const int32_t d[8], int32_t o[8], int pass) {
  int32_t tmp0 = d[0] + d[7], tmp7 = d[0] - d[7];
  int32_t tmp1 = d[1] + d[6], tmp6 = d[1] - d[6];
  int32_t tmp2 = d[2] + d[5], tmp5 = d[2] - d[5];
  int32_t tmp3 = d[3] + d[4], tmp4 = d[3] - d[4];
  int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3;
  int32_t tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  const int sh = pass == 0 ? CONST_BITS - PASS1_BITS : CONST_BITS + PASS1_BITS;
  if (pass == 0) {
    o[0] = (tmp10 + tmp11) * (1 << PASS1_BITS);
    o[4] = (tmp10 - tmp11) * (1 << PASS1_BITS);
  } else {
    o[0] = DESCALE(tmp10 + tmp11, PASS1_BITS);
    o[4] = DESCALE(tmp10 - tmp11, PASS1_BITS);
  }
  int32_t z1 = (tmp12 + tmp13) * F_0_541196100;
  o[2] = DESCALE(z1 + tmp13 * F_0_765366865, sh);
  o[6] = DESCALE(z1 + tmp12 * (-F_1_847759065), sh);
  z1 = tmp4 + tmp7;
  int32_t z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
  int32_t z5 = (z3 + z4) * F_1_175875602;
  tmp4 *= F_0_298631336;
  tmp5 *= F_2_053119869;
  tmp6 *= F_3_072711026;
  tmp7 *= F_1_501321110;
  z1 *= -F_0_899976223;
  z2 *= -F_2_562915447;
  z3 *= -F_1_961570560;
  z4 *= -F_0_390180644;
  z3 += z5;
  z4 += z5;
  o[7] = DESCALE(tmp4 + z1 + z3, sh);
  o[5] = DESCALE(tmp5 + z2 + z4, sh);
  o[3] = DESCALE(tmp6 + z2 + z3, sh);
  o[1] = DESCALE(tmp7 + z1 + z4, sh);
}

void jo_fdct_islow(int16_t blk[64]) {
  int32_t ws[64], in[8], out[8];
  for (int r = 0; r < 8; r++) { /* pass 1: rows */
    for (int i = 0; i < 8; i++) in[i] = blk[r * 8 + i];
    fdct_1d(in, out, 0);
    for (int i = 0; i < 8; i++) ws[r * 8 + i] = out[i];
  }
  for (int c = 0; c < 8; c++) { /* pass 2: columns */
    for (int i = 0; i < 8; i++) in[i] = ws[i * 8 + c];
    fdct_1d(in, out, 1);
    for (int i = 0; i < 8; i++) blk[i * 8 + c] = (int16_t)out[i];
  }
}

/* jcdctmgr.c quantize(): divisor = quantval << 3; result = sign * ((|x| + divisor/2) / divisor).
 * (libjpeg-turbo evaluates this with a reciprocal multiply; that is exact for 16-bit inputs,
 * which the Pillow byte-for-byte stream comparison in the tests confirms.) */
void jo_quantize(const int16_t in[64], const uint16_t q[64], int16_t out[64]) {
  for (int i = 0; i < 64; i++) {
    int32_t d = (int32_t)q[i] << 3;
    int32_t t = in[i];
    if (t < 0) {
      t = -t;
      t += d >> 1;
      t = t >= d ? t / d : 0;
      t = -t;
    } else {
      t += d >> 1;
      t = t >= d ? t / d : 0;
    }
    out[i] = (int16_t)t;
  }
}

void jo_idct_islow(const int16_t coef[64], const uint16_t q[64], uint8_t* out, int out_stride) {
  int32_t ws[64];
  for (int c = 0; c < 8; c++) { /* pass 1: columns */
    int32_t d0 = coef[c] * q[c], d1 = coef[8 + c] * q[8 + c], d2 = coef[16 + c] * q[16 + c],
            d3 = coef[24 + c] * q[24 + c], d4 = coef[32 + c] * q[32 + c],
            d5 = coef[40 + c] * q[40 + c], d6 = coef[48 + c] * q[48 + c],
            d7 = coef[56 + c] * q[56 + c];
    int32_t z2 = d2, z3 = d6;
    int32_t z1 = (z2 + z3) * F_0_541196100;
    int32_t tmp2 = z1 + z3 * (-F_1_847759065);
    int32_t tmp3 = z1 + z2 * F_0_765366865;
    z2 = d0;
    z3 = d4;
    int32_t tmp0 = (z2 + z3) * (1 << CONST_BITS);
    int32_t tmp1 = (z2 - z3) * (1 << CONST_BITS);
    int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = d7;
    tmp1 = d5;
    tmp2 = d3;
    tmp3 = d1;
    z1 = tmp0 + tmp3;
    z2 = tmp1 + tmp2;
    z3 = tmp0 + tmp2;
    int32_t z4 = tmp1 + tmp3;
    int32_t z5 = (z3 + z4) * F_1_175875602;
    tmp0 *= F_0_298631336;
    tmp1 *= F_2_053119869;
    tmp2 *= F_3_072711026;
    tmp3 *= F_1_501321110;
    z1 *= -F_0_899976223;
    z2 *= -F_2_562915447;
    z3 *= -F_1_961570560;
    z4 *= -F_0_390180644;
    z3 += z5;
    z4 += z5;
    tmp0 += z1 + z3;
    tmp1 += z2 + z4;
    tmp2 += z2 + z3;
    tmp3 += z1 + z4;
    ws[0 + c] = DESCALE(tmp10 + tmp3, CONST_BITS - PASS1_BITS);
    ws[56 + c] = DESCALE(tmp10 - tmp3, CONST_BITS - PASS1_BITS);
    ws[8 + c] = DESCALE(tmp11 + tmp2, CONST_BITS - PASS1_BITS);
    ws[48 + c] = DESCALE(tmp11 - tmp2, CONST_BITS - PASS1_BITS);
    ws[16 + c] = DESCALE(tmp12 + tmp1, CONST_BITS - PASS1_BITS);
    ws[40 + c] = DESCALE(tmp12 - tmp1, CONST_BITS - PASS1_BITS);
    ws[24 + c] = DESCALE(tmp13 + tmp0, CONST_BITS - PASS1_BITS);
    ws[32 + c] = DESCALE(tmp13 - tmp0, CONST_BITS - PASS1_BITS);
  }
  for (int r = 0; r < 8; r++) { /* pass 2: rows */
    const int32_t* w = ws + r * 8;
    int32_t z2 = w[2], z3 = w[6];
    int32_t z1 = (z2 + z3) * F_0_541196100;
    int32_t tmp2 = z1 + z3 * (-F_1_847759065);
    int32_t tmp3 = z1 + z2 * F_0_765366865;
    int32_t tmp0 = (w[0] + w[4]) * (1 << CONST_BITS);
    int32_t tmp1 = (w[0] - w[4]) * (1 << CONST_BITS);
    int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = w[7];
    tmp1 = w[5];
    tmp2 = w[3];
    tmp3 = w[1];
    z1 = tmp0 + tmp3;
    z2 = tmp1 + tmp2;
    z3 = tmp0 + tmp2;
    int32_t z4 = tmp1 + tmp3;
    int32_t z5 = (z3 + z4) * F_1_175875602;
    tmp0 *= F_0_298631336;
    tmp1 *= F_2_053119869;
    tmp2 *= F_3_072711026;
    tmp3 *= F_1_501321110;
    z1 *= -F_0_899976223;
    z2 *= -F_2_562915447;
    z3 *= -F_1_961570560;
    z4 *= -F_0_390180644;
    z3 += z5;
    z4 += z5;
    tmp0 += z1 + z3;
    tmp1 += z2 + z4;
    tmp2 += z2 + z3;
    tmp3 += z1 + z4;
    const int sh = CONST_BITS + PASS1_BITS + 3;
    uint8_t* o = out + r * out_stride;
    o[0] = clamp_u8(DESCALE(tmp10 + tmp3, sh) + 128);
    o[7] = clamp_u8(DESCALE(tmp10 - tmp3, sh) + 128);
    o[1] = clamp_u8(DESCALE(tmp11 + tmp2, sh) + 128);
    o[6] = clamp_u8(DESCALE(tmp11 - tmp2, sh) + 128);
    o[2] = clamp_u8(DESCALE(tmp12 + tmp1, sh) + 128);
    o[5] = clamp_u8(DESCALE(tmp12 - tmp1, sh) + 128);
    o[3] = clamp_u8(DESCALE(tmp13 + tmp0, sh) + 128);
    o[4] = clamp_u8(DESCALE(tmp13 - tmp0, sh) + 128);
  }
}

/* ---------------------------------------------------------------------------------------------
 * Frame geometry (jcmaster.c initial_setup / per_scan_setup)
 * ------------------------------------------------------------------------------------------ */
static int ceil_div(int a, int b) { return (a + b - 1) / b; }

static void frame_finish(jo_frame_t* f) {
  f->max_h = f->max_v = 1;
  for (int c = 0; c < f->ncomp; c++) {
    if (f->comp[c].h_samp > f->max_h) f->max_h = f->comp[c].h_samp;
    if (f->comp[c].v_samp > f->max_v) f->max_v = f->comp[c].v_samp;
  }
  for (int c = 0; c < f->ncomp; c++) {
    jo_comp_t* k = &f->comp[c];
    k->width = ceil_div(f->width * k->h_samp, f->max_h);
    k->height = ceil_div(f->height * k->v_samp, f->max_v);
    k->wblocks = ceil_div(f->width * k->h_samp, f->max_h * 8);
    k->hblocks = ceil_div(f->height * k->v_samp, f->max_v * 8);
  }
  if (f->ncomp == 1) { /* non-interleaved: MCU = one block */
    f->mcus_per_row = f->comp[0].wblocks;
    f->mcu_rows = f->comp[0].hblocks;
  } else {
    f->mcus_per_row = ceil_div(f->width, f->max_h * 8);
    f->mcu_rows = ceil_div(f->height, f->max_v * 8);
  }
}

int jo_frame_init(jo_frame_t* f, int fmt, int width, int height, int quality) {
  memset(f, 0, sizeof *f);
  f->width = width;
  f->height = height;
  int hs = 1, vs = 1;
  switch (fmt) {
    case JO_FMT_Y400: f->ncomp = 1; break;
    case JO_FMT_YUV420: f->ncomp = 3; hs = 2; vs = 2; break;
    case JO_FMT_YUV422: f->ncomp = 3; hs = 2; vs = 1; break;
    case JO_FMT_YUV444:
    case JO_FMT_RGB888: f->ncomp = 3; break;
    default: return -1;
  }
  for (int c = 0; c < f->ncomp; c++) {
    f->comp[c].h_samp = c == 0 ? hs : 1;
    f->comp[c].v_samp = c == 0 ? vs : 1;
    f->comp[c].tq = c == 0 ? 0 : 1;
  }
  jo_quant_tables(quality, f->qt[0], f->qt[1]);
  frame_finish(f);
  return 0;
}

/* ---------------------------------------------------------------------------------------------
 * Encode stage 1
 * ------------------------------------------------------------------------------------------ */
static void forward_block(const uint8_t* src, int stride, const uint16_t* q, int16_t* out) {
  int16_t blk[64];
  for (int r = 0; r < 8; r++)
    for (int c = 0; c < 8; c++) blk[r * 8 + c] = (int16_t)(src[r * stride + c] - 128);
  jo_fdct_islow(blk);
  jo_quantize(blk, q, out);
}

int jo_forward(const jo_frame_t* f, int fmt, const uint8_t* const planes[3],
               const unsigned strides[3], int16_t* coefs[3]) {
  for (int c = 0; c < f->ncomp; c++) {
    const jo_comp_t* k = &f->comp[c];
    const int pw = k->wblocks * 8, ph = k->hblocks * 8;
    uint8_t* pad = (uint8_t*)malloc((size_t)pw * ph);
    if (!pad) return -2;
    if (fmt == JO_FMT_RGB888) {
      /* scanline path: jccolor.c conversion, then expand_right_edge / expand_bottom_edge
       * (jcsample.c, jcprepct.c) replicate the last column / row. */
      const uint8_t* rgb = planes[0];
      for (int y = 0; y < ph; y++) {
        int sy = y < f->height ? y : f->height - 1;
        for (int x = 0; x < pw; x++) {
          int sx = x < f->width ? x : f->width - 1;
          const uint8_t* p = rgb + ((size_t)sy * strides[0] + sx) * 3;
          uint8_t yy, cb, cr;
          jo_rgb_to_ycc(p[0], p[1], p[2], &yy, &cb, &cr);
          pad[(size_t)y * pw + x] = c == 0 ? yy : (c == 1 ? cb : cr);
        }
      }
    } else {
      /* raw_data_in path, padding as JpegEncoderHelper::compressYCbCr builds it
       * (jpegencoderhelper.cpp:254-296): rows past the plane height come from a pad row that is
       * 0 for luma and 128 for chroma; when stride < aligned width the row is staged in a
       * scratch buffer whose tail is 0 (luma) / 128 (chroma); otherwise the bytes that follow
       * the row in the caller's buffer are read as they are. */
      const int fill = c == 0 ? 0 : 128;
      const int staged = (int)strides[c] < pw;
      for (int y = 0; y < ph; y++) {
        uint8_t* d = pad + (size_t)y * pw;
        if (y < k->height) {
          const uint8_t* s = planes[c] + (size_t)y * strides[c];
          if (staged) {
            memcpy(d, s, k->width);
            memset(d + k->width, fill, pw - k->width);
          } else {
            memcpy(d, s, pw);
          }
        } else if (staged) {
          /* scratch rows keep what the previous iMCU row left there (or their initial fill) */
          int rows_per_imcu = 8 * k->v_samp;
          int prev = y - rows_per_imcu;
          if (prev >= 0) memcpy(d, pad + (size_t)prev * pw, pw);
          else { memset(d, 0, pw); memset(d + k->width, fill, pw - k->width); }
        } else {
          memset(d, fill, pw);
        }
      }
    }
    for (int by = 0; by < k->hblocks; by++)
      for (int bx = 0; bx < k->wblocks; bx++)
        forward_block(pad + (size_t)by * 8 * pw + bx * 8, pw, f->qt[k->tq],
                      coefs[c] + ((size_t)by * k->wblocks + bx) * 64);
    free(pad);
  }
  return 0;
}

/* ---------------------------------------------------------------------------------------------
 * Huffman tables (jchuff.c jpeg_make_c_derived_tbl)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  uint16_t code[256];
  uint8_t len[256];
} enc_tbl_t;

static void make_enc_tbl(const uint8_t bits[17], const uint8_t* vals, enc_tbl_t* t) {
  memset(t, 0, sizeof *t);
  unsigned code = 0;
  int p = 0;
  for (int l = 1; l <= 16; l++) {
    for (int i = 0; i < bits[l]; i++, p++) {
      t->code[vals[p]] = (uint16_t)code++;
      t->len[vals[p]] = (uint8_t)l;
    }
    code <<= 1;
  }
}

typedef struct {
  uint8_t* buf;
  size_t size, cap;
  uint64_t acc;
  int nbits;
} bitw_t;

static int bw_reserve(bitw_t* w, size_t extra) {
  if (w->size + extra <= w->cap) return 0;
  size_t ncap = w->cap ? w->cap * 2 : 65536;
  while (ncap < w->size + extra) ncap *= 2;
  uint8_t* nb = (uint8_t*)realloc(w->buf, ncap);
  if (!nb) return -1;
  w->buf = nb;
  w->cap = ncap;
  return 0;
}
static void bw_byte(bitw_t* w, uint8_t b) {
  if (bw_reserve(w, 1)) return;
  w->buf[w->size++] = b;
}
static void bw_bytes(bitw_t* w, const void* p, size_t n) {
  if (bw_reserve(w, n)) return;
  memcpy(w->buf + w->size, p, n);
  w->size += n;
}
static void bw_u16(bitw_t* w, unsigned v) {
  bw_byte(w, (uint8_t)(v >> 8));
  bw_byte(w, (uint8_t)v);
}
static void bw_bits(bitw_t* w, unsigned code, int n) {
  if (!n) return;
  w->acc = (w->acc << n) | (code & ((1u << n) - 1));
  w->nbits += n;
  while (w->nbits >= 8) {
    uint8_t b = (uint8_t)(w->acc >> (w->nbits - 8));
    bw_byte(w, b);
    if (b == 0xFF) bw_byte(w, 0);
    w->nbits -= 8;
  }
}
static void bw_flush(bitw_t* w) { /* jchuff.c flush_bits: pad with ones */
  if (w->nbits) bw_bits(w, 0x7F, 8 - w->nbits);
  w->acc = 0;
  w->nbits = 0;
}

static int bitlen(int v) {
  int n = 0;
  while (v) { n++; v >>= 1; }
  return n;
}

static void encode_block(bitw_t* w, const int16_t* blk, int* last_dc, const enc_tbl_t* dc,
                         const enc_tbl_t* ac) {
  int temp = blk[0] - *last_dc, temp2 = temp;
  *last_dc = blk[0];
  if (temp < 0) { temp = -temp; temp2--; }
  int nb = bitlen(temp);
  bw_bits(w, dc->code[nb], dc->len[nb]);
  if (nb) bw_bits(w, (unsigned)temp2, nb);
  int r = 0;
  for (int k = 1; k < 64; k++) {
    temp = blk[k_natural_order[k]];
    if (temp == 0) { r++; continue; }
    while (r > 15) { bw_bits(w, ac->code[0xF0], ac->len[0xF0]); r -= 16; }
    temp2 = temp;
    if (temp < 0) { temp = -temp; temp2--; }
    nb = bitlen(temp);
    int sym = (r << 4) + nb;
    bw_bits(w, ac->code[sym], ac->len[sym]);
    bw_bits(w, (unsigned)temp2, nb);
    r = 0;
  }
  if (r > 0) bw_bits(w, ac->code[0], ac->len[0]);
}

static void emit_dqt(bitw_t* w, int idx, const uint16_t* q) {
  bw_u16(w, 0xFFDB);
  bw_u16(w, 67);
  bw_byte(w, (uint8_t)idx);
  for (int i = 0; i < 64; i++) bw_byte(w, (uint8_t)q[k_natural_order[i]]);
}
static void emit_dht(bitw_t* w, int idx, const uint8_t bits[17], const uint8_t* vals) {
  int n = 0;
  for (int i = 1; i <= 16; i++) n += bits[i];
  bw_u16(w, 0xFFC4);
  bw_u16(w, 2 + 1 + 16 + n);
  bw_byte(w, (uint8_t)idx);
  bw_bytes(w, bits + 1, 16);
  bw_bytes(w, vals, n);
}

int jo_write_stream(const jo_frame_t* f, int16_t* const coefs[3], const uint8_t* icc,
                    size_t icc_size, const char* comment, uint8_t** out, size_t* out_size) {
  bitw_t w;
  memset(&w, 0, sizeof w);
  /* jcmarker.c write_file_header */
  bw_u16(&w, 0xFFD8);
  static const uint8_t jfif[] = {0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  bw_bytes(&w, jfif, sizeof jfif);
  if (icc && icc_size) { /* jpeg_write_marker(APP2) jpegencoderhelper.cpp:202-204 */
    bw_u16(&w, 0xFFE2);
    bw_u16(&w, (unsigned)(icc_size + 2));
    bw_bytes(&w, icc, icc_size);
  }
  if (comment) { /* jpeg_write_marker(COM) jpegencoderhelper.cpp:205-211 */
    size_t n = strlen(comment);
    bw_u16(&w, 0xFFFE);
    bw_u16(&w, (unsigned)(n + 2));
    bw_bytes(&w, comment, n);
  }
  /* write_frame_header */
  emit_dqt(&w, 0, f->qt[0]);
  if (f->ncomp > 1) emit_dqt(&w, 1, f->qt[1]);
  bw_u16(&w, 0xFFC0);
  bw_u16(&w, 8 + 3 * f->ncomp);
  bw_byte(&w, 8);
  bw_u16(&w, (unsigned)f->height);
  bw_u16(&w, (unsigned)f->width);
  bw_byte(&w, (uint8_t)f->ncomp);
  for (int c = 0; c < f->ncomp; c++) {
    bw_byte(&w, (uint8_t)(c + 1));
    bw_byte(&w, (uint8_t)((f->comp[c].h_samp << 4) + f->comp[c].v_samp));
    bw_byte(&w, (uint8_t)f->comp[c].tq);
  }
  /* write_scan_header */
  emit_dht(&w, 0x00, k_bits_dc_lum, k_val_dc);
  emit_dht(&w, 0x10, k_bits_ac_lum, k_val_ac_lum);
  if (f->ncomp > 1) {
    emit_dht(&w, 0x01, k_bits_dc_chr, k_val_dc);
    emit_dht(&w, 0x11, k_bits_ac_chr, k_val_ac_chr);
  }
  bw_u16(&w, 0xFFDA);
  bw_u16(&w, 6 + 2 * f->ncomp);
  bw_byte(&w, (uint8_t)f->ncomp);
  for (int c = 0; c < f->ncomp; c++) {
    bw_byte(&w, (uint8_t)(c + 1));
    bw_byte(&w, c == 0 ? 0x00 : 0x11);
  }
  bw_byte(&w, 0);
  bw_byte(&w, 63);
  bw_byte(&w, 0);

  /* entropy-coded segment: jccoefct.c compress_data MCU walk + jchuff.c encode_mcu_huff */
  enc_tbl_t dcl, acl, dcc, acc;
  make_enc_tbl(k_bits_dc_lum, k_val_dc, &dcl);
  make_enc_tbl(k_bits_ac_lum, k_val_ac_lum, &acl);
  make_enc_tbl(k_bits_dc_chr, k_val_dc, &dcc);
  make_enc_tbl(k_bits_ac_chr, k_val_ac_chr, &acc);
  int last_dc[3] = {0, 0, 0};
  int16_t dummy[64];
  for (int my = 0; my < f->mcu_rows; my++) {
    for (int mx = 0; mx < f->mcus_per_row; mx++) {
      int prev_dc_in_mcu = 0; /* DC of the block coded just before, for dummy blocks */
      for (int c = 0; c < f->ncomp; c++) {
        const jo_comp_t* k = &f->comp[c];
        const int mw = f->ncomp == 1 ? 1 : k->h_samp, mh = f->ncomp == 1 ? 1 : k->v_samp;
        for (int yi = 0; yi < mh; yi++) {
          for (int xi = 0; xi < mw; xi++) {
            int bx = mx * mw + xi, by = my * mh + yi;
            const int16_t* blk;
            if (bx < k->wblocks && by < k->hblocks) {
              blk = coefs[c] + ((size_t)by * k->wblocks + bx) * 64;
            } else { /* dummy block: all-zero AC, DC copied from the preceding block */
              memset(dummy, 0, sizeof dummy);
              dummy[0] = (int16_t)prev_dc_in_mcu;
              blk = dummy;
            }
            prev_dc_in_mcu = blk[0];
            encode_block(&w, blk, &last_dc[c], c == 0 ? &dcl : &dcc, c == 0 ? &acl : &acc);
          }
        }
      }
    }
  }
  bw_flush(&w);
  bw_u16(&w, 0xFFD9);
  *out = w.buf;
  *out_size = w.size;
  return w.buf ? 0 : -2;
}

int jo_encode(const uint8_t* const planes[3], const unsigned strides[3], int width, int height,
              int fmt, int quality, const uint8_t* icc, size_t icc_size, const char* comment,
              uint8_t** out, size_t* out_size) {
  jo_frame_t f;
  if (jo_frame_init(&f, fmt, width, height, quality)) return -1;
  int16_t* coefs[3] = {0, 0, 0};
  for (int c = 0; c < f.ncomp; c++) {
    coefs[c] = (int16_t*)malloc((size_t)f.comp[c].wblocks * f.comp[c].hblocks * 64 * 2);
    if (!coefs[c]) return -2;
  }
  int rc = jo_forward(&f, fmt, planes, strides, coefs);
  if (!rc) rc = jo_write_stream(&f, coefs, icc, icc_size, comment, out, out_size);
  for (int c = 0; c < 3; c++) free(coefs[c]);
  return rc;
}

/* ---------------------------------------------------------------------------------------------
 * Decoder
 * ------------------------------------------------------------------------------------------ */
int jo_read_header(const uint8_t* d, size_t n, jo_header_t* h) {
  memset(h, 0, sizeof *h);
  if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return -1;
  size_t p = 2;
  int have_sof = 0;
  /* default Huffman tables are NOT assumed: baseline streams carry their DHT */
  while (p + 4 <= n) {
    if (d[p] != 0xFF) return -1;
    while (p < n && d[p] == 0xFF) p++; /* fill bytes */
    if (p >= n) return -1;
    uint8_t m = d[p++];
    if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
    if (m == 0xD9) return -1;
    if (p + 2 > n) return -1;
    size_t L = ((size_t)d[p] << 8) | d[p + 1];
    if (L < 2 || p + L > n) return -1;
    const uint8_t* s = d + p + 2;
    size_t sl = L - 2;
    if (m >= 0xE0 && m <= 0xE2) {
      if (h->nmarkers < 64) {
        h->markers[h->nmarkers].id = m;
        h->markers[h->nmarkers].offset = p + 2;
        h->markers[h->nmarkers].length = sl;
        h->nmarkers++;
      }
    } else if (m == 0xDB) {
      size_t i = 0;
      while (i < sl) {
        int prec = s[i] >> 4, idx = s[i] & 15;
        i++;
        if (idx > 1 || i + (prec ? 128 : 64) > sl) return -1;
        for (int k = 0; k < 64; k++) {
          unsigned v = prec ? ((unsigned)s[i] << 8 | s[i + 1]) : s[i];
          i += prec ? 2 : 1;
          h->frame.qt[idx][k_natural_order[k]] = (uint16_t)v;
        }
      }
    } else if (m == 0xC0 || m == 0xC1) {
      if (sl < 6) return -1;
      if (s[0] != 8) return -2;
      h->frame.height = (s[1] << 8) | s[2];
      h->frame.width = (s[3] << 8) | s[4];
      h->frame.ncomp = s[5];
      if ((h->frame.ncomp != 1 && h->frame.ncomp != 3) || sl < 6 + 3u * h->frame.ncomp)
        return -2;
      for (int c = 0; c < h->frame.ncomp; c++) {
        h->comp_id[c] = s[6 + 3 * c];
        h->frame.comp[c].h_samp = s[7 + 3 * c] >> 4;
        h->frame.comp[c].v_samp = s[7 + 3 * c] & 15;
        h->frame.comp[c].tq = s[8 + 3 * c];
        if (h->frame.comp[c].tq > 1) return -2;
      }
      if (h->frame.ncomp == 1) h->frame.comp[0].h_samp = h->frame.comp[0].v_samp = 1;
      frame_finish(&h->frame);
      have_sof = 1;
    } else if (m == 0xC2 || (m >= 0xC5 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC)) {
      return -2; /* progressive / arithmetic etc. unsupported */
    } else if (m == 0xC4) {
      size_t i = 0;
      while (i + 17 <= sl) {
        int cls = s[i] >> 4, idx = s[i] & 15;
        if (cls > 1 || idx > 1) return -2;
        int cnt = 0;
        h->bits[cls][idx][0] = 0;
        for (int k = 1; k <= 16; k++) {
          h->bits[cls][idx][k] = s[i + k];
          cnt += s[i + k];
        }
        i += 17;
        if (cnt > 256 || i + cnt > sl) return -1;
        memcpy(h->vals[cls][idx], s + i, cnt);
        i += cnt;
        h->have_tbl[cls][idx] = 1;
      }
    } else if (m == 0xDD) {
      if (sl < 2) return -1;
      h->restart_interval = (s[0] << 8) | s[1];
    } else if (m == 0xDA) {
      if (!have_sof || sl < 1 || s[0] != h->frame.ncomp || sl < 1 + 2u * s[0] + 3) return -2;
      for (int c = 0; c < h->frame.ncomp; c++) {
        int id = s[1 + 2 * c], k = -1;
        for (int j = 0; j < h->frame.ncomp; j++)
          if (h->comp_id[j] == id) k = j;
        if (k != c) return -2;
        h->dc_sel[c] = s[2 + 2 * c] >> 4;
        h->ac_sel[c] = s[2 + 2 * c] & 15;
        if (h->dc_sel[c] > 1 || h->ac_sel[c] > 1 || !h->have_tbl[0][h->dc_sel[c]] ||
            !h->have_tbl[1][h->ac_sel[c]])
          return -2;
      }
      h->scan_offset = p + L;
      h->scan_end = n;
      return 0;
    }
    p += L;
  }
  return -1;
}

typedef struct {
  /* jdhuff.c style: 9-bit lookahead + canonical maxcode walk */
  uint16_t look[512]; /* (len<<8)|sym, 0 = not resolvable in 9 bits */
  int32_t maxcode[18];
  int32_t valoff[17];
  const uint8_t* vals;
} dec_tbl_t;

static void make_dec_tbl(const uint8_t bits[17], const uint8_t* vals, dec_tbl_t* t) {
  memset(t, 0, sizeof *t);
  t->vals = vals;
  int code = 0, p = 0;
  for (int l = 1; l <= 16; l++) {
    if (bits[l]) {
      t->valoff[l] = p - code;
      for (int i = 0; i < bits[l]; i++, p++, code++) {
        if (l <= 9 && code < (1 << l)) {  /* a table that is no prefix code (legal while no scan selects it) stays in bounds */
          int lo = code << (9 - l);
          for (int k = 0; k < (1 << (9 - l)); k++) t->look[lo + k] = (uint16_t)((l << 8) | vals[p]);
        }
      }
      t->maxcode[l] = code - 1;
    } else {
      t->maxcode[l] = -1;
    }
    code <<= 1;
  }
  t->maxcode[17] = 0xFFFFF;
}

typedef struct {
  const uint8_t* d;
  size_t p, n;
  uint64_t acc;
  int nbits;
  int hit_marker;
} bitr_t;

static void br_fill(bitr_t* r) {
  while (r->nbits <= 56) {
    unsigned b = 0;
    if (!r->hit_marker && r->p < r->n) {
      b = r->d[r->p];
      if (b == 0xFF) {
        if (r->p + 1 < r->n && r->d[r->p + 1] == 0) {
          r->p += 2;
        } else {
          r->hit_marker = 1; /* leave marker in place, feed zeros */
          b = 0;
        }
      } else {
        r->p++;
      }
    }
    r->acc = (r->acc << 8) | b;
    r->nbits += 8;
  }
}
static inline unsigned br_peek(bitr_t* r, int n) {
  if (r->nbits < n) br_fill(r);
  return (unsigned)((r->acc >> (r->nbits - n)) & ((1u << n) - 1));
}
static inline void br_skip(bitr_t* r, int n) { r->nbits -= n; }
static inline unsigned br_get(bitr_t* r, int n) {
  if (!n) return 0;
  unsigned v = br_peek(r, n);
  r->nbits -= n;
  return v;
}
static int huff_decode(bitr_t* r, const dec_tbl_t* t) {
  unsigned look = br_peek(r, 9);
  unsigned e = t->look[look];
  if (e) {
    br_skip(r, e >> 8);
    return e & 255;
  }
  int l = 10;
  int32_t code = 0;
  unsigned all = br_peek(r, 16);
  for (; l <= 16; l++) {
    code = (int32_t)(all >> (16 - l));
    if (code <= t->maxcode[l]) break;
  }
  if (l > 16) return 0;
  br_skip(r, l);
  return t->vals[(code + t->valoff[l]) & 255];
}
static inline int extend(unsigned v, int n) { return v < (1u << (n - 1)) ? (int)v - (1 << n) + 1 : (int)v; }

static int decode_block(bitr_t* r, int16_t* blk, int* last_dc, const dec_tbl_t* dc,
                        const dec_tbl_t* ac) {
  memset(blk, 0, 64 * sizeof(int16_t));
  int s = huff_decode(r, dc);
  int diff = s ? extend(br_get(r, s), s) : 0;
  *last_dc += diff;
  blk[0] = (int16_t)*last_dc;
  for (int k = 1; k < 64; k++) {
    int rs = huff_decode(r, ac);
    int rr = rs >> 4, ss = rs & 15;
    if (ss) {
      k += rr;
      if (k > 63) return -1;
      blk[k_natural_order[k]] = (int16_t)extend(br_get(r, ss), ss);
    } else {
      if (rr != 15) break;
      k += 15;
    }
  }
  return 0;
}

int jo_decode_coefs(const uint8_t* data, size_t size, const jo_header_t* h, int16_t* coefs[3]) {
  const jo_frame_t* f = &h->frame;
  dec_tbl_t dct[2], act[2];
  for (int i = 0; i < 2; i++) {
    if (h->have_tbl[0][i]) make_dec_tbl(h->bits[0][i], h->vals[0][i], &dct[i]);
    if (h->have_tbl[1][i]) make_dec_tbl(h->bits[1][i], h->vals[1][i], &act[i]);
  }
  bitr_t r;
  memset(&r, 0, sizeof r);
  r.d = data;
  r.p = h->scan_offset;
  r.n = size;
  int last_dc[3] = {0, 0, 0};
  int16_t scratch[64];
  int mcu_count = 0;
  for (int my = 0; my < f->mcu_rows; my++) {
    for (int mx = 0; mx < f->mcus_per_row; mx++) {
      if (h->restart_interval && mcu_count && mcu_count % h->restart_interval == 0) {
        /* resync: drop remaining bits, expect RSTn */
        r.nbits = 0;
        r.acc = 0;
        r.hit_marker = 0;
        while (r.p + 1 < r.n && !(r.d[r.p] == 0xFF && r.d[r.p + 1] >= 0xD0 && r.d[r.p + 1] <= 0xD7))
          r.p++;
        r.p += 2;
        last_dc[0] = last_dc[1] = last_dc[2] = 0;
      }
      mcu_count++;
      for (int c = 0; c < f->ncomp; c++) {
        const jo_comp_t* k = &f->comp[c];
        const int mw = f->ncomp == 1 ? 1 : k->h_samp, mh = f->ncomp == 1 ? 1 : k->v_samp;
        for (int yi = 0; yi < mh; yi++)
          for (int xi = 0; xi < mw; xi++) {
            int bx = mx * mw + xi, by = my * mh + yi;
            int16_t* blk = (bx < k->wblocks && by < k->hblocks)
                               ? coefs[c] + ((size_t)by * k->wblocks + bx) * 64
                               : scratch;
            if (decode_block(&r, blk, &last_dc[c], &dct[h->dc_sel[c]], &act[h->ac_sel[c]]))
              return -1;
          }
      }
    }
  }
  return 0;
}

void jo_inverse(const jo_header_t* h, int16_t* const coefs[3], uint8_t* planes[3]) {
  const jo_frame_t* f = &h->frame;
  for (int c = 0; c < f->ncomp; c++) {
    const jo_comp_t* k = &f->comp[c];
    const int pw = k->wblocks * 8;
    for (int by = 0; by < k->hblocks; by++)
      for (int bx = 0; bx < k->wblocks; bx++)
        jo_idct_islow(coefs[c] + ((size_t)by * k->wblocks + bx) * 64, f->qt[k->tq],
                      planes[c] + (size_t)by * 8 * pw + bx * 8, pw);
  }
}

/* Chroma upsampling + colour conversion for RGB output of a subsampled three-component stream:
 * libjpeg-turbo jdsample.c h2v2_fancy_upsample / h2v1_fancy_upsample (do_fancy_upsampling is the
 * library default and the reference does not change it, jpegdecoderhelper.cpp:344-396; components
 * whose downsampled width is <= 2 are replicated instead, jinit_upsampler), row context
 * as jdmainct.c provides it (the row above the first and below the last real row is that row
 * itself), then jdcolor.c ycc_rgb_convert.  planes[] are the padded planes of jo_inverse
 * (stride wblocks*8); rgba is width*height*4 bytes, alpha 0xFF (JCS_EXT_RGBA).
 * Returns -1 for sampling layouts other than 4:4:4, 4:2:2 (h2v1) and 4:2:0 (h2v2). */
int jo_planes_to_rgba(const jo_header_t* h, uint8_t* const planes[3], uint8_t* rgba) {
  const jo_frame_t* f = &h->frame;
  if (f->ncomp != 3) return -1;
  const int hs = f->max_h, vs = f->max_v;
  if (f->comp[0].h_samp != hs || f->comp[0].v_samp != vs) return -1;
  if (f->comp[1].h_samp != 1 || f->comp[1].v_samp != 1 || f->comp[2].h_samp != 1 || f->comp[2].v_samp != 1) return -1;
  if (!((hs == 1 && vs == 1) || (hs == 2 && vs == 1) || (hs == 2 && vs == 2))) return -1;
  const int w = f->width, ht = f->height;
  const int cw = (w + hs - 1) / hs, ch = (ht + vs - 1) / vs; /* downsampled_width / _height */
  const int ypw = f->comp[0].wblocks * 8;
  uint8_t* up[2];
  up[0] = (uint8_t*)malloc((size_t)2 * cw + 2);
  up[1] = (uint8_t*)malloc((size_t)2 * cw + 2);
  if (!up[0] || !up[1]) { free(up[0]); free(up[1]); return -1; }
  for (int y = 0; y < ht; y++) {
    for (int c = 1; c < 3; c++) {
      const int pw = f->comp[c].wblocks * 8;
      uint8_t* o = up[c - 1];
      if (hs == 1) {
        memcpy(o, planes[c] + (size_t)y * pw, (size_t)w);
      } else if (cw <= 2) { /* jinit_upsampler: fancy only when downsampled_width > 2, else replication */
        const uint8_t* in = planes[c] + (size_t)(y / vs) * pw;
        for (int x = 0; x < cw; x++) o[2 * x] = o[2 * x + 1] = in[x];
      } else if (vs == 1) { /* h2v1 fancy */
        const uint8_t* in = planes[c] + (size_t)y * pw;
        if (cw == 1) { o[0] = o[1] = in[0]; }
        else {
          int x = 0;
          o[0] = in[0];
          o[1] = (uint8_t)((in[0] * 3 + in[1] + 2) >> 2);
          for (x = 1; x < cw - 1; x++) {
            o[2 * x] = (uint8_t)((in[x] * 3 + in[x - 1] + 1) >> 2);
            o[2 * x + 1] = (uint8_t)((in[x] * 3 + in[x + 1] + 2) >> 2);
          }
          o[2 * x] = (uint8_t)((in[x] * 3 + in[x - 1] + 1) >> 2);
          o[2 * x + 1] = in[x];
        }
      } else { /* h2v2 fancy: nearest input row, and the next nearest above (even y) / below (odd y) */
        const int r0 = y >> 1;
        int r1 = (y & 1) ? r0 + 1 : r0 - 1;
        if (r1 < 0) r1 = 0;
        if (r1 > ch - 1) r1 = ch - 1;
        const uint8_t* in0 = planes[c] + (size_t)r0 * pw;
        const uint8_t* in1 = planes[c] + (size_t)r1 * pw;
        if (cw == 1) {
          const int s0 = in0[0] * 3 + in1[0];
          o[0] = (uint8_t)((s0 * 4 + 8) >> 4);
          o[1] = (uint8_t)((s0 * 4 + 7) >> 4);
        } else {
          int last, cur = in0[0] * 3 + in1[0], next = in0[1] * 3 + in1[1];
          o[0] = (uint8_t)((cur * 4 + 8) >> 4);
          o[1] = (uint8_t)((cur * 3 + next + 7) >> 4);
          last = cur; cur = next;
          int x;
          for (x = 1; x < cw - 1; x++) {
            next = in0[x + 1] * 3 + in1[x + 1];
            o[2 * x] = (uint8_t)((cur * 3 + last + 8) >> 4);
            o[2 * x + 1] = (uint8_t)((cur * 3 + next + 7) >> 4);
            last = cur; cur = next;
          }
          o[2 * x] = (uint8_t)((cur * 3 + last + 8) >> 4);
          o[2 * x + 1] = (uint8_t)((cur * 4 + 7) >> 4);
        }
      }
    }
    for (int x = 0; x < w; x++) {
      uint8_t* px = rgba + ((size_t)y * w + x) * 4;
      jo_ycc_to_rgb(planes[0][(size_t)y * ypw + x], up[0][x], up[1][x], px, px + 1, px + 2);
      px[3] = 0xFF;
    }
  }
  free(up[0]);
  free(up[1]);
  return 0;
}

