/*
 * jpeg_scaled_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement of libjpeg-turbo's reduced-size decoding (scale_num = 1, scale_denom = k in {1, 2, 4, 8}) on top
 * of the baseline restatement in jpeg_oracle.c, which supplies the header parser, the entropy decoder and the 8x8
 * islow IDCT.  Restated here, in our own words:
 *  - jdmaster.c output geometry: the image is ceil(W / k) x ceil(H / k).  Every component starts at a DCT scaled
 *    size s = 8 / k, doubled while s < 8 and both (max_h * 8/k) % (h_samp * 2s) and (max_v * 8/k) % (v_samp * 2s)
 *    are 0 (chroma is scaled up by the IDCT, not by the upsampler).  A component plane is
 *    ceil(W * h_samp * s / (max_h * 8)) x ceil(H * v_samp * s / (max_v * 8)).
 *  - jidctred.c: the reduced inverse DCTs that output 4x4, 2x2 and 1x1 samples from an 8x8 block, dequantised with
 *    the islow multipliers (the raw quantiser values).  Results are clamped like the SIMD forms, which saturate.
 * Pinned by tests/test_scaled_decode_cpu.py to the real library through jpeg_scaled_ref.c.
 * Built by oracle/scaled.mk into _ref/libjpeg_scaled_oracle.so.
 */
#include <stdint.h>
#include <string.h>

#include "jpeg_oracle.h"

#define CB 13 /* CONST_BITS */
#define PB 2  /* PASS1_BITS */
#define DESC(x, n) (((x) + (1 << ((n)-1))) >> (n))

static int clamp255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

/* 4-point even / odd parts shared by both passes of the 4x4 output (inputs 0, 2, 6 and 1, 3, 5, 7) */
static void idct4(int d0, int d1, int d2, int d3, int d5, int d6, int d7, int shift, int o[4]) {
  const int t0 = d0 * (1 << (CB + 1));
  const int t2 = d2 * 15137 + d6 * -6270;                       /* 1.847759065, -0.765366865 */
  const int t10 = t0 + t2, t12 = t0 - t2;
  const int a = d7 * -1730 + d5 * 11893 + d3 * -17799 + d1 * 8697;  /* -0.211164243 1.451774981 -2.172734803 1.061594337 */
  const int b = d7 * -4176 + d5 * -4926 + d3 * 7373 + d1 * 20995;   /* -0.509795579 -0.601344887 0.899976223 2.562915447 */
  o[0] = DESC(t10 + b, shift);
  o[3] = DESC(t10 - b, shift);
  o[1] = DESC(t12 + a, shift);
  o[2] = DESC(t12 - a, shift);
}

/* 2-point: DC and the odd inputs 1, 3, 5, 7 */
static void idct2(int d0, int d1, int d3, int d5, int d7, int shift, int o[2]) {
  const int t10 = d0 * (1 << (CB + 2));
  const int t0 = d7 * -5906 + d5 * 6967 + d3 * -10426 + d1 * 29692;  /* -0.720959822 0.850430095 -1.272758580 3.624509785 */
  o[0] = DESC(t10 + t0, shift);
  o[1] = DESC(t10 - t0, shift);
}

void jso_idct_4x4(const int16_t coef[64], const uint16_t q[64], uint8_t* out, int stride) {
  int v[64], ws[32], o[4];
  for (int i = 0; i < 64; i++) v[i] = coef[i] * q[i];
  for (int c = 0; c < 8; c++) {  /* columns; column 4 does not contribute */
    if (c == 4) continue;
    idct4(v[c], v[8 + c], v[16 + c], v[24 + c], v[40 + c], v[48 + c], v[56 + c], CB - PB + 1, o);
    for (int r = 0; r < 4; r++) ws[r * 8 + c] = o[r];
  }
  for (int r = 0; r < 4; r++) {
    const int* w = ws + r * 8;
    idct4(w[0], w[1], w[2], w[3], w[5], w[6], w[7], CB + PB + 3 + 1, o);
    for (int c = 0; c < 4; c++) out[r * stride + c] = (uint8_t)clamp255(o[c] + 128);
  }
}

void jso_idct_2x2(const int16_t coef[64], const uint16_t q[64], uint8_t* out, int stride) {
  int ws[16], o[2];
  for (int c = 0; c < 8; c++) {  /* columns 0, 1, 3, 5, 7 */
    if (c == 2 || c == 4 || c == 6) continue;
    const int d[8] = {coef[c] * q[c], coef[8 + c] * q[8 + c], 0, coef[24 + c] * q[24 + c], 0, coef[40 + c] * q[40 + c], 0,
                      coef[56 + c] * q[56 + c]};
    idct2(d[0], d[1], d[3], d[5], d[7], CB - PB + 2, o);
    ws[c] = o[0];
    ws[8 + c] = o[1];
  }
  for (int r = 0; r < 2; r++) {
    const int* w = ws + r * 8;
    idct2(w[0], w[1], w[3], w[5], w[7], CB + PB + 3 + 2, o);
    for (int c = 0; c < 2; c++) out[r * stride + c] = (uint8_t)clamp255(o[c] + 128);
  }
}

/* DC only; libjpeg-turbo has no SIMD form of it, so the C range-limit table applies: the descaled value is taken
 * modulo 1024 as a signed number in [-512, 511], then clamped after the +128 */
void jso_idct_1x1(const int16_t coef[64], const uint16_t q[64], uint8_t* out) {
  int t = DESC(coef[0] * (int)q[0], 3) & 1023;
  if (t >= 512) t -= 1024;
  out[0] = (uint8_t)clamp255(t + 128);
}

/* geometry (12 ints): [0] output width, [1] output height, then per component c: [2 + 3c] DCT scaled size,
 * [3 + 3c] plane width, [4 + 3c] plane height.  Returns 0, or -1 for a k outside {1, 2, 4, 8}. */
int jso_scaled_geometry(const jo_frame_t* f, int k, int g[12]) {
  if (k != 1 && k != 2 && k != 4 && k != 8) return -1;
  memset(g, 0, 12 * sizeof(int));
  g[0] = (f->width + k - 1) / k;
  g[1] = (f->height + k - 1) / k;
  const int m = 8 / k;
  for (int c = 0; c < f->ncomp; c++) {
    const jo_comp_t* p = &f->comp[c];
    int s = m;
    while (s < 8 && (f->max_h * m) % (p->h_samp * s * 2) == 0 && (f->max_v * m) % (p->v_samp * s * 2) == 0) s *= 2;
    g[2 + 3 * c] = s;
    g[3 + 3 * c] = (int)(((long long)f->width * p->h_samp * s + f->max_h * 8 - 1) / (f->max_h * 8));
    g[4 + 3 * c] = (int)(((long long)f->height * p->v_samp * s + f->max_v * 8 - 1) / (f->max_v * 8));
  }
  return 0;
}

/* coefficients (as jo_decode_coefs leaves them) -> plane c of wblocks*s x hblocks*s samples, stride wblocks*s */
int jso_inverse_scaled(const jo_header_t* h, int k, int16_t* const coefs[3], uint8_t* planes[3]) {
  int g[12];
  if (jso_scaled_geometry(&h->frame, k, g)) return -1;
  const jo_frame_t* f = &h->frame;
  for (int c = 0; c < f->ncomp; c++) {
    const jo_comp_t* p = &f->comp[c];
    const uint16_t* q = f->qt[p->tq];
    const int s = g[2 + 3 * c], stride = p->wblocks * s;
    for (int by = 0; by < p->hblocks; by++)
      for (int bx = 0; bx < p->wblocks; bx++) {
        const int16_t* blk = coefs[c] + ((size_t)by * p->wblocks + bx) * 64;
        uint8_t* o = planes[c] + (size_t)by * s * stride + (size_t)bx * s;
        if (s == 8) {
          jo_idct_islow(blk, q, o, stride);
        } else if (s == 4) {
          jso_idct_4x4(blk, q, o, stride);
        } else if (s == 2) {
          jso_idct_2x2(blk, q, o, stride);
        } else {
          jso_idct_1x1(blk, q, o);
        }
      }
  }
  return 0;
}
