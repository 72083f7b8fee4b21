// Bit-exact device evaluation of glibc's powf (2.39, sysdeps/ieee754/flt-32/e_powf.c, the
// x86-64 FMA multiarch variant current x86-64 host CPUs select).  Two sites of the reference
// call float std::pow on a *continuous* argument -- srgbOetf (gainmapmath.cpp:139-148, toneMap)
// and hlgInverseOotfApprox (:303-306, HLG decode output) -- and their results feed 8/10-bit
// quantisers, so a merely "correctly rounded" pow is not enough for bit-exact packed outputs:
// glibc's powf is faithful, not correctly rounded.  The routine below performs the same IEEE
// binary64 operations in the same order (log2 via a 16-entry table + degree-5 polynomial, exp2 via
// a 32-entry table + degree-3 polynomial, FMA where glibc's FMA build contracts), with the
// library's published table values; each DFMA/DMUL/DADD is correctly rounded on the device, so
// the result is identical bit for bit (tests/test_gpu_stages.py::test_device_powf_equals_libm).
// Domain handled: x >= 0 finite (incl. subnormals), y finite with |y*log2(x)| < 126: the only one
// the hot path produces (x in [0,1], y in {1/2.4, 1/1.2, gamma}).
#pragma once
#include <cuda_runtime.h>

namespace uhdr_b200 {

__device__ const double kPowfLog2Tab[32] = {
    0x1.661ec79f8f3bep+0, -0x1.efec65b963019p-2, 0x1.571ed4aaf883dp+0, -0x1.b0b6832d4fca4p-2,
    0x1.49539f0f010b0p+0, -0x1.7418b0a1fb77bp-2, 0x1.3c995b0b80385p+0, -0x1.39de91a6dcf7bp-2,
    0x1.30d190c8864a5p+0, -0x1.01d9bf3f2b631p-2, 0x1.25e227b0b8ea0p+0, -0x1.97c1d1b3b7af0p-3,
    0x1.1bb4a4a1a343fp+0, -0x1.2f9e393af3c9fp-3, 0x1.12358f08ae5bap+0, -0x1.960cbbf788d5cp-4,
    0x1.0953f419900a7p+0, -0x1.a6f9db6475fcep-5, 0x1.0p+0,                0x0.0p+0,
    0x1.e608cfd9a47acp-1, 0x1.338ca9f24f53dp-4,  0x1.ca4b31f026aa0p-1, 0x1.476a9543891bap-3,
    0x1.b2036576afce6p-1, 0x1.e840b4ac4e4d2p-3,  0x1.9c2d163a1aa2dp-1, 0x1.40645f0c6651cp-2,
    0x1.886e6037841edp-1, 0x1.88e9c2c1b9ff8p-2,  0x1.767dcf5534862p-1, 0x1.ce0a44eb17bccp-2};
__device__ const unsigned long long kExp2fTab[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull};

__device__ __forceinline__ float powf_glibc(float x, float y) {
  unsigned ix = __float_as_uint(x);
  if (ix == 0u) return 0.0f;  // pow(+0, y > 0)
  // pow(NaN, y) = NaN, as e_powf.c's special-case branch returns.  Without this the NaN's bits would go
  // through the log as a number near 2^129, and a table index taken from the result overflows.  A NaN
  // reaches here from applyGainMap's HLG output when max_content_boost puts +inf into the gain table.
  if (x != x) return x;
  if (ix < 0x00800000u) {     // subnormal x: normalise like e_powf.c
    ix = __float_as_uint(x * 0x1p23f);
    ix &= 0x7fffffffu;
    ix -= 23u << 23;
  }
  // log2_inline
  const unsigned tmp = ix - 0x3f330000u;
  const int i = (tmp >> 19) & 15;
  const unsigned top = tmp & 0xff800000u;
  const int k = (int)top >> 23;
  const double z = (double)__uint_as_float(ix - top);
  const double r = fma(z, kPowfLog2Tab[2 * i], -1.0);
  const double y0 = __dadd_rn((double)k, kPowfLog2Tab[2 * i + 1]);
  const double r2 = __dmul_rn(r, r);
  const double ya = fma(0x1.27616c9496e0bp-2, r, -0x1.71969a075c67ap-2);
  const double p = fma(0x1.ec70a6ca7baddp-2, r, -0x1.7154748bef6c8p-1);
  const double r4 = __dmul_rn(r2, r2);
  double q = fma(0x1.71547652ab82bp+0, r, y0);
  q = fma(p, r2, q);
  const double logx = fma(ya, r4, q);
  const double ylogx = __dmul_rn((double)y, logx);
  // exp2_inline (sign_bias 0)
  const double kShift = 0x1.8p+47;
  double kd = __dadd_rn(ylogx, kShift);
  const unsigned long long ki = (unsigned long long)__double_as_longlong(kd);
  kd = __dsub_rn(kd, kShift);
  const double rr = __dsub_rn(ylogx, kd);
  const unsigned long long t = kExp2fTab[ki & 31] + (ki << 47);
  const double s = __longlong_as_double((long long)t);
  const double zz = fma(0x1.c6af84b912394p-5, rr, 0x1.ebfce50fac4f3p-3);
  const double rr2 = __dmul_rn(rr, rr);
  double yy = fma(0x1.62e42ff0c52d6p-1, rr, 1.0);
  yy = fma(zz, rr2, yy);
  return __double2float_rn(__dmul_rn(yy, s));
}

}  // namespace uhdr_b200
