/* powf_half.h -- powf(x, 0.5f) exactly as glibc (>= 2.28, x86-64 FMA variant) rounds it, for host and device.
 *
 * Adam's ComputeUpdateValue takes the square root of the second moment with caffe_powx(v, 0.5)
 * (adam_solver.cpp:62-64), and mkl_alternate.hpp's vsPowx is powf.  glibc's powf is NOT sqrtf: it evaluates
 * 2^(y*log2(x)) in double with a 16-entry log2 table, a degree-5 polynomial, a 32-entry exp2 table and a cubic,
 * then rounds to float, and it differs from the correctly rounded sqrtf by one ulp on 1,361,091 of the 2^31
 * non-negative bit patterns (oracle/adam_oracle.c cos_oracle_powf_half_check counts them).  The update kernels
 * therefore evaluate this same sequence of double operations: every double operation below is rounded once
 * (COS_PH_MUL / COS_PH_ADD / COS_PH_FMA map to __dmul_rn / __dadd_rn / __fma_rn on the device and to plain
 * operators + fma() on a host compiled with -ffp-contract=off), so the result is bit-identical to glibc's.
 * The tables and coefficients are those of the published algorithm (the same numbers as musl's powf_data.c
 * and exp2f_data.c, from Arm's optimized-routines).
 *
 * Defined for every input: +-0 -> +0, subnormals are normalised first, +inf -> +inf; negative and NaN inputs
 * (which Adam's v never holds: it is a sum of non-negative products) return a quiet NaN. */
#ifndef COS_POWF_HALF_H_
#define COS_POWF_HALF_H_

#include <stdint.h>

#ifdef __CUDACC__
#define COS_PH_DEVICE 1
#define COS_PH_FN __device__ __forceinline__
#else
#include <math.h>
#include <string.h>
#define COS_PH_FN static inline
#endif

#ifdef COS_PH_DEVICE
#define COS_PH_MUL(a, b) __dmul_rn((a), (b))
#define COS_PH_ADD(a, b) __dadd_rn((a), (b))
#define COS_PH_FMA(a, b, c) __fma_rn((a), (b), (c))
#define COS_PH_TABLE __device__ static const
#else
#define COS_PH_MUL(a, b) ((a) * (b))
#define COS_PH_ADD(a, b) ((a) + (b))
#define COS_PH_FMA(a, b, c) fma((a), (b), (c))
#define COS_PH_TABLE static const
#endif

/* log2 table: {1/c, log2(c)} for 16 subintervals of [0x3f330000, 2 * 0x3f330000) */
COS_PH_TABLE double cos_ph_log2_tab[32] = {
    0x1.661ec79f8f3bep+0, -0x1.efec65b963019p-2, 0x1.571ed4aaf883dp+0, -0x1.b0b6832d4fca4p-2,
    0x1.49539f0f010bp+0,  -0x1.7418b0a1fb77bp-2, 0x1.3c995b0b80385p+0, -0x1.39de91a6dcf7bp-2,
    0x1.30d190c8864a5p+0, -0x1.01d9bf3f2b631p-2, 0x1.25e227b0b8eap+0,  -0x1.97c1d1b3b7afp-3,
    0x1.1bb4a4a1a343fp+0, -0x1.2f9e393af3c9fp-3, 0x1.12358f08ae5bap+0, -0x1.960cbbf788d5cp-4,
    0x1.0953f419900a7p+0, -0x1.a6f9db6475fcep-5, 0x1p+0,               0x0p+0,
    0x1.e608cfd9a47acp-1, 0x1.338ca9f24f53dp-4,  0x1.ca4b31f026aap-1,  0x1.476a9543891bap-3,
    0x1.b2036576afce6p-1, 0x1.e840b4ac4e4d2p-3,  0x1.9c2d163a1aa2dp-1, 0x1.40645f0c6651cp-2,
    0x1.886e6037841edp-1, 0x1.88e9c2c1b9ff8p-2,  0x1.767dcf5534862p-1, 0x1.ce0a44eb17bccp-2,
};
COS_PH_TABLE double cos_ph_log2_poly[5] = {
    0x1.27616c9496e0bp-2, -0x1.71969a075c67ap-2, 0x1.ec70a6ca7baddp-2, -0x1.7154748bef6c8p-1, 0x1.71547652ab82bp+0,
};
/* exp2 table: bits of 2^(i/32) minus i << 47 (the exponent is added back from k) */
COS_PH_TABLE uint64_t cos_ph_exp2_tab[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull,
};
COS_PH_TABLE double cos_ph_exp2_poly[3] = {0x1.c6af84b912394p-5, 0x1.ebfce50fac4f3p-3, 0x1.62e42ff0c52d6p-1};

COS_PH_FN uint32_t cos_ph_f2u(float f) {
#ifdef COS_PH_DEVICE
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}
COS_PH_FN float cos_ph_u2f(uint32_t u) {
#ifdef COS_PH_DEVICE
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}
COS_PH_FN uint64_t cos_ph_d2u(double d) {
#ifdef COS_PH_DEVICE
  return static_cast<uint64_t>(__double_as_longlong(d));
#else
  uint64_t u;
  memcpy(&u, &d, 8);
  return u;
#endif
}
COS_PH_FN double cos_ph_u2d(uint64_t u) {
#ifdef COS_PH_DEVICE
  return __longlong_as_double(static_cast<long long>(u));
#else
  double d;
  memcpy(&d, &u, 8);
  return d;
#endif
}

COS_PH_FN float cos_powf_half(float x) {
  uint32_t ix = cos_ph_f2u(x);
  if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {  /* +-0, subnormal, inf, NaN, negative */
    if ((ix & 0x7fffffffu) == 0) return 0.f;           /* x*x */
    if (ix == 0x7f800000u) return x;                    /* +inf */
    if ((ix & 0x80000000u) || ix > 0x7f800000u) return cos_ph_u2f(0x7fffffffu);
    ix = cos_ph_f2u(x * 0x1p23f);                       /* subnormal: exact scale, exponent corrected below */
    ix -= 23u << 23;
  }
  /* log2(x) = k + log2(c) + log1p(z/c - 1)/ln2, x = 2^k z */
  const uint32_t tmp = ix - 0x3f330000u;
  const int i = (int)((tmp >> 19) % 16u);
  const uint32_t top = tmp & 0xff800000u;
  const uint32_t iz = ix - top;
  const int k = (int32_t)top >> 23;
  const double invc = cos_ph_log2_tab[2 * i], logc = cos_ph_log2_tab[2 * i + 1];
  const double z = (double)cos_ph_u2f(iz);
  const double* A = cos_ph_log2_poly;
  const double r = COS_PH_FMA(z, invc, -1.0);
  const double y0 = COS_PH_ADD(logc, (double)k);
  const double r2 = COS_PH_MUL(r, r);
  double y = COS_PH_FMA(A[0], r, A[1]);
  const double p = COS_PH_FMA(A[2], r, A[3]);
  const double r4 = COS_PH_MUL(r2, r2);
  double q = COS_PH_FMA(A[4], r, y0);
  q = COS_PH_FMA(p, r2, q);
  y = COS_PH_FMA(y, r4, q);
  /* 2^(y/2) = 2^(m/32) * 2^rr, |rr| <= 1/64 */
  const double xd = COS_PH_MUL(0.5, y);
  const double shift = 0x1.8p+47;
  double kd = COS_PH_ADD(xd, shift);
  const uint64_t ki = cos_ph_d2u(kd);
  kd = COS_PH_ADD(kd, -shift);
  const double rr = COS_PH_ADD(xd, -kd);
  const uint64_t t = cos_ph_exp2_tab[ki % 32u] + (ki << 47);
  const double s = cos_ph_u2d(t);
  const double* C = cos_ph_exp2_poly;
  const double zz = COS_PH_FMA(C[0], rr, C[1]);
  const double rr2 = COS_PH_MUL(rr, rr);
  double e = COS_PH_FMA(C[2], rr, 1.0);
  e = COS_PH_FMA(zz, rr2, e);
  e = COS_PH_MUL(e, s);
  return (float)e;
}

#endif
