// cmix_b200/csrc/exact_math.h
//
// Bit-exact device restatements of the three libm entry points the reference's
// floating-point path calls per bit / per byte:
//   expf  — Sigmoid::Logistic (reference src/mixer/sigmoid.cpp:19-21), LSTM gates
//           (src/mixer/lstm-layer.cpp:66-72) and the LSTM softmax (src/mixer/lstm.cpp:143)
//   tanhf — LSTM input node and cell output (src/mixer/lstm-layer.cpp:68,78)
// The parity oracle is the reference built with strict FP flags against glibc
// 2.39 (x86-64, FMA-capable host, so the ifunc'd FMA variant of expf). glibc's
// float functions are not correctly rounded, so "any accurate expf" is not
// enough for a bit-exact per-bit probability stream: these routines reproduce
// the published algorithms operation by operation —
//   expf : the 32-entry-table, double-precision algorithm of ARM's optimized
//          routines that glibc adopted in 2.27 (three multiply-adds contracted
//          to FMA in the x86-64 FMA build),
//   tanhf/expm1f : the single-precision fdlibm algorithms.
// tests/test_exact_math_device.py checks the device build against the host build over all 2^32 inputs
// (tests/exact_math_sweep.cu / .cpp), and the host build against glibc on the special classes (all 2^32
// inputs with CMIXB200_SLOW=1).
//
// Every operation is written with explicit rounding intrinsics so nvcc can
// never contract a multiply-add that the oracle does not contract.
#ifndef CMIXB200_EXACT_MATH_H
#define CMIXB200_EXACT_MATH_H

#include <stdint.h>
#include <string.h>

#if defined(__CUDA_ARCH__)
#define XM_HD __host__ __device__ __forceinline__
#define XM_FADD(a, b) __fadd_rn((a), (b))
#define XM_FSUB(a, b) __fsub_rn((a), (b))
#define XM_FMUL(a, b) __fmul_rn((a), (b))
#define XM_FDIV(a, b) __fdiv_rn((a), (b))
#define XM_DADD(a, b) __dadd_rn((a), (b))
#define XM_DSUB(a, b) __dsub_rn((a), (b))
#define XM_DMUL(a, b) __dmul_rn((a), (b))
#define XM_DFMA(a, b, c) __fma_rn((a), (b), (c))
#define XM_F2U(x) __float_as_uint(x)
#define XM_U2F(x) __uint_as_float(x)
#define XM_D2U(x) ((uint64_t)__double_as_longlong(x))
#define XM_U2D(x) __longlong_as_double((long long)(x))
#else
// Host build (tests / sweep tool): compile with -ffp-contract=off.
#include <math.h>
#if defined(__CUDACC__)
#define XM_HD __host__ __device__ inline
#else
#define XM_HD static inline
#endif
#define XM_FADD(a, b) ((float)(a) + (float)(b))
#define XM_FSUB(a, b) ((float)(a) - (float)(b))
#define XM_FMUL(a, b) ((float)(a) * (float)(b))
#define XM_FDIV(a, b) ((float)(a) / (float)(b))
#define XM_DADD(a, b) ((double)(a) + (double)(b))
#define XM_DSUB(a, b) ((double)(a) - (double)(b))
#define XM_DMUL(a, b) ((double)(a) * (double)(b))
#define XM_DFMA(a, b, c) fma((a), (b), (c))
static inline uint32_t xm_f2u(float x) { uint32_t u; memcpy(&u, &x, 4); return u; }
static inline float xm_u2f(uint32_t u) { float x; memcpy(&x, &u, 4); return x; }
static inline uint64_t xm_d2u(double x) { uint64_t u; memcpy(&u, &x, 8); return u; }
static inline double xm_u2d(uint64_t u) { double x; memcpy(&x, &u, 8); return x; }
#define XM_F2U(x) xm_f2u(x)
#define XM_U2F(x) xm_u2f(x)
#define XM_D2U(x) xm_d2u(x)
#define XM_U2D(x) xm_u2d(x)
#endif

#if defined(__CUDACC__)
// Two IEEE fp32 products, each rounded to nearest (sm_90a has no paired fp32 multiply: two FMULs).
// The explicit rounding keeps nvcc from contracting them into the FADD chain they feed, so that
// chain reproduces the reference's sum bit for bit.
__device__ __forceinline__ void xm_fmul2(float ax, float ay, float bx, float by, float& px, float& py) {
  px = __fmul_rn(ax, bx);
  py = __fmul_rn(ay, by);
}
#endif

// 2^(i/32) as IEEE doubles with i<<47 subtracted from the bit pattern
// (so that adding k<<47 splices in the exponent).
#if defined(__CUDA_ARCH__)
__device__ __constant__
#else
static const
#endif
uint64_t kXmExp2Tab[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull};

XM_HD float xm_expf(float x) {
  const uint32_t ux = XM_F2U(x);
  const uint32_t abstop = (ux >> 20) & 0x7ff;
  if (abstop >= 0x42b) {                       // |x| >= 88 or NaN
    if (ux == 0xff800000u) return 0.0f;
    if (abstop >= 0x7f8) return XM_FADD(x, x);
    if (x > 0x1.62e42ep6f) return XM_U2F(0x7f800000u);          // overflow -> +inf
    if (x < -0x1.9fe368p6f) return 0.0f;                         // underflow -> +0
  }
  const double xd = (double)x;
  const double kInvLn2N = 0x1.71547652b82fep+0 * 32;   // N/ln2, N = 32
  const double kShift = 0x1.8p+52;
  double z = XM_DMUL(kInvLn2N, xd);
  double kd = XM_DADD(z, kShift);
  const uint64_t ki = XM_D2U(kd);
  kd = XM_DSUB(kd, kShift);
  // The FMA build of glibc fuses InvLn2N*xd into this subtraction (found by the
  // exhaustive sweep: 2 of 2^32 inputs differ otherwise).
  const double r = XM_DFMA(kInvLn2N, xd, -kd);
  uint64_t t = kXmExp2Tab[ki & 31];
  t += ki << 47;
  const double s = XM_U2D(t);
  const double c0 = 0x1.c6af84b912394p-5 / 32 / 32 / 32;
  const double c1 = 0x1.ebfce50fac4f3p-3 / 32 / 32;
  const double c2 = 0x1.62e42ff0c52d6p-1 / 32;
  z = XM_DFMA(c0, r, c1);
  const double r2 = XM_DMUL(r, r);
  double y = XM_DFMA(c2, r, 1.0);
  y = XM_DFMA(z, r2, y);
  y = XM_DMUL(y, s);
  return (float)y;
}

// fdlibm single-precision expm1.
XM_HD float xm_expm1f(float x) {
  const float one = 1.0f, huge = 1.0e+30f, tiny = 1.0e-30f;
  const float o_threshold = 8.8721679688e+01f, ln2_hi = 6.9313812256e-01f, ln2_lo = 9.0580006145e-06f,
              invln2 = 1.4426950216e+00f;
  const float Q1 = -3.3333335072e-02f, Q2 = 1.5873016091e-03f, Q3 = -7.9365076090e-05f,
              Q4 = 4.0082177293e-06f, Q5 = -2.0109921195e-07f;
  float y, hi, lo, c = 0.0f, t, e, hxs, hfx, r1;
  int32_t k;
  uint32_t hx = XM_F2U(x);
  const uint32_t xsb = hx & 0x80000000u;
  hx &= 0x7fffffffu;
  if (hx >= 0x4195b844u) {                     // |x| >= 27*ln2
    if (hx >= 0x42b17218u) {                   // |x| >= 88.721...
      if (hx > 0x7f800000u) return XM_FADD(x, x);
      if (hx == 0x7f800000u) return xsb == 0 ? x : -1.0f;
      if (x > o_threshold) return XM_FMUL(huge, huge);
    }
    if (xsb != 0) return XM_FSUB(tiny, one);
  }
  if (hx > 0x3eb17218u) {                      // |x| > 0.5 ln2
    if (hx < 0x3F851592u) {                    // |x| < 1.5 ln2
      if (xsb == 0) { hi = XM_FSUB(x, ln2_hi); lo = ln2_lo; k = 1; }
      else { hi = XM_FADD(x, ln2_hi); lo = -ln2_lo; k = -1; }
    } else {
      k = (int32_t)XM_FADD(XM_FMUL(invln2, x), (xsb == 0) ? 0.5f : -0.5f);
      t = (float)k;
      hi = XM_FSUB(x, XM_FMUL(t, ln2_hi));
      lo = XM_FMUL(t, ln2_lo);
    }
    x = XM_FSUB(hi, lo);
    c = XM_FSUB(XM_FSUB(hi, x), lo);
  } else if (hx < 0x33000000u) {               // |x| < 2^-25
    t = XM_FADD(huge, x);
    return XM_FSUB(x, XM_FSUB(t, XM_FADD(huge, x)));
  } else {
    k = 0;
  }
  hfx = XM_FMUL(0.5f, x);
  hxs = XM_FMUL(x, hfx);
  r1 = XM_FADD(one, XM_FMUL(hxs, XM_FADD(Q1, XM_FMUL(hxs, XM_FADD(Q2, XM_FMUL(hxs, XM_FADD(Q3, XM_FMUL(hxs, XM_FADD(Q4, XM_FMUL(hxs, Q5))))))))));
  t = XM_FSUB(3.0f, XM_FMUL(r1, hfx));
  e = XM_FMUL(hxs, XM_FDIV(XM_FSUB(r1, t), XM_FSUB(6.0f, XM_FMUL(x, t))));
  if (k == 0) return XM_FSUB(x, XM_FSUB(XM_FMUL(x, e), hxs));
  e = XM_FSUB(XM_FMUL(x, XM_FSUB(e, c)), c);
  e = XM_FSUB(e, hxs);
  if (k == -1) return XM_FSUB(XM_FMUL(0.5f, XM_FSUB(x, e)), 0.5f);
  if (k == 1) {
    if (x < -0.25f) return XM_FMUL(-2.0f, XM_FSUB(e, XM_FADD(x, 0.5f)));
    return XM_FADD(one, XM_FMUL(2.0f, XM_FSUB(x, e)));
  }
  if (k <= -2 || k > 56) {
    y = XM_FSUB(one, XM_FSUB(e, x));
    y = XM_U2F(XM_F2U(y) + ((uint32_t)k << 23));
    return XM_FSUB(y, one);
  }
  if (k < 23) {
    t = XM_U2F(0x3f800000u - (0x1000000u >> k));
    y = XM_FSUB(t, XM_FSUB(e, x));
    y = XM_U2F(XM_F2U(y) + ((uint32_t)k << 23));
  } else {
    t = XM_U2F((uint32_t)(0x7f - k) << 23);
    y = XM_FSUB(x, XM_FADD(e, t));
    y = XM_FADD(y, one);
    y = XM_U2F(XM_F2U(y) + ((uint32_t)k << 23));
  }
  return y;
}

// fdlibm single-precision tanh.
XM_HD float xm_tanhf(float x) {
  const float one = 1.0f, two = 2.0f, tiny = 1.0e-30f;
  float t, z;
  const uint32_t jx = XM_F2U(x);
  const uint32_t ix = jx & 0x7fffffffu;
  if (ix >= 0x7f800000u) {
    if ((int32_t)jx >= 0) return XM_FADD(XM_FDIV(one, x), one);
    return XM_FSUB(XM_FDIV(one, x), one);
  }
  if (ix < 0x41b00000u) {                      // |x| < 22
    if (ix == 0) return x;
    if (ix < 0x24000000u) return XM_FMUL(x, XM_FADD(one, x));
    const float ax = XM_U2F(ix);
    if (ix >= 0x3f800000u) {
      t = xm_expm1f(XM_FMUL(two, ax));
      z = XM_FSUB(one, XM_FDIV(two, XM_FADD(t, two)));
    } else {
      t = xm_expm1f(XM_FMUL(-two, ax));
      z = XM_FDIV(-t, XM_FADD(t, two));
    }
  } else {
    z = XM_FSUB(one, tiny);
  }
  return ((int32_t)jx >= 0) ? z : -z;
}

// Sigmoid::Logistic (sigmoid.cpp:19-21): 1 / (1 + exp(-p)), all in float.
XM_HD float xm_logistic(float p) { return XM_FDIV(1.0f, XM_FADD(1.0f, xm_expf(-p))); }

#endif
