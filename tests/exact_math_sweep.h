// tests/exact_math_sweep.h — what the sweeps of cmix_b200/csrc/exact_math.h evaluate, shared by its host build
// (exact_math_sweep.cpp, g++ -ffp-contract=off) and its device build (exact_math_sweep.cu, nvcc for sm_90a), so that
// both sides evaluate and checksum the same way (tests/test_exact_math_device.py).
#ifndef CMIXB200_EXACT_MATH_SWEEP_H
#define CMIXB200_EXACT_MATH_SWEEP_H

#include "../cmix_b200/csrc/exact_math.h"

enum {
  XS_FUNCS = 4,        // xm_expf, xm_expm1f, xm_tanhf, xm_logistic, in this order
  XS_SUB_LOG2 = 16,    // one checksum per function and block of 2^16 consecutive input bit patterns
};

// The result bits of function f at input bits u. Every NaN counts as one value: the device's arithmetic returns the
// canonical NaN where x86 keeps the operand's payload, and nothing downstream reads a payload.
XM_HD uint32_t xs_eval(uint32_t u, int f) {
  const float x = XM_U2F(u);
  float y;
  if (f == 0) y = xm_expf(x);
  else if (f == 1) y = xm_expm1f(x);
  else if (f == 2) y = xm_tanhf(x);
  else y = xm_logistic(x);
  const uint32_t r = XM_F2U(y);
  return (r & 0x7fffffffu) > 0x7f800000u ? 0x7fc00000u : r;
}

// splitmix64's finaliser of (input, result). A block's checksum is the wrapping sum over its inputs, so it does not
// depend on the order in which threads add, and one changed result changes it.
XM_HD uint64_t xs_hash(uint32_t u, uint32_t r) {
  uint64_t z = (((uint64_t)u << 32) | r) + 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

#endif
