// tests/exact_math_sweep.cpp — the host build of cmix_b200/csrc/exact_math.h for tests/test_exact_math_device.py:
// the reference the device build is checked against, and its own exhaustive comparison with glibc.
//   g++ -O2 -std=c++17 -ffp-contract=off -fopenmp -fPIC -shared tests/exact_math_sweep.cpp -o libxs_host.so -lm
#include <math.h>
#include <stddef.h>

#include "exact_math_sweep.h"

// Checksums of blocks first_blk .. first_blk+n_blk-1 (2^16 inputs each): out[b * XS_FUNCS + f].
extern "C" void xs_host_sums(uint32_t first_blk, uint32_t n_blk, uint64_t* out) {
#pragma omp parallel for schedule(dynamic, 1)
  for (long b = 0; b < (long)n_blk; ++b) {
    uint64_t acc[XS_FUNCS] = {0, 0, 0, 0};
    const uint32_t base = (first_blk + (uint32_t)b) << XS_SUB_LOG2;
    for (uint32_t i = 0; i < (1u << XS_SUB_LOG2); ++i)
      for (int f = 0; f < XS_FUNCS; ++f) acc[f] += xs_hash(base | i, xs_eval(base | i, f));
    for (int f = 0; f < XS_FUNCS; ++f) out[b * XS_FUNCS + f] = acc[f];
  }
}

// out[f * n + i]: result bits of function f at input bits in[i].
extern "C" void xs_host_eval(const uint32_t* in, size_t n, uint32_t* out) {
  for (size_t i = 0; i < n; ++i)
    for (int f = 0; f < XS_FUNCS; ++f) out[f * n + i] = xs_eval(in[i], f);
}

// What the reference calls (glibc expf / expm1f / tanhf, Sigmoid::Logistic's 1 / (1 + expf(-x)) in float), laid out
// and NaN-folded as xs_host_eval.
static uint32_t libm_eval(uint32_t u, int f) {
  const float x = XM_U2F(u);
  float y;
  if (f == 0) y = expf(x);
  else if (f == 1) y = expm1f(x);
  else if (f == 2) y = tanhf(x);
  else y = 1.0f / (1.0f + expf(-x));
  const uint32_t r = XM_F2U(y);
  return (r & 0x7fffffffu) > 0x7f800000u ? 0x7fc00000u : r;
}
extern "C" void xs_libm_eval(const uint32_t* in, size_t n, uint32_t* out) {
  for (size_t i = 0; i < n; ++i)
    for (int f = 0; f < XS_FUNCS; ++f) out[f * n + i] = libm_eval(in[i], f);
}

// Host build against glibc over blocks first_blk .. first_blk+n_blk-1: bad[f] counts the differing inputs of function
// f, first[f] is the smallest of them (left as is when there is none).
extern "C" void xs_libm_sweep(uint32_t first_blk, uint32_t n_blk, uint64_t* bad, uint32_t* first) {
#pragma omp parallel for schedule(dynamic, 1)
  for (long b = 0; b < (long)n_blk; ++b) {
    const uint32_t base = (first_blk + (uint32_t)b) << XS_SUB_LOG2;
    for (uint32_t i = 0; i < (1u << XS_SUB_LOG2); ++i)
      for (int f = 0; f < XS_FUNCS; ++f)
        if (xs_eval(base | i, f) != libm_eval(base | i, f)) {
#pragma omp critical
          {
            if (bad[f]++ == 0 || (base | i) < first[f]) first[f] = base | i;
          }
        }
  }
}
