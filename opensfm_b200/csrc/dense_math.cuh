// Arithmetic the dense engine shares in definition with its oracle (oracle/dense_oracle.cpp restates it): the
// counter-based generator, and exp / log built from + - * / alone, so that every variate and everything it passes
// through is the same bit pattern on the device and on the host.  dense.cu is compiled with -fmad=false.
#pragma once
#include <cstdint>

namespace osfm {
namespace dense {

#define DN_HD __host__ __device__ __forceinline__

// Philox4x32-10 (Salmon et al., SC'11): counter c, key k.
struct U4 {
  uint32_t x[4];
};

DN_HD uint32_t dn_mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
  const uint64_t p = (uint64_t)a * (uint64_t)b;
  *hi = (uint32_t)(p >> 32);
  return (uint32_t)p;
}

DN_HD U4 philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, hi1;
    const uint32_t lo0 = dn_mulhilo(0xD2511F53u, c0, &hi0);
    const uint32_t lo1 = dn_mulhilo(0xCD9E8D57u, c2, &hi1);
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  U4 o;
  o.x[0] = c0;
  o.x[1] = c1;
  o.x[2] = c2;
  o.x[3] = c3;
  return o;
}

DN_HD uint64_t dn_bits(double x) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(x);
#else
  uint64_t b;
  __builtin_memcpy(&b, &x, 8);
  return b;
#endif
}
DN_HD double dn_from_bits(uint64_t b) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)b);
#else
  double x;
  __builtin_memcpy(&x, &b, 8);
  return x;
#endif
}

constexpr double DN_LN2 = 0.6931471805599453;
constexpr double DN_INV_LN2 = 1.4426950408889634;
constexpr double DN_SQRT2 = 1.4142135623730951;

// log x for a positive normal x: x = m 2^e with m in [sqrt(1/2), sqrt(2)], then 2 atanh((m - 1) / (m + 1)) by its
// series to s^27, about 1e-20 relative.
DN_HD double dn_log(double x) {
  const uint64_t b = dn_bits(x);
  int e = (int)((b >> 52) & 0x7ff) - 1023;
  double m = dn_from_bits((b & 0x000FFFFFFFFFFFFFull) | (1023ull << 52));
  if (m > DN_SQRT2) {
    m = m * 0.5;
    e = e + 1;
  }
  const double s = (m - 1.0) / (m + 1.0);
  const double s2 = s * s;
  double term = s, sum = 0.0;
  for (int k = 0; k < 14; ++k) {
    sum = sum + term / (double)(2 * k + 1);
    term = term * s2;
  }
  return 2.0 * sum + (double)e * DN_LN2;
}

// exp x: x = k ln2 + r with |r| <= ln2 / 2 + ulp, r's Taylor series to r^20 by Horner, times 2^k.
DN_HD double dn_exp(double x) {
  if (x > 700.0) return dn_from_bits(0x7FF0000000000000ull);
  if (x < -700.0) return 0.0;
  const double q = x * DN_INV_LN2;
  const int k = (int)(q >= 0.0 ? q + 0.5 : q - 0.5);
  const double r = x - (double)k * DN_LN2;
  double p = 1.0;
  for (int n = 20; n >= 1; --n) p = 1.0 + r * p / (double)n;
  return p * dn_from_bits((uint64_t)(k + 1023) << 52);
}

// uniform float in [0, 1) from the top 24 bits
DN_HD float dn_unit(uint32_t x) { return (float)(x >> 8) * 5.9604644775390625e-8f; }
// uniform integer in [lo, lo + n) by multiply-shift
DN_HD int dn_index(uint32_t x, int lo, int n) { return lo + (int)(((uint64_t)x * (uint64_t)n) >> 32); }
// uniform double in [-1, 1), exact
DN_HD double dn_signed(uint32_t x) { return (double)(int32_t)x * 4.656612873077392578125e-10; }

// Standard normal by the Marsaglia polar method: attempt a uses words 0 and 1 of philox(pixel, pass, draw, a);
// the first accepted pair's u gives the variate.
DN_HD float dn_normal(uint32_t pixel, uint32_t pass, uint32_t draw, uint32_t k0, uint32_t k1) {
  for (uint32_t a = 0;; ++a) {
    const U4 r = philox(pixel, pass, draw, a, k0, k1);
    const double u = dn_signed(r.x[0]), v = dn_signed(r.x[1]);
    const double s = u * u + v * v;
    if (s >= 1.0 || s == 0.0) continue;
    return (float)(u * sqrt(-2.0 * dn_log(s) / s));
  }
}

// Draw numbers within one pass of one pixel (the counter's third word).
constexpr uint32_t DRAW_INIT = 0;           // words: log-depth, normal x, normal y, view
constexpr uint32_t DRAW_PERTURB = 1;        // + 3 k + {0 depth, 1 normal x, 2 normal y}, k < 6
constexpr uint32_t DRAW_OTHER_VIEW = 32;    // attempt a: word a % 4 of philox(..., a / 4)

}  // namespace dense
}  // namespace osfm
