// pb200_moments.h -- VAR_POP / VAR_SAMP / STDDEV_POP / STDDEV_SAMP over limb dictionaries (DESIGN.md section 3.9).
//
// A column qualifies when every value of its dictionary is c + k * 2^e, c the smallest value, k an integer in [0, 2^32).
// Its limb dictionaries hold, per dictId, K = k, H = k^2 >> 32 and L = k^2 & 0xFFFFFFFF (pb200_moments.cu).  The scan
// sums them as three ordinary INT-dictionary SUMs: a limb word W is read as the INT value W - 2^31 (the device copy of an
// INT dictionary is biased), so each table holds sum(limb) - n * 2^31, exact in int64 for n < 2^32.  From those sums and
// n the variance is computed exactly in 128-bit integers and rounded ONCE:
//   S1 = sum K, S2 = sum H * 2^32 + sum L = sum k^2, N = n * S2 - S1^2 (>= 0, < 2^128 for n < 2^32)
//   VARPOP = N * 2^2e / n^2, VARSAMP = N * 2^2e / (n (n - 1)), STDDEV* = sqrt of the double variance.
// The arithmetic is plain C++ when not compiled by nvcc: the CPU tests run this same code (tests/moments_probe).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#include "pb200_aggfn.h"

namespace pb200 {

typedef unsigned __int128 u128;

// The grid of one dictionary: value = c + k * 2^e.  c is kept exactly as c_mant * 2^c_exp (the C-ABI's form) and, for the
// build kernel, as the column's own type (c_int: INT / LONG, c_dbl: FLOAT / DOUBLE).
struct MomentGrid {
  int32_t stored_type;
  int32_t e;
  long long c_int;
  double c_dbl;
  long long c_mant;
  int32_t c_exp;
  uint32_t k_max;  // k of the largest value
};

// Exact moments of n values: s1 = sum k, s2 = sum k^2
struct Moments {
  unsigned long long n, s1;
  u128 s2;
};

// From the three limb SUM tables of a row (each holds sum(limb) - n * 2^31) and its row count
PB200_HD Moments moments_from_sums(unsigned long long n, long long sum_k, long long sum_h, long long sum_l) {
  const unsigned long long bias = n << 31;  // n < 2^32
  Moments m;
  m.n = n;
  m.s1 = (unsigned long long)sum_k + bias;  // modulo 2^64: the true sum is < 2^64
  const unsigned long long h = (unsigned long long)sum_h + bias, l = (unsigned long long)sum_l + bias;
  m.s2 = ((u128)h << 32) + (u128)l;
  return m;
}

PB200_HD int bitlen128(u128 x) {
  const unsigned long long hi = (unsigned long long)(x >> 64), lo = (unsigned long long)x;
#ifdef __CUDA_ARCH__
  return hi ? 128 - __clzll((long long)hi) : (lo ? 64 - __clzll((long long)lo) : 0);
#else
  return hi ? 128 - __builtin_clzll(hi) : (lo ? 64 - __builtin_clzll(lo) : 0);
#endif
}

// round-to-nearest-even of (neg ? -1 : 1) * num / den * 2^scale (0 < num < 2^128, 0 < den < 2^64), correctly rounded into
// the subnormal range and to +-inf on overflow.  The quotient is developed bit by bit until it holds at least 55
// significant bits (the remainder is the sticky bit); then exactly the bits the result can hold are kept -- 53, or fewer
// where the result is subnormal -- and rounded once.
PB200_HD double round_dyadic(bool neg, u128 num, unsigned long long den, int scale) {
  u128 q = 0, r = 0;
  for (int i = 127; i >= 0; --i) {
    r = (r << 1) | ((num >> i) & 1u);
    q <<= 1;
    if (r >= den) { r -= den; q |= 1u; }
  }
  int len = bitlen128(q), lsb = scale;   // value = (q + r / den) * 2^lsb
  while (len < 55) {
    r <<= 1;
    q <<= 1;
    if (r >= den) { r -= den; q |= 1u; }
    --lsb;
    len = bitlen128(q);
  }
  int sh = len - 53;                           // bits dropped from q
  if (lsb + sh < -1074) sh = -1074 - lsb;      // subnormal: the last kept bit weighs 2^-1074
  double out;
  if (sh > len) {
    out = 0.0;                                 // below half the smallest subnormal
  } else {
    const unsigned long long keep0 = sh >= 128 ? 0ull : (unsigned long long)(q >> sh);
    const u128 low = sh >= 128 ? q : (q & (((u128)1 << sh) - 1u)), half = (u128)1 << (sh - 1);
    unsigned long long keep = keep0;
    if (low > half || (low == half && (r != 0 || (keep & 1ull)))) ++keep;
    if (keep == (1ull << 53)) { keep >>= 1; ++sh; }
    out = ldexp((double)keep, lsb + sh);       // exact, or +inf beyond the largest double
  }
  return neg ? -out : out;
}

// the positive case (VAR / STDDEV)
PB200_HD double div_round(u128 num, unsigned long long den, int scale) { return round_dyadic(false, num, den, scale); }

// The final value of function fn (PB200_AGG_VARPOP .. STDDEVSAMP) over moments m of values on grid exponent e
PB200_HD double moments_final(int fn, const Moments& m, int e) {
  const bool samp = fn == PB200_AGG_VARSAMP || fn == PB200_AGG_STDDEVSAMP;
  if (m.n == 0 || (samp && m.n == 1)) return -(double)INFINITY;
  const u128 N = (u128)m.n * m.s2 - (u128)m.s1 * m.s1;
  const unsigned long long den = samp ? m.n * (m.n - 1) : m.n * m.n;
  const double var = N == 0 ? 0.0 : div_round(N, den, 2 * e);
  return (fn == PB200_AGG_STDDEVPOP || fn == PB200_AGG_STDDEVSAMP) ? sqrt(var) : var;
}

// ---- host only ----
// exponent of the lowest set bit of a finite non-zero double
inline int lowest_bit_exponent(double d) {
  int x;
  const double m = frexp(fabs(d), &x);
  unsigned long long M = (unsigned long long)ldexp(m, 53);
  return x - 53 + __builtin_ctzll(M);
}

// Whether the sorted dictionary `dict` (native values of `stored_type`, `card` entries) is on a 2^32-unit grid, and the
// grid.  Exact: k is computed in double, and c + k * 2^e must give the value back without rounding (TwoSum).
inline bool moments_grid(int stored_type, const unsigned char* dict, int card, MomentGrid* g) {
  if (!dict || card <= 0) return false;
  memset(g, 0, sizeof *g);
  g->stored_type = stored_type;
  if (stored_type == PB200_INT || stored_type == PB200_LONG) {
    long long lo, hi;
    if (stored_type == PB200_INT) {
      int32_t a, b;
      memcpy(&a, dict, 4); memcpy(&b, dict + 4ull * (card - 1), 4);
      lo = a; hi = b;
    } else {
      memcpy(&lo, dict, 8); memcpy(&hi, dict + 8ull * (card - 1), 8);
    }
    const unsigned long long range = (unsigned long long)hi - (unsigned long long)lo;  // exact: both are int64
    if (hi < lo || range >> 32) return false;
    g->c_int = lo; g->c_mant = lo; g->c_exp = 0; g->e = 0; g->k_max = (uint32_t)range;
    return true;
  }
  if (stored_type != PB200_FLOAT && stored_type != PB200_DOUBLE) return false;
  auto at = [&](int i) -> double {
    if (stored_type == PB200_DOUBLE) { double v; memcpy(&v, dict + 8ull * i, 8); return v; }
    float v; memcpy(&v, dict + 4ull * i, 4); return (double)v;
  };
  const double c = at(0);
  int e = 1 << 30;
  for (int i = 0; i < card; i++) {
    const double v = at(i);
    if (!std::isfinite(v)) return false;
    const double d = v - c;
    if (d != 0.0) e = std::min(e, lowest_bit_exponent(d));
  }
  if (e == (1 << 30)) e = 0;  // a single value
  for (int i = 0; i < card; i++) {
    const double v = at(i);
    const double k = ldexp(v - c, -e);
    if (!(k >= 0.0 && k < 4294967296.0) || k != floor(k)) return false;
    const double t = ldexp(k, e), s = c + t;  // TwoSum(c, t): s + err == c + t exactly
    const double bp = s - c, err = (c - (s - bp)) + (t - bp);
    if (s != v || err != 0.0) return false;
    g->k_max = (uint32_t)k;
  }
  g->c_dbl = c; g->e = e;
  if (c == 0.0) { g->c_mant = 0; g->c_exp = 0; }
  else {
    int x;
    const double m = frexp(c, &x);
    long long M = (long long)ldexp(m, 53);
    int ex = x - 53;
    while (!(M & 1)) { M /= 2; ex++; }
    g->c_mant = M; g->c_exp = ex;
  }
  return true;
}

}  // namespace pb200
