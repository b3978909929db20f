// pb200_distinct_sum.h -- DISTINCTSUM / DISTINCTAVG from DISTINCTCOUNT's dictId bitsets (DESIGN.md section 3.14).
//
// S is the set of distinct stored values a bitset row names.  A qualifying dictionary has every finite value equal to
// j * 2^e with ONE exponent e for the whole dictionary and an integer |j| <= 2^63 (INT / LONG: e = 0, j = the value;
// FLOAT / DOUBLE: see distinct_grid), so the sum of j over S (at most 2^32 members) is exact in an int128.  NaN, +inf
// and -inf members set flags instead.  The final value is that exact sum times 2^e, divided by |S| for DISTINCTAVG,
// rounded ONCE to the nearest double (ties to even), subnormal and overflowing results included.
// The arithmetic is plain C++ when not compiled by nvcc: the CPU tests run this same code (tests/distinct_sum_probe).
#pragma once
#include "pb200_moments.h"

namespace pb200 {

typedef __int128 i128;

// special members of S
enum : uint32_t { DS_NAN = 1, DS_POS_INF = 2, DS_NEG_INF = 4 };

// The state one bitset row finalizes into: u64 words {sum low, sum high, |S|, flags, DISTINCTSUM, DISTINCTAVG} -- the
// int128 sum of j in two's complement, then the two final doubles (bit patterns), rounded by the finalize so that
// extraction, ORDER BY and HAVING only read them.  Group-by: kDsWords words per table entry; aggregation only: kDsWords
// per result and set.
constexpr int kDsWords = 6;
PB200_HD int ds_final_word(int fn) { return fn == PB200_AGG_DISTINCTAVG ? 5 : 4; }

// Decomposes a double into m * 2^x with m an odd integer, |m| < 2^53 (m = 0, x = 0 for +-0.0), so that x is the
// exponent of its lowest set bit.  Finite values only.
PB200_HD void double_parts(double v, long long* m, int* x) {
  unsigned long long b;
  memcpy(&b, &v, 8);
  const int be = (int)((b >> 52) & 0x7FF);
  unsigned long long f = b & ((1ull << 52) - 1);
  if (be) f |= 1ull << 52;
  *x = 0;
  *m = 0;
  if (!f) return;
#ifdef __CUDA_ARCH__
  const int tz = __ffsll((long long)f) - 1;
#else
  const int tz = __builtin_ctzll(f);
#endif
  f >>= tz;
  *x = (be ? be : 1) - 1075 + tz;
  *m = (b >> 63) ? -(long long)f : (long long)f;
}

// One member given as a double: adds its j = v / 2^e to *sum, or returns its flag (0 for a finite member).  The value is
// on the grid (checked when the dictionary was admitted), so the shift is exact.
PB200_HD uint32_t ds_add_double(double v, int e, i128* sum) {
  if (v != v) return DS_NAN;
  if (v == (double)INFINITY) return DS_POS_INF;
  if (v == -(double)INFINITY) return DS_NEG_INF;
  long long m;
  int x;
  double_parts(v, &m, &x);
  if (m) *sum += (i128)m * ((i128)1 << (x - e));
  return 0;
}

// The final value of DISTINCTSUM / DISTINCTAVG (fn) over a row's state: its exact sum of j, |S| and flags, grid exponent e
PB200_HD double distinct_final(int fn, i128 sum, unsigned long long n, uint32_t flags, int e) {
  if ((flags & DS_NAN) || ((flags & DS_POS_INF) && (flags & DS_NEG_INF))) return (double)NAN;
  if (flags & DS_POS_INF) return (double)INFINITY;
  if (flags & DS_NEG_INF) return -(double)INFINITY;
  if (n == 0) return fn == PB200_AGG_DISTINCTAVG ? -(double)INFINITY : 0.0;
  if (sum == 0) return 0.0;
  const bool neg = sum < 0;
  const u128 mag = neg ? (u128)0 - (u128)sum : (u128)sum;
  return round_dyadic(neg, mag, fn == PB200_AGG_DISTINCTAVG ? n : 1ull, e);
}

PB200_HD i128 ds_sum_of(const unsigned long long* st) { return (i128)(((u128)st[1] << 64) | (u128)st[0]); }

// ---- host only ----
// Whether the sorted dictionary `dict` (native values of `stored_type`, `card` entries) qualifies, and its exponent e:
// INT / LONG always (e = 0); FLOAT / DOUBLE when every finite non-zero value is j * 2^e with |j| < 2^63 for the smallest
// exponent e any of them needs (the exponent of the lowest set bit).  NaN, +-inf and +-0.0 never constrain e.
inline bool distinct_grid(int stored_type, const unsigned char* dict, int card, int* e) {
  *e = 0;
  if (stored_type == PB200_INT || stored_type == PB200_LONG) return true;
  if (stored_type != PB200_FLOAT && stored_type != PB200_DOUBLE) return false;
  if (!dict || card <= 0) return false;
  auto at = [&](int i) -> double {
    if (stored_type == PB200_DOUBLE) { double v; memcpy(&v, dict + 8ull * i, 8); return v; }
    float v; memcpy(&v, dict + 4ull * i, 4); return (double)v;
  };
  int lo = 1 << 30;
  for (int i = 0; i < card; i++) {
    const double v = at(i);
    if (!std::isfinite(v) || v == 0.0) continue;
    long long m;
    int x;
    double_parts(v, &m, &x);
    lo = std::min(lo, x);
  }
  if (lo == (1 << 30)) return true;   // no finite non-zero value
  for (int i = 0; i < card; i++) {
    const double v = at(i);
    if (!std::isfinite(v) || v == 0.0) continue;
    long long m;
    int x;
    double_parts(v, &m, &x);
    const unsigned long long a = m < 0 ? 0ull - (unsigned long long)m : (unsigned long long)m;
    if (x - lo + (64 - __builtin_clzll(a)) > 63) return false;   // |j| = |m| * 2^(x - e) must stay below 2^63
  }
  *e = lo;
  return true;
}

}  // namespace pb200
