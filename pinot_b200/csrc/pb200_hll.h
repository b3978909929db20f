// pb200_hll.h -- DISTINCTCOUNTHLL from DISTINCTCOUNT's dictId bitsets (DESIGN.md section 3.17).
//
// The registers of a HyperLogLog depend only on the set S of distinct values it was offered, so the estimate of a bitset
// row is a function of the set it names: every member's 32-bit hash (computed once per dictionary entry, pb200_hll.cu)
// gives a register index j and a rank r, the registers keep the largest rank, and the estimate follows from them.  The
// hash, the offer step and the estimate restate stream-lib's MurmurHash.hash(Object) / HyperLogLog.offerHashed /
// HyperLogLog.cardinality, which Pinot's DistinctCountHLLAggregationFunction uses; all int arithmetic wraps mod 2^32.
// The estimate is exact on the device: registerSum * 2^(33 - p) is an integer below 2^34 (summed in a u64 in any order),
// alpha * m^2 and the m possible linear-counting results are computed on the host (hll_alpha_mm, hll_linear_table), and
// the rest is one IEEE division, one multiplication and an exact Math.round.
// The arithmetic is plain C++ when not compiled by nvcc: the CPU tests run this same code (tests/hll_probe).
#pragma once
#include <math.h>
#include <stdint.h>

#include "pb200_aggfn.h"

namespace pb200 {

// whether every aggregation that reads the set held by aggregation b's bitset is a DISTINCTCOUNTHLL (fns: PB200_AGG_*,
// ds_rep: ScanPlan::ds_rep; a DISTINCTCOUNT reads its own bitset)
inline bool hll_only_set_of(const int* fns, const int* ds_rep, int n, int b) {
  for (int x = 0; x < n; x++)
    if ((ds_rep[x] == b || (x == b && fns[x] == PB200_AGG_DISTINCTCOUNT)) && !is_hll_fn(fns[x])) return false;
  return true;
}

constexpr int kHllDefaultLog2m = 8;   // DistinctCountHLLAggregationFunction's DEFAULT_HYPERLOGLOG_LOG2M
constexpr int kHllMinLog2m = 4, kHllMaxLog2m = 12;   // accelerated; the reference accepts 0..30
constexpr long long kHllSaturated = 0x7FFFFFFFFFFFFFFFll;   // Math.round(+inf)

// MurmurHash.hashLong: a long's two 32-bit halves, low first
PB200_HD uint32_t hll_hash_long(uint64_t data) {
  const uint32_t m = 0x5bd1e995u;
  uint32_t h = 0;
  uint32_t k = (uint32_t)data * m;
  k ^= k >> 24;
  h ^= k * m;
  k = (uint32_t)(data >> 32) * m;
  k ^= k >> 24;
  h *= m;
  h ^= k * m;
  h ^= h >> 13;
  h *= m;
  h ^= h >> 15;
  return h;
}

// MurmurHash.hash(byte[], length, seed): little-endian 4-byte blocks, then the 1..3 tail bytes SIGN-extended (Java's
// byte), unlike C MurmurHash2 for bytes >= 0x80
PB200_HD uint32_t hll_hash_bytes(const unsigned char* b, int len, uint32_t seed) {
  const uint32_t m = 0x5bd1e995u;
  uint32_t h = seed ^ (uint32_t)len;
  const int blocks = len >> 2;
  for (int i = 0; i < blocks; i++) {
    uint32_t k = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
    k *= m;
    k ^= k >> 24;
    k *= m;
    h *= m;
    h ^= k;
  }
  const int left = len & 3;
  if (left) {
    if (left >= 3) h ^= (uint32_t)(int32_t)(int8_t)b[len - 3] << 16;
    if (left >= 2) h ^= (uint32_t)(int32_t)(int8_t)b[len - 2] << 8;
    h ^= (uint32_t)(int32_t)(int8_t)b[len - 1];
    h *= m;
  }
  h ^= h >> 13;
  h *= m;
  h ^= h >> 15;
  return h;
}

// MurmurHash.hash(Object) of a dictionary value of a numeric stored type, given as its raw bits: INT and FLOAT
// (floatToRawIntBits) are sign-extended to a long, LONG and DOUBLE (doubleToRawLongBits) are the long
PB200_HD uint32_t hll_hash_value(int stored_type, uint64_t raw) {
  if (stored_type == PB200_INT || stored_type == PB200_FLOAT) return hll_hash_long((uint64_t)(int64_t)(int32_t)(uint32_t)raw);
  return hll_hash_long(raw);
}

// Whether b[0, len) is well-formed UTF-8 (no overlong forms, no surrogates, nothing above U+10FFFF): the bytes Java's
// new String(bytes, UTF_8).getBytes(UTF_8) gives back unchanged.  Other bytes would be hashed as U+FFFD by the reference.
PB200_HD bool hll_utf8_valid(const unsigned char* b, int len) {
  int i = 0;
  while (i < len) {
    const unsigned c = b[i];
    int n;
    unsigned lo = 0x80, hi = 0xBF;   // the allowed range of the second byte
    if (c < 0x80) { i++; continue; }
    if (c >= 0xC2 && c <= 0xDF) n = 1;
    else if (c >= 0xE0 && c <= 0xEF) { n = 2; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
    else if (c >= 0xF0 && c <= 0xF4) { n = 3; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
    else return false;
    if (i + n >= len) return false;   // truncated sequence
    for (int k = 1; k <= n; k++) {
      const unsigned x = b[i + k];
      if (k == 1 ? (x < lo || x > hi) : (x < 0x80 || x > 0xBF)) return false;
    }
    i += n + 1;
  }
  return true;
}

PB200_HD int hll_clz(uint32_t x) {
#ifdef __CUDA_ARCH__
  return __clz((int)x);
#else
  return x ? __builtin_clz(x) : 32;
#endif
}

// HyperLogLog.offerHashed: register j = x >>> (32 - p), rank r = numberOfLeadingZeros((x << p) | (1 << (p - 1)) + 1) + 1
// (Java's precedence puts the + 1 inside the OR operand), 1 <= r <= 33 - p
PB200_HD uint32_t hll_index(uint32_t x, int p) { return x >> (32 - p); }
PB200_HD uint32_t hll_rank(uint32_t x, int p) { return (uint32_t)hll_clz((x << p) | ((1u << (p - 1)) + 1u)) + 1u; }

// one register's term of registerSum = sum 1.0 / (1 << reg[j]), scaled by 2^(33 - p): an integer
PB200_HD unsigned long long hll_term(uint32_t reg, int p) { return 1ull << (33 - p - (int)reg); }

// Math.round of a finite x >= 0: floor(x + 1/2) taken exactly (x - floor(x) is exact), saturating at Long.MAX_VALUE
PB200_HD long long hll_round(double x) {
  if (!(x < 9223372036854775807.0)) return kHllSaturated;
  const double f = floor(x);
  return (long long)f + (x - f >= 0.5 ? 1 : 0);
}

// HyperLogLog.cardinality from the registers' scaled sum and the number of zero registers.  alpha_mm = hll_alpha_mm(p);
// linear[z] = Math.round(m * Math.log(m / z)) for z = 0..m (hll_linear_table; z = 0 gives Long.MAX_VALUE).
PB200_HD long long hll_estimate(unsigned long long scaled_sum, uint32_t zeros, int p, double alpha_mm, const long long* linear) {
  const int m = 1 << p;
  const double register_sum = ldexp((double)scaled_sum, -(33 - p));   // exact: scaled_sum < 2^34
#ifdef __CUDA_ARCH__
  const double estimate = __dmul_rn(alpha_mm, __ddiv_rn(1.0, register_sum));
#else
  const double estimate = alpha_mm * (1.0 / register_sum);
#endif
  if (estimate <= 2.5 * m) return linear[zeros];
  return hll_round(estimate);
}

// ---- host only ----
// HyperLogLog's alphaMM, evaluated left to right in double as the reference does
inline double hll_alpha_mm(int p) {
  const int m = 1 << p;
  switch (p) {
    case 4: return 0.673 * m * m;
    case 5: return 0.697 * m * m;
    case 6: return 0.709 * m * m;
    default: return (0.7213 / (1 + 1.079 / m)) * m * m;
  }
}

// the linear-counting branch's m + 1 possible results: Math.round(m * Math.log(m / (double)zeros)), zeros = 0..m
inline void hll_linear_table(int p, long long* out) {
  const int m = 1 << p;
  out[0] = kHllSaturated;   // log(+inf): Math.round(+inf) is Long.MAX_VALUE
  for (int z = 1; z <= m; z++) out[z] = hll_round(m * log((double)m / (double)z));
}

}  // namespace pb200
