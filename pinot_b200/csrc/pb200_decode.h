// pb200_decode.h -- how an aggregation's state becomes the values of a result row: {double, long, dictId}.  One decoder
// for both result routes: a GROUP BY result's table entries (the extraction, ORDER BY and HAVING kernels,
// pb200_extract.cu) and an aggregation-only result's one-entry tables (decoded on the host from the pinned copy of the
// call's accumulator block, pb200_api.cu).  An aggregation-only result is a GROUP BY result with one entry and no key.
// Plain C++ when not compiled by nvcc (tests/decode_probe compiles it with g++).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "pb200_desc.h"
#include "pb200_distinct_sum.h"
#include "pb200_expr.h"

namespace pb200 {

// Where aggregation a's state lives: entry g of every table below.  The finalize stages after the scan write the same
// tables (PERCENTILE, FIRST/LASTWITHTIME, DISTINCTSUM / DISTINCTAVG, DISTINCTCOUNTHLL, expressions).
struct AggSource {
  int32_t fn, vk;                    // PB200_AGG_*, VAL_*
  void* src;                         // SUM / AVG: i64 or f64 sums (sum_in_double); MIN / MAX: u32 entries (pb200_desc.h
                                     // max_offset); PERCENTILE: the selected dictId; FIRST/LASTWITHTIME: the data dictId
                                     // (~0: no row); NULL otherwise
  const void* dict;                  // dictionary for the value of a dictId (NULL: the id itself is the value)
  uint32_t dict_bias;                // XOR-ed into INT dictionary values: the device copy is biased, the host copy is not
  int32_t counted;                   // the decoder's `cnt` is the entry's row count (a table without COUNT / AVG or a
                                     // count carrier has none: cnt is 0 there)
  int32_t pack_shift;                // SUM / AVG in a count-carrying table (pb200_plan.cpp): entries hold
  long long pack_vmin;               // sum(value - pack_vmin) + count << pack_shift; 0: a plain sum table
  uint32_t* pct_n;                   // PERCENTILE: values per entry
  long long* wt_time;                // FIRST/LASTWITHTIME: the winning row's time value per entry
  long long* mom[3];                 // VAR / STDDEV: the K, H, L limb sums per entry (pb200_moments.h) ...
  int32_t mom_e;                     // ... and the grid exponent of the column
  unsigned long long* ds;            // DISTINCTSUM / DISTINCTAVG: the finalized state, kDsWords u64 per entry
  long long* hll;                    // DISTINCTCOUNTHLL: the estimate per entry
  unsigned long long* xkey;          // expression MIN / MAX (pb200_expr.cu): the Double.compare key per entry
};

// value of dictId x (raw INT: of the order-preserving encoding x)
PB200_HD double dict_value(const AggSource& s, uint32_t x) {
  const int vk = s.vk;
  if (vk == VAL_RAW_I32) return (double)(int32_t)(x ^ 0x80000000u);
  if (!s.dict) return (double)x;
  if (vk == VAL_DICT_I32) return (double)(int32_t)(static_cast<const uint32_t*>(s.dict)[x] ^ s.dict_bias);
  if (vk == VAL_DICT_I64) return (double)static_cast<const long long*>(s.dict)[x];
  if (vk == VAL_DICT_F32) return (double)static_cast<const float*>(s.dict)[x];
  return static_cast<const double*>(s.dict)[x];
}

// An entry whose count is known and zero has no row.  (A raw INT MIN / MAX entry spans all of u32: only the count tells
// "no row" there.  An entry of a GROUP BY table exists only with a row, so its count, when known, is above zero.)
PB200_HD bool no_row(const AggSource& s, unsigned long long cnt) { return s.counted && cnt == 0; }

// Entry g of aggregation s as a result row holds it: double value, long (count, PERCENTILE values, time value, estimate),
// MIN / MAX / PERCENTILE / WITHTIME dictId (-1: none).  Without a row MIN / MAX give +-inf, PERCENTILE and WITHTIME -inf.
// DISTINCTCOUNT leaves zeros: the set sizes come from the decoded sets.  mom_row: VAR / STDDEV write the exact
// {s1, s2 low, s2 high} there (NULL: not written).
PB200_HD void agg_values(const AggSource& s, long long g, unsigned long long cnt, double& dv, long long& lv, int32_t& id,
                         unsigned long long* mom_row) {
  const int fn = s.fn, vk = s.vk;
  dv = 0.0; lv = 0; id = -1;
  if (fn == PB200_AGG_COUNT) { lv = (long long)cnt; dv = (double)cnt; }
  else if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) {
    if (s.pack_shift) {  // low field = sum(value - vmin): exact integer arithmetic, then to double like every sum
      const unsigned long long f = static_cast<const unsigned long long*>(s.src)[g] & ((1ull << s.pack_shift) - 1ull);
      dv = (double)((long long)f + (long long)cnt * s.pack_vmin);
    } else {
      dv = sum_in_double(vk) ? static_cast<const double*>(s.src)[g] : (double)static_cast<const long long*>(s.src)[g];
    }
    lv = (long long)cnt;
  } else if (s.xkey) {
    dv = expr_key_value(fn, s.xkey[g]);
  } else if (fn == PB200_AGG_MIN || fn == PB200_AGG_MAX) {
    const uint32_t t = static_cast<const uint32_t*>(s.src)[g];
    const bool empty = no_row(s, cnt) || (vk != VAL_RAW_I32 && (fn == PB200_AGG_MIN ? t == 0xFFFFFFFFu : t == 0u));
    if (empty) dv = fn == PB200_AGG_MIN ? INFINITY : -INFINITY;
    else {
      const uint32_t x = fn == PB200_AGG_MIN ? t : t - max_offset(vk);
      id = (int32_t)x;
      dv = dict_value(s, x);
    }
  } else if (fn == PB200_AGG_PERCENTILE) {  // finalized from the histogram (pb200_percentile.cu): dictId, ~0 = no row
    const uint32_t x = static_cast<const uint32_t*>(s.src)[g];
    lv = s.pct_n[g];
    if (no_row(s, cnt) || x == ~0u) dv = -INFINITY;
    else { id = (int32_t)x; dv = dict_value(s, x); }
  } else if (fn == PB200_AGG_FIRSTWITHTIME || fn == PB200_AGG_LASTWITHTIME) {  // finalized (pb200_withtime.cu): ~0 = no row
    const uint32_t x = static_cast<const uint32_t*>(s.src)[g];
    if (no_row(s, cnt) || x == ~0u) dv = -INFINITY;
    else { id = (int32_t)x; dv = dict_value(s, x); lv = s.wt_time[g]; }
  } else if (is_moments_fn(fn)) {  // exact moments from the entry's limb sums and count, rounded once
    const Moments m = moments_from_sums(cnt, s.mom[0][g], s.mom[1][g], s.mom[2][g]);
    if (mom_row) { mom_row[0] = m.s1; mom_row[1] = (unsigned long long)m.s2; mom_row[2] = (unsigned long long)(m.s2 >> 64); }
    dv = moments_final(fn, m, s.mom_e);   // after the row's stores: the pointer is not live across the rounding
    lv = (long long)cnt;
  } else if (is_distinct_value_fn(fn)) {  // rounded once by the finalize (pb200_distinct_sum.cu)
    const unsigned long long* st = s.ds + (size_t)g * kDsWords;
    const long long w = (long long)st[ds_final_word(fn)];
    memcpy(&dv, &w, 8);
    lv = (long long)st[2];
  } else if (is_hll_fn(fn)) {   // the finalize's estimate (pb200_hll.cu), in both columns
    lv = s.hll[g];
    dv = (double)lv;
  }
}

}  // namespace pb200
