// pb200_order.h -- THE order of ORDER BY ... LIMIT over group-by rows (pb200_order_by, include/pinot_b200.h).
//
// One definition for every place that orders rows: the device sort of pb200_extract.cu and the host sort of results built
// on the host (star-tree, FILTER-clause alignment).  An item compares the FINAL value of its column:
//   COUNT, DISTINCTCOUNT      the count / set size (the result's long column)
//   SUM, MIN, MAX             the double (MIN / MAX of a group without rows: +inf / -inf)
//   AVG                       sum / count, -inf when the count is 0
//   group-by column           its dictId (dictId order is value order within one dictionary / domain)
// Doubles compare like Java's Double.compare: -0.0 before 0.0, and every NaN (a SUM over +inf and -inf rows, a MAX over a
// NaN entry, whichever NaN bits the hardware or the dictionary produced) is one value after +inf.  Each item becomes an
// unsigned key whose ascending order is the item's order; rows equal on every item are ordered by their group-key
// values, ascending, in GROUP BY column order.  Plain C++ when not compiled by nvcc (CPU tests compile it with g++).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "pb200_aggfn.h"

namespace pb200 {

// how an item's final value is read from a row's (double, long) pair
enum OrderCmp { ORDER_CMP_LONG = 0, ORDER_CMP_DOUBLE = 1, ORDER_CMP_AVG = 2 };

PB200_HD int order_cmp_of(int fn) {
  return fn == PB200_AGG_AVG ? ORDER_CMP_AVG : (fn == PB200_AGG_COUNT || fn == PB200_AGG_DISTINCTCOUNT) ? ORDER_CMP_LONG : ORDER_CMP_DOUBLE;
}

// Double.compare order as unsigned order: a NaN is the canonical NaN (doubleToLongBits), then negative values have all
// bits flipped, the others only the sign bit
PB200_HD uint64_t double_order_bits(double v) {
  uint64_t u;
  memcpy(&u, &v, 8);
  if ((u & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull) u = 0x7FF8000000000000ull;
  return (u >> 63) ? ~u : (u | (1ull << 63));
}

// (item, row) -> key.  dv / lv are the row's double and long columns of the item's aggregation (for a group-by column:
// lv = its dictId); mask = the key bits in use (all ones for doubles); a DESC item flips them.
PB200_HD uint64_t order_key(int cmp, bool descending, uint64_t mask, double dv, int64_t lv) {
  uint64_t k;
  if (cmp == ORDER_CMP_LONG) k = (uint64_t)lv;
  else if (cmp == ORDER_CMP_DOUBLE) k = double_order_bits(dv);
  else k = double_order_bits(lv ? dv / (double)lv : -(double)INFINITY);
  return descending ? k ^ mask : k;
}

}  // namespace pb200
