// pb200_having.h -- THE predicate of HAVING over group-by rows (pb200_having, include/pinot_b200.h).
//
// One definition for every place that filters rows by HAVING: the device keep-bitmap kernel of pb200_extract.cu, the host
// filter of results built on the host (star-tree, FILTER-clause alignment) and the CPU tests.  A leaf compares the FINAL
// value of one aggregation, as a double:
//   COUNT, DISTINCTCOUNT      the count / set size (the long column; exact below 2^53)
//   AVG                       sum / count, -inf when the count is 0
//   every other function      the double column (MIN / MAX of a group without rows: +inf / -inf)
// with Java's <, <=, ==: a NaN value matches only NEQ (and so NOT IN), -0.0 equals 0.0, +-inf compare as usual.  That is
// the rule of predicates on raw values, NOT the Double.compare order ORDER BY uses (pb200_order.h): HAVING is a value
// predicate, not an order.  NOT negates its operand's outcome, so NOT (x > 1) holds for a NaN x.  The tree is postfix with
// the root last; evaluation keeps one bool per pending operand on a fixed stack.  Plain C++ when not compiled by nvcc
// (CPU tests compile it with g++).
#pragma once
#include <math.h>
#include <stdint.h>

#include "pb200_aggfn.h"

namespace pb200 {

// raw_flags layout of pb200_filter_node
enum { HAVING_LO_UNBOUNDED = 1, HAVING_HI_UNBOUNDED = 2, HAVING_LO_EXCLUSIVE = 4, HAVING_HI_EXCLUSIVE = 8 };

// final value of an aggregation of function fn from a row's double and long columns
PB200_HD double having_value(int fn, double dv, int64_t lv) {
  if (fn == PB200_AGG_COUNT || fn == PB200_AGG_DISTINCTCOUNT) return (double)lv;
  if (fn == PB200_AGG_AVG) return lv ? dv / (double)lv : -(double)INFINITY;
  return dv;
}

PB200_HD bool having_leaf(const pb200_having_node& n, double v) {
  if (n.op == PB200_HAVING_EQ) return v == n.lo;
  if (n.op == PB200_HAVING_NEQ) return !(v == n.lo);
  const bool lo_ok = (n.flags & HAVING_LO_UNBOUNDED) || ((n.flags & HAVING_LO_EXCLUSIVE) ? v > n.lo : v >= n.lo);
  const bool hi_ok = (n.flags & HAVING_HI_UNBOUNDED) || ((n.flags & HAVING_HI_EXCLUSIVE) ? v < n.hi : v <= n.hi);
  return lo_ok && hi_ok;
}

// NULL when `h` is a well-formed tree over num_aggs aggregations, else what is wrong with it.  A RANGE needs at least one
// bound, so that a NaN value never matches one.
inline const char* having_validate(const pb200_having* h, int num_aggs) {
  if (h->num_nodes < 1 || h->num_nodes > PB200_MAX_HAVING_NODES) return "HAVING needs 1 to 32 nodes";
  int depth = 0;
  for (int i = 0; i < h->num_nodes; i++) {
    const pb200_having_node& n = h->nodes[i];
    switch (n.op) {
      case PB200_HAVING_AND:
      case PB200_HAVING_OR:
        if (n.num_children < 1 || n.num_children > depth) return "HAVING AND / OR node without its operands";
        depth -= n.num_children - 1;
        break;
      case PB200_HAVING_NOT:
        if (depth < 1) return "HAVING NOT node without an operand";
        break;
      case PB200_HAVING_RANGE:
      case PB200_HAVING_EQ:
      case PB200_HAVING_NEQ:
        if (n.agg < 0 || n.agg >= num_aggs) return "HAVING leaf names an aggregation out of range";
        if (n.op == PB200_HAVING_RANGE) {
          if ((n.flags & ~15) || (n.flags & 3) == 3) return "HAVING RANGE leaf needs a bound and known flags";
          if ((!(n.flags & HAVING_LO_UNBOUNDED) && isnan(n.lo)) || (!(n.flags & HAVING_HI_UNBOUNDED) && isnan(n.hi)))
            return "HAVING bound is NaN";
        } else if (isnan(n.lo)) {
          return "HAVING bound is NaN";
        }
        depth++;
        break;
      default:
        return "HAVING node of unknown type";
    }
  }
  return depth == 1 ? nullptr : "HAVING tree does not reduce to one root";
}

// The tree's outcome for one row of a validated tree; value(a) = final value of aggregation a (having_value).
// The stack is one 32-bit word: bit i holds pending operand i (a tree has at most 32 nodes, so at most 32 operands), bits
// at and above `top` stay 0.
template <class Value>
PB200_HD bool having_eval(const pb200_having& h, Value&& value) {
  uint32_t st = 0;
  int top = 0;
  for (int i = 0; i < h.num_nodes; i++) {
    const pb200_having_node& n = h.nodes[i];
    if (n.op == PB200_HAVING_AND || n.op == PB200_HAVING_OR) {
      top -= n.num_children;
      const uint32_t m = (uint32_t)(((1ull << n.num_children) - 1ull) << top);
      const bool r = n.op == PB200_HAVING_AND ? (st & m) == m : (st & m) != 0u;
      st = (st & ~m) | ((uint32_t)r << top);
      top++;
    } else if (n.op == PB200_HAVING_NOT) {
      st ^= 1u << (top - 1);
    } else {
      st |= (uint32_t)having_leaf(n, value(n.agg)) << top;
      top++;
    }
  }
  return (st & 1u) != 0u;
}

}  // namespace pb200
