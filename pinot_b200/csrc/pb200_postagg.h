// pb200_postagg.h -- THE value of a post-aggregation expression over group-by rows (pb200_post_program,
// include/pinot_b200.h): arithmetic over the FINAL values of a row's aggregations, e.g. SUM(clicks) / SUM(views).
//
// One definition for every place that orders rows by such an expression: the device order pass of pb200_extract.cu, the
// host order of results built on the host (star-tree, FILTER-clause alignment) and the CPU tests.  An operand is the final
// value of one aggregation as a double (having_value, pb200_having.h: COUNT / DISTINCTCOUNT the count, AVG sum / count or
// -inf at count 0, the other functions their double column); a literal is a finite double; every operator is ONE IEEE-754
// double operation rounded to nearest and never contracted into an FMA (t_add .. t_div, pb200_transform.h), so x / 0 is
// +-inf and 0 / 0 is NaN, as in Java.  The program is postfix with the root last; evaluation keeps the pending operands on
// a fixed stack.  Plain C++ when not compiled by nvcc (CPU tests compile it with g++).
#pragma once
#include <math.h>
#include <stdint.h>

#include "pb200_transform.h"

namespace pb200 {

// NULL when `p` is a well-formed program over num_aggs aggregations, else what is wrong with it
inline const char* postagg_validate(const pb200_post_program* p, int num_aggs) {
  if (p->num_nodes < 1 || p->num_nodes > PB200_MAX_POST_NODES) return "post-aggregation program needs 1 to 16 nodes";
  int depth = 0;
  for (int i = 0; i < p->num_nodes; i++) {
    const pb200_post_node& n = p->nodes[i];
    switch (n.op) {
      case PB200_POST_AGG:
        if (n.agg < 0 || n.agg >= num_aggs) return "post-aggregation operand names an aggregation out of range";
        depth++;
        break;
      case PB200_POST_LITERAL:
        if (!isfinite(n.value)) return "post-aggregation literal is not finite";
        depth++;
        break;
      case PB200_POST_NEG:
        if (depth < 1) return "post-aggregation NEG without an operand";
        break;
      case PB200_POST_ADD:
      case PB200_POST_SUB:
      case PB200_POST_MUL:
      case PB200_POST_DIV:
        if (depth < 2) return "post-aggregation operator without its two operands";
        depth--;
        break;
      default:
        return "post-aggregation node of unknown type";
    }
  }
  return depth == 1 ? nullptr : "post-aggregation program does not reduce to one value";
}

// The value of a validated program for one row; value(a) = final value of aggregation a (having_value).
template <class Value>
PB200_HD double postagg_eval(const pb200_post_program& p, Value&& value) {
  double st[PB200_MAX_POST_NODES];
  int top = 0;
  for (int i = 0; i < p.num_nodes; i++) {
    const pb200_post_node& n = p.nodes[i];
    switch (n.op) {
      case PB200_POST_AGG: st[top++] = value(n.agg); break;
      case PB200_POST_LITERAL: st[top++] = n.value; break;
      case PB200_POST_NEG: st[top - 1] = -st[top - 1]; break;
      case PB200_POST_ADD: --top; st[top - 1] = t_add(st[top - 1], st[top]); break;
      case PB200_POST_SUB: --top; st[top - 1] = t_sub(st[top - 1], st[top]); break;
      case PB200_POST_MUL: --top; st[top - 1] = t_mul(st[top - 1], st[top]); break;
      default: --top; st[top - 1] = t_div(st[top - 1], st[top]); break;
    }
  }
  return st[0];
}

}  // namespace pb200
