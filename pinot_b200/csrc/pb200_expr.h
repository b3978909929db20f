// pb200_expr.h -- multi-column expression programs (DESIGN.md section 3.15): the arithmetic grammar of the single-column
// transforms (pb200_transform.h) over two or more column leaves, evaluated once per matched row by pb200_expr.cu.  CPU
// tests compile this header with g++ and run the same code.
//
// A program is POSTFIX like a pb200_transform_op program.  A PB200_T_COLUMN leaf's `i` names the column: a column id in
// the C-ABI (pb200_expr_program), the leaf index (0 .. kExprMaxLeaves - 1) in the device program.  Every leaf value is a
// double (INT / LONG converted, rounded to nearest beyond 2^53), every operation one IEEE-754 round-to-nearest step
// (t_add / t_sub / t_mul / t_div: never contracted into an FMA), MOD is fmod, x / 0 is +-inf or NaN.
#pragma once
#include "pb200_transform.h"

namespace pb200 {

constexpr int kExprMaxLeaves = 8;   // column leaves per expression (the same column twice counts twice)
constexpr int kExprMaxCols = 6 * kExprMaxLeaves;  // distinct leaf columns of one query (6 aggregations)

PB200_HD bool expr_op_ok(int op) {
  return op == PB200_T_COLUMN || op == PB200_T_LONG_LITERAL || op == PB200_T_DOUBLE_LITERAL || (op >= PB200_T_PLUS && op <= PB200_T_ABS);
}

// Checks a program (host side, before any launch).  Returns 0 with the number of column leaves in *leaves, or a PB200_E_*
// code with a message in `why`: PB200_E_INVALID for a malformed program, PB200_E_UNSUPPORTED for a well-formed one outside
// the supported set (a time function, fewer than two or more than kExprMaxLeaves column leaves, more than 16 operations).
inline int expr_check(const pb200_transform_op* ops, int n, int* leaves, const char** why) {
  if (!ops || n <= 0 || n > kTransformMaxProgram) { *why = "program length out of range"; return PB200_E_INVALID; }
  int sp = 0, columns = 0, operations = 0;
  bool time_fn = false;
  for (int k = 0; k < n; k++) {
    const pb200_transform_op& o = ops[k];
    const int ar = o.op >= PB200_T_COLUMN && o.op <= PB200_T_TOEPOCH_ROUNDED ? transform_arity(o.op) : -1;
    if (ar < 0 || o.reserved != 0) { *why = "unknown operation"; return PB200_E_INVALID; }
    if (sp < ar) { *why = "operand stack underflow"; return PB200_E_INVALID; }
    if (o.op == PB200_T_COLUMN && o.i < 0) { *why = "negative column id"; return PB200_E_INVALID; }
    time_fn |= !expr_op_ok(o.op);
    columns += o.op == PB200_T_COLUMN;
    operations += ar > 0;
    sp += 1 - ar;
  }
  if (sp != 1) { *why = "program does not leave exactly one value"; return PB200_E_INVALID; }
  if (time_fn) { *why = "time functions are not accelerated inside an expression over two or more columns"; return PB200_E_UNSUPPORTED; }
  if (columns < 2) { *why = "an expression over several columns needs two or more column leaves"; return PB200_E_UNSUPPORTED; }
  if (columns > kExprMaxLeaves) { *why = "more than 8 column leaves in one expression"; return PB200_E_UNSUPPORTED; }
  if (operations > kTransformMaxOps) { *why = "more than 16 operations"; return PB200_E_UNSUPPORTED; }
  *leaves = columns;
  return PB200_OK;
}

// A CHECKED device program (column leaf i reads leaf[i]) on one row's leaf values.
PB200_HD double expr_eval(const pb200_transform_op* ops, int n, const double* leaf) {
  double D[kTransformMaxProgram];
  int sp = 0;
  for (int k = 0; k < n; k++) {
    const pb200_transform_op o = ops[k];
    switch (o.op) {
      case PB200_T_COLUMN: D[sp++] = leaf[o.i]; continue;
      case PB200_T_LONG_LITERAL: D[sp++] = (double)o.i; continue;
      case PB200_T_DOUBLE_LITERAL: D[sp++] = o.d; continue;
      default: break;
    }
    const int ar = transform_arity(o.op);
    sp -= ar;
    const double x = D[sp], y = ar == 2 ? D[sp + 1] : 0.0;
    double r;
    switch (o.op) {
      case PB200_T_PLUS: r = t_add(x, y); break;
      case PB200_T_MINUS: r = t_sub(x, y); break;
      case PB200_T_TIMES: r = t_mul(x, y); break;
      case PB200_T_DIVIDE: r = t_div(x, y); break;
      case PB200_T_MOD: r = fmod(x, y); break;
      case PB200_T_FLOOR: r = floor(x); break;
      case PB200_T_CEIL: r = ceil(x); break;
      default: r = fabs(x);
    }
    D[sp++] = r;
  }
  return D[0];
}

// A predicate on an expression's value (DESIGN.md section 3.16), the rule of the reference's raw-value predicate evaluators
// for a DOUBLE: Java's <, > and == against the literal's double.  So NaN matches only NEQ and NOT IN (and no range, not
// even an unbounded one), and 0.0 matches both zeros.  `flags` carries pb200_filter_node.raw_flags' bits (bit0 lower
// unbounded, bit1 upper unbounded, bit2 lower exclusive, bit3 upper exclusive); EQ / NEQ compare values[0].
PB200_HD bool expr_matches(int op, int flags, double lo, double hi, const double* values, int nvalues, double x) {
  if (op == PB200_EXPR_RANGE) {
    if (!(flags & 1) && !((flags & 4) ? x > lo : x >= lo)) return false;
    if (!(flags & 2) && !((flags & 8) ? x < hi : x <= hi)) return false;
    return x == x;
  }
  bool hit = false;
  for (int k = 0; k < nvalues; k++) hit |= x == values[k];
  return (op == PB200_EXPR_EQ || op == PB200_EXPR_IN) ? hit : !hit;
}

// MIN / MAX accumulate the Double.compare order key (transform_key of a DOUBLE); a MIN entry starts at ~0 and a MAX entry
// at 0, neither of which is the key of any double (every NaN has one key), so they mean "no row".
constexpr unsigned long long kExprMinEmpty = ~0ull, kExprMaxEmpty = 0ull;
PB200_HD double expr_key_value(int fn, unsigned long long key) {
  if (key == (fn == PB200_AGG_MIN ? kExprMinEmpty : kExprMaxEmpty)) return fn == PB200_AGG_MIN ? (double)INFINITY : -(double)INFINITY;
  const uint64_t bits = transform_key_bits(TK_DOUBLE, key);
  double d;
  memcpy(&d, &bits, 8);
  return d;
}

}  // namespace pb200
