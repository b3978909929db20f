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

// The operand count of an expression operation: transform_arity, and the CASE WHEN operations (DESIGN.md section 3.19)
// of pb200_execute_exprs_cond; -1 for an unknown operation.
PB200_HD int expr_arity(int op) {
  switch (op) {
    case PB200_T_COND: return 0;
    case PB200_T_NOT: return 1;
    case PB200_T_AND: case PB200_T_OR: return 2;
    case PB200_T_CASE: return 3;
    default: return op >= PB200_T_COLUMN && op <= PB200_T_TOEPOCH_ROUNDED ? transform_arity(op) : -1;
  }
}
PB200_HD bool expr_case_op(int op) { return op >= PB200_T_COND && op <= PB200_T_CASE; }
PB200_HD bool expr_is_condition(int op) { return op == PB200_T_COND || op == PB200_T_AND || op == PB200_T_OR || op == PB200_T_NOT; }

// Checks a program (host side, before any launch).  `nconds` is the size of the call's condition table (0: COND is out of
// range, so no CASE program passes).  Returns 0 with the number of column leaves (COND leaves included) in *leaves, or a
// PB200_E_* code with a message in `why`: PB200_E_INVALID for a malformed program (an unknown operation, a stack
// underflow, a condition index out of range, a condition where a value belongs or the reverse), PB200_E_UNSUPPORTED for
// a well-formed one outside the supported set (a time function, more than kExprMaxLeaves column leaves, more than 16
// operations, fewer than two column leaves in a program without conditions).
inline int expr_check(const pb200_transform_op* ops, int n, int* leaves, const char** why, int nconds = 0) {
  if (!ops || n <= 0 || n > kTransformMaxProgram) { *why = "program length out of range"; return PB200_E_INVALID; }
  int sp = 0, columns = 0, conds = 0, operations = 0;
  uint64_t is_cond = 0;   // bit k: stack entry k is a condition
  bool time_fn = false;
  for (int k = 0; k < n; k++) {
    const pb200_transform_op& o = ops[k];
    const int ar = expr_arity(o.op);
    if (ar < 0 || o.reserved != 0) { *why = "unknown operation"; return PB200_E_INVALID; }
    if (sp < ar) { *why = "operand stack underflow"; return PB200_E_INVALID; }
    if (o.op == PB200_T_COLUMN && o.i < 0) { *why = "negative column id"; return PB200_E_INVALID; }
    if (o.op == PB200_T_COND && (o.i < 0 || o.i >= nconds)) { *why = "condition index out of range"; return PB200_E_INVALID; }
    // operand kinds: AND / OR / NOT take conditions, CASE a condition and two values, everything else values
    const uint64_t args = ar ? (is_cond >> (sp - ar)) & ((1ull << ar) - 1) : 0;
    const uint64_t want = o.op == PB200_T_CASE ? 1 : (o.op == PB200_T_AND || o.op == PB200_T_OR || o.op == PB200_T_NOT) ? (1ull << ar) - 1 : 0;
    if (args != want) { *why = "operand of the wrong kind (a condition where a value belongs, or the reverse)"; return PB200_E_INVALID; }
    time_fn |= !expr_op_ok(o.op) && !expr_case_op(o.op);
    columns += o.op == PB200_T_COLUMN;
    conds += o.op == PB200_T_COND;
    operations += ar > 0;
    sp += 1 - ar;
    is_cond = (is_cond & ((1ull << (sp - 1)) - 1)) | (uint64_t)expr_is_condition(o.op) << (sp - 1);
  }
  if (sp != 1) { *why = "program does not leave exactly one value"; return PB200_E_INVALID; }
  if (is_cond & 1) { *why = "the program's result is a condition, not a value"; return PB200_E_INVALID; }
  if (time_fn) { *why = "time functions are not accelerated inside an expression over two or more columns"; return PB200_E_UNSUPPORTED; }
  if (columns + conds < (conds ? 1 : 2)) { *why = "an expression over several columns needs two or more column leaves"; return PB200_E_UNSUPPORTED; }
  if (columns + conds > kExprMaxLeaves) { *why = "more than 8 column leaves in one expression"; return PB200_E_UNSUPPORTED; }
  if (operations > kTransformMaxOps) { *why = "more than 16 operations"; return PB200_E_UNSUPPORTED; }
  *leaves = columns + conds;
  return PB200_OK;
}

// A CHECKED device program (column leaf i reads leaf[i]) on one row's leaf values.  COND: programs may hold the CASE WHEN
// operations, condition i of the row being bit i of `cond`; a condition is 1.0 or 0.0 on the stack.  Without COND the
// function is the arithmetic evaluator alone, so the kernels of programs without conditions carry none of it.
template <bool COND = false>
PB200_HD double expr_eval(const pb200_transform_op* ops, int n, const double* leaf, uint32_t cond = 0) {
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
    if constexpr (COND) {
      switch (o.op) {
        case PB200_T_COND: D[sp++] = (cond >> o.i) & 1u ? 1.0 : 0.0; continue;
        case PB200_T_NOT: D[sp - 1] = D[sp - 1] != 0.0 ? 0.0 : 1.0; continue;
        case PB200_T_AND: sp--; D[sp - 1] = D[sp - 1] != 0.0 && D[sp] != 0.0 ? 1.0 : 0.0; continue;
        case PB200_T_OR: sp--; D[sp - 1] = D[sp - 1] != 0.0 || D[sp] != 0.0 ? 1.0 : 0.0; continue;
        case PB200_T_CASE: sp -= 2; D[sp - 1] = D[sp - 1] != 0.0 ? D[sp] : D[sp + 1]; continue;
        default: break;
      }
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
