// pb200_transform.h -- single-column transform programs (pb200_transform_op, include/pinot_b200.h): their validation and
// their evaluation on ONE value.  The derivation kernel (pb200_transform.cu) evaluates a program once per dictionary entry
// of the source column; CPU tests compile this header with g++ and run the same code.  Semantics: DESIGN.md section 3.8.
//
// Exactness points:
//   * arithmetic is one IEEE-754 round-to-nearest operation per operator (__dadd_rn / __dmul_rn / __ddiv_rn on the device:
//     never contracted into an FMA), operands converted to double first, like Java's double arithmetic;
//   * calendar fields come from integer civil-from-days arithmetic with floor division (negative instants included);
//   * unit conversions follow java.util.concurrent.TimeUnit: truncation toward 0 to a coarser unit, saturation to
//     Long.MIN_VALUE / Long.MAX_VALUE to a finer one.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "pb200_order.h"

namespace pb200 {

constexpr int kTransformMaxOps = 16;              // operations (leaves not counted) per program
constexpr int kTransformMaxProgram = 2 * kTransformMaxOps + 1;
constexpr int64_t kTransformMaxMillis = 1ll << 53;  // calendar functions refuse instants beyond +-2^53 ms

// java.util.concurrent.TimeUnit, finest first: nanoseconds per unit
PB200_HD int64_t time_unit_nanos(int u) {
  switch (u) {
    case PB200_TU_NANOSECONDS: return 1ll;
    case PB200_TU_MICROSECONDS: return 1000ll;
    case PB200_TU_MILLISECONDS: return 1000000ll;
    case PB200_TU_SECONDS: return 1000000000ll;
    case PB200_TU_MINUTES: return 60000000000ll;
    case PB200_TU_HOURS: return 3600000000000ll;
    default: return 86400000000000ll;
  }
}

// TimeUnit.convert(d, src) into dst (TimeUnit.cvt): coarser -> d / ratio (toward 0), finer -> d * ratio saturated
PB200_HD int64_t time_unit_convert(int64_t d, int src, int dst) {
  const int64_t s = time_unit_nanos(src), t = time_unit_nanos(dst);
  if (s == t) return d;
  if (s < t) return d / (t / s);
  const int64_t r = s / t, max = INT64_MAX / r;
  if (d > max) return INT64_MAX;
  if (d < -max) return INT64_MIN;
  return d * r;
}

PB200_HD int64_t floor_div(int64_t a, int64_t b) { const int64_t q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }

// proleptic Gregorian calendar (H. Hinnant's days_from_civil / civil_from_days)
PB200_HD int64_t days_from_civil(int64_t y, int m, int d) {
  y -= m <= 2;
  const int64_t era = (y >= 0 ? y : y - 399) / 400;
  const int64_t yoe = y - era * 400;
  const int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  const int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + doe - 719468;
}
PB200_HD void civil_from_days(int64_t z, int64_t* y, int* m, int* d) {
  z += 719468;
  const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  const int64_t doe = z - era * 146097;
  const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  const int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const int64_t mp = (5 * doy + 2) / 153;
  *d = (int)(doy - (153 * mp + 2) / 5 + 1);
  *m = (int)(mp < 10 ? mp + 3 : mp - 9);
  *y = yoe + era * 400 + (*m <= 2);
}
PB200_HD int iso_dow(int64_t days) { return (int)((days % 7 + 10) % 7) + 1; }  // 1 = Monday; 1970-01-01 was a Thursday
PB200_HD bool leap_year(int64_t y) { return (y % 4 == 0 && y % 100 != 0) || y % 400 == 0; }
PB200_HD int iso_weeks_in_year(int64_t y) {
  const int jan1 = iso_dow(days_from_civil(y, 1, 1));
  return (jan1 == 4 || (jan1 == 3 && leap_year(y))) ? 53 : 52;
}

// calendar field (PB200_T_YEAR .. PB200_T_MILLISECOND) of an epoch-millisecond instant, UTC
PB200_HD int64_t calendar_field(int op, int64_t ms) {
  const int64_t days = floor_div(ms, 86400000ll), in_day = ms - days * 86400000ll;
  int64_t y; int m, d;
  civil_from_days(days, &y, &m, &d);
  const int64_t doy = days - days_from_civil(y, 1, 1) + 1;
  switch (op) {
    case PB200_T_YEAR: return y;
    case PB200_T_QUARTER: return (m - 1) / 3 + 1;
    case PB200_T_MONTH: return m;
    case PB200_T_DAY: return d;
    case PB200_T_DAYOFWEEK: return iso_dow(days);
    case PB200_T_DAYOFYEAR: return doy;
    case PB200_T_HOUR: return in_day / 3600000ll;
    case PB200_T_MINUTE: return in_day / 60000ll % 60;
    case PB200_T_SECOND: return in_day / 1000ll % 60;
    case PB200_T_MILLISECOND: return in_day % 1000ll;
    default: {  // PB200_T_WEEK: ISO week of the week-based year
      const int64_t w = (doy - iso_dow(days) + 10) / 7;
      if (w < 1) return iso_weeks_in_year(y - 1);
      if (w > iso_weeks_in_year(y)) return 1;
      return w;
    }
  }
}

// start of the UTC unit (PB200_DT_*) holding the instant, in epoch milliseconds
PB200_HD int64_t truncate_millis(int unit, int64_t ms) {
  switch (unit) {
    case PB200_DT_MILLISECOND: return ms;
    case PB200_DT_SECOND: return floor_div(ms, 1000ll) * 1000ll;
    case PB200_DT_MINUTE: return floor_div(ms, 60000ll) * 60000ll;
    case PB200_DT_HOUR: return floor_div(ms, 3600000ll) * 3600000ll;
    case PB200_DT_DAY: return floor_div(ms, 86400000ll) * 86400000ll;
    case PB200_DT_WEEK: { const int64_t days = floor_div(ms, 86400000ll); return (days - (iso_dow(days) - 1)) * 86400000ll; }
    default: {
      int64_t y; int m, d;
      civil_from_days(floor_div(ms, 86400000ll), &y, &m, &d);
      if (unit == PB200_DT_QUARTER) m = (m - 1) / 3 * 3 + 1;
      else if (unit == PB200_DT_YEAR) m = 1;
      return days_from_civil(y, m, 1) * 86400000ll;
    }
  }
}

#ifdef __CUDA_ARCH__
PB200_HD double t_add(double a, double b) { return __dadd_rn(a, b); }
PB200_HD double t_sub(double a, double b) { return __dsub_rn(a, b); }
PB200_HD double t_mul(double a, double b) { return __dmul_rn(a, b); }
PB200_HD double t_div(double a, double b) { return __ddiv_rn(a, b); }
#else
PB200_HD double t_add(double a, double b) { volatile double r = a + b; return r; }  // volatile: no contraction on the host
PB200_HD double t_sub(double a, double b) { volatile double r = a - b; return r; }
PB200_HD double t_mul(double a, double b) { volatile double r = a * b; return r; }
PB200_HD double t_div(double a, double b) { volatile double r = a / b; return r; }
#endif

// Result kinds of a program and of every stack entry.  Integral entries hold int64; kind INT marks an int32 result.
enum TKind { TK_INT = PB200_INT, TK_LONG = PB200_LONG, TK_FLOAT = PB200_FLOAT, TK_DOUBLE = PB200_DOUBLE };
PB200_HD bool tk_integral(int k) { return k == TK_INT || k == TK_LONG; }

PB200_HD int transform_arity(int op) {
  switch (op) {
    case PB200_T_COLUMN: case PB200_T_LONG_LITERAL: case PB200_T_DOUBLE_LITERAL: return 0;
    case PB200_T_PLUS: case PB200_T_MINUS: case PB200_T_TIMES: case PB200_T_DIVIDE: case PB200_T_MOD:
    case PB200_T_TOEPOCH_BUCKET: case PB200_T_TOEPOCH_ROUNDED: return 2;
    default: return 1;
  }
}

// Checks a program against the source column's stored type (host side, before any launch).  Returns 0 and the result
// kind, or a PB200_E_* code with a message in `why` (PB200_E_INVALID: malformed program; PB200_E_UNSUPPORTED: a
// well-formed program outside the supported set).
inline int transform_check(const pb200_transform_op* ops, int n, int source_type, int* result_kind, const char** why) {
  if (!ops || n <= 0 || n > kTransformMaxProgram) { *why = "program length out of range"; return PB200_E_INVALID; }
  if (source_type == PB200_STRING) { *why = "STRING columns have no transforms on this path"; return PB200_E_UNSUPPORTED; }
  if (source_type < PB200_INT || source_type > PB200_STRING) { *why = "unknown source type"; return PB200_E_INVALID; }
  int kinds[kTransformMaxProgram];
  bool literal[kTransformMaxProgram];
  int sp = 0, columns = 0, operations = 0;
  for (int k = 0; k < n; k++) {
    const pb200_transform_op& o = ops[k];
    const int ar = o.op >= PB200_T_COLUMN && o.op <= PB200_T_TOEPOCH_ROUNDED ? transform_arity(o.op) : -1;
    if (ar < 0 || o.reserved != 0) { *why = "unknown operation"; return PB200_E_INVALID; }
    if (sp < ar) { *why = "operand stack underflow"; return PB200_E_INVALID; }
    if (ar == 0) {
      if (o.op == PB200_T_COLUMN) { columns++; kinds[sp] = source_type; literal[sp] = false; }
      else { kinds[sp] = o.op == PB200_T_LONG_LITERAL ? TK_LONG : TK_DOUBLE; literal[sp] = true; }
      sp++;
      continue;
    }
    operations++;
    const int a = kinds[sp - ar];
    int out;
    switch (o.op) {
      case PB200_T_PLUS: case PB200_T_MINUS: case PB200_T_TIMES: case PB200_T_DIVIDE: case PB200_T_MOD:
      case PB200_T_FLOOR: case PB200_T_CEIL: case PB200_T_ABS:
        out = TK_DOUBLE;
        break;
      case PB200_T_DATETRUNC: {
        const int unit = (int)(o.i & 0xff), in = (int)(o.i >> 8 & 0xff), outu = (int)(o.i >> 16 & 0xff);
        if (unit < PB200_DT_MILLISECOND || unit > PB200_DT_YEAR || in > PB200_TU_DAYS || outu > PB200_TU_DAYS || (o.i >> 24) != 0) { *why = "DATETRUNC unit out of range"; return PB200_E_INVALID; }
        if (!tk_integral(a) || literal[sp - 1]) { *why = "DATETRUNC takes an INT / LONG column or time function"; return PB200_E_UNSUPPORTED; }
        out = TK_LONG;
        break;
      }
      case PB200_T_TIMECONVERT:
        if (o.i < 0 || (o.i & 0xff) > PB200_TU_DAYS || (o.i >> 8) > PB200_TU_DAYS) { *why = "TIMECONVERT unit out of range"; return PB200_E_INVALID; }
        if (!tk_integral(a) || literal[sp - 1]) { *why = "TIMECONVERT takes an INT / LONG column or time function"; return PB200_E_UNSUPPORTED; }
        out = TK_LONG;
        break;
      case PB200_T_TOEPOCH: case PB200_T_TOEPOCH_BUCKET: case PB200_T_TOEPOCH_ROUNDED:
        if (o.i < PB200_TU_SECONDS || o.i > PB200_TU_DAYS) { *why = "TOEPOCH unit out of range"; return PB200_E_INVALID; }
        if (!tk_integral(a) || literal[sp - ar]) { *why = "TOEPOCH functions take an INT / LONG column or time function"; return PB200_E_UNSUPPORTED; }
        if (ar == 2 && (!literal[sp - 1] || kinds[sp - 1] != TK_LONG || ops[k - 1].op != PB200_T_LONG_LITERAL || ops[k - 1].i <= 0)) {
          *why = "the bucket of a TOEPOCH function is a positive integer literal";
          return PB200_E_UNSUPPORTED;
        }
        out = TK_LONG;
        break;
      default:  // calendar fields
        if (!tk_integral(a) || literal[sp - 1]) { *why = "calendar functions take an INT / LONG column or time function"; return PB200_E_UNSUPPORTED; }
        out = TK_INT;
    }
    sp -= ar;
    kinds[sp] = out;
    literal[sp] = false;
    sp++;
  }
  if (sp != 1) { *why = "program does not leave exactly one value"; return PB200_E_INVALID; }
  if (columns != 1) { *why = columns ? "more than one column in one expression" : "expression has no column"; return columns ? PB200_E_UNSUPPORTED : PB200_E_INVALID; }
  if (operations == 0) { *why = "program has no operation"; return PB200_E_INVALID; }
  if (operations > kTransformMaxOps) { *why = "more than 16 operations"; return PB200_E_UNSUPPORTED; }
  if (literal[0]) { *why = "program result is a literal"; return PB200_E_INVALID; }
  *result_kind = kinds[0];
  return PB200_OK;
}

// One value of the source column (as stored: INT / LONG as int64, FLOAT / DOUBLE as double) through a CHECKED program.
// Returns false when a calendar function meets an instant beyond +-2^53 ms (the derivation is then refused).
PB200_HD bool transform_eval(const pb200_transform_op* ops, int n, int source_type, int64_t si, double sd, int64_t* oi,
                             double* od) {
  int64_t I[kTransformMaxProgram];
  double D[kTransformMaxProgram];
  bool dbl[kTransformMaxProgram];
  int sp = 0;
  for (int k = 0; k < n; k++) {
    const pb200_transform_op o = ops[k];
    switch (o.op) {
      case PB200_T_COLUMN: if (tk_integral(source_type)) { I[sp] = si; dbl[sp] = false; } else { D[sp] = sd; dbl[sp] = true; } sp++; continue;
      case PB200_T_LONG_LITERAL: I[sp] = o.i; dbl[sp] = false; sp++; continue;
      case PB200_T_DOUBLE_LITERAL: D[sp] = o.d; dbl[sp] = true; sp++; continue;
      default: break;
    }
    const int ar = transform_arity(o.op);
    sp -= ar;
    const int a = sp, b = sp + 1;
    if (o.op <= PB200_T_ABS) {  // arithmetic on doubles
      const double x = dbl[a] ? D[a] : (double)I[a];
      const double y = ar == 2 ? (dbl[b] ? D[b] : (double)I[b]) : 0.0;
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
      D[a] = r; dbl[a] = true;
    } else {
      const int64_t x = I[a];
      int64_t r;
      switch (o.op) {
        case PB200_T_DATETRUNC: {
          const int unit = (int)(o.i & 0xff), in = (int)(o.i >> 8 & 0xff), out = (int)(o.i >> 16 & 0xff);
          const int64_t ms = time_unit_convert(x, in, PB200_TU_MILLISECONDS);
          if (ms > kTransformMaxMillis || ms < -kTransformMaxMillis) return false;
          r = time_unit_convert(truncate_millis(unit, ms), PB200_TU_MILLISECONDS, out);
          break;
        }
        case PB200_T_TIMECONVERT: r = time_unit_convert(x, (int)(o.i & 0xff), (int)(o.i >> 8)); break;
        case PB200_T_TOEPOCH: r = time_unit_convert(x, PB200_TU_MILLISECONDS, (int)o.i); break;
        case PB200_T_TOEPOCH_BUCKET: r = time_unit_convert(x, PB200_TU_MILLISECONDS, (int)o.i) / I[b]; break;
        case PB200_T_TOEPOCH_ROUNDED: r = time_unit_convert(x, PB200_TU_MILLISECONDS, (int)o.i) / I[b] * I[b]; break;
        default:
          if (x > kTransformMaxMillis || x < -kTransformMaxMillis) return false;
          r = calendar_field(o.op, x);
      }
      I[a] = r; dbl[a] = false;
    }
    sp++;
  }
  if (dbl[0]) *od = D[0]; else *oi = I[0];
  return true;
}

// Order key of a typed result: unsigned order == the dictionary order of its kind (INT / LONG numeric; DOUBLE
// Double.compare: -0.0 before 0.0, every NaN one value after +inf).  The inverse gives the dictionary value back.
PB200_HD uint64_t transform_key(int kind, int64_t i, double d) {
  if (kind == TK_INT) return (uint64_t)((uint32_t)(int32_t)i ^ 0x80000000u);
  if (kind == TK_LONG) return (uint64_t)i ^ 0x8000000000000000ull;
  if (d != d) d = NAN;  // Double.doubleToLongBits: one canonical NaN
  return double_order_bits(d);
}
PB200_HD uint64_t transform_key_bits(int kind, uint64_t key) {  // the value's bits (INT: its 32 bits, unbiased)
  if (kind == TK_INT) return (uint32_t)key ^ 0x80000000u;
  if (kind == TK_LONG) return key ^ 0x8000000000000000ull;
  return (key >> 63) ? key & ~(1ull << 63) : ~key;
}

}  // namespace pb200
