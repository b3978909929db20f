// transform.cpp -- value-space face of derived columns (pb200_segment_derive_column): single-column expressions by their
// canonical text, the form of the reference's ExpressionContext.toString() -- function names in lower case without '_',
// arguments separated by ',' without spaces, literals in single quotes: DATETRUNC('DAY', ts) is datetrunc('DAY',ts),
// ts / 1000 is divide(ts,'1000').  Two spellings of one expression normalise to one text and share one derived column.
#include <cctype>
#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "host_internal.h"
#include "../pb200_expr.h"

using pb200::set_error;
using namespace pb200h;

namespace {

struct Node {
  bool call = false, literal = false;
  std::string text;                     // function name (canonical), literal text (normalised), or column name
  std::vector<std::unique_ptr<Node>> args;
};

struct Parser {
  const char* p;
  std::string err;
  void ws() { while (*p && isspace((unsigned char)*p)) p++; }
  std::unique_ptr<Node> parse() {
    ws();
    auto n = std::make_unique<Node>();
    if (*p == '\'') {  // quoted literal ('' escapes a quote)
      p++;
      n->literal = true;
      for (;;) {
        if (!*p) { err = "unterminated literal"; return nullptr; }
        if (*p == '\'') { if (p[1] == '\'') { n->text += '\''; p += 2; continue; } p++; break; }
        n->text += *p++;
      }
      return n;
    }
    if (*p == '-' || *p == '+' || *p == '.' || isdigit((unsigned char)*p)) {  // bare numeric literal
      const char* s = p;
      if (*p == '-' || *p == '+') p++;
      while (isalnum((unsigned char)*p) || *p == '.' || ((*p == '-' || *p == '+') && (p[-1] == 'e' || p[-1] == 'E'))) p++;
      n->literal = true;
      n->text.assign(s, p - s);
      return n;
    }
    const char* s = p;
    while (isalnum((unsigned char)*p) || *p == '_' || *p == '$' || *p == '.') p++;
    if (p == s) { err = "expected a name or a literal"; return nullptr; }
    n->text.assign(s, p - s);
    ws();
    if (*p != '(') return n;  // a column
    p++;
    n->call = true;
    std::string f;
    for (char ch : n->text) if (ch != '_') f += (char)tolower((unsigned char)ch);
    n->text = f;
    ws();
    if (*p == ')') { p++; return n; }
    for (;;) {
      auto a = parse();
      if (!a) return nullptr;
      n->args.push_back(std::move(a));
      ws();
      if (*p == ',') { p++; continue; }
      if (*p == ')') { p++; return n; }
      err = "expected ',' or ')'";
      return nullptr;
    }
  }
};

const char* const kTimeUnits[] = {"NANOSECONDS", "MICROSECONDS", "MILLISECONDS", "SECONDS", "MINUTES", "HOURS", "DAYS"};
const char* const kTruncUnits[] = {"MILLISECOND", "SECOND", "MINUTE", "HOUR", "DAY", "WEEK", "MONTH", "QUARTER", "YEAR"};
struct Fn { const char* name; int op; int min_args, max_args; };
const Fn kFunctions[] = {
    {"plus", PB200_T_PLUS, 2, 2}, {"minus", PB200_T_MINUS, 2, 2}, {"times", PB200_T_TIMES, 2, 2},
    {"divide", PB200_T_DIVIDE, 2, 2}, {"mod", PB200_T_MOD, 2, 2}, {"floor", PB200_T_FLOOR, 1, 1},
    {"ceil", PB200_T_CEIL, 1, 1}, {"abs", PB200_T_ABS, 1, 1}, {"datetrunc", PB200_T_DATETRUNC, 2, 5},
    {"year", PB200_T_YEAR, 1, 1}, {"quarter", PB200_T_QUARTER, 1, 1}, {"month", PB200_T_MONTH, 1, 1},
    {"week", PB200_T_WEEK, 1, 1}, {"day", PB200_T_DAY, 1, 1}, {"dayofweek", PB200_T_DAYOFWEEK, 1, 1},
    {"dayofyear", PB200_T_DAYOFYEAR, 1, 1}, {"hour", PB200_T_HOUR, 1, 1}, {"minute", PB200_T_MINUTE, 1, 1},
    {"second", PB200_T_SECOND, 1, 1}, {"millisecond", PB200_T_MILLISECOND, 1, 1}, {"timeconvert", PB200_T_TIMECONVERT, 3, 3},
    {"toepochseconds", PB200_T_TOEPOCH, 1, 1}, {"toepochminutes", PB200_T_TOEPOCH, 1, 1},
    {"toepochhours", PB200_T_TOEPOCH, 1, 1}, {"toepochdays", PB200_T_TOEPOCH, 1, 1},
    {"toepochsecondsbucket", PB200_T_TOEPOCH_BUCKET, 2, 2}, {"toepochminutesbucket", PB200_T_TOEPOCH_BUCKET, 2, 2},
    {"toepochhoursbucket", PB200_T_TOEPOCH_BUCKET, 2, 2}, {"toepochdaysbucket", PB200_T_TOEPOCH_BUCKET, 2, 2},
    {"toepochsecondsrounded", PB200_T_TOEPOCH_ROUNDED, 2, 2}, {"toepochminutesrounded", PB200_T_TOEPOCH_ROUNDED, 2, 2},
    {"toepochhoursrounded", PB200_T_TOEPOCH_ROUNDED, 2, 2}, {"toepochdaysrounded", PB200_T_TOEPOCH_ROUNDED, 2, 2},
};
const char* const kAliases[][2] = {{"add", "plus"}, {"sub", "minus"}, {"mult", "times"}, {"div", "divide"},
                                   {"weekofyear", "week"}, {"dayofmonth", "day"}, {"dow", "dayofweek"}, {"doy", "dayofyear"}};

const Fn* find_function(std::string& name) {
  for (auto& a : kAliases) if (name == a[0]) name = a[1];
  for (auto& f : kFunctions) if (name == f.name) return &f;
  return nullptr;
}
int toepoch_unit(const std::string& name) {  // toepoch<unit>[bucket|rounded] -> PB200_TU_*
  const std::string u = name.substr(7);
  return u.rfind("seconds", 0) == 0 ? PB200_TU_SECONDS : u.rfind("minutes", 0) == 0 ? PB200_TU_MINUTES
       : u.rfind("hours", 0) == 0 ? PB200_TU_HOURS : PB200_TU_DAYS;
}
int unit_index(const std::string& t, const char* const* names, int n) {
  for (int i = 0; i < n; i++) if (t == names[i]) return i;
  return -1;
}
std::string upper(const std::string& s) { std::string r = s; for (auto& ch : r) ch = (char)toupper((unsigned char)ch); return r; }

// A decimal numeric literal ([+-]digits[.digits][e[+-]digits]: no hex, NaN or infinity): its int64 value when the text
// is an integer or an integral value in the int64 range (is_int: `'10.0'` is the integer 10, so that every spelling of a
// value compiles to one program), and its double (the text rounded to nearest)
bool decimal_text(const std::string& t) {
  size_t k = 0, digits = 0;
  if (k < t.size() && (t[k] == '+' || t[k] == '-')) k++;
  while (k < t.size() && isdigit((unsigned char)t[k])) { k++; digits++; }
  if (k < t.size() && t[k] == '.') { k++; while (k < t.size() && isdigit((unsigned char)t[k])) { k++; digits++; } }
  if (!digits) return false;
  if (k < t.size() && (t[k] == 'e' || t[k] == 'E')) {
    k++;
    if (k < t.size() && (t[k] == '+' || t[k] == '-')) k++;
    size_t e = 0;
    while (k < t.size() && isdigit((unsigned char)t[k])) { k++; e++; }
    if (!e) return false;
  }
  return k == t.size();
}
bool parse_number(const std::string& t, bool* is_int, int64_t* i, double* d) {
  if (!decimal_text(t)) return false;
  const char* s = t.c_str();
  char* end = nullptr;
  errno = 0;
  const long long v = strtoll(s, &end, 10);
  if (*end == 0 && errno == 0) { *is_int = true; *i = v; *d = strtod(s, nullptr); return true; }
  errno = 0;
  const double x = strtod(s, &end);
  if (*end != 0 || end == s) return false;
  *d = x;
  *is_int = std::isfinite(x) && x == std::floor(x) && std::fabs(x) < 9.2e18 && !(x == 0 && std::signbit(x));  // -0.0 stays a double
  if (*is_int) *i = (int64_t)x;
  return true;
}
// numeric literals by value: integral values as integers, the others in their shortest round-trip form
std::string number_text(bool is_int, int64_t i, double d) {
  if (is_int) return std::to_string(i);
  if (std::isfinite(d) && d == std::floor(d) && std::fabs(d) < 9.2e18 && !(d == 0 && std::signbit(d))) return std::to_string((long long)d);
  char buf[40];
  for (int prec = 1; prec <= 17; prec++) {
    snprintf(buf, sizeof buf, "%.*g", prec, d);
    if (strtod(buf, nullptr) == d) break;
  }
  return buf;
}

// Canonical text and, when `seg` is given, the op program (postfix) over the segment's column.  Errors: PB200_E_INVALID
// (malformed), PB200_E_UNSUPPORTED (outside the supported set), with a message.
struct Compiled {
  std::string text;
  std::vector<pb200_transform_op> ops;
  std::string column;
  int columns = 0;
  bool multi = false;                  // any number of columns: leaf k (PB200_T_COLUMN i = k) reads column leaves[k]
  std::vector<std::string> leaves;
  bool in_case = false;                // compiling a CASE's arguments (a nested CASE is refused)
  std::vector<CaseCond> conds;         // CASE conditions: PB200_T_COND i = k tests conds[k]
  std::vector<CaseBranch> branches;    // CASE branch values (THEN and ELSE)
};

int compile(const Node& n, Compiled& c);

// a literal of a CASE condition as canonical text: quoted, '' for a quote
std::string quoted(const std::string& t) {
  std::string r = "'";
  for (char ch : t) { r += ch; if (ch == '\'') r += '\''; }
  return r + "'";
}

// CASE conditions (DESIGN.md section 3.19): the parser's function name (lower case, no '_') -> the canonical one
const char* const kCondNames[][2] = {
    {"and", "and"}, {"or", "or"}, {"not", "not"}, {"equals", "equals"}, {"notequals", "not_equals"},
    {"lessthan", "less_than"}, {"lessthanorequal", "less_than_or_equal"}, {"greaterthan", "greater_than"},
    {"greaterthanorequal", "greater_than_or_equal"}, {"between", "between"}, {"in", "in"}, {"notin", "not_in"},
    {"like", "like"}, {"regexplike", "regexp_like"}};

int compile_cond(const Node& n, Compiled& c) {
  const char* name = nullptr;
  if (n.call)
    for (auto& k : kCondNames) if (n.text == k[0]) name = k[1];
  if (!name) { set_error("a CASE condition must be a comparison, IN, BETWEEN, LIKE or REGEXP_LIKE leaf or AND / OR / NOT over them"); return PB200_E_UNSUPPORTED; }
  const std::string fn = name;
  const int na = (int)n.args.size();
  auto op = [&](int code, int64_t i) { pb200_transform_op o; memset(&o, 0, sizeof o); o.op = code; o.i = i; c.ops.push_back(o); };
  c.text += fn + "(";
  if (fn == "and" || fn == "or" || fn == "not") {
    if (fn == "not" ? na != 1 : na < 2) { set_error("%s takes %s arguments, not %d", name, fn == "not" ? "one" : "two or more", na); return PB200_E_UNSUPPORTED; }
    for (int k = 0; k < na; k++) {
      if (k) c.text += ",";
      if (int rc = compile_cond(*n.args[k], c)) return rc;
      if (k) op(fn == "and" ? PB200_T_AND : PB200_T_OR, 0);
    }
    if (fn == "not") op(PB200_T_NOT, 0);
    c.text += ")";
    return PB200_OK;
  }
  const bool many = fn == "in" || fn == "not_in";
  const int want = fn == "between" ? 3 : 2;
  if (many ? na < 2 : na != want) { set_error("%s takes %d arguments, not %d", name, want, na); return PB200_E_UNSUPPORTED; }
  CaseCond cc;
  cc.fn = fn;
  for (int k = 0; k < na; k++) {
    const Node& a = *n.args[k];
    if (k == 0 ? a.call || a.literal : !a.literal) {
      set_error("%s: a CASE condition compares one column with literals (no column against column, no expression operand)", name);
      return PB200_E_UNSUPPORTED;
    }
    if (k) { c.text += "," + quoted(a.text); cc.literals.push_back(a.text); }
    else { c.text += a.text; cc.column = a.text; }
  }
  c.text += ")";
  op(PB200_T_COND, (int64_t)c.conds.size());
  c.conds.push_back(std::move(cc));
  return PB200_OK;
}

// case(c1,v1,c2,v2,...,e): postfix c1 v1 c2 v2 ... e CASE ... CASE (one CASE per WHEN)
int compile_case(const Node& n, Compiled& c) {
  if (c.in_case) { set_error("a nested CASE is not accelerated"); return PB200_E_UNSUPPORTED; }
  const int na = (int)n.args.size();
  if (na < 3 || na % 2 == 0) { set_error("case takes WHEN / THEN pairs and an ELSE value (an odd number of three or more arguments), not %d", na); return PB200_E_UNSUPPORTED; }
  c.in_case = true;
  c.text += "case(";
  for (int k = 0; k < na; k++) {
    if (k) c.text += ",";
    const Node& a = *n.args[k];
    if (k % 2 == 0 && k + 1 < na) {
      if (int rc = compile_cond(a, c)) return rc;
      continue;
    }
    CaseBranch b;
    b.kind = a.call ? CaseBranch::ARITHMETIC : a.literal ? CaseBranch::DOUBLE_LITERAL : CaseBranch::COLUMN;
    b.column = a.literal ? "" : a.text;
    const size_t first = c.ops.size();
    if (int rc = compile(a, c)) return rc;
    if (a.literal && c.ops[first].op == PB200_T_LONG_LITERAL) { b.kind = CaseBranch::LONG_LITERAL; b.value = c.ops[first].i; }
    c.branches.push_back(b);
  }
  for (int k = 0; k < na / 2; k++) {
    pb200_transform_op o; memset(&o, 0, sizeof o); o.op = PB200_T_CASE; c.ops.push_back(o);
  }
  c.text += ")";
  c.in_case = false;
  return PB200_OK;
}

int compile(const Node& n, Compiled& c) {
  if (n.call && c.multi && n.text == "case") return compile_case(n, c);
  auto op = [&](int code, int64_t i) { pb200_transform_op o; memset(&o, 0, sizeof o); o.op = code; o.i = i; c.ops.push_back(o); };
  if (n.literal) {
    bool is_int; int64_t i = 0; double d = 0;
    if (!parse_number(n.text, &is_int, &i, &d)) { set_error("literal '%s' is not a number", n.text.c_str()); return PB200_E_UNSUPPORTED; }
    pb200_transform_op o; memset(&o, 0, sizeof o);
    o.op = is_int ? PB200_T_LONG_LITERAL : PB200_T_DOUBLE_LITERAL; o.i = i; o.d = d;
    c.ops.push_back(o);
    c.text += "'" + number_text(is_int, i, d) + "'";
    return PB200_OK;
  }
  if (!n.call && c.multi) {
    op(PB200_T_COLUMN, (int64_t)c.leaves.size());
    c.leaves.push_back(n.text);
    c.text += n.text;
    return PB200_OK;
  }
  if (!n.call) {
    c.columns++;
    if (c.columns > 1 && n.text != c.column) { set_error("expressions over two or more columns are not accelerated"); return PB200_E_UNSUPPORTED; }
    if (c.columns > 1) { set_error("an expression may use its column once"); return PB200_E_UNSUPPORTED; }
    c.column = n.text;
    op(PB200_T_COLUMN, 0);
    c.text += n.text;
    return PB200_OK;
  }
  std::string name = n.text;
  const Fn* f = find_function(name);
  if (!f) { set_error("function '%s' has no device transform", n.text.c_str()); return PB200_E_UNSUPPORTED; }
  const int na = (int)n.args.size();
  if (na < f->min_args || na > f->max_args) { set_error("%s takes %d to %d arguments, not %d", f->name, f->min_args, f->max_args, na); return PB200_E_UNSUPPORTED; }
  c.text += name + "(";
  auto unit_arg = [&](int k, const char* const* names, int count, int* out) -> int {
    const Node& a = *n.args[k];
    if (!a.literal) { set_error("%s: argument %d must be a unit literal", f->name, k + 1); return PB200_E_UNSUPPORTED; }
    const std::string u = upper(a.text);
    *out = unit_index(u, names, count);
    if (*out < 0) { set_error("%s: unknown unit '%s'", f->name, a.text.c_str()); return PB200_E_UNSUPPORTED; }
    c.text += (k ? ",'" : "'") + u + "'";
    return PB200_OK;
  };
  int rc = PB200_OK;
  if (f->op == PB200_T_DATETRUNC) {
    int unit = 0, in = PB200_TU_MILLISECONDS, out;
    if ((rc = unit_arg(0, kTruncUnits, 9, &unit))) return rc;
    c.text += ",";
    if (n.args[1]->literal) { set_error("datetrunc: the time value must be a column or a time function"); return PB200_E_UNSUPPORTED; }
    if ((rc = compile(*n.args[1], c))) return rc;
    if (na >= 3 && (rc = unit_arg(2, kTimeUnits, 7, &in))) return rc;
    out = in;
    if (na >= 4) {
      if (!n.args[3]->literal || upper(n.args[3]->text) != "UTC") { set_error("datetrunc: time zone '%s' is not accelerated (UTC only)", n.args[3]->text.c_str()); return PB200_E_UNSUPPORTED; }
      c.text += ",'UTC'";
    }
    if (na >= 5 && (rc = unit_arg(4, kTimeUnits, 7, &out))) return rc;
    op(PB200_T_DATETRUNC, unit | in << 8 | out << 16);
  } else if (f->op == PB200_T_TIMECONVERT) {
    int in, out;
    if ((rc = compile(*n.args[0], c))) return rc;
    if ((rc = unit_arg(1, kTimeUnits, 7, &in)) || (rc = unit_arg(2, kTimeUnits, 7, &out))) return rc;
    op(PB200_T_TIMECONVERT, in | out << 8);
  } else {
    for (int k = 0; k < na; k++) {
      if (k) c.text += ",";
      if ((rc = compile(*n.args[k], c))) return rc;
    }
    op(f->op, f->op >= PB200_T_TOEPOCH ? toepoch_unit(name) : 0);
  }
  c.text += ")";
  return PB200_OK;
}

int compile_text(const char* text, Compiled& c, bool multi = false) {
  c.multi = multi;
  Parser ps{text};
  auto root = ps.parse();
  if (root) { ps.ws(); if (*ps.p) { ps.err = "trailing characters"; root.reset(); } }
  if (!root) { set_error("malformed expression '%s': %s", text, ps.err.c_str()); return PB200_E_INVALID; }
  if (!root->call) { set_error("'%s' is no expression", text); return PB200_E_INVALID; }
  if (int rc = compile(*root, c)) return rc;
  int operations = 0;
  for (const auto& o : c.ops) operations += o.op > PB200_T_DOUBLE_LITERAL && o.op != PB200_T_COND;
  if (operations > pb200::kTransformMaxOps) { set_error("expression '%s' has %d operations (at most %d)", text, operations, pb200::kTransformMaxOps); return PB200_E_UNSUPPORTED; }
  if ((int)c.ops.size() > pb200::kTransformMaxProgram) { set_error("expression '%s' compiles to %zu program entries (at most %d)", text, c.ops.size(), pb200::kTransformMaxProgram); return PB200_E_UNSUPPORTED; }
  return PB200_OK;
}

// Under seg->derive_mu: the column of `expression` on `seg`, derived now if it is not there yet.
int derive_locked(pb200_ctx* ctx, pb200h_segment* seg, const char* expression, int* column) {
  int idx = seg->column_index(expression);
  if (idx >= 0) { *column = idx; return PB200_OK; }
  Compiled c;
  if (int rc = compile_text(expression, c)) return rc;
  idx = seg->column_index(c.text.c_str());
  if (idx >= 0) { *column = idx; return PB200_OK; }
  const int src = seg->column_index(c.column.c_str());
  if (src < 0 || src >= seg->num_stored) { set_error("expression '%s': unknown column '%s'", expression, c.column.c_str()); return PB200_E_INVALID; }
  const HostColumn& s = seg->cols[src];
  if (s.data_type == PB200_STRING) { set_error("expression '%s': STRING column '%s' has no transforms on this path", expression, s.name.c_str()); return PB200_E_UNSUPPORTED; }
  if (!s.has_dictionary) { set_error("expression '%s': raw column '%s' has no dictionary", expression, s.name.c_str()); return PB200_E_UNSUPPORTED; }
  if (seg->num_columns() - seg->num_stored >= PB200_MAX_DERIVED_COLUMNS) {
    set_error("segment '%s' already has %d derived columns", seg->name.c_str(), PB200_MAX_DERIVED_COLUMNS);
    return PB200_E_UNSUPPORTED;
  }
  int dcol = -1;
  if (int rc = pb200_segment_derive_column(ctx, seg->dev, src, (int)c.ops.size(), c.ops.data(), &dcol)) return rc;
  if (dcol != seg->num_columns()) { set_error("segment '%s': device and host column lists diverged", seg->name.c_str()); return PB200_E_INVALID; }
  int64_t info[6];
  if (int rc = pb200_segment_column_info(seg->dev, dcol, info)) return rc;
  HostColumn h;
  h.name = c.text;
  h.derived = true;
  h.data_type = (int)info[1]; h.has_dictionary = 1; h.bits = (int)info[2]; h.cardinality = (int)info[3];
  h.entry_bytes = (h.data_type == PB200_LONG || h.data_type == PB200_DOUBLE) ? 8 : 4;
  const int64_t nb = pb200_segment_read_index(ctx, seg->dev, dcol, 1, nullptr, 0);
  h.dict.resize((size_t)std::max<int64_t>(nb, 0));
  if (nb > 0) pb200_segment_read_index(ctx, seg->dev, dcol, 1, h.dict.data(), (uint64_t)nb);
  seg->cols.push_back(std::move(h));  // within the reserved capacity: no column moves
  seg->published.store(dcol + 1, std::memory_order_release);  // complete: lookups may find it now
  *column = dcol;
  return PB200_OK;
}

}  // namespace

namespace pb200h {

int compile_expression(const char* text, std::string* canonical, std::vector<pb200_transform_op>* ops, std::string* column) {
  Compiled c;
  const int rc = compile_text(text, c);
  if (rc == PB200_OK) { *canonical = c.text; *ops = c.ops; *column = c.column; }
  return rc;
}

int compile_multi_expression(const char* text, std::string* canonical, std::vector<pb200_transform_op>* ops,
                             std::vector<std::string>* leaves, std::vector<CaseCond>* conds, std::vector<CaseBranch>* branches) {
  Compiled c;
  int rc = compile_text(text, c, true);
  if (rc == PB200_OK && !c.conds.empty() && !conds) { set_error("'%s': CASE is accelerated only as the argument of SUM, AVG, MIN, MAX or COUNT", text); rc = PB200_E_UNSUPPORTED; }
  if (rc == PB200_OK && c.leaves.size() < 2 && c.conds.empty()) { set_error("'%s' has fewer than two column leaves", text); rc = PB200_E_UNSUPPORTED; }
  if (rc == PB200_OK)
    for (const auto& o : c.ops)
      if (!pb200::expr_op_ok(o.op) && !pb200::expr_case_op(o.op)) {
        set_error("'%s': time functions are not accelerated inside an expression over two or more columns", text);
        rc = PB200_E_UNSUPPORTED;
        break;
      }
  if (rc == PB200_OK && (int)(c.leaves.size() + c.conds.size()) > pb200::kExprMaxLeaves) {
    set_error("'%s' has %zu column leaves, conditions included (at most %d)", text, c.leaves.size() + c.conds.size(), pb200::kExprMaxLeaves);
    rc = PB200_E_UNSUPPORTED;
  }
  if (rc == PB200_OK) {
    *canonical = c.text; *ops = c.ops; *leaves = c.leaves;
    if (conds) *conds = c.conds;
    if (branches) *branches = c.branches;
  }
  return rc;
}

bool is_multi_column_expression(const char* text) {
  if (!text || !strchr(text, '(')) return false;
  Compiled c;
  char saved[1024];
  memcpy(saved, pb200_last_error(), sizeof saved);  // a failed test leaves the caller's last error alone
  const bool multi = compile_text(text, c, true) == PB200_OK && (c.leaves.size() >= 2 || !c.conds.empty());
  set_error("%s", saved);
  return multi;
}

bool is_expression_filter(const char* text) {
  if (!text || !strchr(text, '(')) return false;
  Compiled c;
  char saved[1024];
  memcpy(saved, pb200_last_error(), sizeof saved);
  bool multi = compile_text(text, c, true) == PB200_OK;
  set_error("%s", saved);
  if (!multi || !c.conds.empty()) return false;   // a CASE leaf is derived, which refuses it
  for (const std::string& l : c.leaves) if (l != c.leaves[0]) return true;
  return false;
}

bool normalize_expression(const char* text, std::string* canonical) {
  Compiled c;
  char saved[1024];
  memcpy(saved, pb200_last_error(), sizeof saved);  // a failed lookup leaves the caller's last error alone
  const bool ok = compile_text(text, c) == PB200_OK;
  set_error("%s", saved);
  if (ok) *canonical = c.text;
  return ok;
}

int derive_names(pb200_ctx* ctx, pb200h_segment* const* segs, int nseg, const std::vector<const char*>& names) {
  for (const char* n : names) {
    if (!n || !strchr(n, '(')) continue;  // a plain column name: resolved (or reported unknown) as before
    int first = -1;
    for (int s = 0; s < nseg; s++) {
      int col = segs[s]->column_index(n);
      if (col < 0) {
        std::lock_guard<std::mutex> g(segs[s]->derive_mu);
        if (int rc = derive_locked(ctx, segs[s], n, &col)) return rc;
      }
      if (first < 0) first = col;
      else if (col != first) {
        set_error("expression '%s' is column %d of one segment and %d of another: derive expressions in one order on every segment", n, first, col);
        return PB200_E_UNSUPPORTED;
      }
    }
  }
  return PB200_OK;
}

int derive_query_names(pb200_ctx* ctx, const pb200h_query& q, pb200h_segment* const* segs, int nseg, const char* const* extra, int nextra) {
  std::vector<const char*> names;
  // a leaf on an expression over several columns is evaluated per row (expr_filters.cpp), not derived
  for (int i = 0; i < q.num_filter_nodes; i++)
    if (q.filter[i].type >= PB200H_EQ && !is_expression_filter(q.filter[i].column)) names.push_back(q.filter[i].column);
  for (int g = 0; g < q.num_group_by; g++) names.push_back(q.group_by[g]);
  for (int a = 0; a < q.num_aggs; a++)   // an expression over several columns is computed per row, not derived
    if (q.aggs && q.aggs[a].function != PB200_AGG_COUNT && !(expression_function(q.aggs[a].function) && is_multi_column_expression(q.aggs[a].column)))
      names.push_back(q.aggs[a].column);
  if (q.agg_filter_count && q.agg_filter_start && q.agg_filter_nodes)
    for (int a = 0; a < q.num_aggs; a++)
      for (int k = 0; k < q.agg_filter_count[a]; k++) {
        const pb200h_filter_node& n = q.agg_filter_nodes[q.agg_filter_start[a] + k];
        if (n.type >= PB200H_EQ && !is_expression_filter(n.column)) names.push_back(n.column);
      }
  for (int k = 0; k < nextra; k++) names.push_back(extra[k]);
  return derive_names(ctx, segs, nseg, names);
}

}  // namespace pb200h

extern "C" int32_t pb200h_segment_derive(pb200_ctx* ctx, pb200h_segment* seg, const char* expression, int32_t* column) {
  if (!ctx || !seg || !expression || !column) { set_error("invalid argument to pb200h_segment_derive"); return PB200_E_INVALID; }
  std::lock_guard<std::mutex> g(seg->derive_mu);
  int col = -1;
  if (int rc = derive_locked(ctx, seg, expression, &col)) return rc;
  *column = col;
  return PB200_OK;
}
