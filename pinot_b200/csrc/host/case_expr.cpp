// case_expr.cpp -- CASE WHEN inside aggregation arguments (DESIGN.md section 3.19): the host half.
//
// transform.cpp compiles `case(c1,v1,...,e)` to a program whose PB200_T_COND leaves name condition leaves.  Here each
// leaf is resolved on every segment to the dictIds it matches, by the WHERE planner's own rule (matching_dict_ids: exact
// value-to-dictId resolution, REGEXP_LIKE / LIKE through the call's pattern scope), and handed to the device as a dictId
// range when the ids are contiguous and as a bitset otherwise.  The device never compares values.
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "host_internal.h"

namespace pb200h {

namespace {

// pb200h_literal of a condition literal on a numeric column (plan_maker.py numeric_literal); false when it is no number
bool numeric(const std::string& t, pb200h_literal* l, bool* integer_text) {
  if (t.empty()) return false;
  char* end = nullptr;
  errno = 0;
  const long long v = strtoll(t.c_str(), &end, 10);
  *integer_text = *end == 0 && end != t.c_str();
  l->s = nullptr;
  if (*integer_text && errno == 0) { l->i = v; l->d = (double)v; return true; }
  const double d = strtod(t.c_str(), &end);
  if (*end != 0 || end == t.c_str() || std::isnan(d)) return false;
  l->d = d;
  l->i = std::isfinite(d) && d == std::floor(d) && d >= -9223372036854775808.0 && d < 9223372036854775808.0 && !*integer_text ? (int64_t)d : 0;
  return true;
}

// sql.py's like_to_regexp: Pinot's RegexpPatternConverterUtils.likeToRegexpLike without escapes
bool like_to_regexp(const std::string& like, std::string* re) {
  if (like.find('\\') != std::string::npos) return false;
  if (like.empty()) { *re = "^$"; return true; }
  if (like.find_first_not_of('%') == std::string::npos) { *re = ""; return true; }
  const size_t lead = like.find_first_not_of('%'), end = like.find_last_not_of('%') + 1;
  std::string body;
  for (size_t k = lead; k < end; k++) {
    const char ch = like[k];
    if (ch == '%') body += ".*";
    else if (ch == '_') body += ".";
    else { if (strchr("\\.^$|?*+()[]{}", ch)) body += '\\'; body += ch; }
  }
  *re = (lead ? "" : "^") + body + (end < like.size() ? "" : "$");
  return true;
}

// FLOAT / DOUBLE dictionaries holding NaN or -0.0: Java's typed compare and Double.compare disagree there
bool has_nan_or_negative_zero(const HostColumn& c) {
  for (int id = 0; id < c.cardinality; id++) {
    const double x = c.as_double(id);
    if (x != x || (x == 0 && std::signbit(x))) return true;
  }
  return false;
}

}  // namespace

int case_result_type_check(const pb200h_segment& s0, const std::vector<CaseBranch>& branches, const char* text) {
  bool fl = false, wide = false, dbl = false;
  for (const CaseBranch& b : branches) {
    int type = -1;
    if (b.kind == CaseBranch::COLUMN) {
      const int ci = s0.column_index(b.column.c_str());
      if (ci >= 0) type = s0.cols[ci].data_type;
    }
    fl |= type == PB200_FLOAT;
    dbl |= type == PB200_DOUBLE || b.kind == CaseBranch::ARITHMETIC || b.kind == CaseBranch::DOUBLE_LITERAL;
    wide |= type == PB200_INT || type == PB200_LONG || (b.kind == CaseBranch::LONG_LITERAL && (b.value > (1ll << 24) || b.value < -(1ll << 24)));
  }
  if (fl && wide && !dbl) {
    set_error("'%s': a FLOAT branch next to INT / LONG branches or integers beyond 2^24 has a result type this library does not restate", text);
    return PB200_E_UNSUPPORTED;
  }
  return PB200_OK;
}

int case_condition_ids(const HostColumn& c, const CaseCond& cc, std::vector<int32_t>* ids) {
  const bool pattern = cc.fn == "like" || cc.fn == "regexp_like";
  const bool range = cc.fn == "less_than" || cc.fn == "less_than_or_equal" || cc.fn == "greater_than" || cc.fn == "greater_than_or_equal" || cc.fn == "between";
  const int type = c.data_type;
  if (type == PB200_STRING && range) { set_error("CASE condition %s on STRING column '%s': a STRING range is not accelerated", cc.fn.c_str(), cc.column.c_str()); return PB200_E_UNSUPPORTED; }
  if (type != PB200_STRING && pattern) { set_error("CASE condition %s on column '%s', which is not STRING", cc.fn.c_str(), cc.column.c_str()); return PB200_E_UNSUPPORTED; }
  if (!c.has_dictionary) { set_error("CASE condition on raw column '%s' (no dictionary) is not accelerated", c.name.c_str()); return PB200_E_UNSUPPORTED; }
  if ((type == PB200_FLOAT || type == PB200_DOUBLE) && has_nan_or_negative_zero(c)) {
    set_error("CASE condition on '%s': its dictionary holds NaN or -0.0", c.name.c_str());
    return PB200_E_UNSUPPORTED;
  }
  // the leaf as a WHERE predicate
  pb200h_filter_node n;
  memset(&n, 0, sizeof n);
  n.column = cc.column.c_str();
  std::vector<pb200h_literal> lits(cc.literals.size());
  std::string regex;
  if (pattern) {
    if (!case_pattern(cc, &regex)) { set_error("LIKE pattern '%s' contains a backslash: LIKE escapes are not supported", cc.literals[0].c_str()); return PB200_E_UNSUPPORTED; }
    lits[0].s = regex.c_str();
    n.type = PB200H_REGEXP_LIKE;
    n.num_values = 1;
    if (!pattern_ids(c, regex.c_str())) { set_error("CASE condition %s on '%s' was not resolved before planning", cc.fn.c_str(), cc.column.c_str()); return PB200_E_INVALID; }
  } else {
    for (size_t j = 0; j < cc.literals.size(); j++) {
      if (type == PB200_STRING) { lits[j].s = cc.literals[j].c_str(); continue; }
      bool integer_text = false;
      if (!numeric(cc.literals[j], &lits[j], &integer_text)) { set_error("CASE condition on numeric column '%s': literal '%s' is not a number", cc.column.c_str(), cc.literals[j].c_str()); return PB200_E_UNSUPPORTED; }
      if (type == PB200_LONG && !integer_text && std::fabs(lits[j].d) >= 9007199254740992.0) {
        set_error("CASE condition on LONG column '%s': the non-integral literal '%s' lies beyond 2^53", cc.column.c_str(), cc.literals[j].c_str());
        return PB200_E_UNSUPPORTED;
      }
    }
    n.num_values = (int)lits.size();
    if (cc.fn == "equals") n.type = PB200H_EQ;
    else if (cc.fn == "not_equals") n.type = PB200H_NEQ;
    else if (cc.fn == "in") n.type = PB200H_IN;
    else if (cc.fn == "not_in") n.type = PB200H_NOT_IN;
    else {
      n.type = PB200H_RANGE;
      n.num_values = 2;
      const bool lower = cc.fn == "greater_than" || cc.fn == "greater_than_or_equal" || cc.fn == "between";
      const bool upper = cc.fn == "less_than" || cc.fn == "less_than_or_equal" || cc.fn == "between";
      if (cc.fn != "between") lits.push_back(lits[0]);   // [lower, upper]: the one literal on its side
      n.lower_unbounded = !lower; n.upper_unbounded = !upper;
      n.lower_inclusive = cc.fn != "greater_than";
      n.upper_inclusive = cc.fn != "less_than";
    }
  }
  *ids = matching_dict_ids(c, n, lits.data());
  return PB200_OK;
}

bool case_pattern(const CaseCond& cc, std::string* regex) {
  if (cc.fn == "regexp_like") { *regex = cc.literals[0]; return true; }
  return like_to_regexp(cc.literals[0], regex);
}

int resolve_case_conditions(pb200_ctx* ctx, pb200h_segment* const* segs, int nseg, const std::vector<CaseCond>& leaves,
                            PatternScope& patterns, CaseTable& out) {
  out = CaseTable();
  if (leaves.empty()) return PB200_OK;
  if ((int)leaves.size() > PB200_MAX_EXPR_CONDS) { set_error("%zu CASE conditions in one query (at most %d)", leaves.size(), PB200_MAX_EXPR_CONDS); return PB200_E_UNSUPPORTED; }
  const pb200h_segment& s0 = *segs[0];
  out.args.resize(leaves.size());
  for (size_t k = 0; k < leaves.size(); k++) {
    const CaseCond& cc = leaves[k];
    const int ci = s0.column_index(cc.column.c_str());
    if (ci < 0 || ci >= s0.num_stored) { set_error("CASE condition: unknown column '%s'", cc.column.c_str()); return PB200_E_INVALID; }
    std::string regex;
    if ((cc.fn == "like" || cc.fn == "regexp_like") && s0.cols[ci].data_type == PB200_STRING && case_pattern(cc, &regex)) {
      // pattern leaves: their ids on every segment of the call, once (patterns.cpp)
      pb200h_filter_node n;
      memset(&n, 0, sizeof n);
      n.type = PB200H_REGEXP_LIKE; n.column = cc.column.c_str(); n.num_values = 1;
      pb200h_literal lit{0, 0.0, regex.c_str()};
      pb200h_query q;
      memset(&q, 0, sizeof q);
      q.num_filter_nodes = 1; q.filter = &n; q.literals = &lit;
      if (int rc = resolve_patterns(ctx, q, segs, nseg, patterns)) return rc;
    }
    std::vector<std::vector<int32_t>> ids(nseg);   // device dictIds per segment
    bool contiguous = true;
    for (int s = 0; s < nseg; s++) {
      const HostColumn& c = segs[s]->cols[ci];
      if (int rc = case_condition_ids(c, cc, &ids[s])) return rc;
      for (int32_t& id : ids[s]) id = c.to_device_id(id);
      contiguous &= ids[s].empty() || ids[s].back() - ids[s].front() + 1 == (int32_t)ids[s].size();
    }
    // one kind per condition: a range when the ids are contiguous in every segment, else a bitset per segment
    out.conds.push_back(pb200_expr_cond{ci, contiguous ? PB200_COND_RANGE : PB200_COND_BITSET, nullptr});
    for (int s = 0; s < nseg; s++) {
      const std::vector<int32_t>& v = ids[s];
      if (contiguous) {
        out.args[k].push_back(v.empty() ? 0 : v.front());
        out.args[k].push_back(v.empty() ? 0 : v.back() + 1);
        continue;
      }
      const int64_t first = (int64_t)out.words.size(), words = ((int64_t)segs[s]->cols[ci].decode_column().cardinality + 31) / 32;
      out.words.resize(out.words.size() + (size_t)words, 0u);
      for (int32_t id : v) out.words[(size_t)first + (size_t)(id >> 5)] |= 1u << (id & 31);
      out.args[k].push_back(first);
      out.args[k].push_back(words);
    }
  }
  for (size_t k = 0; k < leaves.size(); k++) out.conds[k].args = out.args[k].data();
  out.table = pb200_expr_conds{(int32_t)out.conds.size(), 0, out.conds.data(), (int64_t)out.words.size(), out.words.empty() ? nullptr : out.words.data()};
  return PB200_OK;
}

}  // namespace pb200h
