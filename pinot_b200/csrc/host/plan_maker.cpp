// plan_maker.cpp -- native mirror of the JVM-side half of the path (see include/pinot_b200_host.h).
//
// Restates the DECISIONS of (not the code of):
//   core/plan/FilterPlanNode.java:195-320            predicate -> leaf filter operator
//   core/operator/filter/FilterOperatorUtils.java:74-196   leaf choice, AND/OR/NOT simplification
//   core/operator/filter/predicate/*PredicateEvaluatorFactory.java   value -> dictId sets, alwaysTrue/alwaysFalse
//   core/plan/AggregationPlanNode.java:90-121,159-190      NonScanBasedAggregationOperator shortcut
// and hands dictId-space trees to the device through include/pinot_b200.h only.
#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <numeric>
#include <sstream>
#include <string>
#include <vector>

#include "host_internal.h"

using pb200::set_error;

static inline uint32_t be32(const unsigned char* p) { return pb200h::hbe32(p); }
static inline uint64_t be64(const unsigned char* p) { return pb200h::hbe64(p); }

using namespace pb200h;

namespace {

// ---- dictId-space predicate (PredicateEvaluator) -----------------------------------------------------------------
struct Evaluated {
  bool always_true = false, always_false = false, exclusive = false, is_range = false;
  int start = 0, end = 0;       // RANGE [start, end)
  std::vector<int32_t> ids;     // EQ/IN matching ids; NEQ/NOT_IN NON-matching ids (sorted)
};

// The FLOAT / DOUBLE columns the reference has no dictionary for, so it evaluates their predicates per value with Java's
// <, > and == (the *RawValueBased*PredicateEvaluators), not by a dictionary search: a column the segment stores raw, with
// a dictionary synthesised at load, and a DOUBLE expression (ExpressionFilterOperator evaluates it per row), whose
// dictionary the derivation built.  So NaN matches only NEQ / NOT_IN, and 0 matches both zeros.  The matching entries are
// found by one pass over the dictionary; both dictionaries are in Double.compare order with one NaN entry, last, so for a
// RANGE they are contiguous (the zeros are neighbours and NaN, which no range matches, is last).
bool compared_by_value(const HostColumn& c) {
  return (c.synthesized_dictionary || c.derived) && (c.data_type == PB200_FLOAT || c.data_type == PB200_DOUBLE);
}

bool raw_value_matches(const HostColumn& c, int id, const pb200h_filter_node& n, const pb200h_literal* v) {
  const bool fl = c.data_type == PB200_FLOAT;
  const double x = c.as_double(id);
  auto lt = [&](const pb200h_literal& l) { return fl ? (float)x < (float)l.d : x < l.d; };
  auto gt = [&](const pb200h_literal& l) { return fl ? (float)x > (float)l.d : x > l.d; };
  auto eq = [&](const pb200h_literal& l) { return fl ? (float)x == (float)l.d : x == l.d; };
  if (n.type == PB200H_RANGE) {
    if (!n.lower_unbounded && !(n.lower_inclusive ? gt(v[0]) || eq(v[0]) : gt(v[0]))) return false;
    if (!n.upper_unbounded && !(n.upper_inclusive ? lt(v[1]) || eq(v[1]) : lt(v[1]))) return false;
    return x == x;  // an unbounded range matches no NaN either
  }
  for (int i = 0; i < n.num_values; i++) if (eq(v[i])) return true;  // EQ / IN match; NEQ / NOT_IN: the excluded values
  return false;
}

Evaluated evaluate(const HostColumn& c, const pb200h_filter_node& n, const pb200h_literal* lits) {
  Evaluated e;
  const pb200h_literal* v = lits + n.values_offset;
  const int card = c.cardinality;
  if (n.type == PB200H_REGEXP_LIKE) {   // resolved before planning (patterns.cpp): an IN over the matching ids
    if (const std::vector<int32_t>* m = pattern_ids(c, v[0].s)) e.ids = *m;
    const int k = (int)e.ids.size();
    if (k == 0) e.always_false = true; else if (k == card) e.always_true = true;
    return e;
  }
  if (compared_by_value(c)) {
    e.is_range = n.type == PB200H_RANGE;
    e.exclusive = n.type == PB200H_NEQ || n.type == PB200H_NOT_IN;
    for (int id = 0; id < card; id++) if (raw_value_matches(c, id, n, v)) e.ids.push_back(id);
    const int k = (int)e.ids.size();
    if (e.is_range) {
      e.start = k ? e.ids.front() : 0;
      e.end = k ? e.ids.back() + 1 : 0;
      e.ids.clear();
      if (k == 0) e.always_false = true; else if (k == card) e.always_true = true;
    } else if (!e.exclusive) {
      if (k == 0) e.always_false = true; else if (k == card) e.always_true = true;
    } else {
      if (k == 0) e.always_true = true; else if (k == card) e.always_false = true;
    }
    return e;
  }
  if (n.type == PB200H_RANGE) {  // SortedDictionaryBasedRangePredicateEvaluator :126-168
    e.is_range = true;
    if (n.lower_unbounded) e.start = 0;
    else { int ii = c.insertion_index_of(v[0]); e.start = ii < 0 ? -(ii + 1) : (n.lower_inclusive ? ii : ii + 1); }
    if (n.upper_unbounded) e.end = card;
    else { int ii = c.insertion_index_of(v[1]); e.end = ii < 0 ? -(ii + 1) : (n.upper_inclusive ? ii + 1 : ii); }
    int nm = std::max(e.end - e.start, 0);
    if (nm == 0) e.always_false = true; else if (nm == card) e.always_true = true;
    return e;
  }
  e.exclusive = n.type == PB200H_NEQ || n.type == PB200H_NOT_IN;
  for (int i = 0; i < n.num_values; i++) { int id = c.insertion_index_of(v[i]); if (id >= 0) e.ids.push_back(id); }
  std::sort(e.ids.begin(), e.ids.end());
  e.ids.erase(std::unique(e.ids.begin(), e.ids.end()), e.ids.end());
  const int k = (int)e.ids.size();
  if (!e.exclusive) { if (k == 0) e.always_false = true; else if (k == card) e.always_true = true; }
  else { if (k == 0) e.always_true = true; else if (k == card) e.always_false = true; }
  return e;
}


// Predicate on a raw (no-dictionary) INT column -> PB200_F_RAW_RANGE (value space).  EQ is the one-value range; NEQ / IN /
// NOT_IN and the other raw types stay with the reference's operator.
bool raw_leaf(const HostColumn& c, const pb200h_filter_node& n, const pb200h_literal* lits, pb200_filter_node& d) {
  if (c.data_type != PB200_INT) return false;
  const pb200h_literal* v = lits + n.values_offset;
  if (n.type == PB200H_RANGE) {
    d.op = PB200_F_RAW_RANGE;
    // the literals' doubles: fractional bounds reach pb200_execute as they are (it takes ceil / floor), and every int32
    // bound is exact (compare_integral)
    d.raw_lo = n.lower_unbounded ? 0.0 : v[0].d;
    d.raw_hi = n.upper_unbounded ? 0.0 : v[1].d;
    d.raw_flags = (n.lower_unbounded ? 1 : 0) | (n.upper_unbounded ? 2 : 0) | (n.lower_inclusive ? 0 : 4) | (n.upper_inclusive ? 0 : 8);
    return true;
  }
  // EQ with a fractional literal: [ceil, floor] is empty
  if (n.type == PB200H_EQ) { d.op = PB200_F_RAW_RANGE; d.raw_lo = d.raw_hi = v[0].d; d.raw_flags = 0; return true; }
  return false;
}

// A pattern leaf is planned from the ids its call resolved (resolve_patterns); one that was not is a caller's error
int check_resolved(const HostColumn& c, const pb200h_filter_node& n, const pb200h_literal* lits) {
  if (n.type != PB200H_REGEXP_LIKE || pattern_ids(c, lits[n.values_offset].s)) return PB200_OK;
  set_error("REGEXP_LIKE leaf on '%s' was not resolved before planning", c.name.c_str());
  return PB200_E_INVALID;
}

// One segment's device filter tree + the arrays its nodes point to.
struct SegmentFilter {
  std::vector<pb200_filter_node> nodes;
  std::vector<std::unique_ptr<std::vector<int32_t>>> id_store;
  bool root_empty = false, root_all = false;
};

// SortedIndexBasedFilterOperator.getNextBlockWithoutNullHandling :60-135 -> inclusive docId ranges
std::vector<int32_t> sorted_doc_ranges(const HostColumn& c, const Evaluated& e, int num_docs) {
  std::vector<std::pair<int, int>> r;
  if (e.is_range) {
    r.push_back({c.sorted_start(e.start), c.sorted_end(e.end - 1)});
  } else {
    std::pair<int, int> last{c.sorted_start(e.ids[0]), c.sorted_end(e.ids[0])};
    for (size_t i = 1; i < e.ids.size(); i++) {
      std::pair<int, int> cur{c.sorted_start(e.ids[i]), c.sorted_end(e.ids[i])};
      if (cur.first == last.second + 1) last.second = cur.second; else { r.push_back(last); last = cur; }
    }
    r.push_back(last);
    if (e.exclusive) {
      std::vector<std::pair<int, int>> inv;
      if (r[0].first > 0) inv.push_back({0, r[0].first - 1});
      for (size_t i = 0; i + 1 < r.size(); i++) inv.push_back({r[i].second + 1, r[i + 1].first - 1});
      if (r.back().second < num_docs - 1) inv.push_back({r.back().second + 1, num_docs - 1});
      r = inv;
    }
  }
  std::vector<int32_t> flat;
  for (auto& p : r) { flat.push_back(p.first); flat.push_back(p.second); }
  return flat;
}

// Builds the per-segment tree with the SAME SHAPE as the query's tree (the device kernel shares one boolean program
// across segments); what FilterOperatorUtils would simplify away becomes MATCH_ALL / EMPTY leaves, and the root's
// constant-ness is tracked separately for the plan shortcuts.
int build_segment_filter(const pb200h_segment& seg, const pb200h_query& q, SegmentFilter& out, std::string* explain) {
  out.nodes.resize(q.num_filter_nodes);
  std::vector<int> constant;  // per stack entry: 0 unknown, 1 all, 2 empty
  std::vector<std::string> text;
  for (int i = 0; i < q.num_filter_nodes; i++) {
    const pb200h_filter_node& n = q.filter[i];
    pb200_filter_node& d = out.nodes[i];
    memset(&d, 0, sizeof d);
    if (n.type == PB200H_AND || n.type == PB200H_OR) {
      d.op = n.type == PB200H_AND ? PB200_F_AND : PB200_F_OR;
      d.num_children = n.num_children;
      if (n.num_children < 1 || (int)constant.size() < n.num_children) { set_error("malformed filter tree"); return PB200_E_INVALID; }
      bool any_all = false, any_empty = false, all_all = true, all_empty = true;
      std::string t = n.type == PB200H_AND ? "FILTER_AND(" : "FILTER_OR(";
      for (int k = 0; k < n.num_children; k++) {
        int c = constant[constant.size() - n.num_children + k];
        any_all |= c == 1; any_empty |= c == 2; all_all &= c == 1; all_empty &= c == 2;
        t += (k ? "," : "") + text[text.size() - n.num_children + k];
      }
      t += ")";
      constant.resize(constant.size() - n.num_children);
      text.resize(text.size() - n.num_children);
      int c = 0;
      if (n.type == PB200H_AND) c = any_empty ? 2 : (all_all ? 1 : 0); else c = any_all ? 1 : (all_empty ? 2 : 0);
      constant.push_back(c);
      text.push_back(c == 1 ? "FILTER_MATCH_ENTIRE_SEGMENT" : c == 2 ? "FILTER_EMPTY" : t);
      continue;
    }
    if (n.type == PB200H_NOT) {
      d.op = PB200_F_NOT;
      d.num_children = 1;
      if (constant.empty()) { set_error("malformed filter tree"); return PB200_E_INVALID; }
      int c = constant.back();
      constant.back() = c == 1 ? 2 : c == 2 ? 1 : 0;
      text.back() = c == 1 ? "FILTER_EMPTY" : c == 2 ? "FILTER_MATCH_ENTIRE_SEGMENT" : "FILTER_NOT(" + text.back() + ")";
      continue;
    }
    const char* pname = n.type == PB200H_RANGE ? "RANGE" : n.type == PB200H_EQ ? "EQ" : n.type == PB200H_NEQ ? "NOT_EQ" : n.type == PB200H_IN ? "IN" : n.type == PB200H_NOT_IN ? "NOT_IN" : "REGEXP_LIKE";
    if (is_expression_filter(n.column)) {
      // an expression over several columns (DESIGN.md section 3.16): the doc set its call computed on the device, the
      // same leaf in every segment and never folded to a constant
      std::string canonical;
      const uint32_t* mask = nullptr;
      int ncols = 0;
      if (n.type == PB200H_REGEXP_LIKE) { set_error("REGEXP_LIKE / LIKE on the expression '%s' is not accelerated", n.column); return PB200_E_UNSUPPORTED; }
      if (int rc = expr_filter_mask(seg, n, q.literals, &canonical, &mask, &ncols)) return rc;
      if (!mask && !explain) { set_error("predicate on the expression '%s' was not resolved before planning", n.column); return PB200_E_INVALID; }
      d.op = PB200_F_DOC_MASK;
      d.column = -1;
      d.ids = reinterpret_cast<const int32_t*>(mask);
      d.num_ids = (int32_t)pb200::doc_mask_words(seg.num_docs);
      d.reserved = PB200_NODE_IDS_ON_DEVICE;
      constant.push_back(0);
      text.push_back(std::string("FILTER_EXPRESSION(") + pname + "," + canonical + ")");
      continue;
    }
    const int ci = seg.column_index(n.column);
    if (ci < 0) { set_error("unknown column '%s'", n.column ? n.column : "(null)"); return PB200_E_INVALID; }
    const HostColumn& c = seg.cols[ci];
    if (!c.has_dictionary) {
      d.column = ci;
      if (!raw_leaf(c, n, q.literals, d)) { set_error("this predicate on raw column '%s' is not accelerated", c.name.c_str()); return PB200_E_UNSUPPORTED; }
      constant.push_back(0);
      text.push_back(std::string("FILTER_FULL_SCAN(") + (n.type == PB200H_RANGE ? "RANGE," : "EQ,") + c.name + ")");
      continue;
    }
    if (int rc = check_resolved(c, n, q.literals)) return rc;
    Evaluated e = evaluate(c, n, q.literals);
    d.column = ci;
    if (e.always_false) { d.op = PB200_F_EMPTY; constant.push_back(2); text.push_back("FILTER_EMPTY"); continue; }
    if (e.always_true) { d.op = PB200_F_MATCH_ALL; constant.push_back(1); text.push_back("FILTER_MATCH_ENTIRE_SEGMENT"); continue; }
    constant.push_back(0);
    auto store = [&](std::vector<int32_t> v) {
      out.id_store.emplace_back(new std::vector<int32_t>(std::move(v)));
      d.ids = out.id_store.back()->data();
      d.num_ids = (int)out.id_store.back()->size();
    };
    if (c.is_sorted) {  // FilterOperatorUtils :98-101,117-120
      store(sorted_doc_ranges(c, e, seg.num_docs));
      d.op = PB200_F_DOC_RANGES;
      text.push_back(std::string("FILTER_SORTED_INDEX(") + pname + "," + c.name + ")");
    } else if (n.type == PB200H_RANGE) {
      // bound column: the local range [start, end) is the domain range [id(start), id(end-1)] for this segment's rows
      d.op = PB200_F_SCAN_RANGE; d.lo = c.to_device_id(e.start); d.hi = c.to_device_id(e.end - 1) + 1;
      text.push_back(std::string("FILTER_FULL_SCAN(RANGE,") + c.name + ",[" + std::to_string(e.start) + "," + std::to_string(e.end) + "))");
    } else if (c.has_inverted) {  // :121-124
      for (auto& id : e.ids) id = c.to_device_id(id);
      store(e.ids);
      d.op = e.exclusive ? PB200_F_INV_NOT_IN : PB200_F_INV_IN;
      text.push_back(std::string("FILTER_INVERTED_INDEX(") + pname + "," + c.name + ")");
    } else {
      for (auto& id : e.ids) id = c.to_device_id(id);
      store(e.ids);
      d.op = e.exclusive ? PB200_F_SCAN_NOT_IN : PB200_F_SCAN_IN;
      text.push_back(std::string("FILTER_FULL_SCAN(") + pname + "," + c.name + ")");
    }
  }
  if (q.num_filter_nodes == 0) { out.root_all = true; if (explain) *explain = "FILTER_MATCH_ENTIRE_SEGMENT"; return PB200_OK; }
  if (constant.size() != 1) { set_error("malformed filter tree"); return PB200_E_INVALID; }
  out.root_all = constant[0] == 1;
  out.root_empty = constant[0] == 2;
  if (explain) *explain = text[0];
  return PB200_OK;
}

// AggregationPlanNode.java:159-184: filter matches all and every function is answerable from dictionary / metadata
bool non_scan_answerable(const pb200h_segment& seg, const pb200h_query& q) {
  if (q.num_group_by > 0) return false;
  for (int a = 0; a < q.num_aggs; a++) {
    const pb200h_agg& ag = q.aggs[a];
    if (ag.function == PB200_AGG_COUNT) continue;
    const bool set_fn = ag.function == PB200_AGG_DISTINCTCOUNT || ag.function == PB200_AGG_DISTINCTCOUNTHLL;
    if (ag.function != PB200_AGG_MIN && ag.function != PB200_AGG_MAX && !set_fn) return false;
    int ci = seg.column_index(ag.column);
    if (ci < 0 || !seg.cols[ci].has_dictionary) return false;
    // a derived column's dictionary may hold values absent from the segment (derived over a domain), and the reference
    // takes this shortcut for identifiers only
    if (seg.cols[ci].derived) return false;
    if (!set_fn && seg.cols[ci].data_type == PB200_STRING) return false;
  }
  return true;
}

pb200_result* host_result(const pb200h_segment& seg, const pb200h_query& q, bool empty) {
  auto* R = new pb200_result();
  const int nagg = q.num_aggs;
  R->meta.num_groups = q.num_group_by > 0 ? 0 : -1;
  R->meta.num_group_by = q.num_group_by;
  R->meta.num_aggs = nagg;
  R->meta.num_total_docs = seg.num_docs;
  R->meta.num_docs_scanned = empty ? 0 : seg.num_docs;  // NonScanBasedAggregationOperator reports numTotalDocs
  R->dbl.resize(nagg); R->lng.resize(nagg); R->ids.resize(nagg); R->distinct.resize(nagg);
  if (q.num_group_by > 0) return R;
  for (int a = 0; a < nagg; a++) {
    const pb200h_agg& ag = q.aggs[a];
    double d = 0; int64_t l = 0; int32_t id = -1;
    // MIN / MAX read the column's dictionary; an expression argument has no column here (its aggregation is never
    // answered without a scan, so only an empty match reaches this)
    const int ci = ag.column ? seg.column_index(ag.column) : -1;
    const HostColumn* c = ci >= 0 ? &seg.cols[ci] : nullptr;
    switch (ag.function) {
      case PB200_AGG_COUNT: l = empty ? 0 : seg.num_docs; d = (double)l; break;
      case PB200_AGG_SUM: case PB200_AGG_AVG: d = 0; l = 0; break;
      case PB200_AGG_MIN: if (empty || !c) d = INFINITY; else { id = c->to_device_id(0); d = c->as_double(0); } break;
      case PB200_AGG_MAX: if (empty || !c) d = -INFINITY; else { id = c->to_device_id(c->cardinality - 1); d = c->as_double(c->cardinality - 1); } break;
      case PB200_AGG_PERCENTILE: d = -INFINITY; break;   // only reached for an empty match (never answered without a scan)
      case PB200_AGG_FIRSTWITHTIME: case PB200_AGG_LASTWITHTIME: d = -INFINITY; break;   // likewise: no row, dictId -1
      case PB200_AGG_VARPOP: case PB200_AGG_VARSAMP: case PB200_AGG_STDDEVPOP: case PB200_AGG_STDDEVSAMP:
        d = -INFINITY; R->mom.on[a] = true; break;       // likewise: n = 0, zero moments
      case PB200_AGG_DISTINCTSUM: case PB200_AGG_DISTINCTAVG:   // only reached for an empty match: S is empty
        d = ag.function == PB200_AGG_DISTINCTSUM ? 0.0 : -INFINITY;
        R->distinct[a].push_back({});
        break;
      case PB200_AGG_DISTINCTCOUNTHLL:   // an empty S estimates 0; the whole dictionary's estimate is set by the caller
      case PB200_AGG_DISTINCTCOUNT: {
        std::vector<int32_t> ids;
        if (!empty) for (int i = 0; i < c->cardinality; i++) ids.push_back(c->to_device_id(i));
        if (ag.function == PB200_AGG_DISTINCTCOUNT) { l = (int64_t)ids.size(); d = (double)l; }
        R->distinct[a].push_back(std::move(ids));
        break;
      }
    }
    R->dbl[a].push_back(d); R->lng[a].push_back(l); R->ids[a].push_back(id);
  }
  return R;
}

}  // namespace

namespace pb200h {

std::string lower_fn_name(int fn) {
  std::string s = pb200::agg_fn(fn)->name;
  for (char& ch : s) ch = (char)std::tolower((unsigned char)ch);
  return s;
}

std::vector<int> aggs_by_family(const pb200h_query& q, std::initializer_list<int> first) {
  auto rank = [&](int a) {
    const pb200::AggFn* d = pb200::agg_fn(q.aggs[a].function);
    int r = 0;
    for (int fn : first) {
      if (d && strcmp(d->family, pb200::agg_fn(fn)->family) == 0) return r;
      r++;
    }
    return r;
  };
  std::vector<int> order(q.num_aggs);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return rank(x) < rank(y); });
  return order;
}

std::vector<int32_t> matching_dict_ids(const HostColumn& c, const pb200h_filter_node& n, const pb200h_literal* lits) {
  Evaluated e = evaluate(c, n, lits);
  std::vector<int32_t> ids;
  if (e.is_range) { for (int i = e.start; i < e.end; i++) ids.push_back(i); return ids; }
  if (!e.exclusive) return e.ids;
  size_t k = 0;
  for (int i = 0; i < c.cardinality; i++) {
    if (k < e.ids.size() && e.ids[k] == i) { k++; continue; }
    ids.push_back(i);
  }
  return ids;
}

int leaf_to_device(const pb200h_segment& seg, int column, const pb200h_filter_node& n, const pb200h_literal* lits,
                   SegmentFilterStore& store, pb200_filter_node& d) {
  memset(&d, 0, sizeof d);
  const HostColumn& c = seg.cols[column];
  if (!c.has_dictionary) {
    d.column = column;
    if (!raw_leaf(c, n, lits, d)) { set_error("this predicate on raw column '%s' is not accelerated", c.name.c_str()); return PB200_E_UNSUPPORTED; }
    return PB200_OK;
  }
  if (int rc = check_resolved(c, n, lits)) return rc;
  Evaluated e = evaluate(c, n, lits);
  d.column = column;
  if (e.always_false) { d.op = PB200_F_EMPTY; return PB200_OK; }
  if (e.always_true) { d.op = PB200_F_MATCH_ALL; return PB200_OK; }
  auto keep = [&](std::vector<int32_t> v) {
    store.ids.emplace_back(new std::vector<int32_t>(std::move(v)));
    d.ids = store.ids.back()->data();
    d.num_ids = (int)store.ids.back()->size();
  };
  if (c.is_sorted) { keep(sorted_doc_ranges(c, e, seg.num_docs)); d.op = PB200_F_DOC_RANGES; return PB200_OK; }
  if (n.type == PB200H_RANGE) { d.op = PB200_F_SCAN_RANGE; d.lo = c.to_device_id(e.start); d.hi = c.to_device_id(e.end - 1) + 1; return PB200_OK; }
  for (auto& id : e.ids) id = c.to_device_id(id);
  if (c.has_inverted) { keep(e.ids); d.op = e.exclusive ? PB200_F_INV_NOT_IN : PB200_F_INV_IN; }
  else { keep(e.ids); d.op = e.exclusive ? PB200_F_SCAN_NOT_IN : PB200_F_SCAN_IN; }
  return PB200_OK;
}

}  // namespace pb200h

// ------------------------------------------------------------------------------------------------------------------
// segments
// ------------------------------------------------------------------------------------------------------------------
extern "C" int32_t pb200h_segment_create(pb200_ctx* ctx, const char* name, int32_t num_docs, int32_t ncols,
                                         const pb200h_column* cols, pb200h_segment** out) {
  if (!ctx || !cols || !out || ncols <= 0) { set_error("invalid argument to pb200h_segment_create"); return PB200_E_INVALID; }
  std::unique_ptr<pb200h_segment> seg(new pb200h_segment());
  seg->ctx = ctx; seg->name = name ? name : ""; seg->num_docs = num_docs;
  seg->cols.reserve((size_t)ncols + PB200_MAX_DERIVED_COLUMNS);
  seg->num_stored = ncols;
  std::vector<pb200_col_desc> descs(ncols);
  // Raw (no-dictionary) columns: all chunks are decoded once here; a column with at most PB200_RAW_DICT_MAX (default 2^20)
  // distinct values is dictionary-encoded on the fly and is an ordinary dictionary column from here on (raw_forward.cpp)
  std::vector<std::vector<unsigned char>> owned_fwd(ncols), owned_dict(ncols);
  const int raw_dict_max = [&]() { std::lock_guard<std::mutex> g(ctx->mu); return ctx->tune.raw_dict_max; }();
  for (int i = 0; i < ncols; i++) {
    const pb200h_column& c = cols[i];
    HostColumn h;
    h.name = c.name ? c.name : "";
    h.data_type = c.data_type; h.has_dictionary = c.has_dictionary; h.bits = c.bits_per_value;
    h.cardinality = c.cardinality; h.is_sorted = c.is_sorted; h.entry_bytes = c.dict_entry_bytes;
    h.has_inverted = c.inv != nullptr && c.inv_bytes > 0 && !c.is_sorted;
    pb200_col_desc& d = descs[i];
    memset(&d, 0, sizeof d);
    if (!c.has_dictionary) {
      const int width = raw_value_width(c.data_type);
      if (width == 0) { set_error("raw column '%s' of type %d is not loadable (fixed-width numeric types only)", h.name.c_str(), c.data_type); return PB200_E_UNSUPPORTED; }
      std::vector<unsigned char> values;
      int rc = decode_fixed_byte_forward((const unsigned char*)c.fwd, c.fwd_bytes, width, num_docs, values);
      if (rc) return rc;
      int card = 0, nb = 0;
      if (raw_dict_max > 0 && synthesize_dictionary(values, c.data_type, num_docs, raw_dict_max, owned_dict[i], owned_fwd[i], &card, &nb)) {
        h.has_dictionary = 1; h.synthesized_dictionary = true; h.bits = nb; h.cardinality = card; h.entry_bytes = width;
        h.is_sorted = 0; h.has_inverted = false;
        h.dict = owned_dict[i];
        d.fwd_kind = PB200_FWD_DICT_FIXEDBIT;
        d.stored_type = c.data_type; d.bits_per_value = nb; d.cardinality = card;
        d.fwd = owned_fwd[i].data(); d.fwd_bytes = owned_fwd[i].size();
        d.dict = owned_dict[i].data(); d.dict_bytes = owned_dict[i].size();
      } else {
        wrap_pass_through(values, width, num_docs, owned_fwd[i]);
        d.fwd_kind = PB200_FWD_RAW_FIXEDBYTE;
        d.stored_type = c.data_type;
        d.fwd = owned_fwd[i].data(); d.fwd_bytes = owned_fwd[i].size();
      }
      seg->cols.push_back(std::move(h));
      continue;
    }
    if (c.dict && c.dict_bytes) h.dict.assign((const unsigned char*)c.dict, (const unsigned char*)c.dict + c.dict_bytes);
    if (c.is_sorted && c.fwd) h.sorted_idx.assign((const unsigned char*)c.fwd, (const unsigned char*)c.fwd + c.fwd_bytes);
    d.fwd_kind = c.is_sorted ? PB200_FWD_DICT_SORTED : PB200_FWD_DICT_FIXEDBIT;
    d.stored_type = c.data_type; d.bits_per_value = c.bits_per_value; d.cardinality = c.cardinality;
    d.fwd = c.fwd; d.fwd_bytes = c.fwd_bytes;
    d.dict = c.dict; d.dict_bytes = c.dict_bytes;  // STRING: kept on the host by the device layer too (hashing / domains)
    d.reserved = c.data_type == PB200_STRING ? c.dict_entry_bytes : 0;
    d.inv = h.has_inverted ? c.inv : nullptr; d.inv_bytes = h.has_inverted ? c.inv_bytes : 0;
    seg->cols.push_back(std::move(h));
  }
  int rc = pb200_segment_register(ctx, name, num_docs, ncols, descs.data(), &seg->dev);
  if (rc) return rc;
  seg->published.store(ncols, std::memory_order_release);
  *out = seg.release();
  return PB200_OK;
}

extern "C" int32_t pb200h_segment_adopt(pb200_ctx* ctx, pb200_segment* dev, int32_t num_docs, int32_t ncols,
                                        const char* const* names, pb200h_segment** out) {
  if (!ctx || !dev || !out || !names) { set_error("invalid argument to pb200h_segment_adopt"); return PB200_E_INVALID; }
  std::unique_ptr<pb200h_segment> seg(new pb200h_segment());
  seg->ctx = ctx; seg->dev = dev; seg->num_docs = num_docs;
  seg->cols.reserve((size_t)ncols + PB200_MAX_DERIVED_COLUMNS);
  seg->num_stored = ncols;
  for (int i = 0; i < ncols; i++) {
    int64_t info[6];
    int rc = pb200_segment_column_info(dev, i, info);
    if (rc) return rc;
    HostColumn h;
    h.name = names[i];
    h.data_type = (int)info[1]; h.has_dictionary = info[0] != PB200_FWD_RAW_FIXEDBYTE; h.bits = (int)info[2];
    h.cardinality = (int)info[3]; h.has_inverted = info[4] != 0;
    h.entry_bytes = (h.data_type == PB200_LONG || h.data_type == PB200_DOUBLE) ? 8 : 4;
    int64_t n = pb200_segment_read_index(ctx, dev, i, 1, nullptr, 0);
    if (n > 0) { h.dict.resize(n); pb200_segment_read_index(ctx, dev, i, 1, h.dict.data(), n); }
    seg->cols.push_back(std::move(h));
  }
  seg->published.store(ncols, std::memory_order_release);
  *out = seg.release();
  return PB200_OK;
}

extern "C" int32_t pb200h_segment_destroy(pb200h_segment* seg) {
  if (!seg) return PB200_OK;
  if (seg->dev) pb200_segment_release(seg->ctx, seg->dev);
  delete seg;
  return PB200_OK;
}
extern "C" pb200_segment* pb200h_segment_device(pb200h_segment* seg) { return seg ? seg->dev : nullptr; }
extern "C" int32_t pb200h_segment_num_docs(const pb200h_segment* seg) { return seg ? seg->num_docs : -1; }
extern "C" int32_t pb200h_segment_num_columns(const pb200h_segment* seg) { return seg ? seg->num_stored : -1; }  // stored columns only
extern "C" int32_t pb200h_segment_column_index(const pb200h_segment* seg, const char* name) { return seg ? seg->column_index(name) : -1; }
extern "C" const char* pb200h_segment_column_name(const pb200h_segment* seg, int32_t c) {
  return (seg && c >= 0 && c < seg->num_columns()) ? seg->cols[c].name.c_str() : nullptr;
}
extern "C" int32_t pb200h_segment_column_info(const pb200h_segment* seg, int32_t c, int32_t out[6]) {
  if (!seg || c < 0 || c >= seg->num_columns()) { set_error("bad column"); return PB200_E_INVALID; }
  const HostColumn& h = seg->cols[c];
  const HostColumn& g = h.decode_column();  // bound column: the id space results come back in is the domain's
  out[0] = h.data_type; out[1] = h.has_dictionary; out[2] = g.bits; out[3] = g.cardinality; out[4] = h.is_sorted; out[5] = h.has_inverted;
  return PB200_OK;
}
extern "C" int32_t pb200h_dictionary_get(const pb200h_segment* seg, int32_t c, int32_t id, double* num, int64_t* lng,
                                         char* str, int32_t cap) {
  if (!seg || c < 0 || c >= seg->num_columns()) { set_error("bad column"); return PB200_E_INVALID; }
  const HostColumn& h = seg->cols[c].decode_column();
  if (id < 0 || id >= h.cardinality || h.dict.empty()) { set_error("dictId %d out of range", id); return PB200_E_INVALID; }
  if (h.data_type == PB200_STRING) {
    std::string s = h.get_string(id);
    if (str && cap > 0) { size_t n = std::min<size_t>(s.size(), cap - 1); memcpy(str, s.data(), n); str[n] = 0; }
    return PB200_OK;
  }
  if (num) *num = h.as_double(id);
  if (lng) *lng = h.data_type == PB200_INT ? h.get_int(id) : h.data_type == PB200_LONG ? h.get_long(id) : (int64_t)h.as_double(id);
  return PB200_OK;
}

// ---- table-wide dictionaries (value space face of pb200_domain_*) --------------------------------------------------
extern "C" int32_t pb200h_domain_build(pb200_ctx* ctx, pb200h_segment* const* segs, int32_t nseg, int32_t ncols,
                                       const char* const* names, pb200_domain** out) {
  if (!ctx || !segs || !names || !out || nseg <= 0 || ncols <= 0) { set_error("invalid argument to pb200h_domain_build"); return PB200_E_INVALID; }
  std::vector<int32_t> cols(ncols);
  std::vector<pb200_segment*> dev(nseg);
  if (int rc = derive_names(ctx, segs, nseg, std::vector<const char*>(names, names + ncols))) return rc;
  for (int k = 0; k < ncols; k++) {
    cols[k] = segs[0]->column_index(names[k]);
    if (cols[k] < 0) { set_error("unknown column '%s'", names[k] ? names[k] : "(null)"); return PB200_E_INVALID; }
    for (int s = 0; s < nseg; s++) {
      if (segs[s]->column_index(names[k]) != cols[k]) { set_error("column '%s' is not at the same position in every segment", names[k]); return PB200_E_INVALID; }
      if (!segs[s]->cols[cols[k]].has_dictionary) { set_error("column '%s' has no dictionary", names[k]); return PB200_E_INVALID; }
    }
  }
  for (int s = 0; s < nseg; s++) dev[s] = segs[s]->dev;
  return pb200_domain_from_segments(ctx, dev.data(), nseg, ncols, cols.data(), out);
}

extern "C" int32_t pb200h_segment_bind_domain(pb200_ctx* ctx, pb200h_segment* seg, pb200_domain* dom) {
  if (!ctx || !seg || !dom) { set_error("invalid argument to pb200h_segment_bind_domain"); return PB200_E_INVALID; }
  if (!seg->star_trees.empty()) { set_error("segment '%s' has star-trees (their dimension columns share the base dictionaries): not bindable", seg->name.c_str()); return PB200_E_UNSUPPORTED; }
  int rc = pb200_segment_bind_domain(ctx, seg->dev, dom);
  if (rc) return rc;
  for (const auto& dc : dom->cols) {
    HostColumn& h = seg->cols[dc.column];
    auto g = std::make_shared<HostColumn>();
    g->name = h.name; g->data_type = dc.stored_type; g->has_dictionary = 1; g->bits = dc.bits;
    g->cardinality = dc.cardinality; g->entry_bytes = dc.entry_bytes; g->dict = dc.dict_be;
    h.global = g;
    const auto& ids = seg->dev->cols[dc.column].local_ids;
    h.local_ids.assign(ids.begin(), ids.end());
  }
  return PB200_OK;
}

// ---- segment directory loader (V1Constants: metadata.properties, v1 file-per-index, v3 columns.psf + index_map) ----
namespace {
bool read_file(const std::string& p, std::vector<unsigned char>& out) {
  std::ifstream f(p, std::ios::binary);
  if (!f) return false;
  f.seekg(0, std::ios::end);
  std::streamoff n = f.tellg();
  f.seekg(0);
  out.resize((size_t)n);
  if (n) f.read((char*)out.data(), n);
  return (bool)f;
}
std::string trim(const std::string& s) {
  size_t a = s.find_first_not_of(" \t\r"), b = s.find_last_not_of(" \t\r");
  return a == std::string::npos ? std::string() : s.substr(a, b - a + 1);
}
// commons-configuration properties: list values are written either as repeated keys or comma separated; `lists` (optional)
// collects every value of a key in file order, the plain map keeps the last one
std::map<std::string, std::string> read_properties(const std::string& p, std::map<std::string, std::vector<std::string>>* lists = nullptr) {
  std::map<std::string, std::string> m;
  std::ifstream f(p);
  std::string line;
  while (std::getline(f, line)) {
    if (line.empty() || line[0] == '#') continue;
    size_t eq = line.find('=');
    if (eq == std::string::npos) continue;
    const std::string k = trim(line.substr(0, eq)), v = trim(line.substr(eq + 1));
    m[k] = v;
    if (lists) {
      size_t start = 0;
      while (start <= v.size()) {
        size_t comma = v.find(',', start);
        std::string item = trim(v.substr(start, comma == std::string::npos ? std::string::npos : comma - start));
        if (!item.empty()) (*lists)[k].push_back(item);
        if (comma == std::string::npos) break;
        start = comma + 1;
      }
    }
  }
  return m;
}

// StarTreeV2 files of a segment directory (seglocal/startree/v2/store/StarTreeIndexMapUtils.java: `star_tree_index_map`
// lines "<tree>.<column>.<FORWARD_INDEX|STAR_TREE>.<OFFSET|SIZE> = n", the tree itself under column "null";
// metadata.properties keys startree.v2.count / .<t>.total.docs / .split.order / .function.column.pairs): every tree whose
// dimensions are loaded columns is attached; function-column pairs other than COUNT / SUM / MIN / MAX are skipped.
void attach_star_trees_from_dir(pb200_ctx* ctx, const std::string& dir, pb200h_segment* seg) {
  std::map<std::string, std::vector<std::string>> lists;
  std::map<std::string, std::string> meta = read_properties(dir + "/metadata.properties", &lists);
  const int ntrees = meta.count("startree.v2.count") ? atoi(meta["startree.v2.count"].c_str()) : 0;
  if (ntrees <= 0) return;
  std::vector<unsigned char> file;
  if (!read_file(dir + "/star_tree_index", file)) return;
  std::map<std::string, std::string> imap = read_properties(dir + "/star_tree_index_map");
  for (int t = 0; t < ntrees; t++) {
    const std::string pre = "startree.v2." + std::to_string(t) + ".";
    const int total = meta.count(pre + "total.docs") ? atoi(meta[pre + "total.docs"].c_str()) : 0;
    const std::vector<std::string>& dims = lists[pre + "split.order"];
    const std::vector<std::string>& pairs = lists[pre + "function.column.pairs"];
    if (total <= 0 || dims.empty() || pairs.empty()) continue;
    auto slice = [&](const std::string& col, const char* kind, const unsigned char*& p, uint64_t& n) -> bool {
      const std::string k = std::to_string(t) + "." + col + "." + kind;
      auto o = imap.find(k + ".OFFSET"), z = imap.find(k + ".SIZE");
      if (o == imap.end() || z == imap.end()) return false;
      const unsigned long long off = strtoull(o->second.c_str(), nullptr, 10), size = strtoull(z->second.c_str(), nullptr, 10);
      if (off + size > file.size()) return false;
      p = file.data() + off; n = size;
      return true;
    };
    const unsigned char* tree = nullptr; uint64_t tree_bytes = 0;
    if (!slice("null", "STAR_TREE", tree, tree_bytes)) continue;
    std::vector<const char*> dim_names;
    std::vector<const void*> dim_fwd;
    std::vector<uint64_t> dim_bytes;
    bool ok = true;
    for (const std::string& d : dims) {
      const unsigned char* p = nullptr; uint64_t n = 0;
      if (seg->column_index(d.c_str()) < 0 || !slice(d, "FORWARD_INDEX", p, n)) { ok = false; break; }
      dim_names.push_back(d.c_str()); dim_fwd.push_back(p); dim_bytes.push_back(n);
    }
    if (!ok) continue;
    std::vector<pb200h_star_metric> metrics;
    std::vector<std::string> metric_cols(pairs.size());
    for (size_t i = 0; i < pairs.size(); i++) {
      const size_t sep = pairs[i].find("__");
      if (sep == std::string::npos) continue;
      std::string fn = pairs[i].substr(0, sep);
      for (auto& ch : fn) ch = (char)toupper((unsigned char)ch);
      const int code = fn == "COUNT" ? PB200_AGG_COUNT : fn == "SUM" ? PB200_AGG_SUM : fn == "MIN" ? PB200_AGG_MIN : fn == "MAX" ? PB200_AGG_MAX : -1;
      const unsigned char* p = nullptr; uint64_t n = 0;
      if (code < 0 || !slice(pairs[i], "FORWARD_INDEX", p, n)) continue;
      metric_cols[i] = pairs[i].substr(sep + 2);
      if (code != PB200_AGG_COUNT && seg->column_index(metric_cols[i].c_str()) < 0) continue;
      pb200h_star_metric m;
      memset(&m, 0, sizeof m);
      m.function = code; m.column = code == PB200_AGG_COUNT ? nullptr : metric_cols[i].c_str(); m.fwd = p; m.fwd_bytes = n;
      metrics.push_back(m);
    }
    if (metrics.empty()) continue;
    // a tree that cannot be attached (unsupported layout) is simply not used: queries then scan the base columns
    pb200h_startree_attach(ctx, seg, tree, tree_bytes, total, (int)dims.size(), dim_names.data(), dim_fwd.data(), dim_bytes.data(),
                           (int)metrics.size(), metrics.data());
  }
}
}  // namespace

extern "C" int32_t pb200h_segment_load_dir(pb200_ctx* ctx, const char* path, pb200h_segment** out) {
  if (!ctx || !path || !out) { set_error("invalid argument to pb200h_segment_load_dir"); return PB200_E_INVALID; }
  std::string dir = path;
  bool v3 = false;
  std::map<std::string, std::string> meta = read_properties(dir + "/metadata.properties");
  if (meta.empty()) { meta = read_properties(dir + "/v3/metadata.properties"); if (!meta.empty()) { dir += "/v3"; v3 = true; } }
  if (meta.empty()) { set_error("no metadata.properties under %s", path); return PB200_E_INVALID; }
  if (!v3) { std::ifstream probe(dir + "/columns.psf"); v3 = (bool)probe; }
  const int num_docs = atoi(meta["segment.total.docs"].c_str());
  std::vector<std::string> names;
  for (auto& kv : meta) {
    const std::string& k = kv.first;
    const std::string suffix = ".cardinality";
    if (k.rfind("column.", 0) == 0 && k.size() > 7 + suffix.size() && k.compare(k.size() - suffix.size(), suffix.size(), suffix) == 0)
      names.push_back(k.substr(7, k.size() - 7 - suffix.size()));
  }
  std::vector<unsigned char> psf;
  std::map<std::string, std::string> imap;
  if (v3) {
    if (!read_file(dir + "/columns.psf", psf)) { set_error("cannot read %s/columns.psf", dir.c_str()); return PB200_E_INVALID; }
    imap = read_properties(dir + "/index_map");
  }
  struct Bufs { std::vector<unsigned char> fwd, dict, inv; };
  std::vector<Bufs> bufs;
  std::vector<pb200h_column> cols;
  std::vector<std::string> kept;
  auto slice = [&](const std::string& col, const char* kind, std::vector<unsigned char>& dst) -> bool {
    auto so = imap.find(col + "." + kind + ".startOffset"), sz = imap.find(col + "." + kind + ".size");
    if (so == imap.end() || sz == imap.end()) return false;
    unsigned long long off = strtoull(so->second.c_str(), nullptr, 10), size = strtoull(sz->second.c_str(), nullptr, 10);
    if (size < 8 || off > psf.size() || size > psf.size() - off || be64(psf.data() + off) != 0xdeadbeefdeafbeadull) return false;  // SingleFileIndexDirectory magic
    dst.assign(psf.begin() + off + 8, psf.begin() + off + size);
    return true;
  };
  bufs.reserve(names.size());
  for (const std::string& n : names) {
    auto get = [&](const char* k) { auto it = meta.find("column." + n + "." + k); return it == meta.end() ? std::string() : it->second; };
    if (get("isSingleValues") == "false") continue;  // MV columns are outside this path
    const std::string dt = get("dataType");
    int type = dt == "INT" ? PB200_INT : dt == "LONG" ? PB200_LONG : dt == "FLOAT" ? PB200_FLOAT : dt == "DOUBLE" ? PB200_DOUBLE : dt == "STRING" ? PB200_STRING : -1;
    if (type < 0) continue;
    // Only zero padding of STRING dictionaries is supported, as in the reference (ColumnMetadataImpl.java:250-253
    // "Only support zero padding"; segments written before segment.padding.character existed pad with '%').  The
    // reference refuses such a segment as a whole; here the STRING columns are left out and the numeric ones load.
    if (type == PB200_STRING) {
      auto pad = meta.find("segment.padding.character");
      const bool zero = pad != meta.end() && (pad->second == "\\u0000" || pad->second == std::string(1, '\0') || pad->second == "\\0");
      if (!zero) continue;
    }
    const bool has_dict = get("hasDictionary") != "false";
    const bool sorted = get("isSorted") == "true" && has_dict;
    Bufs b;
    bool ok;
    if (v3) {
      ok = slice(n, "forward_index", b.fwd);
      if (has_dict) ok = ok && slice(n, "dictionary", b.dict);
      slice(n, "inverted_index", b.inv);
    } else {
      ok = read_file(dir + "/" + n + (has_dict ? (sorted ? ".sv.sorted.fwd" : ".sv.unsorted.fwd") : ".sv.raw.fwd"), b.fwd);
      if (has_dict) ok = ok && read_file(dir + "/" + n + ".dict", b.dict);
      read_file(dir + "/" + n + ".bitmap.inv", b.inv);
    }
    if (!ok) continue;  // index kinds outside this path: column not registered
    if (!has_dict) {
      // raw columns this loader cannot decode (var-byte types, ZSTANDARD / GZIP chunks) are left out like any other index
      // kind outside the path: queries touching them fall back to the stock operator, the rest of the segment loads
      if (raw_value_width(type) == 0 || b.fwd.size() < 16) continue;
      const int version = (int)hbe32(b.fwd.data());
      const int compression = version > 1 && b.fwd.size() >= 28 ? (int)hbe32(b.fwd.data() + 20) : 1;
      if (compression != 0 && compression != 1 && compression != 3 && compression != 4) continue;
    }
    bufs.push_back(std::move(b));
    kept.push_back(n);
    pb200h_column c;
    memset(&c, 0, sizeof c);
    c.data_type = type; c.has_dictionary = has_dict; c.bits_per_value = atoi(get("bitsPerElement").c_str());
    c.cardinality = atoi(get("cardinality").c_str()); c.is_sorted = sorted;
    int len = atoi(get("lengthOfEachEntry").c_str());
    c.dict_entry_bytes = type == PB200_STRING ? std::max(len, 1) : (type == PB200_LONG || type == PB200_DOUBLE) ? 8 : 4;
    cols.push_back(c);
  }
  if (cols.empty()) { set_error("no loadable single-value columns in %s", path); return PB200_E_UNSUPPORTED; }
  for (size_t i = 0; i < cols.size(); i++) {
    cols[i].name = kept[i].c_str();
    cols[i].fwd = bufs[i].fwd.data(); cols[i].fwd_bytes = bufs[i].fwd.size();
    cols[i].dict = bufs[i].dict.empty() ? nullptr : bufs[i].dict.data(); cols[i].dict_bytes = bufs[i].dict.size();
    cols[i].inv = bufs[i].inv.empty() ? nullptr : bufs[i].inv.data(); cols[i].inv_bytes = bufs[i].inv.size();
  }
  const std::string seg_name = meta.count("segment.name") ? meta["segment.name"] : dir;
  int rc = pb200h_segment_create(ctx, seg_name.c_str(), num_docs, (int)cols.size(), cols.data(), out);
  if (rc) return rc;
  attach_star_trees_from_dir(ctx, dir, *out);
  return PB200_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// plan + execute
// ------------------------------------------------------------------------------------------------------------------
extern "C" int32_t pb200h_explain(pb200_ctx* ctx, const pb200h_query* q, pb200h_segment* seg, char* out, int32_t cap) {
  if (!q || !seg || !out || cap <= 0) { set_error("null argument"); return PB200_E_INVALID; }
  PatternScope patterns;
  pb200h_segment* one = seg;
  if (ctx) {
    if (int rc = derive_query_names(ctx, *q, &one, 1, nullptr, 0)) return rc;
    if (int rc = resolve_patterns(ctx, *q, &one, 1, patterns)) return rc;
  }
  ExprFilterScope exprs;   // checked only: explain names an expression leaf without computing its doc set
  if (int rc = resolve_expr_filters(ctx, *q, &one, 1, exprs, false)) return rc;
  SegmentFilter f;
  std::string text;
  int rc = build_segment_filter(*seg, *q, f, &text);
  if (rc) return rc;
  std::string op = f.root_empty ? "EMPTY" : (f.root_all && non_scan_answerable(*seg, *q)) ? "AGGREGATE_NO_SCAN"
                   : q->num_group_by > 0 ? "GROUP_BY" : "AGGREGATE";
  std::string s = op + "(" + text + ")";
  size_t n = std::min<size_t>(s.size(), (size_t)cap - 1);
  memcpy(out, s.data(), n);
  out[n] = 0;
  return (int32_t)n;
}

extern "C" int32_t pb200h_execute(pb200_ctx* ctx, const pb200h_query* q, pb200h_segment* const* segs, int32_t nseg,
                                  pb200_result** results, int32_t* kinds) {
  return pb200h_execute_ordered(ctx, q, nullptr, segs, nseg, results, kinds);
}

extern "C" int32_t pb200h_execute_ordered(pb200_ctx* ctx, const pb200h_query* q, const pb200_order_by* order,
                                          pb200h_segment* const* segs, int32_t nseg, pb200_result** results, int32_t* kinds) {
  return pb200h_execute_args(ctx, q, order, nullptr, segs, nseg, results, kinds);
}

extern "C" int32_t pb200h_execute_args(pb200_ctx* ctx, const pb200h_query* q, const pb200_order_by* order, const double* agg_args,
                                       pb200h_segment* const* segs, int32_t nseg, pb200_result** results, int32_t* kinds) {
  return pb200h_execute_having(ctx, q, order, agg_args, nullptr, segs, nseg, results, kinds);
}

extern "C" int32_t pb200h_execute_having(pb200_ctx* ctx, const pb200h_query* q, const pb200_order_by* order, const double* agg_args,
                                         const pb200_having* having, pb200h_segment* const* segs, int32_t nseg,
                                         pb200_result** results, int32_t* kinds) {
  if (!q || q->num_aggs < 0 || q->num_aggs > pb200::kMaxAggs || !agg_args)
    return pb200h_execute_agg_args(ctx, q, order, nullptr, having, segs, nseg, results, kinds);
  std::vector<pb200h_agg_arg> args(q->num_aggs);
  for (int a = 0; a < q->num_aggs; a++) args[a] = pb200h_agg_arg{agg_args[a], nullptr, 0};
  return pb200h_execute_agg_args(ctx, q, order, args.data(), having, segs, nseg, results, kinds);
}

extern "C" int32_t pb200h_execute_agg_args(pb200_ctx* ctx, const pb200h_query* q, const pb200_order_by* order, const pb200h_agg_arg* args,
                                           const pb200_having* having, pb200h_segment* const* segs, int32_t nseg,
                                           pb200_result** results, int32_t* kinds) {
  return pb200h_execute_post(ctx, q, order, args, having, nullptr, segs, nseg, results, kinds);
}

extern "C" int32_t pb200h_execute_post(pb200_ctx* ctx, const pb200h_query* q, const pb200_order_by* order, const pb200h_agg_arg* args,
                                       const pb200_having* having, const pb200_post_aggs* post, pb200h_segment* const* segs,
                                       int32_t nseg, pb200_result** results, int32_t* kinds) {
  if (!ctx || !q || !segs || !results || nseg <= 0) { set_error("invalid argument to pb200h_execute"); return PB200_E_INVALID; }
  if (q->num_aggs <= 0) { set_error("selection queries are outside this path"); return PB200_E_UNSUPPORTED; }
  if (int vrc = pb200::order_validate(order, q->num_aggs, q->num_group_by, post)) return vrc;
  if (int hrc = pb200::having_check(having, q->num_aggs, q->num_group_by, q->merge_segments ? 1 : nseg,
                                    q->merge_segments == 2 || q->reduce_world > 1))
    return hrc;
  if (q->num_group_by == 0) order = nullptr;  // aggregation only: one row, nothing to order
  std::vector<const char*> time_names;   // FIRST/LASTWITHTIME time columns: derived like every other name of the query
  for (int a = 0; a < q->num_aggs; a++) {
    if (!pb200::is_withtime_fn(q->aggs[a].function)) continue;
    if (!args || !args[a].time_column) { set_error("FIRST/LASTWITHTIME (aggregation %d) needs its time column: call pb200h_execute_agg_args", a); return PB200_E_INVALID; }
    time_names.push_back(args[a].time_column);
  }
  if (int rc = derive_query_names(ctx, *q, segs, nseg, time_names.data(), (int)time_names.size())) return rc;  // expressions become derived columns once
  PatternScope patterns;
  if (int rc = resolve_patterns(ctx, *q, segs, nseg, patterns)) return rc;      // pattern leaves become dictId sets once
  bool any_clause = false;   // some aggregation has a FILTER (WHERE ...) clause
  if (q->agg_filter_count && q->agg_filter_start && q->agg_filter_nodes)
    for (int a = 0; a < q->num_aggs; a++) any_clause |= q->agg_filter_count[a] > 0;
  // The device path's argument checks, before any segment can be answered on the host.  FILTER clauses run as one
  // submission per clause (host/filtered_agg.cpp), which carries no percentiles, time columns, moments or finalized value
  // sets: such a function anywhere in the query -- with its own clause or next to another function's -- goes to the
  // stock operator.
  std::vector<int> hll_log2m(q->num_aggs, 0);
  for (int a : aggs_by_family(*q, {PB200_AGG_FIRSTWITHTIME, PB200_AGG_PERCENTILE, PB200_AGG_VARPOP, PB200_AGG_DISTINCTSUM, PB200_AGG_DISTINCTCOUNTHLL})) {
    const pb200::AggFn* d = pb200::agg_fn(q->aggs[a].function);
    if (!d) continue;
    if (d->arg == pb200::ARG_PERCENTILE) {
      if (!args) { set_error("PERCENTILE (aggregation %d) needs its percentile: call pb200h_execute_args", a); return PB200_E_INVALID; }
      if (int rc = pb200::check_percentile(args[a].p, a)) return rc;
    }
    if (!d->filter_clause && any_clause) { set_error("%s in a query with FILTER (WHERE ...) clauses is not accelerated", d->family); return PB200_E_UNSUPPORTED; }
    if (d->arg == pb200::ARG_LOG2M)
      if (int rc = pb200::hll_log2m(args ? args[a].p : 0.0, a, &hll_log2m[a])) return rc;
  }
  ExprFilterScope expr_filters;   // expression leaves become device doc sets once, also for the FILTER clauses' submissions
  if (int rc = resolve_expr_filters(ctx, *q, segs, nseg, expr_filters, true)) return rc;
  if (q->agg_filter_count && q->agg_filter_start && q->agg_filter_nodes)
    for (int a = 0; a < q->num_aggs; a++)
      if (q->agg_filter_count[a] > 0) return execute_filtered(ctx, *q, order, having, post, segs, nseg, results, kinds);  // host/filtered_agg.cpp
  const bool merge = q->merge_segments != 0;
  // resolve columns by name against segment 0 (all segments of a table share the schema)
  const pb200h_segment& s0 = *segs[0];
  std::vector<int32_t> gb(q->num_group_by);
  for (int g = 0; g < q->num_group_by; g++) {
    gb[g] = s0.column_index(q->group_by[g]);
    if (gb[g] < 0) { set_error("unknown group-by column '%s'", q->group_by[g]); return PB200_E_INVALID; }
    if (!s0.cols[gb[g]].has_dictionary) { set_error("group-by on raw column '%s' is not accelerated", q->group_by[g]); return PB200_E_UNSUPPORTED; }
  }
  std::vector<pb200_agg> aggs(q->num_aggs);
  std::vector<pb200_agg_arg> dev_args(q->num_aggs, pb200_agg_arg{0.0, -1, 0});
  // SUM / AVG / MIN / MAX over an expression of two or more columns: a program over column ids, evaluated per row
  std::vector<std::vector<pb200_transform_op>> expr_ops(q->num_aggs);
  std::vector<pb200_expr_program> programs(q->num_aggs, pb200_expr_program{0, 0, nullptr});
  std::vector<int> leaf_cols;
  std::vector<CaseCond> case_conds;   // CASE conditions of all aggregations: a COND leaf's i indexes this call-wide list
  bool any_expr = false;
  for (int a = 0; a < q->num_aggs; a++) {
    if (!expression_function(q->aggs[a].function) || !is_multi_column_expression(q->aggs[a].column)) continue;
    std::string canonical;
    std::vector<std::string> leaves;
    std::vector<CaseCond> conds;
    std::vector<CaseBranch> branches;
    if (int rc = compile_multi_expression(q->aggs[a].column, &canonical, &expr_ops[a], &leaves, &conds, &branches)) return rc;
    if (int rc = case_result_type_check(s0, branches, q->aggs[a].column)) return rc;
    for (pb200_transform_op& o : expr_ops[a]) {
      if (o.op == PB200_T_COND) o.i += (int64_t)case_conds.size();
      if (o.op != PB200_T_COLUMN) continue;
      const char* name = leaves[(size_t)o.i].c_str();
      const int ci = s0.column_index(name);
      if (ci < 0 || ci >= s0.num_stored) { set_error("expression '%s': unknown column '%s'", q->aggs[a].column, name); return PB200_E_INVALID; }
      if (s0.cols[ci].data_type == PB200_STRING) { set_error("expression '%s': STRING column '%s' in arithmetic", q->aggs[a].column, name); return PB200_E_UNSUPPORTED; }
      o.i = ci;
      leaf_cols.push_back(ci);
    }
    for (const CaseCond& cc : conds) {
      const int ci = s0.column_index(cc.column.c_str());
      if (ci >= 0) leaf_cols.push_back(ci);
    }
    case_conds.insert(case_conds.end(), conds.begin(), conds.end());
    programs[a] = pb200_expr_program{(int32_t)expr_ops[a].size(), 0, expr_ops[a].data()};
    any_expr = true;
  }
  for (int a = 0; a < q->num_aggs; a++) {
    aggs[a].function = q->aggs[a].function;
    aggs[a].column = -1;
    if (q->aggs[a].function != PB200_AGG_COUNT && !programs[a].num_ops) {
      aggs[a].column = s0.column_index(q->aggs[a].column);
      if (aggs[a].column < 0) { set_error("unknown aggregation column '%s'", q->aggs[a].column ? q->aggs[a].column : "(null)"); return PB200_E_INVALID; }
      const HostColumn& c = s0.cols[aggs[a].column];
      const bool wt = pb200::is_withtime_fn(q->aggs[a].function);
      if (c.data_type == PB200_STRING && q->aggs[a].function != PB200_AGG_DISTINCTCOUNT && !pb200::is_hll_fn(q->aggs[a].function) && !wt) { set_error("%s over STRING column", "aggregation"); return PB200_E_UNSUPPORTED; }
      if (args) dev_args[a].p = args[a].p;
      if (wt) {
        dev_args[a].time_column = s0.column_index(args[a].time_column);
        if (dev_args[a].time_column < 0) { set_error("unknown time column '%s'", args[a].time_column); return PB200_E_INVALID; }
        dev_args[a].value_type = args[a].value_type;
      }
      if (pb200::is_moments_fn(q->aggs[a].function) && !c.has_dictionary) {
        set_error("VAR/STDDEV over raw column '%s' is not accelerated", q->aggs[a].column);
        return PB200_E_UNSUPPORTED;
      }
    }
  }
  // per-segment filters + plan shortcuts
  std::vector<SegmentFilter> filters(nseg);
  std::vector<int> kind(nseg, q->num_group_by > 0 ? PB200H_OP_GROUP_BY : PB200H_OP_AGGREGATION);
  for (int s = 0; s < nseg; s++) {
    if (segs[s]->num_stored != s0.num_stored) { set_error("segments do not share a schema"); return PB200_E_INVALID; }
    // group-by / aggregation columns were resolved by name against segment 0: every segment must hold the same column
    // (name, type, dictionary-encoded or not) at that position
    auto same_column = [&](int idx) {
      const HostColumn &a = s0.cols[idx], &b = segs[s]->cols[idx];
      return a.name == b.name && a.data_type == b.data_type && a.has_dictionary == b.has_dictionary;
    };
    for (int g = 0; g < q->num_group_by; g++) if (!same_column(gb[g])) { set_error("segment %d: column '%s' is not at the position it has in segment 0", s, q->group_by[g]); return PB200_E_INVALID; }
    for (int a = 0; a < q->num_aggs; a++) if (aggs[a].column >= 0 && !same_column(aggs[a].column)) { set_error("segment %d: column '%s' is not at the position it has in segment 0", s, q->aggs[a].column); return PB200_E_INVALID; }
    for (int a = 0; a < q->num_aggs; a++) if (dev_args[a].time_column >= 0 && !same_column(dev_args[a].time_column)) { set_error("segment %d: column '%s' is not at the position it has in segment 0", s, args[a].time_column); return PB200_E_INVALID; }
    for (int c : leaf_cols) if (!same_column(c)) { set_error("segment %d: column '%s' is not at the position it has in segment 0", s, s0.cols[c].name.c_str()); return PB200_E_INVALID; }
    int rc = build_segment_filter(*segs[s], *q, filters[s], nullptr);
    if (rc) return rc;
    if (!merge) {
      if (filters[s].root_empty) kind[s] = PB200H_OP_EMPTY;
      else if (filters[s].root_all && !any_expr && non_scan_answerable(*segs[s], *q)) kind[s] = PB200H_OP_NON_SCAN_AGGREGATION;
    }
  }
  // star-tree substitution (AggregationFunctionUtils.buildAggregationInfo :285-310): first star-tree that fits wins
  std::vector<pb200_result*> star_results(nseg, nullptr);
  if (!merge && !q->skip_star_tree && !any_expr) {   // expressions are computed per row: the raw scan runs
    for (int s = 0; s < nseg; s++) {
      if (kind[s] != PB200H_OP_AGGREGATION && kind[s] != PB200H_OP_GROUP_BY) continue;
      for (auto& st : segs[s]->star_trees) {
        int rc = try_star_tree(ctx, *segs[s], *st, *q, &star_results[s]);
        if (rc < 0) { for (auto r : star_results) if (r) pb200_result_free(r); return rc; }
        if (rc == 1) {
          kind[s] = PB200H_OP_STAR_TREE;
          // the star-tree's own submission computes other functions: filter and order by the query's, on the host
          std::vector<int32_t> fns(q->num_aggs);
          for (int a = 0; a < q->num_aggs; a++) fns[a] = q->aggs[a].function;
          if (having) pb200::having_rows_host(star_results[s], *having, fns.data());
          if (order) pb200::order_rows_host(star_results[s], *order, fns.data(), post);
          break;
        }
      }
    }
  }
  if (kinds) for (int s = 0; s < nseg; s++) kinds[s] = kind[s];
  // device submission for the segments that need a scan
  std::vector<int> dev_idx;
  for (int s = 0; s < nseg; s++) if (kind[s] == PB200H_OP_AGGREGATION || kind[s] == PB200H_OP_GROUP_BY) dev_idx.push_back(s);
  std::vector<pb200_result*> dev_results(merge ? 1 : dev_idx.size(), nullptr);
  if (!dev_idx.empty()) {
    std::vector<pb200_filter_node> flat;
    std::vector<pb200_segment*> dsegs;
    for (int s : dev_idx) { flat.insert(flat.end(), filters[s].nodes.begin(), filters[s].nodes.end()); dsegs.push_back(segs[s]->dev); }
    pb200_query dq;
    memset(&dq, 0, sizeof dq);
    dq.num_filter_nodes = q->num_filter_nodes;
    dq.num_group_by = q->num_group_by;
    dq.num_aggs = q->num_aggs;
    dq.num_groups_limit = q->num_groups_limit > 0 ? q->num_groups_limit : 100000;
    dq.max_initial_result_holder_capacity = q->max_initial_result_holder_capacity > 0 ? q->max_initial_result_holder_capacity : 10000;
    dq.flags = PB200_Q_PER_SEGMENT_FILTER | (merge ? PB200_Q_MERGE_SEGMENTS : 0) | (q->merge_segments == 2 ? PB200_Q_DEFER_FINALIZE : 0) |
               (q->no_count_carrier ? PB200_Q_NO_COUNT_CARRIER : 0);
    dq.reduce_world = q->reduce_world;
    dq.merged_docs_bound = q->merged_docs_bound;
    dq.filter = flat.data();
    dq.group_by_columns = gb.data();
    dq.aggs = aggs.data();
    // the CASE conditions, resolved on the segments of this submission
    CaseTable cases;
    std::vector<pb200h_segment*> hsegs;
    for (int s : dev_idx) hsegs.push_back(segs[s]);
    int rc = resolve_case_conditions(ctx, hsegs.data(), (int)hsegs.size(), case_conds, patterns, cases);
    if (!rc)
      rc = pb200::execute_exprs_post(ctx, &dq, order, args ? dev_args.data() : nullptr, having, any_expr ? programs.data() : nullptr,
                                     case_conds.empty() ? nullptr : &cases.table, post, dsegs.data(), (int)dsegs.size(), dev_results.data());
    if (rc) { for (auto r : star_results) if (r) pb200_result_free(r); return rc; }
    // the mask pass of each expression leaf read its leaf columns at every doc of the segment
    for (size_t k = 0; k < dev_idx.size(); k++) dev_results[merge ? 0 : k]->meta.num_entries_scanned_in_filter += expr_filter_entries(*segs[dev_idx[k]], *q);
  }
  if (merge) { results[0] = dev_results[0]; return PB200_OK; }
  size_t di = 0;
  for (int s = 0; s < nseg; s++) {
    if (kind[s] == PB200H_OP_STAR_TREE) results[s] = star_results[s];
    else if (kind[s] == PB200H_OP_EMPTY) {
      results[s] = host_result(*segs[s], *q, true);
      if (having) results[s]->having = *having;   // no rows to filter, but the result is as final as a filtered one
    }
    else if (kind[s] == PB200H_OP_NON_SCAN_AGGREGATION) results[s] = host_result(*segs[s], *q, false);
    else results[s] = dev_results[di++];
  }
  // DISTINCTCOUNTHLL answered without a scan: the device finalize over the whole dictionary
  for (int s = 0; s < nseg; s++) {
    if (kind[s] != PB200H_OP_NON_SCAN_AGGREGATION) continue;
    for (int a = 0; a < q->num_aggs; a++) {
      if (!pb200::is_hll_fn(q->aggs[a].function)) continue;
      long long est = 0;
      if (int rc = pb200::hll_whole_dictionary(ctx, segs[s]->dev, aggs[a].column, hll_log2m[a], &est)) {
        for (int k = 0; k < nseg; k++) { pb200_result_free(results[k]); results[k] = nullptr; }
        return rc;
      }
      results[s]->lng[a][0] = est;
      results[s]->dbl[a][0] = (double)est;
    }
  }
  return PB200_OK;
}

namespace {
// A selection result without rows, built on the host (every doc of the segments is filtered out before any scan).
pb200_result* empty_selection(pb200h_segment* const* segs, int s0, int s1, int ncols) {
  pb200_result* R = new pb200_result();
  R->selection.present = true;
  R->selection.columns.assign(ncols, nullptr);
  R->meta.regime = PB200_REGIME_NONE;
  for (int s = s0; s < s1; s++) R->meta.num_total_docs += segs[s]->num_docs;
  return R;
}

// pb200h_execute_selection and pb200h_execute_distinct: names resolved, filters folded per segment, `device` (the C-ABI
// call) run over the segments whose filter is not EMPTY, segment indexes mapped back to `segs`.
using RowsDeviceCall = int32_t (*)(pb200_ctx*, const pb200_query*, const pb200_selection*, pb200_segment* const*, int32_t, int32_t,
                                   pb200_result**);
int32_t execute_rows(pb200_ctx* ctx, const pb200h_query* q, const pb200h_selection* sel, pb200h_segment* const* segs, int32_t nseg,
                     pb200_result** results, RowsDeviceCall device) {
  if (sel->num_columns < 0 || (sel->num_columns > 0 && !sel->columns)) { set_error("selection: bad column list"); return PB200_E_INVALID; }
  {
    std::vector<const char*> extra(sel->columns, sel->columns + sel->num_columns);
    for (int k = 0; k < sel->num_order_items && k < PB200_MAX_ORDER_BY; k++) extra.push_back(sel->order[k].column);
    pb200h_query fq = *q;  // the filter part only: the group-by and aggregation fields are ignored here
    fq.num_group_by = 0; fq.num_aggs = 0; fq.agg_filter_count = nullptr;
    if (int rc = derive_query_names(ctx, fq, segs, nseg, extra.data(), (int)extra.size())) return rc;
  }
  PatternScope patterns;
  if (int rc = resolve_patterns(ctx, *q, segs, nseg, patterns)) return rc;
  ExprFilterScope expr_filters;
  if (int rc = resolve_expr_filters(ctx, *q, segs, nseg, expr_filters, true)) return rc;
  const pb200h_segment& s0 = *segs[0];
  std::vector<int32_t> cols(sel->num_columns);
  for (int k = 0; k < sel->num_columns; k++) {
    cols[k] = s0.column_index(sel->columns[k]);
    if (cols[k] < 0) { set_error("unknown selected column '%s'", sel->columns[k] ? sel->columns[k] : "(null)"); return PB200_E_INVALID; }
  }
  pb200_selection dsel;
  memset(&dsel, 0, sizeof dsel);
  dsel.num_columns = sel->num_columns;
  dsel.columns = cols.data();
  dsel.limit = sel->limit;
  if (sel->num_order_items < 0 || sel->num_order_items > PB200_MAX_ORDER_BY) { set_error("selection ORDER BY with %d items (1..%d)", sel->num_order_items, PB200_MAX_ORDER_BY); return PB200_E_INVALID; }
  dsel.num_order_items = sel->num_order_items;
  for (int k = 0; k < sel->num_order_items; k++) {
    dsel.order[k].column = s0.column_index(sel->order[k].column);
    dsel.order[k].descending = sel->order[k].descending;
    if (dsel.order[k].column < 0) { set_error("unknown ORDER BY column '%s'", sel->order[k].column ? sel->order[k].column : "(null)"); return PB200_E_INVALID; }
  }
  if (sel->limit < 0) { set_error("selection: negative LIMIT"); return PB200_E_INVALID; }
  if (sel->limit > PB200_MAX_SELECT_LIMIT) { set_error("selection LIMIT %lld above %d", (long long)sel->limit, PB200_MAX_SELECT_LIMIT); return PB200_E_UNSUPPORTED; }
  const bool merge = q->merge_segments != 0;
  std::vector<SegmentFilter> filters(nseg);
  std::vector<int> dev_idx;
  for (int s = 0; s < nseg; s++) {
    if (segs[s]->num_stored != s0.num_stored) { set_error("segments do not share a schema"); return PB200_E_INVALID; }
    for (int k = 0; k < sel->num_columns; k++) {
      const HostColumn &a = s0.cols[cols[k]], &b = segs[s]->cols[cols[k]];
      if (a.name != b.name || a.data_type != b.data_type) { set_error("segment %d: column '%s' is not at the position it has in segment 0", s, sel->columns[k]); return PB200_E_INVALID; }
    }
    if (int rc = build_segment_filter(*segs[s], *q, filters[s], nullptr)) return rc;
    if (!filters[s].root_empty) dev_idx.push_back(s);
  }
  const int nres = merge ? 1 : nseg;
  std::vector<pb200_result*> dev_results(merge ? 1 : dev_idx.size(), nullptr);
  if (!dev_idx.empty()) {
    std::vector<pb200_filter_node> flat;
    std::vector<pb200_segment*> dsegs;
    for (int s : dev_idx) { flat.insert(flat.end(), filters[s].nodes.begin(), filters[s].nodes.end()); dsegs.push_back(segs[s]->dev); }
    pb200_query dq;
    memset(&dq, 0, sizeof dq);
    dq.num_filter_nodes = q->num_filter_nodes;
    dq.flags = PB200_Q_PER_SEGMENT_FILTER;
    dq.filter = flat.data();
    int rc = device(ctx, &dq, &dsel, dsegs.data(), (int)dsegs.size(), merge ? PB200_Q_MERGE_SEGMENTS : 0, dev_results.data());
    if (rc) return rc;
    for (size_t k = 0; k < dev_idx.size(); k++) dev_results[merge ? 0 : k]->meta.num_entries_scanned_in_filter += expr_filter_entries(*segs[dev_idx[k]], *q);
    // rows name their segment by its position in the device submission: map it back to `segs`
    for (pb200_result* R : dev_results)
      for (int64_t i = 0; i < R->selection.rows; i++) R->selection.segment_index[i] = dev_idx[R->selection.segment_index[i]];
  }
  if (merge) {
    results[0] = dev_idx.empty() ? empty_selection(segs, 0, nseg, sel->num_columns) : dev_results[0];
    results[0]->meta.num_total_docs = 0;
    for (int s = 0; s < nseg; s++) results[0]->meta.num_total_docs += segs[s]->num_docs;
    return PB200_OK;
  }
  size_t di = 0;
  for (int s = 0; s < nres; s++)
    results[s] = (di < dev_idx.size() && dev_idx[di] == s) ? dev_results[di++] : empty_selection(segs, s, s + 1, sel->num_columns);
  return PB200_OK;
}
}  // namespace

extern "C" int32_t pb200h_execute_selection(pb200_ctx* ctx, const pb200h_query* q, const pb200h_selection* sel,
                                            pb200h_segment* const* segs, int32_t nseg, pb200_result** results) {
  if (!ctx || !q || !sel || !segs || !results || nseg <= 0) { set_error("invalid argument to pb200h_execute_selection"); return PB200_E_INVALID; }
  return execute_rows(ctx, q, sel, segs, nseg, results, pb200_execute_selection);
}

extern "C" int32_t pb200h_execute_distinct(pb200_ctx* ctx, const pb200h_query* q, const pb200h_selection* distinct,
                                           pb200h_segment* const* segs, int32_t nseg, pb200_result** results) {
  if (!ctx || !q || !distinct || !segs || !results || nseg <= 0) { set_error("invalid argument to pb200h_execute_distinct"); return PB200_E_INVALID; }
  // also when every segment's filter folds to EMPTY and nothing reaches the device
  for (int k = 0; k < distinct->num_order_items && k < PB200_MAX_ORDER_BY; k++) {
    const char* name = distinct->order[k].column;
    bool found = false;
    for (int c = 0; c < distinct->num_columns && name && distinct->columns && !found; c++)
      found = distinct->columns[c] && strcmp(distinct->columns[c], name) == 0;
    if (!found) { set_error("DISTINCT ORDER BY column '%s' is not one of the DISTINCT columns", name ? name : "(null)"); return PB200_E_INVALID; }
  }
  return execute_rows(ctx, q, distinct, segs, nseg, results, pb200_execute_distinct);
}

