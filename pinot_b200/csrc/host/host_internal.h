// host_internal.h -- shared declarations of the native host layer (plan_maker.cpp, star_tree.cpp).
#pragma once
#include <cmath>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../../include/pinot_b200_host.h"
#include "../pb200_internal.h"

namespace pb200h {
using pb200::set_error;

inline uint32_t hbe32(const unsigned char* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
inline uint64_t hbe64(const unsigned char* p) { return (uint64_t)hbe32(p) << 32 | hbe32(p + 4); }

// Stored INT / LONG value vs a predicate literal, by exact numeric value (-1, 0, 1).  `d` is the literal rounded to
// double; when it is an int64, `i` holds it exactly and (double)i == d.  Otherwise a fractional `d` is the literal
// itself (it equals no integer) and an integral or infinite one lies beyond the int64 range on its side.  This is what
// the reference's broker (NumericalFilterOptimizer) makes of `intCol >= 2.5` or `longCol < 1e19` before a server sees
// them.
inline int compare_integral(int64_t v, const pb200h_literal& l) {
  if ((double)l.i == l.d) return v < l.i ? -1 : v > l.i;
  if (std::isfinite(l.d) && l.d != std::floor(l.d)) return (double)v < l.d ? -1 : 1;   // |d| < 2^52: rounding v keeps its side
  return l.d > 0 ? -1 : 1;
}

struct HostColumn {
  std::string name;
  int data_type = 0, has_dictionary = 0, bits = 0, cardinality = 0, is_sorted = 0, entry_bytes = 0;
  bool has_inverted = false;
  bool synthesized_dictionary = false;    // the segment stores this column raw: `dict` was built from its values at load (raw_forward.cpp)
  bool derived = false;                   // a transform of a stored column (transform.cpp): `name` is its canonical text
  std::vector<unsigned char> dict;        // big-endian values or padded strings (host copy): the SEGMENT's own dictionary
  std::vector<unsigned char> sorted_idx;  // (start,end) BE pairs when is_sorted
  // Bound to a table-wide dictionary domain (pb200h_segment_bind_domain): predicates are still resolved against the
  // segment's own dictionary above (same alwaysTrue / alwaysFalse / index decisions as the reference), then ids are
  // translated with local_ids; everything the device returns for this column is a DOMAIN id, decoded through `global`.
  std::vector<int32_t> local_ids;               // local dictId -> domain id (ascending); empty = unbound
  std::shared_ptr<const HostColumn> global;     // the domain's dictionary as a column (dict, cardinality, bits, entry_bytes)
  int to_device_id(int local) const { return local_ids.empty() ? local : local_ids[local]; }
  const HostColumn& decode_column() const { return global ? *global : *this; }

  int32_t get_int(int id) const { return (int32_t)hbe32(dict.data() + 4ull * id); }
  int64_t get_long(int id) const { return (int64_t)hbe64(dict.data() + 8ull * id); }
  float get_float(int id) const { uint32_t u = hbe32(dict.data() + 4ull * id); float f; memcpy(&f, &u, 4); return f; }
  double get_double(int id) const { uint64_t u = hbe64(dict.data() + 8ull * id); double d; memcpy(&d, &u, 8); return d; }
  std::string get_string(int id) const {
    const char* p = (const char*)dict.data() + (size_t)entry_bytes * id;
    size_t n = 0;
    while (n < (size_t)entry_bytes && p[n]) n++;
    return std::string(p, n);
  }
  double as_double(int id) const {
    switch (data_type) {
      case PB200_INT: return get_int(id);
      case PB200_LONG: return (double)get_long(id);
      case PB200_FLOAT: return get_float(id);
      case PB200_DOUBLE: return get_double(id);
      default: return NAN;
    }
  }
  // Dictionary.insertionIndexOf (BaseImmutableDictionary.java:124-139): >= 0 found, else -(insertion point) - 1
  int insertion_index_of(const pb200h_literal& l) const {
    int lo = 0, hi = cardinality - 1;
    while (lo <= hi) {
      int mid = (lo + hi) >> 1, cmp;
      switch (data_type) {
        case PB200_INT: cmp = compare_integral(get_int(mid), l); break;
        case PB200_LONG: cmp = compare_integral(get_long(mid), l); break;
        case PB200_FLOAT: { float v = get_float(mid), t = (float)l.d; cmp = v < t ? -1 : v > t; break; }
        case PB200_DOUBLE: { double v = get_double(mid); cmp = v < l.d ? -1 : v > l.d; break; }
        default: { int r = get_string(mid).compare(l.s ? l.s : ""); cmp = r < 0 ? -1 : r > 0; }
      }
      if (cmp < 0) lo = mid + 1; else if (cmp > 0) hi = mid - 1; else return mid;
    }
    return -(lo + 1);
  }
  int sorted_start(int id) const { return (int)hbe32(sorted_idx.data() + 8ull * id); }
  int sorted_end(int id) const { return (int)hbe32(sorted_idx.data() + 8ull * id + 4); }
};

// OffHeapStarTree: parsed header + node accessors (7 little-endian ints per node)
struct StarTree {
  std::vector<unsigned char> bytes;
  std::vector<std::string> dim_names;
  const unsigned char* nodes = nullptr;
  int num_nodes = 0;
  bool parse(const unsigned char* b, uint64_t len);
  int field(int n, int f) const { const unsigned char* p = nodes + 28ll * n + 4 * f; return (int)((uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24); }
  int dim_id(int n) const { return field(n, 0); }
  int dim_value(int n) const { return field(n, 1); }
  int start(int n) const { return field(n, 2); }
  int end(int n) const { return field(n, 3); }
  int agg_doc(int n) const { return field(n, 4); }
  int first_child(int n) const { return field(n, 5); }
  int last_child(int n) const { return field(n, 6); }
  bool is_leaf(int n) const { return first_child(n) == -1; }
  int num_children(int n) const { return is_leaf(n) ? 0 : last_child(n) - first_child(n) + 1; }
  int child_for_value(int n, int value) const;
  bool traverse(const std::vector<const std::vector<int32_t>*>& preds, uint32_t group_by_mask,
                std::vector<std::pair<int32_t, int32_t>>& docs,
                uint32_t& remaining_out) const;
};

}  // namespace pb200h

struct pb200h_segment;
namespace pb200h {
struct StarTreeIndex {
  StarTree tree;
  std::vector<int> dim_base_col;     // star dimension -> column index in the base segment
  std::vector<int> metric_fn;        // function of each function-column pair
  std::vector<int> metric_base_col;  // its column in the base segment (-1 for count__*)
  std::vector<int> metric_limb_col;  // built trees, SUM over INT: the first of its three limb columns in the star segment
                                     // (pb200_startree_build.h StarBuildResult::limb_col); -1 otherwise
  int num_docs = 0;
  pb200h_segment* star_segment = nullptr;  // columns: dimensions..., metrics...
  // Traversal results by (predicate dictId sets per dimension, group-by mask): the BFS over a tree with 10^5..10^6 nodes
  // costs more host time than the device scan of the docs it selects, and dashboards repeat their predicates.  The
  // tree is immutable, so an entry never goes stale; a handful of entries, oldest evicted first.
  struct Traversal {
    std::string key; std::vector<uint32_t> mask; uint32_t remaining = 0;
    pb200_ctx* ctx = nullptr; uint32_t* dev_mask = nullptr;   // the mask resident in HBM (pb200_doc_mask_upload): no per-query copy
    ~Traversal() { if (dev_mask) pb200_doc_mask_free(ctx, dev_mask); }
  };
  mutable std::mutex cache_mu;
  mutable std::deque<std::shared_ptr<const Traversal>> cache;
  ~StarTreeIndex();
};
}  // namespace pb200h

namespace pb200h {
// transform.cpp: canonical text of a single-column expression (function names and their aliases to the canonical name,
// time-unit literals in upper case, numeric literals by value); false when `text` is no expression
bool normalize_expression(const char* text, std::string* canonical);
// the canonical text, the postfix program (pb200_transform_op) and the column of an expression; PB200_E_* with a message
int compile_expression(const char* text, std::string* canonical, std::vector<pb200_transform_op>* ops, std::string* column);
}  // namespace pb200h

struct pb200h_segment {
  pb200_ctx* ctx = nullptr;
  pb200_segment* dev = nullptr;
  std::string name;
  int num_docs = 0;
  // Stored columns, then derived ones in the order they were derived (the same ids as in `dev`).  Room for
  // PB200_MAX_DERIVED_COLUMNS more is reserved at creation: a derived column is appended complete, under derive_mu,
  // without moving a column that a running query references.
  // Readers bound column ids by num_columns(), never by cols.size(): the count is published with release only after
  // the appended column is complete.
  std::vector<pb200h::HostColumn> cols;
  int num_stored = 0;
  std::atomic<int> published{-1};  // -1: a column list that never grows (cols.size())
  std::mutex derive_mu;
  int num_columns() const { const int p = published.load(std::memory_order_acquire); return p < 0 ? (int)cols.size() : p; }
  std::vector<std::unique_ptr<pb200h::StarTreeIndex>> star_trees;
  // A stored column whose name is `n`, else the derived column of the expression `n` (any spelling), else -1
  int column_index(const char* n) const {
    if (!n) return -1;
    const int published_now = num_columns();
    for (int i = 0; i < published_now; i++) if (cols[i].name == n) return i;
    std::string canonical;
    if (published_now == num_stored || !strchr(n, '(') || !pb200h::normalize_expression(n, &canonical)) return -1;
    for (int i = num_stored; i < published_now; i++) if (cols[i].name == canonical) return i;
    return -1;
  }
};

namespace pb200h {
// transform.cpp: resolves every name that is no column of a segment as an expression and derives it there once
// (pb200h_segment_derive); afterwards every name is at one position in all segments (else PB200_E_UNSUPPORTED)
int derive_names(pb200_ctx* ctx, pb200h_segment* const* segs, int nseg, const std::vector<const char*>& names);
// Multi-column expressions (DESIGN.md section 3.15): `text` in the grammar of compile_expression with two or more column
// leaves, compiled to a program whose PB200_T_COLUMN leaf k (i = k) reads column leaves[k].  PB200_E_INVALID (malformed)
// or PB200_E_UNSUPPORTED (fewer than two or more than 8 leaves, a time function, outside the grammar), message set.
// CASE WHEN (DESIGN.md section 3.19) compiles to COND leaves (i = k: conds[k]) and CASE / AND / OR / NOT operations; a
// caller that passes no `conds` refuses it (PB200_E_UNSUPPORTED).  COND leaves count against the 8 column leaves, and a
// CASE needs no second column.
struct CaseCond {
  std::string fn;                     // equals, not_equals, less_than, ..., between, in, not_in, like, regexp_like
  std::string column;
  std::vector<std::string> literals;  // as written (quotes removed)
};
struct CaseBranch {                   // a THEN or ELSE value: what decides whether its CASE has one result type
  enum Kind { COLUMN, LONG_LITERAL, DOUBLE_LITERAL, ARITHMETIC } kind = COLUMN;
  std::string column;                 // COLUMN
  int64_t value = 0;                  // LONG_LITERAL
};
int compile_multi_expression(const char* text, std::string* canonical, std::vector<pb200_transform_op>* ops,
                             std::vector<std::string>* leaves, std::vector<CaseCond>* conds = nullptr,
                             std::vector<CaseBranch>* branches = nullptr);
// case_expr.cpp: the condition table of a call's CASE conditions (their COND leaves index `conds`), resolved on every
// segment of the call by the WHERE planner's value-to-dictId rule; LIKE / REGEXP_LIKE leaves go through `patterns`.
// PB200_E_UNSUPPORTED for the refused conditions of DESIGN.md section 3.19 (a STRING range, a raw or NaN / -0.0
// condition column, a non-integral literal beyond 2^53 on a LONG column, ...), PB200_E_INVALID for an unknown column.
struct CaseTable {
  std::vector<pb200_expr_cond> conds;
  std::vector<std::vector<int64_t>> args;
  std::vector<uint32_t> words;
  pb200_expr_conds table{};
};
struct PatternScope;
int resolve_case_conditions(pb200_ctx* ctx, pb200h_segment* const* segs, int nseg, const std::vector<CaseCond>& leaves,
                            PatternScope& patterns, CaseTable& out);
// The local dictIds (ascending) column c matches for one condition (pattern leaves: from the thread's pattern scope), with
// the refusals that concern the column itself
int case_condition_ids(const HostColumn& c, const CaseCond& cc, std::vector<int32_t>* ids);
// the REGEXP_LIKE pattern of a like / regexp_like condition (LIKE as sql.py's like_to_regexp); false for a LIKE escape
bool case_pattern(const CaseCond& cc, std::string* regex);
// PB200_E_UNSUPPORTED for a CASE whose result type this library does not restate: a FLOAT column branch next to an INT /
// LONG column branch or an integer literal beyond 2^24, with no DOUBLE column, decimal literal or arithmetic branch
int case_result_type_check(const pb200h_segment& s0, const std::vector<CaseBranch>& branches, const char* text);
// `text` compiles as a multi-column expression (the last error is left as it was)
bool is_multi_column_expression(const char* text);
// the functions that take a multi-column expression as their argument
inline bool expression_function(int fn) { return fn == PB200_AGG_SUM || fn == PB200_AGG_AVG || fn == PB200_AGG_MIN || fn == PB200_AGG_MAX; }
int derive_query_names(pb200_ctx* ctx, const pb200h_query& q, pb200h_segment* const* segs, int nseg, const char* const* extra, int nextra);
// the name of function fn (PB200_AGG_*) in lower case, as result column names spell it
std::string lower_fn_name(int fn);
// The positions of q's aggregations in the order a check that refuses some functions visits them: those of the families of
// `first` in that order, then the others, each in query order.  So a query with several refused functions is refused
// for the same one whatever their order in the query.
std::vector<int> aggs_by_family(const pb200h_query& q, std::initializer_list<int> first);
}  // namespace pb200h

namespace pb200h {
// raw_forward.cpp: no-dictionary fixed-width SV forward indexes at load time
int raw_value_width(int data_type);
int decode_fixed_byte_forward(const unsigned char* file, uint64_t len, int width, int64_t num_docs, std::vector<unsigned char>& values_be);
void wrap_pass_through(const std::vector<unsigned char>& values_be, int width, int64_t num_docs, std::vector<unsigned char>& file);
bool synthesize_dictionary(const std::vector<unsigned char>& values_be, int data_type, int64_t num_docs, int max_cardinality,
                           std::vector<unsigned char>& dict_be, std::vector<unsigned char>& fwd_packed, int* cardinality, int* bits);
// filtered_agg.cpp: FILTER (WHERE ...) clauses = one device submission per distinct clause, aligned by group key
int execute_filtered(pb200_ctx* ctx, const pb200h_query& q, const pb200_order_by* order, const pb200_having* having,
                     const pb200_post_aggs* post, pb200h_segment* const* segs, int nseg, pb200_result** results, int32_t* kinds);
// ids[] storage that must outlive the pb200_execute call
struct SegmentFilterStore { std::vector<std::unique_ptr<std::vector<int32_t>>> ids; };
// PredicateEvaluator.getMatchingDictIds (sorted) of one predicate on a dictionary column
std::vector<int32_t> matching_dict_ids(const HostColumn& c, const pb200h_filter_node& n, const pb200h_literal* lits);
// one value-space predicate -> the device leaf FilterOperatorUtils.getLeafFilterOperator would build on `seg`.column
int leaf_to_device(const pb200h_segment& seg, int column, const pb200h_filter_node& n, const pb200h_literal* lits,
                   SegmentFilterStore& store, pb200_filter_node& out);
int try_star_tree(pb200_ctx* ctx, const pb200h_segment& seg, const StarTreeIndex& st, const pb200h_query& q,
                  pb200_result** out);

// patterns.cpp: the matching dictIds of the REGEXP_LIKE leaves of one call.  An entry point declares one PatternScope
// (it becomes the calling thread's innermost scope until it goes out of scope) and fills it with resolve_patterns before
// planning; evaluate() then finds a leaf's ids with pattern_ids, which searches the thread's scopes innermost first, so
// a nested call (a FILTER clause's submission) reuses what its caller resolved.
struct PatternScope {
  std::vector<std::pair<std::pair<const HostColumn*, std::string>, std::vector<int32_t>>> ids;  // local dictIds, ascending
  PatternScope* outer;
  PatternScope();
  ~PatternScope();
  PatternScope(const PatternScope&) = delete;
  PatternScope& operator=(const PatternScope&) = delete;
};
// One pb200_match_pattern per distinct (pattern, column) of the query's filter and FILTER clauses not resolved yet, over
// all segments; PB200_E_UNSUPPORTED for a column that is not a STRING dictionary column or is derived
int resolve_patterns(pb200_ctx* ctx, const pb200h_query& q, pb200h_segment* const* segs, int nseg, PatternScope& scope);
// The matching ids of `pattern` on column c, or NULL when no scope of the thread resolved it
const std::vector<int32_t>* pattern_ids(const HostColumn& c, const char* pattern);
// Makes `to` (a star-tree dimension, sharing `from`'s dictionary) resolve `pattern` as `from` does, when `from` does
void pattern_alias(const HostColumn& from, const HostColumn& to, const char* pattern);

// expr_filters.cpp: predicates on expressions of two or more columns (DESIGN.md section 3.16).  Their doc sets are
// computed on the device (pb200_expr_doc_masks) before a call is planned and kept in a scope shaped like PatternScope:
// an entry point declares one, fills it with resolve_expr_filters, and build_segment_filter finds a leaf's mask with
// expr_filter_mask, searching the thread's scopes innermost first, so a FILTER clause's submission reuses its caller's
// masks.  The scope frees its masks when the entry point's frame ends.
struct ExprFilterScope {
  struct Mask { std::string key; const pb200h_segment* seg; uint32_t* mask; int ncols; };
  std::vector<Mask> masks;
  pb200_ctx* ctx = nullptr;
  ExprFilterScope* outer;
  ExprFilterScope();
  ~ExprFilterScope();
  ExprFilterScope(const ExprFilterScope&) = delete;
  ExprFilterScope& operator=(const ExprFilterScope&) = delete;
};
// `text` names an expression with two or more DISTINCT column leaves: as a filter leaf it is evaluated per row, never
// derived (an expression over one column, even used twice, stays a derived column)
bool is_expression_filter(const char* text);
// Every expression leaf of the query's filter and FILTER clauses: compiled, checked, and (launch) one pb200_expr_doc_masks
// call for the distinct (expression, predicate) pairs no scope of the thread holds yet, one mask per segment.
// PB200_E_UNSUPPORTED: REGEXP_LIKE / LIKE on an expression, a string literal, what compile_multi_expression and
// pb200_expr_doc_masks refuse; PB200_E_INVALID: an unknown leaf column or one at different positions in the segments.
int resolve_expr_filters(pb200_ctx* ctx, const pb200h_query& q, pb200h_segment* const* segs, int nseg, ExprFilterScope& scope,
                         bool launch);
// The leaf's canonical text and, when a scope of the thread resolved it on `seg`, its device mask and the number of its
// distinct leaf columns (mask NULL otherwise); PB200_E_* when the leaf does not compile
int expr_filter_mask(const pb200h_segment& seg, const pb200h_filter_node& n, const pb200h_literal* lits, std::string* canonical,
                     const uint32_t** mask, int* ncols);
// num_docs x distinct leaf columns of every expression leaf of the query's filter, on one segment (the statistics the
// mask pass adds to num_entries_scanned_in_filter)
long long expr_filter_entries(const pb200h_segment& seg, const pb200h_query& q);
}  // namespace pb200h
