// patterns.cpp -- REGEXP_LIKE leaves: their matching dictIds, resolved on the device before a call is planned.
//
// The reference turns a pattern predicate on a dictionary column into the set of matching dictIds
// (RegexpLikePredicateEvaluatorFactory) and then builds the leaf like an IN's.  Here every pattern leaf of a call is
// resolved by pb200_match_pattern, one launch per distinct (pattern, column) over all segments of the call, and the ids
// are kept in a scope that lives as long as the entry point's frame; plan_maker.cpp's evaluate() reads them from there.
#include <cstring>
#include <string>
#include <vector>

#include "host_internal.h"

namespace pb200h {

namespace {
thread_local PatternScope* g_scope = nullptr;

const std::vector<int32_t>* find_in(const PatternScope* s, const HostColumn* c, const char* pattern) {
  for (; s; s = s->outer)
    for (const auto& e : s->ids)
      if (e.first.first == c && e.first.second == pattern) return &e.second;
  return nullptr;
}
}  // namespace

PatternScope::PatternScope() : outer(g_scope) { g_scope = this; }
PatternScope::~PatternScope() { g_scope = outer; }

const std::vector<int32_t>* pattern_ids(const HostColumn& c, const char* pattern) {
  return pattern ? find_in(g_scope, &c, pattern) : nullptr;
}

void pattern_alias(const HostColumn& from, const HostColumn& to, const char* pattern) {
  const std::vector<int32_t>* ids = pattern_ids(from, pattern);
  if (ids && g_scope && !pattern_ids(to, pattern)) g_scope->ids.push_back({{&to, pattern}, *ids});
}

int resolve_patterns(pb200_ctx* ctx, const pb200h_query& q, pb200h_segment* const* segs, int nseg, PatternScope& scope) {
  std::vector<const pb200h_filter_node*> leaves;
  for (int i = 0; i < q.num_filter_nodes; i++) if (q.filter[i].type == PB200H_REGEXP_LIKE) leaves.push_back(&q.filter[i]);
  if (q.agg_filter_count && q.agg_filter_start && q.agg_filter_nodes)
    for (int a = 0; a < q.num_aggs; a++)
      for (int k = 0; k < q.agg_filter_count[a]; k++) {
        const pb200h_filter_node& n = q.agg_filter_nodes[q.agg_filter_start[a] + k];
        if (n.type == PB200H_REGEXP_LIKE) leaves.push_back(&n);
      }
  for (const pb200h_filter_node* n : leaves) {
    if (n->num_values != 1 || !q.literals || !q.literals[n->values_offset].s) { set_error("REGEXP_LIKE leaf needs one string literal (the pattern)"); return PB200_E_INVALID; }
    const char* pattern = q.literals[n->values_offset].s;
    if (is_expression_filter(n->column)) { set_error("REGEXP_LIKE / LIKE on the expression '%s' is not accelerated", n->column); return PB200_E_UNSUPPORTED; }
    std::vector<pb200_segment*> dev(nseg);
    std::vector<int32_t> cols(nseg);
    std::vector<const HostColumn*> hcols(nseg);
    bool done = true;
    for (int s = 0; s < nseg; s++) {
      const int ci = segs[s]->column_index(n->column);
      if (ci < 0) { set_error("unknown column '%s'", n->column ? n->column : "(null)"); return PB200_E_INVALID; }
      const HostColumn& c = segs[s]->cols[ci];
      if (c.derived) { set_error("REGEXP_LIKE on the expression '%s' is not accelerated", c.name.c_str()); return PB200_E_UNSUPPORTED; }
      if (c.data_type != PB200_STRING) { set_error("REGEXP_LIKE on column '%s', which is not STRING, is not accelerated", c.name.c_str()); return PB200_E_UNSUPPORTED; }
      if (!c.has_dictionary) { set_error("REGEXP_LIKE on column '%s' without a dictionary is not accelerated", c.name.c_str()); return PB200_E_UNSUPPORTED; }
      dev[s] = segs[s]->dev; cols[s] = ci; hcols[s] = &c;
      done &= pattern_ids(c, pattern) != nullptr;
    }
    if (done) continue;   // an earlier leaf of this call, or the caller's scope, has it
    std::vector<std::vector<uint32_t>> bits(nseg);
    std::vector<uint32_t*> out(nseg);
    for (int s = 0; s < nseg; s++) {
      bits[s].assign(((size_t)hcols[s]->cardinality + 31) / 32 + 1, 0u);
      out[s] = bits[s].data();
    }
    if (int rc = pb200_match_pattern(ctx, pattern, nseg, dev.data(), cols.data(), out.data())) return rc;
    for (int s = 0; s < nseg; s++) {
      if (find_in(&scope, hcols[s], pattern)) continue;   // the same segment twice in the call
      std::vector<int32_t> ids;
      for (int id = 0; id < hcols[s]->cardinality; id++)
        if ((bits[s][id >> 5] >> (id & 31)) & 1u) ids.push_back(id);
      scope.ids.push_back({{hcols[s], pattern}, std::move(ids)});
    }
  }
  return PB200_OK;
}

}  // namespace pb200h
