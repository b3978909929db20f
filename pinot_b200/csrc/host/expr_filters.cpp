// expr_filters.cpp -- predicates on expressions of two or more columns: WHERE a > b, WHERE price * qty > 1000
// (DESIGN.md section 3.16).
//
// The reference builds an ExpressionFilterOperator for such a leaf: the expression is evaluated per row as a DOUBLE and
// compared by a raw-value predicate evaluator.  Here every such leaf of a call -- filter and FILTER (WHERE ...) clauses --
// is compiled (compile_multi_expression) and its doc set computed on the device by pb200_expr_doc_masks, one launch for
// the distinct (expression, predicate) pairs of the call over all its segments.  The masks live in a scope as long as the
// entry point's frame; plan_maker.cpp's build_segment_filter reads them from there and plans the leaf as a
// PB200_F_DOC_MASK | PB200_NODE_IDS_ON_DEVICE leaf in every segment.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "host_internal.h"

namespace pb200h {

namespace {
thread_local ExprFilterScope* g_scope = nullptr;

bool is_leaf(const pb200h_filter_node& n) { return n.type >= PB200H_EQ; }

// Identifies (expression, predicate) by value, so that a FILTER clause's submission, whose nodes are copies, finds the
// masks its caller resolved: canonical text, op, bounds and the literals' doubles bit for bit.
std::string leaf_key(const std::string& canonical, const pb200h_filter_node& n, const pb200h_literal* lits) {
  std::string k = canonical + "|" + std::to_string(n.type);
  auto bits = [&](double d) { uint64_t u; memcpy(&u, &d, 8); char b[20]; snprintf(b, sizeof b, "|%016llx", (unsigned long long)u); k += b; };
  if (n.type == PB200H_RANGE) {
    k += "|" + std::to_string((n.lower_unbounded ? 1 : 0) | (n.upper_unbounded ? 2 : 0) | (n.lower_inclusive ? 0 : 4) | (n.upper_inclusive ? 0 : 8));
    if (!n.lower_unbounded) bits(lits[n.values_offset].d);
    if (!n.upper_unbounded) bits(lits[n.values_offset + 1].d);
  } else {
    for (int v = 0; v < n.num_values; v++) bits(lits[n.values_offset + v].d);
  }
  return k;
}

const ExprFilterScope::Mask* find_in(const ExprFilterScope* s, const pb200h_segment* seg, const std::string& key) {
  for (; s; s = s->outer)
    for (const auto& m : s->masks)
      if (m.seg == seg && m.key == key) return &m;
  return nullptr;
}

// One compiled leaf: its program over the segments' column ids, its predicate and key
struct Leaf {
  std::string key;
  std::vector<pb200_transform_op> ops;
  std::vector<double> values;
  pb200_expr_predicate pred;
  int ncols = 0;
};

int compile_leaf(const pb200h_filter_node& n, const pb200h_literal* lits, pb200h_segment* const* segs, int nseg, Leaf& out) {
  if (n.type == PB200H_REGEXP_LIKE) { set_error("REGEXP_LIKE / LIKE on the expression '%s' is not accelerated", n.column); return PB200_E_UNSUPPORTED; }
  std::string canonical;
  std::vector<std::string> leaves;
  if (int rc = compile_multi_expression(n.column, &canonical, &out.ops, &leaves)) return rc;
  const int nlit = n.type == PB200H_RANGE ? 2 : n.num_values;
  if (nlit < 1 || !lits) { set_error("predicate on '%s' without literals", n.column); return PB200_E_INVALID; }
  for (int v = 0; v < nlit; v++)
    if (lits[n.values_offset + v].s) { set_error("the expression '%s' compared with a string literal is not accelerated", n.column); return PB200_E_UNSUPPORTED; }
  std::vector<int> distinct;
  for (pb200_transform_op& o : out.ops) {
    if (o.op != PB200_T_COLUMN) continue;
    const char* name = leaves[(size_t)o.i].c_str();
    const int ci = segs[0]->column_index(name);
    if (ci < 0 || ci >= segs[0]->num_stored) { set_error("expression '%s': unknown column '%s'", n.column, name); return PB200_E_INVALID; }
    for (int s = 1; s < nseg; s++)
      if (segs[s]->column_index(name) != ci) { set_error("expression '%s': column '%s' is not at the same position in every segment", n.column, name); return PB200_E_INVALID; }
    if (segs[0]->cols[ci].data_type == PB200_STRING) { set_error("expression '%s': STRING column '%s' in arithmetic", n.column, name); return PB200_E_UNSUPPORTED; }
    o.i = ci;
    if (std::find(distinct.begin(), distinct.end(), ci) == distinct.end()) distinct.push_back(ci);
  }
  out.ncols = (int)distinct.size();
  out.key = leaf_key(canonical, n, lits);
  pb200_expr_predicate& p = out.pred;
  memset(&p, 0, sizeof p);
  const pb200h_literal* v = lits + n.values_offset;
  switch (n.type) {
    case PB200H_EQ: p.op = PB200_EXPR_EQ; break;
    case PB200H_NEQ: p.op = PB200_EXPR_NEQ; break;
    case PB200H_IN: p.op = PB200_EXPR_IN; break;
    case PB200H_NOT_IN: p.op = PB200_EXPR_NOT_IN; break;
    default: p.op = PB200_EXPR_RANGE;
  }
  if (p.op == PB200_EXPR_RANGE) {
    p.flags = (n.lower_unbounded ? 1 : 0) | (n.upper_unbounded ? 2 : 0) | (n.lower_inclusive ? 0 : 4) | (n.upper_inclusive ? 0 : 8);
    p.lo = n.lower_unbounded ? 0.0 : v[0].d;
    p.hi = n.upper_unbounded ? 0.0 : v[1].d;
  } else {
    for (int k = 0; k < n.num_values; k++) out.values.push_back(v[k].d);
    p.num_values = n.num_values;
  }
  return PB200_OK;
}

std::vector<const pb200h_filter_node*> expression_leaves(const pb200h_query& q) {
  std::vector<const pb200h_filter_node*> out;
  for (int i = 0; i < q.num_filter_nodes; i++) if (is_leaf(q.filter[i]) && is_expression_filter(q.filter[i].column)) out.push_back(&q.filter[i]);
  if (q.agg_filter_count && q.agg_filter_start && q.agg_filter_nodes)
    for (int a = 0; a < q.num_aggs; a++)
      for (int k = 0; k < q.agg_filter_count[a]; k++) {
        const pb200h_filter_node& n = q.agg_filter_nodes[q.agg_filter_start[a] + k];
        if (is_leaf(n) && is_expression_filter(n.column)) out.push_back(&n);
      }
  return out;
}
}  // namespace

ExprFilterScope::ExprFilterScope() : outer(g_scope) { g_scope = this; }
ExprFilterScope::~ExprFilterScope() {
  g_scope = outer;
  for (const Mask& m : masks) pb200_doc_mask_free(ctx, m.mask);
}

int resolve_expr_filters(pb200_ctx* ctx, const pb200h_query& q, pb200h_segment* const* segs, int nseg, ExprFilterScope& scope,
                         bool launch) {
  std::vector<Leaf> todo;
  for (const pb200h_filter_node* n : expression_leaves(q)) {
    Leaf leaf;
    if (int rc = compile_leaf(*n, q.literals, segs, nseg, leaf)) return rc;
    bool done = true;
    for (int s = 0; s < nseg && done; s++) done = find_in(g_scope, segs[s], leaf.key) != nullptr;
    if (done) continue;   // the caller's scope (a FILTER clause's submission) has it
    bool seen = false;
    for (const Leaf& t : todo) seen |= t.key == leaf.key;
    if (!seen) todo.push_back(std::move(leaf));
  }
  if (todo.empty() || !launch) return PB200_OK;
  if (!ctx) { set_error("predicates on expressions need a context"); return PB200_E_INVALID; }
  std::vector<pb200_expr_predicate> preds;
  for (Leaf& t : todo) {
    t.pred.program = pb200_expr_program{(int32_t)t.ops.size(), 0, t.ops.data()};
    t.pred.values = t.values.empty() ? nullptr : t.values.data();
    preds.push_back(t.pred);
  }
  std::vector<pb200_segment*> dev(nseg);
  for (int s = 0; s < nseg; s++) dev[s] = segs[s]->dev;
  std::vector<uint32_t*> masks(preds.size() * (size_t)nseg, nullptr);
  if (int rc = pb200_expr_doc_masks(ctx, (int)preds.size(), preds.data(), dev.data(), nseg, masks.data())) return rc;
  scope.ctx = ctx;
  for (size_t p = 0; p < todo.size(); p++)
    for (int s = 0; s < nseg; s++) scope.masks.push_back({todo[p].key, segs[s], masks[p * nseg + s], todo[p].ncols});
  return PB200_OK;
}

int expr_filter_mask(const pb200h_segment& seg, const pb200h_filter_node& n, const pb200h_literal* lits, std::string* canonical,
                     const uint32_t** mask, int* ncols) {
  std::vector<pb200_transform_op> ops;
  std::vector<std::string> leaves;
  if (int rc = compile_multi_expression(n.column, canonical, &ops, &leaves)) return rc;
  const ExprFilterScope::Mask* m = find_in(g_scope, &seg, leaf_key(*canonical, n, lits));
  *mask = m ? m->mask : nullptr;
  *ncols = m ? m->ncols : 0;
  return PB200_OK;
}

long long expr_filter_entries(const pb200h_segment& seg, const pb200h_query& q) {
  long long total = 0;
  for (int i = 0; i < q.num_filter_nodes; i++) {
    const pb200h_filter_node& n = q.filter[i];
    if (!is_leaf(n) || !is_expression_filter(n.column)) continue;
    std::string canonical;
    const uint32_t* mask = nullptr;
    int ncols = 0;
    if (expr_filter_mask(seg, n, q.literals, &canonical, &mask, &ncols) == PB200_OK) total += (long long)seg.num_docs * ncols;
  }
  return total;
}

}  // namespace pb200h
