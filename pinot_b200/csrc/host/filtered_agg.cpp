// filtered_agg.cpp -- aggregations with FILTER (WHERE ...) clauses on the accelerated path.
//
// Reference: AggregationFunctionUtils.buildFilteredAggregationInfos (core/query/aggregation/function/
// AggregationFunctionUtils.java:312-403) groups the functions by their FILTER clause; every group becomes one
// "aggregation info" = its own projection over (main filter AND sub filter) (CombinedFilterOperator), the functions without a
// clause run over the main filter, and for GROUP BY queries the main-filter info exists even with no function in it so that
// every group of the main filter appears.  FilteredGroupByOperator.getNextBlock (core/operator/query/
// FilteredGroupByOperator.java:113-160) / FilteredAggregationOperator run the infos one after the other with ONE shared group
// key generator; holders of groups an info never saw keep the function's default; the execution statistics of the infos add up.
//
// Here every info is ONE ordinary device submission (the same scan kernel, filter = main AND sub in one tree, all segments of
// the call) and the per-info results are aligned by group key on the host: the main-filter result defines the rows (it is a
// superset of every info's groups), each info's columns are scattered into them.  Keys are dictIds of the same segment (or of
// the bound domain when merge_segments is set), so equal keys mean equal values.
//
// Deviations (statistics only, never results): the reference folds a sub filter that matches every doc into the main info
// and skips the sub filters when the main filter matches nothing; here such infos still run as their own (cheap) submission,
// so numDocsScanned / numEntriesScanned* can be larger than the reference's in those two corner cases.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <unordered_map>

#include "host_internal.h"

namespace pb200h {
namespace {

struct KeyHash {
  size_t operator()(const std::vector<int32_t>& k) const {
    uint64_t h = 1469598103934665603ull;
    for (int32_t v : k) { h ^= (uint32_t)v; h *= 1099511628211ull; }
    return (size_t)h;
  }
};

struct ResultGuard {
  std::vector<pb200_result*> all;
  ~ResultGuard() { for (auto r : all) if (r) pb200_result_free(r); }
};

}  // namespace

int execute_filtered(pb200_ctx* ctx, const pb200h_query& q, const pb200_order_by* order, const pb200_having* having,
                     const pb200_post_aggs* post, pb200h_segment* const* segs, int nseg, pb200_result** results, int32_t* kinds) {
  if (q.merge_segments == 2) { set_error("FILTER clauses with a deferred (cross-GPU) combine are not accelerated"); return PB200_E_UNSUPPORTED; }
  const int nagg = q.num_aggs, ngb = q.num_group_by;
  const int nres = q.merge_segments ? 1 : nseg;
  // ---- infos: distinct FILTER clauses in order of first appearance, then the main filter ----
  struct Info { int start = 0, count = 0; std::vector<int> aggs; };
  std::vector<Info> infos;
  std::vector<int> non_filtered;
  for (int a = 0; a < nagg; a++) {
    const int cnt = q.agg_filter_count[a];
    if (cnt <= 0) { non_filtered.push_back(a); continue; }
    const int st = q.agg_filter_start[a];
    size_t at = 0;
    while (at < infos.size() && !(infos[at].start == st && infos[at].count == cnt)) at++;
    if (at == infos.size()) { Info i; i.start = st; i.count = cnt; infos.push_back(i); }
    infos[at].aggs.push_back(a);
  }
  const bool main_info = !non_filtered.empty() || ngb > 0;  // AggregationFunctionUtils.java:388-400
  const pb200h_agg probe{PB200_AGG_COUNT, nullptr};          // main info without functions: only its groups are needed

  ResultGuard guard;
  std::vector<std::vector<pb200_result*>> info_results;  // [info][result]
  auto run = [&](const pb200h_filter_node* sub, int nsub, const std::vector<int>& agg_idx) -> int {
    std::vector<pb200h_filter_node> nodes(q.filter, q.filter + q.num_filter_nodes);
    if (nsub > 0) {
      nodes.insert(nodes.end(), sub, sub + nsub);
      if (q.num_filter_nodes > 0) {  // CombinedFilterOperator(main, sub): both must match
        pb200h_filter_node an;
        memset(&an, 0, sizeof an);
        an.type = PB200H_AND; an.num_children = 2;
        nodes.push_back(an);
      }
    }
    std::vector<pb200h_agg> aggs;
    for (int a : agg_idx) aggs.push_back(q.aggs[a]);
    if (aggs.empty()) aggs.push_back(probe);
    pb200h_query sq = q;
    sq.num_filter_nodes = (int)nodes.size();
    sq.filter = nodes.data();
    sq.num_aggs = (int)aggs.size();
    sq.aggs = aggs.data();
    sq.agg_filter_nodes = nullptr; sq.agg_filter_start = nullptr; sq.agg_filter_count = nullptr;
    std::vector<pb200_result*> rs(nres, nullptr);
    int rc = pb200h_execute(ctx, &sq, segs, nseg, rs.data(), nullptr);
    if (rc) return rc;
    guard.all.insert(guard.all.end(), rs.begin(), rs.end());
    info_results.push_back(std::move(rs));
    return PB200_OK;
  };
  for (const Info& inf : infos) { int rc = run(q.agg_filter_nodes + inf.start, inf.count, inf.aggs); if (rc) return rc; }
  if (main_info) { int rc = run(nullptr, 0, non_filtered); if (rc) return rc; }

  // ---- align by group key ----
  std::vector<std::unique_ptr<pb200_result>> aligned(nres);
  for (int r = 0; r < nres; r++) {
    const pb200_result* base = main_info ? info_results.back()[r] : nullptr;  // defines the rows of a GROUP BY result
    pb200_result_meta bm;
    memset(&bm, 0, sizeof bm);
    if (base) pb200_result_meta_get(base, &bm);
    const size_t rows = ngb > 0 ? (size_t)std::max(bm.num_groups, 0) : 1;
    std::unique_ptr<pb200_result> R(new pb200_result());
    R->meta = bm;
    R->meta.num_group_by = ngb; R->meta.num_aggs = nagg;
    R->meta.num_groups = ngb > 0 ? (int32_t)rows : -1;
    R->meta.num_docs_scanned = 0; R->meta.num_entries_scanned_in_filter = 0; R->meta.num_entries_scanned_post_filter = 0;
    R->meta.device_ms = 0;
    R->agg_functions.resize(nagg);
    R->dbl.resize(nagg); R->lng.resize(nagg); R->ids.resize(nagg); R->distinct.resize(nagg);
    for (int a = 0; a < nagg; a++) {
      const int fn = q.aggs[a].function;
      R->agg_functions[a] = fn;
      // defaults of a holder that never saw the group: Sum 0, Min +inf, Max -inf (DoubleGroupByResultHolder default values),
      // Count 0, Avg (0, 0), DistinctCount empty set
      R->dbl[a].assign(rows, fn == PB200_AGG_MIN ? INFINITY : fn == PB200_AGG_MAX ? -INFINITY : 0.0);
      R->lng[a].assign(rows, 0);
      R->ids[a].assign(rows, -1);
      if (fn == PB200_AGG_DISTINCTCOUNT) R->distinct[a].resize(rows);
    }
    std::unordered_map<std::vector<int32_t>, size_t, KeyHash> row_of;
    if (ngb > 0 && rows) {
      const int32_t* bk = nullptr;
      pb200_result_columns(base, &bk, nullptr, nullptr, nullptr);
      R->keys.assign(bk, bk + rows * ngb);
      row_of.reserve(rows * 2);
      for (size_t i = 0; i < rows; i++) row_of.emplace(std::vector<int32_t>(bk + i * ngb, bk + (i + 1) * ngb), i);
    }
    for (size_t i = 0; i < info_results.size(); i++) {
      const bool is_main = main_info && i + 1 == info_results.size();
      const std::vector<int>& agg_idx = is_main ? non_filtered : infos[i].aggs;
      const pb200_result* sr = info_results[i][r];
      pb200_result_meta sm;
      pb200_result_meta_get(sr, &sm);
      R->meta.num_docs_scanned += sm.num_docs_scanned;
      R->meta.num_entries_scanned_in_filter += sm.num_entries_scanned_in_filter;
      // (projected columns of the probe COUNT(*) are the group-by columns only, as for an empty function list)
      R->meta.num_entries_scanned_post_filter += sm.num_entries_scanned_post_filter;
      R->meta.num_total_docs = sm.num_total_docs;
      R->meta.device_ms += sm.device_ms;
      if (!base) { R->meta.regime = sm.regime; R->meta.groups_limit_reached = 0; }
      if (agg_idx.empty()) continue;
      const size_t srows = sm.num_groups < 0 ? 1 : (size_t)sm.num_groups;
      if (srows == 0) continue;
      const int32_t* sk = nullptr;
      const double* sd[8] = {nullptr};
      const int64_t* sl[8] = {nullptr};
      const int32_t* si[8] = {nullptr};
      pb200_result_columns(sr, &sk, sd, sl, si);
      std::vector<int32_t> key(ngb);
      for (size_t g = 0; g < srows; g++) {
        size_t row = 0;
        if (ngb > 0) {
          key.assign(sk + g * ngb, sk + (g + 1) * ngb);
          auto it = row_of.find(key);
          if (it == row_of.end()) { set_error("filtered aggregation: a group of a FILTER clause is missing from the main filter's groups"); return PB200_E_INVALID; }
          row = it->second;
        }
        for (size_t j = 0; j < agg_idx.size(); j++) {
          const int a = agg_idx[j];
          if (sd[j]) R->dbl[a][row] = sd[j][g];
          if (sl[j]) R->lng[a][row] = sl[j][g];
          if (si[j]) R->ids[a][row] = si[j][g];
          if (q.aggs[a].function == PB200_AGG_DISTINCTCOUNT) {
            const int64_t n = pb200_result_distinct(sr, (int)j, (int)g, nullptr, 0);
            if (n > 0) { R->distinct[a][row].resize((size_t)n); pb200_result_distinct(sr, (int)j, (int)g, R->distinct[a][row].data(), n); }
          }
        }
      }
    }
    // HAVING and ORDER BY: the infos ran unfiltered and unordered (each holds partial columns, and a trimmed info could miss
    // a group of the main filter); the aligned rows are filtered, ordered and trimmed here, by the device's rules
    if (having && ngb > 0) pb200::having_rows_host(R.get(), *having, R->agg_functions.data());
    if (order && ngb > 0) pb200::order_rows_host(R.get(), *order, R->agg_functions.data(), post);
    aligned[r] = std::move(R);
  }
  for (int r = 0; r < nres; r++) results[r] = aligned[r].release();  // only when every result was built
  if (kinds) for (int s = 0; s < nseg; s++) kinds[s] = ngb > 0 ? PB200H_OP_GROUP_BY : PB200H_OP_AGGREGATION;
  return PB200_OK;
}

}  // namespace pb200h
