// percentile_probe.cpp -- TEST shim: pb200::plan_scan (pinot_b200/csrc/pb200_plan.cpp) for PERCENTILE queries on segments
// made of column metadata alone, without a GPU.  Built by tests/test_percentile_cpu.py with g++ against the in-tree library.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../pinot_b200/csrc/pb200_plan.h"

extern "C" {

typedef struct {
  int32_t fwd_kind, stored_type, bits, cardinality;
  int32_t dict_native;  // 1: the column has a device dictionary (a sentinel pointer, never dereferenced)
  int32_t dict_hash;    // the dictionary's content hash (equal hashes: one dictionary)
} pct_probe_col;

enum { PP_SEG = 20, PP_AGG = 6 };
typedef struct {  // every field int64: tests/test_percentile_cpu.py mirrors this list
  int64_t nres, group_by, hashed, groups, stride, smem_groups, num_defer_codes, num_agg_codes, hist_total;
  int64_t pct_rep[PP_AGG], code_agg[PP_AGG], code_fn[PP_AGG], hist_per_group[PP_AGG], seg0_entries[PP_AGG];
  int64_t hist_entries[PP_SEG][PP_AGG];
} pct_probe_plan;

int64_t pct_probe_plan_size(void) { return (int64_t)sizeof(pct_probe_plan); }

// pb200::percentile_index, the copy of the index rule the finalize kernel runs (pb200_desc.h)
int64_t pct_probe_index(int64_t n, double p) { return pb200::percentile_index(n, p); }

// cols: nseg x ncols.  agg_args: one per aggregation, or NULL.
int32_t pct_probe_plan_scan(int32_t sm_count, int32_t max_smem_optin, const pb200_query* query, const double* agg_args,
                            const pct_probe_col* cols, int32_t ncols, const int32_t* num_docs, int32_t nseg, int64_t dense_max,
                            pct_probe_plan* out) {
  using namespace pb200;
  static uint32_t sentinel[4];
  std::vector<pb200_segment> segs(nseg);
  std::vector<pb200_segment*> ptrs(nseg);
  for (int s = 0; s < nseg; s++) {
    segs[s].num_docs = num_docs[s];
    segs[s].cols.resize(ncols);
    for (int k = 0; k < ncols; k++) {
      const pct_probe_col& p = cols[(size_t)s * ncols + k];
      DeviceColumn& c = segs[s].cols[k];
      c.fwd_kind = p.fwd_kind; c.stored_type = p.stored_type; c.bits = p.bits; c.cardinality = p.cardinality;
      c.fwd = sentinel;
      c.dict_native = p.dict_native ? sentinel : nullptr;
      c.dict_hash = (uint64_t)(uint32_t)p.dict_hash;
    }
    ptrs[s] = &segs[s];
  }
  pb200_ctx ctx;
  if (dense_max > 0) ctx.tune.dense_max = dense_max;
  ScanPlan plan;
  memset(out, 0, sizeof *out);
  const int rc = plan_scan(ctx.tune, DeviceLimits{sm_count, max_smem_optin}, query, ptrs.data(), nseg, true, &plan, agg_args);
  if (rc) return rc;
  pct_probe_plan& o = *out;
  o.nres = plan.nres; o.group_by = plan.group_by; o.smem_groups = plan.q.smem_groups; o.hist_total = plan.hist_total;
  o.num_defer_codes = plan.segs[0].num_defer_codes; o.num_agg_codes = plan.segs[0].num_agg_codes;
  for (int k = 0; k < plan.segs[0].num_agg_codes && k < PP_AGG; k++) {
    o.code_agg[k] = plan.segs[0].agg_code[k] & 7u;
    o.code_fn[k] = (plan.segs[0].agg_code[k] >> 4) & 7u;
  }
  for (int a = 0; a < query->num_aggs && a < PP_AGG; a++) {
    o.pct_rep[a] = plan.pct_rep[a];
    o.seg0_entries[a] = plan.segs[0].distinct_words[a];
  }
  if (plan.group_by) {
    const TableLayout& t = plan.tables[0];
    o.hashed = t.hashed; o.groups = t.groups; o.stride = t.stride;
    for (int a = 0; a < query->num_aggs && a < PP_AGG; a++) o.hist_per_group[a] = t.hist_per_group[a];
  } else {
    for (int r = 0; r < plan.nres && r < PP_SEG; r++)
      for (int a = 0; a < query->num_aggs && a < PP_AGG; a++) o.hist_entries[r][a] = (int64_t)plan.hist_entries[r][a];
  }
  return PB200_OK;
}

}  // extern "C"
