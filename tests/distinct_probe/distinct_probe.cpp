// distinct_probe.cpp -- TEST shim: pb200::plan_distinct / distinct_rescan (pinot_b200/csrc/pb200_plan.cpp) on segments
// made of column metadata alone, without a GPU.  Built by tests/test_distinct_cpu.py with g++ against the in-tree library.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../pinot_b200/csrc/pb200_plan.h"

extern "C" {

typedef struct {
  int32_t fwd_kind, stored_type, bits, cardinality;
  int32_t dict_native;  // 1: the column has a device dictionary (a sentinel pointer, never dereferenced)
  int32_t dict_hash;    // the dictionary's content hash (equal hashes: one dictionary)
} dist_probe_col;

enum { DP_SEG = 40, DP_COL = 8 };
typedef struct {  // every field int64: tests/test_distinct_cpu.py mirrors this list
  int64_t nres, table_entries, prefix, num_order, num_rescan;
  int64_t order_key[DP_COL], order_desc[DP_COL];
  int64_t table_off[DP_SEG], table_size[DP_SEG], scan_docs[DP_SEG], bound[DP_SEG], rescan[DP_SEG];
  int64_t cards[DP_SEG][DP_COL], mult[DP_SEG][DP_COL];
} dist_probe_plan;

int64_t dist_probe_plan_size(void) { return (int64_t)sizeof(dist_probe_plan); }

// cols: nseg x ncols.  tables: NULL, or the call's first-occurrence table block (table_entries u64, filled in by the
// caller after a first call that returned the layout): the probe counts each result's entries below its bound as the
// device count kernel does and applies distinct_rescan.
int32_t dist_probe_plan_distinct(int32_t sm_count, int32_t max_smem_optin, const pb200_query* filter_only,
                                 const pb200_selection* distinct, const dist_probe_col* cols, int32_t ncols, const int32_t* num_docs,
                                 int32_t nseg, int32_t merge, int32_t prefix, const uint64_t* tables, dist_probe_plan* out) {
  using namespace pb200;
  static uint32_t sentinel[4];
  std::vector<pb200_segment> segs(nseg);
  std::vector<pb200_segment*> ptrs(nseg);
  for (int s = 0; s < nseg; s++) {
    segs[s].num_docs = num_docs[s];
    segs[s].cols.resize(ncols);
    for (int k = 0; k < ncols; k++) {
      const dist_probe_col& p = cols[(size_t)s * ncols + k];
      DeviceColumn& c = segs[s].cols[k];
      c.fwd_kind = p.fwd_kind; c.stored_type = p.stored_type; c.bits = p.bits; c.cardinality = p.cardinality;
      c.fwd = sentinel;
      c.dict_native = p.dict_native ? sentinel : nullptr;
      c.dict_hash = (uint64_t)(uint32_t)p.dict_hash;
    }
    ptrs[s] = &segs[s];
  }
  pb200_ctx ctx;
  DistinctPlan plan;
  memset(out, 0, sizeof *out);
  const int rc = plan_distinct(ctx.tune, DeviceLimits{sm_count, max_smem_optin}, filter_only, distinct, ptrs.data(), nseg,
                               merge != 0, prefix != 0, &plan);
  if (rc) return rc;
  dist_probe_plan& o = *out;
  o.nres = plan.nres; o.table_entries = plan.table_entries; o.prefix = plan.sel.prefix;
  o.num_order = (int64_t)plan.order_key.size();
  for (size_t k = 0; k < plan.order_key.size() && k < DP_COL; k++) { o.order_key[k] = plan.order_key[k]; o.order_desc[k] = plan.order_desc[k]; }
  const std::vector<unsigned long long> bound = distinct_bounds(plan, ptrs.data());
  for (int r = 0; r < plan.nres && r < DP_SEG; r++) {
    o.table_off[r] = plan.table_off[r]; o.table_size[r] = plan.table_size[r]; o.bound[r] = (int64_t)bound[r];
  }
  for (int s = 0; s < nseg && s < DP_SEG; s++) {
    o.scan_docs[s] = plan.sel.scan_docs[s];
    for (size_t k = 0; k < plan.cards[s].size() && k < DP_COL; k++) { o.cards[s][k] = plan.cards[s][k]; o.mult[s][k] = plan.mult[s][k]; }
  }
  if (tables) {
    std::vector<long long> below(plan.nres, 0);
    for (int r = 0; r < plan.nres; r++)
      for (long long i = 0; i < plan.table_size[r]; i++) below[r] += tables[plan.table_off[r] + i] < bound[r];
    const std::vector<int> rs = distinct_rescan(plan, ptrs.data(), below);
    o.num_rescan = (int64_t)rs.size();
    for (size_t i = 0; i < rs.size() && i < DP_SEG; i++) o.rescan[i] = rs[i];
  }
  return PB200_OK;
}

}  // extern "C"
