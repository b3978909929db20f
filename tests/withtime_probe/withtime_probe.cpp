// withtime_probe.cpp -- TEST shim: pb200::plan_scan (pinot_b200/csrc/pb200_plan.cpp) for FIRST/LASTWITHTIME queries on
// segments made of column metadata alone, without a GPU.  Built by tests/test_withtime_cpu.py with g++ against the
// in-tree library.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../pinot_b200/csrc/pb200_plan.h"

extern "C" {

typedef struct {
  int32_t fwd_kind, stored_type, bits, cardinality;
  int32_t dict_native;  // 1: the column has a device dictionary (a sentinel pointer, never dereferenced)
  int32_t dict_hash;    // the dictionary's content hash (equal hashes: one dictionary)
} wt_probe_col;

enum { WP_SEG = 20, WP_AGG = 6 };
typedef struct {  // every field int64: tests/test_withtime_cpu.py mirrors this list
  int64_t nres, group_by, hashed, groups, smem_groups, spec, num_slots, num_agg_codes, warps, ctas_per_sm, smem_bytes;
  int64_t slot_col[12];
  int64_t code_agg[WP_AGG], code_fn[WP_AGG], code_vk[WP_AGG], code_slot_words[WP_AGG], wt_time[WP_AGG], val_kind[WP_AGG];
  int64_t doc_base[WP_SEG][WP_AGG];
} wt_probe_plan;

int64_t wt_probe_plan_size(void) { return (int64_t)sizeof(wt_probe_plan); }
// the launch descriptors the change must leave byte-identical
int64_t wt_probe_segdesc_size(void) { return (int64_t)sizeof(pb200::SegDesc); }
int64_t wt_probe_smem_header_size(void) { return (int64_t)sizeof(pb200::SmemHeader); }
uint64_t wt_probe_key(uint32_t time_id, uint32_t ordinal) { return pb200::withtime_key(time_id, ordinal); }

// cols: nseg x ncols.  args: one per aggregation, or NULL.  SegDesc bytes of segment 0 go to seg0 (sizeof(SegDesc)).
int32_t wt_probe_plan_scan(int32_t sm_count, int32_t max_smem_optin, const pb200_query* query, const pb200_agg_arg* args,
                           const wt_probe_col* cols, int32_t ncols, const int32_t* num_docs, int32_t nseg, int64_t dense_max,
                           wt_probe_plan* out, void* seg0) {
  using namespace pb200;
  static uint32_t sentinel[4];
  std::vector<pb200_segment> segs(nseg);
  std::vector<pb200_segment*> ptrs(nseg);
  for (int s = 0; s < nseg; s++) {
    segs[s].num_docs = num_docs[s];
    segs[s].cols.resize(ncols);
    for (int k = 0; k < ncols; k++) {
      const wt_probe_col& p = cols[(size_t)s * ncols + k];
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
  std::vector<double> p(query->num_aggs > 0 ? query->num_aggs : 1, 0.0);
  for (int a = 0; args && a < query->num_aggs; a++) p[a] = args[a].p;
  const int rc = plan_scan(ctx.tune, DeviceLimits{sm_count, max_smem_optin}, query, ptrs.data(), nseg, true, &plan,
                           args ? p.data() : nullptr, args);
  if (rc) return rc;
  wt_probe_plan& o = *out;
  o.nres = plan.nres; o.group_by = plan.group_by; o.smem_groups = plan.q.smem_groups; o.spec = plan.variant.spec;
  o.num_slots = plan.q.num_slots; o.num_agg_codes = plan.segs[0].num_agg_codes;
  o.warps = plan.warps; o.ctas_per_sm = plan.ctas_per_sm; o.smem_bytes = (int64_t)plan.smem_bytes;
  for (int k = 0; k < plan.q.num_slots && k < 12; k++) o.slot_col[k] = plan.slot_cols[k];
  for (int k = 0; k < plan.segs[0].num_agg_codes && k < WP_AGG; k++) {
    const uint32_t c = plan.segs[0].agg_code[k];
    o.code_agg[k] = c & 7u; o.code_fn[k] = (c >> 4) & 7u; o.code_vk[k] = (c >> 8) & 7u; o.code_slot_words[k] = c >> 18;
  }
  for (int a = 0; a < plan.q.num_aggs && a < WP_AGG; a++) {
    o.wt_time[a] = plan.wt_time[a];
    o.val_kind[a] = plan.q.aggs[a].val_kind;
    for (int s = 0; s < nseg && s < WP_SEG; s++) o.doc_base[s][a] = plan.segs[s].distinct_words[a];
  }
  if (plan.group_by) { o.hashed = plan.tables[0].hashed; o.groups = plan.tables[0].groups; }
  if (seg0) memcpy(seg0, &plan.segs[0], sizeof(SegDesc));
  return PB200_OK;
}

}  // extern "C"
