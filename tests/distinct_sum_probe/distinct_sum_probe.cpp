// distinct_sum_probe.cpp -- TEST shim: the DISTINCTSUM / DISTINCTAVG eligibility rule and finalize arithmetic
// (pinot_b200/csrc/pb200_distinct_sum.h, the same code the device runs) and pb200::plan_scan's bitset sharing, on segments
// made of column metadata and a host dictionary, without a GPU.  Built by tests/test_distinct_sum_cpu.py with g++ against
// the in-tree library.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../pinot_b200/csrc/pb200_plan.h"

extern "C" {

// eligibility of a sorted dictionary (native values): 1 and the exponent, or 0
int32_t ds_probe_grid(int32_t stored_type, const void* dict, int32_t card, int32_t* e) {
  return pb200::distinct_grid(stored_type, static_cast<const unsigned char*>(dict), card, e) ? 1 : 0;
}

// the final value over members given as doubles on grid e (FLOAT / DOUBLE dictionaries), as the device adds them
double ds_probe_final_doubles(int32_t fn, const double* v, int64_t n, int32_t e) {
  pb200::i128 sum = 0;
  uint32_t flags = 0;
  for (int64_t i = 0; i < n; i++) flags |= pb200::ds_add_double(v[i], e, &sum);
  return pb200::distinct_final(fn, sum, (unsigned long long)n, flags, e);
}

// the final value of a state {sum = hi * 2^64 + lo (two's complement), n, flags} on grid e
double ds_probe_final_state(int32_t fn, uint64_t lo, uint64_t hi, uint64_t n, uint32_t flags, int32_t e) {
  const unsigned long long st[4] = {lo, hi, n, flags};
  return pb200::distinct_final(fn, pb200::ds_sum_of(st), n, flags, e);
}

typedef struct {
  int32_t stored_type, bits, cardinality;
  int32_t raw;           // 1: a raw 32-bit column (no dictIds)
  int32_t dict_hash;     // the dictionary's content hash (equal hashes: one dictionary)
  const void* dict;      // host dictionary, native values (NULL: none)
} ds_probe_col;

enum { DP_AGG = 8 };
typedef struct {  // every field int64: tests/test_distinct_sum_cpu.py mirrors this list
  int64_t group_by, num_agg_codes;
  int64_t ds_rep[DP_AGG], code_fn[DP_AGG], code_agg[DP_AGG], slot[DP_AGG], dwords[DP_AGG], distinct_words[DP_AGG];
} ds_probe_plan;

int64_t ds_probe_plan_size(void) { return (int64_t)sizeof(ds_probe_plan); }

static uint32_t g_sentinel[64];

int32_t ds_probe_plan_scan(const pb200_query* query, const ds_probe_col* cols, int32_t ncols, const int32_t* num_docs,
                           int32_t nseg, ds_probe_plan* out) {
  using namespace pb200;
  std::vector<pb200_segment> segs(nseg);
  std::vector<pb200_segment*> ptrs(nseg);
  for (int s = 0; s < nseg; s++) {
    segs[s].num_docs = num_docs[s];
    segs[s].cols.resize(ncols);
    for (int k = 0; k < ncols; k++) {
      const ds_probe_col& p = cols[(size_t)s * ncols + k];
      DeviceColumn& c = segs[s].cols[k];
      c.fwd_kind = PB200_FWD_DICT_FIXEDBIT; c.stored_type = p.stored_type; c.bits = p.raw ? 32 : p.bits; c.cardinality = p.cardinality;
      c.fwd = g_sentinel;
      c.dict_native = p.raw ? nullptr : g_sentinel;
      c.dict_hash = (uint64_t)(uint32_t)p.dict_hash;
      if (p.dict) {
        const size_t w = (p.stored_type == PB200_LONG || p.stored_type == PB200_DOUBLE) ? 8 : 4;
        c.dict_host.assign(static_cast<const unsigned char*>(p.dict), static_cast<const unsigned char*>(p.dict) + w * p.cardinality);
      }
    }
    ptrs[s] = &segs[s];
  }
  pb200_ctx ctx;
  ScanPlan plan;
  memset(out, 0, sizeof *out);
  const int rc = plan_scan(ctx.tune, DeviceLimits{132, 232448}, query, ptrs.data(), nseg, true, &plan, nullptr);
  if (rc) return rc;
  ds_probe_plan& o = *out;
  o.group_by = plan.group_by;
  o.num_agg_codes = plan.segs[0].num_agg_codes;
  for (int a = 0; a < DP_AGG; a++) { o.ds_rep[a] = -1; o.code_fn[a] = -1; o.code_agg[a] = -1; o.slot[a] = -1; }
  for (int a = 0; a < plan.q.num_aggs && a < DP_AGG; a++) {
    o.ds_rep[a] = plan.ds_rep[a];
    o.slot[a] = plan.q.aggs[a].slot;
    if (plan.group_by) o.dwords[a] = plan.tables[0].dwords[a];
    else o.distinct_words[a] = (int64_t)plan.distinct_words[0][a];
  }
  for (int i = 0; i < plan.segs[0].num_agg_codes && i < DP_AGG; i++) {
    o.code_agg[i] = plan.segs[0].agg_code[i] & 7;
    o.code_fn[i] = (plan.segs[0].agg_code[i] >> 4) & 7;
  }
  return PB200_OK;
}

}  // extern "C"
