// moments_probe.cpp -- TEST shim: the VAR / STDDEV eligibility rule and finalize arithmetic (pinot_b200/csrc/pb200_moments.h,
// the same code the device runs) and pb200::plan_scan's expansion into limb sums, on segments made of column metadata
// alone, without a GPU.  Built by tests/test_variance_cpu.py with g++ against the in-tree library.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../pinot_b200/csrc/pb200_plan.h"

extern "C" {

// eligibility of a sorted dictionary (native values): 1 and the grid, or 0
int32_t mom_probe_grid(int32_t stored_type, const void* dict, int32_t card, int64_t* c_mant, int32_t* c_exp, int32_t* e,
                       uint32_t* k_max) {
  pb200::MomentGrid g;
  if (!pb200::moments_grid(stored_type, static_cast<const unsigned char*>(dict), card, &g)) return 0;
  *c_mant = g.c_mant; *c_exp = g.c_exp; *e = g.e; *k_max = g.k_max;
  return 1;
}

// the final value from the three limb sums as the scan leaves them (sum(limb) - n * 2^31) and n; the exact moments back
double mom_probe_final(int32_t fn, uint64_t n, int64_t sum_k, int64_t sum_h, int64_t sum_l, int32_t e, uint64_t* s1,
                       uint64_t* s2_lo, uint64_t* s2_hi) {
  const pb200::Moments m = pb200::moments_from_sums(n, sum_k, sum_h, sum_l);
  *s1 = m.s1; *s2_lo = (uint64_t)m.s2; *s2_hi = (uint64_t)(m.s2 >> 64);
  return pb200::moments_final(fn, m, e);
}

typedef struct {
  int32_t fwd_kind, stored_type, bits, cardinality;
  int32_t dict_native;  // 1: the column has a device dictionary (a sentinel pointer, never dereferenced)
  int32_t dict_hash;    // the dictionary's content hash (equal hashes: one dictionary)
  int32_t eligible;     // the limb dictionaries: -1 not prepared, 0 off the grid, 1 built (sentinel limbs)
} mom_probe_col;

enum { MP_AGG = 6 };
typedef struct {  // every field int64: tests/test_variance_cpu.py mirrors this list
  int64_t num_aggs, num_user_aggs, spec, smem_groups, need_count, carrier_agg, projected, num_slots;
  int64_t mom_first[MP_AGG], limb[MP_AGG], fn[MP_AGG], val_kind[MP_AGG], slot[MP_AGG], dict_off[MP_AGG];
} mom_probe_plan;

int64_t mom_probe_plan_size(void) { return (int64_t)sizeof(mom_probe_plan); }

static uint32_t g_sentinel[64];
static uint32_t g_limbs[3 * 4096];

int32_t mom_probe_plan_scan(int32_t sm_count, int32_t max_smem_optin, const pb200_query* query, const mom_probe_col* cols,
                            int32_t ncols, const int32_t* num_docs, int32_t nseg, mom_probe_plan* out) {
  using namespace pb200;
  std::vector<pb200_segment> segs(nseg);
  std::vector<pb200_segment*> ptrs(nseg);
  for (int s = 0; s < nseg; s++) {
    segs[s].num_docs = num_docs[s];
    segs[s].cols.resize(ncols);
    for (int k = 0; k < ncols; k++) {
      const mom_probe_col& p = cols[(size_t)s * ncols + k];
      DeviceColumn& c = segs[s].cols[k];
      c.fwd_kind = p.fwd_kind; c.stored_type = p.stored_type; c.bits = p.bits; c.cardinality = p.cardinality;
      c.fwd = g_sentinel;
      c.dict_native = p.dict_native ? g_sentinel : nullptr;
      c.dict_hash = (uint64_t)(uint32_t)p.dict_hash;
      if (p.eligible >= 0) {
        c.moments->eligible = p.eligible != 0;
        if (p.eligible) { c.moments->limbs = g_limbs; c.moments->entries = p.cardinality; }
        c.moments->ready.store(true);
      }
    }
    ptrs[s] = &segs[s];
  }
  pb200_ctx ctx;
  ScanPlan plan;
  memset(out, 0, sizeof *out);
  const int rc = plan_scan(ctx.tune, DeviceLimits{sm_count, max_smem_optin}, query, ptrs.data(), nseg, true, &plan, nullptr);
  for (int s = 0; s < nseg; s++)
    for (auto& c : segs[s].cols) c.moments->limbs = nullptr;   // sentinels, never freed
  if (rc) return rc;
  mom_probe_plan& o = *out;
  o.num_aggs = plan.q.num_aggs; o.num_user_aggs = plan.num_user_aggs; o.spec = plan.variant.spec;
  o.smem_groups = plan.q.smem_groups; o.projected = plan.projected; o.num_slots = plan.q.num_slots;
  o.need_count = plan.group_by ? plan.tables[0].need_count : 0;
  o.carrier_agg = plan.group_by ? plan.tables[0].carrier.agg : -1;
  for (int a = 0; a < MP_AGG; a++) { o.mom_first[a] = -1; o.limb[a] = -1; o.dict_off[a] = -1; }
  for (int a = 0; a < plan.num_user_aggs && a < MP_AGG; a++) o.mom_first[a] = plan.mom_first[a];
  for (int a = 0; a < plan.q.num_aggs && a < MP_AGG; a++) {
    o.limb[a] = plan.limb[a];
    o.fn[a] = plan.q.aggs[a].function;
    o.val_kind[a] = plan.q.aggs[a].val_kind;
    o.slot[a] = plan.q.aggs[a].slot;
    const uint32_t* d = static_cast<const uint32_t*>(plan.segs[0].dict[a]);
    if (d >= g_limbs && d < g_limbs + 3 * 4096) o.dict_off[a] = d - g_limbs;
  }
  return PB200_OK;
}

}  // extern "C"
