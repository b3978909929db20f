// spec_probe.cpp -- TEST shim: which scan kernel pb200::plan_scan picks (the shared-table GROUP BY specialisation or the
// generic one), and whether that choice leaves every other part of the plan as it is.  Segments are made of column
// metadata alone, as in tests/host_probe/host_probe.cpp (same probe_col layout).  Built by tests/test_scan_spec_plan_cpu.py
// with g++ against the in-tree library; nothing here ships.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../pinot_b200/csrc/pb200_plan.h"

namespace {
typedef struct {
  int32_t fwd_kind, stored_type, bits, cardinality;
  int32_t dict_native, dict_shared, has_inv, reserved;
  uint64_t dict_hash;
  const void* dict_host;
  uint64_t dict_host_bytes;
} probe_col;

template <class T>
bool same_bytes(const T& a, const T& b) { return memcmp(&a, &b, sizeof(T)) == 0; }

// every field of the plan except variant.spec
bool same_plan(const pb200::ScanPlan& a, const pb200::ScanPlan& b) {
  using namespace pb200;
  if (!same_bytes(a.q, b.q) || a.segs.size() != b.segs.size()) return false;
  for (size_t s = 0; s < a.segs.size(); s++) if (!same_bytes(a.segs[s], b.segs[s])) return false;
  if (a.slot_cols != b.slot_cols || a.leaf_node != b.leaf_node || a.group_by != b.group_by || a.merge != b.merge ||
      a.defer_finalize != b.defer_finalize || a.nres != b.nres || a.warps != b.warps || a.ctas_per_sm != b.ctas_per_sm ||
      a.skip_masks != b.skip_masks || a.smem_bytes != b.smem_bytes || a.variant.warps != b.variant.warps ||
      a.variant.group_by != b.variant.group_by || a.variant.defer != b.variant.defer ||
      a.variant.min_blocks != b.variant.min_blocks || a.chunks.size() != b.chunks.size() ||
      a.leaf_buffers.size() != b.leaf_buffers.size() || a.tables.size() != b.tables.size() ||
      a.distinct_words != b.distinct_words || a.hist_entries != b.hist_entries || a.hist_total != b.hist_total ||
      a.in_filter != b.in_filter || a.projected != b.projected)
    return false;
  for (size_t c = 0; c < a.chunks.size(); c++) {
    const LaunchChunk &x = a.chunks[c], &y = b.chunks[c];
    if (x.first_seg != y.first_seg || x.num_segs != y.num_segs || x.total_tiles != y.total_tiles || x.grid != y.grid) return false;
  }
  for (size_t i = 0; i < a.leaf_buffers.size(); i++) {
    const LeafBuffer &x = a.leaf_buffers[i], &y = b.leaf_buffers[i];
    if (x.kind != y.kind || x.seg != y.seg || x.leaf != y.leaf || x.words != y.words || x.lut != y.lut) return false;
  }
  for (size_t r = 0; r < a.tables.size(); r++) {
    const TableLayout &x = a.tables[r], &y = b.tables[r];
    if (x.cards != y.cards || x.mult != y.mult || x.mult64 != y.mult64 || x.hashed != y.hashed || x.groups != y.groups ||
        x.stride != y.stride || x.need_count != y.need_count || x.need_seen != y.need_seen || x.exists_min != y.exists_min ||
        x.exists_max != y.exists_max || x.carrier.agg != y.carrier.agg || x.carrier.shift != y.carrier.shift ||
        x.carrier.vmin != y.carrier.vmin || x.reduce_world != y.reduce_world || x.flag_slot != y.flag_slot ||
        x.tail_slots != y.tail_slots || x.i64_elems != y.i64_elems || x.f64_elems != y.f64_elems ||
        x.u32max_elems != y.u32max_elems || x.u32min_elems != y.u32min_elems || memcmp(x.index, y.index, sizeof x.index) ||
        memcmp(x.dwords, y.dwords, sizeof x.dwords) || memcmp(x.hist_per_group, y.hist_per_group, sizeof x.hist_per_group))
      return false;
  }
  return true;
}
}  // namespace

extern "C" {

// Plans the query twice: with the knobs as given, and with the same knobs plus spec = 0.  out = {status, spec flag of the
// first plan, spec flag of the second, 1 when the two plans agree in every other field, warps, CTAs per SM}.
int32_t probe_spec_route(int32_t sm_count, int32_t max_smem_optin, const char* const* knob_names, const int64_t* knob_values,
                         int32_t nknobs, const pb200_query* query, const probe_col* cols, int32_t ncols, const int32_t* num_docs,
                         int32_t nseg, int32_t allow_count_carrier, int64_t* out) {
  using namespace pb200;
  pb200_ctx ctx;
  for (int i = 0; i < nknobs; i++) if (int rc = pb200_tuning_set(&ctx, knob_names[i], knob_values[i])) return rc;
  static uint32_t sentinel[4];
  std::vector<pb200_segment> segs(nseg);
  std::vector<pb200_segment*> ptrs(nseg);
  for (int s = 0; s < nseg; s++) {
    segs[s].num_docs = num_docs[s];
    segs[s].cols.resize(ncols);
    for (int k = 0; k < ncols; k++) {
      const probe_col& p = cols[(size_t)s * ncols + k];
      DeviceColumn& c = segs[s].cols[k];
      c.fwd_kind = p.fwd_kind; c.stored_type = p.stored_type; c.bits = p.bits; c.cardinality = p.cardinality;
      c.fwd = sentinel;
      c.dict_native = p.dict_native ? sentinel : nullptr;
      c.dict_shared = p.dict_shared != 0;
      c.dict_hash = p.dict_hash;
      if (p.dict_host) c.dict_host.assign((const unsigned char*)p.dict_host, (const unsigned char*)p.dict_host + p.dict_host_bytes);
      if (p.has_inv) {
        c.inv = (unsigned char*)sentinel;
        for (int id = 0; id <= c.cardinality; id++) c.inv_offsets.push_back(4u * (c.cardinality + 1) + 8u * id);
      }
    }
    ptrs[s] = &segs[s];
  }
  const DeviceLimits lim{sm_count, max_smem_optin};
  ScanPlan a, b;
  memset(out, 0, 6 * sizeof(int64_t));
  const int rc = plan_scan(ctx.tune, lim, query, ptrs.data(), nseg, allow_count_carrier != 0, &a);
  out[0] = rc;
  if (rc) return rc;
  Tuning off = ctx.tune;
  off.spec = 0;
  if (plan_scan(off, lim, query, ptrs.data(), nseg, allow_count_carrier != 0, &b) != PB200_OK) return PB200_E_INVALID;
  out[1] = a.variant.spec;
  out[2] = b.variant.spec;
  out[3] = same_plan(a, b);
  out[4] = a.variant.warps;
  out[5] = a.variant.min_blocks;
  return PB200_OK;
}

}  // extern "C"
