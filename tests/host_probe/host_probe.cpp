// host_probe.cpp -- TEST shim: calls the product's host-side logic (inside libpinot_b200.so) without a GPU, so that the
// CPU test suite can compare it with the oracle:
//   * pb200h::StarTree::parse / traverse   (StarTreeFilterOperator's traversal as the product runs it)
//   * pb200h::matching_dict_ids             (PredicateEvaluator resolution: value-space predicate -> dictIds)
//   * pb200::plan_scan                       (every decision about a scan launch, on segments built from metadata)
//   * probe_plan_sharing                     (which aggregation's state each aggregation reads, and the count carriers)
//   * probe_plan_dump                        (every field of a scan, selection or DISTINCT plan as text: plan_diff.py)
// Built by tests/test_host_logic_cpu.py with g++ against the in-tree library; nothing here ships.
#include <algorithm>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../pinot_b200/csrc/host/host_internal.h"
#include "../../pinot_b200/csrc/pb200_plan.h"

extern "C" {

// preds: npreds entries (dimension, count, ids...) flattened as dims[i], offsets[i]..offsets[i+1] into ids[].
// Returns the number of [start, end) ranges written (pairs), -1 when a predicate matches nothing, -2 malformed tree.
int64_t probe_startree_traverse(const unsigned char* tree, uint64_t len, int32_t num_dims, int32_t npreds, const int32_t* dims,
                                const int32_t* offsets, const int32_t* ids, uint32_t group_by_mask, int32_t* out_pairs,
                                int64_t cap_pairs, uint32_t* remaining) {
  pb200h::StarTree t;
  if (!t.parse(tree, len) || (int)t.dim_names.size() != num_dims) return -2;
  std::vector<std::vector<int32_t>> store(num_dims);
  std::vector<const std::vector<int32_t>*> preds(num_dims, nullptr);
  for (int i = 0; i < npreds; i++) {
    if (dims[i] < 0 || dims[i] >= num_dims) return -2;
    store[dims[i]].assign(ids + offsets[i], ids + offsets[i + 1]);
    preds[dims[i]] = &store[dims[i]];
  }
  std::vector<std::pair<int32_t, int32_t>> docs;
  uint32_t rem = 0;
  if (!t.traverse(preds, group_by_mask, docs, rem)) return -1;
  if (remaining) *remaining = rem;
  int64_t n = 0;
  for (auto& r : docs) {
    if (n < cap_pairs) { out_pairs[2 * n] = r.first; out_pairs[2 * n + 1] = r.second; }
    n++;
  }
  return n;
}

// One predicate against one dictionary column described like pb200h_segment_create's input.
int64_t probe_matching_dict_ids(const pb200h_column* col, const pb200h_filter_node* node, const pb200h_literal* literals,
                                int32_t* out, int64_t cap) {
  pb200h::HostColumn h;
  h.name = col->name ? col->name : "";
  h.data_type = col->data_type; h.has_dictionary = col->has_dictionary; h.bits = col->bits_per_value;
  h.cardinality = col->cardinality; h.is_sorted = col->is_sorted; h.entry_bytes = col->dict_entry_bytes;
  if (col->dict && col->dict_bytes) h.dict.assign((const unsigned char*)col->dict, (const unsigned char*)col->dict + col->dict_bytes);
  std::vector<int32_t> ids = pb200h::matching_dict_ids(h, *node, literals);
  for (size_t i = 0; i < ids.size() && (int64_t)i < cap; i++) out[i] = ids[i];
  return (int64_t)ids.size();
}

// FilterOperatorUtils.getLeafFilterOperator as the product runs it: one predicate on one column of a (host-only) segment ->
// the device leaf.  out4 = {op, column, lo, hi}; ids (<= cap) receives the node's id / doc-range payload; returns num_ids
// or a negative pb200 status.
int64_t probe_leaf_to_device(const pb200h_column* col, int32_t num_docs, const pb200h_filter_node* node,
                             const pb200h_literal* literals, int32_t* out4, int32_t* ids, int64_t cap) {
  pb200h_segment seg;
  seg.num_docs = num_docs;
  pb200h::HostColumn h;
  h.name = col->name ? col->name : "";
  h.data_type = col->data_type; h.has_dictionary = col->has_dictionary; h.bits = col->bits_per_value;
  h.cardinality = col->cardinality; h.is_sorted = col->is_sorted; h.entry_bytes = col->dict_entry_bytes;
  h.has_inverted = col->inv != nullptr && col->inv_bytes > 0 && !col->is_sorted;
  if (col->dict && col->dict_bytes) h.dict.assign((const unsigned char*)col->dict, (const unsigned char*)col->dict + col->dict_bytes);
  if (col->is_sorted && col->fwd) h.sorted_idx.assign((const unsigned char*)col->fwd, (const unsigned char*)col->fwd + col->fwd_bytes);
  seg.cols.push_back(std::move(h));
  pb200h::SegmentFilterStore store;
  pb200_filter_node d;
  int rc = pb200h::leaf_to_device(seg, 0, *node, literals, store, d);
  if (rc) return rc;
  out4[0] = d.op; out4[1] = d.column; out4[2] = d.lo; out4[3] = d.hi;
  for (int i = 0; i < d.num_ids && i < cap; i++) ids[i] = d.ids[i];
  return d.num_ids;
}

// pb200h_explain over a HOST-ONLY segment (no device registration): the filter tree after predicate resolution and
// constant folding (FilterPlanNode / AndFilterOperator / OrFilterOperator always-true / always-false rules) plus the
// operator the plan maker would choose.  Returns the text length or a negative status.
int32_t probe_explain(const pb200h_column* cols, int32_t ncols, int32_t num_docs, const pb200h_query* q, char* out, int32_t cap) {
  pb200h_segment seg;
  seg.num_docs = num_docs;
  for (int i = 0; i < ncols; i++) {
    const pb200h_column& c = cols[i];
    pb200h::HostColumn h;
    h.name = c.name ? c.name : "";
    h.data_type = c.data_type; h.has_dictionary = c.has_dictionary; h.bits = c.bits_per_value;
    h.cardinality = c.cardinality; h.is_sorted = c.is_sorted; h.entry_bytes = c.dict_entry_bytes;
    h.has_inverted = c.inv != nullptr && c.inv_bytes > 0 && !c.is_sorted;
    if (c.dict && c.dict_bytes) h.dict.assign((const unsigned char*)c.dict, (const unsigned char*)c.dict + c.dict_bytes);
    if (c.is_sorted && c.fwd) h.sorted_idx.assign((const unsigned char*)c.fwd, (const unsigned char*)c.fwd + c.fwd_bytes);
    seg.cols.push_back(std::move(h));
  }
  return pb200h_explain(nullptr, q, &seg, out, cap);
}

// raw_forward.cpp: every chunk of a fixed-width raw SV forward index decoded into big-endian values (out: num_docs * width B)
int32_t probe_decode_fixed_byte_forward(const unsigned char* file, uint64_t len, int32_t width, int64_t num_docs, unsigned char* out) {
  std::vector<unsigned char> v;
  int rc = pb200h::decode_fixed_byte_forward(file, len, width, num_docs, v);
  if (rc) return rc;
  memcpy(out, v.data(), v.size());
  return 0;
}

// raw_forward.cpp: dictionary synthesised from raw values.  Returns 1 (built), 0 (more than max_cardinality distinct values).
int32_t probe_synthesize_dictionary(const unsigned char* values_be, int32_t data_type, int64_t num_docs, int32_t max_cardinality,
                                    unsigned char* dict_out, int64_t dict_cap, unsigned char* fwd_out, int64_t fwd_cap,
                                    int32_t* cardinality, int32_t* bits) {
  const int w = pb200h::raw_value_width(data_type);
  std::vector<unsigned char> values(values_be, values_be + (size_t)num_docs * w), dict, fwd;
  int card = 0, nb = 0;
  if (!pb200h::synthesize_dictionary(values, data_type, num_docs, max_cardinality, dict, fwd, &card, &nb)) return 0;
  if ((int64_t)dict.size() > dict_cap || (int64_t)fwd.size() > fwd_cap) return -1;
  memcpy(dict_out, dict.data(), dict.size());
  memcpy(fwd_out, fwd.data(), fwd.size());
  *cardinality = card; *bits = nb;
  return 1;
}

// ---- pb200::plan_scan over segments made of column metadata alone (no device memory: resident pointers are sentinels) ----
typedef struct {
  int32_t fwd_kind, stored_type, bits, cardinality;
  int32_t dict_native;        // 1: the column has a device dictionary (a sentinel pointer, never dereferenced)
  int32_t dict_shared;        // dictionary of a bound domain
  int32_t has_inv;            // an inverted index whose every dictId has a non-empty posting list
  int32_t eligible;           // VAR / STDDEV limb dictionaries: -1 not prepared, 0 off the grid, 1 built (fake limbs)
  uint64_t dict_hash;
  const void* dict_host;      // native little-endian dictionary values (INT: 4 bytes each), or NULL
  uint64_t dict_host_bytes;
} probe_col;

enum { PP_RES = 40, PP_SEG = 40, PP_CHUNK = 4 };
typedef struct {  // every field int64: tests/test_scan_plan_cpu.py mirrors this list
  int64_t warps, ctas_per_sm, stages, stage_words, tile_rows, smem_bytes, queue_off, smem_table_off, queue_max;
  int64_t sparse_max, sparse_max_agg, defer_agg, conj, num_slots, num_leaves, num_nodes, use_pipe;
  int64_t smem_groups, smem_copies, smem_gstride, smem_count, smem_merged, smem_slot[pb200::kMaxAggs];
  int64_t variant[4];  // warps, group_by, defer, min_blocks
  int64_t num_chunks, chunk_first_seg[PP_CHUNK], chunk_num_segs[PP_CHUNK], chunk_total_tiles[PP_CHUNK], chunk_grid[PP_CHUNK];
  int64_t nres, projected, num_leaf_buffers, in_filter[PP_RES];
  int64_t hashed[PP_RES], groups[PP_RES], stride[PP_RES], carrier_agg[PP_RES], carrier_shift[PP_RES], carrier_vmin[PP_RES];
  int64_t need_count[PP_RES], need_seen[PP_RES], exists_min[PP_RES], exists_max[PP_RES], reduce_world[PP_RES];
  int64_t flag_slot[PP_RES], tail_slots[PP_RES], i64_elems[PP_RES], f64_elems[PP_RES], u32max_elems[PP_RES], u32min_elems[PP_RES];
  int64_t dwords[PP_RES * pb200::kMaxAggs], distinct_words[PP_RES * pb200::kMaxAggs];
  int64_t seg_first_tile[PP_SEG], seg_num_tiles[PP_SEG], seg_stage_tx[PP_SEG], seg_num_agg_codes[PP_SEG], seg_num_defer_codes[PP_SEG];
  int64_t seg_agg_code[PP_SEG * pb200::kMaxAggs];
  int64_t seg_leaf_kind[PP_SEG * pb200::kMaxLeaves], seg_leaf_cmp[PP_SEG * pb200::kMaxLeaves], seg_leaf_negate[PP_SEG * pb200::kMaxLeaves];
  int64_t seg_leaf_lo[PP_SEG * pb200::kMaxLeaves], seg_leaf_span[PP_SEG * pb200::kMaxLeaves], seg_leaf_slot[PP_SEG * pb200::kMaxLeaves];
} probe_plan;

int64_t probe_plan_size(void) { return (int64_t)sizeof(probe_plan); }

}  // extern "C"

namespace {

// Limb dictionaries are never read on the host: column k of segment s gets the fake device range
// [kLimbBase + (s ncols + k) kLimbStride, + 3 x 2^31 u32)
constexpr uintptr_t kLimbBase = (uintptr_t)1 << 44, kLimbStride = (uintptr_t)1 << 36;

// Segments made of column metadata (cols: nseg x ncols).  Resident pointers are never dereferenced: the forward index,
// device dictionary and inverted index of column k in segment s are words 3 (s ncols + k) + 0 / 1 / 2 of `sentinels`.
struct ProbeSegments {
  std::vector<uint32_t> sentinels;
  std::vector<pb200_segment> segs;
  std::vector<pb200_segment*> ptrs;
  ProbeSegments(const probe_col* cols, int ncols, const int32_t* num_docs, int nseg)
      : sentinels((size_t)3 * nseg * ncols), segs(nseg), ptrs(nseg) {
    using namespace pb200;
    for (int s = 0; s < nseg; s++) {
      segs[s].num_docs = num_docs[s];
      segs[s].cols.resize(ncols);
      for (int k = 0; k < ncols; k++) {
        const probe_col& p = cols[(size_t)s * ncols + k];
        DeviceColumn& c = segs[s].cols[k];
        uint32_t* sent = &sentinels[3 * ((size_t)s * ncols + k)];
        c.fwd_kind = p.fwd_kind; c.stored_type = p.stored_type; c.bits = p.bits; c.cardinality = p.cardinality;
        c.fwd = sent;
        c.dict_native = p.dict_native ? sent + 1 : nullptr;
        c.dict_shared = p.dict_shared != 0;
        c.dict_hash = p.dict_hash;
        if (p.dict_host) c.dict_host.assign((const unsigned char*)p.dict_host, (const unsigned char*)p.dict_host + p.dict_host_bytes);
        if (p.has_inv) {
          c.inv = (unsigned char*)(sent + 2);
          for (int id = 0; id <= c.cardinality; id++) c.inv_offsets.push_back(4u * (c.cardinality + 1) + 8u * id);
        }
        if (p.eligible >= 0) {
          c.moments->eligible = p.eligible != 0;
          if (p.eligible) {
            c.moments->limbs = reinterpret_cast<uint32_t*>(kLimbBase + ((size_t)s * ncols + k) * kLimbStride);
            c.moments->entries = p.cardinality;
          }
          c.moments->ready.store(true);
        }
      }
      ptrs[s] = &segs[s];
    }
  }
  ~ProbeSegments() { for (auto& s : segs) for (auto& c : s.cols) c.moments->limbs = nullptr; }  // fake: never freed
};

}  // namespace

extern "C" {

// cols: nseg x ncols; knobs: nknobs pb200_tuning_set (name, value) pairs.  Returns plan_scan's status.
int32_t probe_plan_scan(int32_t sm_count, int32_t max_smem_optin, const char* const* knob_names, const int64_t* knob_values,
                        int32_t nknobs, const pb200_query* query, const probe_col* cols, int32_t ncols, const int32_t* num_docs,
                        int32_t nseg, int32_t allow_count_carrier, probe_plan* out) {
  using namespace pb200;
  pb200_ctx ctx;
  for (int i = 0; i < nknobs; i++) if (int rc = pb200_tuning_set(&ctx, knob_names[i], knob_values[i])) return rc;
  ProbeSegments ps(cols, ncols, num_docs, nseg);
  ScanPlan plan;
  const int rc = plan_scan(ctx.tune, DeviceLimits{sm_count, max_smem_optin}, query, ps.ptrs.data(), nseg, allow_count_carrier != 0, &plan);
  memset(out, 0, sizeof *out);
  if (rc) return rc;
  const QueryDesc& q = plan.q;
  probe_plan& o = *out;
  o.warps = plan.warps; o.ctas_per_sm = plan.ctas_per_sm; o.stages = q.num_stages; o.stage_words = q.stage_words;
  o.tile_rows = q.tile_rows; o.smem_bytes = (int64_t)plan.smem_bytes; o.queue_off = q.queue_off; o.smem_table_off = q.smem_table_off;
  o.queue_max = q.queue_max; o.sparse_max = q.sparse_max; o.sparse_max_agg = q.sparse_max_agg; o.defer_agg = q.defer_agg;
  o.conj = q.conj; o.num_slots = q.num_slots; o.num_leaves = q.num_leaves; o.num_nodes = q.num_nodes; o.use_pipe = q.use_pipe;
  o.smem_groups = q.smem_groups; o.smem_copies = q.smem_copies; o.smem_gstride = q.smem_gstride; o.smem_count = q.smem_count;
  o.smem_merged = q.smem_merged;
  for (int a = 0; a < kMaxAggs; a++) o.smem_slot[a] = q.smem_slot[a];
  o.variant[0] = plan.variant.warps; o.variant[1] = plan.variant.group_by; o.variant[2] = plan.variant.defer; o.variant[3] = plan.variant.min_blocks;
  o.num_chunks = (int64_t)plan.chunks.size();
  for (size_t c = 0; c < plan.chunks.size() && c < PP_CHUNK; c++) {
    o.chunk_first_seg[c] = plan.chunks[c].first_seg; o.chunk_num_segs[c] = plan.chunks[c].num_segs;
    o.chunk_total_tiles[c] = plan.chunks[c].total_tiles; o.chunk_grid[c] = plan.chunks[c].grid;
  }
  o.nres = plan.nres; o.projected = plan.projected; o.num_leaf_buffers = (int64_t)plan.leaf_buffers.size();
  for (int r = 0; r < plan.nres && r < PP_RES; r++) {
    o.in_filter[r] = plan.in_filter[r];
    for (int a = 0; a < kMaxAggs && !plan.distinct_words.empty() && a < (int)plan.distinct_words[r].size(); a++)
      o.distinct_words[r * kMaxAggs + a] = (int64_t)plan.distinct_words[r][a];
    if (plan.tables.empty()) continue;
    const TableLayout& t = plan.tables[r];
    o.hashed[r] = t.hashed; o.groups[r] = t.groups; o.stride[r] = t.stride; o.carrier_agg[r] = t.carrier.agg;
    o.carrier_shift[r] = t.carrier.shift; o.carrier_vmin[r] = t.carrier.vmin; o.need_count[r] = t.need_count;
    o.need_seen[r] = t.need_seen; o.exists_min[r] = t.exists_min; o.exists_max[r] = t.exists_max; o.reduce_world[r] = t.reduce_world;
    o.flag_slot[r] = t.flag_slot; o.tail_slots[r] = t.tail_slots; o.i64_elems[r] = t.i64_elems; o.f64_elems[r] = t.f64_elems;
    o.u32max_elems[r] = t.u32max_elems; o.u32min_elems[r] = t.u32min_elems;
    for (int a = 0; a < kMaxAggs; a++) o.dwords[r * kMaxAggs + a] = t.dwords[a];
  }
  for (int s = 0; s < nseg && s < PP_SEG; s++) {
    const SegDesc& sd = plan.segs[s];
    o.seg_first_tile[s] = sd.first_tile; o.seg_num_tiles[s] = sd.num_tiles; o.seg_stage_tx[s] = sd.stage_tx;
    o.seg_num_agg_codes[s] = sd.num_agg_codes; o.seg_num_defer_codes[s] = sd.num_defer_codes;
    for (int a = 0; a < kMaxAggs; a++) o.seg_agg_code[s * kMaxAggs + a] = sd.agg_code[a];
    for (int l = 0; l < kMaxLeaves; l++) {
      const LeafDesc& lf = sd.leaves[l];
      o.seg_leaf_kind[s * kMaxLeaves + l] = lf.kind; o.seg_leaf_cmp[s * kMaxLeaves + l] = lf.cmp;
      o.seg_leaf_negate[s * kMaxLeaves + l] = lf.negate; o.seg_leaf_lo[s * kMaxLeaves + l] = lf.lo;
      o.seg_leaf_span[s * kMaxLeaves + l] = lf.span; o.seg_leaf_slot[s * kMaxLeaves + l] = lf.slot;
    }
  }
  return PB200_OK;
}

// Which aggregation's state each aggregation of a plan reads, and the count carrier of each result
// (tests/test_mixed_aggs_cpu.py).  Per-aggregation arrays are -1 past their length: mom_first has num_user_aggs entries,
// the others num_aggs (the caller's aggregations, then the internal moment sums).
typedef struct {
  int64_t num_user_aggs, num_aggs, nres;
  int64_t function[pb200::kMaxAggs], column[pb200::kMaxAggs];
  int64_t ds_rep[pb200::kMaxAggs], hll_log2m[pb200::kMaxAggs], hll_rep[pb200::kMaxAggs], pct_rep[pb200::kMaxAggs];
  int64_t mom_first[pb200::kMaxAggs], limb[pb200::kMaxAggs];
  int64_t carrier_agg[PP_RES];
} probe_sharing;

int64_t probe_sharing_size(void) { return (int64_t)sizeof(probe_sharing); }

// plan_scan as probe_plan_scan runs it, with the per-aggregation arguments (agg_args: PERCENTILE's p and
// DISTINCTCOUNTHLL's log2m; wt_args: the time columns of FIRST/LASTWITHTIME; either may be NULL).  Returns its status.
int32_t probe_plan_sharing(int32_t sm_count, int32_t max_smem_optin, const char* const* knob_names, const int64_t* knob_values,
                           int32_t nknobs, const pb200_query* query, const double* agg_args, const pb200_agg_arg* wt_args,
                           const probe_col* cols, int32_t ncols, const int32_t* num_docs, int32_t nseg,
                           int32_t allow_count_carrier, probe_sharing* out) {
  using namespace pb200;
  pb200_ctx ctx;
  for (int i = 0; i < nknobs; i++) if (int rc = pb200_tuning_set(&ctx, knob_names[i], knob_values[i])) return rc;
  ProbeSegments ps(cols, ncols, num_docs, nseg);
  ScanPlan plan;
  const int rc = plan_scan(ctx.tune, DeviceLimits{sm_count, max_smem_optin}, query, ps.ptrs.data(), nseg, allow_count_carrier != 0,
                           &plan, agg_args, wt_args);
  probe_sharing& o = *out;
  memset(&o, 0, sizeof o);
  for (int a = 0; a < kMaxAggs; a++) {
    o.function[a] = o.column[a] = o.ds_rep[a] = o.hll_rep[a] = o.pct_rep[a] = o.mom_first[a] = o.limb[a] = -1;
    o.hll_log2m[a] = 0;
  }
  for (int r = 0; r < PP_RES; r++) o.carrier_agg[r] = -1;
  if (rc) return rc;
  o.num_user_aggs = plan.num_user_aggs; o.num_aggs = (int64_t)plan.aggs.size(); o.nres = plan.nres;
  for (int a = 0; a < (int)plan.aggs.size() && a < kMaxAggs; a++) {
    o.function[a] = plan.aggs[a].function; o.column[a] = plan.aggs[a].column;
    o.ds_rep[a] = plan.ds_rep[a]; o.hll_log2m[a] = plan.hll_log2m[a]; o.hll_rep[a] = plan.hll_rep[a];
    o.pct_rep[a] = plan.pct_rep[a]; o.limb[a] = plan.limb[a];
  }
  for (int a = 0; a < plan.num_user_aggs && a < kMaxAggs; a++) o.mom_first[a] = plan.mom_first[a];
  for (int r = 0; r < (int)plan.tables.size() && r < PP_RES; r++) o.carrier_agg[r] = plan.tables[r].carrier.agg;
  return PB200_OK;
}

}  // extern "C"

namespace {

// Text form of a plan.  A pointer is written as (range, byte offset): range 1 is the sentinels, 2 the fake limb
// dictionaries, 3 + i the ids of filter node i of the query; so dumps taken by two processes compare byte for byte.
struct PlanDump {
  const ProbeSegments& ps;
  const pb200_query* query;
  int nnodes_total;
  std::string out;

  uint64_t token(const void* p) const {
    const uintptr_t a = (uintptr_t)p;
    if (!p) return 0;
    const uintptr_t s0 = (uintptr_t)ps.sentinels.data();
    if (a >= s0 && a < s0 + ps.sentinels.size() * 4) return 1ull << 48 | (a - s0);
    if (a >= kLimbBase && a < kLimbBase + ps.ptrs.size() * ps.segs[0].cols.size() * kLimbStride) return 2ull << 48 | (a - kLimbBase);
    for (int i = 0; i < nnodes_total; i++) {
      const pb200_filter_node& n = query->filter[i];
      const uintptr_t b = (uintptr_t)n.ids;
      if (n.ids && a >= b && a < b + (size_t)std::max(n.num_ids, 1) * 4) return (3ull + i) << 48 | (a - b);
    }
    return ~0ull;   // a pointer the plan should not hold
  }
  void line(const char* fmt, ...) __attribute__((format(printf, 2, 3))) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    out += buf;
    out += '\n';
  }
  void bytes(const char* name, const void* p, size_t n) {
    static const char* hex = "0123456789abcdef";
    out += name;
    out += ' ';
    for (size_t i = 0; i < n; i++) { const unsigned char b = ((const unsigned char*)p)[i]; out += hex[b >> 4]; out += hex[b & 15]; }
    out += '\n';
  }
  template <class T> void vec(const char* name, const std::vector<T>& v) {
    out += name;
    for (const T& x : v) { out += ' '; out += std::to_string(x); }
    out += '\n';
  }
  void vec(const char* name, const std::vector<double>& v) {
    out += name;
    for (double x : v) { uint64_t u; memcpy(&u, &x, 8); out += ' '; out += std::to_string(u); }
    out += '\n';
  }
  void vec(const char* name, const std::vector<bool>& v) { vec(name, std::vector<int>(v.begin(), v.end())); }

  void scan(const pb200::ScanPlan& p) {
    using namespace pb200;
    bytes("q", &p.q, sizeof p.q);   // QueryDesc: integers only, no padding
    for (size_t s = 0; s < p.segs.size(); s++) {
      SegDesc d;                    // memset by the planner: padding included, every byte is defined
      memcpy(&d, &p.segs[s], sizeof d);
      for (auto& sl : d.slots) sl.data = (const uint32_t*)token(sl.data);
      for (auto& lf : d.leaves) { lf.bits = (const uint32_t*)token(lf.bits); lf.ranges = (const int32_t*)token(lf.ranges); }
      for (int a = 0; a < kMaxAggs; a++) {
        d.dict[a] = (const void*)token(d.dict[a]); d.distinct_bits[a] = (uint32_t*)token(d.distinct_bits[a]);
        d.g_isum[a] = (long long*)token(d.g_isum[a]); d.g_dsum[a] = (double*)token(d.g_dsum[a]);
        d.g_min[a] = (uint32_t*)token(d.g_min[a]); d.g_max[a] = (uint32_t*)token(d.g_max[a]);
      }
      d.accum = (AggAccum*)token(d.accum); d.g_count = (unsigned long long*)token(d.g_count); d.g_seen = (uint32_t*)token(d.g_seen);
      d.h_keys = (unsigned long long*)token(d.h_keys); d.h_ctl = (uint32_t*)token(d.h_ctl);
      line("seg %zu", s);
      bytes("segdesc", &d, sizeof d);
    }
    vec("slot_cols", p.slot_cols);
    vec("leaf_node", p.leaf_node);
    line("flags %d %d %d nres %d warps %d ctas %d skip %d smem %zu", p.group_by, p.merge, p.defer_finalize, p.nres, p.warps,
         p.ctas_per_sm, p.skip_masks, p.smem_bytes);
    line("variant %d %d %d %d %d", p.variant.warps, p.variant.group_by, p.variant.defer, p.variant.min_blocks, p.variant.spec);
    for (const LaunchChunk& c : p.chunks) line("chunk %d %d %d %d", c.first_seg, c.num_segs, c.total_tiles, c.grid);
    for (const LeafBuffer& b : p.leaf_buffers) {
      uint64_t h = 1469598103934665603ull;   // FNV-1a over the LUT words
      for (uint32_t w : b.lut) { h ^= w; h *= 1099511628211ull; }
      line("leafbuf %d %d %d %zu lut %zu %llx src %llx %zu jobs %zu", (int)b.kind, b.seg, b.leaf, b.words, b.lut.size(),
           (unsigned long long)h, (unsigned long long)token(b.src), b.src_words, b.jobs.size());
      for (const DecodeJob& j : b.jobs)
        line("job %llx %llu %llu %llx %lld", (unsigned long long)token(j.inv), j.offset, j.length, (unsigned long long)token(j.mask), j.num_docs);
    }
    for (const TableLayout& t : p.tables) {
      vec("cards", t.cards); vec("mult", t.mult); vec("mult64", t.mult64);
      line("table %d %lld %d %d %d %d %d carrier %d %d %lld rw %d flag %d tail %d elems %lld %lld %lld %lld", t.hashed, t.groups,
           t.stride, t.need_count, t.need_seen, t.exists_min, t.exists_max, t.carrier.agg, t.carrier.shift, t.carrier.vmin,
           t.reduce_world, t.flag_slot, t.tail_slots, t.i64_elems, t.f64_elems, t.u32max_elems, t.u32min_elems);
      vec("index", std::vector<int>(t.index, t.index + kMaxAggs));
      vec("dwords", std::vector<uint32_t>(t.dwords, t.dwords + kMaxAggs));
      vec("hist_per_group", std::vector<uint32_t>(t.hist_per_group, t.hist_per_group + kMaxAggs));
    }
    for (const auto& v : p.distinct_words) vec("distinct_words", v);
    vec("pct_p", p.pct_p);
    vec("pct_rep", p.pct_rep);
    line("num_user_aggs %d", p.num_user_aggs);
    for (const pb200_agg& a : p.aggs) line("agg %d %d", a.function, a.column);
    vec("mom_first", p.mom_first);
    vec("limb", p.limb);
    for (const auto& v : p.hist_entries) vec("hist_entries", v);
    line("hist_total %lld", p.hist_total);
    vec("in_filter", p.in_filter);
    line("projected %d", p.projected);
  }
  void selection(const pb200::SelectionPlan& p) {
    scan(p.scan);
    vec("columns", p.columns); vec("kinds", p.kinds); vec("order_cols", p.order_cols); vec("order_kinds", p.order_kinds);
    vec("order_desc", p.order_desc);
    line("limit %lld mask_words %lld prefix %d", p.limit, p.mask_words, p.prefix);
    vec("mask_word_off", p.mask_word_off); vec("chunk_word_off", p.chunk_word_off); vec("scan_docs", p.scan_docs);
  }
  void distinct(const pb200::DistinctPlan& p) {
    selection(p.sel);
    line("nres %d table_entries %lld", p.nres, p.table_entries);
    for (const auto& v : p.cards) vec("cards", v);
    for (const auto& v : p.mult) vec("mult", v);
    vec("table_off", p.table_off); vec("table_size", p.table_size); vec("order_key", p.order_key); vec("order_desc", p.order_desc);
  }
};

}  // namespace

extern "C" {

// The whole plan of one input as text into out (cap bytes); returns its length (not truncated when < cap), or a
// negative pb200_tuning_set status.  kind 0: plan_scan (agg_args as for pb200_execute_args, may be NULL), 1:
// plan_selection, 2: plan_distinct (sel: the selection / DISTINCT columns).  A refusal dumps its status and message.
int64_t probe_plan_dump(int32_t kind, int32_t sm_count, int32_t max_smem_optin, const char* const* knob_names,
                        const int64_t* knob_values, int32_t nknobs, const pb200_query* query, const double* agg_args,
                        const pb200_selection* sel, const probe_col* cols, int32_t ncols, const int32_t* num_docs, int32_t nseg,
                        int32_t allow_count_carrier, int32_t merge, int32_t prefix, char* out, int64_t cap) {
  using namespace pb200;
  pb200_ctx ctx;
  for (int i = 0; i < nknobs; i++) if (int rc = pb200_tuning_set(&ctx, knob_names[i], knob_values[i])) return rc;
  ProbeSegments ps(cols, ncols, num_docs, nseg);
  const DeviceLimits lim{sm_count, max_smem_optin};
  const int nnodes_total = query->num_filter_nodes * ((query->flags & PB200_Q_PER_SEGMENT_FILTER) ? nseg : 1);
  PlanDump d{ps, query, nnodes_total, {}};
  int rc;
  if (kind == 0) {
    ScanPlan p;
    rc = plan_scan(ctx.tune, lim, query, ps.ptrs.data(), nseg, allow_count_carrier != 0, &p, agg_args);
    if (!rc) d.scan(p);
  } else if (kind == 1) {
    SelectionPlan p;
    rc = plan_selection(ctx.tune, lim, query, sel, ps.ptrs.data(), nseg, prefix != 0, &p);
    if (!rc) d.selection(p);
  } else {
    DistinctPlan p;
    rc = plan_distinct(ctx.tune, lim, query, sel, ps.ptrs.data(), nseg, merge != 0, prefix != 0, &p);
    if (!rc) d.distinct(p);
  }
  if (rc) d.line("refused %d %s", rc, pb200_last_error());
  memcpy(out, d.out.data(), std::min<size_t>(d.out.size(), (size_t)cap));
  return (int64_t)d.out.size();
}

}  // extern "C"
