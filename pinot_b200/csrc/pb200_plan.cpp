// pb200_plan.cpp -- host-only planning of a scan launch (pb200_plan.h).  No CUDA runtime call in this file.
#include "pb200_plan.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>

namespace pb200 {
namespace {

int slot_of(ScanPlan& p, int col, uint32_t role) {
  for (size_t s = 0; s < p.slot_cols.size(); s++)
    if (p.slot_cols[s] == col) { p.q.slot_roles[s] |= role; return (int)s; }
  if ((int)p.slot_cols.size() >= kMaxSlots) { set_error("too many distinct columns (max %d)", kMaxSlots); return -1; }
  p.slot_cols.push_back(col);
  p.q.slot_roles[p.slot_cols.size() - 1] = role;
  return (int)p.slot_cols.size() - 1;
}

bool is_scan_leaf(int op) { return op == PB200_F_SCAN_RANGE || op == PB200_F_SCAN_IN || op == PB200_F_SCAN_NOT_IN || op == PB200_F_RAW_RANGE; }
bool is_leaf(int op) { return op >= PB200_F_MATCH_ALL; }

// one-sided ranges: every stored dictId is < cardinality, so "hi covers the dictionary" needs no upper compare
void set_cmp(LeafDesc& lf, const DeviceColumn& c) {
  const unsigned long long hi = (unsigned long long)lf.lo + lf.span;
  if (lf.span == 0) { lf.kind = LEAF_NONE; return; }
  if (hi >= (unsigned long long)c.cardinality || hi >= (1ull << c.bits)) lf.cmp = CMP_GE;
  else if (lf.lo == 0) lf.cmp = CMP_LT;
  else lf.cmp = CMP_BOTH;
}

constexpr size_t kHdrBytes = (sizeof(SmemHeader) + 127) / 128 * 128;   // the CTA's header, 128-byte aligned

// Dynamic shared memory a CTA has left for its TMA rings: the opt-in limit shared by `ctas` CTAs per SM, minus the
// header, `extra` bytes (generic-filter stacks, survivor queues or aggregation scratch, a shared-memory group table) and
// 1024 + 256 bytes of alignment slack.
long long ring_budget(const DeviceLimits& lim, int ctas, size_t extra) {
  return (long long)lim.max_smem_optin / ctas - (long long)kHdrBytes - (long long)extra - 1024 - 256;
}

int bits_of(unsigned long long x) { int b = 0; while (b < 64 && (x >> b)) b++; return b; }

}  // namespace

int regime_of(const std::vector<int>& cards, int array_threshold) {
  // DictionaryBasedGroupKeyGenerator.java:128-185
  long long product = 1;
  bool overflow = false;
  for (int c : cards) {
    if (!overflow) {
      if (c > 0 && product > std::numeric_limits<long long>::max() / c) overflow = true; else product *= c;
    }
  }
  if (overflow) return PB200_REGIME_ARRAY_MAP;
  if (product > std::numeric_limits<int>::max()) return PB200_REGIME_LONG_MAP;
  return product > array_threshold ? PB200_REGIME_INT_MAP : PB200_REGIME_ARRAY;
}

// One result for all segments == a merge of dictId-indexed state (group tables, MIN / MAX ids, DISTINCTCOUNT bitsets,
// DISTINCT tables).  That is only a merge BY VALUE (GroupByCombineOperator.java:130-146, AggregationFunction.merge) when
// the column has the same dictionary everywhere: compare content hashes, not cardinalities.  Bound segments
// (pb200_domain_*) pass by construction; anything else is refused so that the caller combines per-segment results itself.
bool same_dictionary(pb200_segment* const* segments, int nseg, int col, const char* what) {
  const DeviceColumn& c0 = segments[0]->cols[col];
  for (int s = 1; s < nseg; s++) {
    const DeviceColumn& c = segments[s]->cols[col];
    if (c.dict_hash != c0.dict_hash || c.cardinality != c0.cardinality || c.stored_type != c0.stored_type) {
      set_error("PB200_Q_MERGE_SEGMENTS: %s column %d has a different dictionary in segment %d than in segment 0 "
                "(bind the segments to a pb200_domain first)", what, col, s);
      return false;
    }
  }
  return true;
}

namespace {

// Numbers the tiles of chunk `ch`'s segments from 0 and sets its tile count and grid; returns its tiles.
long long lay_out_chunk(const Tuning& tune, DeviceLimits lim, ScanPlan& plan, LaunchChunk& ch) {
  long long cursor = 0;
  for (int s = ch.first_seg; s < ch.first_seg + ch.num_segs; s++) { plan.segs[s].first_tile = cursor; cursor += plan.segs[s].num_tiles; }
  ch.total_tiles = (int)cursor;
  ch.grid = tune.grid > 0 ? tune.grid : (int)std::min<long long>((long long)lim.sm_count * plan.ctas_per_sm, std::max<long long>(cursor, 1));
  return cursor;
}

// plan_scan's stages, in the order they run.  Each leaves its decisions in `plan`; the members below carry what a later
// stage needs and ScanPlan does not hold.  The caller's aggregations followed by the internal moment sums are plan.aggs.
struct ScanPlanner {
  const Tuning& tune;
  const DeviceLimits lim;
  const pb200_query* query;
  pb200_segment* const* segments;
  const int nseg, ncols;
  ScanPlan& plan;
  QueryDesc& q = plan.q;
  const bool per_seg_filter = query->flags & PB200_Q_PER_SEGMENT_FILTER, merge = query->flags & PB200_Q_MERGE_SEGMENTS;
  const int nnodes = query->num_filter_nodes, nuser = query->num_aggs, ngb = query->num_group_by;
  int reduce_world = 1;             // GPUs whose tables are summed with this launch's
  std::vector<Carrier> carrier;     // per result
  bool pipelined[kMaxAggs] = {};    // aggregations whose loads are software-pipelined
  int npipe = 0;

  const pb200_filter_node* filter_of(int s) const { return per_seg_filter ? query->filter + (size_t)s * nnodes : query->filter; }
  bool in_result(int s, int r) const { return merge || s == r; }
  unsigned long long result_docs(int r) const {
    unsigned long long docs = 0;
    for (int s = 0; s < nseg; s++) if (in_result(s, r)) docs += (unsigned long long)segments[s]->num_docs;
    return docs;
  }
  int result_max_bits(int r, int col) const {
    int maxbits = 0;
    for (int s = 0; s < nseg; s++) if (in_result(s, r)) maxbits = std::max(maxbits, segments[s]->cols[col].bits);
    return maxbits;
  }
  // PERCENTILE and VAR / STDDEV count or sum per dictId: segment t's column must have them
  int require_dict_ids(int t, int col, const char* what) const {
    const DeviceColumn& c = segments[t]->cols[col];
    if (c.stored_type == PB200_STRING) { set_error("%s over STRING column %d", what, col); return PB200_E_UNSUPPORTED; }
    if (c.bits <= 31 && c.dict_native && c.cardinality > 0) return PB200_OK;
    set_error("%s over column %d: no dictIds in segment %d (raw values): not accelerated", what, col, t);
    return PB200_E_UNSUPPORTED;
  }
  // ---- VAR / STDDEV: each column's moments are three internal INT-dictionary SUMs over its limb dictionaries
  //      (pb200_moments.h), appended behind the caller's aggregations; functions of one column share them ----
  int expand_moments() {
    plan.num_user_aggs = nuser;
    plan.aggs.assign(query->aggs, query->aggs + nuser);
    plan.mom_first.assign(nuser, -1);
    for (int a = 0; a < nuser; a++) {
      const pb200_agg& ag = query->aggs[a];
      if (!is_moments_fn(ag.function)) continue;
      if (ag.column < 0 || ag.column >= ncols) { set_error("aggregation column %d out of range", ag.column); return PB200_E_INVALID; }
      if (merge && (query->flags & PB200_Q_DEFER_FINALIZE)) { set_error("VAR/STDDEV moments are not reducible across GPUs (PB200_Q_DEFER_FINALIZE)"); return PB200_E_UNSUPPORTED; }
      for (int t = 0; t < nseg; t++) {
        if (int rc = require_dict_ids(t, ag.column, "VAR/STDDEV")) return rc;
        const MomentDict& md = *segments[t]->cols[ag.column].moments;
        if (!md.ready.load(std::memory_order_acquire)) { set_error("internal: limb dictionaries of column %d not prepared", ag.column); return PB200_E_INVALID; }
        if (!md.eligible) {
          set_error("VAR/STDDEV over column %d: its values in segment %d are not on a grid of 2^32 steps (c + k * 2^e): not accelerated", ag.column, t);
          return PB200_E_UNSUPPORTED;
        }
      }
      for (int b = 0; b < a && plan.mom_first[a] < 0; b++)
        if (plan.mom_first[b] >= 0 && query->aggs[b].column == ag.column) plan.mom_first[a] = plan.mom_first[b];
      if (plan.mom_first[a] >= 0) continue;
      plan.mom_first[a] = (int)plan.aggs.size();
      for (int j = 0; j < 3; j++) plan.aggs.push_back(pb200_agg{PB200_AGG_SUM, ag.column});
    }
    const int nagg = (int)plan.aggs.size();
    if (nagg > kMaxAggs) {
      set_error("VAR/STDDEV: %d aggregations with the internal moment sums (3 per column), at most %d", nagg, kMaxAggs);
      return PB200_E_UNSUPPORTED;
    }
    plan.limb.assign(nagg, -1);
    for (int a = 0; a < nuser; a++)
      if (plan.mom_first[a] >= 0) for (int j = 0; j < 3; j++) plan.limb[plan.mom_first[a] + j] = j;
    plan.group_by = ngb > 0; plan.merge = merge;
    plan.defer_finalize = merge && (query->flags & PB200_Q_DEFER_FINALIZE);
    plan.nres = merge ? 1 : nseg;
    q.num_segments = nseg; q.num_aggs = nagg; q.num_group_by = ngb;
    plan.pct_p.assign(nagg, std::numeric_limits<double>::quiet_NaN());
    plan.pct_rep.assign(nagg, -1);
    return PB200_OK;
  }
  // ---- slots: filter scan columns, then group-by keys, then aggregation arguments ----
  int assign_slots(const double* agg_args) {
    const pb200_filter_node* f0 = query->filter;
    for (int s = 0; s < (per_seg_filter ? nseg : 1); s++) {
      for (int i = 0; i < nnodes; i++) {
        const pb200_filter_node& n = filter_of(s)[i];
        if (is_leaf(n.op) != is_leaf(f0[i].op) || (!is_leaf(n.op) && (n.op != f0[i].op || n.num_children != f0[i].num_children))) {
          set_error("per-segment filter trees must share their shape"); return PB200_E_INVALID;
        }
        if (is_scan_leaf(n.op)) {
          if (n.column < 0 || n.column >= ncols) { set_error("filter column %d out of range", n.column); return PB200_E_INVALID; }
          if (slot_of(plan, n.column, ROLE_FILTER) < 0) return PB200_E_UNSUPPORTED;
        }
      }
    }
    for (int g = 0; g < ngb; g++) {
      int c = query->group_by_columns[g];
      if (c < 0 || c >= ncols) { set_error("group-by column %d out of range", c); return PB200_E_INVALID; }
      for (int t = 0; t < nseg; t++) {
        const DeviceColumn& gc = segments[t]->cols[c];
        if (gc.bits > 31 || gc.cardinality <= 0 || gc.fwd_kind != PB200_FWD_DICT_FIXEDBIT) {
          set_error("group-by column %d is not dictionary-encoded in segment %d: not accelerated", c, t);
          return PB200_E_UNSUPPORTED;
        }
      }
      if ((q.group_slot[g] = slot_of(plan, c, ROLE_GROUP)) < 0) return PB200_E_UNSUPPORTED;
    }
    for (int a = 0; a < q.num_aggs; a++) {
      const pb200_agg& ag = plan.aggs[a];
      q.aggs[a] = AggDesc{ag.function, -1, VAL_NONE, 0};
      if (ag.function == PB200_AGG_COUNT || is_moments_fn(ag.function)) continue;   // VAR / STDDEV: read their limb sums
      if (ag.function < 0 || ag.function > PB200_AGG_PERCENTILE) { set_error("unknown aggregation function %d", ag.function); return PB200_E_INVALID; }
      if (ag.column < 0 || ag.column >= ncols) { set_error("aggregation column %d out of range", ag.column); return PB200_E_INVALID; }
      if (ag.function == PB200_AGG_PERCENTILE) {
        // the percentile travels beside the query (pb200_execute_args); PercentileAggregationFunction takes 0 <= p <= 100
        if (!agg_args) {   // pb200_execute / pb200_execute_ordered carry no percentile
          set_error("unknown aggregation function %d without arguments: PERCENTILE (aggregation %d) takes its percentile through pb200_execute_args", ag.function, a);
          return PB200_E_INVALID;
        }
        const double pv = agg_args[a];
        if (!(pv >= 0.0 && pv <= 100.0)) { set_error("PERCENTILE (aggregation %d): percentile %g outside [0, 100]", a, pv); return PB200_E_INVALID; }
        if (plan.defer_finalize) { set_error("PERCENTILE histograms are not reducible across GPUs (PB200_Q_DEFER_FINALIZE)"); return PB200_E_UNSUPPORTED; }
        for (int t = 0; t < nseg; t++)
          if (int rc = require_dict_ids(t, ag.column, "PERCENTILE")) return rc;
        plan.pct_p[a] = pv;
        plan.pct_rep[a] = a;
        for (int b = 0; b < a; b++)   // PERCENTILEs of one column share the first one's histogram
          if (plan.aggs[b].function == PB200_AGG_PERCENTILE && plan.aggs[b].column == ag.column) { plan.pct_rep[a] = b; break; }
      }
      if ((q.aggs[a].slot = slot_of(plan, ag.column, ROLE_AGG)) < 0) return PB200_E_UNSUPPORTED;
      const DeviceColumn& c0 = segments[0]->cols[ag.column];
      int vk = VAL_NONE;
      if (c0.bits == 32 && c0.dict_native == nullptr) {
        if (c0.stored_type != PB200_INT) { set_error("raw column type %d not accelerated", c0.stored_type); return PB200_E_UNSUPPORTED; }
        vk = VAL_RAW_I32;
        if (ag.function == PB200_AGG_DISTINCTCOUNT) { set_error("DISTINCTCOUNT on raw column not accelerated"); return PB200_E_UNSUPPORTED; }
      } else {
        switch (c0.stored_type) {
          case PB200_INT: vk = VAL_DICT_I32; break;
          case PB200_LONG: vk = VAL_DICT_I64; break;
          case PB200_FLOAT: vk = VAL_DICT_F32; break;
          case PB200_DOUBLE: vk = VAL_DICT_F64; break;
          default:  // STRING: only functions that work on dictIds (MIN/MAX come back as dictIds, DISTINCTCOUNT as a set)
            if (ag.function == PB200_AGG_SUM || ag.function == PB200_AGG_AVG) { set_error("SUM/AVG over STRING column"); return PB200_E_UNSUPPORTED; }
            vk = VAL_DICT_I32;
        }
      }
      if (plan.limb[a] >= 0) vk = VAL_DICT_I32;   // limb words are read as biased INT dictionary values
      q.aggs[a].val_kind = vk;
    }
    q.num_slots = (int)plan.slot_cols.size();
    return PB200_OK;
  }
  // ---- filter program (shape shared by all segments) ----
  int compile_filter() {
    const pb200_filter_node* f0 = query->filter;
    int nleaves = 0;
    for (int i = 0; i < nnodes; i++) {
      const pb200_filter_node& n = f0[i];
      if (is_leaf(n.op)) {
        if (nleaves >= kMaxLeaves) { set_error("too many filter leaves (max %d)", kMaxLeaves); return PB200_E_UNSUPPORTED; }
        q.prog_op[i] = OP_LEAF;
        q.prog_arg[i] = (uint8_t)nleaves++;
        plan.leaf_node.push_back(i);
      } else if (n.op == PB200_F_NOT) {
        q.prog_op[i] = OP_NOT; q.prog_arg[i] = 1;
      } else if (n.op == PB200_F_AND || n.op == PB200_F_OR) {
        if (n.num_children < 1 || n.num_children > kMaxStack) { set_error("AND/OR with %d operands not supported", n.num_children); return PB200_E_UNSUPPORTED; }
        q.prog_op[i] = n.op == PB200_F_AND ? OP_AND : OP_OR;
        q.prog_arg[i] = (uint8_t)n.num_children;
      } else {
        set_error("unknown filter op %d", n.op);
        return PB200_E_INVALID;
      }
    }
    q.num_nodes = nnodes; q.num_leaves = nleaves;
    q.conj = nnodes == 0 || (nnodes == 1 && nleaves == 1) ||
             (nnodes == nleaves + 1 && f0[nnodes - 1].op == PB200_F_AND && f0[nnodes - 1].num_children == nleaves);
    // validate stack discipline once
    int sp = 0, maxsp = 0;
    for (int i = 0; i < nnodes; i++) {
      if (q.prog_op[i] == OP_LEAF) sp++;
      else if (q.prog_op[i] == OP_NOT) { if (sp < 1) sp = -99; }
      else { sp -= q.prog_arg[i] - 1; }
      if (sp < 1) { set_error("malformed postfix filter"); return PB200_E_INVALID; }
      maxsp = std::max(maxsp, sp);
    }
    if (nnodes > 0 && sp != 1) { set_error("malformed postfix filter (stack %d at end)", sp); return PB200_E_INVALID; }
    if (maxsp > kMaxStack) { set_error("filter too deep"); return PB200_E_UNSUPPORTED; }
    return PB200_OK;
  }
  // ---- count carrier.  Every RED into the global tables is an L2 read-modify-write, and on this path the L2 request
  // rate is the bound.  When the query needs the per-group row count (COUNT / AVG, or only as the group-exists marker)
  // and sums an INT dictionary column, the count rides in the upper bits of that sum: each row adds
  // (value - vmin) + 2^shift with ONE reduction (or, in a shared-memory table, one 8-byte entry instead of 12).
  //   Fields: sum field = `shift` bits, count field = 64 - shift bits, balanced so that both overflow at about the
  //   same rows per group: shift = ceil((64 + bits(R)) / 2), R = vmax - vmin + 1 from the dictionary (a 20-bit value
  //   range leaves 22 bits = 4 M rows per group; a full 32-bit range 65 535).
  //   Either field CAN overflow; both are detected EXACTLY after the launch from one number: a sum field overflow
  //   carries into the count field (counts only grow: value - vmin >= 0), a count overflow drops 2^(64-shift) from
  //   it, so  sum_g count_g == matched docs  iff neither happened -- the two cannot cancel because the carries total
  //   at most docs x R / 2^shift < 2^(64-shift) when docs x R < 2^64 (the admission test below).  On a mismatch the
  //   submission runs again with a separate COUNT table (kRetryWithoutCountCarrier); results are exact either way.
  // Decided once per result here; it sizes the shared-memory table and lays out the result's tables below.
  void choose_carriers(bool allow_count_carrier) {
    reduce_world = plan.defer_finalize ? std::max(query->reduce_world, 1) : 1;
    carrier.assign(plan.nres, Carrier());
    if (!plan.group_by || !allow_count_carrier || (query->flags & PB200_Q_NO_COUNT_CARRIER) || !tune.pack_count) return;
    for (int r = 0; r < plan.nres; r++) {
      unsigned long long docs = result_docs(r);
      // a table that will be summed with the other GPUs' tables: the admission test covers the docs of ALL of them
      if (plan.defer_finalize) docs = query->merged_docs_bound > 0 ? (unsigned long long)query->merged_docs_bound : docs * (unsigned long long)reduce_world;
      for (int a = 0; a < q.num_aggs; a++) {
        const int fn = q.aggs[a].function;
        if ((fn != PB200_AGG_SUM && fn != PB200_AGG_AVG) || q.aggs[a].val_kind != VAL_DICT_I32) continue;
        if (plan.limb[a] >= 0) continue;   // the moments read limb sums as they are: never a carrier
        long long vmin = std::numeric_limits<long long>::max(), vmax = std::numeric_limits<long long>::min();
        bool ok = true;
        for (int s = 0; s < nseg && ok; s++) {
          if (!in_result(s, r)) continue;
          const DeviceColumn& c = segments[s]->cols[plan.aggs[a].column];
          if (c.dict_host.size() < 4ull * std::max(c.cardinality, 1) || c.stored_type != PB200_INT) { ok = false; break; }
          // the other GPUs must subtract the SAME minimum: only a table-wide (domain) dictionary guarantees that
          if (reduce_world > 1 && !c.dict_shared) { ok = false; break; }
          int32_t v0, v1;   // sorted dictionary: first / last entry
          memcpy(&v0, c.dict_host.data(), 4);
          memcpy(&v1, c.dict_host.data() + 4ull * (c.cardinality - 1), 4);
          vmin = std::min<long long>(vmin, v0);
          vmax = std::max<long long>(vmax, v1);
        }
        if (!ok) continue;
        const int rbits = bits_of((unsigned long long)(vmax - vmin));   // value - vmin fits rbits bits
        if (bits_of(docs) + rbits > 63) continue;                        // docs x R < 2^63: the detection is airtight
        carrier[r].agg = a;
        carrier[r].shift = tune.pack_shift > 0 ? tune.pack_shift : (64 + rbits + 1) / 2;
        carrier[r].vmin = vmin;
        break;
      }
    }
  }
  // ---- tile geometry ----
  int choose_geometry() {
    int max_bits_sum = 0;   // streamed bits per row, widest segment
    for (int s = 0; s < nseg; s++) {
      int sum = 0;
      for (int c : plan.slot_cols) sum += segments[s]->cols[c].bits;
      max_bits_sum = std::max(max_bits_sum, sum);
    }
    // CTA tile = W warps x 1024 rows; every warp streams its own 1024-row slices through a private TMA ring.
    // W = 6 (aggregation only): 192-thread CTAs, two per SM, 168 registers, no spills (32 of them hold the software-pipelined
    // dictionary gathers).  Group-by: the survivor-queue path needs 144-145 registers (ptxas, sm_90a); W = 6 with two CTAs per
    // SM leaves room for a 3-deep ring (faster than W = 8 on C3/range); falls back to one CTA when the rows are too wide
    // for two 2-deep rings, or when a shared-memory group table needs the room (below).
    plan.warps = tune.warps;
    plan.ctas_per_sm = tune.ctas_per_sm;  // default 2: the group-by kernel needs < 168 registers, two 192-thread CTAs per SM
    q.sparse_max = tune.sparse_max;
    q.sparse_max_agg = tune.sparse_max_agg >= 0 ? tune.sparse_max_agg : (plan.group_by ? std::min(q.sparse_max, 2) : q.sparse_max);
    const size_t warp_stage_bytes = (size_t)128 * max_bits_sum;
    size_t extra_bytes = 0;   // shared memory besides the header and the rings
    auto extra_for = [&](int w) { return (q.conj ? 0 : (size_t)w * 32 * kMaxStack * 4) + (plan.group_by ? (size_t)w * 2048 : (size_t)q.num_aggs * w * 32 * 16); };
    extra_bytes = extra_for(plan.warps);
    q.queue_max = plan.group_by ? 1024 : 0;  // every group-by slice goes through the survivor queue
  // CTA-private group tables in shared memory when the key space fits next to a 2-deep ring and every function is
  // COUNT or an integer SUM.  A survivor then costs shared atomics instead of a global RED.  Measured on H100 with
  // 10 000 groups (DESIGN.md section 3.1): one 8-warp CTA per SM with the table and the pipelined last batch runs the
  // headline scan in 1.83 ms, two 6-warp CTAs with the global table in 2.11.
    q.smem_groups = 0;
    for (int a = 0; a < kMaxAggs; a++) q.smem_slot[a] = -1;
    if (plan.group_by && tune.smem_groups) {
      long long gmax = 1;
      for (int s = 0; s < nseg && gmax > 0; s++) {
        long long g = 1;
        for (int k = 0; k < ngb; k++) { g *= std::max(segments[s]->cols[query->group_by_columns[k]].cardinality, 1); if (g > tune.smem_groups_max) { g = -1; break; } }
        gmax = g < 0 ? -1 : std::max(gmax, g);
      }
      bool ok = gmax > 0 && gmax <= tune.dense_max;  // hashed: slots, not raw keys
      int nsum = 0;
      for (int a = 0; a < q.num_aggs && ok; a++) {
        const int fn = q.aggs[a].function, vk = q.aggs[a].val_kind;
        if (fn == PB200_AGG_COUNT || is_moments_fn(fn)) continue;   // VAR / STDDEV: the count and their limb sums
        if ((fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) && (vk == VAL_DICT_I32 || vk == VAL_RAW_I32)) q.smem_slot[a] = (int8_t)nsum++;
        else ok = false;
      }
      // no count array when every result of the launch carries its counts in a sum
      bool all_carry = ok;
      for (int r = 0; r < plan.nres && all_carry; r++) all_carry = carrier[r].agg >= 0;
      q.smem_count = all_carry ? 0 : 1;
      const long long gstride = gmax | 1;
      const size_t copy_bytes = ok ? (size_t)gstride * 4 * (q.smem_count + 2 * nsum) : 0;
      // room left after a 2-deep ring
      auto room_for = [&](int w, int ctas) { return ring_budget(lim, ctas, extra_for(w)) - (long long)(2 * warp_stage_bytes * w); };
      bool fits = ok && room_for(plan.warps, plan.ctas_per_sm) >= (long long)copy_bytes;
      if (ok && !fits && room_for(8, 1) >= (long long)copy_bytes) {
        // a table too large for the configured CTA: one CTA of 8 warps per SM.  With 6 warps the CTA hides too little
        // latency (10 000 groups on H100: 2.20 ms against 2.11 for the global table at 2 CTAs/SM; 8 warps: 1.83).
        plan.warps = 8; plan.ctas_per_sm = 1; extra_bytes = extra_for(8); fits = true;
      }
      if (fits) {
        // replicated copies (fewer same-address conflicts) for small key spaces: they may take at most 64 KB
        const long long room = room_for(plan.warps, plan.ctas_per_sm);
        int copies = 1;
        while (copies < 32 && (long long)copy_bytes * copies * 2 <= std::min<long long>(room, 64 << 10)) copies *= 2;
        if (tune.smem_copies > 0) copies = std::max(1, std::min(copies, tune.smem_copies));
        q.smem_groups = (int32_t)gmax; q.smem_copies = copies; q.smem_gstride = (int32_t)gstride; q.smem_merged = merge ? 1 : 0;
        extra_bytes += copy_bytes * copies;
      } else {
        for (int a = 0; a < kMaxAggs; a++) q.smem_slot[a] = -1;
      }
    }
    const int cw = plan.warps;
    auto stages_for = [&](int ctas) {
      const long long budget = ring_budget(lim, ctas, extra_bytes);
      return warp_stage_bytes == 0 ? 2 : (budget <= 0 ? 0 : (int)std::min<long long>(kMaxStages, budget / (long long)(warp_stage_bytes * cw)));
    };
    int stages = stages_for(plan.ctas_per_sm);
    if (stages < 2 && plan.ctas_per_sm > 1) { plan.ctas_per_sm = 1; stages = stages_for(1); }  // wide rows: fall back to one CTA per SM
    if (stages < 2) { set_error("touched columns too wide for the shared-memory pipeline (%d bits per row)", max_bits_sum); return PB200_E_UNSUPPORTED; }
    if (tune.stages > 0) stages = std::max(2, std::min(stages, tune.stages));
    q.tile_rows = cw * 1024;
    q.num_stages = stages;
    q.stage_words = (uint32_t)(32 * max_bits_sum);
    q.use_pipe = q.num_slots > 0;
    q.defer_agg = -1;
    if (!plan.group_by && tune.defer)
      for (int a = 0; a < q.num_aggs; a++)
        if ((q.aggs[a].function == PB200_AGG_SUM || q.aggs[a].function == PB200_AGG_AVG) && q.aggs[a].val_kind == VAL_DICT_I32) { q.defer_agg = a; break; }
    plan.smem_bytes = kHdrBytes + (size_t)cw * stages * q.stage_words * 4 + extra_bytes;
    // the group table sits behind the rings and the generic-filter stack
    q.queue_off = (uint32_t)(kHdrBytes + (size_t)cw * stages * q.stage_words * 4 + (q.conj ? 0 : (size_t)cw * 32 * kMaxStack * 4));
    q.smem_table_off = q.queue_off + (plan.group_by ? (uint32_t)cw * 2048u : 0u);
    // instantiations: W in {6, 8} x {aggregation only (2 CTAs/SM), group-by with 2 or 1 CTAs/SM}
    plan.variant = ScanVariant{cw, plan.group_by, !plan.group_by && !(cw == 8 && !tune.defer), plan.group_by ? plan.ctas_per_sm : 2};
    plan.skip_masks = q.conj && q.num_slots > 0 && tune.skip;
    return PB200_OK;
  }
  // ---- per segment: tiles and slots ----
  void lay_out_segments() {
    plan.segs.resize(nseg);
    long long tile_cursor = 0;
    for (int s = 0; s < nseg; s++) {
      const pb200_segment* seg = segments[s];
      SegDesc& sd = plan.segs[s];
      memset(&sd, 0, sizeof sd);
      sd.num_docs = seg->num_docs;
      sd.first_tile = tile_cursor;
      sd.num_tiles = (seg->num_docs + q.tile_rows - 1) / q.tile_rows;
      tile_cursor += sd.num_tiles;
      uint32_t word_off = 0, tx = 0;
      for (int k = 0; k < q.num_slots; k++) {
        const DeviceColumn& c = seg->cols[plan.slot_cols[k]];
        sd.slots[k] = SlotDesc{c.fwd, c.bits, word_off, (uint32_t)(128 * c.bits), 0};  // tile_bytes: one warp slice = 1024 rows
        word_off += sd.slots[k].tile_bytes / 4;
        tx += sd.slots[k].tile_bytes;
      }
      sd.stage_tx = tx;
    }
    q.total_tiles = (int32_t)std::min<long long>(tile_cursor, 0x7FFFFFFF);
  }

  LeafBuffer& add_buffer(int s, int l, LeafBuffer::Kind kind, size_t words) { plan.leaf_buffers.push_back(LeafBuffer{kind, s, l, words}); return plan.leaf_buffers.back(); }
  // ---- per segment leaves, conjunctions ordered ----
  int build_leaves() {
    for (int s = 0; s < nseg; s++) {
      const pb200_segment* seg = segments[s];
      SegDesc& sd = plan.segs[s];
      const pb200_filter_node* fs = filter_of(s);
      for (int l = 0; l < q.num_leaves; l++) {
        const pb200_filter_node& n = fs[plan.leaf_node[l]];
        LeafDesc& lf = sd.leaves[l];
        lf.slot = -1;
        if (n.op == PB200_F_MATCH_ALL) { lf.kind = LEAF_ALL; continue; }
        if (n.op == PB200_F_EMPTY) { lf.kind = LEAF_NONE; continue; }
        const bool needs_col = n.op != PB200_F_DOC_MASK && n.op != PB200_F_DOC_RANGES;
        if (needs_col && (n.column < 0 || n.column >= ncols)) { set_error("filter column out of range"); return PB200_E_INVALID; }
        const DeviceColumn& c = seg->cols[needs_col ? n.column : 0];
        if (is_scan_leaf(n.op)) {
          const int slot = (int)(std::find(plan.slot_cols.begin(), plan.slot_cols.end(), n.column) - plan.slot_cols.begin());
          if (slot == q.num_slots) { set_error("scan leaf column %d has no slot (per-segment trees must scan the same columns)", n.column); return PB200_E_INVALID; }
          lf.slot = slot;
          if (n.op == PB200_F_RAW_RANGE) {
            // Raw (no-dictionary) INT column, value-space range: IntRawValueBasedRangePredicateEvaluator
            // (core/operator/filter/predicate/RangePredicateEvaluatorFactory.java:227-262).  On two's complement words
            // lo <= x <= hi  <=>  (uint32)(x - lo) < (uint32)(hi - lo + 1): the dictId range compare of the kernel, unchanged.
            if (c.bits != 32 || c.dict_native || c.stored_type != PB200_INT) { set_error("RAW_RANGE is accelerated for raw INT columns only (column %d)", n.column); return PB200_E_UNSUPPORTED; }
            double dlo = (n.raw_flags & 1) ? -2147483648.0 : std::ceil(n.raw_lo), dhi = (n.raw_flags & 2) ? 2147483647.0 : std::floor(n.raw_hi);
            if (!(n.raw_flags & 1) && (n.raw_flags & 4) && dlo == n.raw_lo) dlo += 1.0;   // exclusive bounds on integral literals
            if (!(n.raw_flags & 2) && (n.raw_flags & 8) && dhi == n.raw_hi) dhi -= 1.0;
            dlo = std::max(dlo, -2147483648.0); dhi = std::min(dhi, 2147483647.0);
            if (!(dlo <= dhi)) { lf.kind = LEAF_NONE; lf.slot = -1; continue; }   // also catches NaN bounds
            const long long lo = (long long)dlo, hi = (long long)dhi;
            if (hi - lo + 1 >= (1ll << 32)) { lf.kind = LEAF_ALL; lf.slot = -1; continue; }
            lf.kind = LEAF_RANGE;
            lf.lo = (uint32_t)(int32_t)lo; lf.span = (uint32_t)(hi - lo + 1);
            lf.cmp = CMP_BOTH;   // one-sided shortcuts assume unsigned order
          } else if (n.op == PB200_F_SCAN_RANGE) {
            lf.kind = LEAF_RANGE;
            int lo = std::max(n.lo, 0), hi = std::max(n.hi, lo);
            lf.lo = (uint32_t)lo; lf.span = (uint32_t)(hi - lo);
            set_cmp(lf, c);
          } else {
            lf.negate = n.op == PB200_F_SCAN_NOT_IN;
            if (n.num_ids == 1) {
              lf.kind = LEAF_RANGE; lf.lo = (uint32_t)n.ids[0]; lf.span = 1;
              set_cmp(lf, c);
            } else if (n.num_ids == 0) {
              lf.kind = LEAF_NONE;
            } else {
              // dictId set -> bitmap over the dictionary (what PredicateEvaluator.getMatchingDictIds feeds the scan)
              size_t words = ((size_t)std::max(c.cardinality, 1) + 31) / 32 + 1;
              if (c.bits == 32) { set_error("IN on raw column not accelerated"); return PB200_E_UNSUPPORTED; }
              words = std::max(words, ((size_t)1 << c.bits) / 32 + 1);  // every representable dictId is addressable
              std::vector<uint32_t> lut(words, 0);
              for (int k = 0; k < n.num_ids; k++) {
                int id = n.ids[k];
                if (id < 0 || id >= c.cardinality) { set_error("dictId %d out of range", id); return PB200_E_INVALID; }
                lut[id >> 5] |= 1u << (id & 31);
              }
              add_buffer(s, l, LeafBuffer::LUT, words).lut = std::move(lut);
              lf.kind = LEAF_LUT;
            }
          }
        } else if (n.op == PB200_F_INV_IN || n.op == PB200_F_INV_NOT_IN) {
          if (!c.inv) { set_error("column %d has no inverted index", n.column); return PB200_E_INVALID; }
          LeafBuffer& b = add_buffer(s, l, LeafBuffer::INV_MASK, doc_mask_words(seg->num_docs));
          for (int k = 0; k < n.num_ids; k++) {  // InvertedIndexFilterOperator: OR of the bitmaps of the dictIds
            const int id = n.ids[k];
            if (id < 0 || id >= c.cardinality) { set_error("dictId %d out of range for inverted index (card %d)", id, c.cardinality); return PB200_E_INVALID; }
            if (c.inv_offsets[id + 1] == c.inv_offsets[id]) continue;  // bound column: this domain id does not occur in the segment
            b.jobs.push_back(DecodeJob{c.inv, c.inv_offsets[id], (unsigned long long)c.inv_offsets[id + 1] - c.inv_offsets[id], nullptr, seg->num_docs});
          }
          lf.kind = LEAF_DOCMASK;
          lf.negate = n.op == PB200_F_INV_NOT_IN;
        } else if (n.op == PB200_F_DOC_MASK) {
          const size_t need = ((size_t)seg->num_docs + 31) / 32;
          if ((size_t)n.num_ids < need || !n.ids) { set_error("DOC_MASK needs %zu words, got %d", need, n.num_ids); return PB200_E_INVALID; }
          if (n.reserved & PB200_NODE_IDS_ON_DEVICE) {
            lf.bits = reinterpret_cast<const uint32_t*>(n.ids);  // made by pb200_doc_mask_upload: padded, resident
          } else {
            LeafBuffer& b = add_buffer(s, l, LeafBuffer::DOC_MASK, doc_mask_words(seg->num_docs));
            b.src = n.ids; b.src_words = need;
          }
          lf.kind = LEAF_DOCMASK;
        } else if (n.op == PB200_F_DOC_RANGES) {
          if (n.num_ids % 2) { set_error("DOC_RANGES needs (start,end) pairs"); return PB200_E_INVALID; }
          if (n.num_ids == 0) { lf.kind = LEAF_NONE; continue; }
          LeafBuffer& b = add_buffer(s, l, LeafBuffer::DOC_RANGES, (size_t)n.num_ids);
          b.src = n.ids; b.src_words = (size_t)n.num_ids;
          lf.kind = LEAF_DOCRANGES;
          lf.num_ranges = n.num_ids / 2;
        } else {
          set_error("unsupported leaf op %d", n.op);
          return PB200_E_UNSUPPORTED;
        }
      }
      // conjunctions: cheapest / most selective leaf first (AND is commutative).  The reference orders AND children by
      // operator priority (FilterOperatorUtils.java:205-251) and, with AndScanReordering, by estimated cardinality
      // (AndDocIdSet.java:118-120); here the estimate is the matching fraction of the dictionary.
      const int nleaves = q.num_leaves;
      if (!q.conj || nleaves <= 1) continue;
      auto cost = [&](int l) -> double {
        const LeafDesc& lf = sd.leaves[l];
        if (lf.slot < 0) return -1.0;  // doc masks / ranges / constants: no column to unpack
        const DeviceColumn& c = seg->cols[plan.slot_cols[lf.slot]];
        double frac = 1.0;
        if (lf.kind == LEAF_RANGE) frac = (double)lf.span / std::max(c.cardinality, 1);
        else if (lf.kind == LEAF_LUT) frac = 0.5;
        return lf.negate ? 1.0 - frac : frac;
      };
      int order[kMaxLeaves];
      for (int l = 0; l < nleaves; l++) order[l] = l;
      std::stable_sort(order, order + nleaves, [&](int a, int b) { return cost(a) < cost(b); });
      LeafDesc sorted[kMaxLeaves];
      int rank[kMaxLeaves];
      for (int l = 0; l < nleaves; l++) { sorted[l] = sd.leaves[order[l]]; rank[order[l]] = l; }
      std::copy(sorted, sorted + nleaves, sd.leaves);
      for (LeafBuffer& b : plan.leaf_buffers) if (b.seg == s) b.leaf = rank[b.leaf];  // the buffer follows its leaf
    }
    return PB200_OK;
  }
  // ---- packed dispatch words (pb200_desc.h): everything the tile loop needs per leaf / aggregation in one word ----
  // software-pipelined aggregations go LAST (nothing is waited on after them).  Aggregation only: q.defer_agg.
  // Group-by: up to two of {SUM / AVG over a 4-byte dictionary, MIN, MAX} -- the kernel issues their loads for the
  // last queue batch and reduces one tile later (into the global table, or the CTA's shared table: integer sums only).
  int encode_dispatch() {
    if (!plan.group_by && q.defer_agg >= 0) {
      pipelined[q.defer_agg] = true;
    } else if (plan.group_by && tune.gb_defer) {
      for (int a = 0; a < q.num_aggs && npipe < 2; a++) {
        if (q.aggs[a].slot < 0) continue;
        const int fn = q.aggs[a].function, vk = q.aggs[a].val_kind;
        const bool sum4 = (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) && (vk == VAL_DICT_I32 || vk == VAL_DICT_F32);
        if (sum4 || fn == PB200_AGG_MIN || fn == PB200_AGG_MAX) { pipelined[a] = true; npipe++; }
      }
    }
    for (int s = 0; s < nseg; s++) {
      SegDesc& sd = plan.segs[s];
      for (int l = 0; l < q.num_leaves; l++) {
        LeafDesc& lf = sd.leaves[l];
        const bool has_slot = lf.slot >= 0;
        lf.code = leaf_code(lf.kind, lf.cmp, lf.negate, has_slot ? sd.slots[lf.slot].bits : 0, has_slot ? sd.slots[lf.slot].stage_words : 0u);
      }
      int n = 0;
      for (int pass = 0; pass < 2; pass++)
        for (int a = 0; a < q.num_aggs; a++) {
          if (q.aggs[a].slot < 0 || pipelined[a] != (pass == 1)) continue;
          if (plan.pct_rep[a] >= 0 && plan.pct_rep[a] != a) continue;   // reads another PERCENTILE's histogram
          const SlotDesc& sl = sd.slots[q.aggs[a].slot];
          sd.agg_code[n++] = agg_code(a, q.aggs[a].function, q.aggs[a].val_kind, sl.bits, sl.stage_words);
        }
      sd.num_agg_codes = n;
      sd.num_defer_codes = plan.group_by ? npipe : 0;
      // dictionaries
      for (int a = 0; a < q.num_aggs; a++) {
        if (q.aggs[a].slot < 0) continue;
        const DeviceColumn& c = segments[s]->cols[plan.aggs[a].column];
        sd.dict[a] = c.dict_native;
        if (plan.limb[a] >= 0) {   // K, H or L of the column's limb dictionaries (checked ready above)
          const MomentDict& md = *c.moments;
          sd.dict[a] = md.limbs + (size_t)plan.limb[a] * md.entries;
          continue;
        }
        if ((q.aggs[a].function == PB200_AGG_SUM || q.aggs[a].function == PB200_AGG_AVG) && q.aggs[a].val_kind != VAL_RAW_I32 && !c.dict_native) {
          set_error("SUM/AVG over column %d needs its dictionary on the device", plan.aggs[a].column);
          return PB200_E_INVALID;
        }
      }
    }
    return PB200_OK;
  }
  // ---- result layouts: accumulators and bitsets (aggregation only) or group tables ----
  int lay_out_results() {
    bool any_pct = false, any_mom = false;
    for (int a = 0; a < q.num_aggs; a++) any_pct |= plan.pct_rep[a] >= 0;
    for (int a = 0; a < nuser; a++) any_mom |= plan.mom_first[a] >= 0;
    // histogram bins are u32; the moments' limb sums are exact for n < 2^32: a result over 2^32 docs is refused
    for (int r = 0; r < plan.nres && (any_pct || any_mom); r++)
      if (result_docs(r) >= (1ull << 32)) {
        set_error("%s over %llu docs in one result: at most 2^32 - 1", any_pct ? "PERCENTILE" : "VAR/STDDEV", result_docs(r));
        return PB200_E_UNSUPPORTED;
      }
    if (!plan.group_by) {
      // PERCENTILE: one histogram of 2^bits u32 entries per result and column (every representable dictId is addressable)
      plan.hist_entries.assign(plan.nres, std::vector<size_t>(q.num_aggs, 0));
      for (int r = 0; r < plan.nres; r++)
        for (int a = 0; a < q.num_aggs; a++) {
          if (plan.pct_rep[a] != a) continue;
          const int maxbits = result_max_bits(r, plan.aggs[a].column);
          plan.hist_entries[r][a] = (size_t)1 << maxbits;
          plan.hist_total += 1ll << maxbits;
        }
      // few dictIds: warp-private shared-memory histograms (SegDesc.distinct_words as the flag)
      for (int s = 0; s < nseg; s++)
        for (int a = 0; a < q.num_aggs; a++)
          if (plan.pct_rep[a] == a) plan.segs[s].distinct_words[a] = segments[s]->cols[plan.aggs[a].column].cardinality <= kHistWarpPrivateMaxCard ? 1u : 0u;
      // DISTINCTCOUNT: one dictId bitset per result; a merged result's bitset must hold the dictIds of every segment
      plan.distinct_words.assign(plan.nres, std::vector<size_t>(q.num_aggs, 0));
      for (int r = 0; r < plan.nres; r++)
        for (int a = 0; a < q.num_aggs; a++)
          if (q.aggs[a].function == PB200_AGG_DISTINCTCOUNT) plan.distinct_words[r][a] = ((size_t)1 << result_max_bits(r, plan.aggs[a].column)) / 32 + 1;
    } else {
      plan.tables.resize(plan.nres);
      for (int r = 0; r < plan.nres; r++)
        if (int rc = lay_out_table(r)) return rc;
      // the host-only parts of the segments' table descriptors
      for (int s = 0; s < nseg; s++) {
        SegDesc& sd = plan.segs[s];
        const TableLayout& t = plan.tables[merge ? 0 : s];
        for (int a = 0; a < q.num_aggs; a++) {
          sd.sum_addend[a] = 0ull - (1ull << 31);  // plain INT-dictionary sum: remove the device copy's bias
          if (a == t.carrier.agg) sd.sum_addend[a] = (1ull << t.carrier.shift) - (unsigned long long)((uint32_t)(int32_t)t.carrier.vmin ^ 0x80000000u);
          sd.distinct_words[a] = plan.pct_rep[a] >= 0 ? t.hist_per_group[a] : t.dwords[a];
        }
        for (int g = 0; g < ngb; g++) { sd.group_mult[g] = t.mult[g] * (uint32_t)t.stride; sd.group_mult64[g] = t.mult64[g]; }  // hash tables: stride 1
        sd.h_mask = t.hashed ? (uint32_t)(t.groups - 1) : 0u;
        sd.h_limit = query->num_groups_limit;
      }
    }
    if (plan.hist_total > kMaxHistogramEntries) {
      set_error("PERCENTILE histograms of %lld entries in one call (at most %lld)", plan.hist_total, kMaxHistogramEntries);
      return PB200_E_UNSUPPORTED;
    }
    return PB200_OK;
  }
  // dense group table over the raw key space (column 0 least significant, DictionaryBasedGroupKeyGenerator :311-346)
  int lay_out_table(int r) {
    const pb200_segment* seg = segments[merge ? 0 : r];
    TableLayout& t = plan.tables[r];
    unsigned __int128 space = 1;  // size of the raw key space
    for (int g = 0; g < ngb; g++) {
      const int card = std::max(seg->cols[query->group_by_columns[g]].cardinality, 1);
      // every representable dictId must stay inside the table even for padded / corrupt rows
      t.mult.push_back((uint32_t)(unsigned long long)space);
      t.mult64.push_back((unsigned long long)space);
      t.cards.push_back(card);
      space *= (unsigned)card;
      if (space >> 63) {  // the reference's ARRAY_MAP regime (keys wider than a long): not accelerated
        set_error("group key space does not fit 63 bits (ARRAY_MAP regime): fall back to the reference operator");
        return PB200_E_UNSUPPORTED;
      }
    }
    // dense table up to dense_max raw keys (ARRAY / INT_MAP regimes of the reference), beyond it a hash table over the
    // 64-bit raw key (LONG_MAP regime, and INT_MAP key spaces too large to be worth a dense table)
    t.hashed = space > (unsigned __int128)tune.dense_max;
    if (t.hashed) {
      const long long limit = std::max(query->num_groups_limit, 1);
      long long cap = 1 << 16;
      while (cap < 2 * (limit + 1) && cap < (1ll << 27)) cap <<= 1;
      if (cap < 2 * (limit + 1)) { set_error("numGroupsLimit %lld too large for the device hash table", limit); return PB200_E_UNSUPPORTED; }
      t.groups = cap;
    } else {
      t.groups = (long long)space;
      // Small dense tables are SPREAD: entry of raw key k sits at k * stride.  A 10 000-group table is 80 KB = 312 of the
      // 256-byte chunks the L2 address hash distributes over the L2 slices -- some slices own three chunks, some none, and
      // every surviving row sends a reduction to them (ncu: hottest slice 75 % tag-request utilisation vs 56 % average).
      // With one entry per 128 bytes the same reductions spread over >= 4096 chunks.  Costs table bytes (<= 2 MB each,
      // memset + extraction scan), no instruction in the kernel: the stride is folded into the key multipliers.
      bool any_bitset = false;
      for (int a = 0; a < q.num_aggs; a++) any_bitset |= q.aggs[a].function == PB200_AGG_DISTINCTCOUNT || q.aggs[a].function == PB200_AGG_PERCENTILE;
      if (q.smem_groups == 0 && !any_bitset && tune.table_stride != 1) {
        long long s = 1;
        if (tune.table_stride > 1) s = tune.table_stride;
        else while (s < 16 && t.groups * 8 * s * 2 <= (2ll << 20)) s *= 2;   // keep each table within 2 MB
        while (s > 1 && t.groups * s > (1ll << 26)) s /= 2;
        t.stride = (int)s;
        t.groups *= s;
      }
    }
    // one block per element kind
    // the exact per-group count is kept only when a function needs it; otherwise a dictionary MIN/MAX table (or a flag
    // table) marks the groups that exist -- one atomic less per surviving row.  A raw INT MIN/MAX table cannot: every
    // u32 is a value there, the empty entry included (max_offset in pb200_desc.h)
    bool need_count = tune.always_count != 0;
    auto marks_groups = [&](int a) {
      return (q.aggs[a].function == PB200_AGG_MIN || q.aggs[a].function == PB200_AGG_MAX) && q.aggs[a].val_kind != VAL_RAW_I32;
    };
    bool has_marker = false;
    for (int a = 0; a < q.num_aggs; a++) {
      need_count |= q.aggs[a].function == PB200_AGG_COUNT || q.aggs[a].function == PB200_AGG_AVG || is_moments_fn(q.aggs[a].function);
      has_marker |= marks_groups(a);
    }
    bool need_seen = !need_count && !has_marker && !t.hashed;  // a hash table's keys mark the groups that exist
    t.reduce_world = reduce_world;
    if ((need_count || need_seen) && carrier[r].agg >= 0) {  // the count rides in a sum (see the count carrier above)
      t.carrier = carrier[r];
      need_count = false; need_seen = false;
    }
    // a shared-memory table without a count array relies on every result carrying its counts
    if (q.smem_groups && !q.smem_count && t.carrier.agg < 0) { set_error("internal: shared-memory group table has no count array"); return PB200_E_INVALID; }
    t.need_count = need_count;
    t.need_seen = need_seen;
    long long ii = need_count ? 1 : 0, fi = 0, xi = need_seen ? 1 : 0, ni = 0;
    for (int a = 0; a < q.num_aggs; a++) {
      const int fn = q.aggs[a].function, vk = q.aggs[a].val_kind;
      if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) t.index[a] = (int)(sum_in_double(vk) ? fi++ : ii++);
      else if (fn == PB200_AGG_MIN) { t.index[a] = (int)ni++; if (!need_count && marks_groups(a) && t.exists_max < 0 && t.exists_min < 0) t.exists_min = a; }
      else if (fn == PB200_AGG_MAX) { t.index[a] = (int)xi++; if (!need_count && marks_groups(a) && t.exists_max < 0 && t.exists_min < 0) t.exists_max = a; }
      else if (fn == PB200_AGG_DISTINCTCOUNT) {  // one dictId bitset per group / slot
        const DeviceColumn& c = seg->cols[plan.aggs[a].column];
        const unsigned long long words = ((unsigned long long)c.cardinality + 31) / 32;
        if (words * (unsigned long long)t.groups > (1ull << 28)) {
          set_error("DISTINCTCOUNT with GROUP BY: %lld groups x %d dictIds exceed the device bitset budget", t.groups, c.cardinality);
          return PB200_E_UNSUPPORTED;
        }
        t.dwords[a] = (uint32_t)words;
      } else if (fn == PB200_AGG_PERCENTILE && plan.pct_rep[a] == a) {  // one dictId histogram per group / slot
        const int card = seg->cols[plan.aggs[a].column].cardinality;
        t.hist_per_group[a] = (uint32_t)card;
        plan.hist_total += (long long)card * t.groups;
        // refused in lay_out_results, after the later results' DISTINCTCOUNT budgets were checked
        if ((unsigned long long)card * (unsigned long long)t.groups > (unsigned long long)kMaxHistogramEntries) break;
      }
    }
    t.i64_elems = ii * t.groups; t.f64_elems = fi * t.groups; t.u32max_elems = xi * t.groups; t.u32min_elems = ni * t.groups;
    // cross-GPU combine of a count-carrying table: ONE extra int64 behind the tables carries this rank's "not provably
    // safe" verdict (0 / 1), so that the verdicts of all ranks are summed by the same collective that sums the tables
    // ... and, in front of it, the four execution statistics of this rank: tables, verdict and statistics of a query then
    // cross the GPUs in ONE collective (pb200_comm.cu).  Tail = {docs scanned, entries in filter, entries post filter,
    // total docs, verdict}; the verdict stays the LAST element.
    t.flag_slot = t.carrier.agg >= 0 && t.reduce_world > 1;
    t.tail_slots = (t.reduce_world > 1 && t.i64_elems > 0) ? 5 : 0;
    t.i64_elems += t.tail_slots;
    return PB200_OK;
  }
  // ---- the group-by kernel specialised for the shared-table shape (pb200_scan.cuh SPEC) when the launch has it: a
  //      conjunction of at most two dictionary range leaves (or constant leaves) in every segment, a dense key over one or
  //      two columns, the CTA-private table, and COUNT plus at most two INT dictionary sums, all of them pipelined.  It
  //      runs the same geometry, layouts and descriptors; only the instruction stream differs. ----
  void choose_spec() {
    if (!tune.spec || !plan.group_by || q.smem_groups <= 0 || !q.conj || q.num_leaves > 2 || ngb > 2 ||
        !((plan.warps == 8 && plan.ctas_per_sm == 1) || (plan.warps == 6 && plan.ctas_per_sm == 2))) return;
    bool spec = true;
    for (int a = 0; a < q.num_aggs && spec; a++) {
      const int fn = q.aggs[a].function;
      spec = fn == PB200_AGG_COUNT || ((fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) && q.aggs[a].val_kind == VAL_DICT_I32 && pipelined[a]);
    }
    for (int r = 0; r < plan.nres && spec; r++) spec = !plan.tables[r].hashed;
    for (int s = 0; s < nseg && spec; s++) {
      const SegDesc& sd = plan.segs[s];
      spec = sd.num_agg_codes == sd.num_defer_codes && sd.num_agg_codes <= 2;
      for (int l = 0; l < q.num_leaves && spec; l++) {
        const LeafDesc& lf = sd.leaves[l];
        spec = lf.kind == LEAF_ALL || lf.kind == LEAF_NONE || (lf.kind == LEAF_RANGE && sd.slots[lf.slot].bits <= 31);
      }
    }
    plan.variant.spec = spec;
  }
  // ---- launch chunks of <= kMaxLaunchSegs segments (their TMA table travels in the kernel parameters) ----
  int lay_out_chunks_and_statistics() {
    for (int c0 = 0; c0 < nseg; c0 += kMaxLaunchSegs) {
      LaunchChunk ch{c0, std::min(nseg - c0, (int)kMaxLaunchSegs)};
      if (lay_out_chunk(tune, lim, plan, ch) >= (1 << 30)) { set_error("too many tiles in one launch"); return PB200_E_UNSUPPORTED; }
      plan.chunks.push_back(ch);
    }
    // execution statistics: every scan leaf looks at every doc of its segment
    plan.in_filter.assign(plan.nres, 0);
    for (int s = 0; s < nseg; s++)
      for (int l = 0; l < q.num_leaves; l++) if (is_scan_leaf(filter_of(s)[plan.leaf_node[l]].op)) plan.in_filter[merge ? 0 : s] += segments[s]->num_docs;
    for (int k = 0; k < q.num_slots; k++) if (q.slot_roles[k] & (ROLE_GROUP | ROLE_AGG)) plan.projected++;
    return PB200_OK;
  }
};

}  // namespace

int plan_scan(const Tuning& tune, DeviceLimits lim, const pb200_query* query, pb200_segment* const* segments, int nseg,
              bool allow_count_carrier, ScanPlan* out, const double* agg_args) {
  if (!query || !segments || !out || nseg <= 0) { set_error("invalid argument to pb200_execute"); return PB200_E_INVALID; }
  const bool merge = query->flags & PB200_Q_MERGE_SEGMENTS;
  const int nnodes = query->num_filter_nodes, nuser = query->num_aggs, ngb = query->num_group_by;
  if (nuser < 0 || nuser > kMaxAggs || ngb < 0 || ngb > kMaxGroupBy || nnodes < 0 || nnodes > kMaxNodes) {
    set_error("query exceeds device limits (aggs %d/%d, group-by %d/%d, filter nodes %d/%d)", nuser, kMaxAggs, ngb, kMaxGroupBy, nnodes, kMaxNodes);
    return PB200_E_UNSUPPORTED;
  }
  if (nuser == 0) { set_error("at least one aggregation is required on this path"); return PB200_E_INVALID; }
  if (!segments[0]) { set_error("segment %d does not belong to this context / schema", 0); return PB200_E_INVALID; }
  const int ncols = common_columns(segments, nseg);
  if (ncols < 0) { set_error("the segments do not belong to this context / schema"); return PB200_E_INVALID; }

  if (merge && nseg > 1) {
    for (int g = 0; g < ngb; g++) {
      const int c = query->group_by_columns[g];
      if (c >= 0 && c < ncols && !same_dictionary(segments, nseg, c, "group-by")) return PB200_E_UNSUPPORTED;
    }
    for (int a = 0; a < nuser; a++) {
      const pb200_agg& ag = query->aggs[a];
      if (ag.function != PB200_AGG_MIN && ag.function != PB200_AGG_MAX && ag.function != PB200_AGG_DISTINCTCOUNT &&
          ag.function != PB200_AGG_PERCENTILE && !is_moments_fn(ag.function)) continue;
      if (ag.column < 0 || ag.column >= ncols) continue;
      if (segments[0]->cols[ag.column].bits == 32 && !segments[0]->cols[ag.column].dict_native) continue;  // raw values, no ids
      const char* what = ag.function == PB200_AGG_DISTINCTCOUNT ? "DISTINCTCOUNT" : ag.function == PB200_AGG_PERCENTILE ? "PERCENTILE"
                         : is_moments_fn(ag.function) ? "VAR/STDDEV" : "MIN/MAX";
      if (!same_dictionary(segments, nseg, ag.column, what)) return PB200_E_UNSUPPORTED;
    }
  }
  *out = ScanPlan();
  ScanPlanner p{tune, lim, query, segments, nseg, ncols, *out};
  if (int rc = p.expand_moments()) return rc;
  if (int rc = p.assign_slots(agg_args)) return rc;
  if (int rc = p.compile_filter()) return rc;
  p.choose_carriers(allow_count_carrier);
  if (int rc = p.choose_geometry()) return rc;
  p.lay_out_segments();
  if (int rc = p.build_leaves()) return rc;
  if (int rc = p.encode_dispatch()) return rc;
  if (int rc = p.lay_out_results()) return rc;
  p.choose_spec();
  return p.lay_out_chunks_and_statistics();
}

int plan_selection(const Tuning& tune, DeviceLimits lim, const pb200_query* filter_only, const pb200_selection* sel,
                   pb200_segment* const* segments, int nseg, bool prefix, SelectionPlan* out) {
  if (!filter_only || !sel || !segments || !out || nseg <= 0) { set_error("invalid argument to pb200_execute_selection"); return PB200_E_INVALID; }
  if (sel->limit < 0 || sel->num_columns < 0 || (sel->num_columns > 0 && !sel->columns)) { set_error("selection: bad limit or column list"); return PB200_E_INVALID; }
  if (sel->limit > PB200_MAX_SELECT_LIMIT) { set_error("selection LIMIT %lld above %d", (long long)sel->limit, PB200_MAX_SELECT_LIMIT); return PB200_E_UNSUPPORTED; }
  if (sel->num_order_items < 0 || sel->num_order_items > PB200_MAX_ORDER_BY) { set_error("selection ORDER BY with %d items (1..%d)", sel->num_order_items, PB200_MAX_ORDER_BY); return PB200_E_INVALID; }
  // the select phase puts the segment index in gridDim.y
  if (nseg > kMaxSelectSegments) { set_error("selection over %d segments: at most %d per submission", nseg, kMaxSelectSegments); return PB200_E_UNSUPPORTED; }
  // the scan: the caller's filter, COUNT(*) (matched docs per segment), one result per segment
  static const pb200_agg kCount = {PB200_AGG_COUNT, -1};
  pb200_query q = *filter_only;
  q.num_group_by = 0;
  q.group_by_columns = nullptr;
  q.num_aggs = 1;
  q.aggs = &kCount;
  q.flags = filter_only->flags & PB200_Q_PER_SEGMENT_FILTER;
  q.reduce_world = 0;
  q.merged_docs_bound = 0;
  SelectionPlan& p = *out;
  p = SelectionPlan();
  if (int rc = plan_scan(tune, lim, &q, segments, nseg, false, &p.scan)) return rc;
  ScanPlan& plan = p.scan;
  p.limit = sel->limit;

  // ---- selected and order columns: one value kind for all segments ----
  const int ncols = common_columns(segments, nseg);
  auto kind_of = [&](int c, const char* what, int* out_kind) -> int {
    if (c < 0 || c >= ncols) { set_error("%s column %d out of range", what, c); return PB200_E_INVALID; }
    int kind = -1;
    for (int s = 0; s < nseg; s++) {
      const DeviceColumn& dc = segments[s]->cols[c];
      int ks;
      if (dc.fwd_kind != PB200_FWD_DICT_FIXEDBIT && dc.fwd_kind != PB200_FWD_RAW_FIXEDBYTE) ks = -1;
      else if (dc.bits == 32 && !dc.dict_native) ks = dc.stored_type == PB200_INT ? SEL_RAW_I32 : dc.stored_type == PB200_FLOAT ? SEL_RAW_F32 : -1;
      else if (dc.stored_type == PB200_STRING) ks = SEL_DICT_ID;
      else if (!dc.dict_native) ks = -1;
      else ks = dc.stored_type == PB200_INT ? SEL_DICT_I32 : dc.stored_type == PB200_LONG ? SEL_DICT_I64
              : dc.stored_type == PB200_FLOAT ? SEL_DICT_F32 : SEL_DICT_F64;
      if (ks < 0) { set_error("%s column %d of segment %d has no device dictionary or raw 32-bit values: not accelerated", what, c, s); return PB200_E_UNSUPPORTED; }
      if (kind >= 0 && ks != kind) { set_error("%s column %d is stored differently in segment %d than in segment 0", what, c, s); return PB200_E_UNSUPPORTED; }
      kind = ks;
    }
    *out_kind = kind;
    return PB200_OK;
  };
  for (int k = 0; k < sel->num_columns; k++) {
    int kind = 0;
    if (int rc = kind_of(sel->columns[k], "selected", &kind)) return rc;
    p.columns.push_back(sel->columns[k]);
    p.kinds.push_back(kind);
  }
  for (int k = 0; k < sel->num_order_items; k++) {
    int kind = 0;
    if (int rc = kind_of(sel->order[k].column, "ORDER BY", &kind)) return rc;
    p.order_cols.push_back(sel->order[k].column);
    p.order_kinds.push_back(kind);
    p.order_desc.push_back(sel->order[k].descending != 0);
  }
  // a COUNT(*) launch has no deferred gathers: at 8 warps it runs the variant without them (the one that stores the mask)
  if (plan.variant.warps == 8) plan.variant.defer = false;
  // the top rows by value can sit anywhere in a segment: ORDER BY scans every doc
  if (!p.order_cols.empty()) prefix = false;

  // ---- scanned range: a prefix of whole tiles, or the whole segment ----
  const long long tile_rows = plan.q.tile_rows;
  const long long prefix_tiles = (std::max(kSelectPrefixRows, 2 * p.limit) + tile_rows - 1) / tile_rows;
  p.scan_docs.resize(nseg);
  for (int s = 0; s < nseg; s++) {
    SegDesc& sd = plan.segs[s];
    const long long leaves_per_doc = sd.num_docs > 0 ? plan.in_filter[s] / sd.num_docs : 0;
    p.scan_docs[s] = sd.num_docs;
    if (prefix && sd.num_tiles > prefix_tiles) {
      sd.num_tiles = prefix_tiles;
      p.scan_docs[s] = prefix_tiles * tile_rows;
      p.prefix = true;
    }
    plan.in_filter[s] = leaves_per_doc * p.scan_docs[s];
  }
  // launch chunks over the (possibly shortened) tile ranges -- the grouping of segments into chunks is plan_scan's
  long long cursor = 0;
  p.mask_word_off.resize(nseg);
  for (LaunchChunk& ch : plan.chunks) {
    p.chunk_word_off.push_back(cursor * tile_rows / 32);
    const long long c_tiles = lay_out_chunk(tune, lim, plan, ch);
    for (int s = ch.first_seg; s < ch.first_seg + ch.num_segs; s++) p.mask_word_off[s] = (cursor + plan.segs[s].first_tile) * tile_rows / 32;
    cursor += c_tiles;
  }
  p.mask_words = cursor * tile_rows / 32;
  return PB200_OK;
}

std::vector<int> selection_rescan(const SelectionPlan& p, pb200_segment* const* segments, const std::vector<long long>& matches) {
  std::vector<int> out;
  for (size_t s = 0; s < p.scan_docs.size(); s++)
    if (p.scan_docs[s] < segments[s]->num_docs && matches[s] < p.limit) out.push_back((int)s);
  return out;
}

Rescan rescan_query(const pb200_query& q, pb200_segment* const* segments, const std::vector<int>& rescan) {
  const bool per_seg_filter = q.flags & PB200_Q_PER_SEGMENT_FILTER;
  Rescan r{q, {}, {}};
  for (int s : rescan) {
    r.segs.push_back(segments[s]);
    if (per_seg_filter) r.filter.insert(r.filter.end(), q.filter + (size_t)s * q.num_filter_nodes, q.filter + (size_t)(s + 1) * q.num_filter_nodes);
  }
  if (per_seg_filter) r.query.filter = r.filter.data();   // a moved vector keeps its elements where they are
  return r;
}

int plan_distinct(const Tuning& tune, DeviceLimits lim, const pb200_query* filter_only, const pb200_selection* distinct,
                  pb200_segment* const* segments, int nseg, bool merge, bool prefix, DistinctPlan* out) {
  if (!filter_only || !distinct || !segments || !out || nseg <= 0) { set_error("invalid argument to pb200_execute_distinct"); return PB200_E_INVALID; }
  const int nkeys = distinct->num_columns;
  if (nkeys <= 0 || !distinct->columns) { set_error("DISTINCT needs at least one column"); return PB200_E_INVALID; }
  if (nkeys > kMaxDistinctColumns) { set_error("DISTINCT over %d columns (at most %d)", nkeys, kMaxDistinctColumns); return PB200_E_UNSUPPORTED; }
  if (distinct->num_order_items < 0 || distinct->num_order_items > PB200_MAX_ORDER_BY) { set_error("DISTINCT ORDER BY with %d items (1..%d)", distinct->num_order_items, PB200_MAX_ORDER_BY); return PB200_E_INVALID; }
  DistinctPlan& p = *out;
  p = DistinctPlan();
  // every order item names a DISTINCT column (SQL: ORDER BY items of a SELECT DISTINCT must appear in the select list)
  std::vector<bool> ordered_col(nkeys, false);
  for (int k = 0; k < distinct->num_order_items; k++) {
    const int key = (int)(std::find(distinct->columns, distinct->columns + nkeys, distinct->order[k].column) - distinct->columns);
    if (key == nkeys) { set_error("DISTINCT ORDER BY column %d is not one of the DISTINCT columns", distinct->order[k].column); return PB200_E_INVALID; }
    if (ordered_col[key]) continue;
    ordered_col[key] = true;
    p.order_key.push_back(key);
    p.order_desc.push_back(distinct->order[k].descending != 0);
  }
  if (int rc = plan_selection(tune, lim, filter_only, distinct, segments, nseg, prefix, &p.sel)) return rc;
  // key columns: dictIds (a raw column streamed as 32-bit values has none)
  for (int k = 0; k < nkeys; k++) {
    const int col = distinct->columns[k];
    for (int s = 0; s < nseg; s++) {
      const DeviceColumn& c = segments[s]->cols[col];
      if (c.bits > 31 || c.cardinality <= 0 || c.fwd_kind != PB200_FWD_DICT_FIXEDBIT) {
        set_error("DISTINCT column %d is not dictionary-encoded in segment %d: not accelerated", col, s);
        return PB200_E_UNSUPPORTED;
      }
    }
    if (merge && nseg > 1 && !same_dictionary(segments, nseg, col, "DISTINCT")) return PB200_E_UNSUPPORTED;
  }
  p.nres = merge ? 1 : nseg;
  p.cards.resize(nseg);
  p.mult.resize(nseg);
  for (int s = 0; s < nseg; s++) {
    long long space = 1;
    for (int k = 0; k < nkeys; k++) {
      const int card = segments[s]->cols[distinct->columns[k]].cardinality;
      p.cards[s].push_back(card);
      p.mult[s].push_back((uint32_t)space);
      space *= card;
      if (space > kMaxDistinctKeys) {
        set_error("DISTINCT key space of segment %d above %lld entries: not accelerated", s, kMaxDistinctKeys);
        return PB200_E_UNSUPPORTED;
      }
    }
    if (!merge || s == 0) {
      p.table_off.push_back(p.table_entries);
      p.table_size.push_back(space);
      p.table_entries += space;
    }
  }
  if (p.table_entries > kMaxDistinctEntries) {
    set_error("DISTINCT tables of %lld entries in one call (at most %lld)", p.table_entries, kMaxDistinctEntries);
    return PB200_E_UNSUPPORTED;
  }
  return PB200_OK;
}

std::vector<unsigned long long> distinct_bounds(const DistinctPlan& p, pb200_segment* const* segments) {
  const int nseg = (int)p.sel.scan_docs.size();
  std::vector<unsigned long long> bound(p.nres, kDistinctEmpty);
  for (int s = nseg - 1; s >= 0; s--)   // the earliest truncated segment of each result wins
    if (p.sel.scan_docs[s] < segments[s]->num_docs)
      bound[p.nres == 1 ? 0 : s] = (unsigned long long)s << 32 | (unsigned long long)p.sel.scan_docs[s];
  return bound;
}

std::vector<int> distinct_rescan(const DistinctPlan& p, pb200_segment* const* segments, const std::vector<long long>& below) {
  const int nseg = (int)p.sel.scan_docs.size();
  const std::vector<unsigned long long> bound = distinct_bounds(p, segments);
  std::vector<int> out;
  for (int s = 0; s < nseg; s++) {
    const int r = p.nres == 1 ? 0 : s;
    if (p.sel.scan_docs[s] < segments[s]->num_docs && bound[r] != kDistinctEmpty && below[r] < p.sel.limit) out.push_back(s);
  }
  return out;
}

TmaTable tma_table(const ScanPlan& plan, const LaunchChunk& c) {
  TmaTable tt;
  memset(&tt, 0, sizeof tt);
  for (int s = 0; s < c.num_segs; s++) {
    const SegDesc& sd = plan.segs[c.first_seg + s];
    tt.seg[s].first_tile = (int32_t)sd.first_tile;
    tt.seg[s].end_tile = (int32_t)(sd.first_tile + sd.num_tiles);
    tt.seg[s].stage_tx = sd.stage_tx;
    tt.seg[s].num_docs = (uint32_t)sd.num_docs;
    for (int k = 0; k < plan.q.num_slots; k++) tt.seg[s].slot[k] = TmaSlot{sd.slots[k].data, sd.slots[k].tile_bytes, sd.slots[k].stage_words};
    if (plan.skip_masks) {
      int nm = 0;
      for (int l = 0; l < plan.q.num_leaves && nm < kMaxSkipMasks; l++)
        if (sd.leaves[l].kind == LEAF_DOCMASK && !sd.leaves[l].negate) tt.seg[s].skip_mask[nm++] = sd.leaves[l].bits;
    }
  }
  for (int s = c.num_segs; s < kMaxLaunchSegs; s++) { tt.seg[s].first_tile = c.total_tiles; tt.seg[s].end_tile = 0x7FFFFFFF; }  // sentinel
  return tt;
}

}  // namespace pb200
