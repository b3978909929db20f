// pb200_expr.cu -- aggregations over multi-column expressions (DESIGN.md section 3.15): SUM / AVG / MIN / MAX of a
// per-row value computed from two or more columns.
//
// The scan kernel is not involved in the per-row work.  The query runs its usual scan with each expression aggregation
// replaced by COUNT(*): that scan builds the group tables (dense keys, hash keys) and every count.  This stage then
//   1. gets the match mask from a filter-only scan with the mask output switched on (the launch selection uses,
//      plan_selection); a query whose filter matches every doc skips it;
//   2. runs one pass over the mask: per matched doc it gathers each distinct leaf column's value (read_at / sel_value of
//      pb200_select.cuh), evaluates every expression program (pb200_expr.h), finds the group's table entry -- dense: the
//      key columns' dictIds times the table's multipliers; hashed: a read-only probe of the keys the scan inserted -- and
//      accumulates.  SUM / AVG add into one f64 per entry, MIN / MAX take the u64 min / max of the Double.compare key.
//      Lanes of a warp that hit one entry are combined first (one atomic per entry and warp word); aggregation-only
//      results reduce in registers and once per block.
// Both launches are queued on the call's stream behind the scan; neither synchronises.
//
// CASE WHEN (DESIGN.md section 3.19, pb200_execute_exprs_cond) runs in the same pass, in its own instantiation of the
// kernel: per matched doc it reads each distinct condition column's dictId once, tests it against every condition of
// that column (a dictId range, or a bit of the call's bitset buffer), and hands the row's condition word to the program.
//
// Predicates on such expressions (DESIGN.md section 3.16, pb200_expr_doc_masks) run before the query is planned:
// expr_mask_kernel evaluates every doc of every segment against each predicate and writes the doc mask that the query's
// filter tree then reads as a PB200_F_DOC_MASK leaf.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <type_traits>
#include <vector>

#include "pb200_expr.h"
#include "pb200_plan.h"
#include "pb200_scan.cuh"
#include "pb200_select.cuh"

namespace pb200 {
namespace {

constexpr int kExprThreads = 256;

struct ExprSeg {
  const uint32_t* mask;             // match mask, bit j of word w = doc 32w + j (NULL: every doc matches)
  long long num_docs;
  int32_t ncols, ngb;
  SelCol col[kExprMaxCols];         // the distinct leaf columns
  SelCol key[kMaxGroupBy];          // group-by columns (read_at only)
  uint32_t mult[kMaxGroupBy];       // dense tables: entry = sum dictId_k * mult[k] (the table stride folded in)
  unsigned long long mult64[kMaxGroupBy];  // hash tables: raw key = sum dictId_k * mult64[k]
  const unsigned long long* hkeys;  // hash table keys (NULL: dense)
  uint32_t hmask;
  uint32_t pad;
  void* out[kMaxAggs];              // per expression: its table (group-by) or its one accumulator word
};

struct ExprProg {
  int32_t nx;
  int32_t fn[kMaxAggs];
  int32_t len[kMaxAggs];
  pb200_transform_op ops[kMaxAggs][kTransformMaxProgram];
};

constexpr int kExprMaxConds = PB200_MAX_EXPR_CONDS;
struct CondSeg {                      // one segment's conditions, grouped by column
  int32_t ncc;                        // distinct condition columns
  int32_t first[kExprMaxConds + 1];   // the conditions of column c: entries first[c] .. first[c + 1] - 1
  SelCol ccol[kExprMaxConds];         // read_at only: the dictId
  int32_t kind[kExprMaxConds];        // PB200_COND_*
  int32_t slot[kExprMaxConds];        // the condition's index in the call's table: its bit in the row's condition word
  uint32_t hi[kExprMaxConds];         // RANGE: [lo, hi)
  uint32_t pad;
  long long lo[kExprMaxConds];        // RANGE: lo; BITSET: the first word of this segment's bitset
};

// the table entry of the group of `doc`; false when its key is not in the hash table (only after an overflow, whose
// result is discarded as PB200_E_LIMIT)
__device__ __forceinline__ bool expr_entry(const ExprSeg& s, int32_t doc, unsigned long long& g) {
  if (s.hkeys) {
    unsigned long long key = 0;
    for (int k = 0; k < s.ngb; ++k) key += (unsigned long long)read_at(s.key[k], doc) * s.mult64[k];
    uint32_t h = mix64_32(key) & s.hmask;   // the scan's hash (pb200_scan.cuh): a probe starts where the insert did
    for (uint32_t probe = 0; probe <= s.hmask; ++probe) {
      const unsigned long long cur = __ldg(s.hkeys + h);
      if (cur == key) { g = h; return true; }
      if (cur == ~0ull) return false;
      h = (h + 1u) & s.hmask;
    }
    return false;
  }
  uint32_t e = 0;
  for (int k = 0; k < s.ngb; ++k) e += read_at(s.key[k], doc) * s.mult[k];
  g = e;
  return true;
}

__device__ __forceinline__ double leaf_value(const SelCol& c, int32_t doc) {
  const unsigned long long w = sel_value(c, read_at(c, doc));
  return c.kind == SEL_DICT_F32 || c.kind == SEL_DICT_F64 || c.kind == SEL_RAW_F32 ? __longlong_as_double((long long)w) : (double)(long long)w;
}

// bit k: condition k holds for `doc`
__device__ __forceinline__ uint32_t cond_word(const CondSeg& cs, const uint32_t* __restrict__ bits, int32_t doc) {
  uint32_t w = 0;
  for (int c = 0; c < cs.ncc; ++c) {
    const uint32_t id = read_at(cs.ccol[c], doc);
    for (int k = cs.first[c]; k < cs.first[c + 1]; ++k) {
      const bool hit = cs.kind[k] == PB200_COND_RANGE ? id >= (uint32_t)cs.lo[k] && id < cs.hi[k]
                                                     : ((__ldg(bits + cs.lo[k] + (id >> 5)) >> (id & 31)) & 1u) != 0u;
      w |= (uint32_t)hit << cs.slot[k];
    }
  }
  return w;
}

__device__ __forceinline__ bool is_sum(int fn) { return fn == PB200_AGG_SUM || fn == PB200_AGG_AVG; }
__device__ __forceinline__ unsigned long long key_of(double r) { return transform_key(TK_DOUBLE, 0, r); }
__device__ __forceinline__ unsigned long long key_pick(int fn, unsigned long long a, unsigned long long b) {
  return fn == PB200_AGG_MIN ? (a < b ? a : b) : (a > b ? a : b);
}

// grid: (blocks per segment, segments); one warp per 32-doc mask word at a time.  GB: group-by, COND: programs with
// conditions (csegs: one CondSeg per segment, bits: the call's bitsets).  One instantiation each, so that none carries
// another's live state.
template <bool GB, bool COND>
__global__ void __launch_bounds__(kExprThreads) expr_kernel(const ExprSeg* __restrict__ segs, const ExprProg* __restrict__ gprog,
                                                            const CondSeg* __restrict__ csegs, const uint32_t* __restrict__ bits) {
  constexpr bool group_by = GB;
  __shared__ ExprProg prog;
  __shared__ double red_s[kExprThreads / 32][kMaxAggs];
  __shared__ unsigned long long red_k[kExprThreads / 32][kMaxAggs];
  __shared__ std::conditional_t<COND, CondSeg, int> cs;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(gprog);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&prog);
    for (int i = threadIdx.x; i < (int)(sizeof(ExprProg) / 4); i += blockDim.x) dst[i] = src[i];
    if constexpr (COND) {
      const uint32_t* csrc = reinterpret_cast<const uint32_t*>(csegs + blockIdx.y);
      uint32_t* cdst = reinterpret_cast<uint32_t*>(&cs);
      for (int i = threadIdx.x; i < (int)(sizeof(CondSeg) / 4); i += blockDim.x) cdst[i] = csrc[i];
    }
  }
  __syncthreads();
  const ExprSeg& s = segs[blockIdx.y];
  const int nx = prog.nx, lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long nwords = (s.num_docs + 31) / 32;
  const long long nwarps = (long long)gridDim.x * (kExprThreads / 32);
  double acc_s[kMaxAggs];
  unsigned long long acc_k[kMaxAggs];
#pragma unroll
  for (int x = 0; x < kMaxAggs; ++x) { acc_s[x] = 0.0; acc_k[x] = x < nx && prog.fn[x] == PB200_AGG_MIN ? kExprMinEmpty : kExprMaxEmpty; }
  double v[kExprMaxCols];
  for (long long w = (long long)blockIdx.x * (kExprThreads / 32) + wib; w < nwords; w += nwarps) {
    const uint32_t m = s.mask ? __ldg(s.mask + w) : ~0u;
    const int32_t doc = (int32_t)(32 * w + lane);
    unsigned long long g = 0;
    const bool ok = ((m >> lane) & 1u) && doc < s.num_docs && (!group_by || expr_entry(s, doc, g));
    const unsigned active = __ballot_sync(0xFFFFFFFFu, ok);
    if (active == 0u) continue;
    if (ok)
      for (int c = 0; c < s.ncols; ++c) v[c] = leaf_value(s.col[c], doc);
    uint32_t cw = 0;
    if constexpr (COND)
      if (ok) cw = cond_word(cs, bits, doc);
    if (!group_by) {
#pragma unroll
      for (int x = 0; x < kMaxAggs; ++x) {
        if (x >= nx || !ok) continue;
        const double r = expr_eval<COND>(prog.ops[x], prog.len[x], v, cw);
        if (is_sum(prog.fn[x])) acc_s[x] = t_add(acc_s[x], r);
        else acc_k[x] = key_pick(prog.fn[x], acc_k[x], key_of(r));
      }
      continue;
    }
    // lanes with one entry are peers; lanes without a row group under ~0, which no entry index equals
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, ok ? g : ~0ull);
    const bool uniform = __all_sync(0xFFFFFFFFu, !ok || peers == active);
    const int leader = __ffs(ok ? peers : active) - 1;
    for (int x = 0; x < nx; ++x) {
      const int fn = prog.fn[x];
      const double r = ok ? expr_eval<COND>(prog.ops[x], prog.len[x], v, cw) : 0.0;
      if (is_sum(fn)) {
        double t = ok ? r : 0.0;
        if (uniform) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) t = t_add(t, __shfl_xor_sync(0xFFFFFFFFu, t, o));
        } else {
          double acc = t;
          for (unsigned q = active; q; q &= q - 1u) {
            const int j = __ffs(q) - 1;
            const double tj = __shfl_sync(0xFFFFFFFFu, t, j);
            if (ok && lane == leader && j != lane && ((peers >> j) & 1u)) acc = t_add(acc, tj);
          }
          t = acc;
        }
        if (ok && lane == leader) atomicAdd(static_cast<double*>(s.out[x]) + g, t);
      } else {
        const unsigned long long idle = fn == PB200_AGG_MIN ? kExprMinEmpty : kExprMaxEmpty;
        unsigned long long k = ok ? key_of(r) : idle;
        if (uniform) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) k = key_pick(fn, k, __shfl_xor_sync(0xFFFFFFFFu, k, o));
        } else {
          unsigned long long acc = k;
          for (unsigned q = active; q; q &= q - 1u) {
            const int j = __ffs(q) - 1;
            const unsigned long long kj = __shfl_sync(0xFFFFFFFFu, k, j);
            if (((peers >> j) & 1u) && ok) acc = key_pick(fn, acc, kj);
          }
          k = acc;
        }
        if (ok && lane == leader) {
          unsigned long long* p = static_cast<unsigned long long*>(s.out[x]) + g;
          if (fn == PB200_AGG_MIN) atomicMin(p, k); else atomicMax(p, k);
        }
      }
    }
  }
  if constexpr (!GB) {   // aggregation only: warp, then block, then one atomic per block and expression
#pragma unroll
    for (int x = 0; x < kMaxAggs; ++x) {
      if (x >= nx) break;
      const int fn = prog.fn[x];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        if (is_sum(fn)) acc_s[x] = t_add(acc_s[x], __shfl_xor_sync(0xFFFFFFFFu, acc_s[x], o));
        else acc_k[x] = key_pick(fn, acc_k[x], __shfl_xor_sync(0xFFFFFFFFu, acc_k[x], o));
      }
      if (lane == 0) { red_s[wib][x] = acc_s[x]; red_k[wib][x] = acc_k[x]; }
    }
    __syncthreads();
    if (threadIdx.x < nx) {
      const int x = threadIdx.x, fn = prog.fn[x];
      if (is_sum(fn)) {
        double t = 0.0;
        for (int w = 0; w < kExprThreads / 32; ++w) t = t_add(t, red_s[w][x]);
        atomicAdd(static_cast<double*>(s.out[x]), t);
      } else {
        unsigned long long k = red_k[0][x];
        for (int w = 1; w < kExprThreads / 32; ++w) k = key_pick(fn, k, red_k[w][x]);
        unsigned long long* p = static_cast<unsigned long long*>(s.out[x]);
        if (fn == PB200_AGG_MIN) atomicMin(p, k); else atomicMax(p, k);
      }
    }
  }
}

// ---- predicates on expressions (DESIGN.md section 3.16): the doc-mask pass ----
struct MaskJob {                    // one (predicate, segment)
  uint32_t* mask;                   // doc_mask_words(num_docs) words
  long long num_docs, words;
  int32_t ncols, pad;
  SelCol col[kExprMaxLeaves];       // the predicate's distinct leaf columns in this segment
};
struct MaskPred {
  int32_t len, op, flags, nvalues;
  long long voff;                   // first value in the call's value array
  double lo, hi;
  pb200_transform_op ops[kTransformMaxProgram];
};

// grid: (blocks per job, jobs); jobs are predicate-major, so block row y is predicate y / nseg.  One warp per 32-doc word:
// each lane evaluates its doc, the ballot is the word, lane 0 stores it.  Every word of the padded mask is written.
__global__ void __launch_bounds__(kExprThreads) expr_mask_kernel(const MaskJob* __restrict__ jobs, const MaskPred* __restrict__ preds,
                                                                const double* __restrict__ values, int nseg) {
  extern __shared__ double vals[];
  __shared__ MaskPred p;
  const MaskJob& j = jobs[blockIdx.y];
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(preds + blockIdx.y / nseg);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&p);
    for (int i = threadIdx.x; i < (int)(sizeof(MaskPred) / 4); i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < p.nvalues; i += blockDim.x) vals[i] = values[p.voff + i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * (kExprThreads / 32);
  double v[kExprMaxLeaves];
  for (long long w = (long long)blockIdx.x * (kExprThreads / 32) + (threadIdx.x >> 5); w < j.words; w += nwarps) {
    const long long doc = 32 * w + lane;
    bool hit = false;
    if (doc < j.num_docs) {
      for (int c = 0; c < j.ncols; ++c) v[c] = leaf_value(j.col[c], (int32_t)doc);
      hit = expr_matches(p.op, p.flags, p.lo, p.hi, vals, p.nvalues, expr_eval(p.ops, p.len, v));
    }
    const unsigned word = __ballot_sync(0xFFFFFFFFu, hit);
    if (lane == 0) j.mask[w] = word;
  }
}

// how the pass reads a leaf column: selection's rule, STRING excluded (-1: not readable as a number)
int leaf_kind(const DeviceColumn& dc) { return dc.stored_type == PB200_STRING ? -1 : selection_kind(dc); }

// Points the leaves of `mask_plan` at the buffers `scan_plan` bound for the same leaves; false (nothing changed) unless
// every buffer has its twin: same segment, leaf, kind, size and contents (LUT words, caller's source, posting lists).
bool reuse_leaf_buffers(const ScanPlan& scan_plan, ScanPlan& mask_plan) {
  std::vector<const LeafBuffer*> twin;
  for (const LeafBuffer& b : mask_plan.leaf_buffers) {
    const LeafBuffer* t = nullptr;
    for (const LeafBuffer& c : scan_plan.leaf_buffers) {
      if (c.seg != b.seg || c.leaf != b.leaf || c.kind != b.kind || c.words != b.words || c.lut != b.lut || c.src != b.src ||
          c.src_words != b.src_words || c.jobs.size() != b.jobs.size())
        continue;
      bool same = true;
      for (size_t k = 0; k < b.jobs.size() && same; k++)
        same = c.jobs[k].inv == b.jobs[k].inv && c.jobs[k].offset == b.jobs[k].offset && c.jobs[k].length == b.jobs[k].length;
      if (same) { t = &c; break; }
    }
    if (!t) return false;
    twin.push_back(t);
  }
  for (size_t k = 0; k < twin.size(); k++) {
    const LeafBuffer& b = mask_plan.leaf_buffers[k];
    const LeafDesc& from = scan_plan.segs[b.seg].leaves[b.leaf];
    LeafDesc& to = mask_plan.segs[b.seg].leaves[b.leaf];
    to.bits = from.bits;
    to.ranges = from.ranges;
  }
  return true;
}

// Checks the condition table of pb200_execute_exprs_cond against the segments and collects its distinct columns
int cond_prepare(const pb200_expr_conds& t, pb200_segment* const* segments, int nseg, int ncols, std::vector<int>& ccols) {
  if (t.reserved != 0 || t.num_conds < 1 || t.num_conds > PB200_MAX_EXPR_CONDS || !t.conds || t.num_words < 0 || (t.num_words > 0 && !t.words)) {
    set_error("malformed condition table"); return PB200_E_INVALID;
  }
  for (int k = 0; k < t.num_conds; k++) {
    const pb200_expr_cond& c = t.conds[k];
    if (c.column < 0 || c.column >= ncols) { set_error("condition %d: column %d out of range", k, c.column); return PB200_E_INVALID; }
    if ((c.kind != PB200_COND_RANGE && c.kind != PB200_COND_BITSET) || !c.args) { set_error("condition %d: malformed", k); return PB200_E_INVALID; }
    for (int s = 0; s < nseg; s++) {
      const DeviceColumn& dc = segments[s]->cols[c.column];
      const int kind = selection_kind(dc);
      if (kind < 0 || kind == SEL_RAW_I32 || kind == SEL_RAW_F32) { set_error("condition %d: column %d of segment %d has no dictIds", k, c.column, s); return PB200_E_UNSUPPORTED; }
      const long long a = c.args[2 * s], b = c.args[2 * s + 1];
      const bool ok = c.kind == PB200_COND_RANGE ? 0 <= a && a <= b && b <= dc.cardinality
                                                 : a >= 0 && b >= ((long long)dc.cardinality + 31) / 32 && b <= t.num_words - a;
      if (!ok) { set_error("condition %d: %s outside segment %d's dictIds or the bitset words", k, c.kind == PB200_COND_RANGE ? "range" : "bitset", s); return PB200_E_INVALID; }
    }
    if (std::find(ccols.begin(), ccols.end(), c.column) == ccols.end()) ccols.push_back(c.column);
  }
  return PB200_OK;
}

}  // namespace

int expr_prepare(const pb200_query* query, const pb200_expr_program* exprs, const pb200_expr_conds* conds, pb200_segment* const* segments,
                 int nseg, ExprCall* out) {
  ExprCall& x = *out;
  x = ExprCall();
  if (!query || !segments || nseg <= 0 || query->num_aggs < 0 || query->num_aggs > kMaxAggs || (query->num_aggs > 0 && !query->aggs)) {
    set_error("invalid argument to pb200_execute_exprs"); return PB200_E_INVALID;
  }
  const int ncols = common_columns(segments, nseg);
  if (ncols < 0) { set_error("segments do not share their registered columns"); return PB200_E_INVALID; }
  if (conds) {
    if (int rc = cond_prepare(*conds, segments, nseg, ncols, x.ccols)) return rc;
    x.conds = conds;
  }
  for (int a = 0; a < query->num_aggs; a++) {
    const pb200_expr_program& e = exprs[a];
    if (e.num_ops == 0) continue;
    if (e.num_ops < 0 || !e.ops || e.reserved != 0) { set_error("aggregation %d: malformed expression program", a); return PB200_E_INVALID; }
    const char* why = "";
    int leaves = 0;
    if (int rc = expr_check(e.ops, e.num_ops, &leaves, &why, conds ? conds->num_conds : 0)) { set_error("aggregation %d: %s", a, why); return rc; }
    const int fn = query->aggs[a].function;
    if (fn == PB200_AGG_COUNT) continue;   // COUNT(expr) is COUNT(*)
    if (fn != PB200_AGG_SUM && fn != PB200_AGG_AVG && fn != PB200_AGG_MIN && fn != PB200_AGG_MAX) {
      set_error("aggregation %d: only SUM, AVG, MIN, MAX and COUNT take an expression over several columns", a); return PB200_E_UNSUPPORTED;
    }
    std::vector<pb200_transform_op> ops(e.ops, e.ops + e.num_ops);
    for (pb200_transform_op& o : ops) {
      if (o.op != PB200_T_COLUMN) continue;
      if (o.i >= ncols) { set_error("aggregation %d: column %lld out of range", a, (long long)o.i); return PB200_E_INVALID; }
      const int c = (int)o.i;
      for (int s = 0; s < nseg; s++) {
        const DeviceColumn& dc = segments[s]->cols[c];
        if (dc.stored_type == PB200_STRING) { set_error("aggregation %d: STRING column %d in an arithmetic expression", a, c); return PB200_E_UNSUPPORTED; }
        if (leaf_kind(dc) < 0) { set_error("aggregation %d: column %d of segment %d has no device dictionary or raw 32-bit values", a, c, s); return PB200_E_UNSUPPORTED; }
      }
      const auto at = std::find(x.cols.begin(), x.cols.end(), c);
      o.i = at - x.cols.begin();
      if (at == x.cols.end()) x.cols.push_back(c);
    }
    x.fn_of[a] = fn;
    x.ops[a] = std::move(ops);
    x.count++;
  }
  if (x.count && query->num_group_by > 0 && ((query->flags & PB200_Q_DEFER_FINALIZE) || query->reduce_world > 1)) {
    set_error("expression aggregations with GROUP BY are not combined across GPUs or finalized later");
    return PB200_E_UNSUPPORTED;
  }
  if (x.count && nseg > kMaxSelectSegments) { set_error("expression aggregations over %d segments: at most %d per submission", nseg, kMaxSelectSegments); return PB200_E_UNSUPPORTED; }
  return PB200_OK;
}

int expr_launch(pb200_ctx* ctx, cudaStream_t st, const Tuning& tune, const pb200_query* filter_query, pb200_segment* const* segments,
                int nseg, const ScanPlan& plan, const ExprCall& x, const std::vector<ExprOut>& outs,
                std::vector<std::unique_ptr<DevBufRaw>>& temps) {
  if (!x.count) return PB200_OK;
  auto temp = [&](size_t bytes) -> void* {
    temps.emplace_back(new DevBufRaw(ctx));
    return temps.back()->alloc(bytes) == PB200_OK ? temps.back()->p : nullptr;
  };
  // 1. the match mask: the query's filter, scanned once with the mask output on (none when it matches every doc)
  std::vector<const uint32_t*> masks(nseg, nullptr);
  if (plan.q.num_nodes > 0) {
    pb200_selection sel;
    memset(&sel, 0, sizeof sel);
    SelectionPlan sp;
    if (int rc = plan_selection(tune, DeviceLimits{ctx->sm_count, ctx->max_smem_optin}, filter_query, &sel, segments, nseg, false, &sp)) return rc;
    // the filter's leaf buffers are the ones the query's scan bound (same filter, same leaves): reusing them queues no
    // upload or posting-list decode a second time, and takes none of bind_leaf_buffers' synchronisations
    if (!reuse_leaf_buffers(plan, sp.scan))
      if (int rc = bind_leaf_buffers(ctx, sp.scan, st, temps)) return rc;
    AggAccum* accum = static_cast<AggAccum*>(temp(sizeof(AggAccum) * nseg));
    uint32_t* mask = static_cast<uint32_t*>(temp(std::max<long long>(sp.mask_words, 1) * 4));
    if (!accum || !mask) return PB200_E_CUDA;
    PB200_CUDA(cudaMemsetAsync(accum, 0, sizeof(AggAccum) * nseg, st));
    for (int s = 0; s < nseg; s++) sp.scan.segs[s].accum = accum + s;
    temps.emplace_back(new DevBufRaw(ctx));
    DevBufRaw& dsegs = *temps.back();
    EventPair ev(ctx);
    if (int rc = launch_chunks(ctx, st, sp.scan, dsegs, ev, "expression mask scan", mask, sp.chunk_word_off.data(), nullptr)) return rc;
    for (int s = 0; s < nseg; s++) masks[s] = mask + sp.mask_word_off[s];
  }
  // 2. the expression pass
  ExprProg prog;
  memset(&prog, 0, sizeof prog);
  for (int a = 0; a < kMaxAggs; a++) {
    if (x.fn_of[a] < 0) continue;
    const int k = prog.nx++;
    prog.fn[k] = x.fn_of[a];
    prog.len[k] = (int)x.ops[a].size();
    std::copy(x.ops[a].begin(), x.ops[a].end(), prog.ops[k]);
  }
  std::vector<ExprSeg> es(nseg);
  long long max_words = 1;
  for (int s = 0; s < nseg; s++) {
    ExprSeg& e = es[s];
    memset(&e, 0, sizeof e);
    const pb200_segment& seg = *segments[s];
    const SegDesc& sd = plan.segs[s];
    const int r = plan.merge ? 0 : s;
    e.mask = masks[s];
    e.num_docs = seg.num_docs;
    e.ncols = (int)x.cols.size();
    for (int c = 0; c < e.ncols; c++) {
      const DeviceColumn& dc = seg.cols[x.cols[c]];
      e.col[c] = SelCol{dc.fwd, dc.dict_native, dc.bits, leaf_kind(dc), 0, 0};
    }
    if (plan.group_by) {
      e.ngb = plan.q.num_group_by;
      for (int g = 0; g < e.ngb; g++) {
        const DeviceColumn& dc = seg.cols[filter_query->group_by_columns[g]];
        e.key[g] = SelCol{dc.fwd, nullptr, dc.bits, SEL_DICT_ID, 0, 0};
        e.mult[g] = sd.group_mult[g];
        e.mult64[g] = sd.group_mult64[g];
      }
      e.hkeys = outs[r].hkeys;
      e.hmask = sd.h_mask;
    }
    for (int k = 0, a = 0; a < kMaxAggs; a++) if (x.fn_of[a] >= 0) e.out[k++] = outs[r].out[a];
    max_words = std::max(max_words, (e.num_docs + 31) / 32);
  }
  ExprSeg* dsegs = static_cast<ExprSeg*>(temp(sizeof(ExprSeg) * nseg));
  ExprProg* dprog = static_cast<ExprProg*>(temp(sizeof(ExprProg)));
  if (!dsegs || !dprog) return PB200_E_CUDA;
  PB200_CUDA(cudaMemcpyAsync(dsegs, es.data(), sizeof(ExprSeg) * nseg, cudaMemcpyHostToDevice, st));
  PB200_CUDA(cudaMemcpyAsync(dprog, &prog, sizeof prog, cudaMemcpyHostToDevice, st));
  const long long per_seg = std::max<long long>(1, (long long)ctx->sm_count * 8 / nseg);
  const dim3 grid((unsigned)std::min<long long>((max_words + kExprThreads / 32 - 1) / (kExprThreads / 32), std::max<long long>(per_seg, 2)), (unsigned)nseg);
  if (!x.conds) {
    if (plan.group_by) expr_kernel<true, false><<<grid, kExprThreads, 0, st>>>(dsegs, dprog, nullptr, nullptr);
    else expr_kernel<false, false><<<grid, kExprThreads, 0, st>>>(dsegs, dprog, nullptr, nullptr);
    PB200_CUDA(cudaGetLastError());
    return PB200_OK;
  }
  // the conditions: per segment grouped by column, and the call's bitsets in one buffer
  const pb200_expr_conds& t = *x.conds;
  std::vector<CondSeg> cseg(nseg);
  for (int s = 0; s < nseg; s++) {
    CondSeg& c = cseg[s];
    memset(&c, 0, sizeof c);
    c.ncc = (int)x.ccols.size();
    int n = 0;
    for (int j = 0; j < c.ncc; j++) {
      const DeviceColumn& dc = segments[s]->cols[x.ccols[j]];
      c.ccol[j] = SelCol{dc.fwd, nullptr, dc.bits, SEL_DICT_ID, 0, 0};
      c.first[j] = n;
      for (int k = 0; k < t.num_conds; k++) {
        if (t.conds[k].column != x.ccols[j]) continue;
        c.kind[n] = t.conds[k].kind;
        c.slot[n] = k;
        c.lo[n] = t.conds[k].args[2 * s];
        c.hi[n] = t.conds[k].kind == PB200_COND_RANGE ? (uint32_t)t.conds[k].args[2 * s + 1] : 0u;
        n++;
      }
    }
    c.first[c.ncc] = n;
  }
  CondSeg* dcond = static_cast<CondSeg*>(temp(sizeof(CondSeg) * nseg));
  uint32_t* dbits = static_cast<uint32_t*>(temp(std::max<size_t>((size_t)t.num_words, 1) * 4));
  if (!dcond || !dbits) return PB200_E_CUDA;
  PB200_CUDA(cudaMemcpyAsync(dcond, cseg.data(), sizeof(CondSeg) * nseg, cudaMemcpyHostToDevice, st));
  if (t.num_words > 0) PB200_CUDA(cudaMemcpyAsync(dbits, t.words, (size_t)t.num_words * 4, cudaMemcpyHostToDevice, st));
  if (plan.group_by) expr_kernel<true, true><<<grid, kExprThreads, 0, st>>>(dsegs, dprog, dcond, dbits);
  else expr_kernel<false, true><<<grid, kExprThreads, 0, st>>>(dsegs, dprog, dcond, dbits);
  PB200_CUDA(cudaGetLastError());
  return PB200_OK;
}

}  // namespace pb200

// ---- pb200_expr_doc_masks --------------------------------------------------------------------------------------------
namespace pb200 {
namespace {

// Checks the predicates and fills the pass's descriptors (no CUDA call); PB200_OK or the code of pb200_expr_doc_masks
int mask_prepare(const pb200_expr_predicate* preds, int n, pb200_segment* const* segments, int nseg, std::vector<MaskPred>& mp,
                 std::vector<MaskJob>& jobs, std::vector<double>& values) {
  const int ncols = common_columns(segments, nseg);
  if (ncols < 0) { set_error("segments do not share their registered columns"); return PB200_E_INVALID; }
  if ((long long)n * nseg > kMaxSelectSegments) { set_error("%d predicates over %d segments: at most %d per call", n, nseg, kMaxSelectSegments); return PB200_E_UNSUPPORTED; }
  mp.assign(n, MaskPred());
  jobs.assign((size_t)n * nseg, MaskJob());
  for (int p = 0; p < n; p++) {
    const pb200_expr_predicate& e = preds[p];
    if (e.reserved != 0 || e.program.reserved != 0 || e.program.num_ops <= 0 || !e.program.ops) { set_error("predicate %d: malformed expression program", p); return PB200_E_INVALID; }
    const char* why = "";
    int leaves = 0;
    if (int rc = expr_check(e.program.ops, e.program.num_ops, &leaves, &why)) { set_error("predicate %d: %s", p, why); return rc; }
    if (e.op < PB200_EXPR_EQ || e.op > PB200_EXPR_RANGE) { set_error("predicate %d: unknown op %d", p, e.op); return PB200_E_INVALID; }
    if (e.op == PB200_EXPR_RANGE ? (e.flags & ~15) != 0 || e.num_values != 0 : e.flags != 0) { set_error("predicate %d: bad flags or values for its op", p); return PB200_E_INVALID; }
    if (e.op != PB200_EXPR_RANGE) {
      const bool one = e.op == PB200_EXPR_EQ || e.op == PB200_EXPR_NEQ;
      if (e.num_values < 1 || (one && e.num_values != 1) || !e.values) { set_error("predicate %d: %d values", p, e.num_values); return PB200_E_INVALID; }
      if (e.num_values > PB200_MAX_EXPR_VALUES) { set_error("predicate %d: %d values (at most %d)", p, e.num_values, PB200_MAX_EXPR_VALUES); return PB200_E_UNSUPPORTED; }
    }
    MaskPred& m = mp[p];
    memset(&m, 0, sizeof m);
    m.len = e.program.num_ops; m.op = e.op; m.flags = e.flags; m.lo = e.lo; m.hi = e.hi;
    m.nvalues = e.op == PB200_EXPR_RANGE ? 0 : e.num_values;
    m.voff = (long long)values.size();
    values.insert(values.end(), e.values, e.values + m.nvalues);
    std::vector<int> cols;   // distinct leaf columns: program leaf i reads cols[i]
    for (int k = 0; k < m.len; k++) {
      pb200_transform_op o = e.program.ops[k];
      if (o.op == PB200_T_COLUMN) {
        if (o.i >= ncols) { set_error("predicate %d: column %lld out of range", p, (long long)o.i); return PB200_E_INVALID; }
        const int c = (int)o.i;
        for (int s = 0; s < nseg; s++) {
          const DeviceColumn& dc = segments[s]->cols[c];
          if (dc.stored_type == PB200_STRING) { set_error("predicate %d: STRING column %d in an arithmetic expression", p, c); return PB200_E_UNSUPPORTED; }
          if (leaf_kind(dc) < 0) { set_error("predicate %d: column %d of segment %d has no device dictionary or raw 32-bit values", p, c, s); return PB200_E_UNSUPPORTED; }
        }
        const auto at = std::find(cols.begin(), cols.end(), c);
        o.i = at - cols.begin();
        if (at == cols.end()) cols.push_back(c);
      }
      m.ops[k] = o;
    }
    for (int s = 0; s < nseg; s++) {
      MaskJob& j = jobs[(size_t)p * nseg + s];
      memset(&j, 0, sizeof j);
      j.num_docs = segments[s]->num_docs;
      j.words = (long long)doc_mask_words(j.num_docs);
      j.ncols = (int)cols.size();
      for (int c = 0; c < j.ncols; c++) {
        const DeviceColumn& dc = segments[s]->cols[cols[c]];
        j.col[c] = SelCol{dc.fwd, dc.dict_native, dc.bits, leaf_kind(dc), 0, 0};
      }
    }
  }
  return PB200_OK;
}

int mask_launch(pb200_ctx* ctx, int nseg, const std::vector<MaskPred>& mp, std::vector<MaskJob>& jobs,
                const std::vector<double>& values, std::vector<uint32_t*>& out) {
  PB200_CUDA(cudaSetDevice(ctx->device));
  long long max_words = 1;
  int max_values = 0;
  for (size_t k = 0; k < jobs.size(); k++) {
    void* p = nullptr;
    if (int rc = dev_alloc(ctx, (size_t)jobs[k].words * 4, &p)) return rc;
    out[k] = jobs[k].mask = static_cast<uint32_t*>(p);
    max_words = std::max(max_words, jobs[k].words);
  }
  for (const MaskPred& m : mp) max_values = std::max(max_values, m.nvalues);
  StreamLease st(ctx);
  DevBufRaw djobs(ctx), dpreds(ctx), dvals(ctx);
  if (int rc = djobs.alloc(sizeof(MaskJob) * jobs.size())) return rc;
  if (int rc = dpreds.alloc(sizeof(MaskPred) * mp.size())) return rc;
  if (int rc = dvals.alloc(std::max<size_t>(values.size(), 1) * sizeof(double))) return rc;
  PB200_CUDA(cudaMemcpyAsync(djobs.p, jobs.data(), sizeof(MaskJob) * jobs.size(), cudaMemcpyHostToDevice, st));
  PB200_CUDA(cudaMemcpyAsync(dpreds.p, mp.data(), sizeof(MaskPred) * mp.size(), cudaMemcpyHostToDevice, st));
  if (!values.empty()) PB200_CUDA(cudaMemcpyAsync(dvals.p, values.data(), values.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  const long long per_job = std::max<long long>(2, (long long)ctx->sm_count * 8 / (long long)jobs.size());
  const dim3 grid((unsigned)std::min<long long>((max_words + kExprThreads / 32 - 1) / (kExprThreads / 32), per_job), (unsigned)jobs.size());
  expr_mask_kernel<<<grid, kExprThreads, (size_t)max_values * sizeof(double), st>>>(
      static_cast<const MaskJob*>(djobs.p), static_cast<const MaskPred*>(dpreds.p), static_cast<const double*>(dvals.p), nseg);
  PB200_CUDA(cudaGetLastError());
  PB200_CUDA(cudaStreamSynchronize(st));   // once: the masks are complete for any stream that reads them
  return PB200_OK;
}

}  // namespace
}  // namespace pb200

extern "C" int32_t pb200_expr_doc_masks(pb200_ctx* ctx, int32_t n, const pb200_expr_predicate* preds, pb200_segment* const* segments,
                                        int32_t nseg, uint32_t** masks) {
  using namespace pb200;
  if (!ctx || n < 0 || (n > 0 && !preds) || !segments || nseg <= 0 || !masks) { set_error("invalid argument to pb200_expr_doc_masks"); return PB200_E_INVALID; }
  for (int s = 0; s < nseg; s++) if (!segments[s]) { set_error("invalid argument to pb200_expr_doc_masks"); return PB200_E_INVALID; }
  if (n == 0) return PB200_OK;
  std::vector<MaskPred> mp;
  std::vector<MaskJob> jobs;
  std::vector<double> values;
  if (int rc = mask_prepare(preds, n, segments, nseg, mp, jobs, values)) return rc;
  std::vector<uint32_t*> out(jobs.size(), nullptr);
  if (int rc = mask_launch(ctx, nseg, mp, jobs, values, out)) {
    for (uint32_t* m : out) if (m) dev_free(ctx, m);
    return rc;
  }
  std::copy(out.begin(), out.end(), masks);
  return PB200_OK;
}
