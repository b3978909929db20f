// pb200_distinct.cu -- DISTINCT queries: SELECT DISTINCT columns WHERE ... [ORDER BY columns] LIMIT n (the reference's
// DistinctOperator).
//
// The filter is the selection scan (run_selection_scan, pb200_select.cu): a COUNT(*) launch that leaves every segment's
// match mask.  Then:
//   build: one dense u64 first-occurrence table per result over the raw key space (raw key = sum_k dictId_k x mult_k, the
//     group-by key composition), entry = segment << 32 | doc of the key's first matching doc, empty = ~0.  A warp owns a
//     1024-row slice (lane l: mask word 32 x slice + l) and skips it when all 32 words are zero; otherwise each lane
//     unpacks the B words of every key column for its 32 docs (the read32 group layout, pb200_unpack.cuh) and walks its
//     docs in order.  Per doc position the lanes holding equal keys are found with __match_any_sync; the lowest lane (the
//     lowest doc) reads the entry and issues a 64-bit atomicMin only when the entry is larger.  Entries only decrease, so
//     a stale read can only cost an atomic, never skip a needed one.
//   prefix-final rule (no ORDER BY): segments are first scanned over plan_selection's prefix.  The earliest truncated
//     segment s of a result bounds what has been scanned: every position (segment, doc) below (s, prefix end) has been.
//     If at least LIMIT entries of the result's table lie below that bound, no unscanned doc can hold one of the first
//     LIMIT tuples or lower one of their first occurrences: the result is final.  Otherwise its truncated segments are
//     scanned in full and built into the SAME table (a minimum over a superset of docs: no reset needed).
//   extraction: compaction of the present entries (cub::DeviceSelect), one stable radix sort by first occurrence (segment,
//     doc: this also groups per-segment results), with ORDER BY then one stable pass per order item from the last to the
//     first (key: the item's dictId decoded from the raw key, reversed for DESC) and one by result; the first LIMIT of
//     each result are gathered with selection's value decode (sel_value) into selection's output block layout, so
//     pb200_result_selection reads DISTINCT results unchanged.
//
// Stream synchronisations per call: after each scan and after each table build (once more for a rescan), after the
// prefix count (when a segment was truncated), after compaction (the counts size the output), after the gather.  device_ms = the scan launches
// and the table builds (CUDA events).  pb200_last_phases: PLAN, DEVICE_WAIT (scans, builds, the prefix decision),
// EXTRACT (compaction to output), TOTAL.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <vector>

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "pb200_internal.h"
#include "pb200_plan.h"
#include "pb200_select.cuh"
#include "pb200_unpack.cuh"

namespace pb200 {
namespace {

constexpr int kThreads = 256;

struct DistSeg {                     // one segment of a table build
  const uint32_t* mask;              // its match mask over the scanned range
  long long nwords;                  // words of the scanned range
  unsigned long long* table;         // its result's table
  const uint32_t* fwd[kMaxDistinctColumns];
  int32_t bits[kMaxDistinctColumns];
  uint32_t mult[kMaxDistinctColumns];
  int32_t nkeys;
  uint32_t seg;                      // index in the submission
};
struct DistKey { uint32_t mult, card; };   // one key column of one segment
struct DistRes { long long grp_off, rows, row_off; };

struct KeyAcc {                      // key[i] += dictId of doc i x mult
  uint32_t (&key)[32];
  uint32_t mult;
  int shift;
  __device__ __forceinline__ void operator()(int i, uint32_t xl) { key[i] += (xl >> shift) * mult; }
};

__global__ void __launch_bounds__(kThreads) dist_build_kernel(const DistSeg* __restrict__ segs) {
  const DistSeg& sg = segs[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const long long nslices = (sg.nwords + 31) / 32;
  const long long wpb = blockDim.x / 32;
  for (long long sl = blockIdx.x * wpb + threadIdx.x / 32; sl < nslices; sl += (long long)gridDim.x * wpb) {
    const long long w = sl * 32 + lane;
    const uint32_t m = w < sg.nwords ? __ldg(sg.mask + w) : 0u;
    if (__ballot_sync(0xFFFFFFFFu, m != 0u) == 0u) continue;   // an empty slice: the key columns are not touched
    uint32_t key[32];
#pragma unroll
    for (int i = 0; i < 32; i++) key[i] = 0u;
    if (m != 0u)
      for (int k = 0; k < sg.nkeys; k++) {
        KeyAcc f{key, sg.mult[k], 32 - sg.bits[k]};
        dispatch_left_aligned(sg.bits[k], sg.fwd[k], (int)w, f);
      }
#pragma unroll
    for (int j = 0; j < 32; j++) {
      const bool on = (m >> j) & 1u;
      const uint32_t act = __ballot_sync(0xFFFFFFFFu, on);
      if (!on) continue;
      const uint32_t peers = __match_any_sync(act, key[j]);
      if (lane == __ffs(peers) - 1) {   // the lowest doc holding this key at position j
        const unsigned long long v = (unsigned long long)sg.seg << 32 | (unsigned long long)(32 * w + j);
        unsigned long long* e = sg.table + key[j];
        if (*e > v) atomicMin(e, v);
      }
    }
  }
}

// below[r] = entries of result r's table under bound[r] (bound kDistinctEmpty: not counted)
__global__ void dist_below_kernel(const unsigned long long* __restrict__ tables, const long long* __restrict__ off,
                                  const long long* __restrict__ size, const unsigned long long* __restrict__ bound,
                                  unsigned long long* __restrict__ below) {
  const int r = blockIdx.y;
  const unsigned long long b = bound[r];
  if (b == kDistinctEmpty) return;
  unsigned long long n = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < size[r]; i += (long long)gridDim.x * blockDim.x)
    n += __ldg(tables + off[r] + i) < b;
  for (int o = 16; o; o >>= 1) n += __shfl_down_sync(0xFFFFFFFFu, n, o);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(below + r, n);
}

struct Present {
  const unsigned long long* t;
  __device__ __forceinline__ bool operator()(int i) const { return t[i] != kDistinctEmpty; }
};

// counts[r] = present entries of result r: pos (ascending positions in the table block) between off[r] and off[r]+size[r]
__global__ void dist_count_kernel(const int32_t* __restrict__ pos, const int32_t* __restrict__ npos, const long long* __restrict__ off,
                                  const long long* __restrict__ size, int nres, long long* __restrict__ counts) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nres) return;
  auto lower = [&](long long x) { int lo = 0, hi = *npos; while (lo < hi) { const int m = (lo + hi) >> 1; if (pos[m] < x) lo = m + 1; else hi = m; } return lo; };
  counts[r] = lower(off[r] + size[r]) - lower(off[r]);
}

// compacted entry i: its first occurrence, its raw key and (iota not NULL) the identity permutation
__global__ void dist_fill_kernel(const unsigned long long* __restrict__ tables, const int32_t* __restrict__ pos, long long n,
                                 const long long* __restrict__ off, bool merge, unsigned long long* __restrict__ occ,
                                 uint32_t* __restrict__ raw, int32_t* __restrict__ iota) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long o = tables[pos[i]];
    occ[i] = o;
    raw[i] = (uint32_t)(pos[i] - off[merge ? 0 : (int)(o >> 32)]);
    if (iota) iota[i] = (int32_t)i;
  }
}

// sort key of one ORDER BY pass over the current permutation: key column `key`'s dictId (DESC: card - 1 - dictId), or
// (key < 0) the result index
__global__ void dist_key_kernel(const int32_t* __restrict__ perm, const unsigned long long* __restrict__ occ,
                                const uint32_t* __restrict__ raw, long long n, const DistKey* __restrict__ keys, int nkeys,
                                int key, bool desc, bool merge, uint32_t* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int32_t c = perm[i];
    const uint32_t seg = (uint32_t)(occ[c] >> 32);
    if (key < 0) { out[i] = merge ? 0u : seg; continue; }
    const DistKey dk = keys[(size_t)seg * nkeys + key];
    const uint32_t id = raw[c] / dk.mult % dk.card;
    out[i] = desc ? dk.card - 1u - id : id;
  }
}

// output row -> compacted entry: result r's rows are the first `rows` of its sorted group
__global__ void dist_pick_kernel(const DistRes* __restrict__ res, const int32_t* __restrict__ perm, int32_t* __restrict__ pick) {
  const DistRes g = res[blockIdx.y];
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < g.rows; r += (long long)gridDim.x * blockDim.x)
    pick[g.row_off + r] = perm[g.grp_off + r];
}

// Output block (selection's layout): doc ids int32[rows], segment index int32[rows], per column 8-byte values [rows].
__global__ void dist_gather_kernel(const int32_t* __restrict__ pick, const unsigned long long* __restrict__ occ,
                                   const uint32_t* __restrict__ raw, long long rows, const SelCol* __restrict__ cols,
                                   const DistKey* __restrict__ keys, int ncols, unsigned char* __restrict__ out) {
  int32_t* odoc = reinterpret_cast<int32_t*>(out);
  int32_t* oseg = odoc + rows;
  unsigned long long* ocol = reinterpret_cast<unsigned long long*>(out + 8 * rows);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < rows; i += (long long)gridDim.x * blockDim.x) {
    const int32_t c = pick[i];
    const unsigned long long o = occ[c];
    const uint32_t s = (uint32_t)(o >> 32), key = raw[c];
    odoc[i] = (int32_t)(uint32_t)o;
    oseg[i] = (int32_t)s;
    for (int k = 0; k < ncols; k++) {
      const DistKey dk = keys[(size_t)s * ncols + k];
      ocol[(size_t)k * rows + i] = sel_value(cols[(size_t)s * ncols + k], key / dk.mult % dk.card);
    }
  }
}

int grid_for(pb200_ctx* ctx, long long items) {
  return (int)std::max<long long>(1, std::min<long long>((items + kThreads - 1) / kThreads, (long long)ctx->sm_count * 8));
}

struct EventPair {
  pb200_ctx* c; cudaEvent_t a = nullptr, b = nullptr;
  ~EventPair() { give_event(c, a); give_event(c, b); }
};

// Builds the tables from the masks of segments `ds` (one scan's worth); adds the kernels' event time to *ms.
int build_tables(pb200_ctx* ctx, cudaStream_t st, const std::vector<DistSeg>& ds, float* ms) {
  if (ds.empty()) return PB200_OK;
  long long max_words = 0;
  for (const DistSeg& d : ds) max_words = std::max(max_words, d.nwords);
  DevBufRaw dd(ctx);
  if (int rc = dd.alloc(sizeof(DistSeg) * ds.size())) return rc;
  PB200_CUDA(cudaMemcpyAsync(dd.p, ds.data(), sizeof(DistSeg) * ds.size(), cudaMemcpyHostToDevice, st));
  EventPair ev{ctx};
  ev.a = take_event(ctx);
  ev.b = take_event(ctx);
  if (!ev.a || !ev.b) { set_error("cudaEventCreate failed"); return PB200_E_CUDA; }
  PB200_CUDA(cudaEventRecord(ev.a, st));
  const dim3 grid((unsigned)grid_for(ctx, max_words), (unsigned)ds.size());
  dist_build_kernel<<<grid, kThreads, 0, st>>>(static_cast<const DistSeg*>(dd.p));
  PB200_CUDA(cudaGetLastError());
  PB200_CUDA(cudaEventRecord(ev.b, st));
  const cudaError_t se = cudaStreamSynchronize(st);   // the descriptors live until the build is done
  if (se != cudaSuccess) { set_error("DISTINCT table build failed: %s", cudaGetErrorString(se)); return PB200_E_CUDA; }
  float t = 0.f;
  cudaEventElapsedTime(&t, ev.a, ev.b);
  *ms += t;
  return PB200_OK;
}

}  // namespace
}  // namespace pb200

using namespace pb200;

extern "C" int32_t pb200_execute_distinct(pb200_ctx* ctx, const pb200_query* filter_only, const pb200_selection* distinct,
                                          pb200_segment* const* segments, int32_t nseg, int32_t flags, pb200_result** results) {
  if (!ctx || !filter_only || !distinct || !segments || !results || nseg <= 0) { set_error("invalid argument to pb200_execute_distinct"); return PB200_E_INVALID; }
  if (flags & ~PB200_Q_MERGE_SEGMENTS) { set_error("pb200_execute_distinct: flags other than PB200_Q_MERGE_SEGMENTS"); return PB200_E_INVALID; }
  for (int s = 0; s < nseg; s++)
    if (!segments[s] || segments[s]->ctx != ctx) { set_error("segment %d does not belong to this context / schema", s); return PB200_E_INVALID; }
  const double t_enter = host_ms();
  PB200_CUDA(cudaSetDevice(ctx->device));
  const Tuning tune = [&]() { std::lock_guard<std::mutex> g(ctx->mu); return ctx->tune; }();
  const DeviceLimits lim{ctx->sm_count, ctx->max_smem_optin};
  const bool merge = flags & PB200_Q_MERGE_SEGMENTS;
  DistinctPlan p;
  if (int rc = plan_distinct(tune, lim, filter_only, distinct, segments, nseg, merge, true, &p)) return rc;
  const double t_planned = host_ms();

  cudaStream_t st = take_stream(ctx);
  struct StreamReturn { pb200_ctx* c; cudaStream_t s; ~StreamReturn() { give_stream(c, s); } } stream_return{ctx, st};
  const int nres = p.nres, nkeys = (int)p.sel.columns.size();
  float ms = 0.f;
  DevBufRaw tables(ctx), mask1(ctx), mask2(ctx);
  if (int rc = tables.alloc(std::max<long long>(p.table_entries, 1) * 8)) return rc;
  unsigned long long* tb = static_cast<unsigned long long*>(tables.p);
  PB200_CUDA(cudaMemsetAsync(tb, 0xFF, (size_t)p.table_entries * 8, st));
  std::vector<long long> m1;
  if (int rc = run_selection_scan(ctx, st, p.sel, mask1, m1, &ms)) return rc;
  auto dist_seg = [&](int s, const uint32_t* mask, long long docs) {
    DistSeg d;
    memset(&d, 0, sizeof d);
    d.mask = mask;
    d.nwords = (docs + 31) / 32;
    d.table = tb + p.table_off[merge ? 0 : s];
    d.nkeys = nkeys;
    d.seg = (uint32_t)s;
    for (int k = 0; k < nkeys; k++) {
      const DeviceColumn& c = segments[s]->cols[p.sel.columns[k]];
      d.fwd[k] = c.fwd; d.bits[k] = c.bits; d.mult[k] = p.mult[s][k];
    }
    return d;
  };
  std::vector<long long> matches(m1), in_filter(p.sel.scan.in_filter);
  {
    std::vector<DistSeg> ds;
    for (int s = 0; s < nseg; s++)
      if (m1[s] > 0) ds.push_back(dist_seg(s, static_cast<const uint32_t*>(mask1.p) + p.sel.mask_word_off[s], p.sel.scan_docs[s]));
    if (int rc = build_tables(ctx, st, ds, &ms)) return rc;
  }
  if (p.sel.prefix) {
    // ---- the prefix-final rule: count the entries below each result's bound ----
    const std::vector<unsigned long long> bound = distinct_bounds(p, segments);
    DevBufRaw dmeta(ctx);
    const size_t meta_bytes = (size_t)nres * 8 * 4;
    if (int rc = dmeta.alloc(meta_bytes)) return rc;
    long long* doff = static_cast<long long*>(dmeta.p);
    long long* dsize = doff + nres;
    unsigned long long* dbound = reinterpret_cast<unsigned long long*>(dsize + nres);
    unsigned long long* dbelow = dbound + nres;
    PB200_CUDA(cudaMemcpyAsync(doff, p.table_off.data(), (size_t)nres * 8, cudaMemcpyHostToDevice, st));
    PB200_CUDA(cudaMemcpyAsync(dsize, p.table_size.data(), (size_t)nres * 8, cudaMemcpyHostToDevice, st));
    PB200_CUDA(cudaMemcpyAsync(dbound, bound.data(), (size_t)nres * 8, cudaMemcpyHostToDevice, st));
    PB200_CUDA(cudaMemsetAsync(dbelow, 0, (size_t)nres * 8, st));
    long long max_size = 0;
    for (long long z : p.table_size) max_size = std::max(max_size, z);
    dist_below_kernel<<<dim3((unsigned)grid_for(ctx, max_size), (unsigned)nres), kThreads, 0, st>>>(tb, doff, dsize, dbound, dbelow);
    PB200_CUDA(cudaGetLastError());
    std::vector<long long> below(nres);
    PB200_CUDA(cudaMemcpyAsync(below.data(), dbelow, (size_t)nres * 8, cudaMemcpyDeviceToHost, st));
    PB200_CUDA(cudaStreamSynchronize(st));
    const std::vector<int> rescan = distinct_rescan(p, segments, below);
    if (!rescan.empty()) {
      const Rescan rs = rescan_query(*filter_only, segments, rescan);
      SelectionPlan p2;
      if (int rc = plan_selection(tune, lim, &rs.query, distinct, rs.segs.data(), (int)rs.segs.size(), false, &p2)) return rc;
      std::vector<long long> m2;
      if (int rc = run_selection_scan(ctx, st, p2, mask2, m2, &ms)) return rc;
      std::vector<DistSeg> ds;
      for (size_t i = 0; i < rescan.size(); i++) {
        const int s = rescan[i];
        matches[s] = m2[i]; in_filter[s] = p2.scan.in_filter[i];
        if (m2[i] > 0) ds.push_back(dist_seg(s, static_cast<const uint32_t*>(mask2.p) + p2.mask_word_off[i], p2.scan_docs[i]));
      }
      if (int rc = build_tables(ctx, st, ds, &ms)) return rc;
    }
  }
  const double t_scanned = host_ms();

  // ---- extraction: compact, count per result ----
  const long long nent = p.table_entries;
  DevBufRaw meta(ctx), pos(ctx), tmp(ctx), work(ctx), staging(ctx), dcols(ctx), dkeys(ctx), dres(ctx);
  if (int rc = meta.alloc((size_t)nres * 8 * 3 + 8)) return rc;
  long long* doff = static_cast<long long*>(meta.p);
  long long* dsize = doff + nres;
  long long* dcount = dsize + nres;
  int32_t* dnpos = reinterpret_cast<int32_t*>(dcount + nres);
  PB200_CUDA(cudaMemcpyAsync(doff, p.table_off.data(), (size_t)nres * 8, cudaMemcpyHostToDevice, st));
  PB200_CUDA(cudaMemcpyAsync(dsize, p.table_size.data(), (size_t)nres * 8, cudaMemcpyHostToDevice, st));
  if (int rc = pos.alloc(std::max<long long>(nent, 1) * 4)) return rc;
  size_t sel_bytes = 0;
  thrust::counting_iterator<int32_t> ids(0);
  PB200_CUDA(cub::DeviceSelect::If(nullptr, sel_bytes, ids, static_cast<int32_t*>(pos.p), dnpos, (int)nent, Present{tb}, st));
  if (int rc = tmp.alloc(std::max<size_t>(sel_bytes, 1))) return rc;
  PB200_CUDA(cub::DeviceSelect::If(tmp.p, sel_bytes, ids, static_cast<int32_t*>(pos.p), dnpos, (int)nent, Present{tb}, st));
  dist_count_kernel<<<(nres + kThreads - 1) / kThreads, kThreads, 0, st>>>(static_cast<const int32_t*>(pos.p), dnpos, doff, dsize, nres, dcount);
  PB200_CUDA(cudaGetLastError());
  std::vector<long long> counts(nres);
  PB200_CUDA(cudaMemcpyAsync(counts.data(), dcount, (size_t)nres * 8, cudaMemcpyDeviceToHost, st));
  PB200_CUDA(cudaStreamSynchronize(st));

  std::vector<DistRes> res(nres);
  long long npresent = 0, total_rows = 0;
  for (int r = 0; r < nres; r++) {
    res[r].grp_off = npresent;
    res[r].rows = std::min(counts[r], p.sel.limit);
    res[r].row_off = total_rows;
    npresent += counts[r];
    total_rows += res[r].rows;
  }
  const size_t out_bytes = (size_t)total_rows * 8 * (1 + (size_t)nkeys);
  auto block = std::make_shared<PinnedBlock>();
  block->ctx = ctx;
  if (int rc = pinned_alloc(ctx, std::max<size_t>(out_bytes, 8), &block->p, &block->bytes)) return rc;
  if (total_rows > 0) {
    // ---- sort: by first occurrence (segment, doc), then ORDER BY items last to first, then the result ----
    const long long n = npresent;
    const int nitems = (int)p.order_key.size();
    int seg_bits = 0;
    while ((1 << seg_bits) < nseg) seg_bits++;
    std::vector<SelCol> sc((size_t)nseg * nkeys);
    std::vector<DistKey> dk((size_t)nseg * nkeys);
    int max_key_bits[kMaxDistinctColumns] = {};
    for (int s = 0; s < nseg; s++)
      for (int k = 0; k < nkeys; k++) {
        const DeviceColumn& c = segments[s]->cols[p.sel.columns[k]];
        sc[(size_t)s * nkeys + k] = SelCol{c.fwd, c.dict_native, c.bits, p.sel.kinds[k], 0, 0};
        dk[(size_t)s * nkeys + k] = DistKey{p.mult[s][k], (uint32_t)p.cards[s][k]};
        int b = 0;
        while (b < 32 && ((uint32_t)(p.cards[s][k] - 1) >> b)) b++;
        max_key_bits[k] = std::max(max_key_bits[k], b);
      }
    if (int rc = dcols.alloc(sizeof(SelCol) * sc.size())) return rc;
    if (int rc = dkeys.alloc(sizeof(DistKey) * dk.size())) return rc;
    if (int rc = dres.alloc(sizeof(DistRes) * nres)) return rc;
    PB200_CUDA(cudaMemcpyAsync(dcols.p, sc.data(), sizeof(SelCol) * sc.size(), cudaMemcpyHostToDevice, st));
    PB200_CUDA(cudaMemcpyAsync(dkeys.p, dk.data(), sizeof(DistKey) * dk.size(), cudaMemcpyHostToDevice, st));
    PB200_CUDA(cudaMemcpyAsync(dres.p, res.data(), sizeof(DistRes) * nres, cudaMemcpyHostToDevice, st));
    // work: occ 2 x n u64, raw n u32, keys 2 x n u32, perm 2 x n i32, pick total_rows i32
    if (int rc = work.alloc((size_t)n * 16 + (size_t)n * 4 * 5 + (size_t)total_rows * 4)) return rc;
    unsigned long long* occ0 = static_cast<unsigned long long*>(work.p);
    unsigned long long* occ1 = occ0 + n;
    uint32_t* raw = reinterpret_cast<uint32_t*>(occ1 + n);
    uint32_t* k0 = raw + n;
    uint32_t* k1 = k0 + n;
    int32_t* v0 = reinterpret_cast<int32_t*>(k1 + n);
    int32_t* v1 = v0 + n;
    int32_t* pick = v1 + n;
    const int cgrid = grid_for(ctx, n);
    dist_fill_kernel<<<cgrid, kThreads, 0, st>>>(tb, static_cast<const int32_t*>(pos.p), n, doff, merge, occ0, raw, v0);
    PB200_CUDA(cudaGetLastError());
    size_t sort_bytes = 0, key_bytes = 0;
    cub::DoubleBuffer<unsigned long long> ob(occ0, occ1);
    cub::DoubleBuffer<uint32_t> kb(k0, k1);
    cub::DoubleBuffer<int32_t> vb(v0, v1);
    PB200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, ob, vb, (int)n, 0, 32 + seg_bits, st));
    if (nitems > 0) PB200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, key_bytes, kb, vb, (int)n, 0, 32, st));
    DevBufRaw stmp(ctx);
    if (int rc = stmp.alloc(std::max<size_t>(std::max(sort_bytes, key_bytes), 1))) return rc;
    PB200_CUDA(cub::DeviceRadixSort::SortPairs(stmp.p, sort_bytes, ob, vb, (int)n, 0, 32 + seg_bits, st));
    // the sort reused both occurrence buffers: the permutation indexes the compacted order, filled in again
    dist_fill_kernel<<<cgrid, kThreads, 0, st>>>(tb, static_cast<const int32_t*>(pos.p), n, doff, merge, occ0, raw, nullptr);
    PB200_CUDA(cudaGetLastError());
    const unsigned long long* occ = occ0;
    if (nitems > 0) {
      for (int item = nitems - 1; item >= -1; item--) {
        if (item < 0 && (merge || nres == 1)) break;
        const int key = item < 0 ? -1 : p.order_key[item];
        const int bits = item < 0 ? seg_bits : max_key_bits[key];
        if (bits == 0) continue;   // a key of one value orders nothing
        dist_key_kernel<<<cgrid, kThreads, 0, st>>>(vb.Current(), occ, raw, n, static_cast<const DistKey*>(dkeys.p), nkeys, key,
                                                    item >= 0 && p.order_desc[item], merge, kb.Current());
        PB200_CUDA(cudaGetLastError());
        PB200_CUDA(cub::DeviceRadixSort::SortPairs(stmp.p, key_bytes, kb, vb, (int)n, 0, bits, st));
      }
    }
    dist_pick_kernel<<<dim3((unsigned)grid_for(ctx, p.sel.limit), (unsigned)nres), kThreads, 0, st>>>(static_cast<const DistRes*>(dres.p), vb.Current(), pick);
    PB200_CUDA(cudaGetLastError());
    unsigned char* dst = nullptr;
    const bool mapped = out_bytes <= kSelMappedBytes;
    if (mapped) {
      void* dp = nullptr;
      PB200_CUDA(cudaHostGetDevicePointer(&dp, block->p, 0));
      dst = static_cast<unsigned char*>(dp);
    } else {
      if (int rc = staging.alloc(out_bytes)) return rc;
      dst = static_cast<unsigned char*>(staging.p);
    }
    dist_gather_kernel<<<grid_for(ctx, total_rows), kThreads, 0, st>>>(pick, occ, raw, total_rows, static_cast<const SelCol*>(dcols.p),
                                                                       static_cast<const DistKey*>(dkeys.p), nkeys, dst);
    PB200_CUDA(cudaGetLastError());
    if (!mapped) PB200_CUDA(cudaMemcpyAsync(block->p, staging.p, out_bytes, cudaMemcpyDeviceToHost, st));
    const cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) { set_error("DISTINCT extraction failed: %s", cudaGetErrorString(se)); return PB200_E_CUDA; }
  }

  // ---- results: row ranges of the one block ----
  unsigned char* base = static_cast<unsigned char*>(block->p);
  int32_t* all_docs = reinterpret_cast<int32_t*>(base);
  int32_t* all_segs = all_docs + total_rows;
  const unsigned long long* all_cols = reinterpret_cast<const unsigned long long*>(base + 8 * total_rows);
  for (int r = 0; r < nres; r++) {
    const int s0 = merge ? 0 : r, s1 = merge ? nseg : r + 1;
    std::unique_ptr<pb200_result> R(new pb200_result());
    pb200_result::Selection& v = R->selection;
    v.present = true;
    v.block = block;
    long long docs_scanned = 0, entries = 0, total_docs = 0;
    for (int s = s0; s < s1; s++) { docs_scanned += matches[s]; entries += in_filter[s]; total_docs += segments[s]->num_docs; }
    v.rows = res[r].rows;
    v.doc_ids = all_docs + res[r].row_off;
    v.segment_index = all_segs + res[r].row_off;
    for (int k = 0; k < nkeys; k++) v.columns.push_back(all_cols + (size_t)k * total_rows + res[r].row_off);
    R->meta.num_groups = (int32_t)v.rows;
    R->meta.regime = PB200_REGIME_NONE;
    R->meta.num_docs_scanned = docs_scanned;
    R->meta.num_entries_scanned_in_filter = entries;
    R->meta.num_entries_scanned_post_filter = docs_scanned * nkeys;
    R->meta.num_total_docs = total_docs;
    R->meta.device_ms = ms;
    results[r] = R.release();
  }
  const double t_exit = host_ms();
  for (int ph = 0; ph < PB200_NUM_PHASES; ph++) set_phase_ms(ph, 0.0);
  set_phase_ms(PB200_PHASE_PLAN, t_planned - t_enter);
  set_phase_ms(PB200_PHASE_DEVICE_WAIT, t_scanned - t_planned);
  set_phase_ms(PB200_PHASE_EXTRACT, t_exit - t_scanned);
  set_phase_ms(PB200_PHASE_TOTAL, t_exit - t_enter);
  return PB200_OK;
}
