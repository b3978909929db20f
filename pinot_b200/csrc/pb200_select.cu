// pb200_select.cu -- selection queries: SELECT columns WHERE ... [ORDER BY columns] LIMIT n (the reference's
// SelectionOnlyOperator and SelectionOrderByOperator).
//
// The filter is the scan kernel's (pb200_scan.cuh), launched as an aggregation-only COUNT(*) with the match-mask output
// switched on (QueryDesc.reserved_tail): each thread stores the final 32-row mask of its rows, so the launch leaves the
// doc-id set of every segment in the PB200_F_DOC_MASK layout (the reference's DocIdSet) plus its match count.  Then:
//   selection only: per-word popcounts of every segment's mask, one cub exclusive scan over all of them, compaction of
//     each segment's first `rows` matches in doc order;
//   ORDER BY: a histogram of the first order key's top 12 bits over each segment's matches; the threshold bucket is the
//     first at which the better buckets plus itself hold `rows`; only the matches in buckets up to it are compacted (doc
//     order, same popcount / scan / compaction with that predicate) and sorted: stable cub::DeviceRadixSort passes from
//     the last order item to the first, then one by segment.  Stable over doc-ordered input, so ties keep doc order --
//     the reference keeps the lower doc ids among equal keys.  A merged ORDER BY merges the segments' tops by value on
//     the host (at most LIMIT x segments rows; the dictionaries may differ).
//   projection gather: per row and column, the dictId (or raw 32-bit value) unpacked at the doc from the resident
//     native-order forward index, looked up in the device dictionary, written typed (int64 / double).
// Order keys are 32-bit and order preserving: a dictId left-aligned to 32 bits (dictionary order = value order, STRING
// byte order), a raw INT biased by 2^31, a raw FLOAT with the usual sign flip; DESC complements the key.
// Without ORDER BY a segment is first scanned over a doc prefix (plan_selection); only a segment whose prefix held fewer
// than LIMIT matches is scanned again in full.  ORDER BY scans every doc.
//
// Stream synchronisations per call: one after the scan (the match counts size the output), one after a rescan when any
// segment needs it (selection only), one after the histogram (ORDER BY: the thresholds size the candidates), one after
// the select phase -- 2 or 3, plus the ones bind_leaf_buffers takes for caller-supplied leaf payloads (LUTs, doc masks,
// doc ranges), as for aggregations.  The output goes to a pinned block like group extraction (pb200_extract.cu): up to
// 512 KB the gather writes it straight into mapped memory, larger outputs go to an exact-size device staging buffer and
// come back with one DMA copy.  pb200_last_phases after a selection: PLAN (planning), DEVICE_WAIT (scans and their
// synchronisations), EXTRACT (the select phase up to its synchronisation, host merge included), TOTAL.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <vector>

#include <cub/cub.cuh>

#include "pb200_internal.h"
#include "pb200_plan.h"
#include "pb200_scan_launch.h"
#include "pb200_order.h"
#include "pb200_select.cuh"

namespace pb200 {
namespace {

constexpr int kSelThreads = 256;
constexpr int kHistBits = 12;                 // order-key histogram: the key's top 12 bits
constexpr int kHistBins = 1 << kHistBits;

struct SelSeg {            // one segment of the select phase
  const uint32_t* mask;    // its match mask: bit j of word w = doc 32w + j
  long long nwords;        // words of the scanned range
  long long word_base;     // its first word in the concatenated popcount / position arrays
  long long cand_off;      // its first compacted row (selection only: = row_off)
  long long cands;         // compacted rows: its first `cands` matches in doc order with key bucket <= thresh
  long long row_off;       // its first output row
  long long rows;          // output rows
  uint32_t thresh;         // ORDER BY: largest first-key bucket compacted (kHistBins - 1: every match)
  int32_t seg;             // index in the submission
};
// order-preserving 32-bit key (see the file comment)
__device__ __forceinline__ uint32_t order_key(const SelCol& c, int32_t doc) {
  const uint32_t x = read_at(c, doc);
  uint32_t k;
  if (c.kind == SEL_RAW_I32) k = x ^ 0x80000000u;
  else if (c.kind == SEL_RAW_F32) {   // Float.compare order: every NaN is the canonical one, after +inf
    const uint32_t f = (x & 0x7FFFFFFFu) > 0x7F800000u ? 0x7FC00000u : x;
    k = (f & 0x80000000u) ? ~f : (f | 0x80000000u);
  }
  else k = c.bits >= 32 ? x : x << (32 - c.bits);
  return c.desc ? ~k : k;
}
__device__ __forceinline__ uint32_t bucket_of(uint32_t key) { return key >> (32 - kHistBits); }

// matches of word w that are compacted: all of them, or (ORDER BY) those whose first key is in a bucket <= thresh
__device__ __forceinline__ uint32_t kept_bits(const SelSeg& sg, const SelCol* key0, long long w) {
  uint32_t x = __ldg(sg.mask + w);
  if (key0 == nullptr || sg.thresh >= (uint32_t)(kHistBins - 1)) return x;
  uint32_t keep = 0;
  for (uint32_t y = x; y; y &= y - 1u) {
    const int j = __ffs(y) - 1;
    if (bucket_of(order_key(*key0, (int32_t)(32 * w + j))) <= sg.thresh) keep |= 1u << j;
  }
  return keep;
}

// keys: [nseg x nitems] order-item descriptors (item 0 of segment s at s * nitems) or NULL (selection only)
__global__ void sel_popc_kernel(const SelSeg* __restrict__ segs, const SelCol* __restrict__ keys, int nitems, uint32_t* __restrict__ cnt) {
  const SelSeg sg = segs[blockIdx.y];
  const SelCol* k0 = keys ? keys + (size_t)blockIdx.y * nitems : nullptr;
  for (long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x; w < sg.nwords; w += (long long)gridDim.x * blockDim.x)
    cnt[sg.word_base + w] = sg.cands > 0 ? (uint32_t)__popc(kept_bits(sg, k0, w)) : 0u;
}

// Ranks are differences of the 32-bit exclusive scan inside one segment: exact modulo 2^32 even when the running total
// over all segments wraps (a segment has fewer than 2^31 docs).
__global__ void sel_compact_kernel(const SelSeg* __restrict__ segs, const SelCol* __restrict__ keys, int nitems,
                                   const uint32_t* __restrict__ pos, int32_t* __restrict__ doc_out, int32_t* __restrict__ seg_out) {
  const SelSeg sg = segs[blockIdx.y];
  if (sg.cands <= 0) return;
  const SelCol* k0 = keys ? keys + (size_t)blockIdx.y * nitems : nullptr;
  const uint32_t base = pos[sg.word_base];
  for (long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x; w < sg.nwords; w += (long long)gridDim.x * blockDim.x) {
    uint32_t r = pos[sg.word_base + w] - base;
    if ((long long)r >= sg.cands) continue;
    uint32_t x = kept_bits(sg, k0, w);
    while (x != 0u && (long long)r < sg.cands) {
      const int j = __ffs(x) - 1;
      x &= x - 1u;
      doc_out[sg.cand_off + r] = (int32_t)(32 * w + j);
      seg_out[sg.cand_off + r] = sg.seg;
      ++r;
    }
  }
}

// ORDER BY: histogram of the first key's bucket over each segment's matches (block-private in shared memory)
__global__ void sel_hist_kernel(const SelSeg* __restrict__ segs, const SelCol* __restrict__ keys, int nitems, uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[kHistBins];
  for (int b = threadIdx.x; b < kHistBins; b += blockDim.x) h[b] = 0u;
  __syncthreads();
  const SelSeg sg = segs[blockIdx.y];
  const SelCol k0 = keys[(size_t)blockIdx.y * nitems];
  if (sg.rows > 0)
    for (long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x; w < sg.nwords; w += (long long)gridDim.x * blockDim.x)
      for (uint32_t x = __ldg(sg.mask + w); x; x &= x - 1u)
        atomicAdd(&h[bucket_of(order_key(k0, (int32_t)(32 * w + __ffs(x) - 1)))], 1u);
  __syncthreads();
  uint32_t* out = hist + (size_t)blockIdx.y * kHistBins;
  for (int b = threadIdx.x; b < kHistBins; b += blockDim.x)
    if (h[b]) atomicAdd(out + b, h[b]);
}

__global__ void sel_iota_kernel(int32_t* __restrict__ p, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = (int32_t)i;
}
// sort keys of one pass over the current permutation: item `item` (or, item < 0, the candidate's segment)
__global__ void sel_key_kernel(const int32_t* __restrict__ perm, const int32_t* __restrict__ cdoc, const int32_t* __restrict__ cseg,
                               long long n, const SelCol* __restrict__ keys, int nitems, int item, uint32_t* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int32_t c = perm[i];
    out[i] = item < 0 ? (uint32_t)cseg[c] : order_key(keys[(size_t)cseg[c] * nitems + item], cdoc[c]);
  }
}
// output row -> candidate: segment s's rows are the first `rows` of its sorted candidates
__global__ void sel_pick_kernel(const SelSeg* __restrict__ segs, const int32_t* __restrict__ perm, int32_t* __restrict__ pick) {
  const SelSeg sg = segs[blockIdx.y];
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < sg.rows; r += (long long)gridDim.x * blockDim.x)
    pick[sg.row_off + r] = perm[sg.cand_off + r];
}

// Output block: doc ids int32[rows], segment index int32[rows], then per column 8-byte values [rows].  Row i is candidate
// pick[i] (pick NULL: candidate i).
__global__ void sel_gather_kernel(const int32_t* __restrict__ docs, const int32_t* __restrict__ segs, const int32_t* __restrict__ pick,
                                  long long rows, const SelCol* __restrict__ cols, int ncols, unsigned char* __restrict__ out) {
  int32_t* odoc = reinterpret_cast<int32_t*>(out);
  int32_t* oseg = odoc + rows;
  unsigned long long* ocol = reinterpret_cast<unsigned long long*>(out + 8 * rows);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < rows; i += (long long)gridDim.x * blockDim.x) {
    const long long c = pick ? pick[i] : i;
    const int32_t d = docs[c], s = segs[c];
    odoc[i] = d;
    oseg[i] = s;
    for (int k = 0; k < ncols; k++) {
      const SelCol col = cols[(size_t)s * ncols + k];
      ocol[(size_t)k * rows + i] = sel_value(col, read_at(col, d));
    }
  }
}

struct EventPair {
  pb200_ctx* c; cudaEvent_t a = nullptr, b = nullptr;
  ~EventPair() { give_event(c, a); give_event(c, b); }
};

}  // namespace

int run_selection_scan(pb200_ctx* ctx, cudaStream_t st, SelectionPlan& p, DevBufRaw& mask, std::vector<long long>& matches,
                       float* ms) {
  ScanPlan& plan = p.scan;
  const int nseg = (int)plan.segs.size();
  std::vector<std::unique_ptr<DevBufRaw>> temps;
  if (int rc = bind_leaf_buffers(ctx, plan, st, temps)) return rc;
  const size_t acc_bytes = sizeof(AggAccum) * nseg;
  DevBufRaw accum(ctx), dsegs(ctx);
  if (int rc = accum.alloc(acc_bytes)) return rc;
  if (int rc = dsegs.alloc(sizeof(SegDesc) * nseg)) return rc;
  if (int rc = mask.alloc(std::max<long long>(p.mask_words, 1) * 4)) return rc;  // every word is written by the launch
  PB200_CUDA(cudaMemsetAsync(accum.p, 0, acc_bytes, st));
  for (int s = 0; s < nseg; s++) plan.segs[s].accum = static_cast<AggAccum*>(accum.p) + s;
  PB200_CUDA(cudaMemcpyAsync(dsegs.p, plan.segs.data(), sizeof(SegDesc) * nseg, cudaMemcpyHostToDevice, st));
  EventPair ev{ctx};
  ev.a = take_event(ctx);
  ev.b = take_event(ctx);
  if (!ev.a || !ev.b) { set_error("cudaEventCreate failed"); return PB200_E_CUDA; }
  PB200_CUDA(cudaEventRecord(ev.a, st));
  for (size_t c = 0; c < plan.chunks.size(); c++) {
    const LaunchChunk& ch = plan.chunks[c];
    QueryDesc cq = plan.q;
    cq.num_segments = ch.num_segs;
    cq.total_tiles = ch.total_tiles;
    set_selection_mask(cq, static_cast<uint32_t*>(mask.p) + p.chunk_word_off[c]);
    const cudaError_t le = launch_scan_variant(plan.variant, plan.smem_bytes, ch.grid, cq, tma_table(plan, ch),
                                               static_cast<const SegDesc*>(dsegs.p) + ch.first_seg, st);
    if (le != cudaSuccess) { set_error("selection scan launch failed: %s (smem %zu B, grid %d)", cudaGetErrorString(le), plan.smem_bytes, ch.grid); return PB200_E_CUDA; }
  }
  PB200_CUDA(cudaEventRecord(ev.b, st));
  std::vector<AggAccum> acc(nseg);
  PB200_CUDA(cudaMemcpyAsync(acc.data(), accum.p, acc_bytes, cudaMemcpyDeviceToHost, st));
  const cudaError_t se = cudaStreamSynchronize(st);
  if (se != cudaSuccess) { set_error("selection scan failed: %s", cudaGetErrorString(se)); return PB200_E_CUDA; }
  matches.resize(nseg);
  for (int s = 0; s < nseg; s++) matches[s] = (long long)acc[s].count;
  float t = 0.f;
  cudaEventElapsedTime(&t, ev.a, ev.b);
  *ms += t;
  return PB200_OK;
}

namespace {

// By-value comparison of two output rows on one order item (merged ORDER BY over segments whose dictionaries may differ).
int compare_item(const pb200_segment* const* segments, int col, int kind, bool desc, const unsigned long long* v, int32_t sa,
                 long long ia, int32_t sb, long long ib) {
  int c;
  if (kind == SEL_DICT_ID) {   // STRING: the entries' bytes (zero padded: byte order of the unpadded strings)
    const DeviceColumn& ca = segments[sa]->cols[col];
    const DeviceColumn& cb = segments[sb]->cols[col];
    const int wa = ca.dict_entry_bytes, wb = cb.dict_entry_bytes, w = std::max(wa, wb);
    const unsigned char* pa = ca.dict_be.data() + (size_t)v[ia] * wa;
    const unsigned char* pb = cb.dict_be.data() + (size_t)v[ib] * wb;
    c = 0;
    for (int i = 0; i < w && c == 0; i++) {
      const int x = i < wa ? pa[i] : 0, y = i < wb ? pb[i] : 0;
      c = x < y ? -1 : x > y;
    }
  } else if (selection_kind_is_double(kind)) {   // Double.compare: -0.0 before 0.0, one NaN after +inf (a total order)
    double x, y;
    memcpy(&x, &v[ia], 8); memcpy(&y, &v[ib], 8);
    const uint64_t kx = double_order_bits(x), ky = double_order_bits(y);
    c = kx < ky ? -1 : kx > ky;
  } else {
    const long long x = (long long)v[ia], y = (long long)v[ib];
    c = x < y ? -1 : x > y;
  }
  return desc ? -c : c;
}

}  // namespace
}  // namespace pb200

using namespace pb200;

extern "C" int32_t pb200_execute_selection(pb200_ctx* ctx, const pb200_query* filter_only, const pb200_selection* sel,
                                           pb200_segment* const* segments, int32_t nseg, int32_t flags, pb200_result** results) {
  if (!ctx || !filter_only || !sel || !segments || !results || nseg <= 0) { set_error("invalid argument to pb200_execute_selection"); return PB200_E_INVALID; }
  if (flags & ~PB200_Q_MERGE_SEGMENTS) { set_error("pb200_execute_selection: flags other than PB200_Q_MERGE_SEGMENTS"); return PB200_E_INVALID; }
  for (int s = 0; s < nseg; s++)
    if (!segments[s] || segments[s]->ctx != ctx) { set_error("segment %d does not belong to this context / schema", s); return PB200_E_INVALID; }
  const double t_enter = host_ms();
  PB200_CUDA(cudaSetDevice(ctx->device));
  const Tuning tune = [&]() { std::lock_guard<std::mutex> g(ctx->mu); return ctx->tune; }();
  const DeviceLimits lim{ctx->sm_count, ctx->max_smem_optin};
  SelectionPlan p1;
  if (int rc = plan_selection(tune, lim, filter_only, sel, segments, nseg, true, &p1)) return rc;
  const double t_planned = host_ms();

  cudaStream_t st = take_stream(ctx);
  struct StreamReturn { pb200_ctx* c; cudaStream_t s; ~StreamReturn() { give_stream(c, s); } } stream_return{ctx, st};
  float ms = 0.f;
  DevBufRaw mask1(ctx), mask2(ctx);
  std::vector<long long> m1;
  if (int rc = run_selection_scan(ctx, st, p1, mask1, m1, &ms)) return rc;

  // where each segment's rows come from: the prefix pass, or the full rescan
  std::vector<const uint32_t*> smask(nseg);
  std::vector<long long> sdocs(nseg), matches(nseg), in_filter(nseg);
  for (int s = 0; s < nseg; s++) {
    smask[s] = static_cast<const uint32_t*>(mask1.p) + p1.mask_word_off[s];
    sdocs[s] = p1.scan_docs[s]; matches[s] = m1[s]; in_filter[s] = p1.scan.in_filter[s];
  }
  const std::vector<int> rescan = selection_rescan(p1, segments, m1);
  if (!rescan.empty()) {
    const Rescan rs = rescan_query(*filter_only, segments, rescan);
    SelectionPlan p2;
    if (int rc = plan_selection(tune, lim, &rs.query, sel, rs.segs.data(), (int)rs.segs.size(), false, &p2)) return rc;
    std::vector<long long> m2;
    if (int rc = run_selection_scan(ctx, st, p2, mask2, m2, &ms)) return rc;
    for (size_t i = 0; i < rescan.size(); i++) {
      const int s = rescan[i];
      smask[s] = static_cast<const uint32_t*>(mask2.p) + p2.mask_word_off[i];
      sdocs[s] = p2.scan_docs[i]; matches[s] = m2[i]; in_filter[s] = p2.scan.in_filter[i];
    }
  }
  const double t_scanned = host_ms();

  // ---- rows.  Selection only: per segment its first min(limit, matches) matches, merged: segments in submission order
  //      up to `limit`.  ORDER BY: per segment its top min(limit, matches) rows; merged, the tops are merged by value below.
  const bool merge = flags & PB200_Q_MERGE_SEGMENTS;
  const int nres = merge ? 1 : nseg;
  const int ncols = (int)p1.columns.size();
  const int nitems = (int)p1.order_cols.size();
  const bool ordered = nitems > 0;
  const int gcols = ncols + (ordered && merge ? nitems : 0);   // a merged ORDER BY also gathers the order values
  std::vector<SelSeg> ss(nseg);
  long long total_rows = 0, total_words = 0, max_words = 0, taken = 0;
  for (int s = 0; s < nseg; s++) {
    SelSeg& g = ss[s];
    g.mask = smask[s];
    g.nwords = (sdocs[s] + 31) / 32;
    g.word_base = total_words;
    g.rows = merge && !ordered ? std::min(matches[s], p1.limit - taken) : std::min(matches[s], p1.limit);
    taken += g.rows;
    g.row_off = total_rows;
    g.cand_off = g.row_off;
    g.cands = g.rows;
    g.thresh = kHistBins - 1;
    g.seg = s;
    total_rows += g.rows;
    total_words += g.nwords;
    max_words = std::max(max_words, g.nwords);
  }
  const size_t out_bytes = (size_t)total_rows * 8 * (1 + (size_t)gcols);
  auto block = std::make_shared<PinnedBlock>();
  block->ctx = ctx;
  if (int rc = pinned_alloc(ctx, std::max<size_t>(out_bytes, 8), &block->p, &block->bytes)) return rc;
  if (total_rows > 0) {
    std::vector<SelCol> sc((size_t)nseg * std::max(gcols, 1)), sk((size_t)nseg * std::max(nitems, 1));
    for (int s = 0; s < nseg; s++) {
      for (int k = 0; k < gcols; k++) {
        const int col = k < ncols ? p1.columns[k] : p1.order_cols[k - ncols];
        const DeviceColumn& c = segments[s]->cols[col];
        sc[(size_t)s * gcols + k] = SelCol{c.fwd, c.dict_native, c.bits, k < ncols ? p1.kinds[k] : p1.order_kinds[k - ncols], 0, 0};
      }
      for (int k = 0; k < nitems; k++) {
        const DeviceColumn& c = segments[s]->cols[p1.order_cols[k]];
        sk[(size_t)s * nitems + k] = SelCol{c.fwd, c.dict_native, c.bits, p1.order_kinds[k], p1.order_desc[k] ? 1 : 0, 0};
      }
    }
    DevBufRaw dss(ctx), dsc(ctx), dsk(ctx), cnt(ctx), pos(ctx), tmp(ctx), cand(ctx), staging(ctx), hist(ctx);
    if (int rc = dss.alloc(sizeof(SelSeg) * nseg)) return rc;
    if (int rc = dsc.alloc(sizeof(SelCol) * sc.size())) return rc;
    if (int rc = dsk.alloc(sizeof(SelCol) * sk.size())) return rc;
    PB200_CUDA(cudaMemcpyAsync(dsc.p, sc.data(), sizeof(SelCol) * sc.size(), cudaMemcpyHostToDevice, st));
    PB200_CUDA(cudaMemcpyAsync(dsk.p, sk.data(), sizeof(SelCol) * sk.size(), cudaMemcpyHostToDevice, st));
    const SelCol* keys = ordered ? static_cast<const SelCol*>(dsk.p) : nullptr;
    const dim3 wgrid((unsigned)std::max<long long>(1, std::min<long long>((max_words + kSelThreads - 1) / kSelThreads, (long long)ctx->sm_count * 8)), (unsigned)nseg);
    if (ordered) {
      // ---- threshold bucket per segment: the better buckets plus it hold at least `rows` matches ----
      if (int rc = hist.alloc((size_t)nseg * kHistBins * 4)) return rc;
      PB200_CUDA(cudaMemsetAsync(hist.p, 0, (size_t)nseg * kHistBins * 4, st));
      PB200_CUDA(cudaMemcpyAsync(dss.p, ss.data(), sizeof(SelSeg) * nseg, cudaMemcpyHostToDevice, st));
      sel_hist_kernel<<<wgrid, kSelThreads, 0, st>>>(static_cast<const SelSeg*>(dss.p), keys, nitems, static_cast<uint32_t*>(hist.p));
      PB200_CUDA(cudaGetLastError());
      std::vector<uint32_t> h((size_t)nseg * kHistBins);
      PB200_CUDA(cudaMemcpyAsync(h.data(), hist.p, h.size() * 4, cudaMemcpyDeviceToHost, st));
      PB200_CUDA(cudaStreamSynchronize(st));
      long long cursor = 0;
      for (int s = 0; s < nseg; s++) {
        SelSeg& g = ss[s];
        long long cum = 0;
        uint32_t b = 0;
        if (g.rows > 0)
          for (b = 0; b < (uint32_t)kHistBins; b++) { cum += h[(size_t)s * kHistBins + b]; if (cum >= g.rows) break; }
        g.thresh = std::min<uint32_t>(b, kHistBins - 1);
        g.cands = g.rows > 0 ? cum : 0;
        g.cand_off = cursor;
        cursor += g.cands;
      }
    }
    const long long ncand = ordered ? ss[nseg - 1].cand_off + ss[nseg - 1].cands : total_rows;
    size_t scan_bytes = 0, sort_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)total_words, st);
    if (ordered) {
      cub::DoubleBuffer<uint32_t> kb(nullptr, nullptr);
      cub::DoubleBuffer<int32_t> vb(nullptr, nullptr);
      cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, kb, vb, (int)ncand, 0, 32, st);
    }
    if (int rc = cnt.alloc((size_t)total_words * 4)) return rc;
    if (int rc = pos.alloc((size_t)total_words * 4)) return rc;
    if (int rc = tmp.alloc(std::max<size_t>(std::max(scan_bytes, sort_bytes), 1))) return rc;
    // candidates: doc, segment; ORDER BY also two key and two permutation buffers and the row -> candidate map
    const size_t cand_words = (size_t)ncand * (ordered ? 6 : 2) + (ordered ? (size_t)total_rows : 0);
    if (int rc = cand.alloc(cand_words * 4)) return rc;
    int32_t* cdoc = static_cast<int32_t*>(cand.p);
    int32_t* cseg = cdoc + ncand;
    PB200_CUDA(cudaMemcpyAsync(dss.p, ss.data(), sizeof(SelSeg) * nseg, cudaMemcpyHostToDevice, st));
    sel_popc_kernel<<<wgrid, kSelThreads, 0, st>>>(static_cast<const SelSeg*>(dss.p), keys, nitems, static_cast<uint32_t*>(cnt.p));
    PB200_CUDA(cudaGetLastError());
    PB200_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, scan_bytes, static_cast<const uint32_t*>(cnt.p), static_cast<uint32_t*>(pos.p), (int)total_words, st));
    sel_compact_kernel<<<wgrid, kSelThreads, 0, st>>>(static_cast<const SelSeg*>(dss.p), keys, nitems, static_cast<const uint32_t*>(pos.p), cdoc, cseg);
    PB200_CUDA(cudaGetLastError());
    const int32_t* pick = nullptr;
    if (ordered) {
      // ---- stable radix passes: last order item first, then the segment (candidates are doc ordered per segment) ----
      uint32_t* k0 = reinterpret_cast<uint32_t*>(cseg + ncand);
      uint32_t* k1 = k0 + ncand;
      int32_t* v0 = reinterpret_cast<int32_t*>(k1 + ncand);
      int32_t* v1 = v0 + ncand;
      int32_t* pk = v1 + ncand;
      const int cgrid = (int)std::max<long long>(1, std::min<long long>((ncand + kSelThreads - 1) / kSelThreads, (long long)ctx->sm_count * 8));
      sel_iota_kernel<<<cgrid, kSelThreads, 0, st>>>(v0, ncand);
      cub::DoubleBuffer<uint32_t> kb(k0, k1);
      cub::DoubleBuffer<int32_t> vb(v0, v1);
      int seg_bits = 0;
      while ((1 << seg_bits) < nseg) seg_bits++;
      for (int item = nitems - 1; item >= -1; item--) {
        if (item < 0 && seg_bits == 0) break;
        sel_key_kernel<<<cgrid, kSelThreads, 0, st>>>(vb.Current(), cdoc, cseg, ncand, keys, nitems, item, kb.Current());
        PB200_CUDA(cudaGetLastError());
        PB200_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, sort_bytes, kb, vb, (int)ncand, 0, item < 0 ? seg_bits : 32, st));
      }
      PB200_CUDA(cudaMemcpyAsync(dss.p, ss.data(), sizeof(SelSeg) * nseg, cudaMemcpyHostToDevice, st));
      sel_pick_kernel<<<wgrid, kSelThreads, 0, st>>>(static_cast<const SelSeg*>(dss.p), vb.Current(), pk);
      PB200_CUDA(cudaGetLastError());
      pick = pk;
    }
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
    const int ggrid = (int)std::max<long long>(1, std::min<long long>((total_rows + kSelThreads - 1) / kSelThreads, (long long)ctx->sm_count * 8));
    sel_gather_kernel<<<ggrid, kSelThreads, 0, st>>>(cdoc, cseg, pick, total_rows, static_cast<const SelCol*>(dsc.p), gcols, dst);
    PB200_CUDA(cudaGetLastError());
    if (!mapped) PB200_CUDA(cudaMemcpyAsync(block->p, staging.p, out_bytes, cudaMemcpyDeviceToHost, st));
    const cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) { set_error("selection select phase failed: %s", cudaGetErrorString(se)); return PB200_E_CUDA; }
  }

  // ---- merged ORDER BY: the segments' tops by value, ties by (segment, doc id), first `limit` into a block of their own ----
  unsigned char* base = static_cast<unsigned char*>(block->p);
  long long out_rows = total_rows;
  if (ordered && merge && total_rows > 0) {
    const int32_t* docs = reinterpret_cast<const int32_t*>(base);
    const int32_t* segi = docs + total_rows;
    const unsigned long long* vals = reinterpret_cast<const unsigned long long*>(base + 8 * total_rows);
    std::vector<long long> order(total_rows);
    for (long long i = 0; i < total_rows; i++) order[i] = i;
    std::sort(order.begin(), order.end(), [&](long long a, long long b) {
      for (int k = 0; k < nitems; k++) {
        const int c = compare_item(segments, p1.order_cols[k], p1.order_kinds[k], p1.order_desc[k],
                                   vals + (size_t)(ncols + k) * total_rows, segi[a], a, segi[b], b);
        if (c) return c < 0;
      }
      return segi[a] != segi[b] ? segi[a] < segi[b] : docs[a] < docs[b];
    });
    out_rows = std::min<long long>(p1.limit, total_rows);
    auto merged = std::make_shared<PinnedBlock>();
    merged->ctx = ctx;
    if (int rc = pinned_alloc(ctx, std::max<size_t>((size_t)out_rows * 8 * (1 + (size_t)ncols), 8), &merged->p, &merged->bytes)) return rc;
    unsigned char* mb = static_cast<unsigned char*>(merged->p);
    int32_t* mdocs = reinterpret_cast<int32_t*>(mb);
    int32_t* msegs = mdocs + out_rows;
    unsigned long long* mvals = reinterpret_cast<unsigned long long*>(mb + 8 * out_rows);
    for (long long r = 0; r < out_rows; r++) {
      const long long i = order[r];
      mdocs[r] = docs[i];
      msegs[r] = segi[i];
      for (int k = 0; k < ncols; k++) mvals[(size_t)k * out_rows + r] = vals[(size_t)k * total_rows + i];
    }
    block = merged;
    base = mb;
  }

  // ---- results: row ranges of the one block ----
  int32_t* all_docs = reinterpret_cast<int32_t*>(base);
  int32_t* all_segs = all_docs + out_rows;
  const unsigned long long* all_cols = reinterpret_cast<const unsigned long long*>(base + 8 * out_rows);
  for (int r = 0; r < nres; r++) {
    const int s0 = merge ? 0 : r, s1 = merge ? nseg : r + 1;
    std::unique_ptr<pb200_result> R(new pb200_result());
    pb200_result::Selection& v = R->selection;
    v.present = true;
    v.block = block;
    const long long off = merge ? 0 : ss[s0].row_off;
    long long docs_scanned = 0, entries = 0, total_docs = 0;
    for (int s = s0; s < s1; s++) { docs_scanned += matches[s]; entries += in_filter[s]; total_docs += segments[s]->num_docs; }
    v.rows = merge ? out_rows : ss[r].rows;
    v.doc_ids = all_docs + off;
    v.segment_index = all_segs + off;
    for (int k = 0; k < ncols; k++) v.columns.push_back(all_cols + (size_t)k * out_rows + off);
    R->meta.num_groups = (int32_t)v.rows;
    R->meta.regime = PB200_REGIME_NONE;
    R->meta.num_docs_scanned = docs_scanned;
    R->meta.num_entries_scanned_in_filter = entries;
    R->meta.num_entries_scanned_post_filter = v.rows * ncols;
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

extern "C" int32_t pb200_result_selection(const pb200_result* R, int64_t* rows, const int32_t** doc_ids,
                                          const int32_t** segment_index, const void** columns) {
  if (!R || !R->selection.present) { set_error("not a selection result"); return PB200_E_INVALID; }
  const pb200_result::Selection& v = R->selection;
  if (rows) *rows = v.rows;
  if (doc_ids) *doc_ids = v.doc_ids;
  if (segment_index) *segment_index = v.segment_index;
  if (columns) for (size_t k = 0; k < v.columns.size(); k++) columns[k] = v.columns[k];
  return PB200_OK;
}
