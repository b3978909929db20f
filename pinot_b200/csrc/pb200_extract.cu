// pb200_extract.cu -- group extraction: dense / hash group tables on the device -> the result's FINAL layout in pinned
// host memory, written by the device itself.
//
// What the reference does here: GroupByOperator.nextBlock() walks the group-key iterator and the result holders and
// builds the GroupByResultsBlock (core/operator/query/GroupByOperator.java:116-140,
// DictionaryBasedGroupKeyGenerator.getGroupKeys :577-605; holders: DoubleGroupByResultHolder / ObjectGroupByResultHolder).
// Here, for ALL results of a submission at once, three small launches:
//   count   one CTA per 2048-entry chunk of a table counts its non-empty groups;
//   scan    one CTA per result turns the chunk counts into exclusive offsets and the result's group count;
//   write   every chunk compacts its groups IN RAW-KEY ORDER (the iteration order of the reference's array based holder)
//           and writes, per group, the decoded key dictIds and per aggregation the intermediate the caller reads
//           (double value incl. dictionary lookups for MIN / MAX, long count, MIN / MAX dictId) in the final column layout
//           -- no host conversion loop; accessors read (or hand out) columns of that pinned block.
// Small results (worst case <= kSpeculativeBytes) do all three launches back to back, write STRAIGHT into the mapped
// pinned block and synchronise ONCE.  Larger ones read the group counts first, size the block exactly, compact into a
// device staging buffer and move it with ONE DMA copy: device stores into mapped host memory are far slower than the
// copy engine.
// A result with an ORDER BY spec (pb200_order_by, pb200_order.h) takes one more step between scan and write: the write kernel
// compacts its non-empty entries into an index array (index-only mode), a key kernel turns each row into one u64 key per
// pass, stable LSD radix sorts order the index by the group-key tie key first and then by the items from last to first, and
// the write kernel writes row r from entry idx[r] for r < min(groups, trim_size).  The block is sized for the trimmed rows,
// so a trimmed result stays on the one-synchronisation path.  A PB200_ORDER_POST item's pass evaluates its program
// (pb200_postagg.h) over the row's final values and keys the result in Double.compare order.
// A result with a HAVING tree (pb200_having, pb200_having.h) takes one step before count: a keep kernel evaluates the tree
// on every existing entry's final values and writes a keep bitmap (1 bit per entry, one byte per 8 consecutive entries)
// plus the number of existing entries, which the numGroupsLimit check uses.  Count and write (also index-only) then test
// the keep bit instead of non_empty(), so HAVING runs before the ORDER BY and its trim, and only removes rows.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "pb200_internal.h"
#include "pb200_decode.h"
#include "pb200_having.h"
#include "pb200_order.h"
#include "pb200_postagg.h"

namespace pb200 {

constexpr int kChunk = 2048;             // table entries per CTA
constexpr int kExtractThreads = 256;     // 8 consecutive entries per thread
constexpr size_t kSpeculativeBytes = 512ull << 10;
constexpr unsigned long long kNoCol = ~0ull;

struct ExtractDesc {
  const unsigned long long* count;   // existence markers, see non_empty() below
  const uint32_t* seen;
  const uint32_t* maxk;              // dictionary MIN / MAX tables only (a raw INT entry has no empty value)
  const uint32_t* mink;
  const unsigned long long* hkeys;
  const unsigned long long* packed;  // count-carrying sum table (pb200_plan.cpp): sum(value - vmin) + count << shift
  int32_t pack_shift;
  long long groups;                  // table entries (dense: raw key space x stride, hash: capacity)
  int32_t stride, pad_stride;        // dense tables: only entries at multiples of `stride` are ever written
  int32_t ngb, nagg;
  uint32_t cards[kMaxGroupBy];
  uint32_t first_chunk, num_chunks;  // position in the launch-wide chunk sequence
  unsigned long long cap_rows;       // rows every column has room for
  unsigned long long off_keys;       // int32 [rows x ngb]
  unsigned long long off_idx;        // uint32 [rows] raw key / slot (only when a per-group bitset has to be gathered), else kNoCol
  unsigned long long off_dbl[kMaxAggs], off_lng[kMaxAggs], off_ids[kMaxAggs];  // kNoCol: column not produced
  unsigned long long off_mom[kMaxAggs];  // VAR / STDDEV: {s1, s2 low, s2 high} per row, for pb200_result_moments
  AggSource agg[kMaxAggs];           // each aggregation's tables (pb200_decode.h)
  // ORDER BY only (order_idx == NULL: rows in raw-key order)
  uint32_t* order_idx;               // [idx_cap] non-empty entries in raw-key order (index-only pass), sorted in place...
  const uint32_t* order_sorted;      // ...ending up here (one of the sort's two value buffers)
  unsigned long long idx_cap;        // untrimmed row bound: min(entries, numGroupsLimit + 1)
  const uint32_t* dbits[kMaxAggs];   // DISTINCTCOUNT per-group bitsets (an ORDER BY key is the popcount of a row)
  uint32_t dwords[kMaxAggs];
  const uint8_t* keep;               // HAVING only: bit j of byte i = entry 8i + j is a row (NULL: every non_empty() entry is)
};

__device__ __forceinline__ bool non_empty(const ExtractDesc& d, long long i) {
  if (d.hkeys) return d.hkeys[i] != ~0ull;
  if (d.packed) return d.packed[i] != 0ull;
  return (d.count && d.count[i] != 0ull) || (d.seen && d.seen[i] != 0u) || (d.maxk && d.maxk[i] != 0u) || (d.mink && d.mink[i] != 0xFFFFFFFFu);
}
// bit j = entry base + j exists (base: a multiple of 8)
__device__ __forceinline__ uint32_t exists_flags(const ExtractDesc& d, long long base) {
  uint32_t flags = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) flags |= ((base + j < d.groups && non_empty(d, base + j)) ? 1u : 0u) << j;
  return flags;
}
// bit j = entry base + j is a row of the result
__device__ __forceinline__ uint32_t entry_flags(const ExtractDesc& d, long long base) {
  return d.keep ? d.keep[base >> 3] : exists_flags(d, base);
}
__device__ __forceinline__ int find_result(const ExtractDesc* descs, int nres, uint32_t chunk) {
  int r = 0;
  while (r + 1 < nres && chunk >= descs[r + 1].first_chunk) ++r;
  return r;
}

__global__ void __launch_bounds__(kExtractThreads) extract_count_kernel(const ExtractDesc* __restrict__ descs, int nres,
                                                                        uint32_t* __restrict__ chunk_count) {
  __shared__ uint32_t wsum[kExtractThreads / 32];
  const int r = find_result(descs, nres, blockIdx.x);
  const ExtractDesc& d = descs[r];
  const long long base = (long long)(blockIdx.x - d.first_chunk) * kChunk + threadIdx.x * 8;
  uint32_t c = __popc(entry_flags(d, base));
  c = __reduce_add_sync(0xFFFFFFFFu, c);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < kExtractThreads / 32; ++w) t += wsum[w];
    chunk_count[blockIdx.x] = t;
  }
}

// one CTA per result: chunk counts -> exclusive offsets (in place) + the result's total
__global__ void __launch_bounds__(kExtractThreads) extract_scan_kernel(const ExtractDesc* __restrict__ descs,
                                                                       uint32_t* __restrict__ chunk_count,
                                                                       unsigned long long* __restrict__ totals) {
  __shared__ unsigned long long part[kExtractThreads];
  const ExtractDesc& d = descs[blockIdx.x];
  uint32_t* c = chunk_count + d.first_chunk;
  const uint32_t n = d.num_chunks, per = (n + kExtractThreads - 1) / kExtractThreads;
  const uint32_t lo = min(n, threadIdx.x * per), hi = min(n, lo + per);
  unsigned long long s = 0;
  for (uint32_t i = lo; i < hi; ++i) s += c[i];
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long run = 0;
    for (int t = 0; t < kExtractThreads; ++t) { const unsigned long long v = part[t]; part[t] = run; run += v; }
    totals[blockIdx.x] = run;
  }
  __syncthreads();
  unsigned long long run = part[threadIdx.x];
  for (uint32_t i = lo; i < hi; ++i) { const uint32_t v = c[i]; c[i] = (uint32_t)run; run += v; }  // offsets < 2^32 (tables <= 2^27 entries)
}

__device__ __forceinline__ unsigned long long group_count(const ExtractDesc& d, long long g) {
  return d.packed ? d.packed[g] >> d.pack_shift : (d.count ? d.count[g] : 0ull);
}

// set size of DISTINCTCOUNT aggregation a in entry g: the popcount of its bitset row
__device__ __forceinline__ long long distinct_size(const ExtractDesc& d, int a, long long g) {
  const uint32_t* row = d.dbits[a] + (size_t)g * d.dwords[a];
  long long n = 0;
  for (uint32_t w = 0; w < d.dwords[a]; ++w) n += __popc(row[w]);
  return n;
}

// final value of aggregation a in entry g as HAVING and post-aggregation programs read it (having_value); cnt = the
// entry's group count
__device__ __forceinline__ double final_value(const ExtractDesc& d, int a, long long g, unsigned long long cnt) {
  if (d.agg[a].fn == PB200_AGG_DISTINCTCOUNT) return (double)distinct_size(d, a, g);
  double dv;
  long long lv;
  int32_t id;
  agg_values(d.agg[a], g, cnt, dv, lv, id, nullptr);
  return having_value(d.agg[a].fn, dv, lv);
}

__device__ __forceinline__ unsigned long long raw_key_of(const ExtractDesc& d, long long g) {
  return d.hkeys ? d.hkeys[g] : (unsigned long long)g / (unsigned)d.stride;
}

// row `row` of the result's columns from table entry g
__device__ __forceinline__ void write_row(const ExtractDesc& d, unsigned long long row, long long g, unsigned char* __restrict__ out) {
  // ---- key dictIds: raw key = sum dictId_k * prod_{m<k} card_m (column 0 least significant) ----
  if (d.ngb > 0) {
    int32_t* kp = reinterpret_cast<int32_t*>(out + d.off_keys) + row * d.ngb;
    unsigned long long raw = raw_key_of(d, g);
    for (int k = 0; k < d.ngb; ++k) { kp[k] = (int32_t)(raw % d.cards[k]); raw /= d.cards[k]; }
  }
  if (d.off_idx != kNoCol) reinterpret_cast<uint32_t*>(out + d.off_idx)[row] = (uint32_t)g;
  const unsigned long long cnt = group_count(d, g);
  for (int a = 0; a < d.nagg; ++a) {
    double dv;
    long long lv;
    int32_t id;
    agg_values(d.agg[a], g, cnt, dv, lv, id,
               d.off_mom[a] != kNoCol ? reinterpret_cast<unsigned long long*>(out + d.off_mom[a]) + 3 * row : nullptr);
    if (d.off_dbl[a] != kNoCol) reinterpret_cast<double*>(out + d.off_dbl[a])[row] = dv;
    if (d.off_lng[a] != kNoCol) reinterpret_cast<long long*>(out + d.off_lng[a])[row] = lv;
    if (d.off_ids[a] != kNoCol) reinterpret_cast<int32_t*>(out + d.off_ids[a])[row] = id;
  }
}

// index_only: ordered results compact their entries into order_idx (the others do nothing).  Otherwise unordered results
// compact and write their rows, ordered ones write row r from order_sorted[r] for r < min(groups, cap_rows).
__global__ void __launch_bounds__(kExtractThreads) extract_write_kernel(const ExtractDesc* __restrict__ descs, int nres,
                                                                        const uint32_t* __restrict__ chunk_off,
                                                                        const unsigned long long* __restrict__ totals,
                                                                        unsigned char* __restrict__ out, bool index_only) {
  __shared__ uint32_t wsum[kExtractThreads / 32];
  const int r = find_result(descs, nres, blockIdx.x);
  const ExtractDesc& d = descs[r];
  const long long base = (long long)(blockIdx.x - d.first_chunk) * kChunk + threadIdx.x * 8;
  if (d.order_idx && !index_only) {
    const unsigned long long rows = min(totals[r], d.cap_rows);
    for (int j = 0; j < 8; ++j)
      if ((unsigned long long)(base + j) < rows) write_row(d, base + j, d.order_sorted[base + j], out);
    return;
  }
  if (!d.order_idx && index_only) return;
  const uint32_t flags = entry_flags(d, base);
  const uint32_t mine = __popc(flags);
  // CTA-wide exclusive scan of the per-thread counts (entries stay in raw-key order)
  uint32_t incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if ((threadIdx.x & 31) >= o) incl += t; }
  if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = incl;
  __syncthreads();
  uint32_t before = 0;
  for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) before += wsum[w];
  unsigned long long row = (unsigned long long)chunk_off[blockIdx.x] + before + incl - mine;
  const unsigned long long cap = index_only ? d.idx_cap : d.cap_rows;
  for (int j = 0; j < 8; ++j) {
    if (!((flags >> j) & 1u)) continue;
    if (row >= cap) return;  // more groups than the block has room for (numGroupsLimit bound: the caller discards the result)
    const long long g = base + j;
    if (index_only) d.order_idx[row] = (uint32_t)g;
    else write_row(d, row, g, out);
    ++row;
  }
}

// One sort pass of an ordered result: which key, how many of its bits are in use (pb200_order.h)
enum { PASS_TIE = 0, PASS_GROUP_BY = 1, PASS_AGG = 2, PASS_POST = 3 };
struct OrderPass {
  int32_t what, index;   // PASS_GROUP_BY: group-by column; PASS_AGG: aggregation
  int32_t cmp;           // OrderCmp of an aggregation
  int32_t descending;
  int32_t bits;
  unsigned long long mask;  // (1 << bits) - 1: the key of a padding row (past the group count: sorts last, stays last)
  pb200_post_program prog;  // PASS_POST: the item's program
};

// keys[i] = the pass's key of row i of the current order idx[], for all idx_cap rows
__global__ void __launch_bounds__(kExtractThreads) order_key_kernel(const ExtractDesc* __restrict__ descs, int r, OrderPass p,
                                                                    const unsigned long long* __restrict__ totals,
                                                                    const uint32_t* __restrict__ idx,
                                                                    unsigned long long* __restrict__ keys) {
  const ExtractDesc& d = descs[r];
  const unsigned long long n = totals[r];
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < d.idx_cap;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    if (i >= n) { keys[i] = p.mask; continue; }
    const long long g = idx[i];
    unsigned long long k;
    if (p.what == PASS_AGG) {
      double dv;
      long long lv;
      int32_t id;
      if (d.agg[p.index].fn == PB200_AGG_DISTINCTCOUNT) {
        lv = distinct_size(d, p.index, g);
        dv = (double)lv;
      } else {
        agg_values(d.agg[p.index], g, group_count(d, g), dv, lv, id, nullptr);
      }
      k = order_key(p.cmp, p.descending != 0, p.mask, dv, lv);
    } else if (p.what == PASS_POST) {
      const unsigned long long cnt = group_count(d, g);
      k = order_key(ORDER_CMP_DOUBLE, p.descending != 0, p.mask, postagg_eval(p.prog, [&](int a) { return final_value(d, a, g, cnt); }), 0);
    } else {
      // raw key: column 0 least significant; tie key: column 0 most significant (= ascending key values in GROUP BY order)
      unsigned long long raw = raw_key_of(d, g), tie = 0, id = 0;
      for (int c = 0; c < d.ngb; ++c) {
        const unsigned long long x = raw % d.cards[c];
        raw /= d.cards[c];
        unsigned long long mult = 1;
        for (int m = c + 1; m < d.ngb; ++m) mult *= d.cards[m];
        tie += x * mult;
        if (c == p.index) id = x;
      }
      k = p.what == PASS_TIE ? tie : order_key(ORDER_CMP_LONG, p.descending != 0, p.mask, 0.0, (long long)id);
    }
    keys[i] = k;
  }
}

// keep[i] = the HAVING outcome of entries 8i .. 8i + 7 of result r (bit j: entry 8i + j exists and passes), for every
// entry of the result's chunks; exists[r] += the result's existing entries (the count numGroupsLimit is checked on)
__global__ void __launch_bounds__(kExtractThreads) having_kernel(const ExtractDesc* __restrict__ descs, int r, const pb200_having h,
                                                                 uint8_t* __restrict__ keep, unsigned long long* __restrict__ exists) {
  __shared__ uint32_t wsum[kExtractThreads / 32];
  const ExtractDesc& d = descs[r];
  const long long base = (long long)blockIdx.x * kChunk + threadIdx.x * 8;
  uint32_t flags = exists_flags(d, base);
  const uint32_t c = __reduce_add_sync(0xFFFFFFFFu, __popc(flags));   // counted first: not live across the evaluations
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
  for (int j = 0; j < 8; ++j) {
    if (!((flags >> j) & 1u)) continue;
    const long long g = base + j;
    const unsigned long long cnt = group_count(d, g);
    const bool pass = having_eval(h, [&](int a) { return final_value(d, a, g, cnt); });
    if (!pass) flags &= ~(1u << j);
  }
  keep[base >> 3] = (uint8_t)flags;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < kExtractThreads / 32; ++w) t += wsum[w];
    if (t) atomicAdd(exists + r, t);
  }
}

__global__ void gather_bitset_rows_kernel(const uint32_t* __restrict__ src, const uint32_t* __restrict__ idx, long long n, int words,
                                          uint32_t* __restrict__ dst) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n * words; i += (long long)gridDim.x * blockDim.x)
    dst[i] = src[(size_t)idx[i / words] * words + (i % words)];
}

PinnedBlock::~PinnedBlock() { pinned_free(ctx, p, bytes); }

// Lays the columns of result r out behind `off` for `rows` rows; returns the end offset.
static size_t layout_result(const pb200_result::Dense& d, ExtractDesc& e, size_t off, unsigned long long rows) {
  auto take = [&](size_t esz, size_t n) { const size_t at = off; off += (n * esz + 63) / 64 * 64; return (unsigned long long)at; };
  e.cap_rows = rows;
  e.off_keys = take(4, rows * (size_t)std::max(e.ngb, 1));
  bool need_idx = false;
  for (int a = 0; a < e.nagg; a++) need_idx |= d.dbits[a] != nullptr || e.agg[a].fn == PB200_AGG_PERCENTILE;
  e.off_idx = need_idx ? take(4, rows) : kNoCol;
  for (int a = 0; a < e.nagg; a++) {
    const int fn = e.agg[a].fn;
    e.off_dbl[a] = take(8, rows);
    e.off_lng[a] = agg_fn(fn)->long_col ? take(8, rows) : kNoCol;
    e.off_ids[a] = agg_fn(fn)->ids_col ? take(4, rows) : kNoCol;
    e.off_mom[a] = is_moments_fn(fn) ? take(24, rows) : kNoCol;
  }
  return off;
}

static int bits_for(unsigned long long max_value) {
  int b = 1;
  while (b < 64 && (max_value >> b)) ++b;
  return b;
}

// The sort passes of an ordered result in the order they run: stable LSD, so the tie key first, then the items from last
// to first.  Keys are narrowed to the bits their values can use.
static std::vector<OrderPass> order_passes(const pb200_result::Dense& d, const pb200_order_by& o, const pb200_post_aggs& post) {
  std::vector<OrderPass> ps;
  auto add = [&](OrderPass p) { p.mask = p.bits >= 64 ? ~0ull : (1ull << p.bits) - 1ull; ps.push_back(p); };
  unsigned long long space = 1;  // raw key space: bounded like the raw key (63 bits)
  for (int c : d.cards) space = space > (~0ull >> 1) / (unsigned long long)std::max(c, 1) ? ~0ull : space * (unsigned long long)std::max(c, 1);
  OrderPass tie{};
  tie.what = PASS_TIE;
  tie.bits = bits_for(space - 1);
  add(tie);
  for (int i = o.num_items - 1; i >= 0; --i) {
    const pb200_order_item& it = o.items[i];
    OrderPass p{};
    p.index = it.index;
    p.descending = it.descending != 0;
    if (it.kind == PB200_ORDER_GROUP_BY) {
      p.what = PASS_GROUP_BY; p.cmp = ORDER_CMP_LONG; p.bits = bits_for((unsigned long long)std::max(d.cards[it.index] - 1, 0));
    } else if (it.kind == PB200_ORDER_POST) {
      p.what = PASS_POST; p.cmp = ORDER_CMP_DOUBLE; p.bits = 64; p.prog = post.programs[it.index];
    } else {
      const int fn = d.aggs[it.index].function;
      p.what = PASS_AGG; p.cmp = order_cmp_of(fn);
      p.bits = fn == PB200_AGG_DISTINCTCOUNT ? bits_for(32ull * d.dwords[it.index]) : 64;
    }
    add(p);
  }
  return ps;
}

// rows an ordered result keeps of its n groups
static unsigned long long kept_rows(const pb200_result* R, unsigned long long n) {
  return (R->order.num_items > 0 && R->order.trim_size > 0) ? std::min<unsigned long long>(n, (unsigned long long)R->order.trim_size) : n;
}

int extract_groups(pb200_ctx* ctx, pb200_result* const* Rs, int nres, cudaStream_t st) {
  if (nres <= 0) return PB200_OK;
  int rc;
  std::vector<std::vector<OrderPass>> passes(nres);
  size_t order_bytes = 0;  // per ordered result: 2 index buffers [idx_cap] u32 + 2 key buffers [idx_cap] u64
  std::vector<ExtractDesc> descs(nres);
  uint32_t chunks = 0;
  bool any_having = false;
  for (int r = 0; r < nres; r++) any_having |= Rs[r]->having.num_nodes > 0;
  // header: totals (rows), then with HAVING the existing entries per result (what numGroupsLimit is checked on)
  const size_t head = 64 + 8ull * nres * (any_having ? 2 : 1);
  size_t worst = head;
  for (int r = 0; r < nres; r++) {
    const pb200_result::Dense& d = Rs[r]->dense;
    ExtractDesc& e = descs[r];
    memset(&e, 0, sizeof e);
    e.count = d.count; e.seen = d.seen; e.maxk = d.exists_max; e.mink = d.exists_min; e.hkeys = d.hkeys;
    e.packed = d.exists_packed; e.pack_shift = d.pack_shift;
    e.groups = d.groups;
    e.stride = std::max(d.stride, 1);
    e.ngb = (int)d.cards.size();
    e.nagg = (int)d.aggs.size();
    for (int k = 0; k < e.ngb; k++) e.cards[k] = (uint32_t)d.cards[k];
    agg_sources(*Rs[r], e.agg);
    e.first_chunk = chunks;
    e.num_chunks = (uint32_t)((d.groups + kChunk - 1) / kChunk);
    chunks += e.num_chunks;
    const unsigned long long cap = (unsigned long long)std::min<long long>(d.groups, (long long)d.num_groups_limit + 1);
    e.idx_cap = cap;
    worst = layout_result(d, e, worst, kept_rows(Rs[r], cap));
    if (Rs[r]->order.num_items > 0 || Rs[r]->having.num_nodes > 0) {
      for (int a = 0; a < e.nagg; a++) { e.dbits[a] = d.dbits[a]; e.dwords[a] = d.dwords[a]; }
      for (int i = 0; i < Rs[r]->having.num_nodes; i++) {
        const pb200_having_node& hn = Rs[r]->having.nodes[i];
        const bool leaf = hn.op == PB200_HAVING_RANGE || hn.op == PB200_HAVING_EQ || hn.op == PB200_HAVING_NEQ;
        if (leaf && e.agg[hn.agg].fn == PB200_AGG_DISTINCTCOUNT && !d.dbits[hn.agg]) {
          set_error("HAVING on a DISTINCTCOUNT without per-group sets"); return PB200_E_UNSUPPORTED;
        }
      }
    }
    if (Rs[r]->order.num_items > 0) {
      for (int i = 0; i < Rs[r]->order.num_items; i++) {
        const pb200_order_item& it = Rs[r]->order.items[i];
        if (it.kind == PB200_ORDER_AGG && e.agg[it.index].fn == PB200_AGG_DISTINCTCOUNT && !d.dbits[it.index]) {
          set_error("ORDER BY a DISTINCTCOUNT without per-group sets"); return PB200_E_UNSUPPORTED;
        }
        if (it.kind != PB200_ORDER_POST) continue;
        const pb200_post_program& pp = Rs[r]->post.programs[it.index];
        for (int k = 0; k < pp.num_nodes; k++)
          if (pp.nodes[k].op == PB200_POST_AGG && e.agg[pp.nodes[k].agg].fn == PB200_AGG_DISTINCTCOUNT && !d.dbits[pp.nodes[k].agg]) {
            set_error("ORDER BY an expression over a DISTINCTCOUNT without per-group sets"); return PB200_E_UNSUPPORTED;
          }
      }
      passes[r] = order_passes(d, Rs[r]->order, Rs[r]->post);
      order_bytes += (cap * 24 + 255) / 256 * 256 + 256;
    }
  }
  const bool speculative = worst <= kSpeculativeBytes;
  DevBufRaw ddesc(ctx), dcount(ctx), dtotals(ctx);
  if ((rc = ddesc.alloc(sizeof(ExtractDesc) * nres))) return rc;
  if ((rc = dcount.alloc(4ull * std::max<uint32_t>(chunks, 1)))) return rc;
  auto pin = std::make_shared<PinnedBlock>();
  pin->ctx = ctx;
  if ((rc = pinned_alloc(ctx, speculative ? worst : head, &pin->p, &pin->bytes))) return rc;
  unsigned char* out = static_cast<unsigned char*>(pin->p);
  unsigned long long* totals = reinterpret_cast<unsigned long long*>(out);  // header of the block (written by the scan kernel)
  // ---- ORDER BY buffers: v[0] takes the compaction, pass p sorts (k0, v[p % 2]) -> (k1, v[(p + 1) % 2]) ----
  DevBufRaw obuf(ctx), otemp(ctx);
  struct SortBufs { uint32_t* v[2]; unsigned long long* k[2]; };
  std::vector<SortBufs> sb(nres);
  size_t temp_bytes = 0;
  if (order_bytes) {
    if ((rc = obuf.alloc(order_bytes))) return rc;
    unsigned char* at = static_cast<unsigned char*>(obuf.p);
    for (int r = 0; r < nres; r++) {
      if (passes[r].empty()) continue;
      const size_t cap = descs[r].idx_cap;
      sb[r].k[0] = reinterpret_cast<unsigned long long*>(at); sb[r].k[1] = sb[r].k[0] + cap;
      sb[r].v[0] = reinterpret_cast<uint32_t*>(sb[r].k[1] + cap); sb[r].v[1] = sb[r].v[0] + cap;
      at += (cap * 24 + 255) / 256 * 256 + 256;
      descs[r].order_idx = sb[r].v[0];
      descs[r].order_sorted = sb[r].v[passes[r].size() % 2];
      size_t tb = 0;
      PB200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, sb[r].k[0], sb[r].k[1], sb[r].v[0], sb[r].v[1], (int)cap, 0, 64, st));
      temp_bytes = std::max(temp_bytes, tb);
    }
    if ((rc = otemp.alloc(std::max<size_t>(temp_bytes, 256)))) return rc;
  }
  // ---- HAVING: one keep byte per 8 entries of each filtered result, and its existing-entry counter ----
  DevBufRaw dkeep(ctx), dexist(ctx);
  if (any_having) {
    if ((rc = dkeep.alloc(256ull * std::max<uint32_t>(chunks, 1)))) return rc;   // kChunk / 8 bytes per chunk
    if ((rc = dexist.alloc(8ull * nres))) return rc;
    for (int r = 0; r < nres; r++)
      if (Rs[r]->having.num_nodes > 0) descs[r].keep = static_cast<const uint8_t*>(dkeep.p) + 256ull * descs[r].first_chunk;
  }
  // ---- DISTINCTSUM / DISTINCTAVG / DISTINCTCOUNTHLL: every table entry's bitset row -> its state or estimate, before
  //      HAVING, the order keys and the rows read it (entries without rows have an empty row and finalize to the empty
  //      state) ----
  std::vector<std::unique_ptr<DevBufRaw>> ds_temps;
  for (int r = 0; r < nres; r++) {
    const pb200_result::Dense& d = Rs[r]->dense;
    size_t words[kMaxAggs] = {};
    for (int b = 0; b < descs[r].nagg; b++) words[b] = d.dwords[b];
    if ((rc = finalize_sets(ctx, st, d, d.dbits, words, d.groups, false, descs[r].agg, ds_temps))) return rc;
  }
  const ExtractDesc* ddescs = (const ExtractDesc*)ddesc.p;
  PB200_CUDA(cudaMemcpyAsync(ddesc.p, descs.data(), sizeof(ExtractDesc) * nres, cudaMemcpyHostToDevice, st));
  if (any_having) {
    PB200_CUDA(cudaMemsetAsync(dexist.p, 0, 8ull * nres, st));
    for (int r = 0; r < nres; r++)
      if (descs[r].keep && descs[r].num_chunks)
        having_kernel<<<descs[r].num_chunks, kExtractThreads, 0, st>>>(ddescs, r, Rs[r]->having, const_cast<uint8_t*>(descs[r].keep),
                                                                       static_cast<unsigned long long*>(dexist.p));
    PB200_CUDA(cudaMemcpyAsync(totals + nres, dexist.p, 8ull * nres, cudaMemcpyDeviceToHost, st));
  }
  if (chunks) extract_count_kernel<<<chunks, kExtractThreads, 0, st>>>(ddescs, nres, (uint32_t*)dcount.p);
  extract_scan_kernel<<<nres, kExtractThreads, 0, st>>>(ddescs, (uint32_t*)dcount.p, totals);
  if (order_bytes && chunks) {
    extract_write_kernel<<<chunks, kExtractThreads, 0, st>>>(ddescs, nres, (const uint32_t*)dcount.p, totals, out, true);
    for (int r = 0; r < nres; r++) {
      const size_t cap = descs[r].idx_cap;
      const int grid = grid_for(ctx, (long long)cap, kExtractThreads);
      for (size_t p = 0; p < passes[r].size(); p++) {
        const OrderPass& op = passes[r][p];
        order_key_kernel<<<grid, kExtractThreads, 0, st>>>(ddescs, r, op, totals, sb[r].v[p % 2], sb[r].k[0]);
        size_t tb = temp_bytes;
        PB200_CUDA(cub::DeviceRadixSort::SortPairs(otemp.p, tb, sb[r].k[0], sb[r].k[1], sb[r].v[p % 2], sb[r].v[(p + 1) % 2],
                                                   (int)cap, 0, op.bits, st));
      }
    }
  }
  if (speculative && chunks) extract_write_kernel<<<chunks, kExtractThreads, 0, st>>>(ddescs, nres, (const uint32_t*)dcount.p, totals, out, false);
  PB200_CUDA(cudaGetLastError());
  PB200_CUDA(cudaStreamSynchronize(st));  // descs may be rewritten below: the copy above has completed
  // ---- group counts, limits ----
  std::vector<unsigned long long> n(nres), groups(nres);  // rows kept, existing groups (before HAVING)
  for (int r = 0; r < nres; r++) { n[r] = totals[r]; groups[r] = Rs[r]->having.num_nodes > 0 ? totals[nres + r] : n[r]; }
  for (int r = 0; r < nres; r++) {
    pb200_result* R = Rs[r];
    const pb200_result::Dense& d = R->dense;
    if (d.hctl) {  // hash tables: more groups than numGroupsLimit (or a full table) -> the result is unusable
      uint32_t ctl[2] = {0, 0};
      PB200_CUDA(cudaMemcpy(ctl, d.hctl, 8, cudaMemcpyDeviceToHost));
      if (ctl[1]) {
        set_error("numGroupsLimit %d would bind (hash table saw more groups): fall back to the reference operator", d.num_groups_limit);
        return PB200_E_LIMIT;
      }
    }
    R->meta.num_groups = (int32_t)kept_rows(R, n[r]);
    R->meta.groups_limit_reached = (long long)groups[r] >= d.num_groups_limit;
    if ((long long)groups[r] > d.num_groups_limit) {
      // the reference admits groups in doc order until the limit binds (IntGroupIdMap.getGroupId :1022-1047); that order
      // is not reproducible by a parallel scan -> the caller must run the Java operator for this segment
      set_error("numGroupsLimit %d would bind (%llu groups): fall back to the reference operator", d.num_groups_limit, groups[r]);
      return PB200_E_LIMIT;
    }
  }
  if (!speculative) {  // exact-size block, second pass
    size_t off = head;
    for (int r = 0; r < nres; r++) off = layout_result(Rs[r]->dense, descs[r], off, kept_rows(Rs[r], n[r]));
    auto pin2 = std::make_shared<PinnedBlock>();
    pin2->ctx = ctx;
    if ((rc = pinned_alloc(ctx, off, &pin2->p, &pin2->bytes))) return rc;
    const std::shared_ptr<PinnedBlock> header_block = pin;  // holds `totals`, which the write kernel reads, until the sync below
    pin = pin2;
    out = static_cast<unsigned char*>(pin->p);
    DevBufRaw staging(ctx);
    if ((rc = staging.alloc(off))) return rc;
    PB200_CUDA(cudaMemcpyAsync(ddesc.p, descs.data(), sizeof(ExtractDesc) * nres, cudaMemcpyHostToDevice, st));
    if (chunks) extract_write_kernel<<<chunks, kExtractThreads, 0, st>>>(ddescs, nres, (const uint32_t*)dcount.p, totals, (unsigned char*)staging.p, false);
    PB200_CUDA(cudaGetLastError());
    // the block's header is not written by the kernel
    if (off > head) PB200_CUDA(cudaMemcpyAsync(out + head, (unsigned char*)staging.p + head, off - head, cudaMemcpyDeviceToHost, st));
    PB200_CUDA(cudaStreamSynchronize(st));
  }
  // ---- results point into the block ----
  bool kept_sets = false;   // some set's rows were gathered into a result for later: wait for them before returning
  for (int r = 0; r < nres; r++) {
    pb200_result* R = Rs[r];
    const pb200_result::Dense& d = R->dense;
    const ExtractDesc& e = descs[r];
    const int nagg = e.nagg;
    R->keys.clear();
    R->dbl.assign(nagg, {}); R->lng.assign(nagg, {}); R->ids.assign(nagg, {}); R->distinct.assign(nagg, {});
    pb200_result::View& v = R->view;
    v = pb200_result::View();
    v.block = pin;
    v.rows = kept_rows(R, n[r]);
    v.keys = reinterpret_cast<const int32_t*>(out + e.off_keys);
    R->pct.row_entry = e.off_idx == kNoCol ? nullptr : reinterpret_cast<const uint32_t*>(out + e.off_idx);
    for (int a = 0; a < nagg; a++) {
      v.dbl[a] = e.off_dbl[a] == kNoCol ? nullptr : reinterpret_cast<const double*>(out + e.off_dbl[a]);
      v.lng[a] = e.off_lng[a] == kNoCol ? nullptr : reinterpret_cast<const int64_t*>(out + e.off_lng[a]);
      v.ids[a] = e.off_ids[a] == kNoCol ? nullptr : reinterpret_cast<const int32_t*>(out + e.off_ids[a]);
      R->mom.rows[a] = e.off_mom[a] == kNoCol ? nullptr : reinterpret_cast<const unsigned long long*>(out + e.off_mom[a]);
    }
    // DISTINCTCOUNT with GROUP BY: the groups' bitset rows are gathered on the device and decoded into dictId lists
    // (what extractGroupByResult's value-set conversion starts from, BaseDistinctAggregateAggregationFunction :306-321)
    std::unique_ptr<DevBufRaw> gathered[kMaxAggs];
    DevBufRaw* sets[kMaxAggs] = {};
    size_t words[kMaxAggs] = {};
    double* dbl[kMaxAggs] = {};
    int64_t* lng[kMaxAggs] = {};
    for (int b = 0; b < nagg; b++) {
      dbl[b] = const_cast<double*>(v.dbl[b]);   // the kernel left zeros for DISTINCTCOUNT: the set sizes go here
      lng[b] = const_cast<int64_t*>(v.lng[b]);
      if (!d.dbits[b]) continue;
      gathered[b].reset(new DevBufRaw(ctx));
      sets[b] = gathered[b].get();
      words[b] = d.dwords[b];
      if (!v.rows) continue;
      if ((rc = sets[b]->alloc(v.rows * words[b] * 4))) return rc;
      gather_bitset_rows_kernel<<<grid_for(ctx, (long long)(v.rows * words[b]), 256), 256, 0, st>>>(
          d.dbits[b], reinterpret_cast<const uint32_t*>(out + e.off_idx), (long long)v.rows, (int)words[b], (uint32_t*)sets[b]->p);
    }
    if ((rc = decode_sets(ctx, st, R, sets, words, v.rows, dbl, lng, &kept_sets))) return rc;
  }
  if (kept_sets) PB200_CUDA(cudaStreamSynchronize(st));   // the bitset tables may be freed once this returns
  return PB200_OK;
}

void agg_sources(const pb200_result& R, AggSource* out) {
  const pb200_result::Dense& d = R.dense;
  for (int a = 0; a < (int)d.aggs.size(); a++) {
    AggSource& s = out[a];
    s = AggSource{};
    const int fn = s.fn = d.aggs[a].function, vk = s.vk = d.val_kind[a];
    if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) {
      s.src = sum_in_double(vk) ? (void*)d.dsum[a] : (void*)d.isum[a];
      if (a == d.pack_agg) { s.pack_shift = d.pack_shift; s.pack_vmin = d.pack_vmin; }
    } else if (d.expr_tab[a]) s.xkey = static_cast<unsigned long long*>(d.expr_tab[a]);   // MIN / MAX of an expression
    else if (fn == PB200_AGG_MIN) s.src = d.gmin[a];
    else if (fn == PB200_AGG_MAX) s.src = d.gmax[a];
    else if (fn == PB200_AGG_PERCENTILE) { s.src = R.pct.ids[a]; s.pct_n = R.pct.n[R.pct.rep[a]]; }
    else if (is_withtime_fn(fn)) { s.src = R.wt.ids[a]; s.wt_time = R.wt.time[a]; }
    else if (is_moments_fn(fn)) {
      for (int j = 0; j < 3; j++) s.mom[j] = d.isum[d.mom_first[a] + j];
      s.mom_e = d.mom_e[a];
    } else if (is_distinct_value_fn(fn)) s.ds = d.ds_state[d.ds_rep[a]];
    else if (is_hll_fn(fn)) s.hll = d.hll_est[d.hll_rep[a]];
    const DeviceColumn* c = d.agg_cols[a];
    s.dict = (c && vk != VAL_RAW_I32 && !c->dict_host.empty()) ? c->dict_native : nullptr;
    s.dict_bias = 0x80000000u;   // the device copy of an INT dictionary is biased
    s.counted = d.count || d.exists_packed;
  }
}

int finalize_sets(pb200_ctx* ctx, cudaStream_t st, const pb200_result::Dense& d, const uint32_t* const* bits, const size_t* words,
                  long long rows, bool single, const AggSource* src, std::vector<std::unique_ptr<DevBufRaw>>& temps) {
  for (int a = 0; a < (int)d.aggs.size(); a++) {
    const int fn = d.aggs[a].function, b = d.ds_rep[a];
    if (!reads_distinct_set(fn)) continue;
    const DeviceColumn& c = *d.agg_cols[b];   // a reader of another aggregation's set has no scan slot of its own
    if (is_distinct_value_fn(fn)) {   // one state per set, in the table of the first aggregation that reads it
      bool done = false;
      for (int x = 0; x < a && !done; x++) done = is_distinct_value_fn(d.aggs[x].function) && d.ds_rep[x] == b;
      if (done) continue;
      const DistinctSumJob job{bits[b], words[b], rows, single, c.dict_native, c.stored_type, c.moments->ds_e, src[a].ds};
      if (int rc = distinct_sum_finalize(ctx, st, job, temps)) return rc;
    } else if (is_hll_fn(fn) && d.hll_rep[a] == a) {   // one estimate per column and log2m
      const HllJob job{bits[b], words[b], rows, single, c.moments->hll_hash, d.hll_log2m[a], src[a].hll};
      if (int rc = hll_finalize(ctx, st, job, temps)) return rc;
    }
  }
  return PB200_OK;
}

int decode_sets(pb200_ctx* ctx, cudaStream_t st, pb200_result* R, DevBufRaw* const* sets, const size_t* words, size_t rows,
                double* const* dbl, int64_t* const* lng, bool* kept) {
  const pb200_result::Dense& d = R->dense;
  const int nagg = (int)d.aggs.size();
  std::vector<int> decoded(nagg, -1);   // the bitset aggregation a's set was decoded from
  std::vector<int32_t> fns(nagg);
  for (int a = 0; a < nagg; a++) fns[a] = d.aggs[a].function;
  for (int a = 0; a < nagg; a++) {
    const bool value_fn = reads_distinct_set(fns[a]);
    const int b = value_fn ? d.ds_rep[a] : a;
    if ((fns[a] != PB200_AGG_DISTINCTCOUNT && !value_fn) || b < 0 || !sets[b]) continue;
    decoded[a] = b;
    const bool lazy = hll_only_set_of(fns.data(), d.ds_rep, nagg, b);
    if (lazy) R->lazy.src[a] = b;
    const int same = (int)(std::find(decoded.begin(), decoded.begin() + a, b) - decoded.begin());
    if (same < a) { if (!lazy) R->distinct[a] = R->distinct[same]; continue; }
    if (lazy) {   // owned by the result from here on; the stream orders the rows' writes before any later copy of them
      pb200_result::LazySets& L = R->lazy;
      dev_free(ctx, L.bits[b]);   // a result extracted again (pb200_result_finalize) replaces its rows
      L.ctx = ctx; L.bits[b] = static_cast<uint32_t*>(sets[b]->p); L.words[b] = words[b]; L.rows[b] = rows;
      sets[b]->p = nullptr;
      *kept |= L.bits[b] != nullptr;
      continue;
    }
    std::vector<uint32_t> bits(rows * words[b]);
    if (!bits.empty()) {
      PB200_CUDA(cudaMemcpyAsync(bits.data(), sets[b]->p, bits.size() * 4, cudaMemcpyDeviceToHost, st));
      PB200_CUDA(cudaStreamSynchronize(st));
    }
    R->distinct[a].resize(rows);
    for (size_t i = 0; i < rows; i++) {
      R->distinct[a][i] = bitset_ids(bits.data() + i * words[b], words[b]);
      if (!value_fn) { lng[a][i] = (int64_t)R->distinct[a][i].size(); dbl[a][i] = (double)lng[a][i]; }
    }
  }
  return PB200_OK;
}

std::vector<int32_t> bitset_ids(const uint32_t* bits, size_t words) {
  std::vector<int32_t> ids;
  for (size_t w = 0; w < words; w++) for (uint32_t x = bits[w]; x; x &= x - 1) ids.push_back((int32_t)(w * 32 + __builtin_ctz(x)));
  return ids;
}

// Copies a view-backed result into the std::vector fields (host-side consumers that re-map results: star-tree).
void result_materialize(pb200_result* R) {
  pb200_result::View& v = R->view;
  if (!v.block) return;
  const size_t rows = v.rows, ngb = (size_t)R->meta.num_group_by, nagg = (size_t)R->meta.num_aggs;
  R->keys.assign(v.keys, v.keys + rows * ngb);
  R->dbl.resize(nagg); R->lng.resize(nagg); R->ids.resize(nagg);
  for (size_t a = 0; a < nagg; a++) {
    if (v.dbl[a]) R->dbl[a].assign(v.dbl[a], v.dbl[a] + rows); else R->dbl[a].assign(rows, 0.0);
    if (v.lng[a]) R->lng[a].assign(v.lng[a], v.lng[a] + rows); else R->lng[a].assign(rows, 0);
    if (v.ids[a]) R->ids[a].assign(v.ids[a], v.ids[a] + rows); else R->ids[a].assign(rows, -1);
  }
  v = pb200_result::View();
}

int order_validate(const pb200_order_by* o, int num_aggs, int num_group_by, const pb200_post_aggs* post) {
  if (post) {
    if (post->num_programs < 0 || post->num_programs > PB200_MAX_ORDER_BY) {
      set_error("%d post-aggregation programs (0..%d)", post->num_programs, PB200_MAX_ORDER_BY);
      return PB200_E_INVALID;
    }
    for (int i = 0; i < post->num_programs; i++)
      if (const char* why = postagg_validate(&post->programs[i], num_aggs)) { set_error("program %d: %s", i, why); return PB200_E_INVALID; }
  }
  if (!o) return PB200_OK;
  if (o->num_items < 1 || o->num_items > PB200_MAX_ORDER_BY) {
    set_error("ORDER BY has %d items (1..%d)", o->num_items, PB200_MAX_ORDER_BY);
    return PB200_E_INVALID;
  }
  for (int i = 0; i < o->num_items; i++) {
    const pb200_order_item& it = o->items[i];
    const int bound = it.kind == PB200_ORDER_AGG        ? num_aggs
                      : it.kind == PB200_ORDER_GROUP_BY ? num_group_by
                      : it.kind == PB200_ORDER_POST     ? (post ? post->num_programs : 0)
                                                        : 0;
    if (it.index < 0 || it.index >= bound) {
      set_error("ORDER BY item %d: kind %d index %d is out of range", i, it.kind, it.index);
      return PB200_E_INVALID;
    }
  }
  return PB200_OK;
}

void order_rows_host(pb200_result* R, const pb200_order_by& o, const int32_t* fns, const pb200_post_aggs* post) {
  if (R->meta.num_groups < 0) return;
  const size_t rows = (size_t)R->meta.num_groups, ngb = (size_t)R->meta.num_group_by, nagg = (size_t)R->meta.num_aggs;
  const pb200_result::View& v = R->view;
  // the rows' columns, wherever they live (a view-backed result may alias its vectors: read before anything is rewritten)
  std::vector<int32_t> keys = v.block ? std::vector<int32_t>(v.keys, v.keys + rows * ngb) : R->keys;
  std::vector<std::vector<double>> dbl(nagg);
  std::vector<std::vector<int64_t>> lng(nagg);
  std::vector<std::vector<int32_t>> ids(nagg);
  for (size_t a = 0; a < nagg; a++) {
    if (v.block) {
      dbl[a] = v.dbl[a] ? std::vector<double>(v.dbl[a], v.dbl[a] + rows) : std::vector<double>(rows, 0.0);
      lng[a] = v.lng[a] ? std::vector<int64_t>(v.lng[a], v.lng[a] + rows) : std::vector<int64_t>(rows, 0);
      ids[a] = v.ids[a] ? std::vector<int32_t>(v.ids[a], v.ids[a] + rows) : std::vector<int32_t>(rows, -1);
    } else {
      dbl[a] = R->dbl[a]; lng[a] = R->lng[a]; ids[a] = R->ids[a];
    }
  }
  std::vector<std::vector<uint64_t>> ok(o.num_items, std::vector<uint64_t>(rows));
  for (int i = 0; i < o.num_items; i++) {
    const pb200_order_item& it = o.items[i];
    for (size_t r = 0; r < rows; r++) {
      if (it.kind == PB200_ORDER_POST) {
        const double v = postagg_eval(post->programs[it.index], [&](int a) { return having_value(fns[a], dbl[a][r], lng[a][r]); });
        ok[i][r] = order_key(ORDER_CMP_DOUBLE, it.descending != 0, ~0ull, v, 0);
        continue;
      }
      ok[i][r] = it.kind == PB200_ORDER_GROUP_BY
                     ? order_key(ORDER_CMP_LONG, it.descending != 0, ~0ull, 0.0, (int64_t)(uint32_t)keys[r * ngb + it.index])
                     : order_key(order_cmp_of(fns[it.index]), it.descending != 0, ~0ull, dbl[it.index][r], lng[it.index][r]);
    }
  }
  std::vector<size_t> perm(rows);
  for (size_t r = 0; r < rows; r++) perm[r] = r;
  std::sort(perm.begin(), perm.end(), [&](size_t x, size_t y) {
    for (int i = 0; i < o.num_items; i++) if (ok[i][x] != ok[i][y]) return ok[i][x] < ok[i][y];
    for (size_t k = 0; k < ngb; k++)
      if (keys[x * ngb + k] != keys[y * ngb + k]) return (uint32_t)keys[x * ngb + k] < (uint32_t)keys[y * ngb + k];
    return x < y;
  });
  const size_t kept = o.trim_size > 0 ? std::min(rows, (size_t)o.trim_size) : rows;
  R->keys.resize(kept * ngb);
  R->dbl.assign(nagg, {}); R->lng.assign(nagg, {}); R->ids.assign(nagg, {});
  std::vector<std::vector<std::vector<int32_t>>> distinct(R->distinct.size());
  for (size_t j = 0; j < kept; j++) {
    const size_t r = perm[j];
    for (size_t k = 0; k < ngb; k++) R->keys[j * ngb + k] = keys[r * ngb + k];
    for (size_t a = 0; a < nagg; a++) { R->dbl[a].push_back(dbl[a][r]); R->lng[a].push_back(lng[a][r]); R->ids[a].push_back(ids[a][r]); }
    for (size_t a = 0; a < distinct.size(); a++)
      if (R->distinct[a].size() == rows) distinct[a].push_back(std::move(R->distinct[a][r]));
  }
  R->distinct = std::move(distinct);
  R->view = pb200_result::View();
  R->meta.num_groups = (int32_t)kept;
}

int having_check(const pb200_having* h, int num_aggs, int num_group_by, int nres, bool deferred) {
  if (!h) return PB200_OK;
  if (const char* why = having_validate(h, num_aggs)) { set_error("%s", why); return PB200_E_INVALID; }
  if (num_group_by <= 0) { set_error("HAVING needs a GROUP BY"); return PB200_E_INVALID; }
  if (nres != 1) {
    set_error("HAVING needs a final result: merge the segments or pass one (a call writing %d per-segment results is not final)", nres);
    return PB200_E_INVALID;
  }
  if (deferred) { set_error("HAVING across GPUs (PB200_Q_DEFER_FINALIZE, reduce_world > 1) is not accelerated"); return PB200_E_UNSUPPORTED; }
  return PB200_OK;
}

void having_rows_host(pb200_result* R, const pb200_having& h, const int32_t* fns) {
  R->having = h;
  if (R->meta.num_groups < 0) return;
  result_materialize(R);
  const size_t rows = (size_t)R->meta.num_groups, ngb = (size_t)R->meta.num_group_by, nagg = (size_t)R->meta.num_aggs;
  size_t kept = 0;
  for (size_t r = 0; r < rows; r++) {
    if (!having_eval(h, [&](int a) { return having_value(fns[a], R->dbl[a][r], R->lng[a][r]); })) continue;
    for (size_t k = 0; k < ngb; k++) R->keys[kept * ngb + k] = R->keys[r * ngb + k];
    for (size_t a = 0; a < nagg; a++) { R->dbl[a][kept] = R->dbl[a][r]; R->lng[a][kept] = R->lng[a][r]; R->ids[a][kept] = R->ids[a][r]; }
    if (kept != r)
      for (auto& d : R->distinct) if (d.size() == rows) d[kept] = std::move(d[r]);
    ++kept;
  }
  R->keys.resize(kept * ngb);
  for (size_t a = 0; a < nagg; a++) { R->dbl[a].resize(kept); R->lng[a].resize(kept); R->ids[a].resize(kept); }
  for (auto& d : R->distinct) if (d.size() == rows) d.resize(kept);
  R->meta.num_groups = (int32_t)kept;
}

}  // namespace pb200
