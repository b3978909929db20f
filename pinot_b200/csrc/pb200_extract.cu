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
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "pb200_internal.h"

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
  const unsigned long long* packed;  // count-carrying sum table (pb200_api.cu): sum(value - vmin) + count << shift
  long long pack_vmin;
  int32_t pack_agg, pack_shift;
  long long groups;                  // table entries (dense: raw key space x stride, hash: capacity)
  int32_t stride, pad_stride;        // dense tables: only entries at multiples of `stride` are ever written
  int32_t ngb, nagg;
  uint32_t cards[kMaxGroupBy];
  uint32_t first_chunk, num_chunks;  // position in the launch-wide chunk sequence
  unsigned long long cap_rows;       // rows every column has room for
  unsigned long long off_keys;       // int32 [rows x ngb]
  unsigned long long off_idx;        // uint32 [rows] raw key / slot (only when a per-group bitset has to be gathered), else kNoCol
  unsigned long long off_dbl[kMaxAggs], off_lng[kMaxAggs], off_ids[kMaxAggs];  // kNoCol: column not produced
  const void* src[kMaxAggs];         // accumulator table of the aggregation (NULL: COUNT)
  const void* dict[kMaxAggs];        // device dictionary for the MIN / MAX value lookup (NULL: the id itself is the value)
  int32_t fn[kMaxAggs], vk[kMaxAggs];
};

__device__ __forceinline__ bool non_empty(const ExtractDesc& d, long long i) {
  if (d.hkeys) return d.hkeys[i] != ~0ull;
  if (d.packed) return d.packed[i] != 0ull;
  return (d.count && d.count[i] != 0ull) || (d.seen && d.seen[i] != 0u) || (d.maxk && d.maxk[i] != 0u) || (d.mink && d.mink[i] != 0xFFFFFFFFu);
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
  uint32_t c = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) c += (base + j < d.groups && non_empty(d, base + j)) ? 1u : 0u;
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

__global__ void __launch_bounds__(kExtractThreads) extract_write_kernel(const ExtractDesc* __restrict__ descs, int nres,
                                                                        const uint32_t* __restrict__ chunk_off,
                                                                        unsigned char* __restrict__ out) {
  __shared__ uint32_t wsum[kExtractThreads / 32];
  const int r = find_result(descs, nres, blockIdx.x);
  const ExtractDesc& d = descs[r];
  const long long base = (long long)(blockIdx.x - d.first_chunk) * kChunk + threadIdx.x * 8;
  uint32_t flags = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) flags |= ((base + j < d.groups && non_empty(d, base + j)) ? 1u : 0u) << j;
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
  for (int j = 0; j < 8; ++j) {
    if (!((flags >> j) & 1u)) continue;
    if (row >= d.cap_rows) return;  // more groups than the block has room for (numGroupsLimit bound: the caller discards the result)
    const long long g = base + j;
    // ---- key dictIds: raw key = sum dictId_k * prod_{m<k} card_m (column 0 least significant) ----
    if (d.ngb > 0) {
      int32_t* kp = reinterpret_cast<int32_t*>(out + d.off_keys) + row * d.ngb;
      unsigned long long raw = d.hkeys ? d.hkeys[g] : (unsigned long long)g / (unsigned)d.stride;
      for (int k = 0; k < d.ngb; ++k) { kp[k] = (int32_t)(raw % d.cards[k]); raw /= d.cards[k]; }
    }
    if (d.off_idx != kNoCol) reinterpret_cast<uint32_t*>(out + d.off_idx)[row] = (uint32_t)g;
    const unsigned long long cnt = d.packed ? d.packed[g] >> d.pack_shift : (d.count ? d.count[g] : 0ull);
    for (int a = 0; a < d.nagg; ++a) {
      const int fn = d.fn[a], vk = d.vk[a];
      double dv = 0.0;
      long long lv = 0;
      int32_t id = -1;
      if (fn == PB200_AGG_COUNT) { lv = (long long)cnt; dv = (double)cnt; }
      else if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) {
        if (a == d.pack_agg) {  // low field = sum(value - vmin): exact integer arithmetic, then to double like every sum
          const unsigned long long f = d.packed[g] & ((1ull << d.pack_shift) - 1ull);
          dv = (double)((long long)f + (long long)cnt * d.pack_vmin);
        } else {
          dv = sum_in_double(vk) ? static_cast<const double*>(d.src[a])[g] : (double)static_cast<const long long*>(d.src[a])[g];
        }
        lv = (long long)cnt;
      } else if (fn == PB200_AGG_MIN || fn == PB200_AGG_MAX) {
        const uint32_t t = static_cast<const uint32_t*>(d.src[a])[g];
        // every row of a submission reaches each of its functions, so a group that exists has a MIN / MAX.  Raw INT entries
        // are all values (max_offset): 0xFFFFFFFF / 0 are INT_MAX / INT_MIN there, never "empty"
        const bool empty = vk != VAL_RAW_I32 && (fn == PB200_AGG_MIN ? t == 0xFFFFFFFFu : t == 0u);
        if (empty) dv = fn == PB200_AGG_MIN ? INFINITY : -INFINITY;
        else {
          const uint32_t x = fn == PB200_AGG_MIN ? t : t - max_offset(vk);
          id = (int32_t)x;
          if (vk == VAL_RAW_I32) dv = (double)(int32_t)(x ^ 0x80000000u);
          else if (!d.dict[a]) dv = (double)x;
          else if (vk == VAL_DICT_I32) dv = (double)(int32_t)(static_cast<const uint32_t*>(d.dict[a])[x] ^ 0x80000000u);  // device copy is biased
          else if (vk == VAL_DICT_I64) dv = (double)static_cast<const long long*>(d.dict[a])[x];
          else if (vk == VAL_DICT_F32) dv = (double)static_cast<const float*>(d.dict[a])[x];
          else dv = static_cast<const double*>(d.dict[a])[x];
        }
      }
      if (d.off_dbl[a] != kNoCol) reinterpret_cast<double*>(out + d.off_dbl[a])[row] = dv;
      if (d.off_lng[a] != kNoCol) reinterpret_cast<long long*>(out + d.off_lng[a])[row] = lv;
      if (d.off_ids[a] != kNoCol) reinterpret_cast<int32_t*>(out + d.off_ids[a])[row] = id;
    }
    ++row;
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
  for (int a = 0; a < e.nagg; a++) need_idx |= d.dbits[a] != nullptr;
  e.off_idx = need_idx ? take(4, rows) : kNoCol;
  for (int a = 0; a < e.nagg; a++) {
    const int fn = e.fn[a];
    e.off_dbl[a] = take(8, rows);
    e.off_lng[a] = (fn == PB200_AGG_COUNT || fn == PB200_AGG_AVG || fn == PB200_AGG_SUM || fn == PB200_AGG_DISTINCTCOUNT) ? take(8, rows) : kNoCol;
    e.off_ids[a] = (fn == PB200_AGG_MIN || fn == PB200_AGG_MAX) ? take(4, rows) : kNoCol;
  }
  return off;
}

int extract_groups(pb200_ctx* ctx, pb200_result* const* Rs, int nres, cudaStream_t st) {
  if (nres <= 0) return PB200_OK;
  int rc;
  std::vector<ExtractDesc> descs(nres);
  uint32_t chunks = 0;
  size_t worst = 64 + 8ull * nres;  // header: totals
  for (int r = 0; r < nres; r++) {
    const pb200_result::Dense& d = Rs[r]->dense;
    ExtractDesc& e = descs[r];
    memset(&e, 0, sizeof e);
    e.count = d.count; e.seen = d.seen; e.maxk = d.exists_max; e.mink = d.exists_min; e.hkeys = d.hkeys;
    e.packed = d.exists_packed; e.pack_agg = d.pack_agg; e.pack_shift = d.pack_shift; e.pack_vmin = d.pack_vmin;
    e.groups = d.groups;
    e.stride = std::max(d.stride, 1);
    e.ngb = (int)d.cards.size();
    e.nagg = (int)d.aggs.size();
    for (int k = 0; k < e.ngb; k++) e.cards[k] = (uint32_t)d.cards[k];
    for (int a = 0; a < e.nagg; a++) {
      const int fn = d.aggs[a].function, vk = d.val_kind[a];
      e.fn[a] = fn; e.vk[a] = vk;
      if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) e.src[a] = sum_in_double(vk) ? (const void*)d.dsum[a] : (const void*)d.isum[a];
      else if (fn == PB200_AGG_MIN) e.src[a] = d.gmin[a];
      else if (fn == PB200_AGG_MAX) e.src[a] = d.gmax[a];
      const DeviceColumn* c = d.agg_cols[a];
      e.dict[a] = (c && vk != VAL_RAW_I32 && !c->dict_host.empty()) ? c->dict_native : nullptr;
    }
    e.first_chunk = chunks;
    e.num_chunks = (uint32_t)((d.groups + kChunk - 1) / kChunk);
    chunks += e.num_chunks;
    const unsigned long long cap = (unsigned long long)std::min<long long>(d.groups, (long long)d.num_groups_limit + 1);
    worst = layout_result(d, e, worst, cap);
  }
  const bool speculative = worst <= kSpeculativeBytes;
  DevBufRaw ddesc(ctx), dcount(ctx), dtotals(ctx);
  if ((rc = ddesc.alloc(sizeof(ExtractDesc) * nres))) return rc;
  if ((rc = dcount.alloc(4ull * std::max<uint32_t>(chunks, 1)))) return rc;
  auto pin = std::make_shared<PinnedBlock>();
  pin->ctx = ctx;
  if ((rc = pinned_alloc(ctx, speculative ? worst : 64 + 8ull * nres, &pin->p, &pin->bytes))) return rc;
  unsigned char* out = static_cast<unsigned char*>(pin->p);
  unsigned long long* totals = reinterpret_cast<unsigned long long*>(out);  // header of the block (written by the scan kernel)
  PB200_CUDA(cudaMemcpyAsync(ddesc.p, descs.data(), sizeof(ExtractDesc) * nres, cudaMemcpyHostToDevice, st));
  if (chunks) extract_count_kernel<<<chunks, kExtractThreads, 0, st>>>((const ExtractDesc*)ddesc.p, nres, (uint32_t*)dcount.p);
  extract_scan_kernel<<<nres, kExtractThreads, 0, st>>>((const ExtractDesc*)ddesc.p, (uint32_t*)dcount.p, totals);
  if (speculative && chunks) extract_write_kernel<<<chunks, kExtractThreads, 0, st>>>((const ExtractDesc*)ddesc.p, nres, (const uint32_t*)dcount.p, out);
  PB200_CUDA(cudaGetLastError());
  PB200_CUDA(cudaStreamSynchronize(st));  // descs may be rewritten below: the copy above has completed
  // ---- group counts, limits ----
  std::vector<unsigned long long> n(nres);
  for (int r = 0; r < nres; r++) n[r] = totals[r];
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
    R->meta.num_groups = (int32_t)n[r];
    R->meta.groups_limit_reached = (long long)n[r] >= d.num_groups_limit;
    if ((long long)n[r] > d.num_groups_limit) {
      // the reference admits groups in doc order until the limit binds (IntGroupIdMap.getGroupId :1022-1047); that order
      // is not reproducible by a parallel scan -> the caller must run the Java operator for this segment
      set_error("numGroupsLimit %d would bind (%llu groups): fall back to the reference operator", d.num_groups_limit, n[r]);
      return PB200_E_LIMIT;
    }
  }
  if (!speculative) {  // exact-size block, second pass
    size_t off = 64 + 8ull * nres;
    for (int r = 0; r < nres; r++) off = layout_result(Rs[r]->dense, descs[r], off, n[r]);
    auto pin2 = std::make_shared<PinnedBlock>();
    pin2->ctx = ctx;
    if ((rc = pinned_alloc(ctx, off, &pin2->p, &pin2->bytes))) return rc;
    pin = pin2;
    out = static_cast<unsigned char*>(pin->p);
    DevBufRaw staging(ctx);
    if ((rc = staging.alloc(off))) return rc;
    PB200_CUDA(cudaMemcpyAsync(ddesc.p, descs.data(), sizeof(ExtractDesc) * nres, cudaMemcpyHostToDevice, st));
    if (chunks) extract_write_kernel<<<chunks, kExtractThreads, 0, st>>>((const ExtractDesc*)ddesc.p, nres, (const uint32_t*)dcount.p, (unsigned char*)staging.p);
    PB200_CUDA(cudaGetLastError());
    const size_t head = 64 + 8ull * nres;  // the block's header is not written by the kernel
    if (off > head) PB200_CUDA(cudaMemcpyAsync(out + head, (unsigned char*)staging.p + head, off - head, cudaMemcpyDeviceToHost, st));
    PB200_CUDA(cudaStreamSynchronize(st));
  }
  // ---- results point into the block ----
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
    v.rows = n[r];
    v.keys = reinterpret_cast<const int32_t*>(out + e.off_keys);
    for (int a = 0; a < nagg; a++) {
      v.dbl[a] = e.off_dbl[a] == kNoCol ? nullptr : reinterpret_cast<const double*>(out + e.off_dbl[a]);
      v.lng[a] = e.off_lng[a] == kNoCol ? nullptr : reinterpret_cast<const int64_t*>(out + e.off_lng[a]);
      v.ids[a] = e.off_ids[a] == kNoCol ? nullptr : reinterpret_cast<const int32_t*>(out + e.off_ids[a]);
    }
    // DISTINCTCOUNT with GROUP BY: the groups' bitset rows are gathered on the device and decoded here into dictId lists
    // (what extractGroupByResult's value-set conversion starts from, BaseDistinctAggregateAggregationFunction :306-321)
    for (int a = 0; a < nagg; a++) {
      if (d.aggs[a].function != PB200_AGG_DISTINCTCOUNT || !d.dbits[a]) continue;
      const size_t wpg = d.dwords[a], rows = (size_t)n[r];
      std::vector<uint32_t> bits(rows * wpg);
      if (rows) {
        DevBufRaw g(ctx);
        if ((rc = g.alloc(rows * wpg * 4))) return rc;
        const int gb2 = (int)std::max<size_t>(1, std::min<size_t>((rows * wpg + 255) / 256, (size_t)ctx->sm_count * 8));
        gather_bitset_rows_kernel<<<gb2, 256, 0, st>>>(d.dbits[a], reinterpret_cast<const uint32_t*>(out + e.off_idx), (long long)rows, (int)wpg, (uint32_t*)g.p);
        PB200_CUDA(cudaMemcpyAsync(bits.data(), g.p, rows * wpg * 4, cudaMemcpyDeviceToHost, st));
        PB200_CUDA(cudaStreamSynchronize(st));
      }
      R->distinct[a].resize(rows);
      int64_t* sizes = const_cast<int64_t*>(v.lng[a]);   // the kernel left zeros: the set sizes go here
      double* dsz = const_cast<double*>(v.dbl[a]);
      for (size_t i = 0; i < rows; i++) {
        std::vector<int32_t>& ids = R->distinct[a][i];
        for (size_t w = 0; w < wpg; w++) { uint32_t x = bits[i * wpg + w]; while (x) { ids.push_back((int32_t)(w * 32 + __builtin_ctz(x))); x &= x - 1; } }
        sizes[i] = (int64_t)ids.size(); dsz[i] = (double)ids.size();
      }
    }
  }
  return PB200_OK;
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

}  // namespace pb200
