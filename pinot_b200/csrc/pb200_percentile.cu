// pb200_percentile.cu -- PERCENTILE finalize: per-group dictId histograms -> the selected dictId of every row.
//
// The reference keeps every matched value of a group in a DoubleArrayList, sorts it and takes one index
// (PercentileAggregationFunction.extractFinalResult).  A dictionary is sorted, so the scan kernel keeps a histogram of
// counts over dictIds instead (pb200_scan.cuh, function 6) -- the sorted list in compact form -- and the k-th smallest
// value is the dictionary value at the first dictId whose cumulative count passes k.  Two launches per histogram, both
// spread over the whole GPU (the cost scales with the histogram's bytes, not with one SM per row):
//   chunk sums  one warp per 1024-entry chunk of a row: the chunk's count;
//   select      one warp per row: n = sum of its chunk sums, then per percentile the chunk and, inside it, the entry where
//               the cumulative count first exceeds the index rule's k (pb200_desc.h percentile_index).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>

#include "pb200_internal.h"
#include "pb200_percentile.h"

namespace pb200 {

constexpr uint32_t kHistChunk = 1024;   // entries per chunk (one warp reads 32 per lane)
constexpr int kHistThreads = 256;

__global__ void __launch_bounds__(kHistThreads) hist_chunk_sum_kernel(const uint32_t* __restrict__ hist, long long rows, uint32_t E,
                                                                      uint32_t nchunks, uint32_t* __restrict__ sums) {
  const int lane = threadIdx.x & 31;
  const long long nw = rows * nchunks;
  for (long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; w < nw; w += ((long long)gridDim.x * blockDim.x) >> 5) {
    const long long row = w / nchunks;
    const uint32_t c = (uint32_t)(w - row * nchunks);
    const uint32_t* h = hist + (size_t)row * E;
    const uint32_t lo = c * kHistChunk, hi = min(E, lo + kHistChunk);
    uint32_t s = 0;   // a chunk of one result holds fewer than 2^32 rows (plan_scan refuses larger results)
    for (uint32_t i = lo + lane; i < hi; i += 32) s += __ldg(h + i);
    s = __reduce_add_sync(0xFFFFFFFFu, s);
    if (lane == 0) sums[w] = s;
  }
}

// Position of the (k+1)-th smallest count unit among `n` u32 values read by get(i), i < n, walked 32 at a time by one warp:
// returns the index i and leaves in *k the rank inside entry i.  Requires k < sum of all values.
template <typename Get>
__device__ __forceinline__ uint32_t warp_find(uint32_t n, unsigned long long* k, Get get) {
  const int lane = threadIdx.x & 31;
  unsigned long long before = 0;   // total of the entries already passed
  for (uint32_t base = 0; base < n; base += 32) {
    const uint32_t i = base + lane;
    const unsigned long long v = i < n ? (unsigned long long)get(i) : 0ull;
    unsigned long long incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
    const unsigned found = __ballot_sync(0xFFFFFFFFu, before + incl > *k);
    if (found) {
      const int src = __ffs(found) - 1;
      const unsigned long long excl = __shfl_sync(0xFFFFFFFFu, incl - v, src);
      *k -= before + excl;
      return base + (uint32_t)src;
    }
    before += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
  return n;   // not reached when k < total
}

__global__ void __launch_bounds__(kHistThreads) hist_select_kernel(PercentileJob j, const uint32_t* __restrict__ sums) {
  const int lane = threadIdx.x & 31;
  for (long long row = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; row < j.rows;
       row += ((long long)gridDim.x * blockDim.x) >> 5) {
    const uint32_t* rs = sums + (size_t)row * j.nchunks;
    unsigned long long n = 0;
    for (uint32_t c = lane; c < j.nchunks; c += 32) n += rs[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xFFFFFFFFu, n, o);
    if (lane == 0 && j.n_out) j.n_out[row] = (uint32_t)n;
    const uint32_t* h = j.hist + (size_t)row * j.E;
    for (int a = 0; a < j.np; ++a) {
      uint32_t id = ~0u;   // no matched row: -inf
      if (n > 0) {
        unsigned long long k = (unsigned long long)percentile_index((long long)n, j.p[a]);
        const uint32_t c = warp_find(j.nchunks, &k, [&](uint32_t i) { return rs[i]; });
        const uint32_t lo = c * kHistChunk, cn = min(j.E - lo, kHistChunk);
        id = lo + warp_find(cn, &k, [&](uint32_t i) { return __ldg(h + lo + i); });
      }
      if (lane == 0) j.ids[a][row] = id;
    }
  }
}

__global__ void hist_gather_rows_kernel(const uint32_t* __restrict__ hist, const uint32_t* __restrict__ idx, long long rows,
                                        uint32_t E, uint32_t* __restrict__ dst) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < rows * (long long)E; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / E;
    dst[i] = hist[(size_t)idx[r] * E + (i - r * E)];
  }
}

int percentile_finalize(pb200_ctx* ctx, cudaStream_t st, const PercentileJob& job, std::vector<std::unique_ptr<DevBufRaw>>& temps) {
  if (job.rows <= 0 || job.np <= 0) return PB200_OK;
  PercentileJob j = job;
  j.nchunks = (j.E + kHistChunk - 1) / kHistChunk;
  temps.emplace_back(new DevBufRaw(ctx));
  if (int rc = temps.back()->alloc(4ull * (size_t)j.rows * j.nchunks)) return rc;
  uint32_t* sums = static_cast<uint32_t*>(temps.back()->p);
  const long long warps1 = j.rows * (long long)j.nchunks;
  hist_chunk_sum_kernel<<<grid_for(ctx, warps1 * 32, kHistThreads), kHistThreads, 0, st>>>(j.hist, j.rows, j.E, j.nchunks, sums);
  hist_select_kernel<<<grid_for(ctx, j.rows * 32, kHistThreads), kHistThreads, 0, st>>>(j, sums);
  PB200_CUDA(cudaGetLastError());
  return PB200_OK;
}

int percentile_read_rows(pb200_ctx* ctx, const uint32_t* hist, const uint32_t* idx, long long rows, uint32_t E,
                         std::vector<uint32_t>& out) {
  out.assign((size_t)rows * E, 0u);
  if (!rows || !E) return PB200_OK;
  PB200_CUDA(cudaSetDevice(ctx->device));
  StreamLease st(ctx);
  DevBufRaw rows_dev(ctx), g(ctx);
  const uint32_t* src = hist;
  if (idx) {   // group-by: the histogram rows of the result's rows, in row order
    if (int rc = rows_dev.alloc(4ull * rows)) return rc;
    if (int rc = g.alloc(4ull * rows * E)) return rc;
    PB200_CUDA(cudaMemcpyAsync(rows_dev.p, idx, 4ull * rows, cudaMemcpyHostToDevice, st));
    hist_gather_rows_kernel<<<grid_for(ctx, rows * (long long)E, 256), 256, 0, st>>>(hist, (const uint32_t*)rows_dev.p, rows, E, (uint32_t*)g.p);
    PB200_CUDA(cudaGetLastError());
    src = (const uint32_t*)g.p;
  }
  PB200_CUDA(cudaMemcpyAsync(out.data(), src, 4ull * rows * E, cudaMemcpyDeviceToHost, st));
  PB200_CUDA(cudaStreamSynchronize(st));
  return PB200_OK;
}

}  // namespace pb200

using namespace pb200;

extern "C" int64_t pb200_result_histogram(const pb200_result* Rc, int32_t a, int32_t row, int32_t* dict_ids, int64_t* counts,
                                          int64_t capacity) {
  if (!Rc || a < 0 || a >= Rc->meta.num_aggs || a >= kMaxAggs) { set_error("bad aggregation index"); return PB200_E_INVALID; }
  pb200_result* R = const_cast<pb200_result*>(Rc);   // the lazily copied histograms are a cache of the result's own state
  pb200_result::Pct& p = R->pct;
  const int owner = p.rep[a];
  if (owner < 0 || !p.hist[owner]) {
    if (R->agg_functions.empty()) return 0;   // answered on the host without a scan (no matched doc): no bins
    set_error("aggregation %d has no PERCENTILE histogram", a);
    return PB200_E_INVALID;
  }
  const long long rows = R->meta.num_groups < 0 ? 1 : R->meta.num_groups;
  if (row < 0 || row >= rows) { set_error("bad row %d (%lld rows)", row, rows); return PB200_E_INVALID; }
  const uint32_t E = p.entries[owner];
  if (p.host[owner].empty() && rows > 0) {
    if (R->meta.num_groups >= 0 && !p.row_entry) { set_error("result rows have no table entries"); return PB200_E_INVALID; }
    if (int rc = percentile_read_rows(p.ctx, p.hist[owner], R->meta.num_groups < 0 ? nullptr : p.row_entry, rows, E, p.host[owner])) return rc;
  }
  const uint32_t* h = p.host[owner].data() + (size_t)row * E;
  int64_t m = 0;
  for (uint32_t i = 0; i < E; i++) {
    if (!h[i]) continue;
    if (m < capacity) {
      if (dict_ids) dict_ids[m] = (int32_t)i;
      if (counts) counts[m] = h[i];
    }
    m++;
  }
  return m;
}
