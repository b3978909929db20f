// pb200_withtime.cu -- FIRSTWITHTIME / LASTWITHTIME finalize: one thread per key decodes the winning row.
//
// The scan leaves per result (or per group / slot) the best key (time dictId << 32) | row ordinal.  The ordinal names the
// segment (binary search over the doc bases of the call) and the doc id; the thread unpacks the data column's dictId at
// that doc from the resident forward index and looks the time value up in the time column's dictionary.  The data
// column's value is read once per result row, never per scanned row.
#include "pb200_withtime.h"

#include "pb200_unpack.cuh"

namespace pb200 {
namespace {

constexpr int kWtThreads = 256;

// dictId of doc `doc` in a packed forward index: the doc's 32-row group occupies `bits` words (pb200_scan.cuh layout)
__device__ __forceinline__ uint32_t read_packed(const uint32_t* __restrict__ fwd, uint32_t doc, int bits) {
  const uint32_t* p = fwd + (size_t)(doc >> 5) * bits;
  const int bit = (int)(doc & 31u) * bits;
  const int k = bit >> 5, s = bit & 31;
  const uint32_t hi = fwd_word(p[k]);
  const uint32_t lo = (s + bits > 32) ? fwd_word(p[k + 1]) : 0u;
  return __funnelshift_l(lo, hi, s) >> (32 - bits);
}

__global__ void __launch_bounds__(kWtThreads) withtime_finalize_kernel(WithTimeJob j, const WtSeg* __restrict__ segs, int nseg) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < j.rows; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = j.keys[i];
    const uint32_t tid = (uint32_t)(key >> 32);
    const unsigned long long ord = key & 0xFFFFFFFFull;
    uint32_t id = ~0u;
    long long tv = 0;
    int lo = 0, hi = nseg;   // the last segment whose base <= ord
    while (hi - lo > 1) { const int mid = (lo + hi) / 2; if (segs[mid].base <= ord) lo = mid; else hi = mid; }
    const WtSeg& s = segs[lo];
    if (ord >= s.base && ord - s.base < s.num_docs && tid < s.time_card) {
      id = read_packed(s.fwd, (uint32_t)(ord - s.base), s.bits);
      tv = s.time_long ? static_cast<const long long*>(s.tdict)[tid]
                       : (long long)(int32_t)(static_cast<const uint32_t*>(s.tdict)[tid] ^ 0x80000000u);  // device INT dictionaries are biased
    }
    j.ids[i] = id;
    j.time[i] = tv;
  }
}

}  // namespace

int withtime_segments(pb200_ctx* ctx, cudaStream_t st, pb200_segment* const* segments, int nseg, int data_col, int time_col,
                      const std::vector<unsigned long long>& base, std::vector<std::unique_ptr<DevBufRaw>>& temps,
                      const WtSeg** out) {
  std::vector<WtSeg> h(nseg);
  for (int s = 0; s < nseg; s++) {
    const DeviceColumn &v = segments[s]->cols[data_col], &t = segments[s]->cols[time_col];
    h[s] = WtSeg{base[s], v.fwd, t.dict_native, v.bits, t.stored_type == PB200_LONG ? 1 : 0, (uint32_t)segments[s]->num_docs,
                 (uint32_t)t.cardinality};
  }
  temps.emplace_back(new DevBufRaw(ctx));
  if (int rc = temps.back()->alloc(sizeof(WtSeg) * nseg)) return rc;
  // pageable source: the copy is staged before the call returns, so `h` may go out of scope
  PB200_CUDA(cudaMemcpyAsync(temps.back()->p, h.data(), sizeof(WtSeg) * nseg, cudaMemcpyHostToDevice, st));
  *out = static_cast<const WtSeg*>(temps.back()->p);
  return PB200_OK;
}

int withtime_finalize(pb200_ctx* ctx, cudaStream_t st, const WithTimeJob& job, const WtSeg* segs, int nseg) {
  if (job.rows <= 0) return PB200_OK;
  withtime_finalize_kernel<<<grid_for(ctx, job.rows, kWtThreads), kWtThreads, 0, st>>>(job, segs, nseg);
  PB200_CUDA(cudaGetLastError());
  return PB200_OK;
}

}  // namespace pb200
