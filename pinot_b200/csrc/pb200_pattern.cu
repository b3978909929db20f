// pb200_pattern.cu -- REGEXP_LIKE over STRING dictionaries on the device (pb200_match_pattern, include/pinot_b200.h).
//
// The reference resolves a pattern predicate on a dictionary column to the set of matching dictIds
// (RegexpLikePredicateEvaluatorFactory); this is that resolution for every segment of a call in one launch.  The pattern
// is compiled on the host (pb200_pattern.h) and the automaton, about 18 KB, is staged into each block's shared memory.
// One thread matches one dictionary entry; a warp's 32 consecutive entries fill one 32-bit word of the bitmap with a
// ballot.  STRING dictionaries stay on the host at registration; a column's compact copy (StringDict) is uploaded by its
// first pattern query and lives as long as the segment.
#include <cuda_runtime.h>

#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "pb200_internal.h"
#include "pb200_pattern.h"

namespace pb200 {

StringDict::~StringDict() {
  if (block && ctx) dev_free(ctx, block);
}

struct PatternJob {
  const uint32_t* offsets;      // device: entries + 1 offsets into bytes
  const unsigned char* bytes;
  uint32_t entries;
  uint32_t word0;               // first bitmap word of this segment
};

__global__ void __launch_bounds__(256) pattern_match_kernel(const PatternAutomaton* __restrict__ automaton,
                                                            const PatternJob* __restrict__ jobs, int num_jobs,
                                                            uint32_t total_words, uint32_t* __restrict__ bits) {
  __shared__ PatternAutomaton a;
  {
    const uint4* src = reinterpret_cast<const uint4*>(automaton);
    uint4* dst = reinterpret_cast<uint4*>(&a);
    for (int k = threadIdx.x; k < (int)(sizeof(PatternAutomaton) / 16); k += blockDim.x) dst[k] = src[k];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < total_words; w += warps) {
    int lo = 0, hi = num_jobs - 1;   // the job of word w: the last one starting at or before it
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (jobs[mid].word0 <= w) lo = mid; else hi = mid - 1;
    }
    const PatternJob& j = jobs[lo];
    const uint32_t e = (w - j.word0) * 32 + lane;
    bool m = false;
    if (e < j.entries) {
      const uint32_t s = j.offsets[e];
      m = pattern_match(a, j.bytes + s, (int)(j.offsets[e + 1] - s));
    }
    const uint32_t word = __ballot_sync(0xFFFFFFFFu, m);
    if (lane == 0) bits[w] = word;
  }
}

namespace {

// Entries of the column's own dictionary: the registered one, or (bound) the domain's entries at local_ids
int own_entries(const DeviceColumn& c) { return c.local_ids.empty() ? c.cardinality : (int)c.local_ids.size(); }

// Uploads the compact copy of column c once (two racing callers: one builds, the other waits on the mutex and finds it
// ready).
int ensure_strings(pb200_ctx* ctx, pb200_segment* seg, DeviceColumn& c) {
  StringDict& sd = *c.strings;
  if (sd.ready.load(std::memory_order_acquire)) return PB200_OK;
  std::lock_guard<std::mutex> lock(sd.mu);
  if (sd.ready.load(std::memory_order_relaxed)) return PB200_OK;
  const int n = own_entries(c);
  const size_t w = (size_t)c.dict_entry_bytes;
  std::vector<uint32_t> offsets((size_t)n + 1, 0);
  std::vector<unsigned char> bytes;
  for (int l = 0; l < n; l++) {
    const size_t id = c.local_ids.empty() ? (size_t)l : (size_t)c.local_ids[l];
    const unsigned char* p = c.dict_be.data() + w * id;
    size_t len = 0;
    while (len < w && p[len]) len++;   // the value ends at its first NUL (zero padding)
    bytes.insert(bytes.end(), p, p + len);
    if (bytes.size() > 0xFFFFFFFFull) { set_error("STRING dictionary of more than 4 GiB: REGEXP_LIKE is not accelerated"); return PB200_E_UNSUPPORTED; }
    offsets[l + 1] = (uint32_t)bytes.size();
  }
  const size_t off_bytes = (offsets.size() * 4 + 15) & ~(size_t)15;
  const size_t total = off_bytes + bytes.size() + 16;
  void* p = nullptr;
  if (int rc = dev_alloc(ctx, total, &p)) return rc;
  StreamLease st(ctx);
  cudaError_t e = cudaMemcpyAsync(p, offsets.data(), offsets.size() * 4, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && !bytes.empty())
    e = cudaMemcpyAsync((unsigned char*)p + off_bytes, bytes.data(), bytes.size(), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { dev_free(ctx, p); set_error("STRING dictionary upload failed: %s", cudaGetErrorString(e)); return PB200_E_CUDA; }
  sd.ctx = ctx;
  sd.block = p;
  sd.offsets = (const uint32_t*)p;
  sd.bytes = (const unsigned char*)p + off_bytes;
  sd.entries = (uint32_t)n;
  {
    std::lock_guard<std::mutex> g(seg->derive_mu);
    seg->device_bytes += (int64_t)total;
  }
  sd.ready.store(true, std::memory_order_release);   // published: launches read the copy only after this
  return PB200_OK;
}

}  // namespace
}  // namespace pb200

using namespace pb200;

extern "C" int32_t pb200_match_pattern(pb200_ctx* ctx, const char* pattern, int32_t nseg, pb200_segment* const* segs,
                                       const int32_t* columns, uint32_t* const* match_bits) {
  if (!ctx || !pattern || nseg <= 0 || !segs || !columns || !match_bits) { set_error("invalid argument to pb200_match_pattern"); return PB200_E_INVALID; }
  std::unique_ptr<PatternAutomaton> a(new PatternAutomaton());
  std::string why;
  const int prc = pattern_compile(pattern, a.get(), &why);
  if (prc == PATTERN_INVALID) { set_error("REGEXP_LIKE pattern: %s", why.c_str()); return PB200_E_INVALID; }
  if (prc != PATTERN_OK) { set_error("REGEXP_LIKE pattern outside the accelerated subset: %s", why.c_str()); return PB200_E_UNSUPPORTED; }
  for (int s = 0; s < nseg; s++) {
    pb200_segment* seg = segs[s];
    if (!seg || seg->ctx != ctx || !match_bits[s]) { set_error("pb200_match_pattern: bad segment %d", s); return PB200_E_INVALID; }
    const int col = columns[s];
    if (col < 0 || col >= seg->num_columns()) { set_error("pb200_match_pattern: segment %d has no column %d", s, col); return PB200_E_INVALID; }
    const DeviceColumn& c = seg->cols[col];
    if (col >= seg->num_stored) { set_error("REGEXP_LIKE on a derived column is not accelerated"); return PB200_E_UNSUPPORTED; }
    if (c.stored_type != PB200_STRING) { set_error("REGEXP_LIKE on a column that is not STRING is not accelerated"); return PB200_E_UNSUPPORTED; }
    if (c.fwd_kind == PB200_FWD_RAW_FIXEDBYTE || (c.dict_be.empty() && c.cardinality > 0)) {
      set_error("REGEXP_LIKE on a STRING column without a dictionary is not accelerated");
      return PB200_E_UNSUPPORTED;
    }
  }
  PB200_CUDA(cudaSetDevice(ctx->device));
  std::vector<PatternJob> jobs;
  std::vector<uint32_t> word0(nseg);
  uint32_t total_words = 0;
  for (int s = 0; s < nseg; s++) {
    DeviceColumn& c = segs[s]->cols[columns[s]];
    if (int rc = ensure_strings(ctx, segs[s], c)) return rc;
    const StringDict& sd = *c.strings;
    word0[s] = total_words;
    if (sd.entries == 0) continue;
    jobs.push_back({sd.offsets, sd.bytes, sd.entries, total_words});
    total_words += (sd.entries + 31) / 32;
  }
  if (total_words == 0) return PB200_OK;
  // one staging block: automaton and jobs in, bitmaps out
  const size_t in_bytes = sizeof(PatternAutomaton) + jobs.size() * sizeof(PatternJob);
  const size_t out_off = (in_bytes + 15) & ~(size_t)15;
  const size_t out_bytes = (size_t)total_words * 4;
  PinnedBlock pin;
  pin.ctx = ctx;
  if (int rc = pinned_alloc(ctx, out_off + out_bytes, &pin.p, &pin.bytes)) return rc;
  memcpy(pin.p, a.get(), sizeof(PatternAutomaton));
  memcpy((unsigned char*)pin.p + sizeof(PatternAutomaton), jobs.data(), jobs.size() * sizeof(PatternJob));
  DevBufRaw dev(ctx);
  if (int rc = dev.alloc(out_off + out_bytes)) return rc;
  StreamLease st(ctx);
  const int threads = 256;
  const long long warps_needed = total_words;
  const int grid = (int)std::max<long long>(1, std::min<long long>((warps_needed + 7) / 8, (long long)ctx->sm_count * 8));
  cudaError_t e = cudaMemcpyAsync(dev.p, pin.p, in_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    const unsigned char* base = (const unsigned char*)dev.p;
    pattern_match_kernel<<<grid, threads, 0, st>>>((const PatternAutomaton*)base, (const PatternJob*)(base + sizeof(PatternAutomaton)),
                                                   (int)jobs.size(), total_words, (uint32_t*)(base + out_off));
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync((unsigned char*)pin.p + out_off, (unsigned char*)dev.p + out_off, out_bytes, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { set_error("pattern match failed: %s", cudaGetErrorString(e)); return PB200_E_CUDA; }
  const uint32_t* out = (const uint32_t*)((const unsigned char*)pin.p + out_off);
  for (int s = 0; s < nseg; s++) {
    const uint32_t n = segs[s]->cols[columns[s]].strings->entries;
    if (n) memcpy(match_bits[s], out + word0[s], (size_t)(n + 31) / 32 * 4);
  }
  return PB200_OK;
}
