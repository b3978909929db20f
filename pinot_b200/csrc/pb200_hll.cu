// pb200_hll.cu -- DISTINCTCOUNTHLL on the device (pb200_hll.h, DESIGN.md section 3.17): the per-dictionary hash array,
// and the finalize that turns DISTINCTCOUNT dictId bitsets into HyperLogLog estimates, queued behind the scan.
//
//   hash array        one thread per dictionary entry: MurmurHash of the value (INT unbiased from the device copy, LONG,
//                     FLOAT, DOUBLE raw bits; STRING over its UTF-8 bytes, which are checked), built once per device
//                     dictionary and kept with it (MomentDict::hll_hash, 4 bytes per entry).
//   group-by          each table entry's bitset row -> its estimate.  The set bits gather hash[id], and (j, r) is
//                     max-ed into the row's m registers in shared memory; then the scaled register sum and the zero
//                     registers are reduced and the estimate taken.  log2m <= 8: one warp per row (1 KB of registers);
//                     above: one CTA per row (up to 16 KB).
//   aggregation only  one bitset of up to 2^26 words: each CTA of a grid-stride pass builds partial registers in shared
//                     memory and max-merges them into m global registers; one small block takes the estimate.  A max
//                     does not depend on order, so every schedule gives the same registers.
#include <cuda_runtime.h>

#include <mutex>
#include <vector>

#include "pb200_internal.h"

namespace pb200 {

namespace {
constexpr int kHllThreads = 256;

__global__ void __launch_bounds__(kHllThreads) hll_hash_kernel(int stored_type, const void* __restrict__ dict,
                                                               const uint32_t* __restrict__ offsets,
                                                               const unsigned char* __restrict__ bytes, uint32_t n,
                                                               uint32_t* __restrict__ out, uint32_t* __restrict__ bad) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    uint32_t h;
    if (stored_type == PB200_STRING) {
      const uint32_t s = offsets[i];
      const int len = (int)(offsets[i + 1] - s);
      h = hll_hash_bytes(bytes + s, len, 0xFFFFFFFFu);
      if (!hll_utf8_valid(bytes + s, len)) atomicOr(bad, 1u);
    } else if (stored_type == PB200_INT) {
      h = hll_hash_value(PB200_INT, static_cast<const uint32_t*>(dict)[i] ^ 0x80000000u);   // the device copy is biased
    } else if (stored_type == PB200_FLOAT) {
      h = hll_hash_value(PB200_FLOAT, static_cast<const uint32_t*>(dict)[i]);
    } else {
      h = hll_hash_value(stored_type, static_cast<const unsigned long long*>(dict)[i]);
    }
    out[i] = h;
  }
}

// the members of bitset word w (dictIds 32 w ...) max-ed into registers `reg`
__device__ __forceinline__ void hll_offer_word(uint32_t word, size_t w, const uint32_t* __restrict__ hash, int p, uint32_t* reg) {
  for (; word; word &= word - 1) {
    const uint32_t x = hash[w * 32 + __ffs(word) - 1];
    atomicMax(reg + hll_index(x, p), hll_rank(x, p));
  }
}

__device__ __forceinline__ void warp_sum(unsigned long long* s, uint32_t* z) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    *s += __shfl_xor_sync(0xFFFFFFFFu, *s, o);
    *z += __shfl_xor_sync(0xFFFFFFFFu, *z, o);
  }
}

// group-by: per_row threads (32 or kHllThreads) per bitset row, kHllThreads / per_row rows per block at a time; dynamic
// shared memory: m registers per row
__global__ void __launch_bounds__(kHllThreads) hll_rows_kernel(HllJob j, int per_row, double alpha_mm, const long long* __restrict__ linear) {
  extern __shared__ uint32_t regs[];
  __shared__ unsigned long long part_s[kHllThreads / 32];
  __shared__ uint32_t part_z[kHllThreads / 32];
  const int p = j.log2m, m = 1 << p;
  const int rows_per_block = kHllThreads / per_row, sub = threadIdx.x / per_row, lane = threadIdx.x % per_row;
  uint32_t* reg = regs + (size_t)sub * m;
  for (long long base = (long long)blockIdx.x * rows_per_block; base < j.rows; base += (long long)gridDim.x * rows_per_block) {
    const long long g = base + sub;
    for (int k = lane; k < m; k += per_row) reg[k] = 0;
    __syncthreads();
    if (g < j.rows) {
      const uint32_t* row = j.bits + (size_t)g * j.words;
      for (size_t w = lane; w < j.words; w += per_row) hll_offer_word(row[w], w, j.hash, p, reg);
    }
    __syncthreads();
    unsigned long long s = 0;
    uint32_t z = 0;
    for (int k = lane; k < m; k += per_row) { s += hll_term(reg[k], p); z += reg[k] == 0; }
    warp_sum(&s, &z);
    if (per_row == 32) {
      if (lane == 0 && g < j.rows) j.out[g] = hll_estimate(s, z, p, alpha_mm, linear);
    } else {
      if ((threadIdx.x & 31) == 0) { part_s[threadIdx.x >> 5] = s; part_z[threadIdx.x >> 5] = z; }
      __syncthreads();
      if (threadIdx.x == 0 && g < j.rows) {
        for (int k = 1; k < kHllThreads / 32; k++) { s += part_s[k]; z += part_z[k]; }
        j.out[g] = hll_estimate(s, z, p, alpha_mm, linear);
      }
    }
    __syncthreads();   // the registers are reset for the next rows
  }
}

// aggregation only, pass 1: the block's registers over its words, max-ed into the m global registers `greg` (zeroed)
__global__ void __launch_bounds__(kHllThreads) hll_partial_kernel(HllJob j, uint32_t* __restrict__ greg) {
  extern __shared__ uint32_t reg[];
  const int p = j.log2m, m = 1 << p;
  for (int k = threadIdx.x; k < m; k += kHllThreads) reg[k] = 0;
  __syncthreads();
  for (size_t w = blockIdx.x * (size_t)kHllThreads + threadIdx.x; w < j.words; w += (size_t)gridDim.x * kHllThreads)
    hll_offer_word(j.bits[w], w, j.hash, p, reg);
  __syncthreads();
  for (int k = threadIdx.x; k < m; k += kHllThreads)
    if (reg[k]) atomicMax(greg + k, reg[k]);
}

// aggregation only, pass 2: the global registers -> the estimate (one block)
__global__ void __launch_bounds__(kHllThreads) hll_total_kernel(const uint32_t* __restrict__ greg, int p, double alpha_mm,
                                                                const long long* __restrict__ linear, long long* __restrict__ out) {
  __shared__ unsigned long long part_s[kHllThreads / 32];
  __shared__ uint32_t part_z[kHllThreads / 32];
  unsigned long long s = 0;
  uint32_t z = 0;
  for (int k = threadIdx.x; k < (1 << p); k += kHllThreads) { s += hll_term(greg[k], p); z += greg[k] == 0; }
  warp_sum(&s, &z);
  if ((threadIdx.x & 31) == 0) { part_s[threadIdx.x >> 5] = s; part_z[threadIdx.x >> 5] = z; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < kHllThreads / 32; k++) { s += part_s[k]; z += part_z[k]; }
    *out = hll_estimate(s, z, p, alpha_mm, linear);
  }
}

// the STRING dictionary of column c, every entry (a bound column: the domain's), as offsets + bytes without padding
int pack_strings(const DeviceColumn& c, std::vector<uint32_t>& offsets, std::vector<unsigned char>& bytes) {
  const size_t w = (size_t)c.dict_entry_bytes;
  if (w == 0 || c.dict_be.size() < w * (size_t)c.cardinality) { set_error("DISTINCTCOUNTHLL over a STRING column without dictionary bytes: not accelerated"); return PB200_E_UNSUPPORTED; }
  offsets.assign((size_t)c.cardinality + 1, 0);
  for (int i = 0; i < c.cardinality; i++) {
    const unsigned char* p = c.dict_be.data() + w * i;
    size_t len = 0;
    while (len < w && p[len]) len++;   // the value ends at its first NUL (zero padding)
    bytes.insert(bytes.end(), p, p + len);
    if (bytes.size() > 0xFFFFFFFFull) { set_error("STRING dictionary of more than 4 GiB: DISTINCTCOUNTHLL is not accelerated"); return PB200_E_UNSUPPORTED; }
    offsets[i + 1] = (uint32_t)bytes.size();
  }
  return PB200_OK;
}

// Builds column c's hash array once (two racing callers: one builds, the other waits on the mutex and finds it built)
int ensure_hashes(pb200_ctx* ctx, pb200_segment* seg, DeviceColumn& c) {
  MomentDict& md = *c.moments;
  if (md.hll_state.load(std::memory_order_acquire) != 0) return PB200_OK;
  std::lock_guard<std::mutex> lock(md.mu);
  if (md.hll_state.load(std::memory_order_relaxed) != 0) return PB200_OK;
  const uint32_t n = (uint32_t)c.cardinality;
  std::vector<uint32_t> offsets;
  std::vector<unsigned char> bytes;
  if (c.stored_type == PB200_STRING)
    if (int rc = pack_strings(c, offsets, bytes)) return rc;
  const size_t off_bytes = (offsets.size() * 4 + 15) & ~(size_t)15;
  DevBufRaw scratch(ctx);   // [bad flag | STRING offsets | bytes]
  if (int rc = scratch.alloc(16 + off_bytes + bytes.size() + 16)) return rc;
  void* out = nullptr;
  if (int rc = dev_alloc(ctx, 4ull * n, &out)) return rc;
  unsigned char* const sp = static_cast<unsigned char*>(scratch.p);
  uint32_t bad = 0;
  StreamLease st(ctx);
  cudaError_t e = cudaMemsetAsync(sp, 0, 16, st);
  if (e == cudaSuccess && !offsets.empty()) e = cudaMemcpyAsync(sp + 16, offsets.data(), offsets.size() * 4, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && !bytes.empty()) e = cudaMemcpyAsync(sp + 16 + off_bytes, bytes.data(), bytes.size(), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    hll_hash_kernel<<<grid_for(ctx, n, kHllThreads), kHllThreads, 0, st>>>(c.stored_type, c.dict_native, reinterpret_cast<const uint32_t*>(sp + 16),
                                                                           sp + 16 + off_bytes, n, static_cast<uint32_t*>(out), reinterpret_cast<uint32_t*>(sp));
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, sp, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { dev_free(ctx, out); set_error("DISTINCTCOUNTHLL hash array build failed: %s", cudaGetErrorString(e)); return PB200_E_CUDA; }
  if (bad) {
    dev_free(ctx, out);
    md.hll_state.store(-1, std::memory_order_release);
    return PB200_OK;
  }
  md.ctx = ctx;
  md.hll_hash = static_cast<uint32_t*>(out);
  if (!c.dict_shared) {   // a segment's own dictionary: its hashes count in the segment's resident bytes
    std::lock_guard<std::mutex> g(seg->derive_mu);
    seg->device_bytes += 4ll * n;
  }
  md.hll_state.store(1, std::memory_order_release);   // published: launches read the hashes only after this
  return PB200_OK;
}

// alpha * m^2 and the linear-counting table of log2m p, the table uploaded into `temps`
int hll_constants(pb200_ctx* ctx, cudaStream_t st, int p, std::vector<std::unique_ptr<DevBufRaw>>& temps, double* alpha_mm,
                  const long long** linear) {
  std::vector<long long> table(((size_t)1 << p) + 1);
  hll_linear_table(p, table.data());
  temps.emplace_back(new DevBufRaw(ctx));
  if (int rc = temps.back()->alloc(table.size() * 8)) return rc;
  PB200_CUDA(cudaMemcpyAsync(temps.back()->p, table.data(), table.size() * 8, cudaMemcpyHostToDevice, st));   // pageable: staged before it returns
  *alpha_mm = hll_alpha_mm(p);
  *linear = static_cast<const long long*>(temps.back()->p);
  return PB200_OK;
}
}  // namespace

int hll_prepare(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments, int nseg) {
  if (!query || !segments || nseg <= 0 || query->num_aggs <= 0 || !query->aggs) return PB200_OK;
  for (int a = 0; a < query->num_aggs && a < kMaxAggs; a++) {
    const pb200_agg& ag = query->aggs[a];
    if (!is_hll_fn(ag.function)) continue;
    for (int s = 0; s < nseg; s++) {
      pb200_segment* seg = segments[s];
      if (!seg || seg->ctx != ctx || ag.column < 0 || ag.column >= seg->num_columns()) continue;   // refused by the planner
      DeviceColumn& c = seg->cols[ag.column];
      if (c.bits > 31 || c.cardinality <= 0 || (c.stored_type != PB200_STRING && !c.dict_native)) continue;   // likewise
      if (int rc = ensure_hashes(ctx, seg, c)) return rc;
      if (c.moments->hll_state.load(std::memory_order_acquire) < 0) {
        set_error("DISTINCTCOUNTHLL over column %d: a STRING entry of segment %d is not valid UTF-8: not accelerated", ag.column, s);
        return PB200_E_UNSUPPORTED;
      }
    }
  }
  return PB200_OK;
}

int hll_finalize(pb200_ctx* ctx, cudaStream_t st, const HllJob& j, std::vector<std::unique_ptr<DevBufRaw>>& temps) {
  if (j.rows <= 0) return PB200_OK;
  double alpha_mm;
  const long long* linear;
  if (int rc = hll_constants(ctx, st, j.log2m, temps, &alpha_mm, &linear)) return rc;
  const size_t m = (size_t)1 << j.log2m;
  if (j.rows > 1 || !j.single) {
    const int per_row = j.log2m <= 8 ? 32 : kHllThreads;
    const int rows_per_block = kHllThreads / per_row;
    const size_t smem = (size_t)rows_per_block * m * 4;
    const int grid = (int)std::max<long long>(1, std::min<long long>((j.rows + rows_per_block - 1) / rows_per_block, (long long)ctx->sm_count * 8));
    hll_rows_kernel<<<grid, kHllThreads, smem, st>>>(j, per_row, alpha_mm, linear);
  } else {
    temps.emplace_back(new DevBufRaw(ctx));
    if (int rc = temps.back()->alloc(m * 4)) return rc;
    uint32_t* greg = static_cast<uint32_t*>(temps.back()->p);
    PB200_CUDA(cudaMemsetAsync(greg, 0, m * 4, st));
    hll_partial_kernel<<<grid_for(ctx, (long long)j.words, kHllThreads), kHllThreads, m * 4, st>>>(j, greg);
    hll_total_kernel<<<1, kHllThreads, 0, st>>>(greg, j.log2m, alpha_mm, linear, j.out);
  }
  PB200_CUDA(cudaGetLastError());
  return PB200_OK;
}

int hll_whole_dictionary(pb200_ctx* ctx, pb200_segment* seg, int column, int log2m, long long* out) {
  if (!seg || column < 0 || column >= seg->num_columns()) { set_error("DISTINCTCOUNTHLL: column %d out of range", column); return PB200_E_INVALID; }
  DeviceColumn& c = seg->cols[column];
  if (c.bits > 31 || c.cardinality <= 0 || (c.stored_type != PB200_STRING && !c.dict_native)) {
    set_error("DISTINCTCOUNTHLL over column %d: no dictIds (raw values): not accelerated", column);
    return PB200_E_UNSUPPORTED;
  }
  PB200_CUDA(cudaSetDevice(ctx->device));
  if (int rc = ensure_hashes(ctx, seg, c)) return rc;
  if (c.moments->hll_state.load(std::memory_order_acquire) < 0) {
    set_error("DISTINCTCOUNTHLL over column %d: a STRING entry is not valid UTF-8: not accelerated", column);
    return PB200_E_UNSUPPORTED;
  }
  // the segment's values: every entry of its own dictionary, or (bound to a domain) the domain ids that occur in it
  const size_t n = (size_t)c.cardinality, words = (n + 31) / 32;
  std::vector<uint32_t> ones(words, c.local_ids.empty() ? ~0u : 0u);
  if (c.local_ids.empty() && n % 32) ones.back() = (1u << (n % 32)) - 1u;
  for (uint32_t id : c.local_ids) ones[id >> 5] |= 1u << (id & 31);
  std::vector<std::unique_ptr<DevBufRaw>> temps;
  DevBufRaw bits(ctx), est(ctx);
  if (int rc = bits.alloc(words * 4)) return rc;
  if (int rc = est.alloc(8)) return rc;
  StreamLease st(ctx);
  PB200_CUDA(cudaMemcpyAsync(bits.p, ones.data(), words * 4, cudaMemcpyHostToDevice, st));
  const HllJob job{static_cast<const uint32_t*>(bits.p), words, 1, true, c.moments->hll_hash, log2m, static_cast<long long*>(est.p)};
  if (int rc = hll_finalize(ctx, st, job, temps)) return rc;
  PB200_CUDA(cudaMemcpyAsync(out, est.p, 8, cudaMemcpyDeviceToHost, st));
  PB200_CUDA(cudaStreamSynchronize(st));
  return PB200_OK;
}

const std::vector<std::vector<int32_t>>* result_sets(pb200_result* R, int a) {
  pb200_result::LazySets& L = R->lazy;
  if (a < 0 || a >= kMaxAggs || L.src[a] < 0) return a >= 0 && a < (int)R->distinct.size() ? &R->distinct[a] : nullptr;
  std::lock_guard<std::mutex> lock(L.mu);
  if ((int)R->distinct.size() <= a) R->distinct.resize(a + 1);
  if (R->distinct[a].size() != L.rows[L.src[a]]) {
    const int b = L.src[a];
    std::vector<uint32_t> bits(L.rows[b] * L.words[b]);
    if (!bits.empty()) {
      if (cudaSetDevice(L.ctx->device) != cudaSuccess ||
          cudaMemcpy(bits.data(), L.bits[b], bits.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) {
        set_error("DISTINCTCOUNTHLL set copy failed");
        return nullptr;
      }
    }
    R->distinct[a].resize(L.rows[b]);
    for (size_t i = 0; i < L.rows[b]; i++) R->distinct[a][i] = bitset_ids(bits.data() + i * L.words[b], L.words[b]);
  }
  return &R->distinct[a];
}

}  // namespace pb200
