// pb200_moments.cu -- limb dictionaries for VAR / STDDEV (pb200_moments.h) and the C-ABI reader of exact moments.
//
// A qualifying dictionary gets three u32 arrays indexed by dictId: K = k, H = k^2 >> 32, L = k^2 & 0xFFFFFFFF, with
// value = c + k * 2^e.  They are built once per DEVICE dictionary -- the segment's own, or the domain's when the column is
// bound, so bound segments share them -- by the first query that needs them, one thread per entry, and live as long as
// the dictionary.  12 bytes x cardinality.
#include <cuda_runtime.h>

#include <algorithm>

#include "pb200_internal.h"

namespace pb200 {

MomentDict::~MomentDict() {
  if (limbs && ctx) dev_free(ctx, limbs);
  if (hll_hash && ctx) dev_free(ctx, hll_hash);
}

// k of every dictionary entry from the device copy of the dictionary (INT: biased, value ^ 0x80000000), then its square's
// two words.  The grid was verified exactly on the host: v - c is k * 2^e without rounding.
__global__ void limb_build_kernel(const void* __restrict__ dict, MomentGrid g, int entries, uint32_t* __restrict__ limbs) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < entries; i += gridDim.x * blockDim.x) {
    unsigned long long k;
    switch (g.stored_type) {
      case PB200_INT: k = (unsigned long long)((long long)(int32_t)(static_cast<const uint32_t*>(dict)[i] ^ 0x80000000u) - g.c_int); break;
      case PB200_LONG: k = (unsigned long long)static_cast<const long long*>(dict)[i] - (unsigned long long)g.c_int; break;
      case PB200_FLOAT: k = (unsigned long long)ldexp((double)static_cast<const float*>(dict)[i] - g.c_dbl, -g.e); break;
      default: k = (unsigned long long)ldexp(static_cast<const double*>(dict)[i] - g.c_dbl, -g.e); break;
    }
    const unsigned long long sq = k * k;
    limbs[i] = (uint32_t)k;
    limbs[(size_t)entries + i] = (uint32_t)(sq >> 32);
    limbs[2 * (size_t)entries + i] = (uint32_t)sq;
  }
}

// Evaluates column c's dictionary once (two racing callers: one builds, the other waits on the mutex and finds it ready)
static int ensure_limbs(pb200_ctx* ctx, pb200_segment* seg, DeviceColumn& c) {
  MomentDict& m = *c.moments;
  if (m.ready.load(std::memory_order_acquire)) return PB200_OK;
  std::lock_guard<std::mutex> lock(m.mu);
  if (m.ready.load(std::memory_order_relaxed)) return PB200_OK;
  MomentGrid grid;
  const bool eligible = c.dict_host.size() >= (size_t)c.cardinality * c.dict_width() &&
                        moments_grid(c.stored_type, c.dict_host.data(), c.cardinality, &grid);
  if (eligible) {
    const size_t bytes = 12ull * (size_t)c.cardinality;
    void* p = nullptr;
    if (int rc = dev_alloc(ctx, bytes, &p)) return rc;
    cudaStream_t st = take_stream(ctx);
    limb_build_kernel<<<grid_for(ctx, c.cardinality, 256), 256, 0, st>>>(c.dict_native, grid, c.cardinality, (uint32_t*)p);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    give_stream(ctx, st);
    if (e != cudaSuccess) { dev_free(ctx, p); set_error("limb dictionary build failed: %s", cudaGetErrorString(e)); return PB200_E_CUDA; }
    m.ctx = ctx;
    m.limbs = (uint32_t*)p;
    m.entries = c.cardinality;
    if (!c.dict_shared) {   // a segment's own dictionary: its limbs count in the segment's resident bytes
      std::lock_guard<std::mutex> g(seg->derive_mu);
      seg->device_bytes += (int64_t)bytes;
    }
  }
  m.eligible = eligible;
  m.grid = eligible ? grid : MomentGrid{};
  m.ready.store(true, std::memory_order_release);   // published: launches read the limbs only after this
  return PB200_OK;
}

int moments_prepare(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments, int nseg) {
  if (!query || !segments || nseg <= 0 || query->num_aggs <= 0 || !query->aggs) return PB200_OK;
  for (int a = 0; a < query->num_aggs && a < kMaxAggs; a++) {
    const pb200_agg& ag = query->aggs[a];
    if (!is_moments_fn(ag.function)) continue;
    for (int s = 0; s < nseg; s++) {
      pb200_segment* seg = segments[s];
      if (!seg || seg->ctx != ctx || ag.column < 0 || ag.column >= seg->num_columns()) continue;   // refused by the planner
      DeviceColumn& c = seg->cols[ag.column];
      if (c.stored_type == PB200_STRING || c.bits > 31 || !c.dict_native || c.cardinality <= 0) continue;
      if (int rc = ensure_limbs(ctx, seg, c)) return rc;
    }
  }
  return PB200_OK;
}

}  // namespace pb200

using namespace pb200;

extern "C" int32_t pb200_result_moments(const pb200_result* R, int32_t a, int32_t row, int64_t* n, int64_t* c_mant,
                                        int32_t* c_exp, int32_t* e, uint64_t* s1, uint64_t* s2_lo, uint64_t* s2_hi) {
  if (!R || a < 0 || a >= R->meta.num_aggs || a >= kMaxAggs) { set_error("bad aggregation index"); return PB200_E_INVALID; }
  if (!R->mom.on[a]) { set_error("aggregation %d is not VAR_POP / VAR_SAMP / STDDEV_POP / STDDEV_SAMP", a); return PB200_E_INVALID; }
  const long long rows = R->meta.num_groups < 0 ? 1 : R->meta.num_groups;
  if (row < 0 || row >= rows) { set_error("bad row %d (%lld rows)", row, rows); return PB200_E_INVALID; }
  const int64_t* counts = R->meta.num_groups < 0 ? R->lng[a].data() : R->view.lng[a];
  if (!R->mom.rows[a] || !counts) { set_error("result rows carry no moments"); return PB200_E_INVALID; }
  const unsigned long long* m = R->mom.rows[a] + 3ull * row;
  const long long cnt = counts[row];
  const MomentGrid& g = R->mom.grid[a];
  if (n) *n = cnt;
  if (c_mant) *c_mant = g.c_mant;
  if (c_exp) *c_exp = g.c_exp;
  if (e) *e = g.e;
  if (s1) *s1 = m[0];
  if (s2_lo) *s2_lo = m[1];
  if (s2_hi) *s2_hi = m[2];
  return PB200_OK;
}
