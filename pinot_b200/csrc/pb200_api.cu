// pb200_api.cu -- C-ABI implementation: context, segment residency, query launch (planned by pb200_plan.cpp), result extraction.
//
// Host logic here is the device-facing half of what the reference does between PlanNode.run() and nextBlock():
// choosing what to stream (ProjectPlanNode's column set, core/plan/ProjectPlanNode.java), laying out the group-key
// space (DictionaryBasedGroupKeyGenerator.java:105-186) and extracting results (GroupByOperator.java:116-140,
// AggregationFunction.extractAggregationResult).
#include <cuda_runtime.h>
#include <chrono>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <limits>
#include <memory>
#include <optional>

#include "pb200_decode.h"
#include "pb200_internal.h"
#include "pb200_expr.h"
#include "pb200_percentile.h"
#include "pb200_withtime.h"
#include "pb200_plan.h"
#include "pb200_scan_launch.h"
#include "pb200_unpack.cuh"

namespace pb200 {

static thread_local char g_error[1024] = "";
// Host wall-clock of the calling thread's last pb200_execute, by phase (pb200_last_phases): a few steady_clock reads per query.
static thread_local double g_phase_ms[PB200_NUM_PHASES] = {};
static inline double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

void set_phase_ms(int phase, double ms) { g_phase_ms[phase] = ms; }
double host_ms() { return now_ms(); }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof g_error, fmt, ap);
  va_end(ap);
}

// ------------------------------------------------------------------------------------------------------------------
// caching allocator + stream pool
// ------------------------------------------------------------------------------------------------------------------
static size_t round_block(size_t b) {
  size_t r = 512;
  while (r < b) r <<= 1;
  return b > (64u << 20) ? ((b + (2u << 20) - 1) / (2u << 20)) * (2u << 20) : r;
}

int dev_alloc(pb200_ctx* ctx, size_t bytes, void** out) {
  size_t rb = round_block(bytes ? bytes : 1);
  {
    std::lock_guard<std::mutex> g(ctx->mu);
    auto it = ctx->free_blocks.find(rb);
    if (it != ctx->free_blocks.end()) {
      *out = it->second;
      ctx->free_blocks.erase(it);
      return PB200_OK;
    }
  }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, rb);
  if (e != cudaSuccess) {
    // drop the cache and retry once
    {
      std::lock_guard<std::mutex> g(ctx->mu);
      for (auto& kv : ctx->free_blocks) { cudaFree(kv.second); ctx->block_size.erase(kv.second); }
      ctx->free_blocks.clear();
    }
    cudaGetLastError();
    e = cudaMalloc(&p, rb);
    if (e != cudaSuccess) {
      set_error("cudaMalloc(%zu) failed: %s", rb, cudaGetErrorString(e));
      cudaGetLastError();
      return PB200_E_NOMEM;
    }
  }
  std::lock_guard<std::mutex> g(ctx->mu);
  ctx->block_size[p] = rb;
  *out = p;
  return PB200_OK;
}

void dev_free(pb200_ctx* ctx, void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> g(ctx->mu);
  auto it = ctx->block_size.find(p);
  if (it == ctx->block_size.end()) return;
  if (it->second > (2048ull << 20)) {  // do not hoard very large blocks
    cudaFree(p);
    ctx->block_size.erase(it);
    return;
  }
  ctx->free_blocks.emplace(it->second, p);
}

int pinned_alloc(pb200_ctx* ctx, size_t bytes, void** out, size_t* got) {
  {
    std::lock_guard<std::mutex> g(ctx->mu);
    auto it = ctx->free_pinned.lower_bound(bytes);
    if (it != ctx->free_pinned.end()) { *out = it->second; *got = it->first; ctx->free_pinned.erase(it); return PB200_OK; }
  }
  size_t rb = std::max<size_t>(1 << 20, (bytes + (1 << 20) - 1) >> 20 << 20);
  void* p = nullptr;
  if (cudaHostAlloc(&p, rb, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); set_error("cudaHostAlloc(%zu) failed", rb); return PB200_E_NOMEM; }
  *out = p; *got = rb;
  return PB200_OK;
}
void pinned_free(pb200_ctx* ctx, void* p, size_t bytes) {
  if (!p) return;
  std::lock_guard<std::mutex> g(ctx->mu);
  if (bytes > (256ull << 20) || ctx->free_pinned.size() >= 8) { cudaFreeHost(p); return; }
  ctx->free_pinned.emplace(bytes, p);
}

cudaStream_t take_stream(pb200_ctx* ctx) {
  {
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->free_streams.empty()) {
      cudaStream_t s = ctx->free_streams.back();
      ctx->free_streams.pop_back();
      return s;
    }
  }
  cudaStream_t s = nullptr;
  cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
  return s;
}
void give_stream(pb200_ctx* ctx, cudaStream_t s) {
  std::lock_guard<std::mutex> g(ctx->mu);
  ctx->free_streams.push_back(s);
}
cudaEvent_t take_event(pb200_ctx* ctx) {
  {
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->free_events.empty()) { cudaEvent_t e = ctx->free_events.back(); ctx->free_events.pop_back(); return e; }
  }
  cudaEvent_t e = nullptr;
  if (cudaEventCreate(&e) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  return e;
}
void give_event(pb200_ctx* ctx, cudaEvent_t e) {
  if (!e) return;
  std::lock_guard<std::mutex> g(ctx->mu);
  ctx->free_events.push_back(e);
}

static inline uint32_t be32(const unsigned char* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
static inline uint64_t be64(const unsigned char* p) { return (uint64_t)be32(p) << 32 | be32(p + 4); }

// HBM layout of forward indexes: file order, every 4-byte big-endian word byte-swapped to native order ONCE at upload
// (see pb200_unpack.cuh).  In place, grid-stride, 16 bytes per thread.
__global__ void fwd_words_to_native_kernel(uint4* __restrict__ p, size_t n16) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
    uint4 x = p[i];
    x.x = __byte_perm(x.x, 0u, 0x0123u); x.y = __byte_perm(x.y, 0u, 0x0123u);
    x.z = __byte_perm(x.z, 0u, 0x0123u); x.w = __byte_perm(x.w, 0u, 0x0123u);
    p[i] = x;
  }
}
static cudaError_t fwd_words_to_native(void* p, size_t bytes, int sm_count, cudaStream_t st) {  // bytes: the padded allocation (multiple of 16)
  const size_t n16 = bytes / 16;
  if (!n16) return cudaSuccess;
  const int blocks = (int)std::min<size_t>((n16 + 255) / 256, (size_t)sm_count * 16);
  fwd_words_to_native_kernel<<<blocks, 256, 0, st>>>((uint4*)p, n16);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------------
// small kernels
// ------------------------------------------------------------------------------------------------------------------
__global__ void fill_u32_kernel(uint32_t* p, uint32_t v, long long n) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

}  // namespace pb200

using namespace pb200;

// ------------------------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------------------------
extern "C" const char* pb200_last_error(void) { return g_error; }
extern "C" int32_t pb200_abi_version(void) { return PB200_ABI_VERSION; }
// Structural check of ONE serialized RoaringBitmap (portable RoaringFormatSpec, little-endian) before the device reads it in
// place: header and container table inside the buffer, keys ascending, every container's payload inside the buffer, and the
// largest doc id below num_docs (so that the decode kernel's mask writes stay inside the mask).  O(containers), no decode.
extern "C" int32_t pb200_roaring_validate(const void* bytes, uint64_t len, int64_t num_docs) {
  const unsigned char* b = static_cast<const unsigned char*>(bytes);
  auto l16 = [&](uint64_t at) { return (uint32_t)b[at] | (uint32_t)b[at + 1] << 8; };
  auto l32 = [&](uint64_t at) { return (uint32_t)b[at] | (uint32_t)b[at + 1] << 8 | (uint32_t)b[at + 2] << 16 | (uint32_t)b[at + 3] << 24; };
  if (!b || len < 8) { if (b && len == 0) return PB200_OK; set_error("roaring bitmap shorter than its header"); return PB200_E_INVALID; }
  const uint32_t cookie = l32(0);
  const bool has_run = (cookie & 0xFFFFu) == 12347u;
  uint64_t n, pos;
  uint64_t run_flags = 0;
  if (has_run) { n = (uint64_t)(cookie >> 16) + 1; pos = 4; run_flags = pos; pos += (n + 7) / 8; }
  else if (cookie == 12346u) { n = l32(4); pos = 8; }
  else { set_error("roaring bitmap: unknown cookie %u", cookie); return PB200_E_INVALID; }
  if (n > 65536) { set_error("roaring bitmap: %llu containers", (unsigned long long)n); return PB200_E_INVALID; }
  if (n == 0) return PB200_OK;
  const uint64_t desc = pos;
  pos += 4 * n;
  const bool has_offsets = !has_run || n >= 4;
  const uint64_t offs = pos;
  if (has_offsets) pos += 4 * n;
  if (pos > len) { set_error("roaring bitmap: container table exceeds the buffer"); return PB200_E_INVALID; }
  uint64_t walk = pos;
  int64_t prev_key = -1;
  for (uint64_t c = 0; c < n; c++) {
    const int64_t key = l16(desc + 4 * c);
    const uint32_t card = l16(desc + 4 * c + 2) + 1;
    if (key <= prev_key) { set_error("roaring bitmap: container keys not ascending"); return PB200_E_INVALID; }
    prev_key = key;
    const bool is_run = has_run && ((b[run_flags + (c >> 3)] >> (c & 7)) & 1);
    const uint64_t start = has_offsets ? l32(offs + 4 * c) : walk;
    uint64_t bytes_c;
    if (is_run) {
      if (start + 2 > len) { set_error("roaring bitmap: run container outside the buffer"); return PB200_E_INVALID; }
      bytes_c = 2 + 4ull * l16(start);
    } else bytes_c = card > 4096 ? 8192 : 2ull * card;
    if (start < pos || start + bytes_c > len) { set_error("roaring bitmap: container %llu outside the buffer", (unsigned long long)c); return PB200_E_INVALID; }
    walk = start + bytes_c;
    if (c + 1 == n) {  // largest value of the bitmap
      int64_t top = -1;
      if (is_run) {
        const uint32_t nr = l16(start);
        for (uint32_t r = 0; r < nr; r++) top = std::max<int64_t>(top, (int64_t)l16(start + 2 + 4 * r) + l16(start + 4 + 4 * r));
      } else if (card > 4096) {
        for (int w = 2047; w >= 0 && top < 0; w--) { const uint32_t x = l32(start + 4ull * w); if (x) top = 32ll * w + (31 - __builtin_clz(x)); }
      } else {
        top = l16(start + 2ull * (card - 1));
      }
      if (top > 65535 || (key << 16) + top >= num_docs) { set_error("roaring bitmap: doc id %lld beyond %lld docs", (long long)((key << 16) + top), (long long)num_docs); return PB200_E_INVALID; }
    }
  }
  return PB200_OK;
}

extern "C" int32_t pb200_doc_mask_upload(pb200_ctx* ctx, int32_t num_docs, const uint32_t* words_in, int64_t num_words, uint32_t** out) {
  if (!ctx || !words_in || !out || num_docs < 0) { set_error("invalid argument to pb200_doc_mask_upload"); return PB200_E_INVALID; }
  const size_t need = ((size_t)num_docs + 31) / 32, words = doc_mask_words(num_docs);
  if ((size_t)num_words < need) { set_error("doc mask needs %zu words, got %lld", need, (long long)num_words); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  void* p = nullptr;
  int rc = dev_alloc(ctx, words * 4, &p);
  if (rc) return rc;
  cudaStream_t st = take_stream(ctx);
  cudaError_t e = cudaMemsetAsync((uint32_t*)p + need, 0, (words - need) * 4, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(p, words_in, need * 4, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  give_stream(ctx, st);
  if (e != cudaSuccess) { dev_free(ctx, p); set_error("doc mask upload failed: %s", cudaGetErrorString(e)); return PB200_E_CUDA; }
  *out = (uint32_t*)p;
  return PB200_OK;
}
extern "C" int32_t pb200_doc_mask_free(pb200_ctx* ctx, uint32_t* mask) {
  if (ctx && mask) dev_free(ctx, mask);
  return PB200_OK;
}

extern "C" int32_t pb200_last_phases(double* out_ms) {
  if (!out_ms) { set_error("null argument"); return PB200_E_INVALID; }
  memcpy(out_ms, g_phase_ms, sizeof g_phase_ms);
  return PB200_OK;
}

extern "C" int32_t pb200_init(int32_t device, pb200_ctx** out) {
  if (!out) { set_error("ctx out pointer is NULL"); return PB200_E_INVALID; }
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("no CUDA device available (%s): libpinot_b200 has no CPU fallback", cudaGetErrorString(e));
    cudaGetLastError();
    return PB200_E_CUDA;
  }
  if (device < 0 || device >= n) { set_error("device %d out of range [0,%d)", device, n); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(device));
  auto* ctx = new pb200_ctx();
  ctx->device = device;
  cudaDeviceProp prop;
  PB200_CUDA(cudaGetDeviceProperties(&prop, device));
  ctx->sm_count = prop.multiProcessorCount;
  ctx->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 only
    set_error("device sm_%d%d: this library is built for sm_90a (TMA bulk copies + mbarrier)", prop.major, prop.minor);
    delete ctx;
    return PB200_E_UNSUPPORTED;
  }
  {  // tuning knobs: environment read once here
    Tuning& t = ctx->tune;
    auto env_i = [](const char* n, long long dflt) -> long long { const char* v = getenv(n); return v ? atoll(v) : dflt; };
    const int w = (int)env_i("PB200_W", t.warps);
    if (w == 6 || w == 8) t.warps = w;
    t.sparse_max = (int)env_i("PB200_SPARSE_MAX", t.sparse_max);
    t.sparse_max_agg = (int)env_i("PB200_SPARSE_MAX_AGG", t.sparse_max_agg);
    t.ctas_per_sm = (int)std::max<long long>(1, std::min<long long>(2, env_i("PB200_CTAS", t.ctas_per_sm)));
    t.stages = (int)env_i("PB200_STAGES", 0);
    t.grid = (int)env_i("PB200_GRID", 0);
    t.smem_groups = getenv("PB200_NO_SMEM_GROUPS") ? 0 : 1;
    t.smem_groups_max = env_i("PB200_SMEM_GROUPS_MAX", t.smem_groups_max);
    t.smem_copies = (int)env_i("PB200_SMEM_COPIES", 0);
    t.dense_max = env_i("PB200_DENSE_MAX", t.dense_max);
    t.defer = getenv("PB200_NO_DEFER") ? 0 : 1;
    t.gb_defer = getenv("PB200_NO_GB_DEFER") ? 0 : 1;
    t.spec = getenv("PB200_NO_SPEC") ? 0 : 1;
    t.pack_count = getenv("PB200_NO_PACK_COUNT") ? 0 : 1;
    t.pack_shift = (int)env_i("PB200_PACK_SHIFT", 0);
    t.table_stride = (int)env_i("PB200_TABLE_STRIDE", 0);
    t.skip = getenv("PB200_NO_SKIP") ? 0 : 1;
    t.always_count = getenv("PB200_ALWAYS_COUNT") ? 1 : 0;
    if (const char* e = getenv("PB200_RAW_DICT_MAX")) t.raw_dict_max = std::max(0, atoi(e));
  }
  *out = ctx;
  return PB200_OK;
}

extern "C" int32_t pb200_tuning_set(pb200_ctx* ctx, const char* name, int64_t value) {
  if (!ctx || !name) { set_error("null argument"); return PB200_E_INVALID; }
  Tuning& t = ctx->tune;
  std::lock_guard<std::mutex> g(ctx->mu);
  const std::string n(name);
  if (n == "warps") { if (value != 6 && value != 8) { set_error("warps must be 6 or 8"); return PB200_E_INVALID; } t.warps = (int)value; }
  else if (n == "sparse_max") t.sparse_max = (int)value;
  else if (n == "sparse_max_agg") t.sparse_max_agg = (int)value;
  else if (n == "ctas_per_sm") t.ctas_per_sm = (int)std::max<int64_t>(1, std::min<int64_t>(2, value));
  else if (n == "stages") t.stages = (int)value;
  else if (n == "grid") t.grid = (int)value;
  else if (n == "smem_groups") t.smem_groups = value != 0;
  else if (n == "smem_groups_max") t.smem_groups_max = value;
  else if (n == "smem_copies") t.smem_copies = (int)value;
  else if (n == "dense_max") t.dense_max = value;
  else if (n == "defer") t.defer = value != 0;
  else if (n == "gb_defer") t.gb_defer = value != 0;
  else if (n == "spec") t.spec = value != 0;
  else if (n == "pack_count") t.pack_count = value != 0;
  else if (n == "pack_shift") t.pack_shift = (int)value;
  else if (n == "table_stride") t.table_stride = (int)value;
  else if (n == "skip") t.skip = value != 0;
  else if (n == "always_count") t.always_count = value != 0;
  else if (n == "raw_dict_max") t.raw_dict_max = (int)std::max<int64_t>(0, std::min<int64_t>(value, 1 << 28));
  else { set_error("unknown tuning knob '%s'", name); return PB200_E_INVALID; }
  return PB200_OK;
}

extern "C" int32_t pb200_shutdown(pb200_ctx* ctx) {
  if (!ctx) return PB200_OK;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  pb200_comm_shutdown(ctx);
  for (auto s : ctx->free_streams) cudaStreamDestroy(s);
  for (auto e : ctx->free_events) cudaEventDestroy(e);
  for (auto& kv : ctx->block_size) cudaFree(kv.first);
  for (auto& kv : ctx->free_pinned) cudaFreeHost(kv.second);
  delete ctx;
  return PB200_OK;
}

extern "C" int32_t pb200_device_info(pb200_ctx* ctx, int64_t out[5]) {
  if (!ctx || !out) { set_error("null argument"); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  cudaDeviceProp prop;
  PB200_CUDA(cudaGetDeviceProperties(&prop, ctx->device));
  size_t fr = 0, tot = 0;
  PB200_CUDA(cudaMemGetInfo(&fr, &tot));
  out[0] = prop.multiProcessorCount; out[1] = prop.major; out[2] = prop.minor;
  out[3] = (int64_t)(tot >> 20); out[4] = (int64_t)(fr >> 20);
  return PB200_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// segments
// ------------------------------------------------------------------------------------------------------------------
// Blocks of the caching allocator go back to it (load / evict cycles then cost no cudaMalloc / cudaFree, both of which
// synchronise the device); buffers the generator allocated with cudaMalloc are freed directly.
static void free_any(pb200_ctx* ctx, void* p) {
  if (!p) return;
  bool pooled;
  { std::lock_guard<std::mutex> g(ctx->mu); pooled = ctx->block_size.count(p) != 0; }
  if (pooled) dev_free(ctx, p); else cudaFree(p);
}
static void free_column(pb200_ctx* ctx, DeviceColumn& c) {
  if (c.owns) { free_any(ctx, c.fwd); free_any(ctx, c.inv); }
  if (!c.dict_shared) free_any(ctx, c.dict_native);
  c.fwd = nullptr; c.inv = nullptr; c.dict_native = nullptr;
}

static int convert_dictionary(pb200_ctx* ctx, const pb200_col_desc& d, DeviceColumn& c, const unsigned char* be) {
  // BIG-endian fixed-width values (SegmentDictionaryCreator.java:117-177) -> native little-endian arrays
  const int w = c.dict_width();
  if (d.dict_bytes < (uint64_t)w * c.cardinality) { set_error("dictionary too short: %llu bytes for %d x %d", (unsigned long long)d.dict_bytes, c.cardinality, w); return PB200_E_INVALID; }
  c.dict_be.assign(be, be + (size_t)w * c.cardinality);
  c.dict_entry_bytes = w;
  c.dict_hash = dictionary_hash(c.stored_type, w, c.cardinality, be);
  c.dict_host.resize((size_t)w * c.cardinality);
  for (int i = 0; i < c.cardinality; i++) {
    if (w == 4) { uint32_t v = be32(be + 4ll * i); memcpy(&c.dict_host[4ull * i], &v, 4); }
    else { uint64_t v = be64(be + 8ll * i); memcpy(&c.dict_host[8ull * i], &v, 8); }
  }
  { int rc = dev_alloc(ctx, std::max<size_t>(c.dict_host.size(), 16), &c.dict_native); if (rc) return rc; }
  if (c.stored_type == PB200_INT) {
    // the DEVICE copy of an INT dictionary is biased (value ^ 0x80000000 == value + 2^31 as unsigned): the scan kernel
    // sums unsigned words with 3-input adds and removes count * 2^31 once per tile (SumBiasedU32)
    std::vector<uint32_t> biased(c.cardinality);
    for (int i = 0; i < c.cardinality; i++) { uint32_t v; memcpy(&v, &c.dict_host[4ull * i], 4); biased[i] = v ^ 0x80000000u; }
    PB200_CUDA(cudaMemcpy(c.dict_native, biased.data(), biased.size() * 4, cudaMemcpyHostToDevice));
  } else {
    PB200_CUDA(cudaMemcpy(c.dict_native, c.dict_host.data(), c.dict_host.size(), cudaMemcpyHostToDevice));
  }
  return PB200_OK;
}

extern "C" int32_t pb200_segment_register(pb200_ctx* ctx, const char* name, int32_t num_docs, int32_t ncols,
                                          const pb200_col_desc* cols, pb200_segment** out) {
  if (!ctx || !cols || !out || num_docs < 0 || ncols <= 0) { set_error("invalid argument to pb200_segment_register"); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  // uploads below are asynchronous on a stream of the context's pool (NOT the legacy default stream: concurrent segment
  // loads and queries of other threads must not serialise against each other); whatever way this function returns, they
  // are finished first (the caller's buffers must not be read after the return)
  cudaStream_t up = take_stream(ctx);
  struct DrainUploadStream { pb200_ctx* c; cudaStream_t s; ~DrainUploadStream() { cudaStreamSynchronize(s); give_stream(c, s); } } drain_upload_stream{ctx, up};
  std::unique_ptr<pb200_segment> seg(new pb200_segment());
  seg->ctx = ctx;
  seg->name = name ? name : "";
  seg->num_docs = num_docs;
  seg->cols.reserve((size_t)ncols + PB200_MAX_DERIVED_COLUMNS);  // derived columns append without moving these
  seg->cols.resize(ncols);
  seg->num_stored = ncols;
  seg->published.store(ncols, std::memory_order_release);
  auto fail = [&](int rc) { for (auto& c : seg->cols) free_column(ctx, c); return rc; };
  for (int i = 0; i < ncols; i++) {
    const pb200_col_desc& d = cols[i];
    DeviceColumn& c = seg->cols[i];
    c.fwd_kind = d.fwd_kind; c.stored_type = d.stored_type; c.bits = d.bits_per_value; c.cardinality = d.cardinality;
    const bool on_device = d.flags & PB200_COL_DEVICE_BUFFERS;
    c.owns = !on_device;
    if (d.fwd_kind == PB200_FWD_DICT_FIXEDBIT) {
      if (c.bits < 1 || c.bits > 31) { set_error("column %d: bitsPerElement %d out of range", i, c.bits); return fail(PB200_E_INVALID); }
      uint64_t need = ((uint64_t)num_docs * c.bits + 7) / 8;
      if (d.fwd_bytes < need) { set_error("column %d: forward index has %llu bytes, need %llu", i, (unsigned long long)d.fwd_bytes, (unsigned long long)need); return fail(PB200_E_INVALID); }
      c.fwd_file_bytes = need;
      if (on_device) {
        c.fwd = (uint32_t*)d.fwd;  // generator allocated it padded
        c.fwd_alloc_bytes = d.fwd_bytes;
      } else {
        c.fwd_alloc_bytes = padded_fwd_bytes(num_docs, c.bits);
        void* p = nullptr;
        int rc = dev_alloc(ctx, c.fwd_alloc_bytes, &p);  // pooled: repeated load / evict cycles reuse HBM blocks
        if (rc) return fail(rc);
        c.fwd = (uint32_t*)p;
        c.pooled = true;
        const uint64_t body = need & ~15ull;  // zero only the padding behind the file's bytes
        PB200_CUDA(cudaMemsetAsync((unsigned char*)c.fwd + body, 0, c.fwd_alloc_bytes - body, up));
        // asynchronous on the upload stream: with pinned caller buffers the DMA of this column overlaps the host-side
        // dictionary conversion below and the next column's set-up (pageable buffers are staged synchronously by the
        // runtime); the stream is drained once at the end of the registration
        PB200_CUDA(cudaMemcpyAsync(c.fwd, d.fwd, need, cudaMemcpyHostToDevice, up));
        PB200_CUDA(fwd_words_to_native(c.fwd, c.fwd_alloc_bytes, ctx->sm_count, up));
      }
    } else if (d.fwd_kind == PB200_FWD_DICT_SORTED) {
      // SortedIndexReaderImpl: expand (start,end) pairs into a fixed-bit dictId stream so every kernel sees one format
      if (on_device) { set_error("sorted columns must be registered from host buffers"); return fail(PB200_E_UNSUPPORTED); }
      if (d.fwd_bytes < 8ull * c.cardinality) { set_error("column %d: sorted index too short", i); return fail(PB200_E_INVALID); }
      if (c.bits < 1) c.bits = 1;
      const unsigned char* p = (const unsigned char*)d.fwd;
      c.fwd_file_bytes = ((uint64_t)num_docs * c.bits + 7) / 8;
      c.fwd_alloc_bytes = padded_fwd_bytes(num_docs, c.bits);
      std::vector<unsigned char> packed(c.fwd_alloc_bytes, 0);
      for (int id = 0; id < c.cardinality; id++) {
        int s = (int)be32(p + 8ll * id), e = (int)be32(p + 8ll * id + 4);
        if (s < 0 || e >= num_docs || e < s) { set_error("column %d: bad sorted range", i); return fail(PB200_E_INVALID); }
        for (long long doc = s; doc <= e; doc++) {
          long long bit = doc * c.bits;
          for (int b = c.bits - 1; b >= 0; b--, bit++)
            if ((id >> b) & 1) packed[bit >> 3] |= (unsigned char)(0x80 >> (bit & 7));
        }
      }
      { void* fp = nullptr; int rc = dev_alloc(ctx, c.fwd_alloc_bytes, &fp); if (rc) return fail(rc); c.fwd = (uint32_t*)fp; }
      PB200_CUDA(cudaMemcpyAsync(c.fwd, packed.data(), c.fwd_alloc_bytes, cudaMemcpyHostToDevice, up));  // pageable source: staged before the call returns
      PB200_CUDA(fwd_words_to_native(c.fwd, c.fwd_alloc_bytes, ctx->sm_count, up));
      c.fwd_kind = PB200_FWD_DICT_FIXEDBIT;
    } else if (d.fwd_kind == PB200_FWD_RAW_FIXEDBYTE) {
      // BaseChunkForwardIndexReader header :60-106; only PASS_THROUGH 4-byte values are accelerated
      if (on_device) { set_error("raw columns must be registered from host buffers"); return fail(PB200_E_UNSUPPORTED); }
      const unsigned char* p = (const unsigned char*)d.fwd;
      if (d.fwd_bytes < 28) { set_error("column %d: raw forward index too short", i); return fail(PB200_E_INVALID); }
      int version = (int)be32(p), nchunks = (int)be32(p + 4), entry = (int)be32(p + 12);
      if (version < 2 || be32(p + 20) != 0 || entry != 4 || (d.stored_type != PB200_INT && d.stored_type != PB200_FLOAT)) {
        set_error("column %d: raw forward index version %d / compression %u / width %d not accelerated", i, version, be32(p + 20), entry);
        return fail(PB200_E_UNSUPPORTED);
      }
      uint64_t start = be32(p + 24) + (uint64_t)nchunks * (version <= 2 ? 4 : 8);
      if (d.fwd_bytes < start + 4ull * num_docs) { set_error("column %d: raw data truncated", i); return fail(PB200_E_INVALID); }
      c.bits = 32;
      c.fwd_file_bytes = 4ull * num_docs;
      c.fwd_alloc_bytes = padded_fwd_bytes(num_docs, 32);
      { void* fp = nullptr; int rc = dev_alloc(ctx, c.fwd_alloc_bytes, &fp); if (rc) return fail(rc); c.fwd = (uint32_t*)fp; }
      PB200_CUDA(cudaMemsetAsync(c.fwd, 0, c.fwd_alloc_bytes, up));
      PB200_CUDA(cudaMemcpyAsync(c.fwd, p + start, 4ull * num_docs, cudaMemcpyHostToDevice, up));
      PB200_CUDA(fwd_words_to_native(c.fwd, c.fwd_alloc_bytes, ctx->sm_count, up));
    } else {
      set_error("column %d: unknown forward index kind %d", i, d.fwd_kind);
      return fail(PB200_E_INVALID);
    }
    seg->device_bytes += (int64_t)c.fwd_alloc_bytes;
    if (d.dict && d.stored_type != PB200_STRING && d.fwd_kind != PB200_FWD_RAW_FIXEDBYTE) {
      std::vector<unsigned char> tmp;
      const unsigned char* be = (const unsigned char*)d.dict;
      if (on_device) {
        tmp.resize(d.dict_bytes);
        PB200_CUDA(cudaMemcpy(tmp.data(), d.dict, d.dict_bytes, cudaMemcpyDeviceToHost));
        be = tmp.data();
      }
      int rc = convert_dictionary(ctx, d, c, be);
      if (rc) return fail(rc);
      seg->device_bytes += (int64_t)c.dict_host.size();
    }
    if (d.dict && d.stored_type == PB200_STRING && d.fwd_kind != PB200_FWD_RAW_FIXEDBYTE && !on_device && c.cardinality > 0) {
      // STRING dictionaries never go to the device (keys are dictIds there); the padded entries are kept on the host so
      // that merges can verify / build a common id space (pb200_domain.cu).  Entry width: `reserved`, else bytes / cardinality.
      const int w = d.reserved > 0 ? d.reserved : (int)(d.dict_bytes / (uint64_t)c.cardinality);
      if (w <= 0 || d.dict_bytes < (uint64_t)w * c.cardinality) { set_error("column %d: STRING dictionary too short", i); return fail(PB200_E_INVALID); }
      c.dict_be.assign((const unsigned char*)d.dict, (const unsigned char*)d.dict + (size_t)w * c.cardinality);
      c.dict_entry_bytes = w;
      c.dict_hash = dictionary_hash(PB200_STRING, w, c.cardinality, c.dict_be.data());
    }
    if (d.inv && d.inv_bytes) {
      if (d.inv_bytes < 4ull * (c.cardinality + 1)) { set_error("column %d: inverted index too short", i); return fail(PB200_E_INVALID); }
      c.inv_bytes = d.inv_bytes;
      c.inv_offsets.resize(c.cardinality + 1);
      std::vector<unsigned char> hdr(4ull * (c.cardinality + 1));
      if (on_device) {
        c.inv = (unsigned char*)d.inv;
        PB200_CUDA(cudaMemcpy(hdr.data(), d.inv, hdr.size(), cudaMemcpyDeviceToHost));
      } else {
        { void* ip = nullptr; int rc = dev_alloc(ctx, d.inv_bytes + 16, &ip); if (rc) return fail(rc); c.inv = (unsigned char*)ip; }
        PB200_CUDA(cudaMemcpy(c.inv, d.inv, d.inv_bytes, cudaMemcpyHostToDevice));
        memcpy(hdr.data(), d.inv, hdr.size());
      }
      for (int k = 0; k <= c.cardinality; k++) c.inv_offsets[k] = be32(hdr.data() + 4ll * k);
      if (c.inv_offsets[0] != 4u * (c.cardinality + 1) || c.inv_offsets[c.cardinality] > d.inv_bytes) {
        set_error("column %d: inverted index offsets are not in BitmapInvertedIndexWriter layout", i);
        return fail(PB200_E_INVALID);
      }
      if (!on_device) {  // the device decodes these bitmaps in place: a corrupt file must fail here, not in a kernel
        const unsigned char* ib = (const unsigned char*)d.inv;
        for (int k = 0; k < c.cardinality; k++) {
          if (c.inv_offsets[k + 1] < c.inv_offsets[k]) { set_error("column %d: inverted index offsets not ascending", i); return fail(PB200_E_INVALID); }
          if (pb200_roaring_validate(ib + c.inv_offsets[k], c.inv_offsets[k + 1] - c.inv_offsets[k], num_docs) != PB200_OK) return fail(PB200_E_INVALID);
        }
      }
      seg->device_bytes += (int64_t)d.inv_bytes;
    }
  }
  for (auto& c : seg->cols) c.owns = true;  // adopted device buffers belong to the segment from here on
  {  // every upload / re-layout kernel above ran on the default stream: the caller's buffers may go away after this
    cudaError_t e = cudaStreamSynchronize(up);
    if (e != cudaSuccess) { set_error("segment upload failed: %s", cudaGetErrorString(e)); return fail(PB200_E_CUDA); }
  }
  *out = seg.release();
  return PB200_OK;
}

extern "C" int32_t pb200_segment_release(pb200_ctx* ctx, pb200_segment* seg) {
  if (!seg) return PB200_OK;
  cudaSetDevice(seg->ctx->device);
  for (auto& c : seg->cols) free_column(seg->ctx, c);
  if (seg->domain) pb200_domain_release(seg->ctx, seg->domain);
  delete seg;
  return PB200_OK;
}

extern "C" int64_t pb200_segment_device_bytes(const pb200_segment* seg) { return seg ? seg->device_bytes : 0; }

extern "C" int32_t pb200_segment_column_info(const pb200_segment* seg, int32_t col, int64_t out[6]) {
  if (!seg || col < 0 || col >= seg->num_columns()) { set_error("bad column"); return PB200_E_INVALID; }
  const DeviceColumn& c = seg->cols[col];
  out[0] = c.fwd_kind; out[1] = c.stored_type; out[2] = c.bits; out[3] = c.cardinality; out[4] = c.inv != nullptr;
  out[5] = (int64_t)c.fwd_file_bytes;
  return PB200_OK;
}

extern "C" int64_t pb200_segment_read_index(pb200_ctx* ctx, const pb200_segment* seg, int32_t col, int32_t which,
                                            void* out, uint64_t cap) {
  if (!seg || col < 0 || col >= seg->num_columns()) { set_error("bad column"); return PB200_E_INVALID; }
  const DeviceColumn& c = seg->cols[col];
  cudaSetDevice(seg->ctx->device);
  if (which == 0) {
    if (!out) return (int64_t)c.fwd_file_bytes;
    if (cap < c.fwd_file_bytes) { set_error("buffer too small"); return PB200_E_INVALID; }
    // back to the file's big-endian words (the HBM copy holds native words)
    std::vector<uint32_t> words((c.fwd_file_bytes + 3) / 4);
    if (cudaMemcpy(words.data(), c.fwd, words.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { set_error("D2H failed"); return PB200_E_CUDA; }
    for (auto& w : words) w = bswap32(w);
    memcpy(out, words.data(), c.fwd_file_bytes);
    return (int64_t)c.fwd_file_bytes;
  } else if (which == 1) {
    if (!out) return (int64_t)c.dict_be.size();
    if (cap < c.dict_be.size()) { set_error("buffer too small"); return PB200_E_INVALID; }
    memcpy(out, c.dict_be.data(), c.dict_be.size());
    return (int64_t)c.dict_be.size();
  } else if (which == 2) {
    if (!out) return (int64_t)c.inv_bytes;
    if (cap < c.inv_bytes) { set_error("buffer too small"); return PB200_E_INVALID; }
    if (c.inv_bytes && cudaMemcpy(out, c.inv, c.inv_bytes, cudaMemcpyDeviceToHost) != cudaSuccess) { set_error("D2H failed"); return PB200_E_CUDA; }
    return (int64_t)c.inv_bytes;
  }
  set_error("which must be 0,1,2");
  return PB200_E_INVALID;
}

// ------------------------------------------------------------------------------------------------------------------
// query execution: plan (pb200_plan.cpp) -> bind device buffers -> launch -> verify -> results
// ------------------------------------------------------------------------------------------------------------------
namespace pb200 {
cudaError_t launch_scan_variant(const ScanVariant& v, size_t smem_bytes, int grid, const QueryDesc& q, const TmaTable& tt,
                                const SegDesc* dsegs, cudaStream_t st) {
  if (v.group_by) {
    if (v.spec) {
      if (v.warps == 8 && v.min_blocks == 1) return launch_scan_w8_gb1_spec(smem_bytes, grid, q, tt, dsegs, st);
      if (v.warps == 6 && v.min_blocks == 2) return launch_scan_w6_gb2_spec(smem_bytes, grid, q, tt, dsegs, st);
      return cudaErrorInvalidValue;
    }
    if (v.min_blocks >= 2) return v.warps == 8 ? launch_scan_w8_gb2(smem_bytes, grid, q, tt, dsegs, st) : launch_scan_w6_gb2(smem_bytes, grid, q, tt, dsegs, st);
    return v.warps == 8 ? launch_scan_w8_gb1(smem_bytes, grid, q, tt, dsegs, st) : launch_scan_w6_gb1(smem_bytes, grid, q, tt, dsegs, st);
  }
  if (v.warps == 8) return v.defer ? launch_scan_w8_agg(smem_bytes, grid, q, tt, dsegs, st) : launch_scan_w8_agg_nodefer(smem_bytes, grid, q, tt, dsegs, st);
  return launch_scan_w6_agg(smem_bytes, grid, q, tt, dsegs, st);
}

// Device buffers of the plan's filter leaves: LUTs, doc masks, range lists, and every posting list decoded by ONE launch;
// the leaf descriptors in plan.segs point at them.  They live in `temps` until the caller is done with the launch.
int bind_leaf_buffers(pb200_ctx* ctx, ScanPlan& plan, cudaStream_t st, std::vector<std::unique_ptr<DevBufRaw>>& temps) {
  std::vector<DecodeJob> decode_jobs;
  auto temp = [&](size_t bytes, void** p) -> int {
    temps.emplace_back(new DevBufRaw(ctx));
    const int rc = temps.back()->alloc(bytes);
    *p = temps.back()->p;
    return rc;
  };
  for (const LeafBuffer& b : plan.leaf_buffers) {
    void* vp = nullptr;
    if (int rc = temp(b.words * 4, &vp)) return rc;
    uint32_t* p = static_cast<uint32_t*>(vp);
    LeafDesc& lf = plan.segs[b.seg].leaves[b.leaf];
    if (b.kind == LeafBuffer::DOC_RANGES) lf.ranges = reinterpret_cast<const int32_t*>(p); else lf.bits = p;
    switch (b.kind) {
      case LeafBuffer::LUT:
        PB200_CUDA(cudaMemcpyAsync(p, b.lut.data(), b.words * 4, cudaMemcpyHostToDevice, st));
        PB200_CUDA(cudaStreamSynchronize(st));
        break;
      case LeafBuffer::INV_MASK:
        PB200_CUDA(cudaMemsetAsync(p, 0, b.words * 4, st));
        for (DecodeJob j : b.jobs) { j.mask = p; decode_jobs.push_back(j); }
        break;
      case LeafBuffer::DOC_MASK:
        PB200_CUDA(cudaMemsetAsync(p + b.src_words, 0, (b.words - b.src_words) * 4, st));
        PB200_CUDA(cudaMemcpyAsync(p, b.src, b.src_words * 4, cudaMemcpyHostToDevice, st));
        PB200_CUDA(cudaStreamSynchronize(st));  // caller's buffer may be a temporary
        break;
      case LeafBuffer::DOC_RANGES:
        PB200_CUDA(cudaMemcpyAsync(p, b.src, b.src_words * 4, cudaMemcpyHostToDevice, st));
        PB200_CUDA(cudaStreamSynchronize(st));
        break;
    }
  }
  if (!decode_jobs.empty()) {
    void* jobs_dev = nullptr;
    if (int rc = temp(sizeof(DecodeJob) * decode_jobs.size(), &jobs_dev)) return rc;
    if (int rc = roaring_decode_batch(ctx, st, decode_jobs, jobs_dev)) return rc;
  }
  return PB200_OK;
}

int launch_chunks(pb200_ctx* ctx, cudaStream_t st, const ScanPlan& plan, DevBufRaw& dsegs, EventPair& ev, const char* what,
                  uint32_t* mask, const long long* chunk_word_off, double* t_launch) {
  const size_t bytes = sizeof(SegDesc) * plan.segs.size();
  if (int rc = dsegs.alloc(bytes)) return rc;
  if (int rc = ev.take()) return rc;
  PB200_CUDA(cudaMemcpyAsync(dsegs.p, plan.segs.data(), bytes, cudaMemcpyHostToDevice, st));
  if (t_launch) *t_launch = now_ms();
  PB200_CUDA(cudaEventRecord(ev.a, st));
  for (size_t c = 0; c < plan.chunks.size(); c++) {
    const LaunchChunk& ch = plan.chunks[c];
    QueryDesc cq = plan.q;
    cq.num_segments = ch.num_segs;
    cq.total_tiles = ch.total_tiles;
    if (mask) set_selection_mask(cq, mask + chunk_word_off[c]);
    const cudaError_t le = launch_scan_variant(plan.variant, plan.smem_bytes, ch.grid, cq, tma_table(plan, ch),
                                               static_cast<const SegDesc*>(dsegs.p) + ch.first_seg, st);
    if (le != cudaSuccess) { set_error("%s launch failed: %s (smem %zu B, grid %d)", what, cudaGetErrorString(le), plan.smem_bytes, ch.grid); return PB200_E_CUDA; }
  }
  PB200_CUDA(cudaEventRecord(ev.b, st));
  return PB200_OK;
}
}  // namespace pb200

// Internal return code of execute_impl: a count-carrying sum overflowed its field (detected exactly, see
// ScanCall::read_back_and_verify) -- the caller runs the submission again with separate COUNT reductions.
constexpr int kRetryWithoutCountCarrier = 1;
static int execute_impl(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments, int32_t nseg,
                        pb200_result** results, bool allow_count_carrier, const pb200_order_by* order, const double* agg_args,
                        const pb200_having* having, const pb200_agg_arg* wt_args, const ExprCall* ex = nullptr,
                        const pb200_post_aggs* post = nullptr);
static int execute_checked(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                           const pb200_having* having, pb200_segment* const* segments, int32_t nseg, pb200_result** results,
                           const ExprCall* ex, const pb200_post_aggs* post = nullptr);

extern "C" int32_t pb200_execute_having(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const double* agg_args,
                                        const pb200_having* having, pb200_segment* const* segments, int32_t nseg,
                                        pb200_result** results) {
  if (query) {
    if (const int vrc = order_validate(order, query->num_aggs, query->num_group_by)) return vrc;
    const int nres = (query->flags & PB200_Q_MERGE_SEGMENTS) ? 1 : nseg;
    const bool deferred = (query->flags & PB200_Q_DEFER_FINALIZE) || query->reduce_world > 1;
    if (const int hrc = having_check(having, query->num_aggs, query->num_group_by, nres, deferred)) return hrc;
  }
  int rc = execute_impl(ctx, query, segments, nseg, results, true, order, agg_args, having, nullptr);
  if (rc == kRetryWithoutCountCarrier) rc = execute_impl(ctx, query, segments, nseg, results, false, order, agg_args, having, nullptr);
  return rc;
}

extern "C" int32_t pb200_execute_agg_args(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                                          const pb200_having* having, pb200_segment* const* segments, int32_t nseg,
                                          pb200_result** results) {
  if (!query || !args || query->num_aggs < 0 || query->num_aggs > kMaxAggs || (query->num_aggs > 0 && !query->aggs))
    return pb200_execute_having(ctx, query, order, nullptr, having, segments, nseg, results);
  return execute_checked(ctx, query, order, args, having, segments, nseg, results, nullptr);
}

int pb200::execute_exprs_post(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                              const pb200_having* having, const pb200_expr_program* exprs, const pb200_expr_conds* conds,
                              const pb200_post_aggs* post, pb200_segment* const* segments, int32_t nseg, pb200_result** results) {
  if (!exprs && !post) return pb200_execute_agg_args(ctx, query, order, args, having, segments, nseg, results);
  if (!ctx || !results) { set_error("invalid argument to %s", exprs ? "pb200_execute_exprs" : "pb200_execute_post"); return PB200_E_INVALID; }
  if (post && (!query || query->num_aggs < 0 || (query->num_aggs > 0 && !query->aggs))) {
    set_error("invalid query passed to pb200_execute_post");
    return PB200_E_INVALID;
  }
  if (post && query->num_aggs > kMaxAggs) {   // as the scan planner refuses it: the stock operator runs the query
    set_error("query exceeds device limits (aggs %d/%d)", query->num_aggs, kMaxAggs);
    return PB200_E_UNSUPPORTED;
  }
  ExprCall ex;
  if (exprs)
    if (const int rc = expr_prepare(query, exprs, conds, segments, nseg, &ex)) return rc;
  if (!ex.count)
    return post ? execute_checked(ctx, query, order, args, having, segments, nseg, results, nullptr, post)
                : pb200_execute_agg_args(ctx, query, order, args, having, segments, nseg, results);
  // the scan runs every expression aggregation as COUNT(*): its group tables and counts are what the expressions need
  pb200_query q = *query;
  pb200_agg aggs[kMaxAggs];
  for (int a = 0; a < q.num_aggs; a++) aggs[a] = ex.fn_of[a] >= 0 ? pb200_agg{PB200_AGG_COUNT, -1} : query->aggs[a];
  q.aggs = aggs;
  return execute_checked(ctx, &q, order, args, having, segments, nseg, results, &ex, post);
}

extern "C" int32_t pb200_execute_exprs(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                                       const pb200_having* having, const pb200_expr_program* exprs, pb200_segment* const* segments,
                                       int32_t nseg, pb200_result** results) {
  return pb200::execute_exprs_post(ctx, query, order, args, having, exprs, nullptr, nullptr, segments, nseg, results);
}

extern "C" int32_t pb200_execute_exprs_cond(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                                            const pb200_having* having, const pb200_expr_program* exprs, const pb200_expr_conds* conds,
                                            pb200_segment* const* segments, int32_t nseg, pb200_result** results) {
  if (conds && !exprs) { set_error("invalid argument to pb200_execute_exprs_cond: conditions without programs"); return PB200_E_INVALID; }
  return pb200::execute_exprs_post(ctx, query, order, args, having, exprs, conds, nullptr, segments, nseg, results);
}

extern "C" int32_t pb200_execute_post(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                                      const pb200_having* having, const pb200_post_aggs* post, pb200_segment* const* segments,
                                      int32_t nseg, pb200_result** results) {
  return pb200::execute_exprs_post(ctx, query, order, args, having, nullptr, nullptr, post, segments, nseg, results);
}

// pb200_execute_agg_args past its argument check (args NULL: no percentiles and no *WITHTIME), with the expression
// aggregations of pb200_execute_exprs (ex NULL: none) and the post-aggregation programs of pb200_execute_post (post NULL:
// none)
static int execute_checked(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                           const pb200_having* having, pb200_segment* const* segments, int32_t nseg, pb200_result** results,
                           const ExprCall* ex, const pb200_post_aggs* post) {
  if (const int vrc = order_validate(order, query->num_aggs, query->num_group_by, post)) return vrc;
  const int nres = (query->flags & PB200_Q_MERGE_SEGMENTS) ? 1 : nseg;
  const bool deferred = (query->flags & PB200_Q_DEFER_FINALIZE) || query->reduce_world > 1;
  if (const int hrc = having_check(having, query->num_aggs, query->num_group_by, nres, deferred)) return hrc;
  // ORDER BY / HAVING compare the double column: for a STRING-typed *WITHTIME that is a dictId, not a value
  if (args && segments && nseg > 0 && segments[0] && query->num_group_by > 0) {
    auto string_wt = [&](int a) {
      const pb200_agg& ag = query->aggs[a];
      return is_withtime_fn(ag.function) && ag.column >= 0 && ag.column < (int)segments[0]->cols.size() &&
             segments[0]->cols[ag.column].stored_type == PB200_STRING;
    };
    for (int i = 0; order && i < order->num_items; i++)
      if (order->items[i].kind == PB200_ORDER_AGG && string_wt(order->items[i].index)) {
        set_error("ORDER BY a STRING FIRST/LASTWITHTIME is not accelerated"); return PB200_E_UNSUPPORTED;
      }
    for (int i = 0; order && post && i < order->num_items; i++) {
      if (order->items[i].kind != PB200_ORDER_POST) continue;
      const pb200_post_program& pp = post->programs[order->items[i].index];
      for (int k = 0; k < pp.num_nodes; k++)
        if (pp.nodes[k].op == PB200_POST_AGG && string_wt(pp.nodes[k].agg)) {
          set_error("ORDER BY an expression over a STRING FIRST/LASTWITHTIME is not accelerated"); return PB200_E_UNSUPPORTED;
        }
    }
    for (int i = 0; having && i < having->num_nodes; i++) {
      const pb200_having_node& hn = having->nodes[i];
      if ((hn.op == PB200_HAVING_RANGE || hn.op == PB200_HAVING_EQ || hn.op == PB200_HAVING_NEQ) && string_wt(hn.agg)) {
        set_error("HAVING on a STRING FIRST/LASTWITHTIME is not accelerated"); return PB200_E_UNSUPPORTED;
      }
    }
  }
  double p[kMaxAggs] = {};
  for (int a = 0; args && a < query->num_aggs; a++) p[a] = args[a].p;
  const double* agg_args = args ? p : nullptr;
  // a retry rebuilds every table of the attempt, the expression tables included
  int rc = execute_impl(ctx, query, segments, nseg, results, true, order, agg_args, having, args, ex, post);
  if (rc == kRetryWithoutCountCarrier) rc = execute_impl(ctx, query, segments, nseg, results, false, order, agg_args, having, args, ex, post);
  return rc;
}

extern "C" int32_t pb200_execute_args(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const double* agg_args,
                                      pb200_segment* const* segments, int32_t nseg, pb200_result** results) {
  return pb200_execute_having(ctx, query, order, agg_args, nullptr, segments, nseg, results);
}

extern "C" int32_t pb200_execute_ordered(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order,
                                         pb200_segment* const* segments, int32_t nseg, pb200_result** results) {
  return pb200_execute_args(ctx, query, order, nullptr, segments, nseg, results);
}

extern "C" int32_t pb200_execute(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments,
                                 int32_t nseg, pb200_result** results) {
  return pb200_execute_ordered(ctx, query, nullptr, segments, nseg, results);
}

// Per result: {sum over the table of the carried counts, largest low (sum) field, largest carried count} -- pb200_execute's verification.
__global__ void carrier_verify_kernel(const unsigned long long* __restrict__ tab, long long n, int shift, unsigned long long* __restrict__ out) {
  unsigned long long c = 0, mx = 0, mc = 0;
  const unsigned long long mask = (1ull << shift) - 1ull;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long v = tab[i];
    c += v >> shift;
    mc = max(mc, v >> shift);
    mx = max(mx, v & mask);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
    mx = max(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
    mc = max(mc, __shfl_xor_sync(0xFFFFFFFFu, mc, o));
  }
  if ((threadIdx.x & 31) == 0) { if (c) atomicAdd(out, c); if (mx) atomicMax(out + 1, mx); if (mc) atomicMax(out + 2, mc); }
}

namespace {
// The accumulator block of one call: on the device, and in each half of a pooled pinned block (initial values go up and
// results come back through it, both asynchronously on the call's stream: a pageable cudaMemcpy would synchronise the
// device twice per query).  nres AggAccum records, then 4 words per result for the count-carrier verification {sum of
// carried counts, largest sum field, largest carried count, unused}, then per result kMaxAggs OneEntry records.
// Aggregation only, AggAccum's fields and the OneEntry records are the result's one-entry tables: the scan and the
// finalize stages write them like a GROUP BY result's tables, and one decoder (pb200_decode.h) reads both.
struct OneEntry {
  unsigned long long wt_key;         // FIRST/LASTWITHTIME: the scan's winning key...
  long long wt_time;                 // ... and the finalize's time value ...
  unsigned long long ds[kDsWords];   // DISTINCTSUM / DISTINCTAVG: the set's finalized state (record of ScanPlan::ds_rep)
  unsigned long long xkey;           // expression aggregations (pb200_expr.cu): the f64 sum, or a MIN / MAX Double.compare key
  long long hll;                     // DISTINCTCOUNTHLL: the estimate (record of ScanPlan::hll_rep)
  uint32_t pct_id, pct_n;            // PERCENTILE: the selected dictId; values (record of the histogram's owner)
  uint32_t wt_id;                    // FIRST/LASTWITHTIME: ... and data dictId
};
struct AccumLayout {
  size_t verify_off = 0, one_off = 0, bytes = 0;
  AccumLayout() = default;
  explicit AccumLayout(int nres)
      : verify_off(sizeof(AggAccum) * nres), one_off(verify_off + 32ull * nres), bytes(one_off + sizeof(OneEntry) * kMaxAggs * nres) {}
  static AggAccum* records(void* b) { return static_cast<AggAccum*>(b); }
  unsigned long long* verify(void* b) const { return reinterpret_cast<unsigned long long*>(static_cast<unsigned char*>(b) + verify_off); }
  OneEntry* one(void* b, int r) const { return reinterpret_cast<OneEntry*>(static_cast<unsigned char*>(b) + one_off) + (size_t)r * kMaxAggs; }
};

// The byte every entry of fn's u32 / u64 tables starts at: the min reductions (MIN, FIRSTWITHTIME keys, expression MIN
// keys) at all ones, the rest at zero.
int start_byte(int fn) { return fn == PB200_AGG_MIN || fn == PB200_AGG_FIRSTWITHTIME ? 0xFF : 0; }

// Frees a result's group tables and PERCENTILE selections; its histograms too unless keep_hist (pb200_result_histogram).
void release_tables(pb200_result& R, bool keep_hist) {
  pb200_result::Dense& d = R.dense;
  if (d.ctx) {
    dev_free(d.ctx, d.i64_block); dev_free(d.ctx, d.f64_block); dev_free(d.ctx, d.u32max_block); dev_free(d.ctx, d.u32min_block);
    dev_free(d.ctx, d.hkeys); dev_free(d.ctx, d.hctl);
    for (int a = 0; a < kMaxAggs; a++) { dev_free(d.ctx, d.dbits[a]); d.dbits[a] = nullptr; dev_free(d.ctx, d.ds_state[a]); d.ds_state[a] = nullptr; }
    for (int a = 0; a < kMaxAggs; a++) { dev_free(d.ctx, d.hll_est[a]); d.hll_est[a] = nullptr; }
    for (int a = 0; a < kMaxAggs; a++) { dev_free(d.ctx, d.expr_tab[a]); d.expr_tab[a] = nullptr; }
    d.i64_block = d.f64_block = d.u32max_block = d.u32min_block = nullptr;
    d.hkeys = nullptr; d.hctl = nullptr;
    d.live = false;
  }
  pb200_result::Pct& p = R.pct;
  if (p.ctx)
    for (int a = 0; a < kMaxAggs; a++) {
      if (!keep_hist) { dev_free(p.ctx, p.hist[a]); p.hist[a] = nullptr; }
      dev_free(p.ctx, p.ids[a]); dev_free(p.ctx, p.n[a]); p.ids[a] = p.n[a] = nullptr;
    }
  pb200_result::LazySets& L = R.lazy;
  if (L.ctx && !keep_hist)   // the kept DISTINCTCOUNTHLL sets go with the result, like its histograms
    for (int b = 0; b < kMaxAggs; b++) { dev_free(L.ctx, L.bits[b]); L.bits[b] = nullptr; }
  pb200_result::Wt& w = R.wt;
  if (d.ctx)
    for (int a = 0; a < kMaxAggs; a++) {
      dev_free(d.ctx, w.key[a]); dev_free(d.ctx, w.ids[a]); dev_free(d.ctx, w.time[a]);
      w.key[a] = nullptr; w.ids[a] = nullptr; w.time[a] = nullptr;
    }
}

// One attempt of pb200_execute; execute_impl runs its stages in order.  Members are only the state that crosses stages.
struct ScanCall {
  pb200_ctx* const ctx;
  const pb200_query* const query;
  pb200_segment* const* const segments;
  const int nseg;
  double t_enter = 0, t_launch = 0, t_queued = 0, t_synced = 0, t_results = 0;
  Tuning tune;
  ScanPlan plan;
  std::optional<StreamLease> lease;                  // taken once the plan stands
  cudaStream_t st = nullptr;
  std::vector<std::unique_ptr<pb200_result>> res;    // freed with their device state unless handed out
  std::vector<std::unique_ptr<DevBufRaw>> temps;     // leaf buffers and PERCENTILE scratch, needed until the call returns
  struct PinnedScratch {
    pb200_ctx* c; void* p = nullptr; size_t bytes = 0;
    ~PinnedScratch() { pinned_free(c, p, bytes); }
  } pin{ctx};
  AccumLayout acc;
  DevBufRaw accum{ctx};
  unsigned char* back = nullptr;                     // the pinned half the accumulator block is read back into
  std::vector<std::vector<std::unique_ptr<DevBufRaw>>> distinct_bufs;  // aggregation only: DISTINCTCOUNT bitsets
  DevBufRaw dsegs{ctx};
  EventPair ev{ctx};                                 // around the scan launches
  const ExprCall* ex = nullptr;                      // expression aggregations (pb200_execute_exprs), run as COUNT(*) by the scan
  int expr_fn(int a) const { return ex ? ex->fn_of[a] : -1; }

  ~ScanCall() { for (auto& r : res) if (r) pb200_result_free(r.release()); }

  // 1. the call's arguments and device, and the tuning snapshot the planner reads
  int check_call(pb200_result** results) {
    if (!ctx || !query || !segments || !results || nseg <= 0) { set_error("invalid argument to pb200_execute"); return PB200_E_INVALID; }
    t_enter = now_ms();
    PB200_CUDA(cudaSetDevice(ctx->device));
    for (int s = 0; s < nseg; s++)
      if (segments[s] && segments[s]->ctx != ctx) { set_error("segment %d does not belong to this context / schema", s); return PB200_E_INVALID; }
    std::lock_guard<std::mutex> g(ctx->mu);
    tune = ctx->tune;
    return PB200_OK;
  }

  // 2. VAR / STDDEV limb dictionaries (pb200_moments.cu), then every decision about the launch (pb200_plan.cpp)
  int prepare_and_plan(bool allow_count_carrier, const double* agg_args, const pb200_agg_arg* wt_args) {
    if (int rc = moments_prepare(ctx, query, segments, nseg)) return rc;
    if (int rc = hll_prepare(ctx, query, segments, nseg)) return rc;
    return plan_scan(tune, DeviceLimits{ctx->sm_count, ctx->max_smem_optin}, query, segments, nseg, allow_count_carrier, &plan, agg_args, wt_args);
  }

  // 3. the stream, the results, and the device buffers of the filter leaves
  int alloc_results() {
    lease.emplace(ctx);
    st = *lease;
    for (int r = 0; r < plan.nres; r++) {
      res.emplace_back(new pb200_result());
      res.back()->pct.ctx = ctx;
      for (int a = 0; a < plan.q.num_aggs; a++) res.back()->pct.rep[a] = plan.pct_rep[a];
      describe_aggs(r);
    }
    return bind_leaf_buffers(ctx, plan, st, temps);
  }
  // result r's aggregations, on both routes: functions, value kinds, columns and shared states.  An expression
  // aggregation is the function the caller asked for over a DOUBLE value (the scan runs it as COUNT(*)).
  void describe_aggs(int r) {
    const pb200_segment* seg = segments[plan.merge ? 0 : r];
    pb200_result::Dense& d = res[r]->dense;
    for (int a = 0; a < plan.num_user_aggs; a++) {
      d.aggs.push_back(query->aggs[a]);
      d.val_kind.push_back(plan.q.aggs[a].val_kind);
      if (expr_fn(a) >= 0) { d.aggs[a].function = expr_fn(a); d.val_kind[a] = VAL_DICT_F64; }
      d.agg_cols.push_back(plan.q.aggs[a].slot < 0 ? nullptr : &seg->cols[query->aggs[a].column]);
      d.mom_first[a] = plan.mom_first[a];
      if (plan.mom_first[a] >= 0) d.mom_e[a] = seg->cols[query->aggs[a].column].moments->grid.e;
      d.ds_rep[a] = plan.ds_rep[a];
      d.hll_log2m[a] = plan.hll_log2m[a];
      d.hll_rep[a] = plan.hll_rep[a];
    }
  }

  // 4. the accumulator block, initialised with one copy from the pinned block's first half
  int bind_accumulators() {
    acc = AccumLayout(plan.nres);
    if (int rc = pinned_alloc(ctx, 2 * acc.bytes, &pin.p, &pin.bytes)) return rc;
    unsigned char* const init = static_cast<unsigned char*>(pin.p);
    back = init + acc.bytes;
    AggAccum init_acc;
    memset(&init_acc, 0, sizeof init_acc);
    for (int a = 0; a < kMaxAggs; a++) init_acc.min_id[a] = 0xFFFFFFFFu;
    memset(init, 0, acc.bytes);
    for (int r = 0; r < plan.nres; r++) {
      AccumLayout::records(init)[r] = init_acc;
      for (int a = 0; a < plan.num_user_aggs; a++) {
        OneEntry& o = acc.one(init, r)[a];
        const int fn = expr_fn(a) >= 0 ? expr_fn(a) : plan.q.aggs[a].function;
        memset(&o.wt_key, start_byte(fn), 8);
        memset(&o.xkey, start_byte(fn), 8);
      }
    }
    if (int rc = accum.alloc(acc.bytes)) return rc;
    PB200_CUDA(cudaMemcpyAsync(accum.p, init, acc.bytes, cudaMemcpyHostToDevice, st));
    for (int s = 0; s < nseg; s++) plan.segs[s].accum = AccumLayout::records(accum.p) + (plan.merge ? 0 : s);
    return PB200_OK;
  }

  // 5. aggregation only: DISTINCTCOUNT bitsets, and PERCENTILE dictId histograms (one per result and column, owned by the
  //    result from here on)
  int bind_agg_outputs() {
    const int nagg = plan.q.num_aggs;
    distinct_bufs.resize(plan.nres);
    for (int r = 0; r < plan.nres; r++) {
      distinct_bufs[r].resize(nagg);
      for (int a = 0; a < nagg; a++) {
        const size_t words = plan.distinct_words[r][a];
        if (!words) continue;
        distinct_bufs[r][a].reset(new DevBufRaw(ctx));
        if (int rc = distinct_bufs[r][a]->alloc(words * 4)) return rc;
        PB200_CUDA(cudaMemsetAsync(distinct_bufs[r][a]->p, 0, words * 4, st));
      }
    }
    for (int r = 0; r < plan.nres; r++)
      for (int a = 0; a < nagg; a++) {
        const size_t entries = plan.hist_entries[r][a];
        if (!entries) continue;
        pb200_result::Pct& p = res[r]->pct;
        if (int rc = dev_alloc(ctx, entries * 4, (void**)&p.hist[a])) return rc;
        PB200_CUDA(cudaMemsetAsync(p.hist[a], 0, entries * 4, st));
        p.entries[a] = (uint32_t)entries;
      }
    for (int s = 0; s < nseg; s++) {
      const int r = plan.merge ? 0 : s;
      for (int a = 0; a < nagg; a++) {
        if (distinct_bufs[r][a]) plan.segs[s].distinct_bits[a] = (uint32_t*)distinct_bufs[r][a]->p;
        if (res[r]->pct.hist[a]) plan.segs[s].distinct_bits[a] = res[r]->pct.hist[a];
        if (plan.wt_time[a] >= 0) plan.segs[s].distinct_bits[a] = reinterpret_cast<uint32_t*>(&acc.one(accum.p, r)[a].wt_key);
      }
    }
    return PB200_OK;
  }

  // 6. group-by: each result's tables to the plan's layout (owned by the result from here on), then the segments'
  //    descriptors pointed at them
  int bind_group_tables() {
    for (int r = 0; r < plan.nres; r++)
      if (int rc = build_dense(r)) return rc;
    for (int r = 0; r < plan.nres && ex; r++)
      if (int rc = build_expr_tables(r)) return rc;
    for (int s = 0; s < nseg; s++) {
      SegDesc& sd = plan.segs[s];
      const pb200_result& R = *res[plan.merge ? 0 : s];
      const pb200_result::Dense& d = R.dense;
      sd.g_count = d.count;
      sd.g_seen = d.seen;
      sd.h_keys = d.hkeys;
      sd.h_ctl = d.hctl;
      for (int a = 0; a < plan.q.num_aggs; a++) {
        sd.g_isum[a] = d.isum[a]; sd.g_dsum[a] = d.dsum[a]; sd.g_min[a] = d.gmin[a]; sd.g_max[a] = d.gmax[a];
        sd.distinct_bits[a] = R.pct.hist[a] ? R.pct.hist[a] : R.wt.key[a] ? reinterpret_cast<uint32_t*>(R.wt.key[a]) : d.dbits[a];
      }
    }
    return PB200_OK;
  }
  // expression aggregations: each one's table (the function the caller asked for over a DOUBLE value)
  int build_expr_tables(int r) {
    pb200_result::Dense& d = res[r]->dense;
    for (int a = 0; a < plan.num_user_aggs; a++) {
      const int fn = expr_fn(a);
      if (fn < 0) continue;
      const size_t bytes = (size_t)d.groups * 8;
      if (int rc = dev_alloc(ctx, bytes, &d.expr_tab[a])) return rc;
      PB200_CUDA(cudaMemsetAsync(d.expr_tab[a], start_byte(fn), bytes, st));
      if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) d.dsum[a] = static_cast<double*>(d.expr_tab[a]);
    }
    return PB200_OK;
  }
  int build_dense(int r) {
    const TableLayout& t = plan.tables[r];
    const QueryDesc& q = plan.q;
    pb200_result::Dense& d = res[r]->dense;
    pb200_result::Pct& p = res[r]->pct;
    d.ctx = ctx;
    d.cards = t.cards; d.mult = t.mult; d.mult64 = t.mult64;
    d.groups = t.groups;
    d.stride = t.stride;
    d.live = true;
    d.num_groups_limit = query->num_groups_limit;
    d.pack_agg = t.carrier.agg; d.pack_shift = t.carrier.shift; d.pack_vmin = t.carrier.vmin;
    d.reduce_world = t.reduce_world;
    d.flag_slot = t.flag_slot;
    d.tail_slots = t.tail_slots;
    d.i64_elems = t.i64_elems; d.f64_elems = t.f64_elems; d.u32max_elems = t.u32max_elems; d.u32min_elems = t.u32min_elems;
    auto alloc_block = [&](void** out, long long elems, size_t esz, int fill) -> int {
      if (!elems) return PB200_OK;
      if (int rc = dev_alloc(ctx, (size_t)elems * esz, out)) return rc;
      PB200_CUDA(cudaMemsetAsync(*out, fill, (size_t)elems * esz, st));
      return PB200_OK;
    };
    int rc;
    if (t.hashed) {
      if ((rc = alloc_block((void**)&d.hkeys, t.groups, 8, 0xFF))) return rc;
      if ((rc = alloc_block((void**)&d.hctl, 2, 4, 0))) return rc;
    }
    if ((rc = alloc_block(&d.i64_block, d.i64_elems, 8, 0))) return rc;
    if ((rc = alloc_block(&d.f64_block, d.f64_elems, 8, 0))) return rc;
    if ((rc = alloc_block(&d.u32max_block, d.u32max_elems, 4, 0))) return rc;
    if ((rc = alloc_block(&d.u32min_block, d.u32min_elems, 4, 0xFF))) return rc;
    d.count = t.need_count ? (unsigned long long*)d.i64_block : nullptr;
    d.seen = t.need_seen ? (uint32_t*)d.u32max_block : nullptr;
    for (int a = 0; a < q.num_aggs; a++) {
      const int fn = q.aggs[a].function;
      const long long off = (long long)t.index[a] * t.groups;
      if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) {
        if (sum_in_double(q.aggs[a].val_kind)) d.dsum[a] = (double*)d.f64_block + off;
        else d.isum[a] = (long long*)d.i64_block + off;
      } else if (fn == PB200_AGG_MIN) d.gmin[a] = (uint32_t*)d.u32min_block + off;
      else if (fn == PB200_AGG_MAX) d.gmax[a] = (uint32_t*)d.u32max_block + off;
      else if (owns_bitset(plan, a)) {  // one dictId bitset per group / slot
        const size_t bytes = (size_t)t.dwords[a] * t.groups * 4;
        if ((rc = dev_alloc(ctx, bytes, (void**)&d.dbits[a]))) return rc;
        PB200_CUDA(cudaMemsetAsync(d.dbits[a], 0, bytes, st));
        d.dwords[a] = t.dwords[a];
      }
      if (is_distinct_value_fn(fn)) {   // the set's finalized state per group / slot (pb200_extract.cu runs the finalize)
        unsigned long long*& state = d.ds_state[plan.ds_rep[a]];
        if (!state && (rc = dev_alloc(ctx, (size_t)t.groups * kDsWords * 8, (void**)&state))) return rc;
      } else if (is_hll_fn(fn)) {   // the estimate per group / slot, shared by the HLLs of the column and log2m
        long long*& est = d.hll_est[plan.hll_rep[a]];
        if (!est && (rc = dev_alloc(ctx, (size_t)t.groups * 8, (void**)&est))) return rc;
      } else if (fn == PB200_AGG_PERCENTILE) {  // one dictId histogram per group / slot (owner), a dictId per entry (each)
        if (t.hist_per_group[a]) {
          const size_t entries = (size_t)t.hist_per_group[a] * t.groups;
          if ((rc = dev_alloc(ctx, entries * 4, (void**)&p.hist[a]))) return rc;
          PB200_CUDA(cudaMemsetAsync(p.hist[a], 0, entries * 4, st));
          p.entries[a] = t.hist_per_group[a];
          if ((rc = dev_alloc(ctx, (size_t)t.groups * 4, (void**)&p.n[a]))) return rc;
        }
        if ((rc = dev_alloc(ctx, (size_t)t.groups * 4, (void**)&p.ids[a]))) return rc;
      } else if (is_withtime_fn(fn)) {  // one key per group / slot: u64 min (FIRST) starts at ~0, u64 max (LAST) at 0
        pb200_result::Wt& w = res[r]->wt;
        if ((rc = alloc_block((void**)&w.key[a], t.groups, 8, start_byte(fn)))) return rc;
        if ((rc = dev_alloc(ctx, (size_t)t.groups * 4, (void**)&w.ids[a]))) return rc;
        if ((rc = dev_alloc(ctx, (size_t)t.groups * 8, (void**)&w.time[a]))) return rc;
      }
    }
    if (d.pack_agg >= 0) d.exists_packed = (const unsigned long long*)d.isum[d.pack_agg];
    if (t.exists_min >= 0) d.exists_min = d.gmin[t.exists_min];
    if (t.exists_max >= 0) d.exists_max = d.gmax[t.exists_max];
    return PB200_OK;
  }

  // 7. the descriptors and every chunk's scan, between the call's two events
  int launch() { return launch_chunks(ctx, st, plan, dsegs, ev, "scan kernel", nullptr, nullptr, &t_launch); }

  // entries of result r's tables: its group table's, or the one of an aggregation-only result
  long long entries(int r) const { return plan.group_by ? plan.tables[r].groups : 1; }

  // result r's tables as the finalize stages write them and the decoder reads them: the result's own (group-by), or its
  // one-entry tables in the accumulator block at `block`, the device block or its pinned copy (aggregation only; the
  // host's dictionaries)
  std::array<AggSource, kMaxAggs> sources(int r, unsigned char* block) const {
    std::array<AggSource, kMaxAggs> out{};
    const pb200_result& R = *res[r];
    if (plan.group_by) { agg_sources(R, out.data()); return out; }
    AggAccum& rec = AccumLayout::records(block)[r];
    OneEntry* one = acc.one(block, r);
    const pb200_result::Dense& d = R.dense;
    for (int a = 0; a < (int)d.aggs.size(); a++) {
      AggSource& s = out[a];
      const int fn = s.fn = d.aggs[a].function, vk = s.vk = d.val_kind[a];
      if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG)
        s.src = expr_fn(a) >= 0 ? (void*)&one[a].xkey : sum_in_double(vk) ? (void*)&rec.dsum[a] : (void*)&rec.isum[a];
      else if (expr_fn(a) >= 0) s.xkey = &one[a].xkey;
      else if (fn == PB200_AGG_MIN) s.src = &rec.min_id[a];
      else if (fn == PB200_AGG_MAX) s.src = &rec.max_id_plus1[a];
      else if (fn == PB200_AGG_PERCENTILE) { s.src = &one[a].pct_id; s.pct_n = &one[plan.pct_rep[a]].pct_n; }
      else if (is_withtime_fn(fn)) { s.src = &one[a].wt_id; s.wt_time = &one[a].wt_time; }
      else if (is_moments_fn(fn)) {
        for (int j = 0; j < 3; j++) s.mom[j] = &rec.isum[d.mom_first[a] + j];
        s.mom_e = d.mom_e[a];
      } else if (is_distinct_value_fn(fn)) s.ds = one[d.ds_rep[a]].ds;
      else if (is_hll_fn(fn)) s.hll = &one[d.hll_rep[a]].hll;
      const DeviceColumn* c = d.agg_cols[a];
      s.dict = (c && vk != VAL_RAW_I32 && !c->dict_host.empty()) ? c->dict_host.data() : nullptr;   // unbiased
      s.counted = true;   // the matched docs (AggAccum::count)
    }
    return out;
  }

  // 8. PERCENTILE: histograms -> selected dictIds, queued behind the scan
  int finalize_percentiles() {
    for (int r = 0; r < plan.nres; r++) {
      const auto src = sources(r, static_cast<unsigned char*>(accum.p));
      for (int a = 0; a < plan.q.num_aggs; a++) {
        pb200_result::Pct& p = res[r]->pct;
        if (!p.hist[a]) continue;
        PercentileJob job;
        job.hist = p.hist[a];
        job.E = p.entries[a];
        job.rows = entries(r);
        job.n_out = src[a].pct_n;
        for (int b = 0; b < plan.q.num_aggs; b++) {
          if (plan.pct_rep[b] != a) continue;
          job.p[job.np] = plan.pct_p[b];
          job.ids[job.np++] = static_cast<uint32_t*>(src[b].src);
        }
        if (int rc = percentile_finalize(ctx, st, job, temps)) return rc;
      }
    }
    return PB200_OK;
  }

  // 8b. FIRST/LASTWITHTIME: the scan's winning keys -> data dictIds and time values, queued behind the scan
  int finalize_withtime() {
    if (!plan.any_wt) return PB200_OK;
    for (int a = 0; a < plan.q.num_aggs; a++) {
      if (plan.wt_time[a] < 0) continue;
      const WtSeg* wsegs = nullptr;
      if (int rc = withtime_segments(ctx, st, segments, nseg, query->aggs[a].column, plan.wt_time[a], plan.wt_base, temps, &wsegs)) return rc;
      for (int r = 0; r < plan.nres; r++) {
        const AggSource s = sources(r, static_cast<unsigned char*>(accum.p))[a];
        unsigned long long* key = plan.group_by ? res[r]->wt.key[a] : &acc.one(accum.p, r)[a].wt_key;
        const WithTimeJob job{key, entries(r), static_cast<uint32_t*>(s.src), s.wt_time};
        if (int rc = withtime_finalize(ctx, st, job, wsegs, nseg)) return rc;
      }
    }
    return PB200_OK;
  }

  // 8c. DISTINCTSUM / DISTINCTAVG states and DISTINCTCOUNTHLL estimates, aggregation only, queued behind the scan
  //     (group-by: the extraction finalizes them)
  int finalize_sets() {
    if (plan.group_by) return PB200_OK;
    for (int r = 0; r < plan.nres; r++) {
      const uint32_t* bits[kMaxAggs] = {};
      for (int b = 0; b < plan.num_user_aggs; b++) bits[b] = distinct_bufs[r][b] ? static_cast<const uint32_t*>(distinct_bufs[r][b]->p) : nullptr;
      if (int rc = pb200::finalize_sets(ctx, st, res[r]->dense, bits, plan.distinct_words[r].data(), 1, true,
                                        sources(r, static_cast<unsigned char*>(accum.p)).data(), temps))
        return rc;
    }
    return PB200_OK;
  }

  // 8d. expression aggregations: the mask scan and the expression pass (pb200_expr.cu), queued behind the scan
  int finalize_exprs() {
    if (!ex) return PB200_OK;
    std::vector<ExprOut> outs(plan.nres);
    for (int r = 0; r < plan.nres; r++) {
      const auto src = sources(r, static_cast<unsigned char*>(accum.p));
      for (int a = 0; a < plan.num_user_aggs; a++) {
        if (expr_fn(a) < 0) continue;
        outs[r].out[a] = src[a].xkey ? static_cast<void*>(src[a].xkey) : src[a].src;
        outs[r].hkeys = res[r]->dense.hkeys;
      }
    }
    return expr_launch(ctx, st, tune, query, segments, nseg, plan, *ex, outs, temps);
  }

  // 9. the count carriers' check queued behind the scan, the accumulator block read back, the wait for both, and the
  //    carriers' verdict: kRetryWithoutCountCarrier when a carried sum overflowed its field
  int read_back_and_verify() {
    if (plan.group_by)
      for (int r = 0; r < plan.nres; r++) {
        const pb200_result::Dense& d = res[r]->dense;
        if (d.pack_agg < 0) continue;
        const int vb = (int)std::max<long long>(1, std::min<long long>((d.groups + 1023) / 1024, (long long)ctx->sm_count * 4));
        carrier_verify_kernel<<<vb, 256, 0, st>>>((const unsigned long long*)d.isum[d.pack_agg], d.groups, d.pack_shift, acc.verify(accum.p) + 4 * r);
      }
    PB200_CUDA(cudaMemcpyAsync(back, accum.p, acc.bytes, cudaMemcpyDeviceToHost, st));
    t_queued = now_ms();
    const cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) { set_error("scan kernel failed: %s", cudaGetErrorString(se)); return PB200_E_CUDA; }
    t_synced = now_ms();
    for (int r = 0; r < plan.nres && plan.group_by; r++) {
      pb200_result::Dense& d = res[r]->dense;
      if (d.pack_agg < 0) continue;
      const unsigned long long* vw = acc.verify(back) + 4 * r;   // {sum of counts, largest sum field, largest count}
      const bool exact = vw[0] == AccumLayout::records(back)[r].count;
      if (d.reduce_world > 1) {
        // cross-GPU: the reduce adds `reduce_world` fields of each kind; neither can overflow if every rank's largest one
        // stays below its capacity / reduce_world.  A rank cannot rerun on its own (its peers' tables would have another
        // layout): it marks the result and the combine layer reruns the query on all ranks (PB200_Q_NO_COUNT_CARRIER).
        const unsigned long long w = (unsigned long long)d.reduce_world;
        const unsigned long long sum_lim = ((1ull << d.pack_shift) - 1ull) / w, cnt_lim = ((1ull << (64 - d.pack_shift)) - 1ull) / w;
        d.carrier_unsafe = !exact || vw[1] > sum_lim || vw[2] > cnt_lim;
        if (d.flag_slot) {   // the stream is idle (synchronised above): a blocking 8-byte copy, done before the call returns
          // (callers that bring their own collective read it from the block; pb200_result_combine rewrites the whole tail)
          const long long verdict = d.carrier_unsafe ? 1 : 0;
          PB200_CUDA(cudaMemcpy((long long*)d.i64_block + (d.i64_elems - 1), &verdict, 8, cudaMemcpyHostToDevice));
        }
        continue;
      }
      if (exact) continue;
      if (d.hctl) {  // a hash table that refused rows (numGroupsLimit) also loses counts: that is PB200_E_LIMIT, reported by the extraction
        uint32_t ctl[2] = {0, 0};
        PB200_CUDA(cudaMemcpy(ctl, d.hctl, 8, cudaMemcpyDeviceToHost));
        if (ctl[1]) continue;
      }
      return kRetryWithoutCountCarrier;
    }
    return PB200_OK;
  }

  // 11. every result's metadata and (aggregation only) its row, then the group-by rows extracted, or left for
  //     pb200_result_finalize (deferred); per-segment results release their tables
  int fill_results_and_extract(const pb200_order_by* order, const pb200_having* having, const pb200_post_aggs* post) {
    const int nuser = plan.num_user_aggs;
    const float ms = ev.ms();
    for (int r = 0; r < plan.nres; r++) {
      pb200_result& R = *res[r];
      const unsigned long long count = AccumLayout::records(back)[r].count;
      long long total_docs = 0;
      if (plan.merge) for (int s = 0; s < nseg; s++) total_docs += segments[s]->num_docs; else total_docs = segments[r]->num_docs;
      R.meta.num_group_by = plan.q.num_group_by;
      R.meta.num_aggs = nuser;
      R.agg_functions.resize(nuser);
      for (int a = 0; a < nuser; a++) R.agg_functions[a] = expr_fn(a) >= 0 ? expr_fn(a) : plan.q.aggs[a].function;
      for (int a = 0; a < nuser; a++)
        if (plan.mom_first[a] >= 0) { R.mom.on[a] = true; R.mom.grid[a] = segments[plan.merge ? 0 : r]->cols[query->aggs[a].column].moments->grid; }
      R.meta.num_docs_scanned = (int64_t)count;
      R.meta.num_entries_scanned_in_filter = plan.in_filter[r];
      R.meta.num_entries_scanned_post_filter = (int64_t)count * projected();
      R.meta.num_total_docs = total_docs;
      R.meta.device_ms = ms;
      R.dbl.resize(nuser); R.lng.resize(nuser); R.ids.resize(nuser); R.distinct.resize(nuser);
      if (plan.group_by) {
        R.meta.regime = regime_of(R.dense.cards, query->max_initial_result_holder_capacity);
        R.meta.reserved = (R.dense.pack_agg >= 0 ? 1 : 0) | (R.dense.carrier_unsafe ? 2 : 0) | (R.dense.flag_slot ? 4 : 0);  // include/pinot_b200.h
        if (order) R.order = *order;   // a deferred result keeps it for its extraction
        if (having) R.having = *having;
        if (post) R.post = *post;
        continue;
      }
      R.meta.num_groups = -1;
      R.meta.regime = PB200_REGIME_NONE;
      const AggAccum& rec = AccumLayout::records(back)[r];
      const auto src = sources(r, back);
      for (int a = 0; a < nuser; a++) {
        double dv;
        long long lv;
        int32_t id;
        agg_values(src[a], 0, count, dv, lv, id, R.mom.on[a] ? R.mom.one[a] : nullptr);
        R.dbl[a].push_back(dv); R.lng[a].push_back(lv); R.ids[a].push_back(id);
        const int fn = plan.q.aggs[a].function;   // an INT sum's exact value, for a cross-GPU combine
        if ((fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) && expr_fn(a) < 0 && !sum_in_double(src[a].vk)) { R.exact.on[a] = true; R.exact.sum[a] = rec.isum[a]; }
      }
      DevBufRaw* sets[kMaxAggs] = {};
      double* dbl[kMaxAggs] = {};
      int64_t* lng[kMaxAggs] = {};
      for (int a = 0; a < nuser; a++) { sets[a] = distinct_bufs[r][a].get(); dbl[a] = R.dbl[a].data(); lng[a] = R.lng[a].data(); }
      bool kept = false;   // the sets were complete at the read-back
      if (int rc = decode_sets(ctx, st, &R, sets, plan.distinct_words[r].data(), 1, dbl, lng, &kept)) return rc;
    }
    t_results = now_ms();
    if (!plan.group_by) return PB200_OK;
    if (plan.defer_finalize) {
      for (auto& R : res) { R->meta.num_groups = 0; R->dbl.assign(nuser, {}); R->lng.assign(nuser, {}); R->ids.assign(nuser, {}); R->distinct.assign(nuser, {}); }
      return PB200_OK;
    }
    std::vector<pb200_result*> rs;   // all results of the submission are extracted together (two device round trips in total)
    for (auto& R : res) rs.push_back(R.get());
    if (int rc = extract_groups(ctx, rs.data(), plan.nres, st)) return rc;
    if (!plan.merge)   // per-segment results do not need the dense state any more
      for (auto& R : res) release_tables(*R, true);
    return PB200_OK;
  }

  // columns read after the filter: the scan's group-by and aggregation columns, and every expression leaf and condition
  // column, each once
  int projected() const {
    if (!ex) return plan.projected;
    std::vector<int> cols = ex->cols;
    for (int c : ex->ccols)
      if (std::find(cols.begin(), cols.end(), c) == cols.end()) cols.push_back(c);
    for (int k = 0; k < plan.q.num_slots; k++)
      if ((plan.q.slot_roles[k] & (ROLE_GROUP | ROLE_AGG)) && std::find(cols.begin(), cols.end(), plan.slot_cols[k]) == cols.end())
        cols.push_back(plan.slot_cols[k]);
    return (int)cols.size();
  }

  // 12. the results handed out, and the phases of the call (pb200_last_phases)
  void hand_out(pb200_result** results) {
    for (int r = 0; r < plan.nres; r++) results[r] = res[r].release();
    const double t_exit = now_ms();
    g_phase_ms[PB200_PHASE_PLAN] = t_launch - t_enter;       // validation, plan, table allocation + memsets queued, descriptors
    g_phase_ms[PB200_PHASE_LAUNCH] = t_queued - t_launch;    // kernel launches queued
    g_phase_ms[PB200_PHASE_DEVICE_WAIT] = t_synced - t_queued;
    g_phase_ms[PB200_PHASE_RESULTS] = t_results - t_synced;  // carrier verdict, metadata, scalar results
    g_phase_ms[PB200_PHASE_EXTRACT] = t_exit - t_results;    // group extraction (device kernels + their sync) and table release
    g_phase_ms[PB200_PHASE_TOTAL] = t_exit - t_enter;
  }
};
}  // namespace

static int execute_impl(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments, int32_t nseg,
                        pb200_result** results, bool allow_count_carrier, const pb200_order_by* order, const double* agg_args,
                        const pb200_having* having, const pb200_agg_arg* wt_args, const ExprCall* ex,
                        const pb200_post_aggs* post) {
  ScanCall c{ctx, query, segments, nseg};
  c.ex = ex;
  if (int rc = c.check_call(results)) return rc;
  if (int rc = c.prepare_and_plan(allow_count_carrier, agg_args, wt_args)) return rc;
  if (int rc = c.alloc_results()) return rc;
  if (int rc = c.bind_accumulators()) return rc;
  if (int rc = c.plan.group_by ? c.bind_group_tables() : c.bind_agg_outputs()) return rc;
  if (int rc = c.launch()) return rc;
  if (int rc = c.finalize_percentiles()) return rc;
  if (int rc = c.finalize_withtime()) return rc;
  if (int rc = c.finalize_sets()) return rc;
  if (int rc = c.finalize_exprs()) return rc;
  if (int rc = c.read_back_and_verify()) return rc;   // kRetryWithoutCountCarrier: ~ScanCall frees this attempt's tables
  if (int rc = c.fill_results_and_extract(order, having, post)) return rc;
  c.hand_out(results);
  return PB200_OK;
}

extern "C" int32_t pb200_result_finalize(pb200_ctx* ctx, pb200_result* R) {
  if (!ctx || !R) { set_error("null argument"); return PB200_E_INVALID; }
  pb200_result::Dense& d = R->dense;
  if (!d.ctx || d.groups <= 0 || !d.live) { set_error("result has no dense device state"); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  StreamLease st(ctx);
  pb200_result* one[1] = {R};
  return extract_groups(ctx, one, 1, st);
}

extern "C" int32_t pb200_result_device_buffers(pb200_result* R, int32_t kind, void** p, int64_t* n) {
  if (!R || !p || !n) { set_error("null argument"); return PB200_E_INVALID; }
  pb200_result::Dense& d = R->dense;
  if (d.hkeys) { set_error("hash group tables of different GPUs are not element-wise reducible"); return PB200_E_UNSUPPORTED; }
  for (int a = 0; a < kMaxAggs; a++)
    if (R->mom.on[a]) { set_error("VAR/STDDEV moments are not combined across GPUs"); return PB200_E_UNSUPPORTED; }
  for (int a = 0; a < kMaxAggs; a++)
    if (R->wt.key[a]) { set_error("FIRST/LASTWITHTIME results are not combined across GPUs"); return PB200_E_UNSUPPORTED; }
  for (int a = 0; a < kMaxAggs; a++)
    if (d.expr_tab[a]) {   // not in the four reducible blocks: a reduce of those would keep only this rank's expression values
      set_error("group-by expression aggregations keep their tables outside the reducible blocks: they are not combined across GPUs");
      return PB200_E_UNSUPPORTED;
    }
  for (int a = 0; a < kMaxAggs; a++)
    if (R->pct.hist[a]) {
      set_error("PERCENTILE keeps dictId histograms on the device: a cross-GPU reduce of the tables would drop the other ranks' values");
      return PB200_E_UNSUPPORTED;
    }
  for (int a = 0; a < kMaxAggs; a++)
    if (d.dbits[a]) {  // per-group DISTINCTCOUNT bitsets are not one of the four reducible blocks: never reduce "around" them
      set_error("group-by DISTINCTCOUNT keeps per-group dictId bitsets on the device: a cross-GPU reduce of the tables would drop the other ranks' sets");
      return PB200_E_UNSUPPORTED;
    }
  switch (kind) {
    case 0: *p = d.i64_block; *n = d.i64_elems; break;
    case 1: *p = d.f64_block; *n = d.f64_elems; break;
    case 2: *p = d.u32max_block; *n = d.u32max_elems; break;
    case 3: *p = d.u32min_block; *n = d.u32min_elems; break;
    default: set_error("kind must be 0..3"); return PB200_E_INVALID;
  }
  return PB200_OK;
}

extern "C" int32_t pb200_result_meta_get(const pb200_result* R, pb200_result_meta* m) {
  if (!R || !m) { set_error("null argument"); return PB200_E_INVALID; }
  *m = R->meta;
  return PB200_OK;
}
extern "C" int32_t pb200_result_group_keys(const pb200_result* R, int32_t* out) {
  if (!R) { set_error("null argument"); return PB200_E_INVALID; }
  if (R->view.block) {
    const size_t n = R->view.rows * (size_t)R->meta.num_group_by;
    if (n && !out) { set_error("null argument"); return PB200_E_INVALID; }
    if (n) memcpy(out, R->view.keys, n * 4);
    return PB200_OK;
  }
  if (!out && !R->keys.empty()) { set_error("null argument"); return PB200_E_INVALID; }
  if (!R->keys.empty()) memcpy(out, R->keys.data(), R->keys.size() * 4);
  return PB200_OK;
}
namespace {
// one column of a view-backed result -> caller memory (absent columns: the neutral value)
void copy_dbl(const pb200_result::View& v, int a, double* out) { if (v.dbl[a]) memcpy(out, v.dbl[a], v.rows * 8); else std::fill(out, out + v.rows, 0.0); }
void copy_lng(const pb200_result::View& v, int a, int64_t* out) { if (v.lng[a]) memcpy(out, v.lng[a], v.rows * 8); else std::fill(out, out + v.rows, (int64_t)0); }
void copy_ids(const pb200_result::View& v, int a, int32_t* out) { if (v.ids[a]) memcpy(out, v.ids[a], v.rows * 4); else std::fill(out, out + v.rows, (int32_t)-1); }
}  // namespace
extern "C" int32_t pb200_result_agg(const pb200_result* R, int32_t a, double* od, int64_t* ol) {
  if (!R || a < 0 || a >= R->meta.num_aggs) { set_error("bad aggregation index"); return PB200_E_INVALID; }
  if (R->view.block) {
    if (od && R->view.rows) copy_dbl(R->view, a, od);
    if (ol && R->view.rows) copy_lng(R->view, a, ol);
    return PB200_OK;
  }
  if (a >= (int)R->dbl.size()) { set_error("bad aggregation index"); return PB200_E_INVALID; }
  if (od && !R->dbl[a].empty()) memcpy(od, R->dbl[a].data(), R->dbl[a].size() * 8);
  if (ol && !R->lng[a].empty()) memcpy(ol, R->lng[a].data(), R->lng[a].size() * 8);
  return PB200_OK;
}
extern "C" int32_t pb200_result_exact_sum(const pb200_result* R, int32_t a, int64_t* out) {
  if (!R || a < 0 || a >= R->meta.num_aggs || !out) { set_error("bad aggregation index"); return PB200_E_INVALID; }
  if (R->meta.num_groups >= 0 || a >= kMaxAggs || !R->exact.on[a]) return 0;
  *out = R->exact.sum[a];
  return 1;
}
extern "C" int32_t pb200_result_agg_dict_ids(const pb200_result* R, int32_t a, int32_t* out) {
  if (!R || a < 0 || a >= R->meta.num_aggs || !out) { set_error("bad aggregation index"); return PB200_E_INVALID; }
  if (R->view.block) { if (R->view.rows) copy_ids(R->view, a, out); return PB200_OK; }
  if (a >= (int)R->ids.size()) { set_error("bad aggregation index"); return PB200_E_INVALID; }
  if (!R->ids[a].empty()) memcpy(out, R->ids[a].data(), R->ids[a].size() * 4);
  return PB200_OK;
}
extern "C" int32_t pb200_result_fetch(const pb200_result* R, int32_t* keys, double* dbl, int64_t* lng, int32_t* ids) {
  if (!R) { set_error("null result"); return PB200_E_INVALID; }
  const size_t rows = R->meta.num_groups < 0 ? 1 : (size_t)R->meta.num_groups;
  if (R->view.block) {
    const pb200_result::View& v = R->view;
    if (keys && v.rows && R->meta.num_group_by) memcpy(keys, v.keys, v.rows * (size_t)R->meta.num_group_by * 4);
    for (int a = 0; a < R->meta.num_aggs && v.rows; a++) {
      if (dbl) copy_dbl(v, a, dbl + (size_t)a * rows);
      if (lng) copy_lng(v, a, lng + (size_t)a * rows);
      if (ids) copy_ids(v, a, ids + (size_t)a * rows);
    }
    return PB200_OK;
  }
  if (keys && !R->keys.empty()) memcpy(keys, R->keys.data(), R->keys.size() * 4);
  for (size_t a = 0; a < R->dbl.size(); a++) {
    if (dbl && R->dbl[a].size() == rows && rows) memcpy(dbl + a * rows, R->dbl[a].data(), rows * 8);
    if (lng && R->lng[a].size() == rows && rows) memcpy(lng + a * rows, R->lng[a].data(), rows * 8);
    if (ids && R->ids[a].size() == rows && rows) memcpy(ids + a * rows, R->ids[a].data(), rows * 4);
  }
  return PB200_OK;
}
extern "C" int32_t pb200_result_columns(const pb200_result* R, const int32_t** keys, const double** dbl, const int64_t** lng, const int32_t** ids) {
  if (!R) { set_error("null result"); return PB200_E_INVALID; }
  const size_t rows = R->meta.num_groups < 0 ? 1 : (size_t)R->meta.num_groups;
  const int nagg = R->meta.num_aggs;
  if (R->view.block) {
    const pb200_result::View& v = R->view;
    if (keys) *keys = v.rows && R->meta.num_group_by ? v.keys : nullptr;
    for (int a = 0; a < nagg; a++) {
      if (dbl) dbl[a] = v.rows ? v.dbl[a] : nullptr;
      if (lng) lng[a] = v.rows ? v.lng[a] : nullptr;
      if (ids) ids[a] = v.rows ? v.ids[a] : nullptr;
    }
    return PB200_OK;
  }
  if (keys) *keys = R->keys.empty() ? nullptr : R->keys.data();
  for (int a = 0; a < nagg; a++) {
    if (dbl) dbl[a] = (a < (int)R->dbl.size() && R->dbl[a].size() == rows && rows) ? R->dbl[a].data() : nullptr;
    if (lng) lng[a] = (a < (int)R->lng.size() && R->lng[a].size() == rows && rows) ? R->lng[a].data() : nullptr;
    if (ids) ids[a] = (a < (int)R->ids.size() && R->ids[a].size() == rows && rows) ? R->ids[a].data() : nullptr;
  }
  return PB200_OK;
}
extern "C" int64_t pb200_result_distinct(const pb200_result* R, int32_t a, int32_t row, int32_t* out, int64_t cap) {
  // a DISTINCTCOUNTHLL's kept set is decoded here, once: the result is logically unchanged
  const std::vector<std::vector<int32_t>>* sets = R ? result_sets(const_cast<pb200_result*>(R), a) : nullptr;
  if (!sets || row < 0 || row >= (int)sets->size()) { set_error("bad distinct index"); return PB200_E_INVALID; }
  const auto& v = (*sets)[row];
  for (int64_t i = 0; i < (int64_t)v.size() && i < cap; i++) out[i] = v[i];
  return (int64_t)v.size();
}
extern "C" int32_t pb200_result_free(pb200_result* R) {
  if (!R) return PB200_OK;
  release_tables(*R, false);
  delete R;
  return PB200_OK;
}
