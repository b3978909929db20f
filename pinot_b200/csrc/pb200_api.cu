// pb200_api.cu -- C-ABI implementation: context, segment residency, query planning and launch, result extraction.
//
// Host logic here is the device-facing half of what the reference does between PlanNode.run() and nextBlock():
// choosing what to stream (ProjectPlanNode's column set, core/plan/ProjectPlanNode.java), laying out the group-key
// space (DictionaryBasedGroupKeyGenerator.java:105-186) and extracting results (GroupByOperator.java:116-140,
// AggregationFunction.extractAggregationResult).
#include <cuda_runtime.h>
#include <chrono>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <limits>
#include <memory>

#include "pb200_internal.h"
#include "pb200_scan_launch.h"
#include "pb200_unpack.cuh"

namespace pb200 {

static thread_local char g_error[1024] = "";
// Host wall-clock of the calling thread's last pb200_execute, by phase (pb200_last_phases): a few steady_clock reads per query.
static thread_local double g_phase_ms[PB200_NUM_PHASES] = {};
static inline double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

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

struct DevBuf {  // RAII pooled device buffer
  pb200_ctx* ctx = nullptr;
  void* p = nullptr;
  DevBuf() {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { dev_free(ctx, p); }
  int alloc(pb200_ctx* c, size_t bytes) { ctx = c; return dev_alloc(c, bytes, &p); }
  void* release() { void* r = p; p = nullptr; return r; }
};

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

static uint64_t padded_fwd_bytes(long long num_docs, int bits) {
  // whole tiles for ANY tile size <= kMaxTileRows: ceil(N/t)*t < N + t <= alloc rows
  long long tiles = (num_docs + kMaxTileRows - 1) / kMaxTileRows + 1;
  return (uint64_t)tiles * kMaxTileRows / 8 * bits + 64;
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

// words a device doc mask needs: whole tiles + one spare tile (the kernel reads masks tile-wise) + a tail
static size_t doc_mask_words(long long num_docs) { return (((size_t)num_docs + kMaxTileRows - 1) / kMaxTileRows + 1) * (kMaxTileRows / 32) + 8; }

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
  seg->cols.resize(ncols);
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
  if (!seg || col < 0 || col >= (int)seg->cols.size()) { set_error("bad column"); return PB200_E_INVALID; }
  const DeviceColumn& c = seg->cols[col];
  out[0] = c.fwd_kind; out[1] = c.stored_type; out[2] = c.bits; out[3] = c.cardinality; out[4] = c.inv != nullptr;
  out[5] = (int64_t)c.fwd_file_bytes;
  return PB200_OK;
}

extern "C" int64_t pb200_segment_read_index(pb200_ctx* ctx, const pb200_segment* seg, int32_t col, int32_t which,
                                            void* out, uint64_t cap) {
  if (!seg || col < 0 || col >= (int)seg->cols.size()) { set_error("bad column"); return PB200_E_INVALID; }
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
// query planning
// ------------------------------------------------------------------------------------------------------------------
namespace {

struct Plan {
  QueryDesc q{};
  std::vector<SegDesc> segs;
  std::vector<int> slot_cols;                 // slot -> column id
  std::vector<int> leaf_node;                 // leaf -> index in the postfix node list
  bool group_by = false;
  int cw = 8;
  size_t smem_bytes = 0;
  std::vector<std::unique_ptr<DevBuf>> temps; // LUTs, doc masks, range lists (freed after the launch)
};

int slot_of(Plan& p, int col, uint32_t role) {
  for (size_t s = 0; s < p.slot_cols.size(); s++)
    if (p.slot_cols[s] == col) { p.q.slot_roles[s] |= role; return (int)s; }
  if ((int)p.slot_cols.size() >= kMaxSlots) return -1;
  p.slot_cols.push_back(col);
  p.q.slot_roles[p.slot_cols.size() - 1] = role;
  return (int)p.slot_cols.size() - 1;
}

bool is_scan_leaf(int op) { return op == PB200_F_SCAN_RANGE || op == PB200_F_SCAN_IN || op == PB200_F_SCAN_NOT_IN || op == PB200_F_RAW_RANGE; }
bool is_leaf(int op) { return op >= PB200_F_MATCH_ALL; }

int regime_of(const std::vector<int>& cards, int array_threshold) {
  // DictionaryBasedGroupKeyGenerator.java:128-185
  long long product = 1;
  bool overflow = false;
  for (int c : cards) {
    if (!overflow) {
      if (c > 0 && product > std::numeric_limits<long long>::max() / c) overflow = true; else product *= c;
    }
  }
  if (overflow) return PB200_REGIME_ARRAY_MAP;
  if (product > std::numeric_limits<int>::max()) return PB200_REGIME_LONG_MAP;
  return product > array_threshold ? PB200_REGIME_INT_MAP : PB200_REGIME_ARRAY;
}

// one-sided ranges: every stored dictId is < cardinality, so "hi covers the dictionary" needs no upper compare
void set_cmp(LeafDesc& lf, const DeviceColumn& c) {
  const unsigned long long hi = (unsigned long long)lf.lo + lf.span;
  if (lf.span == 0) { lf.kind = LEAF_NONE; return; }
  if (hi >= (unsigned long long)c.cardinality || hi >= (1ull << c.bits)) lf.cmp = CMP_GE;
  else if (lf.lo == 0) lf.cmp = CMP_LT;
  else lf.cmp = CMP_BOTH;
}

}  // namespace

namespace pb200 {
cudaError_t launch_scan_variant(const ScanVariant& v, size_t smem_bytes, int grid, const QueryDesc& q, const TmaTable& tt,
                                const SegDesc* dsegs, cudaStream_t st) {
  if (v.group_by) {
    if (v.min_blocks >= 2) return v.warps == 8 ? launch_scan_w8_gb2(smem_bytes, grid, q, tt, dsegs, st) : launch_scan_w6_gb2(smem_bytes, grid, q, tt, dsegs, st);
    return v.warps == 8 ? launch_scan_w8_gb1(smem_bytes, grid, q, tt, dsegs, st) : launch_scan_w6_gb1(smem_bytes, grid, q, tt, dsegs, st);
  }
  if (v.warps == 8) return v.defer ? launch_scan_w8_agg(smem_bytes, grid, q, tt, dsegs, st) : launch_scan_w8_agg_nodefer(smem_bytes, grid, q, tt, dsegs, st);
  return launch_scan_w6_agg(smem_bytes, grid, q, tt, dsegs, st);
}
}  // namespace pb200


// Internal return code of execute_impl: a count-carrying sum overflowed its field (detected exactly, see the verification
// after the launch) -- the caller runs the submission again with separate COUNT reductions.
constexpr int kRetryWithoutCountCarrier = 1;
static int execute_impl(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments, int32_t nseg,
                        pb200_result** results, bool allow_count_carrier);

extern "C" int32_t pb200_execute(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments,
                                 int32_t nseg, pb200_result** results) {
  int rc = execute_impl(ctx, query, segments, nseg, results, true);
  if (rc == kRetryWithoutCountCarrier) rc = execute_impl(ctx, query, segments, nseg, results, false);
  return rc;
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

static int execute_impl(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments, int32_t nseg,
                        pb200_result** results, bool allow_count_carrier) {
  if (!ctx || !query || !segments || !results || nseg <= 0) { set_error("invalid argument to pb200_execute"); return PB200_E_INVALID; }
  const double t_enter = now_ms();
  PB200_CUDA(cudaSetDevice(ctx->device));
  const bool per_seg_filter = query->flags & PB200_Q_PER_SEGMENT_FILTER;
  const bool merge = query->flags & PB200_Q_MERGE_SEGMENTS;
  const int nnodes = query->num_filter_nodes, nagg = query->num_aggs, ngb = query->num_group_by;
  if (nagg < 0 || nagg > kMaxAggs || ngb < 0 || ngb > kMaxGroupBy || nnodes < 0 || nnodes > kMaxNodes) {
    set_error("query exceeds device limits (aggs %d/%d, group-by %d/%d, filter nodes %d/%d)", nagg, kMaxAggs, ngb, kMaxGroupBy, nnodes, kMaxNodes);
    return PB200_E_UNSUPPORTED;
  }
  if (nagg == 0) { set_error("at least one aggregation is required on this path"); return PB200_E_INVALID; }
  const int ncols = (int)segments[0]->cols.size();
  for (int s = 0; s < nseg; s++) {
    if (!segments[s] || segments[s]->ctx != ctx || (int)segments[s]->cols.size() != ncols) { set_error("segment %d does not belong to this context / schema", s); return PB200_E_INVALID; }
  }

  if (merge && nseg > 1) {
    // One result for all segments == a merge of dictId-indexed state (group tables, MIN / MAX ids, DISTINCTCOUNT bitsets).
    // That is only a merge BY VALUE (GroupByCombineOperator.java:130-146, AggregationFunction.merge) when the column has
    // the same dictionary everywhere: compare content hashes, not cardinalities.  Bound segments (pb200_domain_*) pass by
    // construction; anything else is refused so that the caller combines per-segment results itself.
    auto same_dictionary = [&](int col, const char* what) -> bool {
      const DeviceColumn& c0 = segments[0]->cols[col];
      for (int s = 1; s < nseg; s++) {
        const DeviceColumn& c = segments[s]->cols[col];
        if (c.dict_hash != c0.dict_hash || c.cardinality != c0.cardinality || c.stored_type != c0.stored_type) {
          set_error("PB200_Q_MERGE_SEGMENTS: %s column %d has a different dictionary in segment %d than in segment 0 "
                    "(bind the segments to a pb200_domain first)", what, col, s);
          return false;
        }
      }
      return true;
    };
    for (int g = 0; g < ngb; g++) {
      const int c = query->group_by_columns[g];
      if (c >= 0 && c < ncols && !same_dictionary(c, "group-by")) return PB200_E_UNSUPPORTED;
    }
    for (int a = 0; a < nagg; a++) {
      const pb200_agg& ag = query->aggs[a];
      if (ag.function != PB200_AGG_MIN && ag.function != PB200_AGG_MAX && ag.function != PB200_AGG_DISTINCTCOUNT) continue;
      if (ag.column < 0 || ag.column >= ncols) continue;
      if (segments[0]->cols[ag.column].bits == 32 && !segments[0]->cols[ag.column].dict_native) continue;  // raw values, no ids
      if (!same_dictionary(ag.column, ag.function == PB200_AGG_DISTINCTCOUNT ? "DISTINCTCOUNT" : "MIN/MAX")) return PB200_E_UNSUPPORTED;
    }
  }

  Plan plan;
  QueryDesc& q = plan.q;
  plan.group_by = ngb > 0;
  q.num_segments = nseg;
  q.num_aggs = nagg;
  q.num_group_by = ngb;

  // ---- slots: filter scan columns, then group-by keys, then aggregation arguments ----
  const pb200_filter_node* f0 = query->filter;
  for (int s = 0; s < (per_seg_filter ? nseg : 1); s++) {
    for (int i = 0; i < nnodes; i++) {
      const pb200_filter_node& n = f0[(size_t)s * nnodes + i];
      if (is_leaf(n.op) != is_leaf(f0[i].op) || (!is_leaf(n.op) && (n.op != f0[i].op || n.num_children != f0[i].num_children))) {
        set_error("per-segment filter trees must share their shape"); return PB200_E_INVALID;
      }
      if (is_scan_leaf(n.op)) {
        if (n.column < 0 || n.column >= ncols) { set_error("filter column %d out of range", n.column); return PB200_E_INVALID; }
        if (slot_of(plan, n.column, ROLE_FILTER) < 0) { set_error("too many distinct columns (max %d)", kMaxSlots); return PB200_E_UNSUPPORTED; }
      }
    }
  }
  for (int g = 0; g < ngb; g++) {
    int c = query->group_by_columns[g];
    if (c < 0 || c >= ncols) { set_error("group-by column %d out of range", c); return PB200_E_INVALID; }
    for (int t = 0; t < nseg; t++) {
      const DeviceColumn& gc = segments[t]->cols[c];
      if (gc.bits > 31 || gc.cardinality <= 0 || gc.fwd_kind != PB200_FWD_DICT_FIXEDBIT) {
        set_error("group-by column %d is not dictionary-encoded in segment %d: not accelerated", c, t);
        return PB200_E_UNSUPPORTED;
      }
    }
    int s = slot_of(plan, c, ROLE_GROUP);
    if (s < 0) { set_error("too many distinct columns (max %d)", kMaxSlots); return PB200_E_UNSUPPORTED; }
    q.group_slot[g] = s;
  }
  for (int a = 0; a < nagg; a++) {
    const pb200_agg& ag = query->aggs[a];
    q.aggs[a].function = ag.function;
    q.aggs[a].slot = -1;
    q.aggs[a].val_kind = VAL_NONE;
    if (ag.function == PB200_AGG_COUNT) continue;
    if (ag.function < 0 || ag.function > PB200_AGG_DISTINCTCOUNT) { set_error("unknown aggregation function %d", ag.function); return PB200_E_INVALID; }
    if (ag.column < 0 || ag.column >= ncols) { set_error("aggregation column %d out of range", ag.column); return PB200_E_INVALID; }
    int s = slot_of(plan, ag.column, ROLE_AGG);
    if (s < 0) { set_error("too many distinct columns (max %d)", kMaxSlots); return PB200_E_UNSUPPORTED; }
    q.aggs[a].slot = s;
    const DeviceColumn& c0 = segments[0]->cols[ag.column];
    int vk = VAL_NONE;
    if (c0.bits == 32 && c0.dict_native == nullptr) {
      if (c0.stored_type != PB200_INT) { set_error("raw column type %d not accelerated", c0.stored_type); return PB200_E_UNSUPPORTED; }
      vk = VAL_RAW_I32;
      if (ag.function == PB200_AGG_DISTINCTCOUNT) { set_error("DISTINCTCOUNT on raw column not accelerated"); return PB200_E_UNSUPPORTED; }
    } else {
      switch (c0.stored_type) {
        case PB200_INT: vk = VAL_DICT_I32; break;
        case PB200_LONG: vk = VAL_DICT_I64; break;
        case PB200_FLOAT: vk = VAL_DICT_F32; break;
        case PB200_DOUBLE: vk = VAL_DICT_F64; break;
        default:  // STRING: only functions that work on dictIds (MIN/MAX come back as dictIds, DISTINCTCOUNT as a set)
          if (ag.function == PB200_AGG_SUM || ag.function == PB200_AGG_AVG) { set_error("SUM/AVG over STRING column"); return PB200_E_UNSUPPORTED; }
          vk = VAL_DICT_I32;
      }
    }
    q.aggs[a].val_kind = vk;
  }
  q.num_slots = (int)plan.slot_cols.size();

  // ---- filter program (shape shared by all segments) ----
  int nleaves = 0;
  for (int i = 0; i < nnodes; i++) {
    const pb200_filter_node& n = f0[i];
    if (is_leaf(n.op)) {
      if (nleaves >= kMaxLeaves) { set_error("too many filter leaves (max %d)", kMaxLeaves); return PB200_E_UNSUPPORTED; }
      q.prog_op[i] = OP_LEAF;
      q.prog_arg[i] = (uint8_t)nleaves++;
      plan.leaf_node.push_back(i);
    } else if (n.op == PB200_F_NOT) {
      q.prog_op[i] = OP_NOT; q.prog_arg[i] = 1;
    } else if (n.op == PB200_F_AND || n.op == PB200_F_OR) {
      if (n.num_children < 1 || n.num_children > kMaxStack) { set_error("AND/OR with %d operands not supported", n.num_children); return PB200_E_UNSUPPORTED; }
      q.prog_op[i] = n.op == PB200_F_AND ? OP_AND : OP_OR;
      q.prog_arg[i] = (uint8_t)n.num_children;
    } else {
      set_error("unknown filter op %d", n.op);
      return PB200_E_INVALID;
    }
  }
  q.num_nodes = nnodes;
  q.num_leaves = nleaves;
  q.conj = nnodes == 0 || (nnodes == 1 && nleaves == 1) ||
           (nnodes == nleaves + 1 && f0[nnodes - 1].op == PB200_F_AND && f0[nnodes - 1].num_children == nleaves);
  {  // validate stack discipline once
    int sp = 0, maxsp = 0;
    for (int i = 0; i < nnodes; i++) {
      if (q.prog_op[i] == OP_LEAF) sp++;
      else if (q.prog_op[i] == OP_NOT) { if (sp < 1) sp = -99; }
      else { sp -= q.prog_arg[i] - 1; }
      if (sp < 1) { set_error("malformed postfix filter"); return PB200_E_INVALID; }
      maxsp = std::max(maxsp, sp);
    }
    if (nnodes > 0 && sp != 1) { set_error("malformed postfix filter (stack %d at end)", sp); return PB200_E_INVALID; }
    if (maxsp > kMaxStack) { set_error("filter too deep"); return PB200_E_UNSUPPORTED; }
  }

  // ---- tile geometry ----
  int max_bits_sum = 0;
  for (int s = 0; s < nseg; s++) {
    int sum = 0;
    for (int c : plan.slot_cols) sum += segments[s]->cols[c].bits;
    max_bits_sum = std::max(max_bits_sum, sum);
  }
  const size_t hdr_bytes = (sizeof(SmemHeader) + 127) / 128 * 128;
  // CTA tile = W warps x 1024 rows; every warp streams its own 1024-row slices through a private TMA ring.
  // W = 6 (aggregation only): 192-thread CTAs, two per SM, 168 registers, no spills (32 of them hold the software-pipelined
  // dictionary gathers).  Group-by: the survivor-queue path needs ~120 registers; W = 6 with two CTAs per SM leaves room
  // for a 3-deep ring (faster than W = 8 on C3/range); falls back to one CTA when the rows are too wide
  // for two 2-deep rings.
  const Tuning tune = [&]() { std::lock_guard<std::mutex> g(ctx->mu); return ctx->tune; }();
  int cw = tune.warps, stages = 0, ctas_per_sm = 1;
  q.sparse_max = tune.sparse_max;
  q.sparse_max_agg = tune.sparse_max_agg >= 0 ? tune.sparse_max_agg : (plan.group_by ? std::min(q.sparse_max, 2) : q.sparse_max);
  ctas_per_sm = tune.ctas_per_sm;  // default 2: the group-by kernel needs < 168 registers, two 192-thread CTAs per SM
  const size_t warp_stage_bytes = (size_t)128 * max_bits_sum;
  size_t extra_bytes = (q.conj ? 0 : (size_t)cw * 32 * kMaxStack * 4) + (plan.group_by ? (size_t)cw * 2048 : (size_t)nagg * cw * 32 * 16);
  q.queue_max = plan.group_by ? 1024 : 0;  // every group-by slice goes through the survivor queue
  // CTA-private group tables in shared memory when the key space is small and every function is COUNT or an integer SUM
  q.smem_groups = 0;
  for (int a = 0; a < kMaxAggs; a++) q.smem_slot[a] = -1;
  if (plan.group_by && tune.smem_groups) {
    // Small key spaces only: there the global table's few addresses serialise in L2, while for thousands of groups the
    // fire-and-forget global REDs beat shared atomics that must return the old low word.
    const long long smem_groups_max = tune.smem_groups_max;
    long long gmax = 1;
    for (int s = 0; s < nseg && gmax > 0; s++) {
      long long g = 1;
      for (int k = 0; k < ngb; k++) { g *= std::max(segments[s]->cols[query->group_by_columns[k]].cardinality, 1); if (g > smem_groups_max) { g = -1; break; } }
      gmax = g < 0 ? -1 : std::max(gmax, g);
    }
    bool ok = gmax > 0;
    if (ok && gmax > tune.dense_max) ok = false;  // hashed: slots, not raw keys
    int nsum = 0;
    for (int a = 0; a < nagg && ok; a++) {
      const int fn = q.aggs[a].function, vk = q.aggs[a].val_kind;
      if (fn == PB200_AGG_COUNT) continue;
      if ((fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) && (vk == VAL_DICT_I32 || vk == VAL_RAW_I32)) q.smem_slot[a] = (int8_t)nsum++;
      else ok = false;
    }
    const long long gstride = gmax | 1;
    const size_t copy_bytes = ok ? (size_t)gstride * 4 * (1 + 2 * nsum) : 0;
    // room left after a 2-deep ring; the table may take at most 64 KB of it
    const long long room = (long long)ctx->max_smem_optin / ctas_per_sm - (long long)hdr_bytes - (long long)extra_bytes - 1024 - 256 - (long long)(2 * warp_stage_bytes * cw);
    if (ok && room >= (long long)copy_bytes) {
      int copies = 1;
      while (copies < 32 && (long long)copy_bytes * copies * 2 <= std::min<long long>(room, 64 << 10)) copies *= 2;
      if (tune.smem_copies > 0) copies = std::max(1, std::min(copies, tune.smem_copies));
      q.smem_groups = (int32_t)gmax;
      q.smem_copies = copies;
      q.smem_gstride = (int32_t)gstride;
      extra_bytes += copy_bytes * copies;
    } else {
      for (int a = 0; a < kMaxAggs; a++) q.smem_slot[a] = -1;
    }
  }
  {
    long long budget = (long long)ctx->max_smem_optin / ctas_per_sm - (long long)hdr_bytes - (long long)extra_bytes - 1024 - 256;
    stages = warp_stage_bytes == 0 ? 2 : (budget <= 0 ? 0 : (int)std::min<long long>(kMaxStages, budget / (long long)(warp_stage_bytes * cw)));
    if (stages < 2 && ctas_per_sm > 1) {  // wide rows: fall back to one CTA per SM
      ctas_per_sm = 1;
      budget = (long long)ctx->max_smem_optin - (long long)hdr_bytes - (long long)extra_bytes - 1024 - 256;
      stages = budget <= 0 ? 0 : (int)std::min<long long>(kMaxStages, budget / (long long)(warp_stage_bytes * cw));
    }
  }
  if (stages < 2) { set_error("touched columns too wide for the shared-memory pipeline (%d bits per row)", max_bits_sum); return PB200_E_UNSUPPORTED; }
  if (tune.stages > 0) stages = std::max(2, std::min(stages, tune.stages));
  plan.cw = cw;
  q.tile_rows = cw * 1024;
  q.num_stages = stages;
  q.stage_words = (uint32_t)(32 * max_bits_sum);
  q.use_pipe = q.num_slots > 0;
  q.defer_agg = -1;
  if (!plan.group_by && tune.defer)
    for (int a = 0; a < nagg; a++)
      if ((q.aggs[a].function == PB200_AGG_SUM || q.aggs[a].function == PB200_AGG_AVG) && q.aggs[a].val_kind == VAL_DICT_I32) { q.defer_agg = a; break; }
  plan.smem_bytes = hdr_bytes + (size_t)cw * stages * q.stage_words * 4 + extra_bytes;
  // the group table sits behind the rings and the generic-filter stack
  q.queue_off = (uint32_t)(hdr_bytes + (size_t)cw * stages * q.stage_words * 4 + (q.conj ? 0 : (size_t)cw * 32 * kMaxStack * 4));
  q.smem_table_off = q.queue_off + (plan.group_by ? (uint32_t)cw * 2048u : 0u);

  cudaStream_t st = take_stream(ctx);
  struct StreamReturn { pb200_ctx* c; cudaStream_t s; ~StreamReturn() { give_stream(c, s); } } stream_return{ctx, st};

  // ---- group table geometry / result buffers ----
  std::vector<std::unique_ptr<pb200_result>> res;
  const int nres = merge ? 1 : nseg;
  for (int r = 0; r < nres; r++) res.emplace_back(new pb200_result());
  struct ResultCleanup {  // frees dense device state if we fail midway
    std::vector<std::unique_ptr<pb200_result>>* r;
    bool armed = true;
    ~ResultCleanup() { if (armed) for (auto& x : *r) if (x) pb200_result_free(x.release()); }
  } cleanup{&res};

  DevBuf accum_buf;  // nres AggAccum records, initialised and read back with ONE copy each
  std::vector<std::vector<std::unique_ptr<DevBuf>>> distinct_bufs(nres);
  plan.segs.resize(nseg);
  long long tile_cursor = 0;
  for (int s = 0; s < nseg; s++) {
    const pb200_segment* seg = segments[s];
    SegDesc& sd = plan.segs[s];
    memset(&sd, 0, sizeof sd);
    sd.num_docs = seg->num_docs;
    sd.first_tile = tile_cursor;
    sd.num_tiles = (seg->num_docs + q.tile_rows - 1) / q.tile_rows;
    tile_cursor += sd.num_tiles;
    uint32_t word_off = 0, tx = 0;
    for (int k = 0; k < q.num_slots; k++) {
      const DeviceColumn& c = seg->cols[plan.slot_cols[k]];
      sd.slots[k].data = c.fwd;
      sd.slots[k].bits = c.bits;
      sd.slots[k].stage_words = word_off;
      sd.slots[k].tile_bytes = (uint32_t)(128 * c.bits);  // one warp slice = 1024 rows
      word_off += sd.slots[k].tile_bytes / 4;
      tx += sd.slots[k].tile_bytes;
    }
    sd.stage_tx = tx;
  }
  q.total_tiles = (int32_t)std::min<long long>(tile_cursor, 0x7FFFFFFF);

  // ---- per segment leaves ----
  std::vector<DecodeJob> decode_jobs;  // every posting list the query needs, decoded by ONE launch
  for (int s = 0; s < nseg; s++) {
    const pb200_segment* seg = segments[s];
    SegDesc& sd = plan.segs[s];
    const pb200_filter_node* fs = per_seg_filter ? query->filter + (size_t)s * nnodes : query->filter;
    for (int l = 0; l < nleaves; l++) {
      const pb200_filter_node& n = fs[plan.leaf_node[l]];
      const pb200_filter_node& n0 = f0[plan.leaf_node[l]];
      LeafDesc& lf = sd.leaves[l];
      lf.slot = -1;
      if (n.op == PB200_F_MATCH_ALL) { lf.kind = LEAF_ALL; continue; }
      if (n.op == PB200_F_EMPTY) { lf.kind = LEAF_NONE; continue; }
      (void)n0;
      const bool needs_col = n.op != PB200_F_DOC_MASK && n.op != PB200_F_DOC_RANGES;
      if (needs_col && (n.column < 0 || n.column >= ncols)) { set_error("filter column out of range"); return PB200_E_INVALID; }
      const DeviceColumn& c = seg->cols[needs_col ? n.column : 0];
      if (is_scan_leaf(n.op)) {
        int slot = -1;
        for (int k = 0; k < q.num_slots; k++) if (plan.slot_cols[k] == n.column) slot = k;
        if (slot < 0) { set_error("scan leaf column %d has no slot (per-segment trees must scan the same columns)", n.column); return PB200_E_INVALID; }
        lf.slot = slot;
        if (n.op == PB200_F_RAW_RANGE) {
          // Raw (no-dictionary) INT column, value-space range: IntRawValueBasedRangePredicateEvaluator
          // (core/operator/filter/predicate/RangePredicateEvaluatorFactory.java:227-262).  On two's complement words
          // lo <= x <= hi  <=>  (uint32)(x - lo) < (uint32)(hi - lo + 1): the dictId range compare of the kernel, unchanged.
          if (c.bits != 32 || c.dict_native || c.stored_type != PB200_INT) { set_error("RAW_RANGE is accelerated for raw INT columns only (column %d)", n.column); return PB200_E_UNSUPPORTED; }
          double dlo = (n.raw_flags & 1) ? -2147483648.0 : std::ceil(n.raw_lo), dhi = (n.raw_flags & 2) ? 2147483647.0 : std::floor(n.raw_hi);
          if (!(n.raw_flags & 1) && (n.raw_flags & 4) && dlo == n.raw_lo) dlo += 1.0;   // exclusive bounds on integral literals
          if (!(n.raw_flags & 2) && (n.raw_flags & 8) && dhi == n.raw_hi) dhi -= 1.0;
          dlo = std::max(dlo, -2147483648.0); dhi = std::min(dhi, 2147483647.0);
          if (!(dlo <= dhi)) { lf.kind = LEAF_NONE; lf.slot = -1; continue; }   // also catches NaN bounds
          const long long lo = (long long)dlo, hi = (long long)dhi;
          if (hi - lo + 1 >= (1ll << 32)) { lf.kind = LEAF_ALL; lf.slot = -1; continue; }
          lf.kind = LEAF_RANGE;
          lf.lo = (uint32_t)(int32_t)lo; lf.span = (uint32_t)(hi - lo + 1);
          lf.cmp = CMP_BOTH;   // one-sided shortcuts assume unsigned order
        } else if (n.op == PB200_F_SCAN_RANGE) {
          lf.kind = LEAF_RANGE;
          int lo = std::max(n.lo, 0), hi = std::max(n.hi, lo);
          lf.lo = (uint32_t)lo; lf.span = (uint32_t)(hi - lo);
          set_cmp(lf, c);
        } else {
          lf.negate = n.op == PB200_F_SCAN_NOT_IN;
          if (n.num_ids == 1) {
            lf.kind = LEAF_RANGE; lf.lo = (uint32_t)n.ids[0]; lf.span = 1;
            set_cmp(lf, c);
          } else if (n.num_ids == 0) {
            lf.kind = LEAF_NONE;
          } else {
            // dictId set -> bitmap over the dictionary (what PredicateEvaluator.getMatchingDictIds feeds the scan)
            size_t words = ((size_t)std::max(c.cardinality, 1) + 31) / 32 + 1;
            if (c.bits == 32) { set_error("IN on raw column not accelerated"); return PB200_E_UNSUPPORTED; }
            words = std::max(words, ((size_t)1 << c.bits) / 32 + 1);  // every representable dictId is addressable
            std::vector<uint32_t> lut(words, 0);
            for (int k = 0; k < n.num_ids; k++) {
              int id = n.ids[k];
              if (id < 0 || id >= c.cardinality) { set_error("dictId %d out of range", id); return PB200_E_INVALID; }
              lut[id >> 5] |= 1u << (id & 31);
            }
            plan.temps.emplace_back(new DevBuf());
            int rc = plan.temps.back()->alloc(ctx, words * 4);
            if (rc) return rc;
            PB200_CUDA(cudaMemcpyAsync(plan.temps.back()->p, lut.data(), words * 4, cudaMemcpyHostToDevice, st));
            PB200_CUDA(cudaStreamSynchronize(st));  // lut is a local
            lf.kind = LEAF_LUT;
            lf.bits = (const uint32_t*)plan.temps.back()->p;
          }
        }
      } else if (n.op == PB200_F_INV_IN || n.op == PB200_F_INV_NOT_IN) {
        if (!c.inv) { set_error("column %d has no inverted index", n.column); return PB200_E_INVALID; }
        size_t words = (((size_t)seg->num_docs + kMaxTileRows - 1) / kMaxTileRows + 1) * (kMaxTileRows / 32) + 8;  // whole tiles
        plan.temps.emplace_back(new DevBuf());
        int rc = plan.temps.back()->alloc(ctx, words * 4);
        if (rc) return rc;
        uint32_t* mask = (uint32_t*)plan.temps.back()->p;
        PB200_CUDA(cudaMemsetAsync(mask, 0, words * 4, st));
        for (int k = 0; k < n.num_ids; k++) {  // InvertedIndexFilterOperator: OR of the bitmaps of the dictIds
          const int id = n.ids[k];
          if (id < 0 || id >= c.cardinality) { set_error("dictId %d out of range for inverted index (card %d)", id, c.cardinality); return PB200_E_INVALID; }
          if (c.inv_offsets[id + 1] == c.inv_offsets[id]) continue;  // bound column: this domain id does not occur in the segment
          decode_jobs.push_back(DecodeJob{c.inv, c.inv_offsets[id], (unsigned long long)c.inv_offsets[id + 1] - c.inv_offsets[id], mask, seg->num_docs});
        }
        lf.kind = LEAF_DOCMASK;
        lf.bits = mask;
        lf.negate = n.op == PB200_F_INV_NOT_IN;
      } else if (n.op == PB200_F_DOC_MASK) {
        const size_t need = ((size_t)seg->num_docs + 31) / 32;
        if ((size_t)n.num_ids < need || !n.ids) { set_error("DOC_MASK needs %zu words, got %d", need, n.num_ids); return PB200_E_INVALID; }
        uint32_t* mask;
        if (n.reserved & PB200_NODE_IDS_ON_DEVICE) {
          mask = reinterpret_cast<uint32_t*>(const_cast<int32_t*>(n.ids));  // made by pb200_doc_mask_upload: padded, resident
        } else {
          const size_t words = doc_mask_words(seg->num_docs);
          plan.temps.emplace_back(new DevBuf());
          int rc = plan.temps.back()->alloc(ctx, words * 4);
          if (rc) return rc;
          mask = (uint32_t*)plan.temps.back()->p;
          PB200_CUDA(cudaMemsetAsync(mask + need, 0, (words - need) * 4, st));
          PB200_CUDA(cudaMemcpyAsync(mask, n.ids, need * 4, cudaMemcpyHostToDevice, st));
          PB200_CUDA(cudaStreamSynchronize(st));  // caller's buffer may be a temporary
        }
        lf.kind = LEAF_DOCMASK;
        lf.bits = mask;
      } else if (n.op == PB200_F_DOC_RANGES) {
        if (n.num_ids % 2) { set_error("DOC_RANGES needs (start,end) pairs"); return PB200_E_INVALID; }
        if (n.num_ids == 0) { lf.kind = LEAF_NONE; continue; }
        plan.temps.emplace_back(new DevBuf());
        int rc = plan.temps.back()->alloc(ctx, (size_t)n.num_ids * 4);
        if (rc) return rc;
        PB200_CUDA(cudaMemcpyAsync(plan.temps.back()->p, n.ids, (size_t)n.num_ids * 4, cudaMemcpyHostToDevice, st));
        PB200_CUDA(cudaStreamSynchronize(st));
        lf.kind = LEAF_DOCRANGES;
        lf.ranges = (const int32_t*)plan.temps.back()->p;
        lf.num_ranges = n.num_ids / 2;
      } else {
        set_error("unsupported leaf op %d", n.op);
        return PB200_E_UNSUPPORTED;
      }
    }
  }

  if (!decode_jobs.empty()) {
    plan.temps.emplace_back(new DevBuf());
    int rc = plan.temps.back()->alloc(ctx, sizeof(DecodeJob) * decode_jobs.size());
    if (rc) return rc;
    rc = roaring_decode_batch(ctx, st, decode_jobs, plan.temps.back()->p);
    if (rc) return rc;
  }

  // ---- conjunctions: cheapest / most selective leaf first (per segment; AND is commutative).  The reference orders
  //      AND children by operator priority (FilterOperatorUtils.java:205-251) and, with AndScanReordering, by estimated
  //      cardinality (AndDocIdSet.java:118-120); here the estimate is the matching fraction of the dictionary. ----
  if (q.conj && nleaves > 1) {
    for (int s = 0; s < nseg; s++) {
      SegDesc& sd = plan.segs[s];
      auto cost = [&](const LeafDesc& lf) -> double {
        if (lf.slot < 0) return -1.0;  // doc masks / ranges / constants: no column to unpack
        const DeviceColumn& c = segments[s]->cols[plan.slot_cols[lf.slot]];
        double frac = 1.0;
        if (lf.kind == LEAF_RANGE) frac = (double)lf.span / std::max(c.cardinality, 1);
        else if (lf.kind == LEAF_LUT) frac = 0.5;
        return lf.negate ? 1.0 - frac : frac;
      };
      std::stable_sort(sd.leaves, sd.leaves + nleaves, [&](const LeafDesc& a, const LeafDesc& b) { return cost(a) < cost(b); });
    }
  }

  // ---- packed dispatch words (pb200_desc.h): everything the tile loop needs per leaf / aggregation in one word ----
  for (int s = 0; s < nseg; s++) {
    SegDesc& sd = plan.segs[s];
    for (int l = 0; l < nleaves; l++) {
      LeafDesc& lf = sd.leaves[l];
      const bool has_slot = lf.slot >= 0;
      lf.code = leaf_code(lf.kind, lf.cmp, lf.negate, has_slot ? sd.slots[lf.slot].bits : 0, has_slot ? sd.slots[lf.slot].stage_words : 0u);
    }
    // software-pipelined aggregations go LAST (nothing is waited on after them).  Aggregation only: q.defer_agg.
    // Group-by (dense / hash tables, not the CTA-private shared tables): up to two of {SUM / AVG over a 4-byte
    // dictionary, MIN, MAX} -- the kernel issues their loads for the last queue batch and reduces one tile later.
    bool pipelined[kMaxAggs] = {};
    int npipe = 0;
    if (!plan.group_by) {
      if (q.defer_agg >= 0) pipelined[q.defer_agg] = true;
    } else if (tune.gb_defer && q.smem_groups == 0) {
      for (int a = 0; a < nagg && npipe < 2; a++) {
        if (q.aggs[a].slot < 0) continue;
        const int fn = q.aggs[a].function, vk = q.aggs[a].val_kind;
        const bool sum4 = (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) && (vk == VAL_DICT_I32 || vk == VAL_DICT_F32);
        if (sum4 || fn == PB200_AGG_MIN || fn == PB200_AGG_MAX) { pipelined[a] = true; npipe++; }
      }
    }
    int n = 0;
    for (int pass = 0; pass < 2; pass++)
      for (int a = 0; a < nagg; a++) {
        if (q.aggs[a].slot < 0 || pipelined[a] != (pass == 1)) continue;
        const SlotDesc& sl = sd.slots[q.aggs[a].slot];
        sd.agg_code[n++] = agg_code(a, q.aggs[a].function, q.aggs[a].val_kind, sl.bits, sl.stage_words);
      }
    sd.num_agg_codes = n;
    sd.num_defer_codes = plan.group_by ? npipe : 0;
  }

  // ---- outputs ----
  AggAccum init_acc;
  memset(&init_acc, 0, sizeof init_acc);
  for (int a = 0; a < kMaxAggs; a++) init_acc.min_id[a] = 0xFFFFFFFFu;
  // initial values go up and results come back through ONE pooled pinned block, both asynchronously on the query's stream
  // (a pageable cudaMemcpy would synchronise the device twice per query)
  struct PinnedScratch {
    pb200_ctx* c; void* p = nullptr; size_t bytes = 0;
    ~PinnedScratch() { pinned_free(c, p, bytes); }
  } pacc{ctx};
  {
    int rc = pinned_alloc(ctx, 2 * (sizeof(AggAccum) + 32) * nres, &pacc.p, &pacc.bytes);
    if (rc) return rc;
  }
  // block layout (device and both pinned halves): nres AggAccum records, then 4 words per result for the count-carrier
  // verification {sum of carried counts, largest sum field, largest carried count, unused}
  const size_t acc_bytes = (sizeof(AggAccum) + 32) * nres;
  unsigned char* const pin_init = static_cast<unsigned char*>(pacc.p);
  unsigned char* const pin_back = pin_init + acc_bytes;
  AggAccum* host_acc = reinterpret_cast<AggAccum*>(pin_back);
  const unsigned long long* host_verify = reinterpret_cast<const unsigned long long*>(pin_back + sizeof(AggAccum) * nres);
  {
    memset(pin_init, 0, acc_bytes);
    AggAccum* init = reinterpret_cast<AggAccum*>(pin_init);
    for (int r = 0; r < nres; r++) init[r] = init_acc;
    int rc = accum_buf.alloc(ctx, acc_bytes);
    if (rc) return rc;
    PB200_CUDA(cudaMemcpyAsync(accum_buf.p, pin_init, acc_bytes, cudaMemcpyHostToDevice, st));
  }
  unsigned long long* const dev_verify = reinterpret_cast<unsigned long long*>(static_cast<unsigned char*>(accum_buf.p) + sizeof(AggAccum) * nres);
  for (int s = 0; s < nseg; s++) {
    const pb200_segment* seg = segments[s];
    SegDesc& sd = plan.segs[s];
    const int r = merge ? 0 : s;
    sd.accum = (AggAccum*)accum_buf.p + r;
    for (int a = 0; a < nagg; a++) {
      if (q.aggs[a].slot < 0) continue;
      const DeviceColumn& c = seg->cols[query->aggs[a].column];
      sd.dict[a] = c.dict_native;
      if ((q.aggs[a].function == PB200_AGG_SUM || q.aggs[a].function == PB200_AGG_AVG) && q.aggs[a].val_kind != VAL_RAW_I32 && !c.dict_native) {
        set_error("SUM/AVG over column %d needs its dictionary on the device", query->aggs[a].column);
        return PB200_E_INVALID;
      }
    }
  }
  if (!plan.group_by) {
    for (int r = 0; r < nres; r++) distinct_bufs[r].resize(nagg);
    for (int s = 0; s < nseg; s++) {
      const int r = merge ? 0 : s;
      for (int a = 0; a < nagg; a++) {
        if (q.aggs[a].function != PB200_AGG_DISTINCTCOUNT) continue;
        const DeviceColumn& c = segments[s]->cols[query->aggs[a].column];
        if (!distinct_bufs[r][a]) {
          int maxbits = c.bits;  // a merged result's bitset must hold the dictIds of every segment that writes into it
          if (merge) for (int t = 0; t < nseg; t++) maxbits = std::max(maxbits, segments[t]->cols[query->aggs[a].column].bits);
          size_t words = ((size_t)1 << maxbits) / 32 + 1;
          distinct_bufs[r][a].reset(new DevBuf());
          int rc = distinct_bufs[r][a]->alloc(ctx, words * 4);
          if (rc) return rc;
          PB200_CUDA(cudaMemsetAsync(distinct_bufs[r][a]->p, 0, words * 4, st));
        }
        plan.segs[s].distinct_bits[a] = (uint32_t*)distinct_bufs[r][a]->p;
      }
    }
  } else {
    // dense group table over the raw key space (column 0 least significant, DictionaryBasedGroupKeyGenerator :311-346)
    for (int r = 0; r < nres; r++) {
      const pb200_segment* seg = segments[merge ? 0 : r];
      pb200_result::Dense& d = res[r]->dense;
      d.ctx = ctx;
      long long groups = 1;
      unsigned __int128 space = 1;  // size of the raw key space
      for (int g = 0; g < ngb; g++) {
        int card = seg->cols[query->group_by_columns[g]].cardinality;
        card = std::max(card, 1);
        // every representable dictId must stay inside the table even for padded / corrupt rows
        d.mult.push_back((uint32_t)(unsigned long long)space);
        d.mult64.push_back((unsigned long long)space);
        d.cards.push_back(card);
        space *= (unsigned)card;
        if (space >> 63) {  // the reference's ARRAY_MAP regime (keys wider than a long): not accelerated
          set_error("group key space does not fit 63 bits (ARRAY_MAP regime): fall back to the reference operator");
          return PB200_E_UNSUPPORTED;
        }
      }
      // dense table up to kDenseMax raw keys (ARRAY / INT_MAP regimes of the reference), beyond it a hash table over the
      // 64-bit raw key (LONG_MAP regime, and INT_MAP key spaces too large to be worth a dense table)
      const long long dense_max = tune.dense_max;
      const bool hashed = space > (unsigned __int128)dense_max;
      if (hashed) {
        const long long limit = std::max(query->num_groups_limit, 1);
        long long cap = 1 << 16;
        while (cap < 2 * (limit + 1) && cap < (1ll << 27)) cap <<= 1;
        if (cap < 2 * (limit + 1)) { set_error("numGroupsLimit %lld too large for the device hash table", limit); return PB200_E_UNSUPPORTED; }
        groups = cap;
        void* hk = nullptr; void* hc = nullptr;
        int rc = dev_alloc(ctx, (size_t)cap * 8, &hk);
        if (rc) return rc;
        d.hkeys = (unsigned long long*)hk;
        PB200_CUDA(cudaMemsetAsync(hk, 0xFF, (size_t)cap * 8, st));
        rc = dev_alloc(ctx, 8, &hc);
        if (rc) return rc;
        d.hctl = (uint32_t*)hc;
        PB200_CUDA(cudaMemsetAsync(hc, 0, 8, st));
      } else {
        groups = (long long)space;
        // Small dense tables are SPREAD: entry of raw key k sits at k * stride.  A 10 000-group table is 80 KB = 312 of the
        // 256-byte chunks the L2 address hash distributes over the L2 slices -- some slices own three chunks, some none, and
        // every surviving row sends a reduction to them (ncu: hottest slice 75 % tag-request utilisation vs 56 % average).
        // With one entry per 128 bytes the same reductions spread over >= 4096 chunks.  Costs table bytes (<= 2 MB each,
        // memset + extraction scan), no instruction in the kernel: the stride is folded into the key multipliers.
        bool any_bitset = false;
        for (int a = 0; a < nagg; a++) any_bitset |= q.aggs[a].function == PB200_AGG_DISTINCTCOUNT;
        if (q.smem_groups == 0 && !any_bitset && tune.table_stride != 1) {
          long long s = 1;
          if (tune.table_stride > 1) s = tune.table_stride;
          else while (s < 16 && groups * 8 * s * 2 <= (2ll << 20)) s *= 2;   // keep each table within 2 MB
          while (s > 1 && groups * s > (1ll << 26)) s /= 2;
          d.stride = (int)s;
          groups *= s;
        }
      }
      d.groups = groups;
      d.live = true;
      d.num_groups_limit = query->num_groups_limit;
      for (int a = 0; a < nagg; a++) { d.aggs.push_back(query->aggs[a]); d.val_kind.push_back(q.aggs[a].val_kind); d.agg_cols.push_back(q.aggs[a].slot < 0 ? nullptr : &seg->cols[query->aggs[a].column]); }
      // one block per element kind
      // the exact per-group count is kept only when a function needs it; otherwise a MIN/MAX table (or a flag table)
      // marks the groups that exist -- one atomic less per surviving row
      bool need_count = tune.always_count != 0;
      bool has_minmax = false;
      for (int a = 0; a < nagg; a++) {
        need_count |= q.aggs[a].function == PB200_AGG_COUNT || q.aggs[a].function == PB200_AGG_AVG;
        has_minmax |= q.aggs[a].function == PB200_AGG_MIN || q.aggs[a].function == PB200_AGG_MAX;
      }
      bool need_seen = !need_count && !has_minmax && !hashed;  // a hash table's keys mark the groups that exist
      // ---- count carrier.  Every RED into the tables is an L2 read-modify-write, and on this path the L2 sector rate is
      // the bound (lts__t_sectors ~ 3.7x the streamed bytes at 10 % selectivity, profiles/r2_*).  When the query needs the
      // per-group row count (COUNT / AVG, or only as the group-exists marker) and sums an INT dictionary column, the
      // count rides in the upper bits of that sum: each row adds (value - vmin) + 2^shift with ONE reduction.
      //   Fields: sum field = `shift` bits, count field = 64 - shift bits, balanced so that both overflow at about the
      //   same rows per group: shift = ceil((64 + bits(R)) / 2), R = vmax - vmin + 1 from the dictionary (a 20-bit value
      //   range leaves 22 bits = 4 M rows per group; a full 32-bit range 65 535).
      //   Either field CAN overflow; both are detected EXACTLY after the launch from one number: a sum field overflow
      //   carries into the count field (counts only grow: value - vmin >= 0), a count overflow drops 2^(64-shift) from
      //   it, so  sum_g count_g == matched docs  iff neither happened -- the two cannot cancel because the carries total
      //   at most docs x R / 2^shift < 2^(64-shift) when docs x R < 2^64 (the admission test below).  On a mismatch the
      //   submission runs again with a separate COUNT table (kRetryWithoutCountCarrier); results are exact either way.
      d.pack_agg = -1;
      const bool deferred = merge && (query->flags & PB200_Q_DEFER_FINALIZE);
      d.reduce_world = deferred ? std::max(query->reduce_world, 1) : 1;
      if (allow_count_carrier && !(query->flags & PB200_Q_NO_COUNT_CARRIER) && tune.pack_count && q.smem_groups == 0 &&
          (need_count || need_seen)) {
        unsigned long long docs = 0;
        for (int s = 0; s < nseg; s++) if (merge || s == r) docs += (unsigned long long)segments[s]->num_docs;
        // a table that will be summed with the other GPUs' tables: the admission test covers the docs of ALL of them
        if (deferred) docs = query->merged_docs_bound > 0 ? (unsigned long long)query->merged_docs_bound : docs * (unsigned long long)d.reduce_world;
        auto bits_of = [](unsigned long long x) { int b = 0; while (b < 64 && (x >> b)) b++; return b; };
        for (int a = 0; a < nagg && d.pack_agg < 0; a++) {
          const int fn = q.aggs[a].function;
          if ((fn != PB200_AGG_SUM && fn != PB200_AGG_AVG) || q.aggs[a].val_kind != VAL_DICT_I32) continue;
          long long vmin = std::numeric_limits<long long>::max(), vmax = std::numeric_limits<long long>::min();
          bool ok = true;
          for (int s = 0; s < nseg && ok; s++) {
            if (!merge && s != r) continue;
            const DeviceColumn& c = segments[s]->cols[query->aggs[a].column];
            if (c.dict_host.size() < 4ull * std::max(c.cardinality, 1) || c.stored_type != PB200_INT) { ok = false; break; }
            // the other GPUs must subtract the SAME minimum: only a table-wide (domain) dictionary guarantees that
            if (d.reduce_world > 1 && !c.dict_shared) { ok = false; break; }
            int32_t v0, v1;   // sorted dictionary: first / last entry
            memcpy(&v0, c.dict_host.data(), 4);
            memcpy(&v1, c.dict_host.data() + 4ull * (c.cardinality - 1), 4);
            vmin = std::min<long long>(vmin, v0);
            vmax = std::max<long long>(vmax, v1);
          }
          if (!ok) continue;
          const int rbits = bits_of((unsigned long long)(vmax - vmin));   // value - vmin fits rbits bits
          if (bits_of(docs) + rbits > 63) continue;                        // docs x R < 2^63: the detection is airtight
          d.pack_agg = a;
          d.pack_shift = tune.pack_shift > 0 ? tune.pack_shift : (64 + rbits + 1) / 2;
          d.pack_vmin = vmin;
        }
        if (d.pack_agg >= 0) { need_count = false; need_seen = false; }
      }
      long long n_i64 = need_count ? 1 : 0, n_f64 = 0, n_max = need_seen ? 1 : 0, n_min = 0;
      for (int a = 0; a < nagg; a++) {
        const int fn = q.aggs[a].function, vk = q.aggs[a].val_kind;
        if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) { if (sum_in_double(vk)) n_f64++; else n_i64++; }
        else if (fn == PB200_AGG_MIN) n_min++;
        else if (fn == PB200_AGG_MAX) n_max++;
      }
      auto alloc_block = [&](void** p, long long elems, size_t esz, int fill) -> int {
        if (!elems) return PB200_OK;
        int rc = dev_alloc(ctx, (size_t)elems * esz, p);
        if (rc) return rc;
        PB200_CUDA(cudaMemsetAsync(*p, fill, (size_t)elems * esz, st));
        return PB200_OK;
      };
      d.i64_elems = n_i64 * groups; d.f64_elems = n_f64 * groups; d.u32max_elems = n_max * groups; d.u32min_elems = n_min * groups;
      // cross-GPU combine of a count-carrying table: ONE extra int64 behind the tables carries this rank's "not provably
      // safe" verdict (0 / 1), so that the verdicts of all ranks are summed by the same collective that sums the tables
      // ... and, in front of it, the four execution statistics of this rank: tables, verdict and statistics of a query then
      // cross the GPUs in ONE collective (pb200_comm.cu).  Tail = {docs scanned, entries in filter, entries post filter,
      // total docs, verdict}; the verdict stays the LAST element.
      d.flag_slot = d.pack_agg >= 0 && d.reduce_world > 1;
      d.tail_slots = (d.reduce_world > 1 && d.i64_elems > 0) ? 5 : 0;
      d.i64_elems += d.tail_slots;
      int rc;
      if ((rc = alloc_block(&d.i64_block, d.i64_elems, 8, 0))) return rc;
      if ((rc = alloc_block(&d.f64_block, d.f64_elems, 8, 0))) return rc;
      if ((rc = alloc_block(&d.u32max_block, d.u32max_elems, 4, 0))) return rc;
      if ((rc = alloc_block(&d.u32min_block, d.u32min_elems, 4, 0xFF))) return rc;
      d.count = need_count ? (unsigned long long*)d.i64_block : nullptr;
      d.seen = need_seen ? (uint32_t*)d.u32max_block : nullptr;
      long long ii = need_count ? 1 : 0, fi = 0, xi = need_seen ? 1 : 0, ni = 0;
      for (int a = 0; a < nagg; a++) {
        const int fn = q.aggs[a].function, vk = q.aggs[a].val_kind;
        if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) {
          if (sum_in_double(vk)) d.dsum[a] = (double*)d.f64_block + (fi++) * groups;
          else d.isum[a] = (long long*)d.i64_block + (ii++) * groups;
          if (a == d.pack_agg) d.exists_packed = (const unsigned long long*)d.isum[a];
        } else if (fn == PB200_AGG_MIN) { d.gmin[a] = (uint32_t*)d.u32min_block + (ni++) * groups; if (!need_count && !d.exists_max && !d.exists_min) d.exists_min = d.gmin[a]; }
        else if (fn == PB200_AGG_MAX) { d.gmax[a] = (uint32_t*)d.u32max_block + (xi++) * groups; if (!need_count && !d.exists_max && !d.exists_min) d.exists_max = d.gmax[a]; }
        else if (fn == PB200_AGG_DISTINCTCOUNT) {  // one dictId bitset per group / slot
          const DeviceColumn& c = seg->cols[query->aggs[a].column];
          const unsigned long long words = ((unsigned long long)c.cardinality + 31) / 32;
          if (words * (unsigned long long)groups > (1ull << 28)) {
            set_error("DISTINCTCOUNT with GROUP BY: %lld groups x %d dictIds exceed the device bitset budget", groups, c.cardinality);
            return PB200_E_UNSUPPORTED;
          }
          void* bp = nullptr;
          if ((rc = dev_alloc(ctx, (size_t)(words * groups) * 4, &bp))) return rc;
          PB200_CUDA(cudaMemsetAsync(bp, 0, (size_t)(words * groups) * 4, st));
          d.dbits[a] = (uint32_t*)bp;
          d.dwords[a] = (uint32_t)words;
        }
      }
    }
    for (int s = 0; s < nseg; s++) {
      SegDesc& sd = plan.segs[s];
      pb200_result::Dense& d = res[merge ? 0 : s]->dense;
      sd.g_count = d.count;
      sd.g_seen = d.seen;
      for (int a = 0; a < nagg; a++) {
        sd.sum_addend[a] = 0ull - (1ull << 31);  // plain INT-dictionary sum: remove the device copy's bias
        if (a == d.pack_agg) sd.sum_addend[a] = (1ull << d.pack_shift) - (unsigned long long)((uint32_t)(int32_t)d.pack_vmin ^ 0x80000000u);
      }
      for (int a = 0; a < nagg; a++) { sd.g_isum[a] = d.isum[a]; sd.g_dsum[a] = d.dsum[a]; sd.g_min[a] = d.gmin[a]; sd.g_max[a] = d.gmax[a]; sd.distinct_bits[a] = d.dbits[a]; sd.distinct_words[a] = d.dwords[a]; }
      for (int g = 0; g < ngb; g++) { sd.group_mult[g] = d.mult[g] * (uint32_t)d.stride; sd.group_mult64[g] = d.mult64[g]; }  // hash tables: stride 1
      sd.h_keys = d.hkeys;
      sd.h_ctl = d.hctl;
      sd.h_mask = d.hkeys ? (uint32_t)(d.groups - 1) : 0u;
      sd.h_limit = query->num_groups_limit;
    }
  }

  // ---- launch: chunks of <= kMaxLaunchSegs segments (their TMA table travels in the kernel parameters) ----
  DevBuf dsegs;
  int rc = dsegs.alloc(ctx, sizeof(SegDesc) * nseg);
  if (rc) return rc;
  struct Events {  // pooled per context (creating / destroying two events per query costs more than the launch itself)
    pb200_ctx* c; cudaEvent_t a = nullptr, b = nullptr;
    ~Events() { give_event(c, a); give_event(c, b); }
  } ev{ctx};
  ev.a = take_event(ctx);
  ev.b = take_event(ctx);
  if (!ev.a || !ev.b) { set_error("cudaEventCreate failed"); return PB200_E_CUDA; }
  cudaEvent_t e0 = ev.a, e1 = ev.b;
  cudaError_t le = cudaSuccess;
  int grid = 0;
  std::vector<SegDesc> launch_segs = plan.segs;
  for (int c0 = 0; c0 < nseg; c0 += kMaxLaunchSegs) {  // first_tile is relative to the chunk
    long long cursor = 0;
    for (int s = c0; s < std::min(nseg, c0 + kMaxLaunchSegs); s++) { launch_segs[s].first_tile = cursor; cursor += launch_segs[s].num_tiles; }
  }
  PB200_CUDA(cudaMemcpyAsync(dsegs.p, launch_segs.data(), sizeof(SegDesc) * nseg, cudaMemcpyHostToDevice, st));
  const double t_launch = now_ms();
  PB200_CUDA(cudaEventRecord(e0, st));
  for (int c0 = 0; c0 < nseg && le == cudaSuccess; c0 += kMaxLaunchSegs) {
    const int cn = std::min(nseg - c0, (int)kMaxLaunchSegs);
    QueryDesc cq = q;
    TmaTable tt;
    memset(&tt, 0, sizeof tt);
    cq.num_segments = cn;
    cq.total_tiles = 0;
    for (int s = 0; s < cn; s++) {
      const SegDesc& sd = launch_segs[c0 + s];
      tt.seg[s].first_tile = (int32_t)sd.first_tile;
      tt.seg[s].end_tile = (int32_t)(sd.first_tile + sd.num_tiles);
      tt.seg[s].stage_tx = sd.stage_tx;
      tt.seg[s].num_docs = (uint32_t)sd.num_docs;
      for (int k = 0; k < q.num_slots; k++) tt.seg[s].slot[k] = TmaSlot{sd.slots[k].data, sd.slots[k].tile_bytes, sd.slots[k].stage_words};
      if (q.conj && q.num_slots > 0 && tune.skip) {
        int nm = 0;
        for (int l = 0; l < nleaves && nm < kMaxSkipMasks; l++)
          if (sd.leaves[l].kind == LEAF_DOCMASK && !sd.leaves[l].negate) tt.seg[s].skip_mask[nm++] = sd.leaves[l].bits;
      }
      cq.total_tiles += sd.num_tiles;
    }
    for (int s = cn; s < kMaxLaunchSegs; s++) { tt.seg[s].first_tile = cq.total_tiles; tt.seg[s].end_tile = 0x7FFFFFFF; }  // sentinel
    grid = (int)std::min<long long>((long long)ctx->sm_count * ctas_per_sm, std::max<long long>(cq.total_tiles, 1));
    if (cq.total_tiles >= (1 << 30)) { set_error("too many tiles in one launch"); return PB200_E_UNSUPPORTED; }
    if (tune.grid > 0) grid = tune.grid;
    const SegDesc* dptr = (const SegDesc*)dsegs.p + c0;
    // instantiations: W in {6, 8} x {aggregation only (2 CTAs/SM), group-by with 2 or 1 CTAs/SM}
    const ScanVariant variant{cw, plan.group_by, !plan.group_by && !(cw == 8 && !tune.defer), plan.group_by ? ctas_per_sm : 2};
    le = launch_scan_variant(variant, plan.smem_bytes, grid, cq, tt, dptr, st);
  }
  if (le != cudaSuccess) { set_error("scan kernel launch failed: %s (smem %zu B, grid %d)", cudaGetErrorString(le), plan.smem_bytes, grid); return PB200_E_CUDA; }
  PB200_CUDA(cudaEventRecord(e1, st));
  if (plan.group_by)
    for (int r = 0; r < nres; r++) {
      const pb200_result::Dense& d = res[r]->dense;
      if (d.pack_agg < 0) continue;
      const int vb = (int)std::max<long long>(1, std::min<long long>((d.groups + 1023) / 1024, (long long)ctx->sm_count * 4));
      carrier_verify_kernel<<<vb, 256, 0, st>>>((const unsigned long long*)d.isum[d.pack_agg], d.groups, d.pack_shift, dev_verify + 4 * r);
    }
  PB200_CUDA(cudaMemcpyAsync(pin_back, accum_buf.p, acc_bytes, cudaMemcpyDeviceToHost, st));
  const double t_queued = now_ms();
  cudaError_t se = cudaStreamSynchronize(st);
  if (se != cudaSuccess) { set_error("scan kernel failed: %s", cudaGetErrorString(se)); return PB200_E_CUDA; }
  const double t_synced = now_ms();
  if (plan.group_by)
    for (int r = 0; r < nres; r++) {
      const pb200_result::Dense& d = res[r]->dense;
      if (d.pack_agg < 0) continue;
      const unsigned long long* vw = host_verify + 4 * r;   // {sum of counts, largest sum field, largest count}
      const bool exact = vw[0] == host_acc[r].count;
      if (d.reduce_world > 1) {
        // cross-GPU: the reduce adds `reduce_world` fields of each kind; neither can overflow if every rank's largest one
        // stays below its capacity / reduce_world.  A rank cannot rerun on its own (its peers' tables would have another
        // layout): it marks the result and the combine layer reruns the query on all ranks (PB200_Q_NO_COUNT_CARRIER).
        const unsigned long long w = (unsigned long long)d.reduce_world;
        const unsigned long long sum_lim = ((1ull << d.pack_shift) - 1ull) / w, cnt_lim = ((1ull << (64 - d.pack_shift)) - 1ull) / w;
        res[r]->dense.carrier_unsafe = !exact || vw[1] > sum_lim || vw[2] > cnt_lim;
        if (d.flag_slot) {   // the stream is idle (synchronised above): a blocking 8-byte copy, done before the call returns
          // (callers that bring their own collective read it from the block; pb200_result_combine rewrites the whole tail)
          const long long verdict = res[r]->dense.carrier_unsafe ? 1 : 0;
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
      return kRetryWithoutCountCarrier;  // ResultCleanup frees the tables
    }
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);

  // ---- results ----
  int projected = 0;
  for (int k = 0; k < q.num_slots; k++) if (q.slot_roles[k] & (ROLE_GROUP | ROLE_AGG)) projected++;
  for (int r = 0; r < nres; r++) {
    pb200_result& R = *res[r];
    const AggAccum acc = host_acc[r];
    long long total_docs = 0;
    if (merge) for (int s = 0; s < nseg; s++) total_docs += segments[s]->num_docs; else total_docs = segments[r]->num_docs;
    R.meta.num_group_by = ngb;
    R.meta.num_aggs = nagg;
    R.agg_functions.resize(nagg);
    for (int a = 0; a < nagg; a++) R.agg_functions[a] = q.aggs[a].function;
    R.meta.num_docs_scanned = (int64_t)acc.count;
    long long in_filter = 0;  // device semantics: every scan leaf looks at every doc of its segment
    for (int s = 0; s < nseg; s++) {
      if (!merge && s != r) continue;
      const pb200_filter_node* fs = per_seg_filter ? query->filter + (size_t)s * nnodes : query->filter;
      for (int l = 0; l < nleaves; l++) if (is_scan_leaf(fs[plan.leaf_node[l]].op)) in_filter += segments[s]->num_docs;
    }
    R.meta.num_entries_scanned_in_filter = in_filter;
    R.meta.num_entries_scanned_post_filter = (int64_t)acc.count * projected;
    R.meta.num_total_docs = total_docs;
    R.meta.device_ms = ms;
    R.dbl.resize(nagg); R.lng.resize(nagg); R.ids.resize(nagg); R.distinct.resize(nagg);
    if (!plan.group_by) {
      R.meta.num_groups = -1;
      R.meta.regime = PB200_REGIME_NONE;
      const pb200_segment* seg = segments[merge ? 0 : r];
      for (int a = 0; a < nagg; a++) {
        const int fn = q.aggs[a].function, vk = q.aggs[a].val_kind;
        double d = 0; int64_t l = 0; int32_t id = -1;
        const DeviceColumn* c = q.aggs[a].slot < 0 ? nullptr : &seg->cols[query->aggs[a].column];
        auto value_of = [&](uint32_t x) -> double {
          if (vk == VAL_RAW_I32) return (double)(int32_t)(x ^ 0x80000000u);
          const unsigned char* h = c->dict_host.data();
          switch (vk) {
            case VAL_DICT_I32: { int32_t v; memcpy(&v, h + 4ull * x, 4); return (double)v; }
            case VAL_DICT_I64: { int64_t v; memcpy(&v, h + 8ull * x, 8); return (double)v; }
            case VAL_DICT_F32: { float v; memcpy(&v, h + 4ull * x, 4); return (double)v; }
            default: { double v; memcpy(&v, h + 8ull * x, 8); return v; }
          }
        };
        if (fn == PB200_AGG_COUNT) { l = (int64_t)acc.count; d = (double)l; }
        else if (fn == PB200_AGG_SUM || fn == PB200_AGG_AVG) {
          d = sum_in_double(vk) ? acc.dsum[a] : (double)acc.isum[a];
          l = (int64_t)acc.count;
        } else if (fn == PB200_AGG_MIN) {
          if (acc.min_id[a] == 0xFFFFFFFFu || acc.count == 0) d = INFINITY; else { id = (int32_t)acc.min_id[a]; d = c->dict_host.empty() && vk != VAL_RAW_I32 ? (double)id : value_of(acc.min_id[a]); }
        } else if (fn == PB200_AGG_MAX) {
          if (acc.max_id_plus1[a] == 0) d = -INFINITY; else { id = (int32_t)(acc.max_id_plus1[a] - 1); d = c->dict_host.empty() && vk != VAL_RAW_I32 ? (double)id : value_of(acc.max_id_plus1[a] - 1); }
        } else if (fn == PB200_AGG_DISTINCTCOUNT) {
          int maxbits = c->bits;
          if (merge) for (int t = 0; t < nseg; t++) maxbits = std::max(maxbits, segments[t]->cols[query->aggs[a].column].bits);
          size_t words = ((size_t)1 << maxbits) / 32 + 1;
          std::vector<uint32_t> bits(words);
          PB200_CUDA(cudaMemcpy(bits.data(), distinct_bufs[r][a]->p, words * 4, cudaMemcpyDeviceToHost));
          std::vector<int32_t> idsv;
          for (size_t w = 0; w < words; w++) { uint32_t x = bits[w]; while (x) { idsv.push_back((int32_t)(w * 32 + __builtin_ctz(x))); x &= x - 1; } }
          l = (int64_t)idsv.size(); d = (double)l;
          R.distinct[a].push_back(std::move(idsv));
        }
        R.dbl[a].push_back(d); R.lng[a].push_back(l); R.ids[a].push_back(id);
      }
    } else {
      std::vector<int> cards = R.dense.cards;
      R.meta.regime = regime_of(cards, query->max_initial_result_holder_capacity);
      R.meta.reserved = (R.dense.pack_agg >= 0 ? 1 : 0) | (R.dense.carrier_unsafe ? 2 : 0) | (R.dense.flag_slot ? 4 : 0);  // include/pinot_b200.h
    }
  }
  const bool defer_finalize = merge && (query->flags & PB200_Q_DEFER_FINALIZE);
  const double t_results = now_ms();
  if (plan.group_by && defer_finalize) {
    for (int r = 0; r < nres; r++) { res[r]->meta.num_groups = 0; res[r]->dbl.assign(nagg, {}); res[r]->lng.assign(nagg, {}); res[r]->ids.assign(nagg, {}); res[r]->distinct.assign(nagg, {}); }
  } else if (plan.group_by) {  // all results of the submission are extracted together (two device round trips in total)
    std::vector<pb200_result*> rs;
    for (int r = 0; r < nres; r++) rs.push_back(res[r].get());
    int frc = extract_groups(ctx, rs.data(), nres, st);
    if (frc) return frc;
    if (!merge) {  // per-segment results do not need the dense state any more
      for (int r = 0; r < nres; r++) {
        pb200_result::Dense& d = res[r]->dense;
        dev_free(ctx, d.i64_block); dev_free(ctx, d.f64_block); dev_free(ctx, d.u32max_block); dev_free(ctx, d.u32min_block);
        dev_free(ctx, d.hkeys); dev_free(ctx, d.hctl);
        d.hkeys = nullptr; d.hctl = nullptr;
        for (int a = 0; a < kMaxAggs; a++) { dev_free(ctx, d.dbits[a]); d.dbits[a] = nullptr; }
        d.i64_block = d.f64_block = d.u32max_block = d.u32min_block = nullptr;
        d.live = false;
      }
    }
  }
  cleanup.armed = false;
  for (int r = 0; r < nres; r++) results[r] = res[r].release();
  const double t_exit = now_ms();
  g_phase_ms[PB200_PHASE_PLAN] = t_launch - t_enter;       // validation, plan, table allocation + memsets queued, descriptors
  g_phase_ms[PB200_PHASE_LAUNCH] = t_queued - t_launch;    // kernel launches queued
  g_phase_ms[PB200_PHASE_DEVICE_WAIT] = t_synced - t_queued;
  g_phase_ms[PB200_PHASE_RESULTS] = t_results - t_synced;  // carrier verdict, metadata, scalar results
  g_phase_ms[PB200_PHASE_EXTRACT] = t_exit - t_results;    // group extraction (device kernels + their sync) and table release
  g_phase_ms[PB200_PHASE_TOTAL] = t_exit - t_enter;
  return PB200_OK;
}

extern "C" int32_t pb200_result_finalize(pb200_ctx* ctx, pb200_result* R) {
  if (!ctx || !R) { set_error("null argument"); return PB200_E_INVALID; }
  pb200_result::Dense& d = R->dense;
  if (!d.ctx || d.groups <= 0 || !d.live) { set_error("result has no dense device state"); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = take_stream(ctx);
  struct StreamReturn { pb200_ctx* c; cudaStream_t s; ~StreamReturn() { give_stream(c, s); } } stream_return{ctx, st};
  pb200_result* one[1] = {R};
  return extract_groups(ctx, one, 1, st);
}

extern "C" int32_t pb200_result_device_buffers(pb200_result* R, int32_t kind, void** p, int64_t* n) {
  if (!R || !p || !n) { set_error("null argument"); return PB200_E_INVALID; }
  pb200_result::Dense& d = R->dense;
  if (d.hkeys) { set_error("hash group tables of different GPUs are not element-wise reducible"); return PB200_E_UNSUPPORTED; }
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
  if (!R || a < 0 || a >= (int)R->distinct.size() || row < 0 || row >= (int)R->distinct[a].size()) { set_error("bad distinct index"); return PB200_E_INVALID; }
  const auto& v = R->distinct[a][row];
  for (int64_t i = 0; i < (int64_t)v.size() && i < cap; i++) out[i] = v[i];
  return (int64_t)v.size();
}
extern "C" int32_t pb200_result_free(pb200_result* R) {
  if (!R) return PB200_OK;
  pb200_result::Dense& d = R->dense;
  if (d.ctx) { dev_free(d.ctx, d.i64_block); dev_free(d.ctx, d.f64_block); dev_free(d.ctx, d.u32max_block); dev_free(d.ctx, d.u32min_block); dev_free(d.ctx, d.hkeys); dev_free(d.ctx, d.hctl); for (int a = 0; a < kMaxAggs; a++) dev_free(d.ctx, d.dbits[a]); }
  delete R;
  return PB200_OK;
}
