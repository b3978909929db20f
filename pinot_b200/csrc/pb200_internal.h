// pb200_internal.h -- host-side objects behind the opaque C-ABI handles.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/pinot_b200.h"
#include "pb200_desc.h"

namespace pb200 {

void set_error(const char* fmt, ...);
#define PB200_CUDA(call)                                                                         \
  do {                                                                                           \
    cudaError_t e__ = (call);                                                                    \
    if (e__ != cudaSuccess) {                                                                    \
      ::pb200::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return PB200_E_CUDA;                                                                       \
    }                                                                                            \
  } while (0)

// Upper bound of the scan kernel's tile (consumer warps x 1024 rows).  Forward indexes are padded so that whole tiles
// of any size up to this can be streamed.
constexpr int kMaxTileRows = 8192;
// words a device doc mask needs: whole tiles + one spare tile (the kernel reads masks tile-wise) + a tail
inline size_t doc_mask_words(long long num_docs) { return (((size_t)num_docs + kMaxTileRows - 1) / kMaxTileRows + 1) * (kMaxTileRows / 32) + 8; }

struct DeviceColumn {
  int fwd_kind = 0, stored_type = 0, bits = 0, cardinality = 0;
  uint32_t* fwd = nullptr;        // packed words, padded to whole max tiles (+ slack)
  uint64_t fwd_file_bytes = 0;    // length of the original index file: ceil(N*bits/8)
  uint64_t fwd_alloc_bytes = 0;
  void* dict_native = nullptr;    // device: little-endian value array
  std::vector<unsigned char> dict_host;  // host copy of the native array (finalisation: dictId -> value)
  std::vector<unsigned char> dict_be;    // original big-endian bytes (read-back / tests)
  unsigned char* inv = nullptr;   // device: inverted index file bytes
  uint64_t inv_bytes = 0;
  std::vector<uint32_t> inv_offsets;  // host: (card+1) offsets into inv (file-relative)
  bool owns = true;
  bool pooled = false;            // fwd came from the context's caching allocator
  int dict_entry_bytes = 0;       // width of one dict_be entry (4 / 8, STRING: lengthOfEachEntry)
  uint64_t dict_hash = 0;         // content hash of the dictionary (pb200_domain.cu dictionary_hash); 0 = no dictionary known
  bool dict_shared = false;       // dict_native belongs to the bound domain, not to this column
  std::vector<uint32_t> local_ids;  // bound to a domain: the (global) ids that occur in THIS segment, ascending
  int dict_width() const { return (stored_type == PB200_LONG || stored_type == PB200_DOUBLE) ? 8 : 4; }
};

}  // namespace pb200

namespace pb200 {
// Tuning knobs of the scan kernel launch.  Read from the environment ONCE, at pb200_init (PB200_W, PB200_CTAS, ... --
// DESIGN.md section 3.1), changeable afterwards with pb200_tuning_set(); read by the scan planner (plan_scan,
// pb200_plan.cpp), which pb200_execute calls with a copy taken under the context's lock -- neither calls getenv.
struct Tuning {
  int warps = 6;                 // PB200_W: 6 | 8 warps per CTA
  int sparse_max = 4;            // PB200_SPARSE_MAX
  int sparse_max_agg = -1;       // PB200_SPARSE_MAX_AGG (-1: rule in plan_scan)
  int ctas_per_sm = 2;           // PB200_CTAS
  int stages = 0;                // PB200_STAGES (0: as many as fit)
  int grid = 0;                  // PB200_GRID (0: SMs x CTAs per SM)
  int smem_groups = 1;           // !PB200_NO_SMEM_GROUPS
  long long smem_groups_max = 1ll << 24;  // PB200_SMEM_GROUPS_MAX: cap on top of the shared-memory budget (default: none)
  int smem_copies = 0;           // PB200_SMEM_COPIES (0: as many as fit)
  long long dense_max = 1ll << 24;   // PB200_DENSE_MAX: dense group table up to this many raw keys, hash table beyond
  int defer = 1;                 // !PB200_NO_DEFER: software-pipelined gathers, aggregation-only kernel
  int gb_defer = 1;              // !PB200_NO_GB_DEFER: software-pipelined last queue batch, group-by kernel
  int pack_count = 1;            // !PB200_NO_PACK_COUNT: group-by COUNT carried inside an INT SUM's reductions (pb200_plan.cpp)
  int table_stride = 0;          // PB200_TABLE_STRIDE: dense group tables hold raw key k at k * stride (0 = auto, 1 = off)
  int pack_shift = 0;            // PB200_PACK_SHIFT: force the carrier's count shift (tests of the overflow fallback); 0 = from the doc count
  int skip = 1;                  // !PB200_NO_SKIP: bitmap-driven slice skipping
  int always_count = 0;          // PB200_ALWAYS_COUNT
  int raw_dict_max = 1 << 20;    // PB200_RAW_DICT_MAX: raw columns with at most this many distinct values are dictionary-encoded at load (0 = never)
};
}  // namespace pb200

struct pb200_ctx {
  pb200::Tuning tune;
  int device = 0;
  int sm_count = 0;
  int max_smem_optin = 0;
  std::mutex mu;
  std::vector<cudaStream_t> free_streams;
  std::vector<cudaEvent_t> free_events;
  void* nccl_comm = nullptr;      // ncclComm_t of the cross-GPU combine (pb200_comm.cu), NULL until pb200_comm_init
  int comm_rank = 0, comm_world = 1;
  long long* comm_scratch = nullptr;  // device: 4 statistics in, 4 reduced out
  long long* comm_pinned = nullptr;   // pinned host staging for the statistics and the carrier verdict
  std::mutex comm_mu;
  std::multimap<size_t, void*> free_blocks;  // caching allocator: size -> block
  std::map<void*, size_t> block_size;
  size_t pooled_bytes = 0;
  std::multimap<size_t, void*> free_pinned;  // pinned host staging blocks (result read-back), size -> block
};

// Table-wide dictionaries (pb200_domain.cu)
struct pb200_domain {
  pb200_ctx* ctx = nullptr;
  struct Col {
    int column = 0, stored_type = 0, entry_bytes = 0, cardinality = 0, bits = 0;
    std::vector<unsigned char> dict_be;    // big-endian sorted values / padded strings
    std::vector<unsigned char> dict_host;  // native little-endian values (numeric types)
    void* dict_native = nullptr;           // device copy (INT: biased), shared by every bound segment
    uint64_t hash = 0;
  };
  std::vector<Col> cols;
  int refs = 1;  // the creator + one per bound segment (guarded by ctx->mu)
};

struct pb200_segment {
  pb200_ctx* ctx = nullptr;
  std::string name;
  int num_docs = 0;
  std::vector<pb200::DeviceColumn> cols;
  int64_t device_bytes = 0;
  pb200_domain* domain = nullptr;  // holds one reference
};

namespace pb200 {
// A pinned (mapped) host block shared by the results whose extracted groups live in it; goes back to the context's pinned
// pool when the last result is freed.
struct PinnedBlock {
  pb200_ctx* ctx = nullptr;
  void* p = nullptr;
  size_t bytes = 0;
  ~PinnedBlock();
};
}  // namespace pb200

struct pb200_result {
  pb200_result_meta meta{};
  // Extracted groups in their final layout inside a pinned block written by the device (pb200_extract.cu); when
  // view.block is set the accessors read these columns, else the vectors below (host-built results).
  struct View {
    std::shared_ptr<pb200::PinnedBlock> block;
    size_t rows = 0;
    const int32_t* keys = nullptr;                 // [rows x num_group_by]
    const double* dbl[pb200::kMaxAggs] = {};       // NULL: all zero
    const int64_t* lng[pb200::kMaxAggs] = {};      // NULL: all zero
    const int32_t* ids[pb200::kMaxAggs] = {};      // NULL: all -1
  } view;
  pb200_order_by order{};                        // ORDER BY spec of a group-by result (num_items 0: none), applied at extraction
  std::vector<int32_t> agg_functions;            // PB200_AGG_* per aggregation (set by pb200_execute)
  std::vector<int32_t> keys;                     // [G x k]
  std::vector<std::vector<double>> dbl;          // per agg [rows]
  std::vector<std::vector<int64_t>> lng;
  std::vector<std::vector<int32_t>> ids;         // per agg [rows] MIN/MAX dictIds (-1 empty)
  std::vector<std::vector<std::vector<int32_t>>> distinct;  // per agg, per row
  // merged dense-table state kept on the device for multi-GPU combine
  struct Dense {
    pb200_ctx* ctx = nullptr;
    long long groups = 0;                        // table entries: dense key space x stride, or hash capacity
    int stride = 1;                              // dense tables: raw key k lives at entry k * stride (pb200_plan.cpp)
    bool live = false;                           // device tables still allocated
    unsigned long long* count = nullptr;         // NULL when no COUNT / AVG
    uint32_t* seen = nullptr;                    // group-exists flags (inside the u32max block) or NULL
    uint32_t* exists_max = nullptr;              // a MAX table doubling as the group-exists marker, or NULL
    uint32_t* exists_min = nullptr;              // a MIN table doubling as the group-exists marker, or NULL
    // count carrier (pb200_plan.cpp): aggregation pack_agg's int64 table holds  sum(value - pack_vmin) + count << pack_shift
    int pack_agg = -1, pack_shift = 0;
    long long pack_vmin = 0;
    const unsigned long long* exists_packed = nullptr;  // that table: non-zero <=> the group exists
    int reduce_world = 1;                               // tables of this many GPUs will be summed into it
    bool carrier_unsafe = false;                        // its sum field may overflow in that reduce: rerun without carrier
    bool flag_slot = false;                             // the i64 block's LAST element is this rank's unsafe verdict (0 / 1)
    int tail_slots = 0;                                 // i64 block ends with {4 execution statistics, verdict} (reduce_world > 1)
    long long* isum[pb200::kMaxAggs] = {};
    double* dsum[pb200::kMaxAggs] = {};
    uint32_t* gmin[pb200::kMaxAggs] = {};
    uint32_t* gmax[pb200::kMaxAggs] = {};
    std::vector<uint32_t> mult;
    std::vector<unsigned long long> mult64;
    uint32_t* dbits[pb200::kMaxAggs] = {};      // DISTINCTCOUNT with GROUP BY: per-group dictId bitsets, dwords[a] words each
    uint32_t dwords[pb200::kMaxAggs] = {};
    unsigned long long* hkeys = nullptr;        // hash table keys (NULL: dense table indexed by raw key)
    uint32_t* hctl = nullptr;                   // [0] inserted, [1] overflow
    std::vector<int> cards;
    std::vector<pb200_agg> aggs;
    std::vector<int> val_kind;
    std::vector<const pb200::DeviceColumn*> agg_cols;
    int num_groups_limit = 0;
    // one contiguous allocation per kind so a collective can reduce it in place
    void* i64_block = nullptr; long long i64_elems = 0;
    void* f64_block = nullptr; long long f64_elems = 0;
    void* u32max_block = nullptr; long long u32max_elems = 0;
    void* u32min_block = nullptr; long long u32min_elems = 0;
  } dense;
};

namespace pb200 {
// caching device allocator + stream pool (thread safe)
int dev_alloc(pb200_ctx* ctx, size_t bytes, void** out);
void dev_free(pb200_ctx* ctx, void* p);
int pinned_alloc(pb200_ctx* ctx, size_t bytes, void** out, size_t* got);  // cudaHostAlloc, cached per context
void pinned_free(pb200_ctx* ctx, void* p, size_t bytes);
cudaStream_t take_stream(pb200_ctx* ctx);
void give_stream(pb200_ctx* ctx, cudaStream_t s);
cudaEvent_t take_event(pb200_ctx* ctx);
void give_event(pb200_ctx* ctx, cudaEvent_t e);

struct DevBufRaw {  // RAII pooled device buffer
  pb200_ctx* ctx;
  void* p = nullptr;
  explicit DevBufRaw(pb200_ctx* c) : ctx(c) {}
  DevBufRaw(const DevBufRaw&) = delete;
  DevBufRaw& operator=(const DevBufRaw&) = delete;
  ~DevBufRaw() { dev_free(ctx, p); }
  int alloc(size_t bytes) { return dev_alloc(ctx, bytes, &p); }
};
// pb200_extract.cu: non-empty groups of the results' device tables -> final layout in pinned memory (all results at once)
int extract_groups(pb200_ctx* ctx, pb200_result* const* results, int nres, cudaStream_t st);
void result_materialize(pb200_result* R);  // view -> the std::vector fields
// pb200_order_by checks shared by the device and host entry points: PB200_OK or PB200_E_INVALID (message set)
int order_validate(const pb200_order_by* order, int num_aggs, int num_group_by);
// Orders and trims a host-built group-by result (rows in its std::vector fields or view) by `order`; fns = PB200_AGG_* per
// aggregation.  Same keys as the device sort (pb200_order.h); the result's rows end up in its std::vector fields.
void order_rows_host(pb200_result* R, const pb200_order_by& order, const int32_t* fns);

// pb200_roaring.cu
// One serialized RoaringBitmap (posting list of one dictId) to be OR-ed into `mask` (1 bit per doc, bit j of 32-bit
// word w = doc 32*w + j; zeroed by the caller).
struct DecodeJob {
  const unsigned char* inv;     // device: inverted index file bytes
  unsigned long long offset;    // byte offset of the bitmap inside the file
  unsigned long long length;
  uint32_t* mask;
  long long num_docs;
};
int roaring_decode_batch(pb200_ctx* ctx, cudaStream_t stream, const std::vector<DecodeJob>& jobs, void* jobs_dev);
// pb200_domain.cu
uint64_t dictionary_hash(int stored_type, int entry_bytes, int cardinality, const unsigned char* be);
int bits_for_cardinality(int card);
// pb200_synth.cu
int synth_build_inverted(pb200_ctx* ctx, cudaStream_t stream, DeviceColumn& col, long long num_docs);
}  // namespace pb200
