// pb200_internal.h -- host-side objects behind the opaque C-ABI handles.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/pinot_b200.h"
#include "pb200_desc.h"
#include "pb200_distinct_sum.h"
#include "pb200_hll.h"
#include "pb200_moments.h"

namespace pb200 {

void set_error(const char* fmt, ...);
// pb200_last_phases of the calling thread: one phase's host wall-clock (PB200_PHASE_*), and the clock it is read from
void set_phase_ms(int phase, double ms);
double host_ms();
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

// Facts of one device dictionary that queries derive once: the DISTINCTSUM / DISTINCTAVG grid (ds_state below), and
// the limb dictionaries for VAR / STDDEV (pb200_moments.h, pb200_moments.cu): built on the first
// query that needs them, under `mu`, and published with `ready` (release) before any launch reads them.  Shared by the
// columns that share the dictionary (a domain's bound segments); freed with the last of them.
struct MomentDict {
  std::mutex mu;
  std::atomic<bool> ready{false};  // evaluated: `eligible`, `grid` and (eligible) `limbs` are final
  bool eligible = false;
  MomentGrid grid{};
  pb200_ctx* ctx = nullptr;
  uint32_t* limbs = nullptr;       // device: K, H, L arrays of `entries` u32 each, one allocation
  int entries = 0;
  // DISTINCTSUM / DISTINCTAVG eligibility of the same dictionary (pb200_distinct_sum.h distinct_grid): evaluated on the
  // host copy by the first query that needs it, under `mu`; 0 not yet, 1 eligible with exponent ds_e, -1 not eligible
  std::atomic<int> ds_state{0};
  int ds_e = 0;
  // DISTINCTCOUNTHLL (pb200_hll.h): the 32-bit MurmurHash of every entry of the same dictionary (device, 4 bytes per
  // entry), built by the first query that needs it (pb200_hll.cu hll_prepare), under `mu`; 0 not yet, 1 built, -1 a
  // STRING entry that is not valid UTF-8 (the reference would hash U+FFFD's bytes: not accelerated)
  std::atomic<int> hll_state{0};
  uint32_t* hll_hash = nullptr;
  ~MomentDict();                   // pb200_moments.cu
};

// Compact device copy of a STRING dictionary for REGEXP_LIKE (pb200_pattern.cu): the entries of the segment's OWN
// dictionary (also once the column is bound to a domain) without their zero padding, `entries + 1` u32 offsets followed by
// the bytes, in one allocation.  Built on the first pattern query, under `mu`, and published with `ready` (release).
struct StringDict {
  std::mutex mu;
  std::atomic<bool> ready{false};
  pb200_ctx* ctx = nullptr;
  void* block = nullptr;
  const uint32_t* offsets = nullptr;
  const unsigned char* bytes = nullptr;
  uint32_t entries = 0;
  ~StringDict();                   // pb200_pattern.cu
};

struct DeviceColumn {
  int fwd_kind = 0, stored_type = 0, bits = 0, cardinality = 0;
  std::shared_ptr<MomentDict> moments = std::make_shared<MomentDict>();  // replaced by the domain's when bound
  std::shared_ptr<StringDict> strings = std::make_shared<StringDict>();  // STRING columns; stays the segment's when bound
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
  int spec = 1;                  // !PB200_NO_SPEC: the group-by kernel specialised for the shared-table shape when it qualifies
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
    std::shared_ptr<pb200::MomentDict> moments = std::make_shared<pb200::MomentDict>();  // shared by every bound segment
  };
  std::vector<Col> cols;
  int refs = 1;  // the creator + one per bound segment (guarded by ctx->mu)
};

struct pb200_segment {
  pb200_ctx* ctx = nullptr;
  std::string name;
  int num_docs = 0;
  // Registered columns, then derived ones (pb200_transform.cu).  Registration reserves room for
  // PB200_MAX_DERIVED_COLUMNS more, so appending a derived column (under derive_mu) never moves a column that a
  // running query references.  Readers bound their column ids by num_columns(), never by cols.size(): the count is
  // published with release only after the appended column is complete.
  std::vector<pb200::DeviceColumn> cols;
  int num_stored = 0;              // registered columns: segments of one table agree on these
  std::atomic<int> published{-1};  // columns queries may read; -1: a column list that never grows (cols.size())
  std::mutex derive_mu;
  int num_columns() const { const int p = published.load(std::memory_order_acquire); return p < 0 ? (int)cols.size() : p; }
  int64_t device_bytes = 0;
  pb200_domain* domain = nullptr;  // holds one reference
};

namespace pb200 {
// Columns every segment of a submission has (derived columns may have been added to some segments only); -1 when the
// segments do not share their registered columns
inline int common_columns(pb200_segment* const* segments, int nseg) {
  int n = segments[0]->num_columns();
  for (int s = 0; s < nseg; s++) {
    if (!segments[s] || segments[s]->num_stored != segments[0]->num_stored) return -1;
    n = std::min(n, segments[s]->num_columns());
  }
  return n;
}
}  // namespace pb200

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
  // Selection result (pb200_select.cu): rows in a pinned block shared by the results of one submission
  struct Selection {
    bool present = false;
    std::shared_ptr<pb200::PinnedBlock> block;
    int64_t rows = 0;
    int32_t* doc_ids = nullptr;
    int32_t* segment_index = nullptr;
    std::vector<const void*> columns;            // int64 or double [rows] each
  } selection;
  // PERCENTILE (pb200_percentile.cu): the histograms stay on the device until pb200_result_histogram copies them
  struct Pct {
    Pct() { std::fill(rep, rep + pb200::kMaxAggs, -1); }
    pb200_ctx* ctx = nullptr;
    int rep[pb200::kMaxAggs];                    // aggregation -> owner of its histogram (-1: not a PERCENTILE)
    uint32_t* hist[pb200::kMaxAggs] = {};        // owners: device histogram, one row per result row / table entry
    uint32_t entries[pb200::kMaxAggs] = {};      // owners: entries per row
    uint32_t* ids[pb200::kMaxAggs] = {};         // group-by: selected dictId per table entry (device, ~0: no row)
    uint32_t* n[pb200::kMaxAggs] = {};           // group-by, owners: values per table entry (device)
    const uint32_t* row_entry = nullptr;         // group-by: table entry of each extracted row (inside view.block)
    std::vector<uint32_t> host[pb200::kMaxAggs]; // owners: histogram rows of the result's rows, copied on first use
  } pct;
  // FIRST/LASTWITHTIME with GROUP BY (pb200_withtime.cu): per table entry the winning key, then the data dictId (~0: no
  // row) and the time value the finalize decoded from it; allocated with the dense tables and freed with them
  struct Wt {
    unsigned long long* key[pb200::kMaxAggs] = {};
    uint32_t* ids[pb200::kMaxAggs] = {};
    long long* time[pb200::kMaxAggs] = {};
  } wt;
  // VAR / STDDEV (pb200_moments.h): the grid of each such aggregation's dictionary and its exact moments per row
  struct Mom {
    Mom() { for (int a = 0; a < pb200::kMaxAggs; a++) rows[a] = one[a]; }
    bool on[pb200::kMaxAggs] = {};
    pb200::MomentGrid grid[pb200::kMaxAggs] = {};
    const unsigned long long* rows[pb200::kMaxAggs];      // {s1, s2 low, s2 high} per row: `one`, or (group-by) in view.block
    unsigned long long one[pb200::kMaxAggs][3] = {};       // aggregation only: the one row's
  } mom;
  // aggregation only: the exact int64 sum behind an INT SUM / AVG (the double column holds it rounded), so that a
  // cross-GPU combine adds exact sums and rounds once (pb200_result_exact_sum, pb200_comm.cu: combine_scalars)
  struct ExactSum {
    bool on[pb200::kMaxAggs] = {};
    long long sum[pb200::kMaxAggs] = {};
  } exact;
  // DISTINCTCOUNTHLL sets that nothing else in the query reads: the result rows' bitset rows stay on the device
  // (rows x words u32, owned per bitset b) and pb200_result_distinct decodes them into `distinct` on its first call for an
  // aggregation a with src[a] = b -- a caller that reads only the estimates never pays for the decode
  struct LazySets {
    LazySets() { std::fill(src, src + pb200::kMaxAggs, -1); }
    pb200_ctx* ctx = nullptr;
    std::mutex mu;
    int src[pb200::kMaxAggs];
    uint32_t* bits[pb200::kMaxAggs] = {};
    size_t words[pb200::kMaxAggs] = {};
    size_t rows[pb200::kMaxAggs] = {};
  } lazy;
  pb200_order_by order{};                      // ORDER BY spec of a group-by result (num_items 0: none), applied at extraction
  pb200_having having{};                       // HAVING of a group-by result (num_nodes 0: none), applied at extraction before
                                               // the order; set on every result whose rows it filtered
  pb200_post_aggs post{};                      // the programs PB200_ORDER_POST items of `order` name (num_programs 0: none)
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
    int mom_first[pb200::kMaxAggs];             // VAR / STDDEV: the first of the three limb sums (isum) of aggregation a, -1 if none
    int mom_e[pb200::kMaxAggs] = {};            // ... and the grid exponent of its column
    Dense() {
      std::fill(mom_first, mom_first + pb200::kMaxAggs, -1);
      std::fill(ds_rep, ds_rep + pb200::kMaxAggs, -1);
      std::fill(hll_rep, hll_rep + pb200::kMaxAggs, -1);
    }
    uint32_t* dbits[pb200::kMaxAggs] = {};      // DISTINCTCOUNT with GROUP BY: per-group dictId bitsets, dwords[a] words each
    uint32_t dwords[pb200::kMaxAggs] = {};
    // DISTINCTSUM / DISTINCTAVG (pb200_distinct_sum.h): the aggregation b whose bitset holds the set (-1: neither
    // function); indexed by b, the set's finalized state per table entry (kDsWords u64 each, device), shared by every
    // function that reads the set
    int ds_rep[pb200::kMaxAggs];
    unsigned long long* ds_state[pb200::kMaxAggs] = {};
    // DISTINCTCOUNTHLL (pb200_hll.h): log2m of aggregation a (0: not one); indexed by the first HLL of a column and log2m
    // (ScanPlan::hll_rep), the estimate per table entry (int64, device), shared by the HLLs with that column and log2m
    int hll_log2m[pb200::kMaxAggs] = {};
    int hll_rep[pb200::kMaxAggs];
    long long* hll_est[pb200::kMaxAggs] = {};
    // expression aggregations (pb200_expr.cu): per aggregation its own table, f64 sums (also pointed to by dsum) or u64
    // Double.compare keys of MIN / MAX; NULL: not an expression
    void* expr_tab[pb200::kMaxAggs] = {};
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
struct StreamLease {  // RAII stream of the context's pool; converts to the stream
  pb200_ctx* ctx;
  cudaStream_t s;
  explicit StreamLease(pb200_ctx* c) : ctx(c), s(take_stream(c)) {}
  StreamLease(const StreamLease&) = delete;
  StreamLease& operator=(const StreamLease&) = delete;
  ~StreamLease() { give_stream(ctx, s); }
  operator cudaStream_t() const { return s; }
};
struct EventPair {  // two pooled events around queued work (creating / destroying them per query costs more than a launch)
  pb200_ctx* ctx;
  cudaEvent_t a = nullptr, b = nullptr;
  explicit EventPair(pb200_ctx* c) : ctx(c) {}
  EventPair(const EventPair&) = delete;
  EventPair& operator=(const EventPair&) = delete;
  ~EventPair() { give_event(ctx, a); give_event(ctx, b); }
  int take() {
    a = take_event(ctx);
    b = take_event(ctx);
    if (!a || !b) { set_error("cudaEventCreate failed"); return PB200_E_CUDA; }
    return PB200_OK;
  }
  float ms() const { float t = 0.f; cudaEventElapsedTime(&t, a, b); return t; }
};
// grid of a grid-stride kernel over `items`: one thread per item, at most 8 blocks per SM
inline int grid_for(const pb200_ctx* ctx, long long items, int threads) {
  return (int)std::max<long long>(1, std::min<long long>((items + threads - 1) / threads, (long long)ctx->sm_count * 8));
}
// dictIds of the set bits of a DISTINCTCOUNT bitset (bit j of word w = dictId 32w + j), ascending
std::vector<int32_t> bitset_ids(const uint32_t* bits, size_t words);
// pb200_extract.cu: non-empty groups of the results' device tables -> final layout in pinned memory (all results at once)
int extract_groups(pb200_ctx* ctx, pb200_result* const* results, int nres, cudaStream_t st);
struct AggSource;   // pb200_decode.h
// The decoder's sources of a GROUP BY result's aggregations (out: one per aggregation), over its device tables.
void agg_sources(const pb200_result& R, AggSource* out);
// DISTINCTSUM / DISTINCTAVG states and DISTINCTCOUNTHLL estimates of one result's sets, queued on `st`: the `rows` rows of
// set b (bits[b], words[b] u32 per row; b the aggregation whose bitset holds the set) into the tables of `src`, once per
// set and once per column and log2m.  d: the result's aggregations.  single: the one row of an aggregation-only result.
int finalize_sets(pb200_ctx* ctx, cudaStream_t st, const pb200_result::Dense& d, const uint32_t* const* bits, const size_t* words,
                  long long rows, bool single, const AggSource* src, std::vector<std::unique_ptr<DevBufRaw>>& temps);
// The value sets of R's `rows` rows: DISTINCTCOUNT's, and those DISTINCTSUM / DISTINCTAVG / DISTINCTCOUNTHLL read, decoded
// once per set from its rows on the device (sets[b], words[b] u32 per row).  DISTINCTCOUNT's set sizes go to dbl[a] /
// lng[a].  A set only DISTINCTCOUNTHLLs read is not decoded: R takes its device rows for pb200_result_distinct to decode
// on first use (sets[b] gives them up; *kept is set when rows are still being written on `st`).
int decode_sets(pb200_ctx* ctx, cudaStream_t st, pb200_result* R, DevBufRaw* const* sets, const size_t* words, size_t rows,
                double* const* dbl, int64_t* const* lng, bool* kept);
void result_materialize(pb200_result* R);  // view -> the std::vector fields
// pb200_execute_exprs (exprs NULL: no expression aggregations) whose ORDER BY may name the post-aggregation programs of
// pb200_execute_post (post NULL: none); both NULL is pb200_execute_agg_args.  The host layer's one device entry point.
// conds: the CASE WHEN conditions of the programs (pb200_execute_exprs_cond; NULL: none).
int execute_exprs_post(pb200_ctx* ctx, const pb200_query* query, const pb200_order_by* order, const pb200_agg_arg* args,
                       const pb200_having* having, const pb200_expr_program* exprs, const pb200_expr_conds* conds,
                       const pb200_post_aggs* post, pb200_segment* const* segments, int32_t nseg, pb200_result** results);
// pb200_order_by checks shared by the device and host entry points, with the post-aggregation programs its
// PB200_ORDER_POST items may name (post NULL: none): PB200_OK or PB200_E_INVALID (message set)
int order_validate(const pb200_order_by* order, int num_aggs, int num_group_by, const pb200_post_aggs* post = nullptr);
// Orders and trims a host-built group-by result (rows in its std::vector fields or view) by `order`; fns = PB200_AGG_* per
// aggregation, post = the programs of its PB200_ORDER_POST items (NULL: none).  Same keys as the device sort (pb200_order.h,
// pb200_postagg.h); the result's rows end up in its std::vector fields.
void order_rows_host(pb200_result* R, const pb200_order_by& order, const int32_t* fns, const pb200_post_aggs* post = nullptr);
// pb200_having checks of the device and host entry points (having may be NULL): PB200_OK, or PB200_E_INVALID /
// PB200_E_UNSUPPORTED (message set).  nres = results the call writes, deferred = PB200_Q_DEFER_FINALIZE or reduce_world > 1.
int having_check(const pb200_having* having, int num_aggs, int num_group_by, int nres, bool deferred);
// Keeps the rows of a host-built group-by result that pass `having` (pb200_having.h, fns = PB200_AGG_* per aggregation)
// and marks the result as filtered; the kept rows end up in its std::vector fields, in their order.
void having_rows_host(pb200_result* R, const pb200_having& having, const int32_t* fns);

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
uint64_t padded_fwd_bytes(long long num_docs, int bits);  // allocation of a forward index (whole max tiles + slack)
// Launches the re-encode of a fixed-bit column on `st`: value v of `src` (sb bits, card values) becomes remap[v] in `dst`
// (db bits, zeroed by the caller); padding rows stay 0.
cudaError_t reencode_column(pb200_ctx* ctx, cudaStream_t st, const uint32_t* src, int sb, uint32_t* dst, int db,
                            const uint32_t* remap, uint32_t card, long long num_docs);
// pb200_moments.cu: builds (once per device dictionary) the limb dictionaries of every VAR / STDDEV column of the query
// that has dictIds, before it is planned; columns the planner refuses are skipped
int moments_prepare(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments, int nseg);
// pb200_distinct_sum.cu: DISTINCTSUM / DISTINCTAVG states (kDsWords u64 per row, pb200_distinct_sum.h) of `rows` bitset
// rows of `words` words each, queued on `st`.  single: one row of an aggregation-only result (a grid-wide pass; its
// scratch goes to `temps`).
struct DistinctSumJob {
  const uint32_t* bits;
  size_t words;
  long long rows;
  bool single;
  const void* dict;           // the column's device dictionary (INT: biased)
  int stored_type, e;
  unsigned long long* out;
};
int distinct_sum_finalize(pb200_ctx* ctx, cudaStream_t st, const DistinctSumJob& job, std::vector<std::unique_ptr<DevBufRaw>>& temps);
// pb200_hll.cu: builds (once per device dictionary) the hash array of every DISTINCTCOUNTHLL column of the query that has
// dictIds, before it is planned; PB200_E_UNSUPPORTED for a STRING dictionary with an entry that is not valid UTF-8
int hll_prepare(pb200_ctx* ctx, const pb200_query* query, pb200_segment* const* segments, int nseg);
// DISTINCTCOUNTHLL estimates (int64 per row) of `rows` bitset rows of `words` words each, queued on `st`.  single: one row
// of an aggregation-only result (a grid-wide pass; its scratch goes to `temps`).
struct HllJob {
  const uint32_t* bits;
  size_t words;
  long long rows;
  bool single;
  const uint32_t* hash;       // the column's hash array (MomentDict::hll_hash)
  int log2m;
  long long* out;
};
int hll_finalize(pb200_ctx* ctx, cudaStream_t st, const HllJob& job, std::vector<std::unique_ptr<DevBufRaw>>& temps);
// pb200_hll.cu: the DISTINCTCOUNTHLL estimate over every value of column `column` in the segment (the host layer's answer
// without a scan for a filter that matches every doc), computed by the finalize; synchronous
int hll_whole_dictionary(pb200_ctx* ctx, pb200_segment* seg, int column, int log2m, long long* out);
// pb200_hll.cu: the dictId set of pb200_result_distinct for aggregation a of R, decoding a lazily kept set first
const std::vector<std::vector<int32_t>>* result_sets(pb200_result* R, int a);
// pb200_synth.cu
int synth_build_inverted(pb200_ctx* ctx, cudaStream_t stream, DeviceColumn& col, long long num_docs);
}  // namespace pb200
