// pb200_plan.h -- scan-launch planning: every decision pb200_execute takes before it touches the device.
//
// plan_scan() validates a query against the segments it runs on and chooses the launch: slots, the filter program, the
// kernel geometry (warps, CTAs per SM, ring stages, shared-memory layout, variant), the count carrier, the shared-memory
// group table, the per-segment descriptors, the result tables' layout and the launch chunks.  It calls nothing from the
// CUDA runtime and never dereferences a device pointer (segment-resident ones are copied into the descriptors), so the
// whole decision can be checked on a machine without a GPU (tests/test_scan_plan_cpu.py).  pb200_api.cu then allocates
// what the plan lists, fills the device pointers in and launches.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

#include "pb200_internal.h"
#include "pb200_scan_launch.h"

namespace pb200 {

struct DeviceLimits {
  int sm_count = 0;
  int max_smem_optin = 0;  // cudaDeviceProp::sharedMemPerBlockOptin
};

// Count carrier of one result: aggregation `agg`'s int64 table holds  sum(value - vmin) + count << shift  (agg -1: none)
struct Carrier { int agg = -1; int shift = 0; long long vmin = 0; };

// A device buffer one filter leaf needs; the executor allocates it and points segs[seg].leaves[leaf] at it.
struct LeafBuffer {
  enum Kind { LUT, INV_MASK, DOC_MASK, DOC_RANGES } kind;
  int seg = 0, leaf = 0;
  size_t words = 0;                 // 32-bit words to allocate
  std::vector<uint32_t> lut;        // LUT: the whole contents
  const void* src = nullptr;        // DOC_MASK / DOC_RANGES: the caller's host words, copied in ...
  size_t src_words = 0;             // ... this many; the rest of a doc mask is zeroed
  std::vector<DecodeJob> jobs;      // INV_MASK (zeroed): posting lists OR-ed into it; `mask` is filled in by the executor
};

// Layout of one group-by result's device tables (pb200_result::Dense).  Each aggregation's table is the index[a]-th
// `groups`-entry array of its block: SUM / AVG in the i64 or f64 block (sum_in_double), MIN in u32min, MAX in u32max.
struct TableLayout {
  std::vector<int> cards;
  std::vector<uint32_t> mult;
  std::vector<unsigned long long> mult64;
  bool hashed = false;              // hash table of `groups` (power of two) slots over the 64-bit raw key
  long long groups = 0;             // table entries: dense key space x stride, or the hash capacity
  int stride = 1;
  bool need_count = false;          // i64 block starts with the per-group count
  bool need_seen = false;           // u32max block starts with group-exists flags
  int exists_min = -1, exists_max = -1;  // a dictionary MIN / MAX table that marks the groups that exist
  Carrier carrier;
  int reduce_world = 1;
  bool flag_slot = false;
  int tail_slots = 0;
  long long i64_elems = 0, f64_elems = 0, u32max_elems = 0, u32min_elems = 0;
  int index[kMaxAggs] = {};
  uint32_t dwords[kMaxAggs] = {};   // DISTINCTCOUNT: bitset words per group
  uint32_t hist_per_group[kMaxAggs] = {};  // PERCENTILE (the histogram's owner, ScanPlan::pct_rep): entries per group
};

// One kernel launch: segments [first_seg, first_seg + num_segs), their tiles numbered from 0
struct LaunchChunk { int first_seg = 0, num_segs = 0; int total_tiles = 0; int grid = 0; };

struct ScanPlan {
  QueryDesc q{};                    // the launch's query descriptor (num_segments / total_tiles: per chunk)
  std::vector<SegDesc> segs;        // host parts filled in; device buffers are bound by the executor
  std::vector<int> slot_cols;       // slot -> column id
  std::vector<int> leaf_node;       // leaf -> index in the postfix node list
  bool group_by = false, merge = false, defer_finalize = false;
  int nres = 0;
  int warps = 0, ctas_per_sm = 0;
  bool skip_masks = false;          // the TMA table lists top-level doc masks for slice skipping
  size_t smem_bytes = 0;
  ScanVariant variant{};
  std::vector<LaunchChunk> chunks;
  std::vector<LeafBuffer> leaf_buffers;
  std::vector<TableLayout> tables;                    // group-by: one per result
  std::vector<std::vector<size_t>> distinct_words;    // aggregation only: [result][agg] DISTINCTCOUNT bitset words (0: none)
  // PERCENTILE: percentile of aggregation a (NaN: not a PERCENTILE) and the aggregation whose histogram it reads -- the
  // first PERCENTILE of its column, the only one with an agg code (-1: not a PERCENTILE)
  std::vector<double> pct_p;
  std::vector<int> pct_rep;
  // VAR / STDDEV (pb200_moments.h): the caller's aggregations come first, then three internal INT-dictionary SUMs per
  // column (K, H, L limbs) -- q.num_aggs and every per-aggregation array count them all
  int num_user_aggs = 0;
  std::vector<pb200_agg> aggs;                        // the launch's aggregations, internal ones included
  std::vector<int> mom_first;                         // [user agg] the first of its column's limb sums (-1: not VAR / STDDEV)
  std::vector<int> limb;                              // [agg] 0 / 1 / 2 for the K / H / L limb sums, else -1
  std::vector<std::vector<size_t>> hist_entries;      // aggregation only: [result][agg] histogram entries of an owner (0: none)
  long long hist_total = 0;                           // histogram entries of all results of the call
  std::vector<long long> in_filter;                   // per result: num_entries_scanned_in_filter
  int projected = 0;                                  // num_entries_scanned_post_filter = matched docs x this
};

// PB200_OK, or the PB200_E_* code of pb200_execute_args for this input (message set with set_error).  agg_args: one per
// aggregation, the percentile of a PERCENTILE (NULL: PERCENTILE is refused, as pb200_execute does).
constexpr long long kMaxHistogramEntries = 1ll << 28;  // PERCENTILE histogram entries of one call (u32 each)
// Aggregation-only PERCENTILE over at most this many dictIds: each warp counts into a private histogram in its own
// accumulator slots in shared memory (32 threads x 8 bytes = 64 u32 bins), flushed once per segment, instead of one
// same-address L2 reduction per row (DESIGN.md section 3.7 has the measurements)
constexpr int kHistWarpPrivateMaxCard = 64;
int plan_scan(const Tuning& tune, DeviceLimits lim, const pb200_query* query, pb200_segment* const* segments, int nseg,
              bool allow_count_carrier, ScanPlan* out, const double* agg_args = nullptr);

// ---- selection (pb200_execute_selection): plan_scan with COUNT(*) as the only aggregation, plus the match mask ----
constexpr long long kSelectPrefixRows = 1ll << 20;  // first pass of a selection without ORDER BY: at least this many docs
constexpr int kMaxSelectSegments = 65535;           // segments of one selection submission (gridDim.y of the select phase)
// how a selected column's value is produced at a doc (pb200_select.cu gather)
enum : int32_t { SEL_DICT_I32 = 0, SEL_DICT_I64 = 1, SEL_DICT_F32 = 2, SEL_DICT_F64 = 3, SEL_DICT_ID = 4, SEL_RAW_I32 = 5,
                 SEL_RAW_F32 = 6 };
inline bool selection_kind_is_double(int k) { return k == SEL_DICT_F32 || k == SEL_DICT_F64 || k == SEL_RAW_F32; }

struct SelectionPlan {
  ScanPlan scan;                          // the launch; segments keep their submission order and results are per segment
  std::vector<int> columns;               // selected column ids
  std::vector<int> kinds;                 // SEL_* per selected column (the same in every segment)
  std::vector<int> order_cols, order_kinds;  // ORDER BY items: column id, SEL_* kind
  std::vector<bool> order_desc;
  long long limit = 0;
  // Launch-wide match mask: doc d of segment s is bit d % 32 of word mask_word_off[s] + d / 32 (bit j of word w = doc
  // 32w + j inside the segment, the PB200_F_DOC_MASK layout).  Chunk c's launch writes from word chunk_word_off[c] on.
  std::vector<long long> mask_word_off;
  std::vector<long long> chunk_word_off;
  long long mask_words = 0;
  std::vector<long long> scan_docs;       // per segment: docs [0, scan_docs) scanned (a prefix, or num_docs)
  bool prefix = false;                    // some segment is scanned over a prefix only
};

// prefix: scan each segment over its first max(kSelectPrefixRows, 2 x limit) docs rounded up to whole tiles (selection
// without ORDER BY: the first `limit` matches are usually there; with ORDER BY every doc is scanned).  PB200_OK or the PB200_E_* code of
// pb200_execute_selection for this input.  No CUDA runtime call.
int plan_selection(const Tuning& tune, DeviceLimits lim, const pb200_query* filter_only, const pb200_selection* sel,
                   pb200_segment* const* segments, int nseg, bool prefix, SelectionPlan* out);
// Segments a prefix pass must scan again over all their docs: prefix shorter than the segment and fewer than `limit`
// matches in it (matches[s] = matched docs of segment s in the prefix).
std::vector<int> selection_rescan(const SelectionPlan& p, pb200_segment* const* segments, const std::vector<long long>& matches);
// A full pass over segments `rescan` (selection or DISTINCT): the filter-only query `q` with a per-segment filter cut
// down to those segments' trees (held in `filter`), and the segments in the same order.
struct Rescan { pb200_query query; std::vector<pb200_segment*> segs; std::vector<pb200_filter_node> filter; };
Rescan rescan_query(const pb200_query& q, pb200_segment* const* segments, const std::vector<int>& rescan);

// ---- DISTINCT (pb200_execute_distinct): a selection scan, then a dense first-occurrence table per result ----
constexpr int kMaxDistinctColumns = 8;                 // the group-by limit
constexpr long long kMaxDistinctKeys = 1ll << 24;      // raw key space of one result's table
constexpr long long kMaxDistinctEntries = 1ll << 27;   // table entries of all results of one call
constexpr unsigned long long kDistinctEmpty = ~0ull;   // table entry without a match; else segment << 32 | doc

struct DistinctPlan {
  SelectionPlan sel;                      // the scan: columns = the DISTINCT columns, order items as given
  int nres = 0;
  // [segment][key column]: cardinality and multiplier, raw key = sum_k dictId_k x mult_k, mult_k = prod_{j<k} card_j
  // (merged: the same in every segment, their dictionaries are one)
  std::vector<std::vector<int>> cards;
  std::vector<std::vector<uint32_t>> mult;
  std::vector<long long> table_off, table_size;   // per result: first entry in the call's table block, entries
  long long table_entries = 0;
  std::vector<int> order_key;             // per order item kept: index of its column among the key columns
  std::vector<bool> order_desc;           // (an item repeating an earlier item's column is dropped: it orders nothing)
};

// PB200_OK or the PB200_E_* code of pb200_execute_distinct for this input (refusals: see include/pinot_b200.h).  merge:
// one result over all segments.  prefix as for plan_selection (ignored with order items).  No CUDA runtime call.
int plan_distinct(const Tuning& tune, DeviceLimits lim, const pb200_query* filter_only, const pb200_selection* distinct,
                  pb200_segment* const* segments, int nseg, bool merge, bool prefix, DistinctPlan* out);
// The prefix-final rule.  bound[r]: (segment << 32 | prefix end) of the earliest segment of result r whose scan was cut
// short, kDistinctEmpty when none was.  Every position before the bound has been scanned, so result r is final when at
// least `limit` of its table's entries lie below it (below[r]).  Returns the truncated segments of every result that is
// not final, to be scanned again in full into the same tables.
std::vector<unsigned long long> distinct_bounds(const DistinctPlan& p, pb200_segment* const* segments);
std::vector<int> distinct_rescan(const DistinctPlan& p, pb200_segment* const* segments, const std::vector<long long>& below);

// PB200_Q_MERGE_SEGMENTS over dictIds: true when column `col` has the same dictionary in every segment; otherwise sets
// the error ("`what` column ... bind the segments to a pb200_domain first") and returns false.
bool same_dictionary(pb200_segment* const* segments, int nseg, int col, const char* what);

// DictionaryBasedGroupKeyGenerator's key-holder regime for these group-by cardinalities (informational)
int regime_of(const std::vector<int>& cards, int array_threshold);

// The TMA table of chunk `c` (device pointers as bound into plan.segs).
TmaTable tma_table(const ScanPlan& plan, const LaunchChunk& c);

// pb200_api.cu: allocates and fills the device buffers plan.leaf_buffers lists on `st` and points the leaf descriptors of
// plan.segs at them; the buffers stay in `temps` until the launch that reads them is done.
int bind_leaf_buffers(pb200_ctx* ctx, ScanPlan& plan, cudaStream_t st, std::vector<std::unique_ptr<DevBufRaw>>& temps);

// pb200_select.cu: one scan launch of a selection plan on `st`: fills `mask` (p.mask_words words) and the matched docs of
// each segment, adds the scan's CUDA-event time to *ms; ends in a stream synchronisation.
int run_selection_scan(pb200_ctx* ctx, cudaStream_t st, SelectionPlan& p, DevBufRaw& mask, std::vector<long long>& matches,
                       float* ms);

}  // namespace pb200
