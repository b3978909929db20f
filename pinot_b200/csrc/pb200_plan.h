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
  std::vector<long long> in_filter;                   // per result: num_entries_scanned_in_filter
  int projected = 0;                                  // num_entries_scanned_post_filter = matched docs x this
};

// PB200_OK, or the PB200_E_* code of pb200_execute for this input (message set with set_error).
int plan_scan(const Tuning& tune, DeviceLimits lim, const pb200_query* query, pb200_segment* const* segments, int nseg,
              bool allow_count_carrier, ScanPlan* out);

// DictionaryBasedGroupKeyGenerator's key-holder regime for these group-by cardinalities (informational)
int regime_of(const std::vector<int>& cards, int array_threshold);

// The TMA table of chunk `c` (device pointers as bound into plan.segs).
TmaTable tma_table(const ScanPlan& plan, const LaunchChunk& c);

}  // namespace pb200
