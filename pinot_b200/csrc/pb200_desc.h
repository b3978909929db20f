// pb200_desc.h -- launch descriptors shared by the host planner (pb200_plan.cpp), the launch (pb200_api.cu) and the scan kernels.
#pragma once
#include <cstdint>

namespace pb200 {

constexpr int kMaxSlots = 12;    // distinct columns one query may touch on the device
constexpr int kMaxLeaves = 8;    // filter leaves
constexpr int kMaxNodes = 16;    // filter tree nodes (postfix program length)
constexpr int kMaxAggs = 6;      // aggregation functions per query
constexpr int kMaxGroupBy = 8;   // group-by columns (dense table or 64-bit-key hash table)
constexpr int kRowsPerThread = 32;
constexpr int kMaxStack = 8;

// slot roles
enum : uint32_t { ROLE_FILTER = 1, ROLE_GROUP = 2, ROLE_AGG = 4 };

// device leaf kinds
enum : int32_t { LEAF_ALL = 0, LEAF_NONE = 1, LEAF_RANGE = 2, LEAF_LUT = 3, LEAF_DOCMASK = 4, LEAF_DOCRANGES = 5 };

// program ops (postfix over 32-row masks)
enum : uint8_t { OP_LEAF = 0, OP_AND = 1, OP_OR = 2, OP_NOT = 3 };

// LEAF_RANGE comparison shape (one-sided ranges need one compare per value instead of subtract + compare)
enum : int32_t { CMP_BOTH = 0, CMP_GE = 1, CMP_LT = 2 };

// aggregation value kinds (how a dictId / raw word becomes a number)
enum : int32_t { VAL_NONE = 0, VAL_DICT_I32 = 1, VAL_DICT_I64 = 2, VAL_DICT_F32 = 3, VAL_DICT_F64 = 4, VAL_RAW_I32 = 5 };

// SUM / AVG accumulate in double for FLOAT / DOUBLE and for LONG dictionaries -- what SumAggregationFunction does for every
// type (core/query/aggregation/function/SumAggregationFunction.java:69-145: `sum += values[i]` on a double).  A 64-bit
// integer accumulator over LONG values would wrap silently (epoch millis x 5 M rows > 2^63); INT values keep the exact
// int64 accumulator (|v| x rows < 2^31 x 2^31, cannot wrap).
__host__ __device__ constexpr bool sum_in_double(int vk) { return vk == VAL_DICT_F32 || vk == VAL_DICT_F64 || vk == VAL_DICT_I64; }

// MIN / MAX entries hold an order-preserving u32: the dictId, or for a raw INT column x = value ^ 0x80000000.  A MIN entry
// starts at 0xFFFFFFFF, a MAX entry at 0; MAX stores x + max_offset(vk).  DictIds are below 2^31, so dictId + 1 never
// wraps and 0 / 0xFFFFFFFF mean "no row".  A raw INT spans all of u32 (INT_MAX is 0xFFFFFFFF, INT_MIN is 0): its MAX is
// stored as x, and whether the group has a row at all comes from its count, seen flag, count carrier or hash key -- never
// from a raw MIN / MAX entry.
__host__ __device__ constexpr uint32_t max_offset(int vk) { return vk == VAL_RAW_I32 ? 0u : 1u; }

// PERCENTILE(col, p) over n > 0 sorted values (PercentileAggregationFunction.extractFinalResult): p == 100 selects the
// largest, otherwise index (int64)((double)n * p / 100.0) -- product, division, truncation, in that order -- clamped to
// n - 1 (rounding near p = 100 can reach n, where the reference would throw).
__host__ __device__ inline long long percentile_index(long long n, double p) {
  if (p == 100.0) return n - 1;
  const long long k = (long long)((double)n * p / 100.0);
  return k < n - 1 ? k : n - 1;
}

// FIRSTWITHTIME / LASTWITHTIME (DESIGN.md section 3.13) in SegDesc.agg_code: function field kFnWithTime over the TIME
// column's slot, the value-kind field says which end wins.  A row's key is (time dictId << 32) | row ordinal, the
// ordinal being the segment's doc base in the call plus the doc id: u64 max is the last row by (time, call order), u64
// min the first.  The key table is SegDesc.distinct_bits[a] (as u64: one per result, or one per group / slot) and the
// segment's doc base is SegDesc.distinct_words[a].
constexpr int kFnWithTime = 7;
enum : int32_t { WT_MAX = 0, WT_MIN = 1 };
__host__ __device__ constexpr unsigned long long withtime_key(uint32_t time_id, uint32_t ordinal) {
  return (unsigned long long)time_id << 32 | ordinal;
}

struct SlotDesc {
  const uint32_t* data;  // device: packed words, padded to whole tiles
  int32_t bits;          // 1..32 (32 = raw big-endian 32-bit values)
  uint32_t stage_words;  // offset of this slot inside a warp's stage buffer, in 32-bit words
  uint32_t tile_bytes;   // bytes of this slot per 1024-row warp slice: 128 * bits
  uint32_t pad;
};

// LeafDesc.code packs everything the tile loop needs to dispatch a leaf into ONE word (one LDS.128 then brings code,
// slot, lo and span): kind [0:3)  cmp [4:6)  negate [8]  bits of the slot [12:18)  stage_words of the slot [18:32)
__host__ __device__ constexpr uint32_t leaf_code(int kind, int cmp, int negate, int bits, uint32_t stage_words) {
  return (uint32_t)kind | (uint32_t)cmp << 4 | (uint32_t)(negate ? 1 : 0) << 8 | (uint32_t)bits << 12 | stage_words << 18;
}
// SegDesc.agg_code: one word per aggregation that reads a column (COUNT(*) never appears), the software-pipelined one
// LAST: index [0:3)  function [4:7)  value kind [8:11)  bits [12:18)  stage_words [18:32)
__host__ __device__ constexpr uint32_t agg_code(int a, int fn, int vk, int bits, uint32_t stage_words) {
  return (uint32_t)a | (uint32_t)fn << 4 | (uint32_t)vk << 8 | (uint32_t)bits << 12 | stage_words << 18;
}

struct alignas(16) LeafDesc {
  uint32_t code;    // leaf_code(...); kind = code & 7
  int32_t slot;
  uint32_t lo;      // RANGE: dictId lower bound
  uint32_t span;    // RANGE: hi - lo  (match iff (v - lo) < span, unsigned)
  const uint32_t* bits;  // LUT: bitmap over dictIds; DOCMASK: 1 bit per doc (bit j of word w = doc 32w+j)
  const int32_t* ranges; // DOCRANGES: inclusive (start,end) pairs
  int32_t num_ranges;
  int32_t negate;
  int32_t cmp;      // LEAF_RANGE: CMP_*
  int32_t kind;     // LEAF_* (host side; the kernel reads it from code)
};

// Per-aggregation outputs of the aggregation-only kernel (one per segment or one merged)
struct AggAccum {
  unsigned long long count;             // matched docs
  long long isum[kMaxAggs];             // exact integer sums (INT / LONG dictionaries)
  double dsum[kMaxAggs];                // FLOAT / DOUBLE sums
  uint32_t min_id[kMaxAggs];            // dictId (or order-preserving raw encoding); 0xFFFFFFFF = empty (raw: count == 0)
  uint32_t max_id_plus1[kMaxAggs];      // dictId + 1; 0 = empty (raw INT: the encoding itself, see max_offset)
};

struct SegDesc {
  long long num_docs;
  long long first_tile;   // index of this segment's first tile in the launch-wide tile sequence
  long long num_tiles;
  uint32_t stage_tx;      // bytes TMA delivers per warp slice for THIS segment (sum of its slots' tile_bytes)
  int32_t num_agg_codes;
  uint32_t agg_code[kMaxAggs];
  int32_t num_defer_codes;  // group-by: the LAST num_defer_codes entries of agg_code are software-pipelined (pb200_scan.cuh drain_gb)
  uint32_t pad1;
  SlotDesc slots[kMaxSlots];
  LeafDesc leaves[kMaxLeaves];
  const void* dict[kMaxAggs];          // native (little-endian) dictionary value array of the aggregation's column
  // per-group dictId tables, indexed by the aggregation (group-by: distinct_words[a] entries per group / slot):
  //   DISTINCTCOUNT: bitset over dictIds, distinct_words[a] = words per group;
  //   PERCENTILE:    u32 histogram of dictId counts, distinct_words[a] = entries per group (the column's cardinality);
  //                  aggregation only: 1 when the warps count into private shared-memory histograms first (at most
  //                  64 dictIds, in the aggregation's accumulator slots), else 0
  //   FIRST/LASTWITHTIME: u64 key table (kFnWithTime above), distinct_words[a] = the segment's doc base in the call
  uint32_t* distinct_bits[kMaxAggs];
  uint32_t distinct_words[kMaxAggs];
  AggAccum* accum;                     // aggregation-only output
  // dense group table (group-by): indexed by raw key = sum_j dictId_j * mult_j
  unsigned long long* g_count;   // per-group row count; NULL when no COUNT / AVG needs it
  uint32_t* g_seen;              // then: group-exists flags (NULL if a dictionary MIN/MAX table already tells)
  long long* g_isum[kMaxAggs];
  double* g_dsum[kMaxAggs];
  uint32_t* g_min[kMaxAggs];
  uint32_t* g_max[kMaxAggs];
  uint32_t group_mult[kMaxGroupBy];
  // hash group table (key spaces beyond the dense limit, the reference's LONG_MAP regime): open addressing over the
  // 64-bit raw key; the accumulator tables above are then indexed by SLOT instead of by raw key
  unsigned long long* h_keys;          // NULL = dense table; else capacity (h_mask + 1) keys, empty = ~0
  uint32_t* h_ctl;                     // [0] = inserted keys, [1] = overflow flag (more groups than h_limit, or table full)
  uint32_t h_mask;
  int32_t h_limit;
  unsigned long long group_mult64[kMaxGroupBy];
  // group-by SUM / AVG over an INT dictionary: the 64-bit value added to the table is (zero-extended biased dictionary
  // word) + sum_addend[a].  Plain sums: -2^31 (removes the bias).  The sum that CARRIES the row count of its group
  // (pb200_plan.cpp "count carrier"): 2^shift - biased(min value), i.e. one reduction adds (value - min) to the low `shift`
  // bits and 1 to the bits above them -- the separate COUNT reduction (an L2 read-modify-write per surviving row) is gone.
  unsigned long long sum_addend[kMaxAggs];
};

// Everything lane 0 needs to refill a warp's TMA ring, for every segment of the launch, passed BY VALUE as a kernel
// parameter so it sits in the constant bank (a global-memory descriptor read per tile costs an L2 round trip because
// the dictionary gathers keep evicting L1).
constexpr int kMaxLaunchSegs = 16;
constexpr int kMaxSkipMasks = 3;
struct TmaSlot {
  const void* data;
  uint32_t tile_bytes;
  uint32_t stage_words;
};
struct TmaSeg {
  int32_t first_tile;   // CTA-tile index (launch relative) of the segment's first tile
  int32_t end_tile;     // exclusive
  uint32_t stage_tx;
  uint32_t num_docs;
  // doc masks (1 bit per doc) that are top-level AND operands of the filter: a 1024-row slice whose mask words are all
  // zero is never loaded (the GPU analogue of iterating only the doc ids a bitmap index produced)
  const uint32_t* skip_mask[kMaxSkipMasks];
  TmaSlot slot[kMaxSlots];
};
struct TmaTable {
  TmaSeg seg[kMaxLaunchSegs];
};

struct AggDesc {
  int32_t function;  // PB200_AGG_*
  int32_t slot;      // -1 for COUNT(*)
  int32_t val_kind;  // VAL_*
  int32_t pad;
};

struct QueryDesc {
  int32_t num_segments;
  int32_t num_slots;
  int32_t num_leaves;
  int32_t num_nodes;       // program length; 0 = match all
  int32_t conj;            // 1: root is a flat AND (or single leaf) of leaves -> no stack
  int32_t sparse_max;      // per-row probing instead of unpacking when <= this many rows per thread survive
  int32_t sparse_max_agg;  // same decision for the projection / aggregation phase
  int32_t defer_agg;       // aggregation whose dictionary gathers are software-pipelined across tiles (-1: none)
  int32_t num_aggs;
  int32_t num_group_by;
  int32_t tile_rows;       // warps per CTA * 1024
  int32_t num_stages;
  uint32_t stage_words;    // words per WARP stage buffer: 32 * sum of bits (max over segments)
  uint32_t use_pipe;       // 0: no column is streamed (e.g. COUNT(*) over doc masks only)
  uint32_t slot_roles[kMaxSlots];
  int32_t group_slot[kMaxGroupBy];
  uint8_t prog_op[kMaxNodes];
  uint8_t prog_arg[kMaxNodes];  // OP_LEAF: leaf index; AND/OR: operand count
  AggDesc aggs[kMaxAggs];
  int32_t total_tiles;     // CTA tiles in this launch
  // CTA-private group table in shared memory (group-by with a small key space and COUNT / integer SUM only): rows
  // update it with native 32-bit shared atomics and it is merged into the global dense table once per segment.
  // Layout at byte offset smem_table_off: count u32[G] (when smem_count), then per summed aggregation lo u32[G],
  // hi u32[G].  A sum that carries its group's row count (SegDesc.sum_addend) needs no count array: with the carrier
  // admitted for every result of the launch an entry is 8 bytes, and the flushed table equals what global REDs build.
  int32_t smem_groups;     // 0 = off, else the size G of the dense key space (max over the launch's segments)
  uint32_t smem_table_off;
  // the table is replicated `smem_copies` (power of two) times, lane l updates copy l % copies: same-address conflicts
  // inside a warp (the norm for a handful of groups) drop by that factor; each array is smem_copies * smem_gstride words,
  // entry of (copy c, group g) at c * smem_gstride + g; smem_gstride is odd so that the copies start in different banks
  int32_t smem_copies;
  int32_t smem_gstride;
  // group-by survivor queue: u16[1024] per warp at byte offset queue_off; used when a warp slice has <= queue_max survivors
  uint32_t queue_off;
  int32_t queue_max;
  int8_t smem_slot[kMaxAggs];  // aggregation -> index of its (lo, hi) pair, -1: none (COUNT)
  int8_t smem_count;           // 1: the shared table has a count array
  int8_t smem_merged;          // 1: every segment of the launch adds into the same global table (flush at exit only)
  // Selection launches (pb200_select.cu): the launch-wide match mask, as two 32-bit halves (lo, hi) of the pointer because
  // the field is only 4-byte aligned.  Non-NULL: every thread stores its final 32-row mask at word
  // (T * W + warp) * 32 + lane, T the launch tile.  NULL (both halves 0) in every aggregation launch.
  int32_t reserved_tail[2];
};

__host__ __device__ inline uint32_t* selection_mask_of(const QueryDesc& q) {
  return reinterpret_cast<uint32_t*>((unsigned long long)(uint32_t)q.reserved_tail[1] << 32 | (uint32_t)q.reserved_tail[0]);
}
inline void set_selection_mask(QueryDesc& q, uint32_t* p) {
  const unsigned long long v = reinterpret_cast<unsigned long long>(p);
  q.reserved_tail[0] = (int32_t)(uint32_t)v;
  q.reserved_tail[1] = (int32_t)(uint32_t)(v >> 32);
}

// ---- shared-memory header of the scan kernel (the host sizes the dynamic shared memory with it) ----
constexpr int kMaxWarps = 8;    // warps per CTA (all of them consume; there is no producer warp)
constexpr int kMaxStages = 4;

struct SmemHeader {
  SegDesc seg;                              // CTA-wide copy of the current segment's descriptor
  AggDesc aggs[kMaxAggs];                   // q.aggs: indexed with a runtime `a` (an indexed LDC costs a long-scoreboard wait)
  uint32_t slot_roles[kMaxSlots];           // q.slot_roles, same reason
  int32_t group_slot[kMaxGroupBy];          // q.group_slot, same reason
  uint64_t full[kMaxWarps][kMaxStages];     // per-warp ring: "stage filled by TMA"
};

}  // namespace pb200
