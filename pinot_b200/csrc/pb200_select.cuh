// pb200_select.cuh -- what the selection (pb200_select.cu) and DISTINCT (pb200_distinct.cu) output phases share: the
// per-column descriptor, the value read at a doc and the typed decode of a stored 32-bit word, and the output rule.
#pragma once
#include <cstdint>
#include <memory>
#include <utility>
#include <vector>

#include "pb200_plan.h"

namespace pb200 {

// Outputs up to this size are written by the gather straight into mapped pinned memory; larger ones go to a device
// staging buffer and come back with one DMA copy.
constexpr size_t kSelMappedBytes = 512ull << 10;

// ---- host steps of both rows executors (pb200_select.cu) ----
struct RowsCall {
  pb200_segment* const* segments = nullptr;
  int nseg = 0;
  bool merge = false;                         // PB200_Q_MERGE_SEGMENTS: one result over all segments
  double t_enter = 0, t_planned = 0, t_scanned = 0;
  Tuning tune;
  DeviceLimits lim;
  float ms = 0.f;                             // CUDA-event time of the call's scans (and DISTINCT table builds)
  std::vector<long long> matches, in_filter;  // per segment, from the scan its rows come from
};
// The entry checks of pb200_execute_<fn> (args_ok: its own arguments are set), then the call's device, tuning snapshot
// and limits
int rows_call_enter(pb200_ctx* ctx, bool args_ok, pb200_segment* const* segments, int nseg, int32_t flags, const char* fn,
                    RowsCall* c);
// Where the gather writes `bytes` of output for `block`: the block through its mapped device pointer (up to
// kSelMappedBytes), else `staging` (allocated here), which the caller copies into the block after the gather
int rows_output(const PinnedBlock& block, size_t bytes, DevBufRaw& staging, unsigned char** dst);
// The call's results: result r is rows [ranges[r].first, + ranges[r].second) of `block` (doc ids int32[total_rows],
// segment index int32[total_rows], then `ncols` columns of 8-byte values [total_rows]).  Post-filter entries: the
// result's rows (per_row) or its matched docs, times ncols.  Then the call's phases (pb200_last_phases).
void rows_results(const RowsCall& c, const std::shared_ptr<PinnedBlock>& block, long long total_rows, int ncols,
                  const std::vector<std::pair<long long, long long>>& ranges, bool per_row, pb200_result** results);

struct SelCol {            // one column (selected or order item) of one segment
  const uint32_t* fwd;     // resident forward index, native word order (pb200_unpack.cuh)
  const void* dict;        // device dictionary (INT: biased by 2^31) or NULL
  int32_t bits, kind;      // kind: SEL_*
  int32_t desc, pad;       // order items: DESC
};

// the stored 32-bit word at `doc`: dictId, or the raw value (MSB-first bit stream; a value may straddle two words)
__device__ __forceinline__ uint32_t read_at(const SelCol& c, int32_t doc) {
  const unsigned long long bit = (unsigned long long)doc * (unsigned)c.bits;
  const uint32_t* p = c.fwd + (bit >> 5);
  const int sh = (int)(bit & 31u);
  const uint32_t hi = __ldg(p);
  const uint32_t lo = sh + c.bits > 32 ? __ldg(p + 1) : 0u;
  const uint32_t x = __funnelshift_l(lo, hi, sh);
  return c.bits == 32 ? x : x >> (32 - c.bits);
}

// the output word of stored word `id` (dictId or raw value): int64, or a double's bits (selection_kind_is_double)
__device__ __forceinline__ unsigned long long sel_value(const SelCol& col, uint32_t id) {
  switch (col.kind) {
    case SEL_DICT_I32: return (unsigned long long)(long long)(int32_t)(__ldg(static_cast<const uint32_t*>(col.dict) + id) ^ 0x80000000u);
    case SEL_DICT_I64: return (unsigned long long)__ldg(static_cast<const long long*>(col.dict) + id);
    case SEL_DICT_F32: return (unsigned long long)__double_as_longlong((double)__ldg(static_cast<const float*>(col.dict) + id));
    case SEL_DICT_F64: return (unsigned long long)__double_as_longlong(__ldg(static_cast<const double*>(col.dict) + id));
    case SEL_RAW_I32: return (unsigned long long)(long long)(int32_t)id;
    case SEL_RAW_F32: return (unsigned long long)__double_as_longlong((double)__int_as_float((int)id));
    default: return (unsigned long long)id;  // SEL_DICT_ID: STRING dictIds
  }
}

}  // namespace pb200
