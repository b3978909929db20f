// pb200_select.cuh -- what the selection (pb200_select.cu) and DISTINCT (pb200_distinct.cu) output phases share: the
// per-column descriptor, the value read at a doc and the typed decode of a stored 32-bit word, and the output rule.
#pragma once
#include <cstdint>

#include "pb200_plan.h"

namespace pb200 {

// Outputs up to this size are written by the gather straight into mapped pinned memory; larger ones go to a device
// staging buffer and come back with one DMA copy.
constexpr size_t kSelMappedBytes = 512ull << 10;

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
