// decode_probe.cpp -- TEST shim: the result decoder of pinot_b200/csrc/pb200_decode.h (the code the extraction kernels
// and the aggregation-only route run) over one-entry tables, without a GPU.  Built by tests/test_decode_cpu.py with g++.
#include <cuda_runtime.h>   // __host__ / __device__ of pb200_desc.h as plain C++

#include <cstdint>

#include "../../pinot_b200/csrc/pb200_decode.h"

extern "C" {

// One aggregation over one-entry tables: `word` is the entry of its source table (a u32 table uses the low half), the
// other tables hold the given values.  dict: the dictionary (NULL: none), bias: its INT bias.  Writes {double, long,
// dictId} and, for VAR / STDDEV, the moments row.
void dp_decode(int32_t fn, int32_t vk, int32_t counted, uint64_t cnt, uint64_t word, const void* dict, uint32_t bias,
               int32_t pack_shift, int64_t pack_vmin, uint32_t pct_n, int64_t wt_time, const int64_t* mom, int32_t mom_e,
               const uint64_t* ds, int64_t hll, int32_t has_xkey, uint64_t xkey, double* dv, int64_t* lv, int32_t* id,
               unsigned long long* mom_row) {
  union { uint64_t u64; uint32_t u32; } src;
  src.u64 = word;
  if (vk != pb200::VAL_NONE && fn != PB200_AGG_SUM && fn != PB200_AGG_AVG) src.u32 = (uint32_t)word;
  long long limbs[3] = {mom[0], mom[1], mom[2]};
  unsigned long long state[pb200::kDsWords];
  for (int i = 0; i < pb200::kDsWords; i++) state[i] = ds[i];
  long long est = hll, time = wt_time;
  unsigned long long key = xkey;
  uint32_t n = pct_n;
  pb200::AggSource s{};
  s.fn = fn; s.vk = vk; s.src = &src; s.dict = dict; s.dict_bias = bias; s.counted = counted;
  s.pack_shift = pack_shift; s.pack_vmin = pack_vmin;
  s.pct_n = &n; s.wt_time = &time;
  for (int j = 0; j < 3; j++) s.mom[j] = &limbs[j];
  s.mom_e = mom_e; s.ds = state; s.hll = &est; s.xkey = has_xkey ? &key : nullptr;
  long long l;
  pb200::agg_values(s, 0, cnt, *dv, l, *id, mom_row);
  *lv = l;
}

}
