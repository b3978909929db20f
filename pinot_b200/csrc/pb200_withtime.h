// pb200_withtime.h -- FIRSTWITHTIME / LASTWITHTIME finalize (pb200_withtime.cu): winning keys -> data dictIds and time
// values on the device (DESIGN.md section 3.13).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <vector>

#include "pb200_internal.h"

namespace pb200 {

// One segment of the call as the finalize sees it: its rows are ordinals [base, base + num_docs).
struct WtSeg {
  unsigned long long base;
  const uint32_t* fwd;     // the data column's packed dictIds (native word order, pb200_unpack.cuh)
  const void* tdict;       // the time column's device dictionary: biased u32 (INT) or int64 (LONG)
  int32_t bits;            // of the data column
  int32_t time_long;       // 1: LONG time column
  uint32_t num_docs;
  uint32_t time_card;
};

// One key table: `rows` keys (withtime_key in pb200_desc.h).  Row i gets the data dictId of the winning row in ids[i]
// and its time value in time[i]; a key that names no row of the call (an initial value) gives ~0 and 0.
struct WithTimeJob {
  const unsigned long long* keys = nullptr;
  long long rows = 0;
  uint32_t* ids = nullptr;
  long long* time = nullptr;
};

// The call's segments for the finalize of aggregation `agg` (data column data_col, time column time_col), uploaded on `st`
// into a buffer kept in `temps`.
int withtime_segments(pb200_ctx* ctx, cudaStream_t st, pb200_segment* const* segments, int nseg, int data_col, int time_col,
                      const std::vector<unsigned long long>& base, std::vector<std::unique_ptr<DevBufRaw>>& temps,
                      const WtSeg** out);
// Queues the finalize of one key table on `st` behind the scan (no synchronisation).
int withtime_finalize(pb200_ctx* ctx, cudaStream_t st, const WithTimeJob& job, const WtSeg* segs, int nseg);

}  // namespace pb200
