// pb200_percentile.h -- PERCENTILE finalize (pb200_percentile.cu): dictId histograms -> selected dictIds on the device.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <vector>

#include "pb200_internal.h"

namespace pb200 {

// One histogram block: `rows` rows of E u32 counts (row-major).  For each of its np percentiles p[a] the selected dictId
// of every row goes to ids[a][row] (~0 when the row has no count); n_out[row] (may be NULL) receives the row's total.
struct PercentileJob {
  const uint32_t* hist = nullptr;
  long long rows = 0;
  uint32_t E = 0;
  uint32_t nchunks = 0;   // set by percentile_finalize
  int np = 0;
  double p[kMaxAggs] = {};
  uint32_t* ids[kMaxAggs] = {};
  uint32_t* n_out = nullptr;
};

// Queues the finalize of one histogram block on `st` (no synchronisation); its scratch stays in `temps` until the
// stream has passed it.
int percentile_finalize(pb200_ctx* ctx, cudaStream_t st, const PercentileJob& job, std::vector<std::unique_ptr<DevBufRaw>>& temps);
// Copies histogram rows to the host: all `rows` rows of the block (idx == NULL) or the rows idx[0 .. rows) (host array).
int percentile_read_rows(pb200_ctx* ctx, const uint32_t* hist, const uint32_t* idx, long long rows, uint32_t E,
                         std::vector<uint32_t>& out);

}  // namespace pb200
