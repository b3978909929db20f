// pb200_scan_launch.h -- the scan kernel's instantiations live in one translation unit each (pb200_scan_k*.cu, built in
// parallel); pb200_api.cu only sees these launchers.
#pragma once
#include <cuda_runtime.h>

#include "pb200_desc.h"

namespace pb200 {

// W warps per CTA, aggregation-only or group-by kernel, software-pipelined gathers, CTAs per SM the kernel is bounded for
struct ScanVariant {
  int warps;       // 6 | 8
  bool group_by;
  bool defer;      // aggregation only: dictionary gathers of the deferred SUM are software-pipelined across tiles
  int min_blocks;  // __launch_bounds__ minBlocksPerMultiprocessor
  bool spec;       // group-by: the kernel specialised for the shared-table shape (pb200_scan.cuh SPEC; 8 x 1 or 6 x 2 only)
};

// Launches the matching instantiation on `st`.  cudaErrorInvalidValue if the variant was not built.
cudaError_t launch_scan_variant(const ScanVariant& v, size_t smem_bytes, int grid, const QueryDesc& q, const TmaTable& tt,
                                const SegDesc* dsegs, cudaStream_t st);

#define PB200_SCAN_LAUNCHER(NAME) \
  cudaError_t NAME(size_t smem_bytes, int grid, const QueryDesc& q, const TmaTable& tt, const SegDesc* dsegs, cudaStream_t st)
PB200_SCAN_LAUNCHER(launch_scan_w6_agg);        // <6, false, true, 2>
PB200_SCAN_LAUNCHER(launch_scan_w8_agg);        // <8, false, true, 2>
PB200_SCAN_LAUNCHER(launch_scan_w8_agg_nodefer);  // <8, false, false, 2>
PB200_SCAN_LAUNCHER(launch_scan_w6_gb1);        // <6, true, false, 1>
PB200_SCAN_LAUNCHER(launch_scan_w8_gb1);        // <8, true, false, 1>
PB200_SCAN_LAUNCHER(launch_scan_w6_gb2);        // <6, true, false, 2>
PB200_SCAN_LAUNCHER(launch_scan_w8_gb2);        // <8, true, false, 2>
PB200_SCAN_LAUNCHER(launch_scan_w8_gb1_spec);   // <8, true, false, 1, true>
PB200_SCAN_LAUNCHER(launch_scan_w6_gb2_spec);   // <6, true, false, 2, true>

}  // namespace pb200
