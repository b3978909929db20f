// pb200_distinct_sum.cu -- DISTINCTSUM / DISTINCTAVG finalize: DISTINCTCOUNT dictId bitsets -> per row the exact int128
// sum of the members' j, |S| and the special-value flags (pb200_distinct_sum.h), queued behind the scan on its stream.
//
//   group-by         one warp per table entry: the lanes stride the entry's bitset row coalesced, each set bit gathers
//                    its dictionary value, and a shuffle reduction writes the entry's state.  Entries without rows have
//                    an all-zero row and finalize to the empty state.
//   aggregation only one bitset of up to 2^26 words per result: a grid-stride pass leaves one int128 partial per block,
//                    one small block adds them.  The sum is exact, so the result does not depend on the schedule.
#include <cuda_runtime.h>

#include "pb200_internal.h"

namespace pb200 {

namespace {
constexpr int kDsThreads = 256;

// member dictId x of a dictionary of `stored_type` (device copy: INT biased): adds j to *sum or returns its flag
__device__ __forceinline__ uint32_t ds_member(const void* dict, int stored_type, int e, uint32_t x, i128* sum) {
  switch (stored_type) {
    case PB200_INT: *sum += (i128)(int32_t)(static_cast<const uint32_t*>(dict)[x] ^ 0x80000000u); return 0;
    case PB200_LONG: *sum += (i128)static_cast<const long long*>(dict)[x]; return 0;
    case PB200_FLOAT: return ds_add_double((double)static_cast<const float*>(dict)[x], e, sum);
    default: return ds_add_double(static_cast<const double*>(dict)[x], e, sum);
  }
}

// the members of one bitset word (dictIds 32 w ...)
__device__ __forceinline__ void ds_word(const DistinctSumJob& j, uint32_t word, size_t w, i128* sum, unsigned long long* n,
                                        uint32_t* flags) {
  *n += __popc(word);
  for (; word; word &= word - 1) *flags |= ds_member(j.dict, j.stored_type, j.e, (uint32_t)(w * 32 + __ffs(word) - 1), sum);
}

__device__ __forceinline__ void warp_reduce(i128* sum, unsigned long long* n, uint32_t* flags) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long lo = __shfl_xor_sync(0xFFFFFFFFu, (unsigned long long)(u128)*sum, o);
    const unsigned long long hi = __shfl_xor_sync(0xFFFFFFFFu, (unsigned long long)((u128)*sum >> 64), o);
    *sum += (i128)(((u128)hi << 64) | lo);
    *n += __shfl_xor_sync(0xFFFFFFFFu, *n, o);
    *flags |= __shfl_xor_sync(0xFFFFFFFFu, *flags, o);
  }
}

// final: also the two rounded values (a row's state, not a block's partial)
__device__ __forceinline__ void store_state(unsigned long long* out, i128 sum, unsigned long long n, uint32_t flags, int e,
                                            bool final) {
  out[0] = (unsigned long long)(u128)sum;
  out[1] = (unsigned long long)((u128)sum >> 64);
  out[2] = n;
  out[3] = flags;
  if (!final) return;
  out[4] = (unsigned long long)__double_as_longlong(distinct_final(PB200_AGG_DISTINCTSUM, sum, n, flags, e));
  out[5] = (unsigned long long)__double_as_longlong(distinct_final(PB200_AGG_DISTINCTAVG, sum, n, flags, e));
}

__global__ void __launch_bounds__(kDsThreads) distinct_sum_rows_kernel(DistinctSumJob j) {
  const long long warps = (long long)gridDim.x * (kDsThreads / 32);
  const int lane = threadIdx.x & 31;
  for (long long g = blockIdx.x * (long long)(kDsThreads / 32) + (threadIdx.x >> 5); g < j.rows; g += warps) {
    const uint32_t* row = j.bits + (size_t)g * j.words;
    i128 sum = 0;
    unsigned long long n = 0;
    uint32_t flags = 0;
    for (size_t w = lane; w < j.words; w += 32) ds_word(j, row[w], w, &sum, &n, &flags);
    warp_reduce(&sum, &n, &flags);
    if (lane == 0) store_state(j.out + (size_t)g * kDsWords, sum, n, flags, j.e, true);
  }
}

// aggregation only, pass 1: block b's partial state to part + kDsWords * b
__global__ void __launch_bounds__(kDsThreads) distinct_sum_partial_kernel(DistinctSumJob j, unsigned long long* __restrict__ part) {
  __shared__ unsigned long long sh[kDsThreads / 32][kDsWords];
  i128 sum = 0;
  unsigned long long n = 0;
  uint32_t flags = 0;
  for (size_t w = blockIdx.x * (size_t)kDsThreads + threadIdx.x; w < j.words; w += (size_t)gridDim.x * kDsThreads)
    ds_word(j, j.bits[w], w, &sum, &n, &flags);
  warp_reduce(&sum, &n, &flags);
  if ((threadIdx.x & 31) == 0) store_state(sh[threadIdx.x >> 5], sum, n, flags, j.e, false);
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < kDsThreads / 32; k++) { sum += ds_sum_of(sh[k]); n += sh[k][2]; flags |= (uint32_t)sh[k][3]; }
    store_state(part + (size_t)kDsWords * blockIdx.x, sum, n, flags, j.e, false);
  }
}

// aggregation only, pass 2: the blocks' partials -> out (one warp)
__global__ void distinct_sum_total_kernel(const unsigned long long* __restrict__ part, int blocks, int e, unsigned long long* __restrict__ out) {
  i128 sum = 0;
  unsigned long long n = 0;
  uint32_t flags = 0;
  for (int b = threadIdx.x; b < blocks; b += 32) { sum += ds_sum_of(part + (size_t)kDsWords * b); n += part[(size_t)kDsWords * b + 2]; flags |= (uint32_t)part[(size_t)kDsWords * b + 3]; }
  warp_reduce(&sum, &n, &flags);
  if (threadIdx.x == 0) store_state(out, sum, n, flags, e, true);
}
}  // namespace

int distinct_sum_finalize(pb200_ctx* ctx, cudaStream_t st, const DistinctSumJob& j, std::vector<std::unique_ptr<DevBufRaw>>& temps) {
  if (j.rows <= 0) return PB200_OK;
  if (j.rows > 1 || !j.single) {
    distinct_sum_rows_kernel<<<grid_for(ctx, j.rows * 32, kDsThreads), kDsThreads, 0, st>>>(j);
  } else {
    const int blocks = grid_for(ctx, (long long)j.words, kDsThreads);
    temps.emplace_back(new DevBufRaw(ctx));
    if (int rc = temps.back()->alloc((size_t)blocks * kDsWords * 8)) return rc;
    unsigned long long* part = static_cast<unsigned long long*>(temps.back()->p);
    distinct_sum_partial_kernel<<<blocks, kDsThreads, 0, st>>>(j, part);
    distinct_sum_total_kernel<<<1, 32, 0, st>>>(part, blocks, j.e, j.out);
  }
  PB200_CUDA(cudaGetLastError());
  return PB200_OK;
}

}  // namespace pb200
