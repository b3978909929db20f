// pb200_transform.cu -- derived columns: a single-column transform program (pb200_transform.h) turned into an ordinary
// dictionary column of the segment.
//
// A function of one dictionary column is a function of its dictId.  With D' the sorted distinct values of f over the
// column's dictionary and remap[id] the rank of f(dict[id]) in D', re-encoding the forward index through remap (the
// domain machinery's re-encode) gives a column with a sorted dictionary, so every query route serves it unchanged:
//   1. one thread per dictionary entry evaluates the program and writes the result's order key and the entry's id;
//   2. one radix sort of (key, id), adjacent-difference flags and an inclusive scan give the ranks: remap[id] and D';
//   3. the forward index is re-encoded at bits_for_cardinality(|D'|);
//   4. D' becomes the dictionary in its three forms (device, native host, big-endian) from one device-to-host copy.
// A time column's LONG dictionary can hold tens of millions of entries, which is why all of this runs on the device.
#include <cuda_runtime.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <cstring>
#include <vector>

#include "pb200_internal.h"
#include "pb200_transform.h"

namespace pb200 {
namespace {

constexpr int kMaxProgramBytes = kTransformMaxProgram * (int)sizeof(pb200_transform_op);

struct Program {
  pb200_transform_op ops[kTransformMaxProgram];
  int n;
};

__global__ void eval_kernel(Program prog, int source_type, const void* __restrict__ dict, uint32_t card, int kind,
                            uint64_t* __restrict__ keys, uint32_t* __restrict__ ids, uint32_t* __restrict__ out_of_range) {
  __shared__ pb200_transform_op ops[kTransformMaxProgram];
  for (int k = threadIdx.x; k < prog.n; k += blockDim.x) ops[k] = prog.ops[k];
  __syncthreads();
  for (uint32_t id = blockIdx.x * blockDim.x + threadIdx.x; id < card; id += gridDim.x * blockDim.x) {
    int64_t si = 0;
    double sd = 0.0;
    switch (source_type) {  // the device dictionary: INT biased (convert_dictionary), the others native
      case PB200_INT: si = (int32_t)(static_cast<const uint32_t*>(dict)[id] ^ 0x80000000u); break;
      case PB200_LONG: si = static_cast<const int64_t*>(dict)[id]; break;
      case PB200_FLOAT: sd = static_cast<const float*>(dict)[id]; break;
      default: sd = static_cast<const double*>(dict)[id];
    }
    int64_t ri = 0;
    double rd = 0.0;
    if (!transform_eval(ops, prog.n, source_type, si, sd, &ri, &rd)) atomicOr(out_of_range, 1u);
    keys[id] = transform_key(kind, ri, rd);
    ids[id] = id;
  }
}

__global__ void flag_kernel(const uint64_t* __restrict__ keys, uint32_t n, uint32_t* __restrict__ flags) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    flags[k] = k > 0 && keys[k] != keys[k - 1];
}

// ranks -> remap[source id]; each distinct key once, as the dictionary's native device value (INT biased)
__global__ void rank_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ids, const uint32_t* __restrict__ rank,
                            uint32_t n, int kind, uint32_t* __restrict__ remap, void* __restrict__ dict_out, uint32_t* __restrict__ card_out) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const uint32_t r = rank[k];
    remap[ids[k]] = r;
    if (k == 0 || keys[k] != keys[k - 1]) {
      const uint64_t bits = transform_key_bits(kind, keys[k]);
      if (kind == TK_INT) static_cast<uint32_t*>(dict_out)[r] = (uint32_t)bits ^ 0x80000000u;
      else static_cast<uint64_t*>(dict_out)[r] = bits;
    }
    if (k == n - 1) *card_out = r + 1;
  }
}

inline void put_be(unsigned char* p, uint64_t v, int w) { for (int b = 0; b < w; b++) p[b] = (unsigned char)(v >> (8 * (w - 1 - b))); }

}  // namespace
}  // namespace pb200

using namespace pb200;

extern "C" int32_t pb200_segment_derive_column(pb200_ctx* ctx, pb200_segment* seg, int32_t source, int32_t num_ops,
                                               const pb200_transform_op* ops, int32_t* new_column) {
  if (!ctx || !seg || !new_column || seg->ctx != ctx) { set_error("invalid argument to pb200_segment_derive_column"); return PB200_E_INVALID; }
  std::lock_guard<std::mutex> derive_lock(seg->derive_mu);
  if (source < 0 || source >= seg->num_columns()) { set_error("derive: no column %d", source); return PB200_E_INVALID; }
  const DeviceColumn& src = seg->cols[source];
  int kind = 0;
  const char* why = "";
  if (int rc = transform_check(ops, num_ops, src.stored_type, &kind, &why)) { set_error("derive from column %d: %s", source, why); return rc; }
  if (src.fwd_kind != PB200_FWD_DICT_FIXEDBIT || !src.dict_native || src.bits > 31) {
    set_error("derive: column %d has no dictIds (a raw column streamed as 32-bit values)", source);
    return PB200_E_UNSUPPORTED;
  }
  if (seg->num_columns() - seg->num_stored >= PB200_MAX_DERIVED_COLUMNS) {
    set_error("segment '%s' already has %d derived columns", seg->name.c_str(), PB200_MAX_DERIVED_COLUMNS);
    return PB200_E_UNSUPPORTED;
  }
  PB200_CUDA(cudaSetDevice(ctx->device));
  Program prog;
  memcpy(prog.ops, ops, sizeof(pb200_transform_op) * num_ops);
  prog.n = num_ops;
  static_assert(sizeof(Program) <= kMaxProgramBytes + 16, "program travels as a kernel parameter");

  const uint32_t n = (uint32_t)src.cardinality;
  const int width = kind == TK_INT ? 4 : 8;
  StreamLease st(ctx);
  // scratch: keys and ids in and out of the sort, flags / ranks, the sort's temporary storage
  size_t sort_bytes = 0, scan_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)n);
  cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
  DevBufRaw keys(ctx), keys_sorted(ctx), ids(ctx), ids_sorted(ctx), flags(ctx), rank(ctx), temp(ctx), flag(ctx), dict_tmp(ctx);
  void* remap = nullptr;
  const size_t nn = std::max<size_t>(n, 1);
  int rc = 0;
  if (!rc) rc = keys.alloc(nn * 8);
  if (!rc) rc = keys_sorted.alloc(nn * 8);
  if (!rc) rc = ids.alloc(nn * 4);
  if (!rc) rc = ids_sorted.alloc(nn * 4);
  if (!rc) rc = flags.alloc(nn * 4);
  if (!rc) rc = rank.alloc(nn * 4);
  if (!rc) rc = temp.alloc(std::max<size_t>(std::max(sort_bytes, scan_bytes), 16));
  if (!rc) rc = flag.alloc(16);
  if (!rc) rc = dict_tmp.alloc(nn * width);
  if (!rc) rc = dev_alloc(ctx, nn * 4, &remap);
  if (rc) { dev_free(ctx, remap); return rc; }
  // declared after the scratch buffers, so destroyed before them: on every return the stream has drained before the
  // scratch goes back to the pool
  struct Drain { cudaStream_t s; ~Drain() { cudaStreamSynchronize(s); } } drain{st};
  const int end_bit = kind == TK_INT ? 32 : 64;  // INT keys are zero above bit 31
  const int blocks = (int)std::min<long long>((n + 255) / 256 + 1, (long long)ctx->sm_count * 8);
  uint32_t host_flags[2] = {0, 0};  // {out of range, cardinality}
  cudaError_t e = cudaMemsetAsync(flag.p, 0, 16, st);
  if (e == cudaSuccess && n > 0) {
    eval_kernel<<<blocks, 256, 0, st>>>(prog, src.stored_type, src.dict_native, n, kind, (uint64_t*)keys.p, (uint32_t*)ids.p, (uint32_t*)flag.p);
    e = cudaGetLastError();
    if (e == cudaSuccess)
      e = cub::DeviceRadixSort::SortPairs(temp.p, sort_bytes, (const uint64_t*)keys.p, (uint64_t*)keys_sorted.p, (const uint32_t*)ids.p,
                                          (uint32_t*)ids_sorted.p, (int)n, 0, end_bit, st);
    if (e == cudaSuccess) { flag_kernel<<<blocks, 256, 0, st>>>((const uint64_t*)keys_sorted.p, n, (uint32_t*)flags.p); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cub::DeviceScan::InclusiveSum(temp.p, scan_bytes, (const uint32_t*)flags.p, (uint32_t*)rank.p, (int)n, st);
    if (e == cudaSuccess) {
      rank_kernel<<<blocks, 256, 0, st>>>((const uint64_t*)keys_sorted.p, (const uint32_t*)ids_sorted.p, (const uint32_t*)rank.p, n, kind,
                                          (uint32_t*)remap, dict_tmp.p, (uint32_t*)flag.p + 1);
      e = cudaGetLastError();
    }
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(host_flags, flag.p, 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { dev_free(ctx, remap); set_error("derive: evaluation failed: %s", cudaGetErrorString(e)); return PB200_E_CUDA; }
  if (host_flags[0]) {
    dev_free(ctx, remap);
    set_error("derive from column %d: a dictionary value lies beyond +-2^53 ms, outside the calendar functions' range", source);
    return PB200_E_UNSUPPORTED;
  }
  const int card = (int)host_flags[1];

  DeviceColumn c;
  c.fwd_kind = PB200_FWD_DICT_FIXEDBIT;
  c.stored_type = kind;
  c.cardinality = card;
  c.bits = bits_for_cardinality(std::max(card, 1));
  c.fwd_alloc_bytes = padded_fwd_bytes(seg->num_docs, c.bits);
  c.fwd_file_bytes = ((uint64_t)seg->num_docs * c.bits + 7) / 8;
  c.pooled = true;
  c.dict_entry_bytes = width;
  auto fail = [&](int code) { dev_free(ctx, remap); dev_free(ctx, c.fwd); dev_free(ctx, c.dict_native); return code; };
  { void* p = nullptr; rc = dev_alloc(ctx, c.fwd_alloc_bytes, &p); c.fwd = (uint32_t*)p; if (rc) return fail(rc); }
  rc = dev_alloc(ctx, std::max<size_t>((size_t)card * width, 16), &c.dict_native);
  if (rc) return fail(rc);
  std::vector<unsigned char> native((size_t)card * width);
  std::vector<uint32_t> remap_host(src.local_ids.empty() ? 0 : n);
  e = cudaMemsetAsync(c.fwd, 0, c.fwd_alloc_bytes, st);
  if (e == cudaSuccess) e = reencode_column(ctx, st, src.fwd, src.bits, c.fwd, c.bits, (const uint32_t*)remap, n, seg->num_docs);
  if (e == cudaSuccess && card) e = cudaMemcpyAsync(c.dict_native, dict_tmp.p, native.size(), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess && card) e = cudaMemcpyAsync(native.data(), dict_tmp.p, native.size(), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && !remap_host.empty()) e = cudaMemcpyAsync(remap_host.data(), remap, (size_t)n * 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { set_error("derive: re-encode failed: %s", cudaGetErrorString(e)); return fail(PB200_E_CUDA); }
  dev_free(ctx, remap);
  remap = nullptr;

  c.dict_host = native;
  c.dict_be.resize(native.size());
  for (int i = 0; i < card; i++) {
    uint64_t v;
    if (width == 4) { uint32_t u; memcpy(&u, &native[4ull * i], 4); u ^= 0x80000000u; memcpy(&c.dict_host[4ull * i], &u, 4); v = u; }
    else memcpy(&v, &native[8ull * i], 8);
    put_be(&c.dict_be[(size_t)width * i], v, width);
  }
  c.dict_hash = dictionary_hash(kind, width, card, c.dict_be.data());
  if (!remap_host.empty()) {  // bound source: the derived ids this segment holds are the ranks of its own ids
    for (uint32_t g : src.local_ids) c.local_ids.push_back(remap_host[g]);
    std::sort(c.local_ids.begin(), c.local_ids.end());
    c.local_ids.erase(std::unique(c.local_ids.begin(), c.local_ids.end()), c.local_ids.end());
  }
  seg->device_bytes += (int64_t)c.fwd_alloc_bytes + (int64_t)c.dict_host.size();
  const int id = seg->num_columns();
  seg->cols.push_back(std::move(c));  // within the reserved capacity: no column moves
  seg->published.store(id + 1, std::memory_order_release);  // the column is complete: queries may name it now
  *new_column = id;
  return PB200_OK;
}
