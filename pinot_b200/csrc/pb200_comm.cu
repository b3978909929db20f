// pb200_comm.cu -- the cross-GPU combine inside the library: NCCL over NVLink 5 / NVSwitch, one communicator per context.
//
// What it replaces in the reference: the merge of the per-server partial results that the broker (and, per server, the
// combine operator) does by VALUE on the JVM (GroupByCombineOperator.java:130-146, AggregationFunction.merge).  With one
// process per GPU and table-wide dictionaries (pb200_domain.cu) the per-GPU group tables are element-wise mergeable:
//   int64 block   COUNT / integer SUM (and count-carrying sums)   ncclSum
//   double block  FLOAT / DOUBLE / LONG sums                        ncclSum
//   u32max block  MAX as dictId + 1, 0 = empty                      ncclMax on ncclUint32
//                 (raw INT: value ^ 0x80000000, 0 = INT_MIN or empty; group-exists flags)
//   u32min block  MIN as dictId, 0xFFFFFFFF = empty                 ncclMin on ncclUint32
//                 (raw INT: value ^ 0x80000000, 0xFFFFFFFF = INT_MAX or empty)
// A raw INT entry's emptiness is never read from the entry: the group's count, seen flag, carrier or hash key tells
// (max_offset in pb200_desc.h).  Both stay neutral elements of their reduce, so the reduces are the same for both kinds.
// pb200_result_combine issues ALL of a result's reduces as ONE NCCL group on the context's stream, reads the carrier verdict
// that rides behind the int64 block (pb200_plan.cpp), and lets the root extract the groups -- one library call per rank and
// query instead of four Python-driven collectives, a tensor-alias step and a second call for the extraction.
//
// NCCL is bound at RUN time (dlopen "libnccl.so.2"): the library loads and every single-GPU entry point works on a box
// without NCCL; in a torch process the already loaded NCCL is reused.  Only types and enum values come from <nccl.h>.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <cmath>
#include <cstring>
#include <mutex>

#include "pb200_internal.h"

namespace pb200 {
namespace {

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Reduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      api.handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (api.handle) break;
    }
    if (!api.handle) return;
    auto sym = [&](const char* n) { return dlsym(api.handle, n); };
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(sym("ncclAllReduce"));
    api.Reduce = reinterpret_cast<decltype(api.Reduce)>(sym("ncclReduce"));
    api.GroupStart = reinterpret_cast<decltype(api.GroupStart)>(sym("ncclGroupStart"));
    api.GroupEnd = reinterpret_cast<decltype(api.GroupEnd)>(sym("ncclGroupEnd"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllReduce || !api.Reduce || !api.GroupStart || !api.GroupEnd) {
      dlclose(api.handle);
      api.handle = nullptr;
    }
  });
  return api.handle ? &api : nullptr;
}

#define PB200_NCCL(api, call)                                                                                  \
  do {                                                                                                         \
    ncclResult_t r__ = (call);                                                                                 \
    if (r__ != ncclSuccess) {                                                                                  \
      set_error("%s failed: %s", #call, (api)->GetErrorString ? (api)->GetErrorString(r__) : "NCCL error");   \
      return PB200_E_CUDA;                                                                                     \
    }                                                                                                          \
  } while (0)

}  // namespace
}  // namespace pb200

using namespace pb200;

static_assert(sizeof(ncclUniqueId) == PB200_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");

extern "C" int32_t pb200_comm_unique_id(void* id_out) {
  if (!id_out) { set_error("null argument"); return PB200_E_INVALID; }
  NcclApi* api = nccl_api();
  if (!api) { set_error("libnccl.so.2 is not available: the cross-GPU combine needs NCCL"); return PB200_E_UNSUPPORTED; }
  ncclUniqueId id;
  PB200_NCCL(api, api->GetUniqueId(&id));
  memcpy(id_out, &id, sizeof id);
  return PB200_OK;
}

extern "C" int32_t pb200_comm_init(pb200_ctx* ctx, const void* id_bytes, int32_t rank, int32_t world_size) {
  if (!ctx || !id_bytes || world_size < 1 || rank < 0 || rank >= world_size) { set_error("invalid argument to pb200_comm_init"); return PB200_E_INVALID; }
  NcclApi* api = nccl_api();
  if (!api) { set_error("libnccl.so.2 is not available: the cross-GPU combine needs NCCL"); return PB200_E_UNSUPPORTED; }
  if (ctx->nccl_comm) { set_error("the context already has a communicator"); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  ncclUniqueId id;
  memcpy(&id, id_bytes, sizeof id);
  ncclComm_t comm = nullptr;
  PB200_NCCL(api, api->CommInitRank(&comm, world_size, id, rank));
  PB200_CUDA(cudaMalloc(&ctx->comm_scratch, 128 * sizeof(long long)));
  PB200_CUDA(cudaHostAlloc(&ctx->comm_pinned, 128 * sizeof(long long), cudaHostAllocDefault));
  ctx->nccl_comm = comm;
  ctx->comm_rank = rank;
  ctx->comm_world = world_size;
  return PB200_OK;
}

extern "C" int32_t pb200_comm_shutdown(pb200_ctx* ctx) {
  if (!ctx || !ctx->nccl_comm) return PB200_OK;
  NcclApi* api = nccl_api();
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  if (api) api->CommDestroy(static_cast<ncclComm_t>(ctx->nccl_comm));
  ctx->nccl_comm = nullptr;
  ctx->comm_world = 1;
  if (ctx->comm_scratch) cudaFree(ctx->comm_scratch);
  if (ctx->comm_pinned) cudaFreeHost(ctx->comm_pinned);
  ctx->comm_scratch = nullptr;
  ctx->comm_pinned = nullptr;
  return PB200_OK;
}

// Aggregation-only results (AggregationResultsBlockMerger.java:34-44): a handful of scalars per rank -- sums and counts add,
// MIN / MAX compare by VALUE (ids of different ranks are only comparable under a domain: dropped).  One NCCL group.
static int combine_scalars(NcclApi* api, pb200_ctx* ctx, pb200_result* R, int root) {
  const int nagg = R->meta.num_aggs;
  if (nagg > kMaxAggs || (int)R->dbl.size() < nagg || (int)R->lng.size() < nagg) { set_error("result is not an aggregation-only result"); return PB200_E_INVALID; }
  for (int a = 0; a < nagg; a++)
    if (((int)R->distinct.size() > a && !R->distinct[a].empty()) || R->lazy.src[a] >= 0) { set_error("DISTINCTCOUNT sets are merged on the host"); return PB200_E_UNSUPPORTED; }
  for (int a = 0; a < nagg; a++)
    if (R->pct.rep[a] >= 0) { set_error("PERCENTILE histograms are merged on the host"); return PB200_E_UNSUPPORTED; }
  for (int a = 0; a < nagg; a++)
    if (R->mom.on[a]) { set_error("VAR/STDDEV moments are merged on the host"); return PB200_E_UNSUPPORTED; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  ncclComm_t comm = static_cast<ncclComm_t>(ctx->nccl_comm);
  StreamLease st(ctx);
  std::lock_guard<std::mutex> g(ctx->comm_mu);
  // pinned / device scratch (8-byte slots): [0,4) statistics | [8,16) double sums | [16,24) long counts | [24,32) double mins |
  // [32,40) double maxs | [40,48) exact int64 sums of INT SUM / AVG; outputs at +64
  static_assert(64 + 48 <= 128, "comm scratch holds 128 slots");
  long long* pin = ctx->comm_pinned;
  double* pd = reinterpret_cast<double*>(pin);
  pin[0] = R->meta.num_docs_scanned; pin[1] = R->meta.num_entries_scanned_in_filter;
  pin[2] = R->meta.num_entries_scanned_post_filter; pin[3] = R->meta.num_total_docs;
  for (int a = 0; a < kMaxAggs; a++) { pd[8 + a] = 0.0; pin[16 + a] = 0; pd[24 + a] = INFINITY; pd[32 + a] = -INFINITY; pin[40 + a] = 0; }
  for (int a = 0; a < nagg; a++) {
    const double dv = R->dbl[a].empty() ? 0.0 : R->dbl[a][0];
    const long long lv = R->lng[a].empty() ? 0 : R->lng[a][0];
    pd[8 + a] = dv; pin[16 + a] = lv; pd[24 + a] = dv; pd[32 + a] = dv;
    if (R->exact.on[a]) pin[40 + a] = R->exact.sum[a];
  }
  long long* dev = ctx->comm_scratch;
  PB200_CUDA(cudaMemcpyAsync(dev, pin, 48 * sizeof(long long), cudaMemcpyHostToDevice, st));
  PB200_NCCL(api, api->GroupStart());
  ncclResult_t r = api->Reduce(dev, dev + 64, 4, ncclInt64, ncclSum, root, comm, st);
  if (r == ncclSuccess) r = api->Reduce(dev + 8, dev + 64 + 8, 8, ncclFloat64, ncclSum, root, comm, st);
  if (r == ncclSuccess) r = api->Reduce(dev + 16, dev + 64 + 16, 8, ncclInt64, ncclSum, root, comm, st);
  if (r == ncclSuccess) r = api->Reduce(dev + 24, dev + 64 + 24, 8, ncclFloat64, ncclMin, root, comm, st);
  if (r == ncclSuccess) r = api->Reduce(dev + 32, dev + 64 + 32, 8, ncclFloat64, ncclMax, root, comm, st);
  if (r == ncclSuccess) r = api->Reduce(dev + 40, dev + 64 + 40, 8, ncclInt64, ncclSum, root, comm, st);
  ncclResult_t e = api->GroupEnd();
  if (r != ncclSuccess || e != ncclSuccess) { set_error("NCCL reduce of the aggregation scalars failed"); return PB200_E_CUDA; }
  PB200_CUDA(cudaMemcpyAsync(pin + 64, dev + 64, 48 * sizeof(long long), cudaMemcpyDeviceToHost, st));
  PB200_CUDA(cudaStreamSynchronize(st));
  if (ctx->comm_rank != root) return PB200_OK;
  R->meta.num_docs_scanned = pin[64]; R->meta.num_entries_scanned_in_filter = pin[65];
  R->meta.num_entries_scanned_post_filter = pin[66]; R->meta.num_total_docs = pin[67];
  // which function each aggregation is: MIN leaves +inf / MAX -inf on empty input, sums 0 -- the caller told us through the
  // values' roles at execute time (R->agg_functions)
  for (int a = 0; a < nagg; a++) {
    const int fn = a < (int)R->agg_functions.size() ? R->agg_functions[a] : PB200_AGG_SUM;
    if (fn == PB200_AGG_MIN) R->dbl[a][0] = pd[64 + 24 + a];
    else if (fn == PB200_AGG_MAX) R->dbl[a][0] = pd[64 + 32 + a];
    else if (fn == PB200_AGG_COUNT) { R->lng[a][0] = pin[64 + 16 + a]; R->dbl[a][0] = (double)pin[64 + 16 + a]; }
    else if (R->exact.on[a]) {   // INT SUM / AVG: the exact total, rounded once (the ranks' doubles are rounded already)
      R->exact.sum[a] = pin[64 + 40 + a];
      R->dbl[a][0] = (double)pin[64 + 40 + a]; R->lng[a][0] = pin[64 + 16 + a];
    } else { R->dbl[a][0] = pd[64 + 8 + a]; R->lng[a][0] = pin[64 + 16 + a]; }
    if ((fn == PB200_AGG_MIN || fn == PB200_AGG_MAX) && a < (int)R->ids.size() && !R->ids[a].empty()) R->ids[a][0] = -1;
  }
  return PB200_OK;
}

extern "C" int32_t pb200_result_combine(pb200_ctx* ctx, pb200_result* R, int32_t root, int32_t* retry) {
  if (!ctx || !R || !retry) { set_error("null argument"); return PB200_E_INVALID; }
  *retry = 0;
  NcclApi* api = nccl_api();
  if (!api || !ctx->nccl_comm) { set_error("no communicator: call pb200_comm_init first"); return PB200_E_INVALID; }
  if (root < 0 || root >= ctx->comm_world) { set_error("root %d out of range", root); return PB200_E_INVALID; }
  if (R->meta.num_groups < 0) return combine_scalars(api, ctx, R, root);
  pb200_result::Dense& d = R->dense;
  if (!d.ctx || !d.live || d.groups <= 0) { set_error("result has no device tables (execute with PB200_Q_MERGE_SEGMENTS | PB200_Q_DEFER_FINALIZE)"); return PB200_E_INVALID; }
  if (d.hkeys) { set_error("hash group tables of different GPUs are not element-wise reducible"); return PB200_E_UNSUPPORTED; }
  for (int a = 0; a < kMaxAggs; a++) {
    if (d.dbits[a]) { set_error("group-by DISTINCTCOUNT bitsets are not reducible by NCCL (no bitwise OR): merge on the host"); return PB200_E_UNSUPPORTED; }
    if (d.expr_tab[a]) { set_error("group-by expression aggregations are not combined across GPUs: merge on the host"); return PB200_E_UNSUPPORTED; }
  }
  (void)root;
  if (d.pack_agg >= 0 && ctx->comm_world > 1 && !d.flag_slot) {
    set_error("count-carrying table was not sized for a reduce: execute with pb200_query.reduce_world = world size");
    return PB200_E_INVALID;
  }
  PB200_CUDA(cudaSetDevice(ctx->device));
  ncclComm_t comm = static_cast<ncclComm_t>(ctx->nccl_comm);
  StreamLease st(ctx);
  long long verdict = 0;
  {
    std::lock_guard<std::mutex> g(ctx->comm_mu);  // one communicator: collectives of concurrent queries must not interleave
    // Execution statistics of the whole table (the broker sums them over servers) and the carrier verdict travel in the
    // TAIL of the int64 table block when there is one -- the headline query then needs exactly ONE collective.  Every block
    // is all-reduced (NVSwitch: an all-reduce of 1-2 MB is latency bound and at least as fast as a rooted reduce; the other
    // ranks free their tables anyway).
    long long* pin = ctx->comm_pinned;
    pin[0] = R->meta.num_docs_scanned; pin[1] = R->meta.num_entries_scanned_in_filter;
    pin[2] = R->meta.num_entries_scanned_post_filter; pin[3] = R->meta.num_total_docs;
    pin[4] = d.carrier_unsafe ? 1 : 0;
    long long* tail = d.tail_slots == 5 ? (long long*)d.i64_block + (d.i64_elems - 5) : ctx->comm_scratch;
    PB200_CUDA(cudaMemcpyAsync(tail, pin, 5 * sizeof(long long), cudaMemcpyHostToDevice, st));
    int nops = (d.tail_slots == 5 ? 0 : 1) + (d.i64_elems ? 1 : 0) + (d.f64_elems ? 1 : 0) + (d.u32max_elems ? 1 : 0) + (d.u32min_elems ? 1 : 0);
    if (nops > 1) PB200_NCCL(api, api->GroupStart());
    ncclResult_t r = ncclSuccess;
    if (d.tail_slots != 5) r = api->AllReduce(tail, tail, 5, ncclInt64, ncclSum, comm, st);
    if (r == ncclSuccess && d.i64_elems) r = api->AllReduce(d.i64_block, d.i64_block, (size_t)d.i64_elems, ncclInt64, ncclSum, comm, st);
    if (r == ncclSuccess && d.f64_elems) r = api->AllReduce(d.f64_block, d.f64_block, (size_t)d.f64_elems, ncclFloat64, ncclSum, comm, st);
    if (r == ncclSuccess && d.u32max_elems) r = api->AllReduce(d.u32max_block, d.u32max_block, (size_t)d.u32max_elems, ncclUint32, ncclMax, comm, st);
    if (r == ncclSuccess && d.u32min_elems) r = api->AllReduce(d.u32min_block, d.u32min_block, (size_t)d.u32min_elems, ncclUint32, ncclMin, comm, st);
    ncclResult_t e = nops > 1 ? api->GroupEnd() : ncclSuccess;
    if (r != ncclSuccess || e != ncclSuccess) {
      set_error("NCCL reduce of the group tables failed: %s", api->GetErrorString ? api->GetErrorString(r != ncclSuccess ? r : e) : "error");
      return PB200_E_CUDA;
    }
    PB200_CUDA(cudaMemcpyAsync(pin + 8, tail, 5 * sizeof(long long), cudaMemcpyDeviceToHost, st));
    if (ctx->comm_rank == root) {
      // the root extracts SPECULATIVELY behind the reduce on the same stream (the verdict is almost always "safe"): one
      // host sync for reduce + verdict + extraction instead of two; an unsafe verdict just discards the extraction
      pb200_result* one[1] = {R};
      const int rc = extract_groups(ctx, one, 1, st);   // synchronises the stream: pin[8..13) has landed
      if (rc && !(d.pack_agg >= 0 && pin[12] != 0)) return rc;
    }
    PB200_CUDA(cudaStreamSynchronize(st));
    verdict = d.pack_agg >= 0 ? pin[12] : 0;
    if (ctx->comm_rank == root && verdict == 0) {
      R->meta.num_docs_scanned = pin[8]; R->meta.num_entries_scanned_in_filter = pin[9];
      R->meta.num_entries_scanned_post_filter = pin[10]; R->meta.num_total_docs = pin[11];
    }
  }
  if (verdict != 0) *retry = 1;  // identical on every rank: all free the result and rerun without the carrier
  return PB200_OK;
}
