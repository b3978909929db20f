// pb200_startree_build.cu -- builds a segment's star-tree on the device from its resident columns: the tree of
// BaseSingleTreeBuilder.build (restated by oracle/startree_builder.py) and its star docs as a device segment, in the
// layout pb200h_startree_attach produces (host/star_tree.cpp), so traversal and scan treat both alike.
//
// Every doc-sized step is one PASS over a list of doc ranges, each range tagged with the node (owner) it belongs to:
//   expand the ranges into items -> optionally sort the items by (owner, key dimensions) -> flag where the owner or a
//   key dimension changes -> inclusive scan = run ids -> one new doc per run: the dimensions of its first item with the
//   zeroed dimensions set to STAR_IN_FORWARD_INDEX (0), and one ReduceByKey per metric.
// The passes:
//   base docs      all rows, keys = the split order                                  (sortAndAggregateSegmentRecords)
//   children       per level: the ranges of the nodes being split, keys = the child dimension; reports the runs only
//   star children  per level, one pass for all parents that get one: keys = (parent, dimensions after the starred one)
//   aggregated     per level, bottom up: multi-doc leaves' ranges and the aggregated docs of a STAR-less node's
//                  children, no keys: one run per node                                (createAggregatedDocs)
// Nodes are few next to docs: the host keeps them (split decisions, breadth-first numbering) and hands ranges down, so
// launches and stream synchronisations grow with the number of levels, never with the number of nodes or docs.
//
// Metrics travel as 64-bit accumulators: COUNT and SUM over INT as exact int64, the other SUMs as the double's bits
// (accumulated in double, as ValueAggregatorFactory does), MIN / MAX as the Double.compare order key (pb200_order.h), so
// that a star-tree MIN / MAX equals the raw scan's at NaN and -0.0.
#include <cuda_runtime.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <climits>
#include <cstring>
#include <vector>

#include "pb200_order.h"
#include "pb200_startree_build.h"
#include "pb200_unpack.cuh"

namespace pb200 {
namespace {

constexpr int kMaxDims = 30;
constexpr int kThreads = 256;
enum Acc { ACC_I64 = 0, ACC_F64 = 1, ACC_MIN = 2, ACC_MAX = 3 };
enum Src { SRC_COUNT = 0, SRC_DICT = 1, SRC_RAW32 = 2 };

struct DimPtrs { const uint32_t* p[kMaxDims]; };
struct OutDims { uint32_t* p[kMaxDims]; };
struct KeyCols { const uint32_t* p[kMaxDims]; int bits[kMaxDims]; int n; };

struct SumI64 { __device__ uint64_t operator()(uint64_t a, uint64_t b) const { return a + b; } };
struct SumF64 {
  __device__ uint64_t operator()(uint64_t a, uint64_t b) const {
    return (uint64_t)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)b)));
  }
};
struct MinU64 { __device__ uint64_t operator()(uint64_t a, uint64_t b) const { return a < b ? a : b; } };
struct MaxU64 { __device__ uint64_t operator()(uint64_t a, uint64_t b) const { return a > b ? a : b; } };

#define PB200_GRID_LOOP(i, n) for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (n); i += (long long)gridDim.x * blockDim.x)

__global__ void unpack_kernel(const uint32_t* __restrict__ fwd, int bits, long long n, uint32_t* __restrict__ out) {
  PB200_GRID_LOOP(i, n) out[i] = read_one(fwd, i, bits);
}

// one row's metric as its accumulator
__global__ void row_metric_kernel(int src, const uint32_t* __restrict__ fwd, int bits, const void* __restrict__ dict, int type,
                                  int acc, long long n, uint64_t* __restrict__ out) {
  PB200_GRID_LOOP(i, n) {
    int64_t iv = 1;
    double dv = 1.0;
    if (src != SRC_COUNT) {
      const uint32_t w = src == SRC_RAW32 ? fwd[i] : 0u;
      const uint32_t id = src == SRC_DICT ? read_one(fwd, i, bits) : 0u;
      switch (type) {  // device dictionaries: INT biased (convert_dictionary), the others native
        case PB200_INT: iv = src == SRC_RAW32 ? (int32_t)w : (int32_t)(static_cast<const uint32_t*>(dict)[id] ^ 0x80000000u); dv = (double)iv; break;
        case PB200_LONG: iv = static_cast<const int64_t*>(dict)[id]; dv = (double)iv; break;
        case PB200_FLOAT: dv = __uint_as_float(src == SRC_RAW32 ? w : static_cast<const uint32_t*>(dict)[id]); break;
        default: dv = static_cast<const double*>(dict)[id];
      }
    }
    out[i] = acc == ACC_I64 ? (uint64_t)iv : acc == ACC_F64 ? (uint64_t)__double_as_longlong(dv) : double_order_bits(dv);
  }
}

// item p of the concatenated ranges: range r with off[r] <= p < off[r + 1]
__global__ void expand_kernel(const uint32_t* __restrict__ start, const uint32_t* __restrict__ off, const uint32_t* __restrict__ owner,
                              int nr, long long n, uint32_t* __restrict__ items, uint32_t* __restrict__ item_owner) {
  PB200_GRID_LOOP(p, n) {
    int lo = 0, hi = nr - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (off[mid] <= (uint32_t)p) lo = mid; else hi = mid - 1;
    }
    items[p] = start[lo] + ((uint32_t)p - off[lo]);
    item_owner[p] = owner[lo];
  }
}

// the sort key of item `pos`: owner (when owner_bits > 0), then the key columns, most significant first
__global__ void key64_kernel(const uint32_t* __restrict__ items, const uint32_t* __restrict__ owner, int owner_bits, KeyCols k,
                             long long n, uint64_t* __restrict__ key, uint32_t* __restrict__ pos) {
  PB200_GRID_LOOP(i, n) {
    uint64_t v = owner_bits ? owner[i] : 0u;
    const uint32_t s = items[i];
    for (int j = 0; j < k.n; j++) v = (v << k.bits[j]) | k.p[j][s];
    key[i] = v;
    pos[i] = (uint32_t)i;
  }
}

// one pass of the multi-pass sort: the 32-bit key of column `col` (-1: the owner) of the items in the current order
__global__ void key32_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ items, const uint32_t* __restrict__ owner,
                             const uint32_t* __restrict__ col, long long n, uint32_t* __restrict__ key) {
  PB200_GRID_LOOP(i, n) key[i] = col ? col[items[perm[i]]] : owner[perm[i]];
}

__global__ void iota_kernel(uint32_t* __restrict__ p, long long n) { PB200_GRID_LOOP(i, n) p[i] = (uint32_t)i; }

__global__ void permute_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ items, const uint32_t* __restrict__ owner,
                               long long n, uint32_t* __restrict__ items_out, uint32_t* __restrict__ owner_out) {
  PB200_GRID_LOOP(i, n) { items_out[i] = items[perm[i]]; owner_out[i] = owner[perm[i]]; }
}

__global__ void flag_kernel(const uint32_t* __restrict__ items, const uint32_t* __restrict__ owner, KeyCols k, long long n,
                            uint32_t* __restrict__ flags) {
  PB200_GRID_LOOP(i, n) {
    bool f = i == 0 || owner[i] != owner[i - 1];
    for (int j = 0; j < k.n && !f; j++) f = k.p[j][items[i]] != k.p[j][items[i - 1]];
    flags[i] = f;
  }
}

__global__ void first_kernel(const uint32_t* __restrict__ flags, const uint32_t* __restrict__ run, long long n, uint32_t* __restrict__ first) {
  PB200_GRID_LOOP(i, n) if (flags[i]) first[run[i] - 1] = (uint32_t)i;
}

// children of the nodes being split: per run its first doc, its value of the child dimension and its parent
__global__ void children_kernel(const uint32_t* __restrict__ first, const uint32_t* __restrict__ items, const uint32_t* __restrict__ owner,
                                const uint32_t* __restrict__ dim, long long runs, uint32_t* __restrict__ out) {
  PB200_GRID_LOOP(r, runs) {
    const uint32_t i = first[r], doc = items[i];
    out[r] = doc; out[runs + r] = dim[doc]; out[2 * runs + r] = owner[i];
  }
}

// one new doc per run at off + r: the dimensions of the run's first item, [z0, z1) set to 0; per owner its new docs
__global__ void emit_kernel(const uint32_t* __restrict__ first, const uint32_t* __restrict__ items, const uint32_t* __restrict__ owner,
                            long long runs, DimPtrs src, OutDims dst, int nd, int z0, int z1, long long off,
                            uint32_t* __restrict__ owner_first, uint32_t* __restrict__ owner_end) {
  PB200_GRID_LOOP(r, runs) {
    const uint32_t i = first[r], s = items[i], o = owner[i];
    for (int j = 0; j < nd; j++) dst.p[j][off + r] = (j >= z0 && j < z1) ? 0u : src.p[j][s];
    if (r == 0 || owner[first[r - 1]] != o) owner_first[o] = (uint32_t)(off + r);
    if (r == runs - 1 || owner[first[r + 1]] != o) owner_end[o] = (uint32_t)(off + r + 1);
  }
}

__global__ void gather_kernel(const uint32_t* __restrict__ items, const uint64_t* __restrict__ src, long long n, uint64_t* __restrict__ out) {
  PB200_GRID_LOOP(i, n) out[i] = src[items[i]];
}

// u32 values -> fixed-bit forward index in the HBM layout (pb200_unpack.cuh): one thread per 32-row group
__global__ void pack_kernel(const uint32_t* __restrict__ v, long long n, int bits, long long groups, uint32_t* __restrict__ out) {
  PB200_GRID_LOOP(g, groups) {
    uint32_t* o = out + g * bits;
    uint64_t acc = 0;
    int have = 0, k = 0;
    for (int i = 0; i < 32; i++) {
      const long long row = g * 32 + i;
      acc = (acc << bits) | (row < n ? v[row] : 0u);
      have += bits;
      if (have >= 32) { o[k++] = (uint32_t)(acc >> (have - 32)); have -= 32; }
    }
  }
}

// the final value of a star doc's metric as an order key: LONG (count__*) sign-flipped, DOUBLE double_order_bits
enum Final { FIN_LONG = 0, FIN_INT_SUM = 1, FIN_DOUBLE = 2, FIN_KEY = 3 };
__global__ void metric_key_kernel(const uint64_t* __restrict__ acc, int kind, long long n, uint64_t* __restrict__ key, uint32_t* __restrict__ pos) {
  PB200_GRID_LOOP(i, n) {
    const uint64_t a = acc[i];
    uint64_t k;
    if (kind == FIN_LONG) k = a ^ (1ull << 63);
    else if (kind == FIN_INT_SUM) k = double_order_bits((double)(long long)a);  // the exact int64 sum, rounded once
    else if (kind == FIN_DOUBLE) k = double_order_bits(__longlong_as_double((long long)a));
    else k = a;                                                                // MIN / MAX: already the key
    key[i] = k;
    pos[i] = (uint32_t)i;
  }
}

// limb k of an exact INT sum x (|x| < 2^62): x = l2 * 2^42 + l1 * 2^21 + l0, l0 and l1 in [0, 2^21), l2 signed
__global__ void limb_kernel(const uint64_t* __restrict__ acc, int k, long long n, uint32_t* __restrict__ out) {
  PB200_GRID_LOOP(i, n) {
    const long long x = (long long)acc[i];
    out[i] = k == 2 ? (uint32_t)(int32_t)(x >> 42) : (uint32_t)((x >> (21 * k)) & 0x1FFFFF);
  }
}

__global__ void key_flag_kernel(const uint64_t* __restrict__ key, long long n, uint32_t* __restrict__ flags) {
  PB200_GRID_LOOP(i, n) flags[i] = i > 0 && key[i] != key[i - 1];
}

// ranks -> ids[doc]; each distinct key once as its native value (LONG: the int64, DOUBLE: the bits, NaN canonical)
__global__ void rank_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ pos, const uint32_t* __restrict__ rank,
                            long long n, bool is_long, uint32_t* __restrict__ ids, uint64_t* __restrict__ dict) {
  PB200_GRID_LOOP(i, n) {
    const uint32_t r = rank[i];
    ids[pos[i]] = r;
    if (i == 0 || key[i] != key[i - 1]) {
      const uint64_t k = key[i];
      dict[r] = is_long ? k ^ (1ull << 63) : ((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k);
    }
  }
}

struct Range { uint32_t start, end, owner; };

class Builder {
 public:
  Builder(pb200_ctx* c, cudaStream_t s, int nd, const std::vector<int>& acc) : ctx(c), st(s), D(nd), acc_(acc) {
    blocks = ctx->sm_count * 8;
  }
  ~Builder() {
    cudaStreamSynchronize(st);
    for (auto* p : dim) dev_free(ctx, p);
    for (auto* p : met) dev_free(ctx, p);
  }
  pb200_ctx* ctx;
  cudaStream_t st;
  int D, blocks;
  std::vector<int> acc_;
  std::vector<uint32_t*> dim;  // star docs: per dimension the dictIds, per metric the accumulators; `cap` entries each
  std::vector<uint64_t*> met;
  long long cap = 0, total = 0;

  int grow(long long need) {
    if (need <= cap) return PB200_OK;
    const long long nc = std::max(need, cap + cap / 2);
    std::vector<uint32_t*> nd(D, nullptr);
    std::vector<uint64_t*> nm(acc_.size(), nullptr);
    int rc = PB200_OK;
    for (int j = 0; j < D && !rc; j++) rc = dev_alloc(ctx, (size_t)nc * 4, (void**)&nd[j]);
    for (size_t m = 0; m < nm.size() && !rc; m++) rc = dev_alloc(ctx, (size_t)nc * 8, (void**)&nm[m]);
    cudaError_t e = cudaSuccess;
    for (int j = 0; j < D && !rc && total && e == cudaSuccess; j++) e = cudaMemcpyAsync(nd[j], dim[j], (size_t)total * 4, cudaMemcpyDeviceToDevice, st);
    for (size_t m = 0; m < nm.size() && !rc && total && e == cudaSuccess; m++) e = cudaMemcpyAsync(nm[m], met[m], (size_t)total * 8, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (!rc && e != cudaSuccess) { set_error("star-tree build: copy failed: %s", cudaGetErrorString(e)); rc = PB200_E_CUDA; }
    if (rc) { for (auto* p : nd) dev_free(ctx, p); for (auto* p : nm) dev_free(ctx, p); return rc; }
    for (auto* p : dim) dev_free(ctx, p);
    for (auto* p : met) dev_free(ctx, p);
    dim = nd; met = nm; cap = nc;
    return PB200_OK;
  }

  // One pass (see the top of the file).  sdim / smet: the source docs (the rows for the base pass, else the star docs).
  // children_dim >= 0: report the runs of that dimension (start doc, value, owner) in `runs_out` and emit nothing.
  // Otherwise the runs become docs [total, total + R) and owner_first / owner_end receive each owner's new docs.
  int pass(const std::vector<Range>& ranges, int num_owners, const uint32_t* const* sdim, const uint64_t* const* smet,
           const std::vector<int>& key_dims, bool sort, int z0, int z1, int children_dim, std::vector<uint32_t>* runs_out,
           std::vector<uint32_t>* owner_first, std::vector<uint32_t>* owner_end) {
    const int nr = (int)ranges.size();
    std::vector<uint32_t> hr(3ull * nr + 1);
    long long n = 0;
    for (int r = 0; r < nr; r++) { hr[r] = ranges[r].start; hr[nr + r] = (uint32_t)n; hr[2 * nr + 1 + r] = ranges[r].owner; n += ranges[r].end - ranges[r].start; }
    hr[2 * nr] = (uint32_t)n;
    if (n == 0) { if (runs_out) runs_out->clear(); return PB200_OK; }
    const bool emit = children_dim < 0;
    if (emit) {  // a pass makes at most one doc per item
      if (total >= INT_MAX) { set_error("star-tree build: 2^31 or more star docs"); return PB200_E_UNSUPPORTED; }
      if (int rc = grow(std::min<long long>(total + n, INT_MAX))) return rc;
    }
    if (sdim == nullptr) { sdim = (const uint32_t* const*)dim.data(); smet = (const uint64_t* const*)met.data(); }
    KeyCols keys{};
    keys.n = (int)key_dims.size();
    int key_bits = 0;
    for (int j = 0; j < keys.n; j++) { keys.p[j] = sdim[key_dims[j]]; keys.bits[j] = bit_width[key_dims[j]]; key_bits += keys.bits[j]; }
    const int owner_bits = num_owners > 1 ? bits_for_cardinality(num_owners) : 0;
    sort = sort && keys.n > 0;
    const bool key64 = owner_bits + key_bits <= 64;

    size_t t_sort = 0, t_scan = 0, t_red = 0, t = 0;
    if (sort && key64) cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
    if (sort && !key64) cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
    cub::DeviceScan::InclusiveSum(nullptr, t_scan, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
    if (emit) cub::DeviceReduce::ReduceByKey(nullptr, t_red, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint64_t*)nullptr,
                                             (uint64_t*)nullptr, (uint32_t*)nullptr, SumF64(), (int)n);
    t = std::max({t_sort, t_scan, t_red, (size_t)16});
    DevBufRaw b_ranges(ctx), b_items(ctx), b_owner(ctx), b_items2(ctx), b_owner2(ctx), b_perm(ctx), b_perm2(ctx), b_key(ctx),
        b_key2(ctx), b_flags(ctx), b_run(ctx), b_first(ctx), b_vals(ctx), b_temp(ctx), b_small(ctx), b_out(ctx);
    int rc = PB200_OK;
    const size_t n4 = (size_t)n * 4;
    if (!rc) rc = b_ranges.alloc(hr.size() * 4);
    if (!rc) rc = b_items.alloc(n4);
    if (!rc) rc = b_owner.alloc(n4);
    if (!rc) rc = b_flags.alloc(n4);
    if (!rc) rc = b_run.alloc(n4);
    if (!rc) rc = b_first.alloc(n4);
    if (!rc) rc = b_temp.alloc(t);
    if (!rc) rc = b_small.alloc(16 + 8ull * num_owners);
    if (!rc && sort) rc = b_items2.alloc(n4);
    if (!rc && sort) rc = b_owner2.alloc(n4);
    if (!rc && sort) rc = b_perm.alloc(n4);
    if (!rc && sort) rc = b_perm2.alloc(n4);
    if (!rc && sort) rc = b_key.alloc((size_t)n * (key64 ? 8 : 4));
    if (!rc && sort) rc = b_key2.alloc((size_t)n * (key64 ? 8 : 4));
    if (!rc && emit) rc = b_vals.alloc((size_t)n * 8);
    if (!rc && !emit) rc = b_out.alloc(n4 * 3);
    if (rc) return rc;
    struct Drain { cudaStream_t s; ~Drain() { cudaStreamSynchronize(s); } } drain{st};  // before the scratch goes back to the pool
    uint32_t* items = (uint32_t*)b_items.p;
    uint32_t* owner = (uint32_t*)b_owner.p;
    const uint32_t* rg = (const uint32_t*)b_ranges.p;
    const int grid = (int)std::min<long long>((n + kThreads - 1) / kThreads, blocks);
    PB200_CUDA(cudaMemcpyAsync(b_ranges.p, hr.data(), hr.size() * 4, cudaMemcpyHostToDevice, st));
    expand_kernel<<<grid, kThreads, 0, st>>>(rg, rg + nr, rg + 2 * nr + 1, nr, n, items, owner);
    PB200_CUDA(cudaGetLastError());
    if (sort) {
      uint32_t* perm = (uint32_t*)b_perm.p;
      uint32_t* perm2 = (uint32_t*)b_perm2.p;
      if (key64) {
        key64_kernel<<<grid, kThreads, 0, st>>>(items, owner, owner_bits, keys, n, (uint64_t*)b_key.p, perm2);
        PB200_CUDA(cudaGetLastError());
        PB200_CUDA(cub::DeviceRadixSort::SortPairs(b_temp.p, t_sort, (const uint64_t*)b_key.p, (uint64_t*)b_key2.p, (const uint32_t*)perm2,
                                                   perm, (int)n, 0, owner_bits + key_bits, st));
      } else {  // stable passes, least significant column first, the owner last
        iota_kernel<<<grid, kThreads, 0, st>>>(perm, n);
        PB200_CUDA(cudaGetLastError());
        std::vector<int> order;  // -1: the owner
        for (int j = keys.n - 1; j >= 0; j--) order.push_back(j);
        if (owner_bits) order.push_back(-1);
        for (int j : order) {
          const uint32_t* col = j >= 0 ? keys.p[j] : nullptr;
          const int bits = j >= 0 ? keys.bits[j] : owner_bits;
          key32_kernel<<<grid, kThreads, 0, st>>>(perm, items, owner, col, n, (uint32_t*)b_key.p);
          PB200_CUDA(cudaGetLastError());
          PB200_CUDA(cub::DeviceRadixSort::SortPairs(b_temp.p, t_sort, (const uint32_t*)b_key.p, (uint32_t*)b_key2.p, (const uint32_t*)perm,
                                                     perm2, (int)n, 0, bits, st));
          std::swap(perm, perm2);
        }
      }
      permute_kernel<<<grid, kThreads, 0, st>>>(perm, items, owner, n, (uint32_t*)b_items2.p, (uint32_t*)b_owner2.p);
      PB200_CUDA(cudaGetLastError());
      items = (uint32_t*)b_items2.p;
      owner = (uint32_t*)b_owner2.p;
    }
    uint32_t* flags = (uint32_t*)b_flags.p;
    uint32_t* run = (uint32_t*)b_run.p;
    uint32_t* first = (uint32_t*)b_first.p;
    flag_kernel<<<grid, kThreads, 0, st>>>(items, owner, keys, n, flags);
    PB200_CUDA(cudaGetLastError());
    PB200_CUDA(cub::DeviceScan::InclusiveSum(b_temp.p, t_scan, (const uint32_t*)flags, run, (int)n, st));
    first_kernel<<<grid, kThreads, 0, st>>>(flags, run, n, first);
    PB200_CUDA(cudaGetLastError());
    uint32_t runs32 = 0;
    PB200_CUDA(cudaMemcpyAsync(&runs32, run + n - 1, 4, cudaMemcpyDeviceToHost, st));
    PB200_CUDA(cudaStreamSynchronize(st));
    const long long runs = runs32;
    const int rgrid = (int)std::min<long long>((runs + kThreads - 1) / kThreads, blocks);
    if (!emit) {
      children_kernel<<<rgrid, kThreads, 0, st>>>(first, items, owner, sdim[children_dim], runs, (uint32_t*)b_out.p);
      PB200_CUDA(cudaGetLastError());
      runs_out->resize(3 * runs);
      PB200_CUDA(cudaMemcpyAsync(runs_out->data(), b_out.p, 12ull * runs, cudaMemcpyDeviceToHost, st));
      PB200_CUDA(cudaStreamSynchronize(st));
      return PB200_OK;
    }
    if (total + runs > INT_MAX) { set_error("star-tree build: 2^31 or more star docs"); return PB200_E_UNSUPPORTED; }
    DimPtrs src{};
    OutDims dst{};
    for (int j = 0; j < D; j++) { src.p[j] = sdim[j]; dst.p[j] = dim[j]; }
    uint32_t* of = (uint32_t*)b_small.p + 4;
    emit_kernel<<<rgrid, kThreads, 0, st>>>(first, items, owner, runs, src, dst, D, z0, z1, total, of, of + num_owners);
    PB200_CUDA(cudaGetLastError());
    uint64_t* vals = (uint64_t*)b_vals.p;
    for (size_t m = 0; m < met.size(); m++) {
      gather_kernel<<<grid, kThreads, 0, st>>>(items, smet[m], n, vals);
      PB200_CUDA(cudaGetLastError());
      uint64_t* out = met[m] + total;
      uint32_t* nruns = (uint32_t*)b_small.p;
      cudaError_t e;
      switch (acc_[m]) {
        case ACC_I64: e = cub::DeviceReduce::ReduceByKey(b_temp.p, t_red, (const uint32_t*)run, (uint32_t*)flags, (const uint64_t*)vals, out, nruns, SumI64(), (int)n, st); break;
        case ACC_F64: e = cub::DeviceReduce::ReduceByKey(b_temp.p, t_red, (const uint32_t*)run, (uint32_t*)flags, (const uint64_t*)vals, out, nruns, SumF64(), (int)n, st); break;
        case ACC_MIN: e = cub::DeviceReduce::ReduceByKey(b_temp.p, t_red, (const uint32_t*)run, (uint32_t*)flags, (const uint64_t*)vals, out, nruns, MinU64(), (int)n, st); break;
        default: e = cub::DeviceReduce::ReduceByKey(b_temp.p, t_red, (const uint32_t*)run, (uint32_t*)flags, (const uint64_t*)vals, out, nruns, MaxU64(), (int)n, st);
      }
      PB200_CUDA(e);
    }
    owner_first->resize(num_owners);
    owner_end->resize(num_owners);
    PB200_CUDA(cudaMemcpyAsync(owner_first->data(), of, 4ull * num_owners, cudaMemcpyDeviceToHost, st));
    PB200_CUDA(cudaMemcpyAsync(owner_end->data(), of + num_owners, 4ull * num_owners, cudaMemcpyDeviceToHost, st));
    PB200_CUDA(cudaStreamSynchronize(st));
    total += runs;
    return PB200_OK;
  }

  std::vector<int> bit_width;  // per dimension: bits of its dictIds
};

struct Node { int dim, value; uint32_t start, end; int agg = -1, first = -1, last = -1; };

inline void put_be(unsigned char* p, uint64_t v, int w) { for (int b = 0; b < w; b++) p[b] = (unsigned char)(v >> (8 * (w - 1 - b))); }

// star docs -> device segment columns: dimensions packed at their base bits sharing the base dictionaries, metrics
// dictionary-encoded (sort -> flags -> scan -> rank, as derived columns are)
int encode_segment(pb200_ctx* ctx, cudaStream_t st, const pb200_segment* seg, const StarBuildSpec& spec, Builder& b,
                   pb200_segment** out, std::vector<int>* limb_col) {
  const long long T = b.total;
  const int blocks = ctx->sm_count * 8;
  std::unique_ptr<pb200_segment> s(new pb200_segment());
  const int D = (int)spec.dim_cols.size(), M = (int)spec.metric_fn.size();
  s->ctx = ctx;
  s->name = seg->name + "$startree";
  s->num_docs = (int)T;
  s->cols.reserve((size_t)D + 4 * M + PB200_MAX_DERIVED_COLUMNS);
  struct FreeOnFail {
    pb200_ctx* ctx; cudaStream_t st; pb200_segment* s; bool armed = true;
    ~FreeOnFail() {
      if (!armed) return;
      cudaStreamSynchronize(st);
      for (auto& c : s->cols) { dev_free(ctx, c.fwd); dev_free(ctx, c.dict_native); }
    }
  } guard{ctx, st, s.get()};
  auto pack = [&](const uint32_t* v, int bits, DeviceColumn& c) -> int {
    c.fwd_kind = PB200_FWD_DICT_FIXEDBIT;
    c.bits = bits;
    c.fwd_alloc_bytes = padded_fwd_bytes(T, bits);
    c.fwd_file_bytes = ((uint64_t)T * bits + 7) / 8;
    c.pooled = true;
    if (int rc = dev_alloc(ctx, c.fwd_alloc_bytes, (void**)&c.fwd)) return rc;
    PB200_CUDA(cudaMemsetAsync(c.fwd, 0, c.fwd_alloc_bytes, st));
    const long long groups = (T + 31) / 32;
    pack_kernel<<<(int)std::min<long long>((groups + kThreads - 1) / kThreads, blocks), kThreads, 0, st>>>(v, T, bits, groups, c.fwd);
    PB200_CUDA(cudaGetLastError());
    s->device_bytes += (int64_t)c.fwd_alloc_bytes;
    return PB200_OK;
  };
  for (int j = 0; j < D; j++) {
    const DeviceColumn& base = seg->cols[spec.dim_cols[j]];
    s->cols.emplace_back();
    DeviceColumn& c = s->cols.back();
    c.stored_type = base.stored_type; c.cardinality = base.cardinality;
    c.dict_entry_bytes = base.dict_entry_bytes; c.dict_be = base.dict_be; c.dict_host = base.dict_host; c.dict_hash = base.dict_hash;
    if (int rc = pack(b.dim[j], base.bits, c)) return rc;
    if (base.dict_native) {
      const size_t bytes = std::max<size_t>((size_t)c.dict_width() * c.cardinality, 16);
      if (int rc = dev_alloc(ctx, bytes, &c.dict_native)) return rc;
      PB200_CUDA(cudaMemcpyAsync(c.dict_native, base.dict_native, (size_t)c.dict_width() * c.cardinality, cudaMemcpyDeviceToDevice, st));
      s->device_bytes += (int64_t)c.dict_host.size();
    }
  }
  size_t t_sort = 0, t_scan = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)T);
  cub::DeviceScan::InclusiveSum(nullptr, t_scan, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)T);
  DevBufRaw key(ctx), key2(ctx), pos(ctx), pos2(ctx), flags(ctx), rank(ctx), ids(ctx), dict(ctx), temp(ctx);
  int rc = PB200_OK;
  if (!rc) rc = key.alloc((size_t)T * 8);
  if (!rc) rc = key2.alloc((size_t)T * 8);
  if (!rc) rc = pos.alloc((size_t)T * 4);
  if (!rc) rc = pos2.alloc((size_t)T * 4);
  if (!rc) rc = flags.alloc((size_t)T * 4);
  if (!rc) rc = rank.alloc((size_t)T * 4);
  if (!rc) rc = ids.alloc((size_t)T * 4);
  if (!rc) rc = dict.alloc((size_t)T * 8);
  if (!rc) rc = temp.alloc(std::max({t_sort, t_scan, (size_t)16}));
  if (rc) return rc;
  struct Drain { cudaStream_t s; ~Drain() { cudaStreamSynchronize(s); } } drain{st};
  const int grid = (int)std::min<long long>((T + kThreads - 1) / kThreads, blocks);
  for (int m = 0; m < M; m++) {
    const bool is_long = spec.metric_fn[m] == PB200_AGG_COUNT;
    const int fin = is_long ? FIN_LONG : b.acc_[m] == ACC_I64 ? FIN_INT_SUM : b.acc_[m] == ACC_F64 ? FIN_DOUBLE : FIN_KEY;
    metric_key_kernel<<<grid, kThreads, 0, st>>>(b.met[m], fin, T, (uint64_t*)key.p, (uint32_t*)pos.p);
    PB200_CUDA(cudaGetLastError());
    PB200_CUDA(cub::DeviceRadixSort::SortPairs(temp.p, t_sort, (const uint64_t*)key.p, (uint64_t*)key2.p, (const uint32_t*)pos.p, (uint32_t*)pos2.p, (int)T, 0, 64, st));
    key_flag_kernel<<<grid, kThreads, 0, st>>>((const uint64_t*)key2.p, T, (uint32_t*)flags.p);
    PB200_CUDA(cudaGetLastError());
    PB200_CUDA(cub::DeviceScan::InclusiveSum(temp.p, t_scan, (const uint32_t*)flags.p, (uint32_t*)rank.p, (int)T, st));
    rank_kernel<<<grid, kThreads, 0, st>>>((const uint64_t*)key2.p, (const uint32_t*)pos2.p, (const uint32_t*)rank.p, T, is_long,
                                           (uint32_t*)ids.p, (uint64_t*)dict.p);
    PB200_CUDA(cudaGetLastError());
    uint32_t last = 0;
    PB200_CUDA(cudaMemcpyAsync(&last, (uint32_t*)rank.p + T - 1, 4, cudaMemcpyDeviceToHost, st));
    PB200_CUDA(cudaStreamSynchronize(st));
    const int card = (int)last + 1;
    s->cols.emplace_back();
    DeviceColumn& c = s->cols.back();
    c.stored_type = is_long ? PB200_LONG : PB200_DOUBLE;
    c.cardinality = card;
    c.dict_entry_bytes = 8;
    c.dict_host.resize(8ull * card);
    if (int r2 = dev_alloc(ctx, std::max<size_t>(8ull * card, 16), &c.dict_native)) return r2;
    PB200_CUDA(cudaMemcpyAsync(c.dict_native, dict.p, 8ull * card, cudaMemcpyDeviceToDevice, st));
    PB200_CUDA(cudaMemcpyAsync(c.dict_host.data(), dict.p, 8ull * card, cudaMemcpyDeviceToHost, st));
    if (int r2 = pack((const uint32_t*)ids.p, bits_for_cardinality(card), c)) return r2;
    PB200_CUDA(cudaStreamSynchronize(st));
    c.dict_be.resize(8ull * card);
    for (int i = 0; i < card; i++) { uint64_t v; memcpy(&v, &c.dict_host[8ull * i], 8); put_be(&c.dict_be[8ull * i], v, 8); }
    c.dict_hash = dictionary_hash(c.stored_type, 8, card, c.dict_be.data());
    s->device_bytes += (int64_t)c.dict_host.size();
  }
  // an INT SUM's exact sums, also as three raw INT limb columns (see StarBuildResult::limb_col)
  limb_col->assign(M, -1);
  for (int m = 0; m < M; m++) {
    if (spec.metric_fn[m] != PB200_AGG_SUM || b.acc_[m] != ACC_I64) continue;
    (*limb_col)[m] = (int)s->cols.size();
    for (int k = 0; k < 3; k++) {
      limb_kernel<<<grid, kThreads, 0, st>>>(b.met[m], k, T, (uint32_t*)ids.p);
      PB200_CUDA(cudaGetLastError());
      s->cols.emplace_back();
      DeviceColumn& c = s->cols.back();
      c.stored_type = PB200_INT;
      if (int r2 = pack((const uint32_t*)ids.p, 32, c)) return r2;
      c.fwd_kind = PB200_FWD_RAW_FIXEDBYTE;   // bits 32 and no dictionary: the scan reads signed words (VAL_RAW_I32)
    }
  }
  const int ncols = (int)s->cols.size();
  s->num_stored = ncols;
  PB200_CUDA(cudaStreamSynchronize(st));
  s->published.store(ncols, std::memory_order_release);
  guard.armed = false;
  *out = s.release();
  return PB200_OK;
}

}  // namespace

int startree_build(pb200_ctx* ctx, const pb200_segment* seg, const StarBuildSpec& spec, StarBuildResult* out) {
  const int D = (int)spec.dim_cols.size(), M = (int)spec.metric_fn.size();
  const long long N = seg->num_docs;
  if (D < 1 || D > kMaxDims || M < 1) { set_error("star-tree build: %d dimensions, %d metrics", D, M); return PB200_E_UNSUPPORTED; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  StreamLease st(ctx);
  std::vector<int> acc(M);
  for (int m = 0; m < M; m++) {
    const int fn = spec.metric_fn[m];
    const bool int_col = spec.metric_col[m] >= 0 && seg->cols[spec.metric_col[m]].stored_type == PB200_INT;
    acc[m] = fn == PB200_AGG_COUNT || (fn == PB200_AGG_SUM && int_col) ? ACC_I64 : fn == PB200_AGG_SUM ? ACC_F64 : fn == PB200_AGG_MIN ? ACC_MIN : ACC_MAX;
  }
  Builder b(ctx, st, D, acc);
  for (int j = 0; j < D; j++) b.bit_width.push_back(seg->cols[spec.dim_cols[j]].bits);
  const int blocks = ctx->sm_count * 8;
  const int grid = (int)std::min<long long>((N + kThreads - 1) / kThreads, blocks);
  double t0 = host_ms();

  // ---- 1. base docs: the rows sorted by the split order, identical dimension tuples merged -----------------------
  {
    std::vector<std::unique_ptr<DevBufRaw>> rows;  // the rows' dimensions and metric accumulators
    std::vector<const uint32_t*> sdim;
    std::vector<const uint64_t*> smet;
    for (int j = 0; j < D; j++) {
      rows.emplace_back(new DevBufRaw(ctx));
      if (int rc = rows.back()->alloc((size_t)N * 4)) return rc;
      const DeviceColumn& c = seg->cols[spec.dim_cols[j]];
      unpack_kernel<<<grid, kThreads, 0, st>>>(c.fwd, c.bits, N, (uint32_t*)rows.back()->p);
      PB200_CUDA(cudaGetLastError());
      sdim.push_back((const uint32_t*)rows.back()->p);
    }
    for (int m = 0; m < M; m++) {
      rows.emplace_back(new DevBufRaw(ctx));
      if (int rc = rows.back()->alloc((size_t)N * 8)) return rc;
      int src = SRC_COUNT, bits = 0, type = PB200_INT;
      const uint32_t* fwd = nullptr;
      const void* dict = nullptr;
      if (spec.metric_col[m] >= 0) {
        const DeviceColumn& c = seg->cols[spec.metric_col[m]];
        src = c.fwd_kind == PB200_FWD_RAW_FIXEDBYTE ? SRC_RAW32 : SRC_DICT;
        fwd = c.fwd; bits = c.bits; type = c.stored_type; dict = c.dict_native;
      }
      row_metric_kernel<<<grid, kThreads, 0, st>>>(src, fwd, bits, dict, type, acc[m], N, (uint64_t*)rows.back()->p);
      PB200_CUDA(cudaGetLastError());
      smet.push_back((const uint64_t*)rows.back()->p);
    }
    std::vector<int> all(D);
    for (int j = 0; j < D; j++) all[j] = j;
    std::vector<uint32_t> f, e;
    struct Drain { cudaStream_t s; ~Drain() { cudaStreamSynchronize(s); } } drain{st};
    if (int rc = b.pass({{0u, (uint32_t)N, 0u}}, 1, sdim.data(), smet.data(), all, true, 0, 0, -1, nullptr, &f, &e)) return rc;
  }
  out->num_base_docs = b.total;
  double t1 = host_ms();
  out->ms[STAR_PHASE_BASE] = t1 - t0;

  // ---- 2. construction, level by level (constructStarTree) ---------------------------------------------------------
  std::vector<Node> nodes;
  nodes.push_back(Node{-1, -1, 0u, (uint32_t)b.total});
  std::vector<std::pair<int, int>> levels{{0, 1}};
  std::vector<int> split{0};  // the root is always split on dimension 0
  for (int cd = 0; cd < D && !split.empty(); cd++) {
    const int K = (int)split.size();
    std::vector<Range> ranges(K);
    for (int k = 0; k < K; k++) ranges[k] = {nodes[split[k]].start, nodes[split[k]].end, (uint32_t)k};
    std::vector<uint32_t> ch;
    if (int rc = b.pass(ranges, K, nullptr, nullptr, {cd}, false, 0, 0, cd, &ch, nullptr, nullptr)) return rc;
    const size_t C = ch.size() / 3;
    const uint32_t* cstart = ch.data();
    const uint32_t* cvalue = ch.data() + C;
    const uint32_t* cowner = ch.data() + 2 * C;
    std::vector<int> nchild(K, 0);
    for (size_t c = 0; c < C; c++) nchild[cowner[c]]++;
    std::vector<Range> star_ranges;
    std::vector<int> star_of(K, -1);
    if (!spec.skip_star[cd])
      for (int k = 0; k < K; k++)
        if (nchild[k] > 1) { star_of[k] = (int)star_ranges.size(); star_ranges.push_back({ranges[k].start, ranges[k].end, (uint32_t)star_ranges.size()}); }
    std::vector<uint32_t> sfirst, send;
    if (!star_ranges.empty()) {
      std::vector<int> rest;
      for (int j = cd + 1; j < D; j++) rest.push_back(j);
      if (int rc = b.pass(star_ranges, (int)star_ranges.size(), nullptr, nullptr, rest, true, cd, cd + 1, -1, nullptr, &sfirst, &send)) return rc;
    }
    const int level_begin = (int)nodes.size();
    size_t c = 0;
    for (int k = 0; k < K; k++) {
      const int parent = split[k];
      const int first = (int)nodes.size();
      if (star_of[k] >= 0) nodes.push_back(Node{cd, -1, sfirst[star_of[k]], send[star_of[k]]});
      for (; c < C && cowner[c] == (uint32_t)k; c++) {
        const uint32_t end = (c + 1 < C && cowner[c + 1] == (uint32_t)k) ? cstart[c + 1] : nodes[parent].end;
        nodes.push_back(Node{cd, (int)cvalue[c], cstart[c], end});
      }
      nodes[parent].first = first;
      nodes[parent].last = (int)nodes.size() - 1;
    }
    levels.push_back({level_begin, (int)nodes.size()});
    std::vector<int> next;
    if (cd + 1 < D)
      for (int id = level_begin; id < (int)nodes.size(); id++)
        if ((long long)nodes[id].end - nodes[id].start > spec.max_leaf_records) next.push_back(id);
    split.swap(next);
  }
  double t2 = host_ms();
  out->ms[STAR_PHASE_CONSTRUCT] = t2 - t1;

  // ---- 3. aggregated docs, deepest level first (createAggregatedDocs) -------------------------------------------
  for (int L = (int)levels.size() - 1; L >= 0; L--) {
    std::vector<Range> ranges;
    std::vector<int> owners;
    for (int id = levels[L].first; id < levels[L].second; id++) {
      Node& nd = nodes[id];
      if (nd.first < 0) {
        if (nd.end - nd.start == 1) { nd.agg = (int)nd.start; continue; }
        ranges.push_back({nd.start, nd.end, (uint32_t)owners.size()});
      } else if (nodes[nd.first].value == -1) {
        nd.agg = nodes[nd.first].agg;
        continue;
      } else {
        for (int ch = nd.first; ch <= nd.last; ch++) ranges.push_back({(uint32_t)nodes[ch].agg, (uint32_t)nodes[ch].agg + 1, (uint32_t)owners.size()});
      }
      owners.push_back(id);
    }
    if (owners.empty()) continue;
    std::vector<uint32_t> f, e;
    // the nodes of level L split on dimension L - 1: their aggregated docs zero dimensions L.. (the root's: all)
    if (int rc = b.pass(ranges, (int)owners.size(), nullptr, nullptr, {}, false, L, D, -1, nullptr, &f, &e)) return rc;
    for (size_t k = 0; k < owners.size(); k++) nodes[owners[k]].agg = (int)f[k];
  }
  double t3 = host_ms();
  out->ms[STAR_PHASE_AGGREGATE] = t3 - t2;

  // ---- 4. the star docs as a device segment --------------------------------------------------------------------
  pb200_segment* docs = nullptr;
  if (int rc = encode_segment(ctx, st, seg, spec, b, &docs, &out->limb_col)) return rc;
  out->ms[STAR_PHASE_ENCODE] = host_ms() - t3;
  out->nodes.resize(7 * nodes.size());
  for (size_t i = 0; i < nodes.size(); i++) {
    const Node& nd = nodes[i];
    int32_t* r = &out->nodes[7 * i];
    r[0] = nd.dim; r[1] = nd.value; r[2] = i ? (int32_t)nd.start : -1; r[3] = i ? (int32_t)nd.end : -1;
    r[4] = nd.agg; r[5] = nd.first; r[6] = nd.last;
  }
  out->docs = docs;
  return PB200_OK;
}

}  // namespace pb200
