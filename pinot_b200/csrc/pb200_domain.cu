// pb200_domain.cu -- table-wide dictionaries ("dictionary domains"): the common key space that makes per-segment results
// mergeable BY VALUE on the device and across GPUs.
//
// In the reference dictIds are segment local and every cross-segment merge goes through VALUES: GroupByCombineOperator
// upserts Key(Object[] values) into an IndexedTable (core/operator/combine/GroupByCombineOperator.java:130-146,
// core/data/table/IndexedTable.java:101-136), MIN / MAX merge doubles, DISTINCTCOUNT merges value sets
// (BaseDistinctAggregateAggregationFunction.java:109-121).  A dense device table indexed by dictIds, an NCCL reduce of
// such tables, or a dictId bitset can only be merged when all contributors share ONE id space.  A domain provides it:
//
//   * pb200_domain_create          sorted union of any number of sorted per-segment dictionaries per column (Pinot's
//                                  dictionary order: numeric ascending / Float.compare order / unpadded UTF-8 bytes);
//   * pb200_segment_bind_domain    once, at segment load: dictId -> globalId remap (both sides sorted: one merge walk),
//                                  the column's forward index is RE-ENCODED into global ids by one streaming kernel
//                                  (unpack, remap gather, repack with the domain's bit width) and the column adopts the
//                                  domain's dictionary, which is shared by all bound segments (one copy in HBM / L2);
//   * afterwards a bound segment simply IS a segment whose dictionary is the table-wide one: the scan kernel needs no
//     per-row remap, PB200_Q_MERGE_SEGMENTS and the cross-GPU reduce are merges by value.
#include <cuda_runtime.h>

#include <algorithm>
#include <memory>
#include <cstring>
#include <string>

#include "pb200_internal.h"

namespace pb200 {

uint64_t fnv1a(const void* p, size_t n, uint64_t h) {
  const unsigned char* b = static_cast<const unsigned char*>(p);
  for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 0x100000001B3ull; }
  return h;
}

// Content hash of a dictionary: equal for equal value sequences (STRING entries are hashed without their padding, so the
// per-segment lengthOfEachEntry does not matter).  Never 0 (0 = "no dictionary known").
uint64_t dictionary_hash(int stored_type, int entry_bytes, int cardinality, const unsigned char* be) {
  uint64_t h = fnv1a(&stored_type, sizeof stored_type, 0xCBF29CE484222325ull);
  h = fnv1a(&cardinality, sizeof cardinality, h);
  if (stored_type == PB200_STRING) {
    for (int i = 0; i < cardinality; i++) {
      const unsigned char* e = be + (size_t)i * entry_bytes;
      int n = 0;
      while (n < entry_bytes && e[n]) n++;
      h = fnv1a(e, n, h);
      h = fnv1a("\0", 1, h);
    }
  } else {
    h = fnv1a(be, (size_t)cardinality * entry_bytes, h);
  }
  return h ? h : 1;
}

int bits_for_cardinality(int card) {  // PinotDataBitSet.getNumBitsPerValue(card - 1), seglocal/io/util/PinotDataBitSet.java:61-72
  int b = 1;
  while (b < 31 && (1ll << b) < card) b++;
  return b;
}

namespace {

inline uint32_t rd32(const unsigned char* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
inline uint64_t rd64(const unsigned char* p) { return (uint64_t)rd32(p) << 32 | rd32(p + 4); }

// Order key of a fixed-width dictionary entry: comparing keys as unsigned integers == the order Pinot sorted the
// dictionary in (Integer / Long natural order; Float.compare / Double.compare order incl. -0.0 < 0.0).  Every NaN bit
// pattern gets the canonical NaN's key (floatToIntBits / doubleToLongBits): one value, after +inf.  A dictionary written
// by Java stores the raw bits of the first NaN it saw, so its last entry may be a NaN with the sign bit set.
inline uint64_t order_key(int type, const unsigned char* e) {
  switch (type) {
    case PB200_INT: return (uint64_t)(rd32(e) ^ 0x80000000u);
    case PB200_LONG: return rd64(e) ^ 0x8000000000000000ull;
    case PB200_FLOAT: {
      uint32_t u = rd32(e);
      if ((u & 0x7FFFFFFFu) > 0x7F800000u) u = 0x7FC00000u;
      return (uint64_t)((u & 0x80000000u) ? ~u : (u | 0x80000000u));
    }
    default: {
      uint64_t u = rd64(e);
      if ((u & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull) u = 0x7FF8000000000000ull;
      return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
    }
  }
}
inline std::string unpadded(const unsigned char* e, int width) {
  int n = 0;
  while (n < width && e[n]) n++;
  return std::string(reinterpret_cast<const char*>(e), n);
}

// Re-encodes a fixed-bit column: value i of the source stream (sb bits, native-word HBM layout of pb200_unpack.cuh) is
// replaced by remap[value] and written as db bits.  One thread per 32-row group (sb words in, db words out).
__global__ void reencode_kernel(const uint32_t* __restrict__ src, int sb, uint32_t* __restrict__ dst, int db,
                                const uint32_t* __restrict__ remap, uint32_t card, long long num_docs, long long groups) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
    const uint32_t* p = src + g * sb;
    uint32_t* o = dst + g * db;
    unsigned long long acc = 0;
    int nb = 0, wi = 0;
    for (int j = 0; j < 32; ++j) {
      const int bit = j * sb, k = bit >> 5, s = bit & 31;
      const uint32_t hi = p[k];
      const uint32_t lo = (s + sb > 32) ? p[k + 1] : 0u;
      const uint32_t x = __funnelshift_l(lo, hi, s) >> (32 - sb);
      const uint32_t id = (g * 32 + j < num_docs && x < card) ? remap[x] : 0u;  // padding rows stay 0
      acc = (acc << db) | id;
      nb += db;
      if (nb >= 32) { o[wi++] = (uint32_t)(acc >> (nb - 32)); nb -= 32; }
    }
  }
}

}  // namespace

uint64_t padded_fwd_bytes(long long num_docs, int bits) {
  // whole tiles for ANY tile size <= kMaxTileRows: ceil(N/t)*t < N + t <= alloc rows
  long long tiles = (num_docs + kMaxTileRows - 1) / kMaxTileRows + 1;
  return (uint64_t)tiles * kMaxTileRows / 8 * bits + 64;
}

cudaError_t reencode_column(pb200_ctx* ctx, cudaStream_t st, const uint32_t* src, int sb, uint32_t* dst, int db,
                            const uint32_t* remap, uint32_t card, long long num_docs) {
  const long long groups = (num_docs + 31) / 32;
  if (groups <= 0) return cudaSuccess;
  const int blocks = (int)std::min<long long>((groups + 255) / 256, (long long)ctx->sm_count * 16);
  reencode_kernel<<<blocks, 256, 0, st>>>(src, sb, dst, db, remap, card, num_docs, groups);
  return cudaGetLastError();
}
}  // namespace pb200

using namespace pb200;

extern "C" int32_t pb200_domain_create(pb200_ctx* ctx, int32_t ncols, const pb200_domain_col* cols, pb200_domain** out) {
  if (!ctx || !cols || !out || ncols <= 0) { set_error("invalid argument to pb200_domain_create"); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<pb200_domain> dom(new pb200_domain());
  dom->ctx = ctx;
  auto fail = [&](int rc) { for (auto& c : dom->cols) dev_free(ctx, c.dict_native); return rc; };
  for (int k = 0; k < ncols; k++) {
    const pb200_domain_col& d = cols[k];
    if (d.column < 0 || d.num_parts <= 0 || !d.parts || !d.cardinalities) { set_error("domain column %d: bad description", k); return fail(PB200_E_INVALID); }
    if (d.stored_type < PB200_INT || d.stored_type > PB200_STRING) { set_error("domain column %d: unknown type", k); return fail(PB200_E_INVALID); }
    for (auto& e : dom->cols) if (e.column == d.column) { set_error("domain lists column %d twice", d.column); return fail(PB200_E_INVALID); }
    pb200_domain::Col c;
    c.column = d.column;
    c.stored_type = d.stored_type;
    const bool str = d.stored_type == PB200_STRING;
    const int fixed = (d.stored_type == PB200_LONG || d.stored_type == PB200_DOUBLE) ? 8 : 4;
    if (!str) {
      // k-way union of sorted parts == sort + unique of their order keys (parts are small next to the columns)
      std::vector<std::pair<uint64_t, const unsigned char*>> all;
      for (int p = 0; p < d.num_parts; p++) {
        const unsigned char* b = static_cast<const unsigned char*>(d.parts[p]);
        if (!b && d.cardinalities[p] > 0) { set_error("domain column %d: part %d is NULL", k, p); return fail(PB200_E_INVALID); }
        uint64_t prev = 0;
        for (int i = 0; i < d.cardinalities[p]; i++) {
          const uint64_t key = order_key(d.stored_type, b + (size_t)i * fixed);
          if (i && key <= prev) { set_error("domain column %d: part %d is not a sorted dictionary", k, p); return fail(PB200_E_INVALID); }
          prev = key;
          all.emplace_back(key, b + (size_t)i * fixed);
        }
      }
      // stable: of entries with one key (NaNs with different bits), the first part's is the domain's entry
      std::stable_sort(all.begin(), all.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
      all.erase(std::unique(all.begin(), all.end(), [](const auto& a, const auto& b) { return a.first == b.first; }), all.end());
      c.entry_bytes = fixed;
      c.cardinality = (int)all.size();
      c.dict_be.resize((size_t)fixed * all.size());
      for (size_t i = 0; i < all.size(); i++) memcpy(&c.dict_be[i * fixed], all[i].second, fixed);
    } else {
      std::vector<std::string> all;
      size_t width = 1;
      for (int p = 0; p < d.num_parts; p++) {
        const int w = d.entry_bytes ? d.entry_bytes[p] : 0;
        const unsigned char* b = static_cast<const unsigned char*>(d.parts[p]);
        if (w <= 0 || (!b && d.cardinalities[p] > 0)) { set_error("domain column %d: STRING part %d needs its entry width", k, p); return fail(PB200_E_INVALID); }
        for (int i = 0; i < d.cardinalities[p]; i++) { all.push_back(unpadded(b + (size_t)i * w, w)); width = std::max(width, all.back().size()); }
      }
      std::sort(all.begin(), all.end());  // std::string compares bytes as unsigned char: UTF-8 byte order
      all.erase(std::unique(all.begin(), all.end()), all.end());
      c.entry_bytes = (int)width;
      c.cardinality = (int)all.size();
      c.dict_be.assign(width * all.size(), 0);
      for (size_t i = 0; i < all.size(); i++) memcpy(&c.dict_be[i * width], all[i].data(), all[i].size());
    }
    if (c.cardinality <= 0) { set_error("domain column %d: empty dictionary", k); return fail(PB200_E_INVALID); }
    c.bits = bits_for_cardinality(c.cardinality);
    c.hash = dictionary_hash(c.stored_type, c.entry_bytes, c.cardinality, c.dict_be.data());
    if (!str) {  // native host copy + device copy (INT: biased, see convert_dictionary in pb200_api.cu)
      c.dict_host.resize(c.dict_be.size());
      std::vector<unsigned char> dev(c.dict_be.size());
      for (int i = 0; i < c.cardinality; i++) {
        if (fixed == 4) {
          uint32_t v = rd32(&c.dict_be[4ull * i]);
          memcpy(&c.dict_host[4ull * i], &v, 4);
          if (c.stored_type == PB200_INT) v ^= 0x80000000u;
          memcpy(&dev[4ull * i], &v, 4);
        } else {
          uint64_t v = rd64(&c.dict_be[8ull * i]);
          memcpy(&c.dict_host[8ull * i], &v, 8);
          memcpy(&dev[8ull * i], &v, 8);
        }
      }
      int rc = dev_alloc(ctx, std::max<size_t>(dev.size(), 16), &c.dict_native);
      if (rc) return fail(rc);
      if (cudaMemcpy(c.dict_native, dev.data(), dev.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
        dev_free(ctx, c.dict_native);
        set_error("domain dictionary upload failed");
        cudaGetLastError();
        return fail(PB200_E_CUDA);
      }
    }
    dom->cols.push_back(std::move(c));
  }
  *out = dom.release();
  return PB200_OK;
}

extern "C" int32_t pb200_domain_from_segments(pb200_ctx* ctx, pb200_segment* const* segs, int32_t nseg, int32_t ncols,
                                              const int32_t* columns, pb200_domain** out) {
  if (!ctx || !segs || !columns || !out || nseg <= 0 || ncols <= 0) { set_error("invalid argument to pb200_domain_from_segments"); return PB200_E_INVALID; }
  std::vector<pb200_domain_col> cols(ncols);
  std::vector<std::vector<const void*>> parts(ncols);
  std::vector<std::vector<int32_t>> cards(ncols), widths(ncols);
  for (int k = 0; k < ncols; k++) {
    for (int s = 0; s < nseg; s++) {
      if (!segs[s] || columns[k] < 0 || columns[k] >= segs[s]->num_columns()) { set_error("segment %d has no column %d", s, columns[k]); return PB200_E_INVALID; }
      const DeviceColumn& c = segs[s]->cols[columns[k]];
      if (c.dict_be.empty()) { set_error("segment %d column %d was registered without dictionary bytes", s, columns[k]); return PB200_E_INVALID; }
      if (c.stored_type != segs[0]->cols[columns[k]].stored_type) { set_error("column %d changes type between segments", columns[k]); return PB200_E_INVALID; }
      parts[k].push_back(c.dict_be.data());
      cards[k].push_back(c.cardinality);
      widths[k].push_back(c.dict_entry_bytes);
    }
    cols[k].column = columns[k];
    cols[k].stored_type = segs[0]->cols[columns[k]].stored_type;
    cols[k].num_parts = nseg;
    cols[k].parts = parts[k].data();
    cols[k].cardinalities = cards[k].data();
    cols[k].entry_bytes = widths[k].data();
  }
  return pb200_domain_create(ctx, ncols, cols.data(), out);
}

extern "C" int32_t pb200_domain_column_info(const pb200_domain* dom, int32_t column, int64_t out[4]) {
  if (!dom || !out) { set_error("null argument"); return PB200_E_INVALID; }
  for (const auto& c : dom->cols)
    if (c.column == column) { out[0] = c.stored_type; out[1] = c.cardinality; out[2] = c.bits; out[3] = c.entry_bytes; return PB200_OK; }
  set_error("column %d is not part of the domain", column);
  return PB200_E_INVALID;
}

extern "C" int64_t pb200_domain_dictionary(const pb200_domain* dom, int32_t column, void* out, uint64_t cap) {
  if (!dom) { set_error("null argument"); return PB200_E_INVALID; }
  for (const auto& c : dom->cols) {
    if (c.column != column) continue;
    if (!out) return (int64_t)c.dict_be.size();
    if (cap < c.dict_be.size()) { set_error("buffer too small"); return PB200_E_INVALID; }
    memcpy(out, c.dict_be.data(), c.dict_be.size());
    return (int64_t)c.dict_be.size();
  }
  set_error("column %d is not part of the domain", column);
  return PB200_E_INVALID;
}

extern "C" int32_t pb200_domain_release(pb200_ctx* ctx, pb200_domain* dom) {
  if (!dom) return PB200_OK;
  pb200_ctx* c = dom->ctx;
  bool last;
  { std::lock_guard<std::mutex> g(c->mu); last = --dom->refs == 0; }
  if (last) {
    cudaSetDevice(c->device);
    for (auto& col : dom->cols) dev_free(c, col.dict_native);
    delete dom;
  }
  return PB200_OK;
}

extern "C" int32_t pb200_segment_bind_domain(pb200_ctx* ctx, pb200_segment* seg, pb200_domain* dom) {
  if (!ctx || !seg || !dom || seg->ctx != ctx || dom->ctx != ctx) { set_error("invalid argument to pb200_segment_bind_domain"); return PB200_E_INVALID; }
  if (seg->domain) { set_error("segment '%s' is already bound to a domain", seg->name.c_str()); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  // ---- pass 1: validate and compute every remap before touching the segment ----
  struct Work { int col; const pb200_domain::Col* dc; std::vector<uint32_t> remap; };
  std::vector<Work> work;
  for (const auto& dc : dom->cols) {
    if (dc.column >= seg->num_columns()) { set_error("domain column %d is outside segment '%s'", dc.column, seg->name.c_str()); return PB200_E_INVALID; }
    const DeviceColumn& c = seg->cols[dc.column];
    if (c.fwd_kind != PB200_FWD_DICT_FIXEDBIT || c.bits > 31) { set_error("column %d is not dictionary-encoded: it cannot join a domain", dc.column); return PB200_E_INVALID; }
    if (c.dict_be.empty()) { set_error("column %d was registered without dictionary bytes", dc.column); return PB200_E_INVALID; }
    if (c.stored_type != dc.stored_type) { set_error("column %d: type differs from the domain's", dc.column); return PB200_E_INVALID; }
    Work w{dc.column, &dc, std::vector<uint32_t>((size_t)c.cardinality)};
    int g = 0;
    for (int l = 0; l < c.cardinality; l++) {  // both sorted in the same order: one merge walk
      if (dc.stored_type == PB200_STRING) {
        const std::string v = unpadded(&c.dict_be[(size_t)l * c.dict_entry_bytes], c.dict_entry_bytes);
        while (g < dc.cardinality && unpadded(&dc.dict_be[(size_t)g * dc.entry_bytes], dc.entry_bytes) < v) g++;
        if (g >= dc.cardinality || unpadded(&dc.dict_be[(size_t)g * dc.entry_bytes], dc.entry_bytes) != v) {
          set_error("column %d: dictionary value '%s' of segment '%s' is not in the domain", dc.column, v.c_str(), seg->name.c_str());
          return PB200_E_INVALID;
        }
      } else {
        const uint64_t key = order_key(dc.stored_type, &c.dict_be[(size_t)l * dc.entry_bytes]);
        while (g < dc.cardinality && order_key(dc.stored_type, &dc.dict_be[(size_t)g * dc.entry_bytes]) < key) g++;
        if (g >= dc.cardinality || order_key(dc.stored_type, &dc.dict_be[(size_t)g * dc.entry_bytes]) != key) {
          set_error("column %d: dictionary entry %d of segment '%s' is not in the domain", dc.column, l, seg->name.c_str());
          return PB200_E_INVALID;
        }
      }
      w.remap[l] = (uint32_t)g;
    }
    work.push_back(std::move(w));
  }
  // ---- pass 2: re-encode ----
  StreamLease st(ctx);
  for (auto& w : work) {
    DeviceColumn& c = seg->cols[w.col];
    const pb200_domain::Col& dc = *w.dc;
    // a subset of equal size is the same dictionary; a stream registered wider than the domain's width is still repacked
    const bool identity = c.cardinality == dc.cardinality && c.bits == dc.bits;
    if (!identity) {
      void* remap_dev = nullptr;
      void* nf = nullptr;
      int rc = dev_alloc(ctx, std::max<size_t>(w.remap.size() * 4, 16), &remap_dev);
      if (rc) return rc;
      const uint64_t nbytes = padded_fwd_bytes(seg->num_docs, dc.bits);
      rc = dev_alloc(ctx, nbytes, &nf);
      if (rc) { dev_free(ctx, remap_dev); return rc; }
      cudaError_t e = cudaMemcpyAsync(remap_dev, w.remap.data(), w.remap.size() * 4, cudaMemcpyHostToDevice, st);
      if (e == cudaSuccess) e = cudaMemsetAsync(nf, 0, nbytes, st);
      if (e == cudaSuccess)
        e = reencode_column(ctx, st, c.fwd, c.bits, (uint32_t*)nf, dc.bits, (const uint32_t*)remap_dev, (uint32_t)c.cardinality, seg->num_docs);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      dev_free(ctx, remap_dev);
      if (e != cudaSuccess) { dev_free(ctx, nf); set_error("re-encoding column %d failed: %s", w.col, cudaGetErrorString(e)); return PB200_E_CUDA; }
      // swap the forward index (the old buffer came from the pool or from the generator's cudaMalloc)
      {
        bool pooled;
        { std::lock_guard<std::mutex> g(ctx->mu); pooled = ctx->block_size.count(c.fwd) != 0; }
        if (pooled) dev_free(ctx, c.fwd); else cudaFree(c.fwd);
      }
      seg->device_bytes += (int64_t)nbytes - (int64_t)c.fwd_alloc_bytes;
      c.fwd = (uint32_t*)nf;
      c.fwd_alloc_bytes = nbytes;
      c.fwd_file_bytes = ((uint64_t)seg->num_docs * dc.bits + 7) / 8;
      c.pooled = true;
      if (!c.inv_offsets.empty()) {  // posting lists are looked up by the column's (now global) ids: re-index the offsets
        std::vector<uint32_t> og((size_t)dc.cardinality + 1);
        og[dc.cardinality] = c.inv_offsets[c.cardinality];
        int l = c.cardinality - 1;
        for (int g = dc.cardinality - 1; g >= 0; g--) {
          if (l >= 0 && w.remap[l] == (uint32_t)g) { og[g] = c.inv_offsets[l]; l--; }
          else og[g] = og[g + 1];  // id absent from this segment: empty posting list
        }
        c.inv_offsets.swap(og);
      }
    }
    // adopt the domain's dictionary (device copy shared by all bound segments)
    if (c.dict_native && !c.dict_shared) { seg->device_bytes -= (int64_t)c.dict_host.size(); dev_free(ctx, c.dict_native); }
    if (!c.dict_shared && c.moments->limbs) seg->device_bytes -= 12ll * c.moments->entries;
    c.moments = dc.moments;   // VAR / STDDEV limb dictionaries: one set per domain dictionary
    c.dict_native = dc.dict_native;
    c.dict_shared = true;
    c.dict_host = dc.dict_host;
    c.dict_be = dc.dict_be;
    c.dict_entry_bytes = dc.entry_bytes;
    c.dict_hash = dc.hash;
    c.local_ids.swap(w.remap);
    c.bits = dc.bits;
    c.cardinality = dc.cardinality;
  }
  { std::lock_guard<std::mutex> g(ctx->mu); dom->refs++; }
  seg->domain = dom;
  return PB200_OK;
}

extern "C" int64_t pb200_segment_local_ids(const pb200_segment* seg, int32_t column, int32_t* out, int64_t cap) {
  if (!seg || column < 0 || column >= seg->num_columns()) { set_error("bad column"); return PB200_E_INVALID; }
  const DeviceColumn& c = seg->cols[column];
  if (c.local_ids.empty()) {  // unbound: every id of the dictionary occurs (Pinot dictionaries hold only present values)
    if (out) for (int64_t i = 0; i < c.cardinality && i < cap; i++) out[i] = (int32_t)i;
    return c.cardinality;
  }
  if (out) for (int64_t i = 0; i < (int64_t)c.local_ids.size() && i < cap; i++) out[i] = (int32_t)c.local_ids[i];
  return (int64_t)c.local_ids.size();
}
