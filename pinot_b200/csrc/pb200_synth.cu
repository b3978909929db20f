// pb200_synth.cu -- synthetic segment creator running on the device.
//
// Stand-in for the reference's SegmentIndexCreationDriverImpl when benchmarking: 100 M-row segments are generated
// straight into HBM, but the BYTES are exactly what the reference's writers would produce for the same values:
//   forward index  = FixedBitSVForwardIndexWriter / PinotDataBitSet.writeInt (MSB-first big-endian bit stream,
//                    seglocal/io/writer/impl/FixedBitSVForwardIndexWriter.java:39-46)
//   dictionary     = SegmentDictionaryCreator (sorted INT values, big-endian, :117)
//   inverted index = BitmapInvertedIndexWriter layout (:33-50) with RoaringBitmap portable serialization per dictId
//                    (array container <= 4096 values, bitmap container above; no run containers -- a valid encoding,
//                    byte parity of Roaring serialization is unpinned anyway, see oracle/pinot_oracle.h)
// tests/test_gpu_synth.py reads the buffers back and compares them with the oracle's CPU writers.
//
// Values: dictId(doc) = mix64(seed + doc * 0x9E3779B97F4A7C15) % cardinality (SplitMix64 finaliser; reproducible in
// numpy), value(dictId) = value_base + value_step * dictId.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "pb200_internal.h"
#include "pb200_unpack.cuh"

namespace pb200 {

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
  z ^= z >> 27; z *= 0x94D049BB133111EBull;
  z ^= z >> 31;
  return z;
}
__host__ __device__ __forceinline__ uint32_t synth_dict_id(uint64_t seed, long long doc, uint32_t card) {
  return (uint32_t)(mix64(seed + (uint64_t)doc * 0x9E3779B97F4A7C15ull) % card);
}

// one thread = one 32-row group = `bits` output words
__global__ void synth_fwd_kernel(uint32_t* __restrict__ out, long long num_groups, long long num_docs, int bits,
                                 uint32_t card, uint64_t seed) {
  long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (; g < num_groups; g += (long long)gridDim.x * blockDim.x) {
    uint32_t* o = out + g * bits;
    uint64_t acc = 0;
    int have = 0, k = 0;
    for (int i = 0; i < 32; i++) {
      long long doc = g * 32 + i;
      uint32_t v = doc < num_docs ? synth_dict_id(seed, doc, card) : 0u;
      acc = (acc << bits) | v;
      have += bits;
      if (have >= 32) {
        o[k++] = (uint32_t)(acc >> (have - 32));  // native word order (the HBM layout; see pb200_unpack.cuh)
        have -= 32;
      }
    }
  }
}

__global__ void synth_dict_kernel(unsigned char* __restrict__ out, int card, int base, int step) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < card) {
    uint32_t v = (uint32_t)(base + step * i);
    out[4 * i + 0] = v >> 24; out[4 * i + 1] = v >> 16; out[4 * i + 2] = v >> 8; out[4 * i + 3] = v;
  }
}

// ---- inverted index ----------------------------------------------------------------------------------------------
__global__ void inv_count_kernel(const uint32_t* __restrict__ fwd, int bits, long long num_docs, int nchunks,
                                 uint32_t* __restrict__ counts) {
  long long doc = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (; doc < num_docs; doc += (long long)gridDim.x * blockDim.x) {
    uint32_t id = read_one(fwd, doc, bits);
    atomicAdd(counts + (size_t)id * nchunks + (doc >> 16), 1u);
  }
}

struct ContainerJob {
  uint32_t dict_id;
  uint32_t chunk;
  uint32_t card;
  uint32_t pad;
  unsigned long long dst;  // byte offset of the container payload in the index file
};

__global__ void __launch_bounds__(256) inv_fill_kernel(const uint32_t* __restrict__ fwd, int bits, long long num_docs,
                                                       const ContainerJob* __restrict__ jobs, long long njobs,
                                                       unsigned char* __restrict__ out) {
  __shared__ uint32_t words[2048];
  __shared__ uint32_t scan[256];
  for (long long j = blockIdx.x; j < njobs; j += gridDim.x) {
    const ContainerJob job = jobs[j];
    const long long base = (long long)job.chunk << 16;
    for (int w = threadIdx.x; w < 2048; w += 256) words[w] = 0;
    __syncthreads();
    // each thread owns 256 consecutive docs of the chunk = 8 mask words
    const int t = threadIdx.x;
    uint32_t mine = 0;
    for (int w = 0; w < 8; w++) {
      uint32_t m = 0;
      for (int b = 0; b < 32; b++) {
        long long doc = base + t * 256 + w * 32 + b;
        if (doc < num_docs && read_one(fwd, doc, bits) == job.dict_id) m |= 1u << b;
      }
      words[t * 8 + w] = m;
      mine += __popc(m);
    }
    scan[t] = mine;
    __syncthreads();
    unsigned char* dst = out + job.dst;
    if (job.card > 4096) {
      for (int w = threadIdx.x; w < 2048; w += 256) {
        uint32_t x = words[w];
        dst[4 * w + 0] = x; dst[4 * w + 1] = x >> 8; dst[4 * w + 2] = x >> 16; dst[4 * w + 3] = x >> 24;
      }
    } else {
      // exclusive prefix over the 256 per-thread counts (serial by one warp-0 thread is fine for a setup kernel)
      if (t == 0) {
        uint32_t run = 0;
        for (int i = 0; i < 256; i++) { uint32_t c = scan[i]; scan[i] = run; run += c; }
      }
      __syncthreads();
      uint32_t pos = scan[t];
      for (int w = 0; w < 8; w++) {
        uint32_t m = words[t * 8 + w];
        while (m) {
          uint32_t v = (uint32_t)(t * 256 + w * 32 + __ffs(m) - 1);
          dst[2 * pos + 0] = v; dst[2 * pos + 1] = v >> 8;
          pos++;
          m &= m - 1;
        }
      }
    }
    __syncthreads();
  }
}

static void put_le16(std::vector<unsigned char>& b, size_t at, uint32_t v) { b[at] = v; b[at + 1] = v >> 8; }
static void put_le32(std::vector<unsigned char>& b, size_t at, uint32_t v) { b[at] = v; b[at + 1] = v >> 8; b[at + 2] = v >> 16; b[at + 3] = v >> 24; }
static void put_be32(std::vector<unsigned char>& b, size_t at, uint32_t v) { b[at] = v >> 24; b[at + 1] = v >> 16; b[at + 2] = v >> 8; b[at + 3] = v; }

int synth_build_inverted(pb200_ctx* ctx, cudaStream_t st, DeviceColumn& col, long long num_docs) {
  const int card = col.cardinality;
  if (card > 1024) { set_error("synthetic inverted index limited to cardinality <= 1024"); return PB200_E_UNSUPPORTED; }
  const int nchunks = (int)((num_docs + 65535) >> 16);
  uint32_t* dcounts = nullptr;
  PB200_CUDA(cudaMalloc(&dcounts, (size_t)card * nchunks * 4));
  PB200_CUDA(cudaMemsetAsync(dcounts, 0, (size_t)card * nchunks * 4, st));
  inv_count_kernel<<<ctx->sm_count * 8, 256, 0, st>>>(col.fwd, col.bits, num_docs, nchunks, dcounts);
  std::vector<uint32_t> counts((size_t)card * nchunks);
  PB200_CUDA(cudaMemcpyAsync(counts.data(), dcounts, counts.size() * 4, cudaMemcpyDeviceToHost, st));
  PB200_CUDA(cudaStreamSynchronize(st));
  cudaFree(dcounts);

  // layout: (card+1) BE offsets, then per dictId: cookie 12346, n, n x (key, card-1), n x offset, payloads
  std::vector<ContainerJob> jobs;
  std::vector<uint64_t> bm_off(card + 1);
  uint64_t pos = 4ull * (card + 1);
  struct Hdr { uint64_t at; std::vector<unsigned char> bytes; };
  std::vector<Hdr> hdrs(card);
  for (int d = 0; d < card; d++) {
    bm_off[d] = pos;
    std::vector<std::pair<uint32_t, uint32_t>> cs;
    for (int c = 0; c < nchunks; c++) if (counts[(size_t)d * nchunks + c]) cs.push_back({(uint32_t)c, counts[(size_t)d * nchunks + c]});
    const uint32_t n = (uint32_t)cs.size();
    std::vector<unsigned char>& h = hdrs[d].bytes;
    hdrs[d].at = pos;
    h.resize(8 + 8ull * n);
    put_le32(h, 0, 12346u);
    put_le32(h, 4, n);
    uint64_t payload = 8 + 8ull * n;  // relative to the bitmap start
    for (uint32_t i = 0; i < n; i++) {
      put_le16(h, 8 + 4ull * i, cs[i].first);
      put_le16(h, 8 + 4ull * i + 2, cs[i].second - 1);
      put_le32(h, 8 + 4ull * n + 4ull * i, (uint32_t)payload);
      jobs.push_back({(uint32_t)d, cs[i].first, cs[i].second, 0u, pos + payload});
      payload += cs[i].second > 4096 ? 8192 : 2ull * cs[i].second;
    }
    pos += payload;
  }
  bm_off[card] = pos;
  if (pos > 0xFFFFFFFFull) { set_error("inverted index exceeds 4 GB (offsets are u32 in Pinot's layout)"); return PB200_E_UNSUPPORTED; }
  PB200_CUDA(cudaMalloc(&col.inv, pos + 16));
  col.inv_bytes = pos;
  std::vector<unsigned char> offs(4ull * (card + 1));
  col.inv_offsets.resize(card + 1);
  for (int d = 0; d <= card; d++) { put_be32(offs, 4ull * d, (uint32_t)bm_off[d]); col.inv_offsets[d] = (uint32_t)bm_off[d]; }
  PB200_CUDA(cudaMemcpyAsync(col.inv, offs.data(), offs.size(), cudaMemcpyHostToDevice, st));
  for (int d = 0; d < card; d++)
    PB200_CUDA(cudaMemcpyAsync(col.inv + hdrs[d].at, hdrs[d].bytes.data(), hdrs[d].bytes.size(), cudaMemcpyHostToDevice, st));
  ContainerJob* djobs = nullptr;
  if (!jobs.empty()) {
    PB200_CUDA(cudaMalloc(&djobs, jobs.size() * sizeof(ContainerJob)));
    PB200_CUDA(cudaMemcpyAsync(djobs, jobs.data(), jobs.size() * sizeof(ContainerJob), cudaMemcpyHostToDevice, st));
    int grid = (int)std::min<size_t>(jobs.size(), (size_t)ctx->sm_count * 16);
    inv_fill_kernel<<<grid, 256, 0, st>>>(col.fwd, col.bits, num_docs, djobs, (long long)jobs.size(), col.inv);
    PB200_CUDA(cudaGetLastError());
  }
  PB200_CUDA(cudaStreamSynchronize(st));
  if (djobs) cudaFree(djobs);
  return PB200_OK;
}

}  // namespace pb200

using namespace pb200;

extern "C" int32_t pb200_synth_segment(pb200_ctx* ctx, const char* name, int32_t num_docs, int32_t ncols,
                                       const pb200_synth_col* cols, pb200_segment** out) {
  if (!ctx || !cols || !out || num_docs <= 0 || ncols <= 0) { set_error("invalid argument to pb200_synth_segment"); return PB200_E_INVALID; }
  PB200_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = take_stream(ctx);
  struct StreamReturn { pb200_ctx* c; cudaStream_t s; ~StreamReturn() { give_stream(c, s); } } stream_return{ctx, st};
  std::vector<pb200_col_desc> descs(ncols);
  std::vector<void*> tmp_dicts;
  std::vector<void*> fwds;
  auto cleanup = [&](bool keep_fwd) {
    for (void* p : tmp_dicts) cudaFree(p);
    if (!keep_fwd) for (void* p : fwds) cudaFree(p);
  };
  for (int i = 0; i < ncols; i++) {
    const pb200_synth_col& sc = cols[i];
    if (sc.cardinality < 1) { set_error("cardinality must be >= 1"); cleanup(false); return PB200_E_INVALID; }
    int bits = 1;
    while (bits < 31 && (1ll << bits) < sc.cardinality) bits++;  // PinotDataBitSet.getNumBitsPerValue(card - 1)
    long long tiles = ((long long)num_docs + kMaxTileRows - 1) / kMaxTileRows + 1;  // see padded_fwd_bytes()
    uint64_t alloc = (uint64_t)tiles * kMaxTileRows / 8 * bits + 64;
    uint32_t* fwd = nullptr;
    cudaError_t e = cudaMalloc(&fwd, alloc);
    if (e != cudaSuccess) { set_error("cudaMalloc(%llu) failed: %s", (unsigned long long)alloc, cudaGetErrorString(e)); cleanup(false); cudaGetLastError(); return PB200_E_NOMEM; }
    fwds.push_back(fwd);
    long long groups = tiles * (kMaxTileRows / 32);
    synth_fwd_kernel<<<ctx->sm_count * 8, 256, 0, st>>>(fwd, groups, num_docs, bits, (uint32_t)sc.cardinality, sc.seed);
    cudaMemsetAsync((unsigned char*)fwd + (alloc - 64), 0, 64, st);
    unsigned char* dict = nullptr;
    e = cudaMalloc(&dict, 4ull * sc.cardinality);
    if (e != cudaSuccess) { set_error("cudaMalloc failed: %s", cudaGetErrorString(e)); cleanup(false); cudaGetLastError(); return PB200_E_NOMEM; }
    tmp_dicts.push_back(dict);
    synth_dict_kernel<<<(sc.cardinality + 255) / 256, 256, 0, st>>>(dict, sc.cardinality, sc.value_base, sc.value_step);
    pb200_col_desc& d = descs[i];
    memset(&d, 0, sizeof d);
    d.fwd_kind = PB200_FWD_DICT_FIXEDBIT;
    d.stored_type = PB200_INT;
    d.bits_per_value = bits;
    d.cardinality = sc.cardinality;
    d.flags = PB200_COL_DEVICE_BUFFERS;
    d.fwd = fwd;
    d.fwd_bytes = alloc;
    d.dict = dict;
    d.dict_bytes = 4ull * sc.cardinality;
  }
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { set_error("synthetic generation failed: %s", cudaGetErrorString(e)); cleanup(false); return PB200_E_CUDA; }
  pb200_segment* seg = nullptr;
  int rc = pb200_segment_register(ctx, name, num_docs, ncols, descs.data(), &seg);
  if (rc) { cleanup(false); return rc; }
  cleanup(true);
  for (int i = 0; i < ncols; i++) {
    if (!cols[i].with_inverted) continue;
    rc = synth_build_inverted(ctx, st, seg->cols[i], num_docs);
    if (rc) { pb200_segment_release(ctx, seg); return rc; }
    seg->device_bytes += (int64_t)seg->cols[i].inv_bytes;
  }
  *out = seg;
  return PB200_OK;
}
