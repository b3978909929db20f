// pb200_scan.cuh -- the fused scan kernel: DocIdSet -> Projection -> Aggregation / GroupBy in one pass over HBM.
//
// What the reference does per segment, block (<=10 000 docs) at a time, on one CPU thread
//   FilterOperator tree -> DocIdSetOperator -> ProjectionOperator -> GroupByOperator/AggregationOperator
//   (core/operator/DocIdSetOperator.java:59-86, ProjectionOperator.java:68-79, query/GroupByOperator.java:101-140,
//    query/AggregationOperator.java:64-80; bit unpack in seglocal/io/reader/impl/FixedBitIntReader.java)
// is done here for ALL segments of a query by one persistent kernel:
//
//   * every WARP streams its own 1024-row slices of every touched column HBM -> shared memory with TMA 1-D bulk copies
//     (cp.async.bulk ... mbarrier::complete_tx) through a private ring of stage buffers -- no producer warp;
//   * each thread owns 32 consecutive rows: unpacks its B words per column (pb200_unpack.cuh; native word order in HBM),
//     evaluates every filter leaf into a 32-bit row mask (compare through the carry flag), combines masks with the
//     filter's boolean program, then aggregates the surviving rows:
//       aggregation only: per-thread accumulators in shared memory + warp reduction + one atomic per warp and segment,
//                         dictionary gathers software-pipelined across tiles;
//       group-by:         survivors compacted into a per-warp queue, then dense gathers / reductions over the queue into a
//                         dense table indexed by the raw key (sum dictId_j * mult_j, DictionaryBasedGroupKeyGenerator
//                         :311-346), a CTA-private shared-memory table (small key spaces) or a hash table (LONG_MAP);
//   * integer work only: no tensor cores; the bound is HBM bandwidth (algorithmic bytes = sum of bits/8 per row).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "pb200_desc.h"
#include "pb200_unpack.cuh"

namespace pb200 {

// ------------------------------------------------------------------------------------------------------------------
// mbarrier / TMA bulk-copy primitives (PTX ISA 8.x; SASS: SYNCS.*, UBLKCP)
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// The ring primitives take 32-bit shared-window addresses computed ONCE per thread (a generic -> shared conversion
// per call costs an S2UR/ULEA/IMAD chain in the tile loop).
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}" ::"r"(bar),
      "r"(parity)
      : "memory");
}
// 1-D TMA bulk copy global -> shared, completion counted in bytes on `bar`; streaming data: L2 evict-first policy.
__device__ __forceinline__ void tma_load_1d(uint32_t dst_smem, const void* src_gmem, uint32_t bytes, uint32_t bar,
                                            uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          dst_smem),
      "l"(src_gmem), "r"(bytes), "r"(bar), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void consumer_bar_sync(int nthreads) {
  asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory");
}

// ------------------------------------------------------------------------------------------------------------------
// leaf evaluation on a thread's 32 unpacked dictIds
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t eval_range(const uint32_t (&v)[32], uint32_t lo, uint32_t span) {
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < 32; ++j) m |= ((v[j] - lo) < span ? 1u : 0u) << j;
  return m;
}
__device__ __forceinline__ uint32_t eval_lut(const uint32_t (&v)[32], const uint32_t* __restrict__ bits) {
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < 32; ++j) m |= ((__ldg(bits + (v[j] >> 5)) >> (v[j] & 31)) & 1u) << j;
  return m;
}
// rows [row0, row0+32) against inclusive doc-id ranges
__device__ __forceinline__ uint32_t eval_doc_ranges(uint32_t row0u, const int32_t* __restrict__ r, int n) {
  const long long row0 = row0u;
  uint32_t m = 0;
  for (int i = 0; i < n; ++i) {
    long long lo = (long long)__ldg(r + 2 * i) - row0, hi = (long long)__ldg(r + 2 * i + 1) - row0 + 1;  // [lo, hi)
    lo = lo < 0 ? 0 : lo;
    hi = hi > 32 ? 32 : hi;
    if (hi > lo) {
      uint32_t upto_hi = hi >= 32 ? 0xFFFFFFFFu : ((1u << hi) - 1u);
      uint32_t upto_lo = (1u << lo) - 1u;  // lo < 32 here
      m |= upto_hi & ~upto_lo;
    }
  }
  return m;
}


// One value of a thread's 32-row group straight from the tile: bit offset j*bits inside the group's `bits` words.
__device__ __forceinline__ uint32_t read_one_group(const uint32_t* __restrict__ p, int j, int bits) {
  const int bit = j * bits;
  const int k = bit >> 5, s = bit & 31;
  const uint32_t hi = fwd_word(p[k]);
  const uint32_t lo = (s + bits > 32) ? fwd_word(p[k + 1]) : 0u;
  const uint32_t x = __funnelshift_l(lo, hi, s);
  return bits == 32 ? x : (x >> (32 - bits));
}
// Branch-free predicated gathers: the load is skipped (not just masked) for rows that did not survive the filter.
__device__ __forceinline__ int ldg_pred_s32(const int* p, uint32_t pred) {
  int x;
  asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\tmov.b32 %0, 0;\n\t@p ld.global.nc.b32 %0, [%1];\n\t}" : "=r"(x) : "l"(p), "r"(pred));
  return x;
}
// same, predicate = (mask & bit) != 0 with `bit` a compile-time constant after unrolling: LOP3 + ISETP, no shift
__device__ __forceinline__ uint32_t ldg_bit_u32(const uint32_t* p, uint32_t mask, uint32_t bit) {
  uint32_t x;
  asm("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\tand.b32 t, %2, %3;\n\tsetp.ne.u32 p, t, 0;\n\tmov.b32 %0, 0;\n\t"
      "@p ld.global.nc.b32 %0, [%1];\n\t}" : "=r"(x) : "l"(p), "r"(mask), "r"(bit));
  return x;
}
__device__ __forceinline__ long long ldg_pred_s64(const long long* p, uint32_t pred) {
  long long x;
  asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\tmov.b64 %0, 0;\n\t@p ld.global.nc.b64 %0, [%1];\n\t}" : "=l"(x) : "l"(p), "r"(pred));
  return x;
}

template <typename T>
__device__ __forceinline__ T warp_sum(T x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, o);
  return x;
}
__device__ __forceinline__ uint32_t warp_min(uint32_t x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = min(x, __shfl_xor_sync(0xFFFFFFFFu, x, o));
  return x;
}
__device__ __forceinline__ uint32_t warp_max(uint32_t x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = max(x, __shfl_xor_sync(0xFFFFFFFFu, x, o));
  return x;
}



// fire-and-forget global reductions (the result is never needed: RED, not ATOM)
__device__ __forceinline__ void red_add_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_add_f64(double* p, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}

// Hash group table: slot of `key` in the open-addressing table (linear probing, 64-bit CAS on the key itself -- exact,
// no fingerprints).  Returns false once the table holds more than h_limit groups (the caller's result is then discarded:
// numGroupsLimit would bind, PB200_E_LIMIT) or is full.
__device__ __forceinline__ uint32_t mix64_32(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return (uint32_t)(z ^ (z >> 31));
}
__device__ __forceinline__ bool hash_slot(const SegDesc& sd, unsigned long long key, uint32_t& slot) {
  constexpr unsigned long long kEmpty = ~0ull;
  if (*reinterpret_cast<volatile uint32_t*>(sd.h_ctl + 1)) return false;
  uint32_t h = mix64_32(key) & sd.h_mask;
  for (uint32_t probe = 0; probe <= sd.h_mask; ++probe) {
    unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(sd.h_keys + h);
    if (cur == kEmpty) {
      cur = atomicCAS(sd.h_keys + h, kEmpty, key);
      if (cur == kEmpty) {
        if (atomicAdd(sd.h_ctl, 1u) >= (uint32_t)sd.h_limit) { sd.h_ctl[1] = 1u; return false; }
        slot = h;
        return true;
      }
    }
    if (cur == key) { slot = h; return true; }
    h = (h + 1u) & sd.h_mask;
  }
  sd.h_ctl[1] = 1u;
  return false;
}

// 64-bit signed accumulate into a CTA-private shared-memory table kept as two u32 words: shared 64-bit atomic adds
// compile to a CAS spin loop (ATOMS.CAST.SPIN.64) while 32-bit ones are native, and the high word only moves on a
// carry or a negative addend.
__device__ __forceinline__ void smem_add64(uint32_t* lo, uint32_t* hi, uint32_t g, int x) {
  const uint32_t xl = (uint32_t)x;
  const uint32_t old = atomicAdd(lo + g, xl);
  const int h = (x >> 31) + ((uint32_t)(old + xl) < xl ? 1 : 0);  // sign extension + carry out of the low word
  if (h) atomicAdd(hi + g, (uint32_t)h);
}

// ------------------------------------------------------------------------------------------------------------------
// streaming functors for dispatch_left_aligned(): consume one left-aligned value at a time (pb200_unpack.cuh)
// ------------------------------------------------------------------------------------------------------------------
// dictId range predicate -> 32-bit row mask.
// Mask building through the carry flag: compare = one subtract whose carry-out lands in CC.CF, and `addc m, m, m`
// shifts it into the mask (m = 2m + CF) -- 2 instructions per value (IADD3 + IMAD.X, the second one on the FMA pipe)
// instead of ISETP + SEL + OR.  After `sub.cc.u32 t, a, b` ptxas / sm_90a leave CF = 1 iff there was NO borrow, i.e.
// a >= b (the hardware carry of a + ~b + 1; measured by tests/workloads/cc_probe and guarded by every parity test).
// Four chains of 8 values (rows 8k .. 8k+7 in chain k, first row in the chain's highest bit) keep the adds independent;
// the chains are concatenated and bit-reversed once per leaf.
__device__ __forceinline__ void ge_into(uint32_t& m, uint32_t a, uint32_t b) {  // m = 2m + (a >= b)
  asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\taddc.u32 %0, %0, %0;\n\t}" : "+r"(m) : "r"(a), "r"(b));
}
struct CarryMask {
  uint32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
  __device__ __forceinline__ void push(int j, uint32_t a, uint32_t b) {
    if (j < 8) ge_into(c0, a, b); else if (j < 16) ge_into(c1, a, b); else if (j < 24) ge_into(c2, a, b); else ge_into(c3, a, b);
  }
  // bit j = (a_j >= b_j)
  __device__ __forceinline__ uint32_t ge_mask() const { return __brev((c0 << 24) | (c1 << 16) | (c2 << 8) | c3); }
};
struct RangeBoth {   // lo <= v < hi   as   (xl - LO) < SPAN,  LO = lo << (32-B), SPAN = (hi-lo) << (32-B)
  uint32_t LO, SPAN;
  CarryMask cm;
  __device__ __forceinline__ void operator()(int j, uint32_t xl) { cm.push(j, xl - LO, SPAN); }
  __device__ __forceinline__ uint32_t mask() const { return ~cm.ge_mask(); }
};
struct RangeGE {     // v >= lo  (upper bound is the whole dictionary: every stored dictId is < cardinality)
  uint32_t LO;
  CarryMask cm;
  __device__ __forceinline__ void operator()(int j, uint32_t xl) { cm.push(j, xl, LO); }
  __device__ __forceinline__ uint32_t mask() const { return cm.ge_mask(); }
};
struct RangeLT {     // v < hi  (lower bound 0)
  uint32_t HI;
  CarryMask cm;
  __device__ __forceinline__ void operator()(int j, uint32_t xl) { cm.push(j, xl, HI); }
  __device__ __forceinline__ uint32_t mask() const { return ~cm.ge_mask(); }
};
// SUM over an INT dictionary: gather the BIASED value (value ^ 0x80000000, i.e. value + 2^31 as unsigned) of every
// surviving row and add pairs with one 3-input 64-bit add; the bias is removed once per tile (popc * 2^31).
struct SumBiasedU32 {
  const uint32_t* __restrict__ d;
  uint32_t m, sh;
  unsigned long long a0 = 0, a1 = 0;
  uint32_t pend = 0;
  __device__ __forceinline__ void operator()(int j, uint32_t xl) {
    const uint32_t x = ldg_bit_u32(d + (xl >> sh), m, 1u << j);
    if ((j & 1) == 0) {
      pend = x;
    } else if ((j & 2) == 0) {
      a0 += (unsigned long long)pend + (unsigned long long)x;
    } else {
      a1 += (unsigned long long)pend + (unsigned long long)x;
    }
  }
};
// Deferred variant: only issues the gathers (into x[j]); the caller sums them one tile later.
struct GatherBiasedU32 {
  const uint32_t* __restrict__ d;
  uint32_t m, sh;
  uint32_t (&x)[32];
  __device__ __forceinline__ void operator()(int j, uint32_t xl) { x[j] = ldg_bit_u32(d + (xl >> sh), m, 1u << j); }
};
// MIN / MAX of dictIds on the left-aligned form (order preserving; shift back once at the end)
struct MinMaxLeft {
  uint32_t m, mn = 0xFFFFFFFFu, mx = 0u;
  __device__ __forceinline__ void operator()(int j, uint32_t xl) {
    if ((m >> j) & 1u) { mn = min(mn, xl); mx = max(mx, xl); }
  }
};

// ------------------------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------------------------
// Execution model
//   * a CTA tile is W x 1024 consecutive rows of ONE segment; CTA c takes CTA tiles c, c + grid, ...;
//   * inside it every WARP owns a private slice of 1024 rows and a private TMA ring: lane 0 arms the warp's mbarrier
//     with the slice's byte count and issues one 1-D bulk copy per touched column (128 x bits bytes each); when the
//     warp has consumed a slice, the same lane refills that buffer with the slice `num_stages` CTA tiles ahead.  No
//     producer warp, no CTA-wide barrier per tile -- warps only meet at segment boundaries (<= #segments times);
//   * a THREAD owns 32 consecutive rows (one FixedBitIntReader.read32 group): B words per column.
// Shared-memory layout (dynamic):
//   [SmemHeader][W x num_stages x stage_words][filter stack (generic filters only)]
//   [acc64: num_aggs x threads x 8 B][accmm: num_aggs x threads x 8 B]                        (aggregation-only kernel)
//   [survivor queue: W x 1024 u16][group table copies: count, (lo, hi) per sum -- optional]     (group-by kernel)
// acc64/accmm are the per-thread running aggregates; they live in shared memory (private slot per thread, touched once
// per tile) instead of registers so that two CTAs fit on an SM.
template <int W, bool GROUPBY, bool DEFER = !GROUPBY, int MINB = (GROUPBY ? 1 : 2)>
__global__ void __launch_bounds__(W * 32, MINB)
scan_kernel(const __grid_constant__ QueryDesc q, const __grid_constant__ TmaTable tt, const SegDesc* __restrict__ segs) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  // The shared-window base is made opaque to the compiler once: otherwise every access through hdr-> / the accumulator
  // pointers rematerialises it as S2R SR_CgaCtaId + LEA (a variable-latency special-register read per access).
  uint32_t smem_base_s = smem_u32(smem_raw);
  asm volatile("" : "+r"(smem_base_s));
  unsigned char* const smem_base = static_cast<unsigned char*>(__cvta_shared_to_generic(smem_base_s));
  SmemHeader* hdr = reinterpret_cast<SmemHeader*>(smem_base);
  constexpr int kHdrBytes = (sizeof(SmemHeader) + 127) / 128 * 128;
  constexpr int kConsumers = W * 32;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  uint32_t* stages_all = reinterpret_cast<uint32_t*>(smem_base + kHdrBytes);
  uint32_t* wstages = stages_all + (size_t)warp * q.num_stages * q.stage_words;   // this warp's ring
  uint32_t* fstack = stages_all + (size_t)W * q.num_stages * q.stage_words;       // generic-filter mask stack
  unsigned long long* acc64 = reinterpret_cast<unsigned long long*>(fstack + (q.conj ? 0 : kConsumers * kMaxStack));
  uint2* accmm = reinterpret_cast<uint2*>(acc64 + (size_t)q.num_aggs * kConsumers);
  const bool use_pipe = q.use_pipe != 0;

  if (lane == 0) {
    for (int s = 0; s < q.num_stages; ++s) mbar_init(&hdr->full[warp][s], 1);
    mbar_fence_init();
  }
  // CTA-private group table (see QueryDesc.smem_groups)
  uint32_t* const tcnt = reinterpret_cast<uint32_t*>(smem_base + q.smem_table_off);
  const uint32_t TG = (uint32_t)q.smem_groups;
  const uint32_t TA = (uint32_t)(q.smem_copies * q.smem_gstride);                  // words per table array (all copies)
  const uint32_t tcopy = (uint32_t)((threadIdx.x & (q.smem_copies - 1)) * q.smem_gstride);  // this lane's copy
  const uint32_t tcnt_s = smem_base_s + q.smem_table_off + 4u * tcopy;             // shared-window address, lane's copy
  if (GROUPBY && TG) {
    int nsl = 0;
#pragma unroll
    for (int a = 0; a < kMaxAggs; ++a) nsl = max(nsl, (int)q.smem_slot[a] + 1);
    for (uint32_t i = threadIdx.x; i < TA * (1u + 2u * nsl); i += W * 32) tcnt[i] = 0u;
  }
  if (threadIdx.x < kMaxAggs) hdr->aggs[threadIdx.x] = q.aggs[threadIdx.x];
  if (threadIdx.x < kMaxSlots) hdr->slot_roles[threadIdx.x] = q.slot_roles[threadIdx.x];
  if (threadIdx.x < kMaxGroupBy) hdr->group_slot[threadIdx.x] = q.group_slot[threadIdx.x];
  __syncthreads();

  const int group = threadIdx.x;  // index of this thread's per-thread accumulators
  const SegDesc& sd = hdr->seg;
  unsigned long long cnt = 0;

  // ---- warp-private TMA ring.  Prefetch cursor state lives in registers and advances incrementally (lane k < num_slots
  //      owns slot k's source pointer); the constant-bank table is consulted only when the cursor enters a new segment.
  const uint64_t policy = policy_evict_first();
  const uint32_t fullw = smem_u32(&hdr->full[warp][0]);  // + 8 * stage
  const uint32_t wstages_s = smem_u32(wstages);
  int pidx = 0, p_end = 0;            // prefetch segment cursor and its exclusive end tile
  int Tp = blockIdx.x;                // next CTA tile to prefetch
  const unsigned char* p_src = nullptr;
  unsigned long long p_stride = 0;
  uint32_t p_tb = 0, p_dst = 0, p_tx = 0, p_docs = 0, skipbits = 0;
  int p_first = 0;
  const uint32_t *p_skip0 = nullptr, *p_skip1 = nullptr, *p_skip2 = nullptr;
  auto issue = [&](int stage) {  // whole warp: lane 0 arms the barrier, lane k < num_slots copies slot k
    if (Tp >= p_end) {
      while (Tp >= tt.seg[pidx].end_tile) ++pidx;
      const TmaSeg& ps = tt.seg[pidx];
      p_end = ps.end_tile;
      p_first = ps.first_tile;
      p_docs = ps.num_docs;
      p_skip0 = ps.skip_mask[0]; p_skip1 = ps.skip_mask[1]; p_skip2 = ps.skip_mask[2];
      p_tx = ps.stage_tx;
      const TmaSlot& sl = ps.slot[lane < q.num_slots ? lane : 0];
      p_tb = sl.tile_bytes;
      p_dst = sl.stage_words;
      p_src = reinterpret_cast<const unsigned char*>(sl.data) + (unsigned long long)((Tp - ps.first_tile) * W + warp) * p_tb;
      p_stride = (unsigned long long)p_tb * (unsigned)(W * gridDim.x);
    }
    // bitmap-index driven skipping: if the AND of the slice's doc-mask words is zero, nothing in it can match
    bool skip = false;
    if (p_skip0 != nullptr) {
      const uint32_t slice = (uint32_t)((Tp - p_first) * W + warp);
      uint32_t wv = 0;
      if (slice * 1024u < p_docs) {
        const uint32_t wi = slice * 32u + lane;
        wv = __ldg(p_skip0 + wi);
        if (p_skip1) wv &= __ldg(p_skip1 + wi);
        if (p_skip2) wv &= __ldg(p_skip2 + wi);
      }
      skip = !__any_sync(0xFFFFFFFFu, wv != 0u);
    }
    if (skip) {
      skipbits |= 1u << stage;
      if (lane == 0) mbar_arrive(fullw + 8u * stage);  // completes the phase without any bytes
    } else {
      skipbits &= ~(1u << stage);
      // WAR on the stage buffer: every lane's generic-proxy reads of it have completed (their values were consumed
      // before the __syncwarp() that precedes issue()), so the async-proxy write may follow without a proxy fence --
      // the same consumer-release -> producer-TMA ordering CUTLASS pipelines rely on.  (A fence.proxy.async here
      // compiles to MEMBAR.ALL.CTA, which also drains the deferred dictionary gathers.)
      if (lane == 0) mbar_expect_tx(fullw + 8u * stage, p_tx);
      __syncwarp();
      if (lane < q.num_slots) tma_load_1d(wstages_s + 4u * (stage * q.stage_words + p_dst), p_src, p_tb, fullw + 8u * stage, policy);
    }
    p_src += p_stride;
    Tp += gridDim.x;
  };
  if (use_pipe) {
    for (int s = 0; s < q.num_stages; ++s)
      if (Tp < q.total_tiles) issue(s);
  }

  // deferred dictionary gathers (software pipelining across tiles): the biased values of tile t's surviving rows are
  // loaded into x[] while tile t+1 is being filtered and are summed afterwards -- one L2 latency hidden per tile
  uint32_t x[DEFER ? 32 : 1];
  int pend_pc = -1;  // >= 0: x[] holds a tile's gathers (pend_pc surviving rows in this thread)
  auto drain = [&]() {
    if (DEFER && pend_pc >= 0) {
      unsigned long long a0 = 0, a1 = 0;
#pragma unroll
      for (int j = 0; j < (DEFER ? 32 : 0); j += 4) {
        a0 += (unsigned long long)x[j] + (unsigned long long)x[j + 1];
        a1 += (unsigned long long)x[j + 2] + (unsigned long long)x[j + 3];
      }
      acc64[q.defer_agg * kConsumers + group] += (a0 + a1) - ((unsigned long long)pend_pc << 31);
      pend_pc = -1;
    }
  };

  // Group-by: the LAST batch of a slice's survivor queue (all of it when <= 32 * kQB rows survive) is software-pipelined
  // too.  Its table indices and the loads its reductions wait for -- the dictionary value of a SUM / AVG argument, the
  // current table entry of a MIN / MAX -- are issued in this tile and consumed after the NEXT tile's filter phase, so the
  // L2 round trip of the gathers is hidden behind ~1000 cycles of independent work instead of stalling the warp.
  // Up to kGD aggregations are pipelined (the host lists them last in SegDesc.agg_code, num_defer_codes of them).
  constexpr int kQB = 4;   // queue entries per lane and step
  constexpr int kGD = 2;
  uint32_t pg[GROUPBY ? kQB : 1];            // table index (raw key or hash slot) of the pending entries
  uint32_t px[GROUPBY ? kGD : 1][GROUPBY ? kQB : 1];  // loaded word: biased / float dictionary value, or current MIN / MAX entry
  uint32_t pq[GROUPBY ? kGD : 1][GROUPBY ? kQB : 1];  // MIN / MAX: the row's order-preserving encoding
  uint32_t pend_ok = 0;                      // bit u: entry u is pending
  auto drain_gb = [&]() {
    if constexpr (GROUPBY) {
      if (pend_ok) {
        const int n = sd.num_agg_codes, nd = sd.num_defer_codes;
#pragma unroll
        for (int k = 0; k < kGD; ++k) {
          if (k < nd) {
            const uint32_t ac = sd.agg_code[n - nd + k];
            const int a = (int)(ac & 7u), fn = (int)((ac >> 4) & 7u), vk = (int)((ac >> 8) & 7u);
            if (fn == 1 || fn == 4) {
              if (vk == VAL_DICT_F32) {
                double* t = sd.g_dsum[a];
#pragma unroll
                for (int u = 0; u < kQB; ++u) if ((pend_ok >> u) & 1u) red_add_f64(t + pg[u], (double)__uint_as_float(px[k][u]));
              } else {
                // device INT dictionaries are biased (value + 2^31): the addend removes the bias -- or, when this sum
                // CARRIES the group's row count (SegDesc.sum_addend), re-bases the value to (value - min) + 2^shift
                unsigned long long* t = reinterpret_cast<unsigned long long*>(sd.g_isum[a]);
                const unsigned long long addend = sd.sum_addend[a];
#pragma unroll
                for (int u = 0; u < kQB; ++u)
                  if ((pend_ok >> u) & 1u) red_add_u64(t + pg[u], (unsigned long long)px[k][u] + addend);
              }
            } else if (fn == 2) {
              uint32_t* t = sd.g_min[a];
#pragma unroll
              for (int u = 0; u < kQB; ++u) if (((pend_ok >> u) & 1u) && pq[k][u] < px[k][u]) atomicMin(t + pg[u], pq[k][u]);
            } else {
              uint32_t* t = sd.g_max[a];
#pragma unroll
              for (int u = 0; u < kQB; ++u) if (((pend_ok >> u) & 1u) && pq[k][u] + 1u > px[k][u]) atomicMax(t + pg[u], pq[k][u] + 1u);
            }
          }
        }
        pend_ok = 0;
      }
    }
  };

  auto reset_acc = [&]() {
    if (!GROUPBY) {
      for (int a = 0; a < q.num_aggs; ++a) {
        acc64[a * kConsumers + group] = 0ull;
        accmm[a * kConsumers + group] = make_uint2(0xFFFFFFFFu, 0u);
      }
    }
  };
  auto flush = [&]() {
    // one atomic per warp per accumulator into the segment's AggAccum
    drain();
    drain_gb();
    unsigned long long c = warp_sum(cnt);
    if (lane == 0 && c) atomicAdd(&sd.accum->count, c);
    cnt = 0;
    if (!GROUPBY) {
      for (int a = 0; a < q.num_aggs; ++a) {
        if (hdr->aggs[a].slot < 0) continue;
        const int fn = hdr->aggs[a].function;
        if (fn == 1 || fn == 4) {  // SUM / AVG
          const unsigned long long raw = acc64[a * kConsumers + group];
          if (sum_in_double(hdr->aggs[a].val_kind)) {
            double d = warp_sum(__longlong_as_double((long long)raw));
            if (lane == 0) atomicAdd(&sd.accum->dsum[a], d);
          } else {
            unsigned long long s = warp_sum(raw);
            if (lane == 0) atomicAdd(reinterpret_cast<unsigned long long*>(&sd.accum->isum[a]), s);
          }
        } else if (fn == 2 || fn == 3) {
          const uint2 mm = accmm[a * kConsumers + group];
          if (fn == 2) { uint32_t v = warp_min(mm.x); if (lane == 0) atomicMin(&sd.accum->min_id[a], v); }
          else { uint32_t v = warp_max(mm.y); if (lane == 0) atomicMax(&sd.accum->max_id_plus1[a], v); }
        }
      }
      reset_acc();
    }
  };
  reset_acc();
  // merges the CTA-private group table into the segment's dense global table and clears it (whole CTA, between barriers)
  auto table_flush = [&]() {
    for (uint32_t g = threadIdx.x; g < TG; g += W * 32) {
      uint32_t c = 0;
      for (int r = 0; r < q.smem_copies; ++r) { c += tcnt[r * q.smem_gstride + g]; tcnt[r * q.smem_gstride + g] = 0u; }
      if (c == 0u) continue;
      if (sd.g_count) atomicAdd(sd.g_count + g, (unsigned long long)c);
      else if (sd.g_seen) sd.g_seen[g] = 1u;
#pragma unroll
      for (int a = 0; a < kMaxAggs; ++a) {
        const int k = q.smem_slot[a];
        if (k < 0 || a >= q.num_aggs) continue;
        uint32_t* lo = tcnt + TA * (1u + 2u * k);
        unsigned long long v = 0;
        for (int r = 0; r < q.smem_copies; ++r) {
          const uint32_t i = r * q.smem_gstride + g;
          v += (unsigned long long)lo[i] | (unsigned long long)lo[TA + i] << 32;
          lo[i] = 0u; lo[TA + i] = 0u;
        }
        atomicAdd(reinterpret_cast<unsigned long long*>(sd.g_isum[a] + g), v);
      }
    }
  };

  int sidx = -1, stage = 0, c_first = 0, c_end = 0;
  uint32_t phase = 0, c_docs = 0;
  for (int T = blockIdx.x; T < q.total_tiles; T += gridDim.x) {
    // ---- segment change: flush accumulators, refresh the shared descriptor copy (the only CTA-wide barriers) ----
    if (T >= c_end) {
      int ns = sidx < 0 ? 0 : sidx;
      while (T >= tt.seg[ns].end_tile) ++ns;
      if (sidx >= 0) flush();
      consumer_bar_sync(kConsumers);  // everyone done reading the old descriptor
      if (GROUPBY && TG && sidx >= 0) { table_flush(); consumer_bar_sync(kConsumers); }
      const uint32_t* src = reinterpret_cast<const uint32_t*>(segs + ns);
      uint32_t* dstw = reinterpret_cast<uint32_t*>(&hdr->seg);
      for (int i = threadIdx.x; i < (int)(sizeof(SegDesc) / 4); i += kConsumers) dstw[i] = __ldg(src + i);
      consumer_bar_sync(kConsumers);
      sidx = ns;
      c_first = tt.seg[ns].first_tile;
      c_end = tt.seg[ns].end_tile;
      c_docs = tt.seg[ns].num_docs;
    }
    const uint32_t row0 = (uint32_t)((T - c_first) * W + warp) * 1024u + (uint32_t)lane * kRowsPerThread;
    const int left = row0 >= c_docs ? 0 : (c_docs - row0 >= 32u ? 32 : (int)(c_docs - row0));
    uint32_t m = left >= 32 ? 0xFFFFFFFFu : ((1u << left) - 1u);

    if (use_pipe) mbar_wait(fullw + 8u * stage, phase);
    if (use_pipe && ((skipbits >> stage) & 1u)) m = 0u;  // slice was never loaded: no doc of it passes the bitmap leaves
    const uint32_t* st = wstages + stage * q.stage_words;
    const int group_in_stage = lane;  // the thread's 32-row group inside the warp's slice

    // ---------------- phase 1: filter -> row mask ----------------
    // Conjunctions (the common case) evaluate leaf by leaf, most selective first (host order); once few rows per
    // thread survive, the remaining columns are probed per surviving row straight from the shared-memory tile
    // (the GPU form of ScanBasedDocIdIterator.applyAnd on the bitmap of survivors, AndDocIdSet.java:167-169)
    // instead of unpacking all 32 values.
    if (q.num_nodes > 0 && __any_sync(0xFFFFFFFFu, m != 0u)) {
      if (q.conj) {
#pragma unroll 1
        for (int l = 0; l < q.num_leaves; ++l) {
          const LeafDesc& lf = sd.leaves[l];
          const uint4 L = *reinterpret_cast<const uint4*>(&lf);  // code, slot, lo, span in one LDS.128
          const uint32_t code = L.x, lf_lo = L.z, lf_span = L.w;
          const int kind = (int)(code & 7u);
          uint32_t lm;
          if (kind == LEAF_ALL) lm = 0xFFFFFFFFu;
          else if (kind == LEAF_NONE) lm = 0u;
          else if (kind == LEAF_DOCMASK) lm = left > 0 ? __ldg(lf.bits + (row0 >> 5)) : 0u;
          else if (kind == LEAF_DOCRANGES) lm = eval_doc_ranges(row0, lf.ranges, lf.num_ranges);
          else {
            const int sbits = (int)((code >> 12) & 63u);
            const uint32_t* base = st + (code >> 18);
            // the first leaf sees (almost) full masks: no need to count survivors to pick the dense path
            const int wmax = l == 0 ? 32 : __reduce_max_sync(0xFFFFFFFFu, __popc(m));
            if (wmax == 0) {
              lm = 0u;  // nothing left to test (m == 0 in every lane)
            } else if (wmax <= q.sparse_max) {
              const uint32_t* p = base + group_in_stage * sbits;
              uint32_t keep = 0, mm = m;
              while (mm) {
                const int j = 31 - __clz(mm);
                mm &= ~(1u << j);
                const uint32_t id = read_one_group(p, j, sbits);
                const bool hit = kind == LEAF_RANGE ? ((id - lf_lo) < lf_span)
                                                    : (((__ldg(lf.bits + (id >> 5)) >> (id & 31)) & 1u) != 0u);
                keep |= (hit ? 1u : 0u) << j;
              }
              lm = keep;  // bits outside m are irrelevant (m &= lm below)
            } else if (kind == LEAF_RANGE) {
              const int sh = 32 - sbits;
              const int cmp = (int)((code >> 4) & 3u);
              if (cmp == CMP_GE) { RangeGE f; f.LO = lf_lo << sh; dispatch_left_aligned(sbits, base, group_in_stage, f); lm = f.mask(); }
              else if (cmp == CMP_LT) { RangeLT f; f.HI = (lf_lo + lf_span) << sh; dispatch_left_aligned(sbits, base, group_in_stage, f); lm = f.mask(); }
              else { RangeBoth f; f.LO = lf_lo << sh; f.SPAN = lf_span << sh; dispatch_left_aligned(sbits, base, group_in_stage, f); lm = f.mask(); }
            } else {
              uint32_t v[32];
              unpack_group(sbits, base, group_in_stage, v);
              lm = eval_lut(v, lf.bits);
            }
          }
          if ((code >> 8) & 1u) lm = ~lm;
          m &= lm;
        }
      } else {
        uint32_t lm[kMaxLeaves];
#pragma unroll
        for (int l = 0; l < kMaxLeaves; ++l) {
          lm[l] = 0xFFFFFFFFu;
          if (l < q.num_leaves) {
            const LeafDesc& lf = sd.leaves[l];
            if ((lf.code & 7u) == LEAF_NONE) lm[l] = 0u;
            else if ((lf.code & 7u) == LEAF_DOCMASK) lm[l] = left > 0 ? __ldg(lf.bits + (row0 >> 5)) : 0u;
            else if ((lf.code & 7u) == LEAF_DOCRANGES) lm[l] = eval_doc_ranges(row0, lf.ranges, lf.num_ranges);
          }
        }
        for (int s = 0; s < q.num_slots; ++s) {
          if (!(hdr->slot_roles[s] & ROLE_FILTER)) continue;
          uint32_t v[32];
          unpack_group(sd.slots[s].bits, st + sd.slots[s].stage_words, group_in_stage, v);
#pragma unroll
          for (int l = 0; l < kMaxLeaves; ++l) {
            if (l < q.num_leaves && sd.leaves[l].slot == s) {
              const LeafDesc& lf = sd.leaves[l];
              if ((lf.code & 7u) == LEAF_RANGE) lm[l] = eval_range(v, lf.lo, lf.span);
              else if ((lf.code & 7u) == LEAF_LUT) lm[l] = eval_lut(v, lf.bits);
            }
          }
        }
#pragma unroll
        for (int l = 0; l < kMaxLeaves; ++l)
          if (l < q.num_leaves && sd.leaves[l].negate) lm[l] = ~lm[l];
        // postfix boolean program over masks; the stack lives in shared memory (column per thread: conflict free)
        uint32_t* stk = fstack + group;
        int sp = 0;
        for (int i = 0; i < q.num_nodes; ++i) {
          const int op = q.prog_op[i], arg = q.prog_arg[i];
          if (op == OP_LEAF) {
            uint32_t x = 0;
#pragma unroll
            for (int l = 0; l < kMaxLeaves; ++l) x = (l == arg) ? lm[l] : x;
            stk[(sp++) * kConsumers] = x;
          } else if (op == OP_NOT) {
            stk[(sp - 1) * kConsumers] = ~stk[(sp - 1) * kConsumers];
          } else {
            uint32_t x = stk[(sp - 1) * kConsumers];
            for (int c = 1; c < arg; ++c) {
              uint32_t y = stk[(sp - 1 - c) * kConsumers];
              x = op == OP_AND ? (x & y) : (x | y);
            }
            sp -= arg;
            stk[(sp++) * kConsumers] = x;
          }
        }
        m &= stk[0];
      }
    }

    drain();  // the previous tile's gathers have had this tile's whole filter phase to arrive
    drain_gb();

    // ---------------- phase 2: aggregate the surviving rows ----------------
    const int pc = __popc(m);
    cnt += pc;
    const int wmax2 = __reduce_max_sync(0xFFFFFFFFu, pc);
    // Aggregation-only kernels, few survivors: one surviving row (row j of this thread's group) is read straight from the
    // tile (FixedBitIntReader.readUnchecked shape; what DataFetcher does with sparse docIds, core/common/DataFetcher.java:335-338)
    auto process_row = [&](const int j) {
#pragma unroll 1
      for (int ai = 0; ai < sd.num_agg_codes; ++ai) {
        const uint32_t ac = sd.agg_code[ai];  // index | function | value kind | bits | stage_words (pb200_desc.h)
        const int a = (int)(ac & 7u), fn = (int)((ac >> 4) & 7u), vk = (int)((ac >> 8) & 7u);
        const int abits = (int)((ac >> 12) & 63u);
        const uint32_t id = read_one_group(st + (ac >> 18) + group_in_stage * abits, j, abits);
        if (fn == 1 || fn == 4) {
          if (sum_in_double(vk)) {
            const double x = vk == VAL_DICT_F32 ? (double)__ldg(static_cast<const float*>(sd.dict[a]) + id)
                           : vk == VAL_DICT_I64 ? (double)__ldg(static_cast<const long long*>(sd.dict[a]) + id)
                                                : __ldg(static_cast<const double*>(sd.dict[a]) + id);
            double* slot = reinterpret_cast<double*>(acc64 + a * kConsumers + group);
            *slot += x;
          } else {
            const long long x = vk == VAL_DICT_I32 ? (long long)(int)(__ldg(static_cast<const uint32_t*>(sd.dict[a]) + id) ^ 0x80000000u)
                                                   : (long long)(int)id;
            acc64[a * kConsumers + group] += (unsigned long long)x;
          }
        } else if (fn == 2 || fn == 3) {
          const uint32_t x = id ^ (vk == VAL_RAW_I32 ? 0x80000000u : 0u);
          uint2 mmx = accmm[a * kConsumers + group];
          mmx.x = min(mmx.x, x); mmx.y = max(mmx.y, x + 1u);
          accmm[a * kConsumers + group] = mmx;
        } else if (fn == 5) {
          atomicOr(sd.distinct_bits[a] + (id >> 5), 1u << (id & 31));
        }
      }
    };
    bool handled = false;
    if (GROUPBY && wmax2 == 0) handled = true;
    if (GROUPBY && !handled) {
      // ---- survivor queue: the warp's surviving rows are compacted into a shared-memory queue (exclusive scan of the
      //      per-thread counts), then the lanes take queue entries round-robin: every table update and dictionary gather
      //      is a DENSE warp instruction over survivors (the DocIdSet -> Projection step of the reference) instead of a
      //      predicated one per row slot.  At 10 % selectivity that is ~4 dense iterations instead of 32 row slots.
      int incl = pc;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
      const int S = __shfl_sync(0xFFFFFFFFu, incl, 31);
      if (S == 0) handled = true;
      else {
        unsigned short* wq = reinterpret_cast<unsigned short*>(smem_base + q.queue_off) + warp * 1024;
        int pos = incl - pc;
        uint32_t mm = m;
        while (mm) {
          const int j = 31 - __clz(mm);
          mm &= ~(1u << j);
          wq[pos++] = (unsigned short)((lane << 5) | j);
        }
        __syncwarp();
        // kQB queue entries per lane and step: their smem probes, dictionary gathers and table updates are issued as
        // groups (all keys, all gathers, all reductions) so that kQB latency chains overlap instead of running back to back.
        // The loop is warp-uniform (validity is per entry) so that "last batch" is a uniform decision.
        const int ncodes = sd.num_agg_codes;
        const int ndefer = sd.num_defer_codes;
        for (int b0 = 0; b0 < S; b0 += 32 * kQB) {
          const int i0 = b0 + lane;
          const bool last = b0 + 32 * kQB >= S;
          uint32_t e[kQB], g[kQB];
          bool ok[kQB];
#pragma unroll
          for (int u = 0; u < kQB; ++u) { ok[u] = i0 + 32 * u < S; e[u] = ok[u] ? (uint32_t)wq[i0 + 32 * u] : 0u; g[u] = 0u; }
          if (sd.h_keys) {  // hash table: 64-bit raw key -> slot
            unsigned long long key[kQB];
#pragma unroll
            for (int u = 0; u < kQB; ++u) key[u] = 0ull;
#pragma unroll 1
            for (int gi = 0; gi < q.num_group_by; ++gi) {
              const SlotDesc& sl = sd.slots[hdr->group_slot[gi]];
              const uint32_t* gb = st + sl.stage_words;
              const unsigned long long mult = sd.group_mult64[gi];
#pragma unroll
              for (int u = 0; u < kQB; ++u) key[u] += read_one_group(gb + (e[u] >> 5) * sl.bits, (int)(e[u] & 31u), sl.bits) * mult;
            }
#pragma unroll
            for (int u = 0; u < kQB; ++u) if (ok[u]) ok[u] = hash_slot(sd, key[u], g[u]);
          } else {
#pragma unroll 1
            for (int gi = 0; gi < q.num_group_by; ++gi) {
              const SlotDesc& sl = sd.slots[hdr->group_slot[gi]];
              const uint32_t* gb = st + sl.stage_words;
              const uint32_t mult = sd.group_mult[gi];
#pragma unroll
              for (int u = 0; u < kQB; ++u) g[u] += read_one_group(gb + (e[u] >> 5) * sl.bits, (int)(e[u] & 31u), sl.bits) * mult;
            }
          }
          if (TG) {
#pragma unroll
            for (int u = 0; u < kQB; ++u) if (ok[u]) atomicAdd(tcnt + tcopy + g[u], 1u);
          } else if (sd.g_count) {
#pragma unroll
            for (int u = 0; u < kQB; ++u) if (ok[u]) red_add_u64(sd.g_count + g[u], 1ull);
          } else if (sd.g_seen) {
            uint32_t cur[kQB];
#pragma unroll
            for (int u = 0; u < kQB; ++u) cur[u] = ok[u] ? __ldcg(sd.g_seen + g[u]) : 1u;
#pragma unroll
            for (int u = 0; u < kQB; ++u) if (cur[u] == 0u) sd.g_seen[g[u]] = 1u;
          }
          // ---- software-pipelined aggregations of the last batch: issue the loads, reduce one tile later (drain_gb) ----
          const int nimm = last ? ncodes - ndefer : ncodes;
          if (last && ndefer > 0) {
            uint32_t okm = 0;
#pragma unroll
            for (int u = 0; u < kQB; ++u) { okm |= (ok[u] ? 1u : 0u) << u; pg[u] = g[u]; }
#pragma unroll
            for (int k = 0; k < kGD; ++k) {
              if (k < ndefer) {
                const uint32_t ac = sd.agg_code[ncodes - ndefer + k];
                const int a = (int)(ac & 7u), fn = (int)((ac >> 4) & 7u), vk = (int)((ac >> 8) & 7u);
                const int abits = (int)((ac >> 12) & 63u);
                const uint32_t* base = st + (ac >> 18);
                uint32_t id[kQB];
#pragma unroll
                for (int u = 0; u < kQB; ++u) id[u] = read_one_group(base + (e[u] >> 5) * abits, (int)(e[u] & 31u), abits);
                if (fn == 1 || fn == 4) {   // 4-byte dictionaries only (host rule): biased INT or FLOAT bits
                  const uint32_t* d = static_cast<const uint32_t*>(sd.dict[a]);
#pragma unroll
                  for (int u = 0; u < kQB; ++u) px[k][u] = (uint32_t)ldg_pred_s32(reinterpret_cast<const int*>(d + id[u]), ok[u] ? 1u : 0u);
                } else {
                  const uint32_t bias = vk == VAL_RAW_I32 ? 0x80000000u : 0u;
                  const uint32_t* tab = fn == 2 ? sd.g_min[a] : sd.g_max[a];
#pragma unroll
                  for (int u = 0; u < kQB; ++u) {
                    pq[k][u] = id[u] ^ bias;
                    px[k][u] = ok[u] ? __ldcg(tab + g[u]) : (fn == 2 ? 0u : 0xFFFFFFFFu);
                  }
                }
              }
            }
            pend_ok = okm;
          }
#pragma unroll 1
          for (int ai = 0; ai < nimm; ++ai) {
            const uint32_t ac = sd.agg_code[ai];  // index | function | value kind | bits | stage_words (pb200_desc.h)
            const int a = (int)(ac & 7u), fn = (int)((ac >> 4) & 7u), vk = (int)((ac >> 8) & 7u);
            const int abits = (int)((ac >> 12) & 63u);
            const uint32_t* base = st + (ac >> 18);
            uint32_t id[kQB];
#pragma unroll
            for (int u = 0; u < kQB; ++u) id[u] = read_one_group(base + (e[u] >> 5) * abits, (int)(e[u] & 31u), abits);
            if (fn == 1 || fn == 4) {
              if (sum_in_double(vk)) {
                double x[kQB];
#pragma unroll
                for (int u = 0; u < kQB; ++u)
                  x[u] = vk == VAL_DICT_F32 ? (double)__ldg(static_cast<const float*>(sd.dict[a]) + id[u])
                       : vk == VAL_DICT_I64 ? (double)__ldg(static_cast<const long long*>(sd.dict[a]) + id[u])
                                            : __ldg(static_cast<const double*>(sd.dict[a]) + id[u]);
#pragma unroll
                for (int u = 0; u < kQB; ++u) if (ok[u]) red_add_f64(sd.g_dsum[a] + g[u], x[u]);
              } else {
                long long x[kQB];
#pragma unroll
                for (int u = 0; u < kQB; ++u)
                  x[u] = vk == VAL_DICT_I32 ? (long long)((unsigned long long)__ldg(static_cast<const uint32_t*>(sd.dict[a]) + id[u]) + sd.sum_addend[a])
                                            : (long long)(int)id[u];
                if (TG) {
                  uint32_t* lo = tcnt + tcopy + TA * (1u + 2u * q.smem_slot[a]);
#pragma unroll
                  for (int u = 0; u < kQB; ++u) if (ok[u]) smem_add64(lo, lo + TA, g[u], (int)x[u]);
                } else {
                  unsigned long long* gs = reinterpret_cast<unsigned long long*>(sd.g_isum[a]);
#pragma unroll
                  for (int u = 0; u < kQB; ++u) if (ok[u]) red_add_u64(gs + g[u], (unsigned long long)x[u]);
                }
              }
            } else if (fn == 5) {  // DISTINCTCOUNT: the group's dictId bitset (RoaringBitmap per group in the reference)
              uint32_t* bits = sd.distinct_bits[a];
              const size_t wpg = sd.distinct_words[a];
#pragma unroll
              for (int u = 0; u < kQB; ++u) if (ok[u]) atomicOr(bits + (size_t)g[u] * wpg + (id[u] >> 5), 1u << (id[u] & 31u));
            } else if (fn == 2 || fn == 3) {
              // MIN / MAX tables change for only O(log n) of a group's rows: read the current entries first, then issue
              // a reduction only where the row can win (a stale read costs a redundant reduction, never a wrong result)
              const uint32_t bias = vk == VAL_RAW_I32 ? 0x80000000u : 0u;
              uint32_t* tab = fn == 2 ? sd.g_min[a] : sd.g_max[a];
              uint32_t cur[kQB];
#pragma unroll
              for (int u = 0; u < kQB; ++u) cur[u] = ok[u] ? __ldcg(tab + g[u]) : (fn == 2 ? 0u : 0xFFFFFFFFu);
#pragma unroll
              for (int u = 0; u < kQB; ++u) {
                const uint32_t x = id[u] ^ bias;
                if (fn == 2) { if (x < cur[u]) atomicMin(tab + g[u], x); }
                else { if (x + 1u > cur[u]) atomicMax(tab + g[u], x + 1u); }
              }
            }
          }
        }
        handled = true;  // the __syncwarp() before the ring refill also orders the queue reads before the next appends
      }
    }
    if (handled) {
    } else if (wmax2 > 0 && wmax2 <= q.sparse_max_agg) {
      uint32_t mm = m;
      while (mm) {
        const int j = 31 - __clz(mm);
        mm &= ~(1u << j);
        process_row(j);
      }
    } else if (wmax2 > 0) {
      // ---- dense projection ----
      if (!GROUPBY) {
#pragma unroll 1
        for (int ai = 0; ai < sd.num_agg_codes; ++ai) {
          const uint32_t ac = sd.agg_code[ai];  // index | function | value kind | bits | stage_words (pb200_desc.h)
          const int a = (int)(ac & 7u), fn = (int)((ac >> 4) & 7u), vk = (int)((ac >> 8) & 7u);
          const int abits = (int)((ac >> 12) & 63u);
          const uint32_t* base = st + (ac >> 18);
          if (DEFER && (fn == 1 || fn == 4) && vk == VAL_DICT_I32 && a == q.defer_agg) {
            // gathers of biased INT dictionary values (device copy holds value ^ 0x80000000) are only ISSUED here;
            // they are summed after the next tile's filter phase (drain())
            if constexpr (DEFER) {
              GatherBiasedU32 f{static_cast<const uint32_t*>(sd.dict[a]), m, (uint32_t)(32 - abits), x};
              dispatch_left_aligned(abits, base, group_in_stage, f);
              pend_pc = pc;
            }
          } else if ((fn == 1 || fn == 4) && vk == VAL_DICT_I32) {
            SumBiasedU32 f;
            f.d = static_cast<const uint32_t*>(sd.dict[a]); f.m = m; f.sh = 32 - abits;
            dispatch_left_aligned(abits, base, group_in_stage, f);
            acc64[a * kConsumers + group] += (f.a0 + f.a1) - ((unsigned long long)pc << 31);
          } else if ((fn == 2 || fn == 3) && vk != VAL_RAW_I32) {
            MinMaxLeft f;
            f.m = m;
            dispatch_left_aligned(abits, base, group_in_stage, f);
            if (pc) {
              const int sh = 32 - abits;
              uint2 mmx = accmm[a * kConsumers + group];
              mmx.x = min(mmx.x, f.mn >> sh);
              mmx.y = max(mmx.y, (f.mx >> sh) + 1u);
              accmm[a * kConsumers + group] = mmx;
            }
          } else {
            uint32_t v[32];
            unpack_group(abits, base, group_in_stage, v);
            if (fn == 1 || fn == 4) {
              if (vk == VAL_RAW_I32) {
                long long acc = 0;
#pragma unroll
                for (int j = 0; j < 32; ++j) acc += ((m >> j) & 1u) ? (long long)(int)v[j] : 0ll;
                acc64[a * kConsumers + group] += (unsigned long long)acc;
              } else {
                double acc = 0.0;
                if (vk == VAL_DICT_I64) {
                  const long long* __restrict__ d = static_cast<const long long*>(sd.dict[a]);
#pragma unroll
                  for (int j = 0; j < 32; ++j) acc += (double)ldg_pred_s64(d + v[j], (m >> j) & 1u);
                } else if (vk == VAL_DICT_F32) {
                  const float* __restrict__ d = static_cast<const float*>(sd.dict[a]);
#pragma unroll
                  for (int j = 0; j < 32; ++j) acc += (double)__int_as_float(ldg_pred_s32(reinterpret_cast<const int*>(d + v[j]), (m >> j) & 1u));
                } else {
                  const double* __restrict__ d = static_cast<const double*>(sd.dict[a]);
#pragma unroll
                  for (int j = 0; j < 32; ++j) acc += __longlong_as_double(ldg_pred_s64(reinterpret_cast<const long long*>(d + v[j]), (m >> j) & 1u));
                }
                double* slot = reinterpret_cast<double*>(acc64 + a * kConsumers + group);
                *slot += acc;
              }
            } else if (fn == 2 || fn == 3) {  // raw INT: signed -> unsigned order
              uint32_t tmn = 0xFFFFFFFFu, tmx = 0u;
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if ((m >> j) & 1u) { const uint32_t x = v[j] ^ 0x80000000u; tmn = min(tmn, x); tmx = max(tmx, x + 1u); }
              uint2 mmx = accmm[a * kConsumers + group];
              mmx.x = min(mmx.x, tmn); mmx.y = max(mmx.y, tmx);
              accmm[a * kConsumers + group] = mmx;
            } else if (fn == 5) {  // DISTINCTCOUNT: bitset of dictIds (RoaringBitmap.addN in the reference)
              uint32_t* bits = sd.distinct_bits[a];
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if ((m >> j) & 1u) atomicOr(bits + (v[j] >> 5), 1u << (v[j] & 31));
            }
          }
        }
      }
    }

    if (use_pipe) {
      __syncwarp();  // every lane is done reading this buffer
      if (Tp < q.total_tiles) issue(stage);
      if (++stage == q.num_stages) { stage = 0; phase ^= 1u; }
    }
  }
  if (sidx >= 0) flush();
  if (GROUPBY && TG) {
    consumer_bar_sync(kConsumers);  // every warp's rows are in the table
    if (sidx >= 0) table_flush();
  }
}

}  // namespace pb200
