// pb200_unpack.cuh -- device-side decode of Pinot's fixed-bit forward index.
//
// Format (reference: pinot-segment-local/.../io/util/PinotDataBitSet.java:143-170 writer,
// .../io/reader/impl/FixedBitIntReader.java read32 per width): value i occupies bits [i*B, (i+1)*B) of an MSB-first,
// big-endian bit stream.  Consequence used here (same as FixedBitIntReader.read32): 32 consecutive values whose first
// index is a multiple of 32 occupy exactly B consecutive, 4-byte aligned big-endian words -- no carry between groups.
//
// HBM layout: the B-word groups are kept in the file's order, but every 4-byte word is stored in the GPU's native
// (little-endian) byte order -- the byte swap of the big-endian file words is done ONCE when the segment is uploaded
// (fwd_words_to_native in pb200_api.cu) instead of once per value group per query (a PRMT per word otherwise).
//
// GPU mapping: ONE THREAD owns one such group (32 rows).  Its B words sit contiguously in shared memory (the tile was
// brought in by a TMA bulk copy, so the layout is the HBM layout); lane l of a warp reads words
// [l*B, (l+1)*B).  With the widest naturally aligned load (LDS.128 when B%4==0, LDS.64 when B%2==0, else LDS.32) the
// lane stride is an odd multiple of the access width for every B except 8, 16 and 24, i.e. bank-conflict free; all
// shift amounts are compile-time constants after unrolling, so a value costs ~2 ALU ops (SHF/funnel + mask).
#pragma once
#include <cstdint>

namespace pb200 {

__host__ __device__ __forceinline__ uint32_t bswap32(uint32_t x) {
  return (x >> 24) | ((x >> 8) & 0xFF00u) | ((x << 8) & 0xFF0000u) | (x << 24);
}
// a forward-index word as the unpackers want it (MSB-first bit stream): identity on the native HBM layout
__device__ __forceinline__ uint32_t fwd_word(uint32_t x) { return x; }

template <int B>
struct Unpack32 {
  static_assert(B >= 1 && B <= 32, "bits per value");
  // p: this thread's first word (16-byte aligned when B%4==0, 8-byte aligned when B%2==0)
  static __device__ __forceinline__ void run(const uint32_t* __restrict__ p, uint32_t (&v)[32]) {
    uint32_t w[B];
    if constexpr (B % 4 == 0) {
      const uint4* p4 = reinterpret_cast<const uint4*>(p);
#pragma unroll
      for (int k = 0; k < B / 4; ++k) {
        uint4 x = p4[k];
        w[4 * k + 0] = fwd_word(x.x);
        w[4 * k + 1] = fwd_word(x.y);
        w[4 * k + 2] = fwd_word(x.z);
        w[4 * k + 3] = fwd_word(x.w);
      }
    } else if constexpr (B % 2 == 0) {
      const uint2* p2 = reinterpret_cast<const uint2*>(p);
#pragma unroll
      for (int k = 0; k < B / 2; ++k) {
        uint2 x = p2[k];
        w[2 * k + 0] = fwd_word(x.x);
        w[2 * k + 1] = fwd_word(x.y);
      }
    } else {
#pragma unroll
      for (int k = 0; k < B; ++k) w[k] = fwd_word(p[k]);
    }
    constexpr uint32_t kMask = B == 32 ? 0xFFFFFFFFu : ((1u << (B & 31)) - 1u);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int o = i * B;
      const int k = o >> 5;
      const int s = o & 31;
      if (s + B <= 32) {
        const int sh = 32 - s - B;
        if (s == 0) {
          v[i] = B == 32 ? w[k] : (w[k] >> sh);  // top of word: no mask needed
        } else if (sh == 0) {
          v[i] = w[k] & kMask;
        } else {
          v[i] = (w[k] >> sh) & kMask;
        }
      } else {
        // straddles w[k] (high part) and w[k+1]: funnel-shift left by s, keep the top B bits
        const int k1 = (k + 1 < B) ? k + 1 : k;  // (always k+1 < B when straddling; keeps indexing static)
        v[i] = __funnelshift_l(w[k1], w[k], s) >> (32 - B);
      }
    }
  }
};

// Streaming form: calls f(j, xl) for the 32 values in order, j a compile-time constant after unrolling and xl the value
// LEFT-aligned in 32 bits (top B bits = the value, lower bits = whatever follows it in the stream).  Left alignment
// costs ONE shift (a funnel shift when the value straddles two words) and is enough for order comparisons:
//   v >= lo  <=>  xl >= (lo << (32-B)),   v < hi  <=>  xl < (hi << (32-B))        (low garbage bits < 2^(32-B))
// while v itself is xl >> (32-B).  Only the B loaded words stay live (no 32-value register array), which is what lets
// two CTAs share an SM.
template <int B, class F>
__device__ __forceinline__ void for_each_left_aligned(const uint32_t* __restrict__ p, F& f) {
  static_assert(B >= 1 && B <= 32, "bits per value");
  uint32_t w[B];
  if constexpr (B % 4 == 0) {
    const uint4* p4 = reinterpret_cast<const uint4*>(p);
#pragma unroll
    for (int k = 0; k < B / 4; ++k) {
      uint4 x = p4[k];
      w[4 * k + 0] = fwd_word(x.x);
      w[4 * k + 1] = fwd_word(x.y);
      w[4 * k + 2] = fwd_word(x.z);
      w[4 * k + 3] = fwd_word(x.w);
    }
  } else if constexpr (B % 2 == 0) {
    const uint2* p2 = reinterpret_cast<const uint2*>(p);
#pragma unroll
    for (int k = 0; k < B / 2; ++k) {
      uint2 x = p2[k];
      w[2 * k + 0] = fwd_word(x.x);
      w[2 * k + 1] = fwd_word(x.y);
    }
  } else {
#pragma unroll
    for (int k = 0; k < B; ++k) w[k] = fwd_word(p[k]);
  }
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int o = i * B;
    const int k = o >> 5;
    const int s = o & 31;
    uint32_t xl;
    if (s == 0) {
      xl = w[k];
    } else if (s + B <= 32) {
      xl = w[k] << s;
    } else {
      const int k1 = (k + 1 < B) ? k + 1 : k;
      xl = __funnelshift_l(w[k1], w[k], s);
    }
    f(i, xl);
  }
}

template <class F>
__device__ __forceinline__ void dispatch_left_aligned(int bits, const uint32_t* __restrict__ base, int group, F& f) {
  switch (bits) {
#define PB200_CASE(B) \
  case B:             \
    for_each_left_aligned<B>(base + group * B, f); \
    break;
    PB200_CASE(1) PB200_CASE(2) PB200_CASE(3) PB200_CASE(4) PB200_CASE(5) PB200_CASE(6) PB200_CASE(7) PB200_CASE(8)
    PB200_CASE(9) PB200_CASE(10) PB200_CASE(11) PB200_CASE(12) PB200_CASE(13) PB200_CASE(14) PB200_CASE(15)
    PB200_CASE(16) PB200_CASE(17) PB200_CASE(18) PB200_CASE(19) PB200_CASE(20) PB200_CASE(21) PB200_CASE(22)
    PB200_CASE(23) PB200_CASE(24) PB200_CASE(25) PB200_CASE(26) PB200_CASE(27) PB200_CASE(28) PB200_CASE(29)
    PB200_CASE(30) PB200_CASE(31) PB200_CASE(32)
#undef PB200_CASE
    default:
      break;
  }
}

// Width is a per-(segment, column) runtime value but uniform across the whole tile: one switch, 32 specialisations.
// `group` is the thread's 32-row group index inside the tile; `base` the slot's first word in the stage buffer.
__device__ __forceinline__ void unpack_group(int bits, const uint32_t* __restrict__ base, int group,
                                             uint32_t (&v)[32]) {
  switch (bits) {
#define PB200_CASE(B) \
  case B:             \
    Unpack32<B>::run(base + group * B, v); \
    break;
    PB200_CASE(1) PB200_CASE(2) PB200_CASE(3) PB200_CASE(4) PB200_CASE(5) PB200_CASE(6) PB200_CASE(7) PB200_CASE(8)
    PB200_CASE(9) PB200_CASE(10) PB200_CASE(11) PB200_CASE(12) PB200_CASE(13) PB200_CASE(14) PB200_CASE(15)
    PB200_CASE(16) PB200_CASE(17) PB200_CASE(18) PB200_CASE(19) PB200_CASE(20) PB200_CASE(21) PB200_CASE(22)
    PB200_CASE(23) PB200_CASE(24) PB200_CASE(25) PB200_CASE(26) PB200_CASE(27) PB200_CASE(28) PB200_CASE(29)
    PB200_CASE(30) PB200_CASE(31) PB200_CASE(32)
#undef PB200_CASE
    default:
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = 0;
  }
}

// Random access to one value (FixedBitIntReader.readUnchecked shape; used by the sparse / post-bitmap paths):
// two aligned words cover any value of width <= 32.
__device__ __forceinline__ uint32_t read_one(const uint32_t* __restrict__ words, long long index, int bits) {
  const long long bit = index * bits;
  const long long k = bit >> 5;
  const int s = (int)(bit & 31);
  const uint32_t hi = fwd_word(words[k]);
  const uint32_t lo = (s + bits > 32) ? fwd_word(words[k + 1]) : 0u;
  const uint32_t x = __funnelshift_l(lo, hi, s);
  return bits == 32 ? x : (x >> (32 - bits));
}

}  // namespace pb200
