// raw_forward.cpp -- no-dictionary (raw) fixed-width single-value forward indexes at segment load.
//
// Reference: seglocal/segment/index/readers/forward/BaseChunkForwardIndexReader.java:60-106 (header: version, numChunks,
// numDocsPerChunk, lengthOfLongestEntry, [v2+: totalDocs, compressionType, dataHeaderStart], chunk offsets: int up to v2,
// long from v3), :204-240 (a chunk = the bytes up to the next chunk's offset / the end of the file, decompressed as a whole),
// FixedByteChunkSVForwardIndexReader.java:52-100 (value i of a chunk at i * width, big-endian),
// segment/spi/compression/ChunkCompressionType.java (PASS_THROUGH 0, SNAPPY 1, ZSTANDARD 2, LZ4 3, LZ4_LENGTH_PREFIXED 4, GZIP 5).
//
// What the reference does per VALUE at query time (decompress the chunk the doc falls into, read the value) happens here
// ONCE at load: all chunks are decoded into one flat big-endian value array.  Then
//   * columns with at most `max_cardinality` distinct values get a dictionary SYNTHESISED from their values (sorted like an
//     immutable Pinot dictionary) and a fixed-bit forward index of dictIds -- from there on the column is an ordinary
//     dictionary column for every device path (value predicates, GROUP BY, MIN / MAX / DISTINCTCOUNT, count carrier ...);
//     the reference's NoDictionary group-key generators and raw-value predicate evaluators produce the same VALUES, only
//     the internal ids differ (and those never leave the boundary un-decoded: pb200h_dictionary_get serves both kinds);
//   * wider value sets stay raw (pb200_api.cu streams 4-byte INT values; other widths are refused to the stock operator).
// Snappy (raw format) and LZ4 (block format) decoders are written from the formats' published descriptions; ZSTD / GZIP
// chunks are refused.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <unordered_map>

#include "host_internal.h"

namespace pb200h {
namespace {

inline uint32_t rd_be32(const unsigned char* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
inline uint64_t rd_be64(const unsigned char* p) { return (uint64_t)rd_be32(p) << 32 | rd_be32(p + 4); }

// Snappy raw format: varint uncompressed length, then elements tagged by the low 2 bits of their first byte:
// 00 literal (length - 1 in the upper 6 bits, 60..63 = that many - 59 length bytes follow), 01 copy with 11-bit offset,
// 10 copy with 16-bit offset, 11 copy with 32-bit offset (little-endian); copies may overlap their own output.
bool snappy_decode(const unsigned char* ip, size_t n, unsigned char* dst, size_t cap, size_t* produced) {
  const unsigned char* end = ip + n;
  uint64_t ulen = 0;
  int shift = 0;
  while (true) {
    if (ip >= end || shift > 35) return false;
    const unsigned char b = *ip++;
    ulen |= (uint64_t)(b & 0x7F) << shift;
    if (!(b & 0x80)) break;
    shift += 7;
  }
  if (ulen > cap) return false;
  size_t op = 0;
  while (ip < end) {
    const unsigned char tag = *ip++;
    size_t len, off;
    if ((tag & 3) == 0) {
      len = (size_t)(tag >> 2) + 1;
      if (len > 60) {
        const int nb = (int)len - 60;
        if (ip + nb > end) return false;
        len = 0;
        for (int i = 0; i < nb; i++) len |= (size_t)ip[i] << (8 * i);
        len += 1;
        ip += nb;
      }
      if (ip + len > end || op + len > ulen) return false;
      memcpy(dst + op, ip, len);
      ip += len; op += len;
      continue;
    }
    if ((tag & 3) == 1) {
      if (ip >= end) return false;
      len = 4 + ((tag >> 2) & 7);
      off = ((size_t)(tag >> 5) << 8) | *ip++;
    } else if ((tag & 3) == 2) {
      if (ip + 2 > end) return false;
      len = (size_t)(tag >> 2) + 1;
      off = (size_t)ip[0] | (size_t)ip[1] << 8;
      ip += 2;
    } else {
      if (ip + 4 > end) return false;
      len = (size_t)(tag >> 2) + 1;
      off = (size_t)ip[0] | (size_t)ip[1] << 8 | (size_t)ip[2] << 16 | (size_t)ip[3] << 24;
      ip += 4;
    }
    if (off == 0 || off > op || op + len > ulen) return false;
    for (size_t i = 0; i < len; i++) dst[op + i] = dst[op + i - off];
    op += len;
  }
  *produced = op;
  return op == ulen;
}

// LZ4 block format: sequences of [token][literal length extension][literals][offset LE16][match length extension];
// token = literal length (high nibble) | match length - 4 (low nibble), 15 = extended by 255-bytes; the last sequence ends
// after its literals.
bool lz4_block_decode(const unsigned char* ip, size_t n, unsigned char* dst, size_t cap, size_t* produced) {
  const unsigned char* end = ip + n;
  size_t op = 0;
  while (ip < end) {
    const unsigned char token = *ip++;
    size_t lit = token >> 4;
    if (lit == 15) {
      unsigned char b;
      do { if (ip >= end) return false; b = *ip++; lit += b; } while (b == 255);
    }
    if (ip + lit > end || op + lit > cap) return false;
    memcpy(dst + op, ip, lit);
    ip += lit; op += lit;
    if (ip >= end) break;  // last sequence: literals only
    if (ip + 2 > end) return false;
    const size_t off = (size_t)ip[0] | (size_t)ip[1] << 8;
    ip += 2;
    size_t ml = token & 15;
    if (ml == 15) {
      unsigned char b;
      do { if (ip >= end) return false; b = *ip++; ml += b; } while (b == 255);
    }
    ml += 4;
    if (off == 0 || off > op || op + ml > cap) return false;
    for (size_t i = 0; i < ml; i++) dst[op + i] = dst[op + i - off];
    op += ml;
  }
  *produced = op;
  return true;
}

// order-preserving 64-bit key of a stored value (Pinot dictionaries are sorted by Integer / Long / Float / Double.compare).
// Equal keys are one dictionary entry: every NaN bit pattern becomes the canonical NaN first (Float.floatToIntBits /
// Double.doubleToLongBits), so all NaNs are one value, sorted after +inf; -0.0 and 0.0 stay two values.
inline uint64_t sort_key(const unsigned char* p, int data_type) {
  switch (data_type) {
    case PB200_INT: return (uint64_t)((int64_t)(int32_t)rd_be32(p)) ^ 0x8000000000000000ull;
    case PB200_LONG: return rd_be64(p) ^ 0x8000000000000000ull;
    case PB200_FLOAT: {
      uint32_t u = rd_be32(p);
      if ((u & 0x7FFFFFFFu) > 0x7F800000u) u = 0x7FC00000u;
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
      return u;
    }
    default: {
      uint64_t u = rd_be64(p);
      if ((u & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull) u = 0x7FF8000000000000ull;
      return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
    }
  }
}
inline void store_key(uint64_t k, int data_type, unsigned char* p) {
  if (data_type == PB200_INT || data_type == PB200_FLOAT) {
    uint32_t u;
    if (data_type == PB200_INT) u = (uint32_t)(int32_t)(int64_t)(k ^ 0x8000000000000000ull);
    else { u = (uint32_t)k; u = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u; }
    p[0] = (unsigned char)(u >> 24); p[1] = (unsigned char)(u >> 16); p[2] = (unsigned char)(u >> 8); p[3] = (unsigned char)u;
    return;
  }
  uint64_t u;
  if (data_type == PB200_LONG) u = k ^ 0x8000000000000000ull;
  else u = (k & 0x8000000000000000ull) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
  for (int i = 0; i < 8; i++) p[i] = (unsigned char)(u >> (56 - 8 * i));
}

}  // namespace

int raw_value_width(int data_type) {
  return data_type == PB200_INT || data_type == PB200_FLOAT ? 4 : data_type == PB200_LONG || data_type == PB200_DOUBLE ? 8 : 0;
}

int decode_fixed_byte_forward(const unsigned char* b, uint64_t len, int width, int64_t num_docs, std::vector<unsigned char>& out) {
  if (!b || len < 16 || width <= 0) { set_error("raw forward index too short"); return PB200_E_INVALID; }
  const int version = (int)rd_be32(b), nchunks = (int)rd_be32(b + 4), per_chunk = (int)rd_be32(b + 8), entry = (int)rd_be32(b + 12);
  int compression = 1;  // version 1: always Snappy (BaseChunkForwardIndexReader.java:92-96)
  uint64_t header = 16;
  if (version > 1) {
    if (len < 28) { set_error("raw forward index header truncated"); return PB200_E_INVALID; }
    compression = (int)rd_be32(b + 20);
    header = rd_be32(b + 24);
  }
  if (version < 1 || version > 4 || nchunks < 0 || per_chunk <= 0 || entry != width) {
    set_error("raw forward index: version %d, %d chunks of %d docs, entry width %d (expected %d) not understood", version, nchunks, per_chunk, entry, width);
    return PB200_E_UNSUPPORTED;
  }
  if ((uint64_t)per_chunk * (uint64_t)width > (1ull << 30)) { set_error("raw forward index: %d docs per chunk is not plausible", per_chunk); return PB200_E_INVALID; }
  const int osz = version <= 2 ? 4 : 8;
  const uint64_t data_start = header + (uint64_t)nchunks * osz;
  if (data_start > len || (int64_t)nchunks * per_chunk < num_docs) { set_error("raw forward index: chunk table does not cover %lld docs", (long long)num_docs); return PB200_E_INVALID; }
  out.assign((size_t)num_docs * width, 0);
  if (compression == 0) {
    if (len < data_start + (uint64_t)num_docs * width) { set_error("raw forward index: data truncated"); return PB200_E_INVALID; }
    memcpy(out.data(), b + data_start, (size_t)num_docs * width);
    return PB200_OK;
  }
  if (compression != 1 && compression != 3 && compression != 4) {
    set_error("raw forward index: chunk compression %d (ZSTANDARD / GZIP) is not decoded by this loader", compression);
    return PB200_E_UNSUPPORTED;
  }
  std::vector<unsigned char> chunk((size_t)per_chunk * width);
  for (int c = 0; c < nchunks; c++) {
    const int64_t first = (int64_t)c * per_chunk;
    if (first >= num_docs) break;
    const unsigned char* e = b + header + (uint64_t)c * osz;
    const uint64_t pos = osz == 4 ? rd_be32(e) : rd_be64(e);
    const uint64_t next = c + 1 < nchunks ? (osz == 4 ? rd_be32(e + osz) : rd_be64(e + osz)) : len;
    if (pos > next || next > len) { set_error("raw forward index: chunk %d offsets out of range", c); return PB200_E_INVALID; }
    const unsigned char* src = b + pos;
    size_t n = (size_t)(next - pos), produced = 0;
    bool ok;
    if (compression == 1) ok = snappy_decode(src, n, chunk.data(), chunk.size(), &produced);
    else {
      if (compression == 4) {  // LZ4CompressorWithLength: little-endian decompressed length, then the block
        if (n < 4) { set_error("raw forward index: chunk %d too short", c); return PB200_E_INVALID; }
        src += 4; n -= 4;
      }
      ok = lz4_block_decode(src, n, chunk.data(), chunk.size(), &produced);
    }
    const int64_t docs_here = std::min<int64_t>(per_chunk, num_docs - first);
    if (!ok || produced < (size_t)docs_here * width) { set_error("raw forward index: chunk %d does not decompress (compression %d)", c, compression); return PB200_E_INVALID; }
    memcpy(out.data() + (size_t)first * width, chunk.data(), (size_t)docs_here * width);
  }
  return PB200_OK;
}

void wrap_pass_through(const std::vector<unsigned char>& values_be, int width, int64_t num_docs, std::vector<unsigned char>& out) {
  // one-chunk version-2 PASS_THROUGH file around already decoded values (what pb200_segment_register parses)
  out.assign(32 + values_be.size(), 0);
  auto put = [&](size_t at, uint32_t v) { out[at] = (unsigned char)(v >> 24); out[at + 1] = (unsigned char)(v >> 16); out[at + 2] = (unsigned char)(v >> 8); out[at + 3] = (unsigned char)v; };
  put(0, 2); put(4, 1); put(8, (uint32_t)std::max<int64_t>(num_docs, 1)); put(12, (uint32_t)width); put(16, (uint32_t)num_docs); put(20, 0); put(24, 28); put(28, 32);
  memcpy(out.data() + 32, values_be.data(), values_be.size());
}

bool synthesize_dictionary(const std::vector<unsigned char>& values_be, int data_type, int64_t num_docs, int max_cardinality,
                           std::vector<unsigned char>& dict_be, std::vector<unsigned char>& fwd_packed, int* cardinality, int* bits) {
  const int width = raw_value_width(data_type);
  if (width == 0 || num_docs <= 0) return false;
  // pass 1: distinct keys in an open-addressing set that gives up once the column is wider than max_cardinality
  size_t cap = 1;
  while (cap < (size_t)max_cardinality * 2 + 2) cap <<= 1;
  const uint64_t kEmpty = ~0ull;  // also the key of LONG Long.MAX_VALUE: handled below
  std::vector<uint64_t> slots(cap, kEmpty);
  std::vector<uint64_t> distinct;
  bool has_all_ones = false;
  auto hash = [&](uint64_t k) { k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; return (size_t)k & (cap - 1); };
  const unsigned char* p = values_be.data();
  for (int64_t i = 0; i < num_docs; i++, p += width) {
    const uint64_t k = sort_key(p, data_type);
    if (k == kEmpty) { if (!has_all_ones) { has_all_ones = true; distinct.push_back(k); } continue; }
    size_t h = hash(k);
    while (slots[h] != kEmpty && slots[h] != k) h = (h + 1) & (cap - 1);
    if (slots[h] == k) continue;
    if ((int64_t)distinct.size() >= max_cardinality) return false;
    slots[h] = k;
    distinct.push_back(k);
  }
  std::sort(distinct.begin(), distinct.end());
  const int card = (int)distinct.size();
  int nb = 1;
  while (nb < 31 && (1ll << nb) < card) nb++;  // PinotDataBitSet.getNumBitsPerValue(cardinality - 1)
  dict_be.assign((size_t)card * width, 0);
  for (int i = 0; i < card; i++) store_key(distinct[i], data_type, dict_be.data() + (size_t)i * width);
  // pass 2: ids (the set's slots now carry the id next to the key)
  std::vector<int32_t> slot_id(cap, -1);
  int all_ones_id = -1;
  for (int i = 0; i < card; i++) {
    const uint64_t k = distinct[i];
    if (k == kEmpty) { all_ones_id = i; continue; }
    size_t h = hash(k);
    while (slots[h] != k) h = (h + 1) & (cap - 1);
    slot_id[h] = i;
  }
  // FixedBitSVForwardIndexWriter layout: value i occupies bits [i * nb, (i + 1) * nb), most significant bit first
  const size_t bytes = ((size_t)num_docs * nb + 7) / 8;
  fwd_packed.assign(bytes, 0);
  p = values_be.data();
  uint64_t acc = 0; int have = 0; size_t at = 0;
  for (int64_t i = 0; i < num_docs; i++, p += width) {
    const uint64_t k = sort_key(p, data_type);
    int id;
    if (k == kEmpty) id = all_ones_id;
    else { size_t h = hash(k); while (slots[h] != k) h = (h + 1) & (cap - 1); id = slot_id[h]; }
    acc = (acc << nb) | (uint64_t)(uint32_t)id;
    have += nb;
    while (have >= 8) { fwd_packed[at++] = (unsigned char)(acc >> (have - 8)); have -= 8; }
  }
  if (have > 0) fwd_packed[at++] = (unsigned char)(acc << (8 - have));
  *cardinality = card;
  *bits = nb;
  return true;
}

}  // namespace pb200h
