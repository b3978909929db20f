// pinot_oracle.cpp -- CPU parity oracle (TEST INFRASTRUCTURE ONLY; see pinot_oracle.h).
//
// A restatement, not a translation: every function cites the reference code (y-scope/pinot @ 1.3.0-SNAPSHOT,
// paths relative to /root/reference) whose behaviour it reproduces.  Abbreviations:
//   core/     = pinot-core/src/main/java/org/apache/pinot/core/
//   seglocal/ = pinot-segment-local/src/main/java/org/apache/pinot/segment/local/
//
// Shape: the executor is deliberately "reference shaped" -- doc-id iterators with next()/advance(), 256-doc scan
// batches, 10 000-doc projection blocks, per-block double accumulation in Java's order -- so that (a) SUM/AVG values are
// the ones the JVM would produce (the 1e-6 tolerance is tested against Java-order doubles), (b) ExecutionStatistics
// (numEntriesScannedInFilter ...) can be compared with the reference's asserted numbers, and (c) timing it is a fair
// stand-in for the JVM path's algorithmic shape (kind "port" in bench.py's cpu_baseline).

#include "pinot_oracle.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <limits>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

namespace {

constexpr int kEOF = std::numeric_limits<int>::min();  // core/common/Constants.java EOF = Integer.MIN_VALUE
constexpr int kMaxDocPerCall = 10000;                  // core/plan/DocIdSetPlanNode.java:29
constexpr int kScanBatch = 256;                        // core/common/BlockDocIdIterator.java:49

// ------------------------------------------------------------------------------------------------------------------
// Big-endian loads (PinotDataBuffer views of index files are BIG_ENDIAN: segspi/memory/PinotDataBuffer.java:54-55)
// ------------------------------------------------------------------------------------------------------------------
inline uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
inline uint64_t be64(const uint8_t* p) { return (uint64_t)be32(p) << 32 | be32(p + 4); }
inline uint16_t le16(const uint8_t* p) { return (uint16_t)(p[0] | p[1] << 8); }
inline uint32_t le32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
inline uint64_t le64(const uint8_t* p) { return (uint64_t)le32(p) | (uint64_t)le32(p + 4) << 32; }

// ------------------------------------------------------------------------------------------------------------------
// PinotDataBitSet (seglocal/io/util/PinotDataBitSet.java)
// ------------------------------------------------------------------------------------------------------------------
// getNumBitsPerValue :61-72 -- at least one bit; position of the highest set bit of maxValue.
int num_bits_per_value(int max_value) {
  if (max_value <= 1) return 1;
  int bits = 0;
  uint32_t v = (uint32_t)max_value;
  while (v) { bits++; v >>= 1; }
  return bits;
}

// writeInt(index, numBits, value) :143-170 -- MSB-first bit stream, byte at a time, preserving neighbouring bits.
void bitset_write_one(uint8_t* buf, int64_t index, int bits, int32_t value) {
  int64_t bit_offset = index * bits;
  int64_t byte_offset = bit_offset / 8;
  int in_first = (int)(bit_offset % 8);
  int first_byte = buf[byte_offset];
  int first_mask = 0xFF >> in_first;
  int left = bits - (8 - in_first);
  if (left <= 0) {
    first_mask &= 0xFF << -left;
    buf[byte_offset] = (uint8_t)((first_byte & ~first_mask) | ((value << -left) & first_mask));
  } else {
    buf[byte_offset] = (uint8_t)((first_byte & ~first_mask) | (((uint32_t)value >> left) & first_mask));
    while (left > 8) {
      left -= 8;
      byte_offset++;
      buf[byte_offset] = (uint8_t)(value >> left);
    }
    byte_offset++;
    int last = buf[byte_offset];
    buf[byte_offset] = (uint8_t)((last & (0xFF >> left)) | (value << (8 - left)));
  }
}

// readInt(index, numBits) :80-102 -- the byte-wise (bounds-safe) reader.
int32_t bitset_read_one(const uint8_t* buf, int64_t index, int bits) {
  int64_t bit_offset = index * bits;
  int64_t byte_offset = bit_offset / 8;
  int in_first = (int)(bit_offset % 8);
  int cur = buf[byte_offset] & (0xFF >> in_first);
  int left = bits - (8 - in_first);
  if (left <= 0) return cur >> -left;
  while (left > 8) {
    byte_offset++;
    cur = (cur << 8) | buf[byte_offset];
    left -= 8;
  }
  return (int32_t)(((uint32_t)cur << left) | (buf[byte_offset + 1] >> (8 - left)));
}

// ------------------------------------------------------------------------------------------------------------------
// FixedBitIntReader (seglocal/io/reader/impl/FixedBitIntReader.java)
// The reference hand-unrolls 31 classes; all follow one pattern which is restated generically here:
//   readUnchecked: b<=25 -> one BE int load at byte (i*b)>>>3, shift by (32-b-bit) (e.g. 17-bit :1278-1283, 25-bit
//                  :1960-1965); b>=26 -> one BE long load, shift by (64-b-bit) (31-bit :2515-2520).
//   read:          bounds-safe variant (byte/short loads); value-identical to PinotDataBitSet.readInt.
//   read32:        index%32==0; consumes exactly b BE ints at byte offset (index>>>3)*b (e.g. 17-bit :1286-1340).
// ------------------------------------------------------------------------------------------------------------------
int32_t fixedbit_read_unchecked(const uint8_t* buf, int64_t index, int bits) {
  int64_t bit_offset = index * bits;
  int64_t off = bit_offset >> 3;
  int bit = (int)(bit_offset & 7);
  if (bits <= 25) return (int32_t)((be32(buf + off) >> (32 - bits - bit)) & ((1u << bits) - 1));
  return (int32_t)((be64(buf + off) >> (64 - bits - bit)) & ((1ull << bits) - 1));
}

void fixedbit_read32(const uint8_t* buf, int64_t index, int bits, int32_t* out) {
  const uint8_t* p = buf + (index >> 3) * bits;
  // 32 values == `bits` big-endian 32-bit words; walk a 64-bit window over them.
  uint64_t window = 0;
  int have = 0, w = 0;
  const uint32_t mask = bits == 32 ? 0xFFFFFFFFu : ((1u << bits) - 1);
  for (int i = 0; i < 32; i++) {
    if (have < bits) {
      window = (window << 32) | be32(p + 4 * w++);
      have += 32;
    }
    out[i] = (int32_t)((window >> (have - bits)) & mask);
    have -= bits;
  }
}

// FixedBitSVForwardIndexReaderV2.readDictIds
// (seglocal/segment/index/readers/forward/FixedBitSVForwardIndexReaderV2.java:65-99)
void fwd_read_dict_ids(const uint8_t* buf, int num_docs, int bits, const int32_t* doc_ids, int length, int32_t* out) {
  if (length <= 0) return;
  int first = doc_ids[0], last = doc_ids[length - 1];
  int index = 0;
  if (last - first + 1 == length && length >= 64) {  // bulk path only for contiguous doc ids
    int bulk_start = (first + 31) & ~31;
    int bulk_end = last & ~31;
    for (int i = first; i < bulk_start; i++) out[index++] = fixedbit_read_unchecked(buf, i, bits);
    for (int i = bulk_start; i < bulk_end; i += 32) {
      fixedbit_read32(buf, i, bits, out + index);
      index += 32;
    }
  }
  if (last < num_docs - 2) {
    for (int i = index; i < length; i++) out[i] = fixedbit_read_unchecked(buf, doc_ids[i], bits);
  } else {  // the last two docs must use the bounds-safe reader
    out[length - 1] = bitset_read_one(buf, last, bits);
    int unchecked_end = length - 2;
    if (unchecked_end >= index) {
      out[unchecked_end] = bitset_read_one(buf, doc_ids[unchecked_end], bits);
      for (int i = index; i < unchecked_end; i++) out[i] = fixedbit_read_unchecked(buf, doc_ids[i], bits);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// RoaringBitmap portable serialization (third party, restated from RoaringFormatSpec; call sites:
// seglocal/segment/creator/impl/inv/BitmapInvertedIndexWriter.java:90-97 (serialize),
// seglocal/segment/index/readers/BitmapInvertedIndexReader.java:53-57 (ImmutableRoaringBitmap over the bytes)).
//   cookie 12346: [u32 cookie][u32 n] [n x (u16 key, u16 card-1)] [n x u32 offset] containers
//   cookie 12347: [u16 cookie][u16 n-1] [ceil(n/8) run flags] [n x (u16 key,u16 card-1)] [if n>=4: n x u32 offset] ...
//   containers: array (card<=4096): card x u16; bitmap: 1024 x u64; run: u16 nruns, nruns x (u16 start, u16 len-1)
// ------------------------------------------------------------------------------------------------------------------
constexpr uint32_t kCookieNoRun = 12346, kCookieRun = 12347;
constexpr int kNoOffsetThreshold = 4;

struct DenseBitmap {  // oracle's in-memory doc-id set: dense bitset over [0, num_docs)
  std::vector<uint64_t> w;
  int64_t n = 0;
  explicit DenseBitmap(int64_t nbits = 0) : w((nbits + 63) / 64, 0), n(nbits) {}
  void set(uint32_t i) { w[i >> 6] |= 1ull << (i & 63); }
  bool get(uint32_t i) const { return w[i >> 6] >> (i & 63) & 1; }
  void set_range(int64_t lo, int64_t hi) {  // [lo, hi)
    for (int64_t i = lo; i < hi;) {
      if ((i & 63) == 0 && i + 64 <= hi) { w[i >> 6] = ~0ull; i += 64; } else { set((uint32_t)i); i++; }
    }
  }
  int64_t cardinality() const { int64_t c = 0; for (uint64_t x : w) c += __builtin_popcountll(x); return c; }
  void and_with(const DenseBitmap& o) { for (size_t i = 0; i < w.size(); i++) w[i] &= o.w[i]; }
  void or_with(const DenseBitmap& o) { for (size_t i = 0; i < w.size(); i++) w[i] |= o.w[i]; }
  void flip_all() {  // flip(0, numDocs)
    for (auto& x : w) x = ~x;
    if (n & 63) w.back() &= (1ull << (n & 63)) - 1;
  }
  // next set bit >= from, or -1
  int64_t next_set(int64_t from) const {
    if (from >= n) return -1;
    size_t wi = from >> 6;
    uint64_t x = w[wi] & (~0ull << (from & 63));
    while (true) {
      if (x) { int64_t r = (int64_t)wi * 64 + __builtin_ctzll(x); return r < n ? r : -1; }
      if (++wi >= w.size()) return -1;
      x = w[wi];
    }
  }
};

// Iterate a serialized roaring bitmap, calling f(value) in ascending order. Returns cardinality or -1 if malformed.
template <class F>
int64_t roaring_for_each(const uint8_t* buf, int64_t len, F&& f) {
  if (len < 8) return -1;
  uint32_t cookie = le32(buf);
  int64_t pos;
  uint32_t n;
  const uint8_t* run_flags = nullptr;
  bool has_run = (cookie & 0xFFFF) == kCookieRun;
  if (has_run) {
    n = (cookie >> 16) + 1;
    pos = 4;
    run_flags = buf + pos;
    pos += (n + 7) / 8;
  } else if (cookie == kCookieNoRun) {
    n = le32(buf + 4);
    pos = 8;
  } else {
    return -1;
  }
  if (pos + 4ll * n > len) return -1;
  const uint8_t* desc = buf + pos;
  pos += 4ll * n;
  if (!has_run || (int)n >= kNoOffsetThreshold) pos += 4ll * n;  // offset header (not needed for sequential decode)
  int64_t total = 0;
  for (uint32_t c = 0; c < n; c++) {
    uint32_t key = le16(desc + 4 * c);
    uint32_t card = (uint32_t)le16(desc + 4 * c + 2) + 1;
    uint32_t base = key << 16;
    bool is_run = has_run && (run_flags[c >> 3] >> (c & 7) & 1);
    if (is_run) {
      if (pos + 2 > len) return -1;
      uint32_t nruns = le16(buf + pos);
      pos += 2;
      if (pos + 4ll * nruns > len) return -1;
      for (uint32_t r = 0; r < nruns; r++) {
        uint32_t start = le16(buf + pos), lenm1 = le16(buf + pos + 2);
        pos += 4;
        for (uint32_t v = start; v <= start + lenm1; v++) f(base | v);
      }
    } else if (card > 4096) {
      if (pos + 8192 > len) return -1;
      for (int wi = 0; wi < 1024; wi++) {
        uint64_t x = le64(buf + pos + 8 * wi);
        while (x) { f(base | (uint32_t)(wi * 64 + __builtin_ctzll(x))); x &= x - 1; }
      }
      pos += 8192;
    } else {
      if (pos + 2ll * card > len) return -1;
      for (uint32_t i = 0; i < card; i++) f(base | le16(buf + pos + 2 * i));
      pos += 2ll * card;
    }
    total += card;
  }
  return total;
}

struct ByteSink {
  uint8_t* out; int64_t cap; int64_t pos = 0;
  void u8(uint8_t v) { if (out && pos < cap) out[pos] = v; pos++; }
  void u16(uint16_t v) { u8(v & 0xFF); u8(v >> 8); }
  void u32(uint32_t v) { u16(v & 0xFFFF); u16(v >> 16); }
  void u64(uint64_t v) { u32((uint32_t)v); u32((uint32_t)(v >> 32)); }
  void be_u32(uint32_t v) { u8(v >> 24); u8(v >> 16); u8(v >> 8); u8(v); }
};

// Serialize sorted distinct values.  Container choice follows RoaringBitmap's rules: <=4096 values -> array, else
// bitmap; with run_optimize (RoaringBitmapWriter.writer() default, OnHeapBitmapInvertedIndexCreator.java:41-45) a
// container becomes a run container when that is strictly smaller (2+4*runs < 2*card resp. < 8192).
int64_t roaring_serialize(const uint32_t* v, int64_t n, bool run_optimize, uint8_t* out, int64_t cap) {
  struct C { uint32_t key; int64_t lo, hi; int kind; uint32_t nruns; };  // kind 0 array 1 bitmap 2 run
  std::vector<C> cs;
  for (int64_t i = 0; i < n;) {
    uint32_t key = v[i] >> 16;
    int64_t j = i;
    uint32_t nruns = 0;
    while (j < n && (v[j] >> 16) == key) {
      if (j == i || v[j] != v[j - 1] + 1) nruns++;
      j++;
    }
    int64_t card = j - i;
    int kind = card > 4096 ? 1 : 0;
    if (run_optimize) {
      int64_t cur = kind ? 8192 : 2 * card;
      if (2 + 4ll * nruns < cur) kind = 2;
    }
    cs.push_back({key, i, j, kind, nruns});
    i = j;
  }
  bool has_run = false;
  for (auto& c : cs) has_run |= c.kind == 2;
  ByteSink s{out, cap};
  uint32_t nc = (uint32_t)cs.size();
  if (has_run) {
    s.u32(kCookieRun | ((nc - 1) << 16));
    std::vector<uint8_t> flags((nc + 7) / 8, 0);
    for (uint32_t c = 0; c < nc; c++) if (cs[c].kind == 2) flags[c >> 3] |= 1 << (c & 7);
    for (uint8_t b : flags) s.u8(b);
  } else {
    s.u32(kCookieNoRun);
    s.u32(nc);
  }
  for (auto& c : cs) { s.u16((uint16_t)c.key); s.u16((uint16_t)(c.hi - c.lo - 1)); }
  if (!has_run || (int)nc >= kNoOffsetThreshold) {
    int64_t off = s.pos + 4ll * nc;
    for (auto& c : cs) {
      s.u32((uint32_t)off);
      off += c.kind == 0 ? 2 * (c.hi - c.lo) : c.kind == 1 ? 8192 : 2 + 4ll * c.nruns;
    }
  }
  for (auto& c : cs) {
    if (c.kind == 0) {
      for (int64_t i = c.lo; i < c.hi; i++) s.u16((uint16_t)(v[i] & 0xFFFF));
    } else if (c.kind == 1) {
      uint64_t words[1024];
      memset(words, 0, sizeof words);
      for (int64_t i = c.lo; i < c.hi; i++) { uint32_t x = v[i] & 0xFFFF; words[x >> 6] |= 1ull << (x & 63); }
      for (int wi = 0; wi < 1024; wi++) s.u64(words[wi]);
    } else {
      s.u16((uint16_t)c.nruns);
      for (int64_t i = c.lo; i < c.hi;) {
        int64_t j = i;
        while (j + 1 < c.hi && v[j + 1] == v[j] + 1) j++;
        s.u16((uint16_t)(v[i] & 0xFFFF));
        s.u16((uint16_t)(j - i));
        i = j + 1;
      }
    }
  }
  return s.pos;
}

// ------------------------------------------------------------------------------------------------------------------
// Column accessors
// ------------------------------------------------------------------------------------------------------------------
struct RawChunkHeader {  // seglocal/segment/index/readers/forward/BaseChunkForwardIndexReader.java:60-106
  int version = 0, num_chunks = 0, docs_per_chunk = 0, entry_len = 0, compression = 0;
  int64_t raw_data_start = 0;
  bool ok = false;
};

RawChunkHeader parse_raw_header(const uint8_t* b, int64_t len) {
  RawChunkHeader h;
  if (len < 16) return h;
  h.version = (int)be32(b);
  h.num_chunks = (int)be32(b + 4);
  h.docs_per_chunk = (int)be32(b + 8);
  h.entry_len = (int)be32(b + 12);
  int64_t data_header_start = 16;
  if (h.version > 1) {
    h.compression = (int)be32(b + 20);  // ChunkCompressionType: 0 = PASS_THROUGH
    data_header_start = (int)be32(b + 24);
  } else {
    h.compression = 1;  // v1 is always snappy
  }
  int off_size = h.version <= 2 ? 4 : 8;
  h.raw_data_start = data_header_start + (int64_t)h.num_chunks * off_size;
  h.ok = h.compression == 0;
  return h;
}

// INT / LONG value vs literal by exact numeric value (NumericalFilterOptimizer: a fractional literal equals no integer,
// range bounds become ceil / floor, a literal beyond the column's range makes the predicate constant).  `d` is the
// literal rounded to double, `i` the literal when it is an int64 ((double)i == d); otherwise a fractional `d` is the
// literal and an integral or infinite one lies beyond int64 on its side.
int cmp_integral(int64_t v, const po_literal_t& l) {
  if ((double)l.i == l.d) return v < l.i ? -1 : v > l.i ? 1 : 0;
  if (std::isfinite(l.d) && l.d != std::floor(l.d)) return (double)v < l.d ? -1 : 1;   // |d| < 2^52: rounding v keeps its side
  return l.d > 0 ? -1 : 1;
}

struct Column {
  const po_column_t* c;
  RawChunkHeader raw;
  explicit Column(const po_column_t* col) : c(col) {
    if (!c->has_dictionary) raw = parse_raw_header(c->fwd, c->fwd_len);
  }
  int card() const { return c->cardinality; }
  // Dictionary values (seglocal/segment/index/readers/{Int,Long,Float,Double}Dictionary.java; BE fixed width:
  // seglocal/io/util/FixedByteValueReaderWriter.java:36-54)
  int32_t dict_int(int id) const { return (int32_t)be32(c->dict + 4ll * id); }
  int64_t dict_long(int id) const { return (int64_t)be64(c->dict + 8ll * id); }
  float dict_float(int id) const { uint32_t u = be32(c->dict + 4ll * id); float f; memcpy(&f, &u, 4); return f; }
  double dict_double_raw(int id) const { uint64_t u = be64(c->dict + 8ll * id); double d; memcpy(&d, &u, 8); return d; }
  // Dictionary.getDoubleValue(dictId)
  double dict_as_double(int id) const {
    switch (c->data_type) {
      case PO_INT: return (double)dict_int(id);
      case PO_LONG: return (double)dict_long(id);
      case PO_FLOAT: return (double)dict_float(id);
      case PO_DOUBLE: return dict_double_raw(id);
      default: return std::nan("");
    }
  }
  std::string dict_string(int id) const {  // padded with '\0' (StringDictionary, numBytesPerValue)
    const char* p = (const char*)c->dict + (int64_t)c->dict_entry_bytes * id;
    size_t n = 0;
    while (n < (size_t)c->dict_entry_bytes && p[n] != 0) n++;
    return std::string(p, n);
  }
  // Raw (no dictionary) fixed-byte PASS_THROUGH values
  // (seglocal/segment/index/readers/forward/FixedByteChunkSVForwardIndexReader.java:52-100)
  double raw_as_double(int doc) const {
    const uint8_t* p = c->fwd + raw.raw_data_start;
    switch (c->data_type) {
      case PO_INT: return (double)(int32_t)be32(p + 4ll * doc);
      case PO_LONG: return (double)(int64_t)be64(p + 8ll * doc);
      case PO_FLOAT: { uint32_t u = be32(p + 4ll * doc); float f; memcpy(&f, &u, 4); return (double)f; }
      case PO_DOUBLE: { uint64_t u = be64(p + 8ll * doc); double d; memcpy(&d, &u, 8); return d; }
      default: return std::nan("");
    }
  }
  // identity of a raw value as a group key: the long for INT / LONG, doubleToLongBits of the (widened) value for FLOAT / DOUBLE
  uint64_t raw_value_bits(int doc) const {
    if (c->data_type == PO_INT || c->data_type == PO_LONG) return (uint64_t)raw_as_long(doc);
    const double d = raw_as_double(doc);
    uint64_t u; memcpy(&u, &d, 8);
    return u;
  }
  int64_t raw_as_long(int doc) const {
    const uint8_t* p = c->fwd + raw.raw_data_start;
    return c->data_type == PO_INT ? (int64_t)(int32_t)be32(p + 4ll * doc) : (int64_t)be64(p + 8ll * doc);
  }
  // Sorted index (seglocal/segment/index/readers/sorted/SortedIndexReaderImpl.java): (start,end) inclusive per dictId
  int sorted_start(int id) const { return (int)be32(c->fwd + 8ll * id); }
  int sorted_end(int id) const { return (int)be32(c->fwd + 8ll * id + 4); }
  int sorted_dict_id(int doc) const {  // binary search over the ranges (SortedIndexReaderImpl.getDictId)
    int lo = 0, hi = c->cardinality - 1;
    while (lo < hi) {
      int mid = (lo + hi) >> 1;
      if (sorted_end(mid) < doc) lo = mid + 1; else hi = mid;
    }
    return lo;
  }
  void read_dict_ids(int num_docs, const int32_t* doc_ids, int length, int32_t* out) const {
    if (c->is_sorted) {
      for (int i = 0; i < length; i++) out[i] = sorted_dict_id(doc_ids[i]);
    } else {
      fwd_read_dict_ids(c->fwd, num_docs, c->bits_per_value, doc_ids, length, out);
    }
  }
  int get_dict_id(int doc) const {
    return c->is_sorted ? sorted_dict_id(doc) : bitset_read_one(c->fwd, doc, c->bits_per_value);
  }

  // BaseImmutableDictionary.insertionIndexOf / binarySearch (seglocal/segment/index/readers/BaseImmutableDictionary.java
  // :124-139,245-259): >=0 found, else -(insertion point)-1.
  int insertion_index_of(const po_literal_t& lit) const {
    int lo = 0, hi = c->cardinality - 1;
    while (lo <= hi) {
      int mid = (lo + hi) >> 1;
      int cmp;
      switch (c->data_type) {
        case PO_INT: cmp = cmp_integral(dict_int(mid), lit); break;
        case PO_LONG: cmp = cmp_integral(dict_long(mid), lit); break;
        case PO_FLOAT: { float v = dict_float(mid), t = (float)lit.d; cmp = v < t ? -1 : v > t ? 1 : 0; break; }
        case PO_DOUBLE: { double v = dict_double_raw(mid); cmp = v < lit.d ? -1 : v > lit.d ? 1 : 0; break; }
        default: { int r = dict_string(mid).compare(lit.s ? lit.s : ""); cmp = r < 0 ? -1 : r > 0 ? 1 : 0; }
      }
      if (cmp < 0) lo = mid + 1; else if (cmp > 0) hi = mid - 1; else return mid;
    }
    return -(lo + 1);
  }
  // raw value at `doc` vs a literal in the column's type (the *RawValueBased*PredicateEvaluators): INT / LONG exact,
  // FLOAT as float, DOUBLE as double
  int raw_compare(int doc, const po_literal_t& lit) const {
    switch (c->data_type) {
      case PO_INT: case PO_LONG: return cmp_integral(raw_as_long(doc), lit);
      case PO_FLOAT: { float v = (float)raw_as_double(doc), t = (float)lit.d; return v < t ? -1 : v > t ? 1 : 0; }
      default: { double v = raw_as_double(doc); return v < lit.d ? -1 : v > lit.d ? 1 : 0; }
    }
  }
  // BitmapInvertedIndexReader.getDocIds (seglocal/segment/index/readers/BitmapInvertedIndexReader.java:45-62)
  bool inverted_bitmap(int dict_id, const uint8_t** p, int64_t* len) const {
    int64_t off = be32(c->inv + 4ll * dict_id), end = be32(c->inv + 4ll * (dict_id + 1));
    int64_t first = be32(c->inv);
    int64_t base = 4ll * (c->cardinality + 1);
    *p = c->inv + base + (off - first);
    *len = end - off;
    return true;
  }
};

// ------------------------------------------------------------------------------------------------------------------
// Predicate evaluators (dictionary based) -- core/operator/filter/predicate/
//   RangePredicateEvaluatorFactory.java:119-246 (SortedDictionaryBasedRangePredicateEvaluator)
//   EqualsPredicateEvaluatorFactory / NotEqualsPredicateEvaluatorFactory / InPredicateEvaluatorFactory /
//   NotInPredicateEvaluatorFactory (DictionaryBased* inner classes)
// ------------------------------------------------------------------------------------------------------------------
struct Predicate {
  int type = PO_EQ;
  bool always_true = false, always_false = false;
  bool exclusive = false;      // NEQ / NOT_IN
  bool is_range = false;
  int start = 0, end = 0;      // RANGE: [start, end)
  std::vector<int> ids;        // EQ/IN: matching; NEQ/NOT_IN: NON-matching (sorted)
  std::vector<uint8_t> lut;    // dictId -> match
  int card = 0;
  // raw (no dictionary) numeric predicate
  bool raw = false;
  po_literal_t lo{}, hi{}; bool lo_inc = true, hi_inc = true, lo_unb = true, hi_unb = true;
  std::vector<po_literal_t> raw_values;

  bool apply(int dict_id) const { return is_range ? (start <= dict_id && end > dict_id) : lut[dict_id] != 0; }
  bool apply_raw(const Column& col, int doc) const {
    if (is_range) {
      if (!lo_unb) { int c = col.raw_compare(doc, lo); if (lo_inc ? c < 0 : c <= 0) return false; }
      if (!hi_unb) { int c = col.raw_compare(doc, hi); if (hi_inc ? c > 0 : c >= 0) return false; }
      return true;
    }
    bool in = false;
    for (const po_literal_t& l : raw_values) in |= col.raw_compare(doc, l) == 0;
    return exclusive ? !in : in;
  }
  int num_matching() const {  // getNumMatchingItems (negative for exclusive predicates)
    if (is_range) return std::max(end - start, 0);
    return exclusive ? -(int)ids.size() : (int)ids.size();
  }
  std::vector<int> matching_ids() const {
    std::vector<int> r;
    if (is_range) { for (int i = start; i < end; i++) r.push_back(i); return r; }
    if (!exclusive) return ids;
    for (int i = 0; i < card; i++) if (lut[i]) r.push_back(i);
    return r;
  }
};

Predicate make_predicate(const Column& col, const po_filter_node_t& n, const po_literal_t* lits) {
  Predicate p;
  p.type = n.type;
  p.card = col.card();
  const po_literal_t* v = lits + n.values_offset;
  if (!col.c->has_dictionary) {
    p.raw = true;
    if (n.type == PO_RANGE) {
      p.is_range = true;
      p.lo_unb = n.lower_unbounded; p.hi_unb = n.upper_unbounded;
      p.lo_inc = n.lower_inclusive; p.hi_inc = n.upper_inclusive;
      if (!p.lo_unb) p.lo = v[0];
      if (!p.hi_unb) p.hi = v[1];
    } else {
      p.exclusive = n.type == PO_NEQ || n.type == PO_NOT_IN;
      for (int i = 0; i < n.num_values; i++) p.raw_values.push_back(v[i]);
    }
    return p;
  }
  if (n.type == PO_RANGE) {
    p.is_range = true;
    if (n.lower_unbounded) {
      p.start = 0;
    } else {
      int ii = col.insertion_index_of(v[0]);
      p.start = ii < 0 ? -(ii + 1) : (n.lower_inclusive ? ii : ii + 1);
    }
    if (n.upper_unbounded) {
      p.end = p.card;
    } else {
      int ii = col.insertion_index_of(v[1]);
      p.end = ii < 0 ? -(ii + 1) : (n.upper_inclusive ? ii + 1 : ii);
    }
    int nm = std::max(p.end - p.start, 0);
    if (nm == 0) p.always_false = true; else if (nm == p.card) p.always_true = true;
    return p;
  }
  p.exclusive = n.type == PO_NEQ || n.type == PO_NOT_IN;
  for (int i = 0; i < n.num_values; i++) {
    int id = col.insertion_index_of(v[i]);
    if (id >= 0) p.ids.push_back(id);
  }
  std::sort(p.ids.begin(), p.ids.end());
  p.ids.erase(std::unique(p.ids.begin(), p.ids.end()), p.ids.end());
  p.lut.assign(p.card, p.exclusive ? 1 : 0);
  for (int id : p.ids) p.lut[id] = p.exclusive ? 0 : 1;
  int k = (int)p.ids.size();
  if (!p.exclusive) {
    if (k == 0) p.always_false = true; else if (k == p.card) p.always_true = true;
  } else {
    if (k == 0) p.always_true = true; else if (k == p.card) p.always_false = true;
  }
  return p;
}

// ------------------------------------------------------------------------------------------------------------------
// Doc-id iterators -- core/operator/dociditerators/
// ------------------------------------------------------------------------------------------------------------------
struct DocIdIterator {
  virtual ~DocIdIterator() {}
  virtual int next() = 0;
  virtual int advance(int target) = 0;
  virtual int64_t entries_scanned() const { return 0; }
  virtual int kind() const = 0;  // 0 scan, 1 bitmap, 2 sorted, 3 other
};
using ItPtr = std::unique_ptr<DocIdIterator>;

struct MatchAllIterator : DocIdIterator {  // MatchAllDocIdIterator
  int n, nxt = 0;
  explicit MatchAllIterator(int num_docs) : n(num_docs) {}
  int next() override { return nxt < n ? nxt++ : kEOF; }
  int advance(int t) override { nxt = t; return next(); }
  int kind() const override { return 3; }
};
struct EmptyIterator : DocIdIterator {
  int next() override { return kEOF; }
  int advance(int) override { return kEOF; }
  int kind() const override { return 3; }
};

// SVScanDocIdIterator.java:76-112,115-142
struct ScanIterator : DocIdIterator {
  const Column& col;
  Predicate pred;
  int num_docs;
  int batch[kScanBatch], dict_buf[kScanBatch];
  int first_mismatch = 0, cursor = 0, next_doc = 0;
  int64_t scanned = 0;
  ScanIterator(const Column& c, Predicate p, int n) : col(c), pred(std::move(p)), num_docs(n) {}
  int match_values(int limit, int* doc_ids) {  // DictIdMatcher.matchValues / raw matchers
    int m = 0;
    if (pred.raw) {
      for (int i = 0; i < limit; i++) if (pred.apply_raw(col, doc_ids[i])) doc_ids[m++] = doc_ids[i];
      return m;
    }
    col.read_dict_ids(num_docs, doc_ids, limit, dict_buf);
    for (int i = 0; i < limit; i++) if (pred.apply(dict_buf[i])) doc_ids[m++] = doc_ids[i];
    return m;
  }
  bool does_match(int doc) { return pred.raw ? pred.apply_raw(col, doc) : pred.apply(col.get_dict_id(doc)); }
  int next() override {
    if (cursor >= first_mismatch) {
      int limit, bs = 0;
      do {
        limit = std::min(num_docs - next_doc, kScanBatch);
        if (limit > 0) {
          for (int i = 0; i < limit; i++) batch[i] = next_doc + i;
          bs = match_values(limit, batch);
          next_doc += limit;
          scanned += limit;
        }
      } while (limit > 0 && bs == 0);
      first_mismatch = bs;
      cursor = 0;
      if (first_mismatch == 0) return kEOF;
    }
    return batch[cursor++];
  }
  int advance(int target) override {
    next_doc = target;
    first_mismatch = 0;
    while (next_doc < num_docs) {
      int d = next_doc++;
      scanned++;
      if (does_match(d)) return d;
    }
    return kEOF;
  }
  // applyAnd(bitmap): evaluate the predicate only on the docs of `in`, in batches of 256
  DenseBitmap apply_and(const DenseBitmap& in) {
    DenseBitmap out(in.n);
    int buf[kScanBatch];
    int64_t d = in.next_set(0);
    while (d >= 0) {
      int limit = 0;
      while (d >= 0 && limit < kScanBatch) { buf[limit++] = (int)d; d = in.next_set(d + 1); }
      int m = match_values(limit, buf);
      for (int i = 0; i < m; i++) out.set(buf[i]);
      scanned += limit;
    }
    return out;
  }
  int64_t entries_scanned() const override { return scanned; }
  int kind() const override { return 0; }
  float estimated_cardinality() const {  // getEstimatedCardinality :154-163
    int nm = pred.num_matching();
    nm = nm > 0 ? nm : nm + col.card();
    return (float)col.card() / nm;
  }
};

// BitmapDocIdIterator / RangelessBitmapDocIdIterator
struct BitmapIterator : DocIdIterator {
  std::shared_ptr<DenseBitmap> bm;
  int64_t cur = 0;
  explicit BitmapIterator(std::shared_ptr<DenseBitmap> b) : bm(std::move(b)) {}
  int next() override {
    int64_t r = bm->next_set(cur);
    if (r < 0) { cur = bm->n; return kEOF; }
    cur = r + 1;
    return (int)r;
  }
  int advance(int t) override { cur = t; return next(); }
  int kind() const override { return 1; }
};

// SortedDocIdIterator: list of inclusive doc-id ranges
struct SortedIterator : DocIdIterator {
  std::vector<std::pair<int, int>> ranges;
  size_t ri = 0;
  int nxt;
  explicit SortedIterator(std::vector<std::pair<int, int>> r) : ranges(std::move(r)) { nxt = ranges.empty() ? 0 : ranges[0].first; }
  int next() override {
    while (ri < ranges.size()) {
      if (nxt < ranges[ri].first) nxt = ranges[ri].first;
      if (nxt <= ranges[ri].second) return nxt++;
      ri++;
    }
    return kEOF;
  }
  int advance(int t) override {
    while (ri < ranges.size() && ranges[ri].second < t) ri++;
    if (ri == ranges.size()) return kEOF;
    nxt = std::max(t, ranges[ri].first);
    return next();
  }
  int kind() const override { return 2; }
};

// AndDocIdIterator.java:40-67
struct AndIterator : DocIdIterator {
  std::vector<ItPtr> its;
  int nxt = 0;
  explicit AndIterator(std::vector<ItPtr> v) : its(std::move(v)) {}
  int next() override {
    int max_doc = nxt, max_idx = -1, n = (int)its.size(), idx = 0;
    while (idx < n) {
      if (idx == max_idx) { idx++; continue; }
      int d = its[idx]->advance(max_doc);
      if (d == kEOF) return kEOF;
      if (d == max_doc) { idx++; } else { max_doc = d; max_idx = idx; idx = 0; }
    }
    nxt = max_doc;
    return nxt++;
  }
  int advance(int t) override { nxt = t; return next(); }
  int64_t entries_scanned() const override { int64_t s = 0; for (auto& i : its) s += i->entries_scanned(); return s; }
  int kind() const override { return 3; }
};

// OrDocIdIterator.java:52-110
struct OrIterator : DocIdIterator {
  std::vector<ItPtr> its;   // never shrinks (for stats); `live` indexes the not-exhausted ones
  std::vector<int> live, next_ids;
  int prev = -1;
  explicit OrIterator(std::vector<ItPtr> v) : its(std::move(v)) {
    for (int i = 0; i < (int)its.size(); i++) { live.push_back(i); next_ids.push_back(-1); }
  }
  template <class F>
  int step(F&& fetch, bool by_target, int target) {
    int nd = std::numeric_limits<int>::max();
    bool exhausted = false;
    for (size_t k = 0; k < live.size(); k++) {
      int d = next_ids[k];
      if (by_target ? d < target : d == prev) {
        d = fetch(*its[live[k]]);
        next_ids[k] = d;
        if (d == kEOF) { exhausted = true; continue; }
      }
      nd = std::min(nd, d);
    }
    if (exhausted) {
      size_t w = 0;
      for (size_t k = 0; k < live.size(); k++) if (next_ids[k] != kEOF) { live[w] = live[k]; next_ids[w] = next_ids[k]; w++; }
      live.resize(w); next_ids.resize(w);
    }
    if (nd != std::numeric_limits<int>::max()) { prev = nd; return nd; }
    return kEOF;
  }
  int next() override { return step([](DocIdIterator& i) { return i.next(); }, false, 0); }
  int advance(int t) override { return step([t](DocIdIterator& i) { return i.advance(t); }, true, t); }
  int64_t entries_scanned() const override { int64_t s = 0; for (auto& i : its) s += i->entries_scanned(); return s; }
  int kind() const override { return 3; }
};

// NotDocIdIterator.java:28-75
struct NotIterator : DocIdIterator {
  ItPtr child;
  int num_docs, nxt = 0, next_non_matching;
  NotIterator(ItPtr c, int n) : child(std::move(c)), num_docs(n) {
    int d = child->next();
    next_non_matching = d == kEOF ? n : d;
  }
  int next() override {
    if (nxt >= num_docs) return kEOF;
    while (nxt == next_non_matching) {
      nxt++;
      int d = child->next();
      next_non_matching = d == kEOF ? num_docs : d;
    }
    if (nxt >= num_docs) return kEOF;
    return nxt++;
  }
  int advance(int t) override {
    nxt = t;
    if (t > next_non_matching) {
      int d = child->advance(t);
      next_non_matching = d == kEOF ? num_docs : d;
    }
    return next();
  }
  int64_t entries_scanned() const override { return child->entries_scanned(); }
  int kind() const override { return 3; }
};

// ------------------------------------------------------------------------------------------------------------------
// Filter operators -> BlockDocIdSet -- core/operator/filter/, core/operator/docidsets/
// A "DocIdSet" here is a factory producing the iterator (BlockDocIdSet.iterator()) exactly once.
// ------------------------------------------------------------------------------------------------------------------
struct FilterOp {
  enum Kind { EMPTY, MATCH_ALL, SCAN, BITMAP, SORTED, AND, OR, NOT, DOCIDS } kind = EMPTY;
  const int32_t* doc_ids = nullptr;  // DOCIDS: BitmapBasedFilterOperator over an explicit doc-id list
  int64_t num_doc_ids = 0;
  const Column* col = nullptr;
  Predicate pred;
  std::vector<std::unique_ptr<FilterOp>> children;
  int num_docs = 0;

  int priority() const {  // FilterOperatorUtils.java:205-251 (PrioritizedFilterOperator constants)
    switch (kind) {
      case SORTED: return 0;      // HIGH_PRIORITY
      case BITMAP: case DOCIDS: return 100;    // MEDIUM_PRIORITY
      case AND: return 300;       // AND_PRIORITY
      case OR: return 400;        // OR_PRIORITY
      case NOT: return children[0]->priority();
      case SCAN: return 500;      // SCAN_PRIORITY (SV columns keep the base priority :252-262)
      default: return 600;
    }
  }
};
using OpPtr = std::unique_ptr<FilterOp>;

struct Segment {
  const po_segment_t* s;
  std::vector<Column> cols;
  explicit Segment(const po_segment_t* seg) : s(seg) {
    for (int i = 0; i < seg->num_columns; i++) cols.emplace_back(&seg->columns[i]);
  }
  int num_docs() const { return s->num_docs; }
};

// FilterOperatorUtils.getLeafFilterOperator :74-133
OpPtr leaf_operator(const Segment& seg, const po_filter_node_t& n, const po_literal_t* lits) {
  const Column& col = seg.cols[n.column];
  auto op = std::make_unique<FilterOp>();
  op->num_docs = seg.num_docs();
  op->col = &col;
  op->pred = make_predicate(col, n, lits);
  if (op->pred.always_false) { op->kind = FilterOp::EMPTY; return op; }
  if (op->pred.always_true) { op->kind = FilterOp::MATCH_ALL; return op; }
  bool sorted = col.c->is_sorted && col.c->has_dictionary;
  if (n.type == PO_RANGE) {
    op->kind = sorted ? FilterOp::SORTED : FilterOp::SCAN;  // (no range index in scope)
  } else {
    op->kind = sorted ? FilterOp::SORTED : (col.c->inv && col.c->has_dictionary) ? FilterOp::BITMAP : FilterOp::SCAN;
  }
  return op;
}

OpPtr make_empty(int n) { auto o = std::make_unique<FilterOp>(); o->kind = FilterOp::EMPTY; o->num_docs = n; return o; }
OpPtr make_match_all(int n) { auto o = std::make_unique<FilterOp>(); o->kind = FilterOp::MATCH_ALL; o->num_docs = n; return o; }

// FilterPlanNode.constructPhysicalOperator (core/plan/FilterPlanNode.java:195-320) + FilterOperatorUtils and/or/not
OpPtr build_filter_nodes(const Segment& seg, const po_query_t& q, const po_filter_node_t* nodes, int num_nodes) {
  int nd = seg.num_docs();
  if (num_nodes == 0) return make_match_all(nd);
  std::vector<OpPtr> stack;
  for (int i = 0; i < num_nodes; i++) {
    const po_filter_node_t& n = nodes[i];
    if (n.type == PO_DOCIDS) {
      auto o = std::make_unique<FilterOp>();
      o->kind = FilterOp::DOCIDS; o->num_docs = nd; o->doc_ids = q.doc_ids; o->num_doc_ids = q.num_doc_ids;
      stack.push_back(std::move(o));
      continue;
    }
    if (n.type >= PO_EQ) { stack.push_back(leaf_operator(seg, n, q.literals)); continue; }
    if (n.type == PO_NOT) {
      OpPtr c = std::move(stack.back()); stack.pop_back();
      if (c->kind == FilterOp::MATCH_ALL) stack.push_back(make_empty(nd));
      else if (c->kind == FilterOp::EMPTY) stack.push_back(make_match_all(nd));
      else { auto o = std::make_unique<FilterOp>(); o->kind = FilterOp::NOT; o->num_docs = nd; o->children.push_back(std::move(c)); stack.push_back(std::move(o)); }
      continue;
    }
    std::vector<OpPtr> kids(n.num_children);
    for (int k = n.num_children - 1; k >= 0; k--) { kids[k] = std::move(stack.back()); stack.pop_back(); }
    bool is_and = n.type == PO_AND;
    std::vector<OpPtr> kept;
    bool shortcut = false;
    for (auto& k : kids) {
      if (is_and ? k->kind == FilterOp::EMPTY : k->kind == FilterOp::MATCH_ALL) { shortcut = true; break; }
      if (is_and ? k->kind != FilterOp::MATCH_ALL : k->kind != FilterOp::EMPTY) kept.push_back(std::move(k));
    }
    if (shortcut) { stack.push_back(is_and ? make_empty(nd) : make_match_all(nd)); continue; }
    if (kept.empty()) { stack.push_back(is_and ? make_match_all(nd) : make_empty(nd)); continue; }
    if (kept.size() == 1) { stack.push_back(std::move(kept[0])); continue; }
    if (is_and) std::stable_sort(kept.begin(), kept.end(), [](const OpPtr& a, const OpPtr& b) { return a->priority() < b->priority(); });
    auto o = std::make_unique<FilterOp>();
    o->kind = is_and ? FilterOp::AND : FilterOp::OR;
    o->num_docs = nd;
    o->children = std::move(kept);
    stack.push_back(std::move(o));
  }
  return std::move(stack.back());
}

OpPtr build_filter(const Segment& seg, const po_query_t& q) { return build_filter_nodes(seg, q, q.filter, q.num_filter_nodes); }

struct ExecCtx {
  bool and_scan_reordering = false;
  std::vector<ScanIterator*> scans;  // every scan iterator created (for numEntriesScannedInFilter)
};

std::shared_ptr<DenseBitmap> bitmap_from_inverted(const FilterOp& op) {
  // InvertedIndexFilterOperator.getNextBlockWithoutNullHandling :60-96
  const Column& col = *op.col;
  auto bm = std::make_shared<DenseBitmap>(op.num_docs);
  const std::vector<int>& ids = op.pred.ids;  // matching (EQ/IN) or non-matching (NEQ/NOT_IN)
  for (int id : ids) {
    const uint8_t* p; int64_t len;
    col.inverted_bitmap(id, &p, &len);
    roaring_for_each(p, len, [&](uint32_t d) { bm->set(d); });
  }
  if (op.pred.exclusive) bm->flip_all();
  return bm;
}

std::vector<std::pair<int, int>> sorted_ranges(const FilterOp& op) {
  // SortedIndexBasedFilterOperator.getNextBlockWithoutNullHandling :60-135
  const Column& col = *op.col;
  std::vector<std::pair<int, int>> r;
  if (op.pred.is_range) {
    r.push_back({col.sorted_start(op.pred.start), col.sorted_end(op.pred.end - 1)});
    return r;
  }
  const std::vector<int>& ids = op.pred.ids;
  std::pair<int, int> last{col.sorted_start(ids[0]), col.sorted_end(ids[0])};
  for (size_t i = 1; i < ids.size(); i++) {
    std::pair<int, int> cur{col.sorted_start(ids[i]), col.sorted_end(ids[i])};
    if (cur.first == last.second + 1) last.second = cur.second; else { r.push_back(last); last = cur; }
  }
  r.push_back(last);
  if (op.pred.exclusive) {
    std::vector<std::pair<int, int>> inv;
    if (r[0].first > 0) inv.push_back({0, r[0].first - 1});
    for (size_t i = 0; i + 1 < r.size(); i++) inv.push_back({r[i].second + 1, r[i + 1].first - 1});
    if (r.back().second < op.num_docs - 1) inv.push_back({r.back().second + 1, op.num_docs - 1});
    r = inv;
  }
  return r;
}

ItPtr make_iterator(const FilterOp& op, ExecCtx& ctx);

// AndDocIdSet.iterator() (core/operator/docidsets/AndDocIdSet.java:72-186)
ItPtr and_iterator(const FilterOp& op, ExecCtx& ctx) {
  std::vector<ItPtr> all;
  for (auto& c : op.children) all.push_back(make_iterator(*c, ctx));
  std::vector<size_t> sorted_idx, bitmap_idx, scan_idx, rest_idx;
  for (size_t i = 0; i < all.size(); i++) {
    switch (all[i]->kind()) {
      case 2: sorted_idx.push_back(i); break;
      case 1: bitmap_idx.push_back(i); break;
      case 0: scan_idx.push_back(i); break;
      default: rest_idx.push_back(i);
    }
  }
  auto bm_of = [&](size_t i) { return static_cast<BitmapIterator*>(all[i].get())->bm; };
  std::stable_sort(bitmap_idx.begin(), bitmap_idx.end(), [&](size_t a, size_t b) { return bm_of(a)->cardinality() < bm_of(b)->cardinality(); });
  if (ctx.and_scan_reordering) {
    std::stable_sort(scan_idx.begin(), scan_idx.end(), [&](size_t a, size_t b) {
      return -static_cast<ScanIterator*>(all[a].get())->estimated_cardinality() < -static_cast<ScanIterator*>(all[b].get())->estimated_cardinality();
    });
  }
  size_t n_index = sorted_idx.size() + bitmap_idx.size();
  if ((n_index > 0 && !scan_idx.empty()) || n_index > 1) {
    std::shared_ptr<DenseBitmap> docs;
    if (!sorted_idx.empty()) {
      docs = std::make_shared<DenseBitmap>(op.num_docs);
      // intersect the sorted range sets (SortedRangeIntersection) by AND-ing dense range bitmaps
      bool first = true;
      for (size_t i : sorted_idx) {
        DenseBitmap r(op.num_docs);
        for (auto& pr : static_cast<SortedIterator*>(all[i].get())->ranges) r.set_range(pr.first, pr.second + 1ll);
        if (first) { *docs = r; first = false; } else docs->and_with(r);
      }
      for (size_t i : bitmap_idx) docs->and_with(*bm_of(i));
    } else {
      docs = std::make_shared<DenseBitmap>(*bm_of(bitmap_idx[0]));
      for (size_t k = 1; k < bitmap_idx.size(); k++) docs->and_with(*bm_of(bitmap_idx[k]));
    }
    for (size_t i : scan_idx) docs = std::make_shared<DenseBitmap>(static_cast<ScanIterator*>(all[i].get())->apply_and(*docs));
    ItPtr merged = std::make_unique<BitmapIterator>(docs);
    if (rest_idx.empty()) {
      // keep the scan iterators alive for stats: they are registered in ctx.scans and owned below
      struct Holder : BitmapIterator { std::vector<ItPtr> keep; using BitmapIterator::BitmapIterator; };
      auto h = std::make_unique<Holder>(docs);
      for (auto& a : all) h->keep.push_back(std::move(a));
      return h;
    }
    std::vector<ItPtr> its;
    its.push_back(std::move(merged));
    for (size_t i : rest_idx) its.push_back(std::move(all[i]));
    struct Holder : AndIterator { std::vector<ItPtr> keep; using AndIterator::AndIterator; };
    auto h = std::make_unique<Holder>(std::move(its));
    for (auto& a : all) if (a) h->keep.push_back(std::move(a));
    return h;
  }
  return std::make_unique<AndIterator>(std::move(all));
}

// OrDocIdSet.iterator() (core/operator/docidsets/OrDocIdSet.java:62-130)
ItPtr or_iterator(const FilterOp& op, ExecCtx& ctx) {
  std::vector<ItPtr> all;
  for (auto& c : op.children) all.push_back(make_iterator(*c, ctx));
  std::vector<size_t> index_idx, rest_idx;
  for (size_t i = 0; i < all.size(); i++) (all[i]->kind() == 1 || all[i]->kind() == 2 ? index_idx : rest_idx).push_back(i);
  if (index_idx.size() > 1) {
    auto docs = std::make_shared<DenseBitmap>(op.num_docs);
    for (size_t i : index_idx) {
      if (all[i]->kind() == 2) {
        for (auto& pr : static_cast<SortedIterator*>(all[i].get())->ranges) docs->set_range(pr.first, pr.second + 1ll);
      } else {
        docs->or_with(*static_cast<BitmapIterator*>(all[i].get())->bm);
      }
    }
    if (rest_idx.empty()) return std::make_unique<BitmapIterator>(docs);
    std::vector<ItPtr> its;
    its.push_back(std::make_unique<BitmapIterator>(docs));
    for (size_t i : rest_idx) its.push_back(std::move(all[i]));
    return std::make_unique<OrIterator>(std::move(its));
  }
  return std::make_unique<OrIterator>(std::move(all));
}

ItPtr make_iterator(const FilterOp& op, ExecCtx& ctx) {
  switch (op.kind) {
    case FilterOp::EMPTY: return std::make_unique<EmptyIterator>();
    case FilterOp::MATCH_ALL: return std::make_unique<MatchAllIterator>(op.num_docs);
    case FilterOp::SCAN: {
      auto it = std::make_unique<ScanIterator>(*op.col, op.pred, op.num_docs);
      ctx.scans.push_back(it.get());
      return it;
    }
    case FilterOp::BITMAP: return std::make_unique<BitmapIterator>(bitmap_from_inverted(op));
    case FilterOp::DOCIDS: {
      auto bm = std::make_shared<DenseBitmap>(op.num_docs);
      for (int64_t i = 0; i < op.num_doc_ids; i++) bm->set((uint32_t)op.doc_ids[i]);
      return std::make_unique<BitmapIterator>(bm);
    }
    case FilterOp::SORTED: return std::make_unique<SortedIterator>(sorted_ranges(op));
    case FilterOp::AND: return and_iterator(op, ctx);
    case FilterOp::OR: return or_iterator(op, ctx);
    case FilterOp::NOT: return std::make_unique<NotIterator>(make_iterator(*op.children[0], ctx), op.num_docs);
  }
  return nullptr;
}

// ------------------------------------------------------------------------------------------------------------------
// Group keys -- core/query/aggregation/groupby/DictionaryBasedGroupKeyGenerator.java
// ------------------------------------------------------------------------------------------------------------------
struct GroupKeyGenerator {
  int regime = PO_REGIME_ARRAY;
  std::vector<int> cards;
  int k = 0;
  int upper_bound = 0;     // _globalGroupIdUpperBound
  int num_groups_limit = 0;
  // ARRAY: flags over raw key space
  std::vector<uint8_t> flags;
  int num_keys = 0;
  // INT_MAP / LONG_MAP: raw key -> group id in first-seen order (IntGroupIdMap.getGroupId :1022-1047 returns
  // INVALID_ID = -1 once size >= limit); ARRAY_MAP: the dictId tuple itself
  std::unordered_map<int64_t, int> map;
  std::vector<int64_t> keys_in_order;
  std::map<std::vector<int>, int> array_map;
  std::vector<std::vector<int>> array_keys_in_order;

  void init(const std::vector<int>& cardinalities, int groups_limit, int array_threshold) {
    cards = cardinalities;
    k = (int)cards.size();
    num_groups_limit = groups_limit;
    int64_t product = 1;
    bool overflow = false;
    for (int c : cards) {
      if (!overflow) {
        if (product > std::numeric_limits<int64_t>::max() / c) overflow = true; else product *= c;
      }
    }
    if (overflow) {
      regime = PO_REGIME_ARRAY_MAP;
      upper_bound = groups_limit;
    } else if (product > std::numeric_limits<int32_t>::max()) {
      regime = PO_REGIME_LONG_MAP;
      upper_bound = groups_limit;
    } else {
      upper_bound = (int)std::min<int64_t>(product, groups_limit);
      if (product > array_threshold) regime = PO_REGIME_INT_MAP; else { regime = PO_REGIME_ARRAY; flags.assign(upper_bound, 0); }
    }
  }
  // generateKeysForBlock: dict_ids[j][i] -> out[i]
  void generate(int n, const std::vector<std::vector<int>>& dict_ids, int* out) {
    if (regime == PO_REGIME_ARRAY_MAP) {
      std::vector<int> key(k);
      for (int i = 0; i < n; i++) {
        for (int j = 0; j < k; j++) key[j] = dict_ids[j][i];
        auto it = array_map.find(key);
        if (it != array_map.end()) { out[i] = it->second; continue; }
        if ((int)array_map.size() < upper_bound) {
          int id = (int)array_map.size();
          array_map.emplace(key, id);
          array_keys_in_order.push_back(key);
          out[i] = id;
        } else {
          out[i] = -1;
        }
      }
      return;
    }
    for (int i = 0; i < n; i++) {
      int64_t raw = 0;
      for (int j = k - 1; j >= 0; j--) raw = raw * cards[j] + dict_ids[j][i];  // column 0 least significant :311-346
      if (regime == PO_REGIME_ARRAY) {
        out[i] = (int)raw;
        if (!flags[raw]) { flags[raw] = 1; num_keys++; }
      } else {
        auto it = map.find(raw);
        if (it != map.end()) { out[i] = it->second; continue; }
        if ((int)map.size() < upper_bound) {
          int id = (int)map.size();
          map.emplace(raw, id);
          keys_in_order.push_back(raw);
          out[i] = id;
        } else {
          out[i] = -1;  // GroupKeyGenerator.INVALID_ID
        }
      }
    }
  }
  // ---- NoDictionarySingleColumnGroupKeyGenerator.java:60-147,  NoDictionaryMultiColumnGroupKeyGenerator.java ----
  // Chosen by DefaultGroupByExecutor.java:87-117 as soon as ONE group-by expression has no dictionary.  Raw columns get an
  // on-the-fly dictionary (value -> id in first-seen order, ValueToIdMap), dictionary columns keep their dictIds; the id
  // tuple maps to a group id in first-seen order, INVALID_ID once numGroupsLimit groups exist.  (With a single column the
  // value itself is the map key -- the same first-seen numbering.)  Group keys of raw columns are VALUES in the result.
  std::vector<uint8_t> col_raw;
  std::vector<std::unordered_map<uint64_t, int>> otf;   // per raw column: value bits -> on-the-fly id
  std::vector<std::vector<uint64_t>> otf_values;        // per raw column: value bits in id order
  void init_no_dictionary(const std::vector<uint8_t>& raw_flags, int groups_limit) {
    col_raw = raw_flags;
    k = (int)raw_flags.size();
    cards.assign(k, 0);
    regime = PO_REGIME_NO_DICT;
    num_groups_limit = groups_limit;
    upper_bound = groups_limit;
    otf.assign(k, {});
    otf_values.assign(k, {});
  }
  // ids[j][i]: dictId (dictionary column) ; bits[j][i]: value bits (raw column)
  void generate_no_dictionary(int n, const std::vector<std::vector<int>>& ids, const std::vector<std::vector<uint64_t>>& bits, int* out) {
    std::vector<int> key(k);
    for (int i = 0; i < n; i++) {
      for (int j = 0; j < k; j++) {
        if (!col_raw[j]) { key[j] = ids[j][i]; continue; }
        auto f = otf[j].find(bits[j][i]);
        if (f != otf[j].end()) key[j] = f->second;
        else { key[j] = (int)otf_values[j].size(); otf[j].emplace(bits[j][i], key[j]); otf_values[j].push_back(bits[j][i]); }
      }
      auto it = array_map.find(key);
      if (it != array_map.end()) { out[i] = it->second; continue; }
      if ((int)array_map.size() < upper_bound) {
        int id = (int)array_map.size();
        array_map.emplace(key, id);
        array_keys_in_order.push_back(key);
        out[i] = id;
      } else {
        out[i] = -1;
      }
    }
  }
  int current_upper_bound() const {  // getCurrentGroupKeyUpperBound
    if (regime == PO_REGIME_NO_DICT) return (int)array_map.size();
    if (regime == PO_REGIME_ARRAY) return upper_bound;
    if (regime == PO_REGIME_ARRAY_MAP) return (int)array_map.size();
    return (int)map.size();
  }
  int num_keys_total() const {
    if (regime == PO_REGIME_ARRAY) return num_keys;
    if (regime == PO_REGIME_ARRAY_MAP || regime == PO_REGIME_NO_DICT) return (int)array_map.size();
    return (int)map.size();
  }
};

}  // namespace

// ------------------------------------------------------------------------------------------------------------------
// Result + executor
// ------------------------------------------------------------------------------------------------------------------
struct po_result {
  std::string error;
  int num_groups = -1;
  int regime = PO_REGIME_NONE;
  bool limit_reached = false;
  int64_t stats[4] = {0, 0, 0, 0};
  int num_group_by = 0;
  std::vector<int32_t> keys;                       // [G x k]: dictIds; for raw group-by columns ids of raw_key_bits[j]
  std::vector<std::vector<uint64_t>> raw_key_bits; // per group-by column: on-the-fly dictionary (empty for dictionary columns)
  std::vector<int> raw_key_type;                   // per group-by column: PO_* stored type of a raw column, else -1
  std::vector<std::vector<uint64_t>> raw_distinct_bits;  // per aggregation: on-the-fly value numbering of a raw DISTINCTCOUNT
  std::vector<int> raw_distinct_type;
  std::vector<std::vector<double>> dbl;            // per agg: [G]
  std::vector<std::vector<int64_t>> lng;           // per agg: [G]
  std::vector<std::vector<std::vector<int32_t>>> distinct;  // per agg: per group: sorted dictIds
};

namespace {

struct AggState {
  po_agg_t spec;
  const Column* col = nullptr;
  // holders indexed by group id (aggregation only: index 0)
  std::vector<double> dbl;    // SUM / MIN / MAX / AVG.sum / COUNT (double holder, CountAggregationFunction.java:112-116)
  std::vector<int64_t> cnt;   // AVG.count
  std::vector<std::vector<uint8_t>> bits;  // DISTINCTCOUNT: dictId bitset per group (RoaringBitmap of dictIds)
  // DISTINCTCOUNT over a raw column: value sets (DistinctCountAggregationFunction keeps an IntOpenHashSet / LongOpenHashSet /
  // FloatOpenHashSet / DoubleOpenHashSet of VALUES when there is no dictionary, BaseDistinctAggregateAggregationFunction
  // .java:157-200).  Values are numbered in first-seen order (raw_values) and the per-group sets hold those numbers.
  std::unordered_map<uint64_t, int> raw_ids;
  std::vector<uint64_t> raw_values;
  std::vector<std::vector<uint8_t>> raw_bits;  // per group: bitset over raw value numbers
  double def() const { return spec.function == PO_MIN ? INFINITY : spec.function == PO_MAX ? -INFINITY : 0.0; }
  void ensure(int n) {
    if ((int)dbl.size() < n) { dbl.resize(n, def()); cnt.resize(n, 0); }
    if (spec.function == PO_DISTINCTCOUNT && (int)bits.size() < n) { bits.resize(n); raw_bits.resize(n); }
  }
};

void run_query(const Segment& seg, const po_query_t& q, po_result& res, std::vector<int32_t>* doc_ids_out,
               int64_t doc_ids_cap) {
  const int num_docs = seg.num_docs();
  const int nagg = q.num_aggs, k = q.num_group_by;

  // ---- aggregation infos: AggregationFunctionUtils.buildFilteredAggregationInfos (:312-403).  Without FILTER clauses: one
  // info = (main filter, all functions).  With them: one info per distinct FILTER, its filter = main AND sub
  // (CombinedFilterOperator; sub alone when the main filter matches everything or the sub filter matches nothing; a sub
  // filter that matches everything makes its functions non-filtered), then the main info with the non-filtered functions --
  // for GROUP BY queries even when that list is empty, so that every group of the main filter exists (:388-400).
  struct Info { OpPtr filter; std::vector<int> aggs; };
  std::vector<Info> infos;
  bool any_filtered = false;
  for (int a = 0; a < nagg && q.agg_filter_count; a++) any_filtered |= q.agg_filter_count[a] > 0;
  {
    OpPtr main_op = build_filter(seg, q);
    if (!any_filtered || main_op->kind == FilterOp::EMPTY) {
      Info one; one.filter = std::move(main_op);
      for (int a = 0; a < nagg; a++) one.aggs.push_back(a);
      infos.push_back(std::move(one));
    } else {
      std::vector<int> non_filtered;
      std::vector<std::pair<int, int>> seen;  // (start, count) of distinct FILTER trees, first-appearance order
      for (int a = 0; a < nagg; a++) {
        if (q.agg_filter_count[a] <= 0) { non_filtered.push_back(a); continue; }
        const std::pair<int, int> key(q.agg_filter_start[a], q.agg_filter_count[a]);
        size_t at = std::find(seen.begin(), seen.end(), key) - seen.begin();
        if (at == seen.size()) {
          seen.push_back(key);
          OpPtr sub = build_filter_nodes(seg, q, q.agg_filter_nodes + key.first, key.second);
          Info inf;
          if (sub->kind == FilterOp::MATCH_ALL && main_op->kind != FilterOp::MATCH_ALL) inf.filter = nullptr;  // == main: non-filtered
          else if (main_op->kind == FilterOp::MATCH_ALL || sub->kind == FilterOp::EMPTY) inf.filter = std::move(sub);
          else {
            auto o = std::make_unique<FilterOp>();
            o->kind = FilterOp::AND; o->num_docs = num_docs;
            o->children.push_back(build_filter(seg, q));
            o->children.push_back(std::move(sub));
            inf.filter = std::move(o);
          }
          infos.push_back(std::move(inf));
        }
        infos[at].aggs.push_back(a);
      }
      std::vector<Info> kept;
      for (auto& inf : infos) {
        if (!inf.filter) non_filtered.insert(non_filtered.end(), inf.aggs.begin(), inf.aggs.end());
        else kept.push_back(std::move(inf));
      }
      infos = std::move(kept);
      if (!non_filtered.empty() || k > 0) {
        Info m; m.filter = std::move(main_op); m.aggs = non_filtered;
        infos.push_back(std::move(m));
      }
    }
  }

  std::vector<AggState> aggs(nagg);
  for (int a = 0; a < nagg; a++) {
    aggs[a].spec = q.aggs[a];
    if (q.aggs[a].function != PO_COUNT) aggs[a].col = &seg.cols[q.aggs[a].column];
  }

  GroupKeyGenerator gkg;
  if (k > 0) {
    std::vector<int> cards;
    std::vector<uint8_t> raw_flags;
    bool any_raw = false;
    for (int j = 0; j < k; j++) {
      const Column& c = seg.cols[q.group_by_columns[j]];
      raw_flags.push_back(c.c->has_dictionary ? 0 : 1);
      any_raw |= !c.c->has_dictionary;
      if (!c.c->has_dictionary && (!c.raw.ok || c.c->data_type == PO_STRING)) { res.error = "group-by on this raw column is not supported by the oracle"; return; }
      cards.push_back(c.card());
    }
    if (any_raw) gkg.init_no_dictionary(raw_flags, q.num_groups_limit);
    else gkg.init(cards, q.num_groups_limit, q.max_initial_result_holder_capacity);
    res.regime = gkg.regime;
  }
  std::vector<std::vector<uint64_t>> gb_raw_bits(k);

  std::vector<int> doc_ids(kMaxDocPerCall), group_keys(kMaxDocPerCall);
  std::vector<std::vector<int>> gb_dict_ids(k, std::vector<int>(kMaxDocPerCall));
  std::map<int, std::vector<int>> col_dict_ids;   // DataBlockCache: dictIds per projected dict column per block
  int64_t total_docs_scanned = 0, total_in_filter = 0, total_post_filter = 0;

  for (int a = 0; a < nagg; a++) aggs[a].ensure(1);

  // FilteredGroupByOperator.getNextBlock :113-160 / FilteredAggregationOperator: the infos run one after the other and
  // SHARE the group key generator; statistics add up.  (One info = GroupByOperator :101-140 / AggregationOperator :64-80.)
  for (Info& info : infos) {
  ExecCtx ctx;
  ctx.and_scan_reordering = q.and_scan_reordering != 0;
  ItPtr it = make_iterator(*info.filter, ctx);
  std::vector<int> projected;  // distinct columns this info projects (its aggregation arguments + group-by)
  auto add_projected = [&](int c) { if (c >= 0 && std::find(projected.begin(), projected.end(), c) == projected.end()) projected.push_back(c); };
  for (int a : info.aggs) if (q.aggs[a].function != PO_COUNT) add_projected(q.aggs[a].column);
  for (int j = 0; j < k; j++) add_projected(q.group_by_columns[j]);
  int64_t docs_scanned = 0;
  while (true) {
    // DocIdSetOperator.getNextBlock :59-86
    int n = 0;
    while (n < kMaxDocPerCall) {
      int d = it->next();
      if (d == kEOF) break;
      doc_ids[n++] = d;
    }
    if (n == 0) break;
    docs_scanned += n;
    if (doc_ids_out) {
      for (int i = 0; i < n && (int64_t)doc_ids_out->size() < doc_ids_cap; i++) doc_ids_out->push_back(doc_ids[i]);
    }
    if (nagg == 0 && k == 0) continue;
    col_dict_ids.clear();
    auto dict_ids_of = [&](int cidx) -> const std::vector<int>& {
      auto f = col_dict_ids.find(cidx);
      if (f != col_dict_ids.end()) return f->second;
      std::vector<int>& v = col_dict_ids[cidx];
      v.resize(n);
      seg.cols[cidx].read_dict_ids(num_docs, doc_ids.data(), n, v.data());
      return v;
    };
    if (k > 0) {
      for (int j = 0; j < k; j++) {
        const Column& gc = seg.cols[q.group_by_columns[j]];
        if (!gc.c->has_dictionary) {  // values of the block (ProjectionBlockValSet.get{Int,Long,Float,Double}ValuesSV)
          gb_raw_bits[j].resize(n);
          for (int i = 0; i < n; i++) gb_raw_bits[j][i] = gc.raw_value_bits(doc_ids[i]);
          continue;
        }
        const std::vector<int>& v = dict_ids_of(q.group_by_columns[j]);
        std::copy(v.begin(), v.begin() + n, gb_dict_ids[j].begin());
      }
      if (gkg.regime == PO_REGIME_NO_DICT) gkg.generate_no_dictionary(n, gb_dict_ids, gb_raw_bits, group_keys.data());
      else gkg.generate(n, gb_dict_ids, group_keys.data());
      int cap = gkg.current_upper_bound();
      for (auto& a : aggs) a.ensure(cap);
    }
    for (int ai : info.aggs) {
      AggState& a = aggs[ai];
      const int fn = a.spec.function;
      if (fn == PO_COUNT) {  // CountAggregationFunction.java:84-143
        if (k == 0) a.dbl[0] += n;
        else for (int i = 0; i < n; i++) { int g = group_keys[i]; if (g >= 0) a.dbl[g] += 1; }
        continue;
      }
      const Column& col = *a.col;
      const bool dict = col.c->has_dictionary;
      const std::vector<int>* ids = dict ? &dict_ids_of(a.spec.column) : nullptr;
      auto value_at = [&](int i) -> double { return dict ? col.dict_as_double((*ids)[i]) : col.raw_as_double(doc_ids[i]); };
      if (fn == PO_DISTINCTCOUNT && !dict) {  // value set of a raw column
        if (!col.raw.ok || col.c->data_type == PO_STRING) { res.error = "DISTINCTCOUNT on this raw column is not supported by the oracle"; return; }
        for (int i = 0; i < n; i++) {
          int g = k == 0 ? 0 : group_keys[i];
          if (g < 0) continue;
          const uint64_t vb = col.raw_value_bits(doc_ids[i]);
          auto f = a.raw_ids.find(vb);
          int id;
          if (f != a.raw_ids.end()) id = f->second;
          else { id = (int)a.raw_values.size(); a.raw_ids.emplace(vb, id); a.raw_values.push_back(vb); }
          auto& b = a.raw_bits[g];
          if ((int)b.size() <= id) b.resize(id + 1, 0);
          b[id] = 1;
        }
        continue;
      }
      if (fn == PO_DISTINCTCOUNT) {  // BaseDistinctAggregateAggregationFunction.java:144-155,306-321
        for (int i = 0; i < n; i++) {
          int g = k == 0 ? 0 : group_keys[i];
          if (g < 0) continue;
          auto& b = a.bits[g];
          if (b.empty()) b.assign(col.card(), 0);
          b[(*ids)[i]] = 1;
        }
        continue;
      }
      if (k == 0) {
        if (fn == PO_SUM || fn == PO_AVG) {  // SumAggregationFunction.java:69-145 (per-block innerSum), Avg :63-103
          double inner = 0;
          for (int i = 0; i < n; i++) inner += value_at(i);
          a.dbl[0] += inner;
          a.cnt[0] += n;
        } else if (fn == PO_MIN) {  // MinAggregationFunction (typed per-block min, then Math.min with holder)
          double m = value_at(0);
          for (int i = 1; i < n; i++) m = std::min(m, value_at(i));
          a.dbl[0] = std::min(a.dbl[0], m);
        } else {
          double m = value_at(0);
          for (int i = 1; i < n; i++) m = std::max(m, value_at(i));
          a.dbl[0] = std::max(a.dbl[0], m);
        }
      } else {
        for (int i = 0; i < n; i++) {
          int g = group_keys[i];
          if (g < 0) continue;  // DoubleGroupByResultHolder ignores INVALID_ID
          double v = value_at(i);
          if (fn == PO_SUM) a.dbl[g] += v;                       // :160-178
          else if (fn == PO_AVG) { a.dbl[g] += v; a.cnt[g]++; }  // AvgAggregationFunction.java:106-127
          else if (fn == PO_MIN) { if (v < a.dbl[g]) a.dbl[g] = v; }  // MinAggregationFunction group-by (strict <)
          else { if (v > a.dbl[g]) a.dbl[g] = v; }                    // MaxAggregationFunction.java:163-187
        }
      }
    }
  }

  // ExecutionStatistics (GroupByOperator.java:148-153 / AggregationOperator; FilteredGroupByOperator.java:148-150 sums them)
  int64_t in_filter = 0;
  for (ScanIterator* s : ctx.scans) in_filter += s->entries_scanned();
  total_docs_scanned += docs_scanned;
  total_in_filter += in_filter;
  total_post_filter += docs_scanned * (int64_t)projected.size();
  }  // infos
  res.stats[0] = total_docs_scanned;
  res.stats[1] = total_in_filter;
  res.stats[2] = total_post_filter;
  res.stats[3] = num_docs;

  res.num_group_by = k;
  res.dbl.resize(nagg);
  res.lng.resize(nagg);
  res.distinct.resize(nagg);
  auto emit_group = [&](int a, int g) {
    AggState& s = aggs[a];
    const int fn = s.spec.function;
    double d = s.dbl[g];
    int64_t l = 0;
    if (fn == PO_COUNT) l = (int64_t)d;  // extract: (long) double :178-185
    if (fn == PO_AVG) l = s.cnt[g];
    if (fn == PO_DISTINCTCOUNT) {
      std::vector<int32_t> ids;
      if (g < (int)s.bits.size()) for (int i = 0; i < (int)s.bits[g].size(); i++) if (s.bits[g][i]) ids.push_back(i);
      if (g < (int)s.raw_bits.size()) for (int i = 0; i < (int)s.raw_bits[g].size(); i++) if (s.raw_bits[g][i]) ids.push_back(i);
      l = (int64_t)ids.size();
      d = (double)l;
      res.distinct[a].push_back(std::move(ids));
    }
    res.dbl[a].push_back(d);
    res.lng[a].push_back(l);
  };
  res.raw_distinct_bits.resize(nagg);
  res.raw_distinct_type.assign(nagg, -1);
  for (int a = 0; a < nagg; a++)
    if (!aggs[a].raw_values.empty()) { res.raw_distinct_bits[a] = aggs[a].raw_values; res.raw_distinct_type[a] = aggs[a].col->c->data_type; }
  if (k == 0) {
    res.num_groups = -1;
    for (int a = 0; a < nagg; a++) emit_group(a, 0);
    return;
  }
  // group keys: ARRAY regime iterates raw keys with flag set (ascending); map regimes in group-id order
  res.limit_reached = gkg.num_keys_total() >= q.num_groups_limit;  // GroupByOperator.java:116-119
  std::vector<std::pair<int64_t, int>> groups;  // (raw key or index, group id)
  if (gkg.regime == PO_REGIME_ARRAY) {
    for (int r = 0; r < gkg.upper_bound; r++) if (gkg.flags[r]) groups.push_back({r, r});
  } else if (gkg.regime == PO_REGIME_ARRAY_MAP || gkg.regime == PO_REGIME_NO_DICT) {
    for (int g = 0; g < (int)gkg.array_keys_in_order.size(); g++) groups.push_back({g, g});
  } else {
    for (int g = 0; g < (int)gkg.keys_in_order.size(); g++) groups.push_back({gkg.keys_in_order[g], g});
  }
  res.num_groups = (int)groups.size();
  for (auto& a : aggs) a.ensure(gkg.regime == PO_REGIME_ARRAY ? gkg.upper_bound : res.num_groups);
  if (gkg.regime == PO_REGIME_NO_DICT) {
    res.raw_key_bits = gkg.otf_values;
    for (int j = 0; j < k; j++) res.raw_key_type.push_back(gkg.col_raw[j] ? seg.cols[q.group_by_columns[j]].c->data_type : -1);
  }
  for (auto& gr : groups) {
    if (gkg.regime == PO_REGIME_ARRAY_MAP || gkg.regime == PO_REGIME_NO_DICT) {
      for (int j = 0; j < k; j++) res.keys.push_back(gkg.array_keys_in_order[gr.second][j]);
    } else {
      int64_t raw = gr.first;
      for (int j = 0; j < k; j++) { res.keys.push_back((int32_t)(raw % gkg.cards[j])); raw /= gkg.cards[j]; }  // getKeys :577-605
    }
    for (int a = 0; a < nagg; a++) emit_group(a, gr.second);
  }
}

}  // namespace

extern "C" {

int32_t po_num_bits_per_value(int32_t max_value) { return num_bits_per_value(max_value); }

void po_bitset_write(uint8_t* buf, int64_t start_index, int32_t bits, int64_t n, const int32_t* values) {
  for (int64_t i = 0; i < n; i++) bitset_write_one(buf, start_index + i, bits, values[i]);
}
int32_t po_bitset_read(const uint8_t* buf, int64_t index, int32_t bits) { return bitset_read_one(buf, index, bits); }
int32_t po_fixedbit_read(const uint8_t* buf, int64_t index, int32_t bits) { return bitset_read_one(buf, index, bits); }
int32_t po_fixedbit_read_unchecked(const uint8_t* buf, int64_t index, int32_t bits) { return fixedbit_read_unchecked(buf, index, bits); }
void po_fixedbit_read32(const uint8_t* buf, int64_t index, int32_t bits, int32_t* out) { fixedbit_read32(buf, index, bits, out); }
void po_fwd_read_dict_ids(const uint8_t* buf, int32_t num_docs, int32_t bits, const int32_t* doc_ids, int32_t length, int32_t* out) {
  fwd_read_dict_ids(buf, num_docs, bits, doc_ids, length, out);
}

int64_t po_roaring_serialize(const uint32_t* v, int64_t n, int32_t run_optimize, uint8_t* out, int64_t cap) {
  return roaring_serialize(v, n, run_optimize != 0, out, cap);
}
int64_t po_roaring_deserialize(const uint8_t* buf, int64_t len, uint32_t* out, int64_t cap) {
  int64_t i = 0;
  return roaring_for_each(buf, len, [&](uint32_t v) { if (i < cap) out[i] = v; i++; });
}

// BitmapInvertedIndexWriter layout (seglocal/segment/creator/impl/inv/BitmapInvertedIndexWriter.java:33-50,90-97):
// (card+1) BE u32 offsets relative to the start of the file, then the serialized bitmaps.
int64_t po_inverted_index_build(const int32_t* dict_ids, int32_t num_docs, int32_t cardinality, uint8_t* out, int64_t cap) {
  std::vector<int64_t> counts(cardinality + 1, 0);
  for (int i = 0; i < num_docs; i++) counts[dict_ids[i] + 1]++;
  for (int i = 0; i < cardinality; i++) counts[i + 1] += counts[i];
  std::vector<uint32_t> docs(num_docs);
  std::vector<int64_t> fill(counts.begin(), counts.end() - 1);
  for (int i = 0; i < num_docs; i++) docs[fill[dict_ids[i]]++] = (uint32_t)i;
  int64_t pos = 4ll * (cardinality + 1);
  ByteSink offs{out, cap};
  for (int d = 0; d < cardinality; d++) {
    offs.be_u32((uint32_t)pos);
    int64_t n = counts[d + 1] - counts[d];
    int64_t room = out && cap > pos ? cap - pos : 0;
    pos += roaring_serialize(docs.data() + counts[d], n, true, room ? out + pos : nullptr, room);
  }
  offs.be_u32((uint32_t)pos);
  return pos;
}

po_result_t* po_execute(const po_segment_t* segment, const po_query_t* query) {
  auto* r = new po_result();
  try {
    Segment seg(segment);
    run_query(seg, *query, *r, nullptr, 0);
  } catch (const std::exception& e) {
    r->error = e.what();
  }
  return r;
}

int64_t po_filter_doc_ids(const po_segment_t* segment, const po_query_t* query, int32_t* out, int64_t cap, int64_t* entries) {
  po_result r;
  Segment seg(segment);
  po_query_t q = *query;
  q.num_aggs = 0;
  q.num_group_by = 0;
  std::vector<int32_t> ids;
  run_query(seg, q, r, &ids, cap);
  for (size_t i = 0; i < ids.size(); i++) out[i] = ids[i];
  if (entries) *entries = r.stats[1];
  return r.stats[0];
}

const char* po_result_error(const po_result_t* r) { return r->error.empty() ? nullptr : r->error.c_str(); }
int32_t po_result_num_groups(const po_result_t* r) { return r->num_groups; }
int32_t po_result_regime(const po_result_t* r) { return r->regime; }
int32_t po_result_groups_limit_reached(const po_result_t* r) { return r->limit_reached; }
void po_result_stats(const po_result_t* r, int64_t out[4]) { memcpy(out, r->stats, sizeof r->stats); }
void po_result_group_keys(const po_result_t* r, int32_t* out) { if (!r->keys.empty()) memcpy(out, r->keys.data(), r->keys.size() * 4); }
void po_result_agg_double(const po_result_t* r, int32_t a, double* out) { if (!r->dbl[a].empty()) memcpy(out, r->dbl[a].data(), r->dbl[a].size() * 8); }
void po_result_agg_long(const po_result_t* r, int32_t a, int64_t* out) { if (!r->lng[a].empty()) memcpy(out, r->lng[a].data(), r->lng[a].size() * 8); }
int64_t po_result_distinct(const po_result_t* r, int32_t a, int32_t g, int32_t* out, int64_t cap) {
  if (a >= (int)r->distinct.size() || g >= (int)r->distinct[a].size()) return 0;
  const auto& v = r->distinct[a][g];
  for (int64_t i = 0; i < (int64_t)v.size() && i < cap; i++) out[i] = v[i];
  return (int64_t)v.size();
}
// Raw group-by column j: the on-the-fly dictionary (id -> value); returns its size, 0 for dictionary columns.
int64_t po_result_raw_key_values(const po_result_t* r, int32_t j, double* out_d, int64_t* out_l, int64_t cap) {
  if (j < 0 || j >= (int)r->raw_key_bits.size()) return 0;
  const auto& v = r->raw_key_bits[j];
  const bool integral = r->raw_key_type[j] == PO_INT || r->raw_key_type[j] == PO_LONG;
  for (int64_t i = 0; i < (int64_t)v.size() && i < cap; i++) {
    double d; int64_t l;
    if (integral) { l = (int64_t)v[i]; d = (double)l; } else { memcpy(&d, &v[i], 8); l = (int64_t)d; }
    if (out_d) out_d[i] = d;
    if (out_l) out_l[i] = l;
  }
  return (int64_t)v.size();
}
// Raw DISTINCTCOUNT of aggregation a: the value numbering its id sets (po_result_distinct) refer to; 0 for dictionary columns.
int64_t po_result_raw_distinct_values(const po_result_t* r, int32_t a, double* out_d, int64_t* out_l, int64_t cap) {
  if (a < 0 || a >= (int)r->raw_distinct_bits.size()) return 0;
  const auto& v = r->raw_distinct_bits[a];
  const bool integral = r->raw_distinct_type[a] == PO_INT || r->raw_distinct_type[a] == PO_LONG;
  for (int64_t i = 0; i < (int64_t)v.size() && i < cap; i++) {
    double d; int64_t l;
    if (integral) { l = (int64_t)v[i]; d = (double)l; } else { memcpy(&d, &v[i], 8); l = (int64_t)d; }
    if (out_d) out_d[i] = d;
    if (out_l) out_l[i] = l;
  }
  return (int64_t)v.size();
}
void po_result_free(po_result_t* r) { delete r; }

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------------
// Star-tree: OffHeapStarTree (seglocal/startree/OffHeapStarTree.java:39-82: LITTLE-endian buffer; magic
// 0xBADDA55B00DAD00D, version 1, header size, dimensions, numNodes; then 7 x int32 per node,
// seglocal/startree/OffHeapStarTreeNode.java:30-47) and the BFS of
// core/startree/operator/StarTreeFilterOperator.java:217-370 (traverseStarTree).
// ------------------------------------------------------------------------------------------------------------------
namespace {
constexpr int kStarAll = -1;  // StarTreeNode.ALL
struct StarTree {
  int num_dims = 0, num_nodes = 0;
  std::vector<std::string> dims;
  const uint8_t* nodes = nullptr;
  int field(int node, int f) const { return (int)le32(nodes + 28ll * node + 4 * f); }
  int dim_id(int n) const { return field(n, 0); }
  int dim_value(int n) const { return field(n, 1); }
  int start(int n) const { return field(n, 2); }
  int end(int n) const { return field(n, 3); }
  int agg_doc(int n) const { return field(n, 4); }
  int first_child(int n) const { return field(n, 5); }
  int last_child(int n) const { return field(n, 6); }
  bool is_leaf(int n) const { return first_child(n) == -1; }
  int num_children(int n) const { return is_leaf(n) ? 0 : last_child(n) - first_child(n) + 1; }
  // getChildForDimensionValue: children are sorted by dimension value (star = -1 first) -> binary search
  int child_for_value(int n, int value) const {
    if (is_leaf(n)) return -1;
    int lo = first_child(n), hi = last_child(n);
    while (lo <= hi) {
      int mid = (lo + hi) >> 1, v = dim_value(mid);
      if (v == value) return mid;
      if (v < value) lo = mid + 1; else hi = mid - 1;
    }
    return -1;
  }
};
bool parse_star_tree(const uint8_t* b, int64_t len, StarTree& t) {
  if (len < 24 || le64(b) != 0xBADDA55B00DAD00Dull || le32(b + 8) != 1) return false;
  int64_t root_off = le32(b + 12);
  t.num_dims = (int)le32(b + 16);
  int64_t off = 20;
  t.dims.assign(t.num_dims, "");
  for (int i = 0; i < t.num_dims; i++) {
    if (off + 8 > len) return false;
    int id = (int)le32(b + off), n = (int)le32(b + off + 4);
    off += 8;
    if (id < 0 || id >= t.num_dims || off + n > len) return false;
    t.dims[id] = std::string((const char*)b + off, n);
    off += n;
  }
  t.num_nodes = (int)le32(b + off);
  off += 4;
  if (off != root_off || off + 28ll * t.num_nodes != len) return false;
  t.nodes = b + off;
  return true;
}
}  // namespace

extern "C" int32_t po_startree_info(const uint8_t* tree, int64_t len, int32_t out[2], char* names, int32_t cap) {
  StarTree t;
  if (!parse_star_tree(tree, len, t)) return -1;
  out[0] = t.num_dims; out[1] = t.num_nodes;
  int pos = 0;
  for (auto& d : t.dims) for (size_t i = 0; i <= d.size() && pos < cap; i++) names[pos++] = i < d.size() ? d[i] : '\0';
  return 0;
}

extern "C" int64_t po_startree_traverse(const uint8_t* tree, int64_t len, int32_t num_predicates,
                                        const po_star_predicate_t* predicates, int32_t num_group_by,
                                        const int32_t* group_by_dims, int32_t* out_docs, int64_t cap,
                                        uint32_t* remaining_predicate_mask) {
  StarTree t;
  if (!parse_star_tree(tree, len, t)) return -2;
  std::vector<const po_star_predicate_t*> pred_of(t.num_dims, nullptr);
  uint32_t remaining_pred = 0, remaining_gb = 0;
  for (int i = 0; i < num_predicates; i++) { pred_of[predicates[i].dimension] = &predicates[i]; remaining_pred |= 1u << predicates[i].dimension; }
  for (int i = 0; i < num_group_by; i++) remaining_gb |= 1u << group_by_dims[i];
  std::vector<int> docs;
  auto add_range = [&](long long s, long long e) { for (long long d = s; d < e; d++) docs.push_back((int)d); };
  bool found_leaf = t.is_leaf(0);
  bool have_global = false;
  uint32_t global_remaining = 0;
  if (found_leaf) { global_remaining = remaining_pred; have_global = true; }
  std::vector<int> queue{0};
  size_t head = 0;
  int current_dim = -1;
  const po_star_predicate_t* matching = nullptr;
  while (head < queue.size()) {
    int node = queue[head++];
    int dim = t.dim_id(node);
    if (dim > current_dim) {  // previous level finished
      remaining_pred &= ~(1u << dim);
      remaining_gb &= ~(1u << dim);
      if (found_leaf && !have_global) { global_remaining = remaining_pred; have_global = true; }
      matching = nullptr;
      current_dim = dim;
    }
    if (remaining_pred == 0 && remaining_gb == 0) { docs.push_back(t.agg_doc(node)); continue; }
    if (t.is_leaf(node)) { add_range(t.start(node), t.end(node)); continue; }
    const int child_dim = dim + 1;
    int star_node = -1;
    if ((!have_global || !(global_remaining >> child_dim & 1)) && !(remaining_gb >> child_dim & 1))
      star_node = t.child_for_value(node, kStarAll);
    const int first = t.first_child(node), nchild = t.num_children(node);
    if (remaining_pred >> child_dim & 1) {
      if (!matching) {
        matching = pred_of[child_dim];
        if (matching->num_ids == 0) return -1;
      }
      auto contains = [&](int v) { return std::binary_search(matching->ids, matching->ids + matching->num_ids, v); };
      if ((long long)matching->num_ids * 10 > nchild) {  // USE_SCAN_TO_TRAVERSE_NODES_THRESHOLD
        if (star_node >= 0 && matching->num_ids >= nchild - 1) {
          std::vector<int> match_children;
          bool leaf_child = false;
          for (int c = first; c < first + nchild; c++)
            if (contains(t.dim_value(c))) { match_children.push_back(c); leaf_child |= t.is_leaf(c); }
          if ((int)match_children.size() == nchild - 1) { queue.push_back(star_node); found_leaf |= t.is_leaf(star_node); }
          else { for (int c : match_children) queue.push_back(c); found_leaf |= leaf_child; }
        } else {
          for (int c = first; c < first + nchild; c++)
            if (contains(t.dim_value(c))) { queue.push_back(c); found_leaf |= t.is_leaf(c); }
        }
      } else {
        for (int i = 0; i < matching->num_ids; i++) {
          int c = t.child_for_value(node, matching->ids[i]);
          if (c >= 0) { queue.push_back(c); found_leaf |= t.is_leaf(c); }
        }
      }
    } else if (star_node >= 0) {
      queue.push_back(star_node);
      found_leaf |= t.is_leaf(star_node);
    } else {
      for (int c = first; c < first + nchild; c++)
        if (t.dim_value(c) != kStarAll) { queue.push_back(c); found_leaf |= t.is_leaf(c); }
    }
  }
  std::sort(docs.begin(), docs.end());
  docs.erase(std::unique(docs.begin(), docs.end()), docs.end());
  for (int64_t i = 0; i < (int64_t)docs.size() && i < cap; i++) out_docs[i] = docs[i];
  if (remaining_predicate_mask) *remaining_predicate_mask = have_global ? global_remaining : 0u;
  return (int64_t)docs.size();
}

// ------------------------------------------------------------------------------------------------------------------
// Benchmark table generator (CPU twin of pinot_b200/csrc/pb200_synth.cu; tests/test_gpu_synth.py compares the bytes).
// NOT part of the reference: it only lets bench.py's CPU arm (--impl reference) create the SAME synthetic segments
// without touching the device library.  dictId(doc) = mix64(seed + doc * 0x9E3779B97F4A7C15) % cardinality (SplitMix64
// finaliser), written as FixedBitSVForwardIndexWriter would (MSB-first big-endian bit stream); dictionary =
// { base + step * i } as sorted big-endian INT values (SegmentDictionaryCreator).
// ------------------------------------------------------------------------------------------------------------------
#include <thread>

namespace {
inline uint64_t synth_mix64(uint64_t z) {
  z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
  z ^= z >> 27; z *= 0x94D049BB133111EBull;
  z ^= z >> 31;
  return z;
}
}  // namespace

extern "C" void po_synth_fwd(uint64_t seed, int32_t cardinality, int64_t num_docs, int32_t bits, uint8_t* out, int32_t threads) {
  const int64_t groups = (num_docs + 31) / 32;          // 32 docs = `bits` whole 4-byte words
  const int64_t out_bytes = (num_docs * bits + 7) / 8;  // the last group may be cut short
  auto work = [&](int64_t g0, int64_t g1) {
    for (int64_t g = g0; g < g1; g++) {
      uint64_t acc = 0;
      int have = 0;
      int64_t o = g * bits * 4;
      for (int i = 0; i < 32; i++) {
        const int64_t doc = g * 32 + i;
        const uint32_t v = doc < num_docs ? (uint32_t)(synth_mix64(seed + (uint64_t)doc * 0x9E3779B97F4A7C15ull) % (uint32_t)cardinality) : 0u;
        acc = (acc << bits) | v;
        have += bits;
        while (have >= 8) {
          if (o < out_bytes) out[o] = (uint8_t)(acc >> (have - 8));
          o++;
          have -= 8;
        }
      }
    }
  };
  const int nt = (int)std::max<int64_t>(1, std::min<int64_t>(threads, groups / 4096 + 1));
  std::vector<std::thread> pool;
  for (int t = 0; t < nt; t++) pool.emplace_back(work, groups * t / nt, groups * (t + 1) / nt);
  for (auto& th : pool) th.join();
}

extern "C" void po_synth_dict(int32_t cardinality, int32_t base, int32_t step, uint8_t* out) {
  for (int32_t i = 0; i < cardinality; i++) {
    const uint32_t v = (uint32_t)(base + step * i);
    out[4 * i + 0] = (uint8_t)(v >> 24); out[4 * i + 1] = (uint8_t)(v >> 16); out[4 * i + 2] = (uint8_t)(v >> 8); out[4 * i + 3] = (uint8_t)v;
  }
}
