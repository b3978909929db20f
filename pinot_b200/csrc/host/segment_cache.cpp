// segment_cache.cpp -- HBM residency manager: which segments live on the device, keyed by (segment name, CRC).
//
// The reference keeps a loaded segment in its TableDataManager until the table drops or replaces it
// (pinot-core/.../data/manager/BaseTableDataManager.java: addSegment / replaceSegment / offloadSegment), identifies a segment
// version by its CRC (SegmentMetadata.getCrc(), segment-spi/.../SegmentMetadata.java; refresh = same name, new CRC) and
// reference-counts it around every query (SegmentDataManager.increaseReferenceCount / decreaseReferenceCount, acquired in
// ServerQueryExecutorV1Impl.java:217 and released in its finally block).  HBM is smaller than the page cache a JVM server
// leans on, so the device side adds what the reference gets from the OS for free: a byte budget and least-recently-used
// eviction of segments no query holds.
//
//   acquire(name, crc, dir)  hit: pin + touch.  miss: evict LRU unpinned segments until the estimate fits, load the
//                            directory (pb200h_segment_load_dir == ImmutableSegmentLoader.load), pin.  A different CRC
//                            under the same name is a refresh: the old version is dropped as soon as nobody holds it.
//   release(segment)         unpin (the query is done with it).
//   evict(name, crc)         the table dropped the segment (IndexSegment.destroy()): freed now, or when the last holder
//                            releases it.
#include <algorithm>
#include <cstring>
#include <list>
#include <map>
#include <mutex>
#include <string>

#include "host_internal.h"

using pb200::set_error;

struct pb200h_cache {
  pb200_ctx* ctx = nullptr;
  int64_t budget = 0;
  struct Entry {
    std::string name;
    uint64_t crc = 0;
    pb200h_segment* seg = nullptr;
    int64_t bytes = 0;
    int pins = 0;
    bool doomed = false;  // dropped / superseded while pinned: freed by the last release
    uint64_t last_use = 0;
  };
  std::mutex mu;
  std::list<Entry> entries;
  uint64_t clock = 0;
  int64_t resident_bytes = 0, hits = 0, misses = 0, evictions = 0;
};

namespace {
void drop(pb200h_cache* c, std::list<pb200h_cache::Entry>::iterator it) {  // caller holds mu; entry is unpinned
  c->resident_bytes -= it->bytes;
  pb200h_segment_destroy(it->seg);
  c->entries.erase(it);
}
// a segment grows when queries derive columns on it (host/transform.cpp): the resident bytes follow (caller holds mu)
void refresh_bytes(pb200h_cache* c) {
  for (auto& e : c->entries) {
    const int64_t now = pb200_segment_device_bytes(pb200h_segment_device(e.seg));
    c->resident_bytes += now - e.bytes;
    e.bytes = now;
  }
}
// frees least-recently-used unpinned segments until `need` more bytes fit the budget; false if they cannot
bool make_room(pb200h_cache* c, int64_t need) {
  refresh_bytes(c);
  while (c->resident_bytes + need > c->budget) {
    auto victim = c->entries.end();
    for (auto it = c->entries.begin(); it != c->entries.end(); ++it)
      if (it->pins == 0 && (victim == c->entries.end() || it->last_use < victim->last_use)) victim = it;
    if (victim == c->entries.end()) return false;
    drop(c, victim);
    c->evictions++;
  }
  return true;
}
}  // namespace

extern "C" int32_t pb200h_cache_create(pb200_ctx* ctx, int64_t max_device_bytes, pb200h_cache** out) {
  if (!ctx || !out) { set_error("null argument"); return PB200_E_INVALID; }
  if (max_device_bytes <= 0) {  // default: 80 % of the device's memory
    int64_t info[5];
    int rc = pb200_device_info(ctx, info);
    if (rc) return rc;
    max_device_bytes = (info[3] << 20) / 10 * 8;
  }
  auto* c = new pb200h_cache();
  c->ctx = ctx;
  c->budget = max_device_bytes;
  *out = c;
  return PB200_OK;
}

extern "C" int32_t pb200h_cache_acquire(pb200h_cache* c, const char* name, uint64_t crc, const char* index_dir,
                                        int64_t size_hint, pb200h_segment** out) {
  if (!c || !name || !out) { set_error("null argument"); return PB200_E_INVALID; }
  std::lock_guard<std::mutex> g(c->mu);  // loads are serialised: two queries missing the same segment must not load it twice
  for (auto it = c->entries.begin(); it != c->entries.end(); ++it) {
    if (it->name != name || it->doomed) continue;
    if (it->crc == crc) {
      it->pins++;
      it->last_use = ++c->clock;
      c->hits++;
      *out = it->seg;
      return PB200_OK;
    }
    // same name, other CRC: the segment was refreshed (BaseTableDataManager.replaceSegment) -- the old version goes
    if (it->pins == 0) { drop(c, it); c->evictions++; } else it->doomed = true;
    break;
  }
  c->misses++;
  if (!index_dir) { set_error("segment %s (crc %llu) is not resident and no index directory was given", name, (unsigned long long)crc); return PB200_E_INVALID; }
  if (size_hint > c->budget) { set_error("segment %s (%lld bytes) exceeds the residency budget (%lld)", name, (long long)size_hint, (long long)c->budget); return PB200_E_NOMEM; }
  if (size_hint > 0 && !make_room(c, size_hint)) { set_error("HBM budget exhausted: every resident segment is in use"); return PB200_E_NOMEM; }
  pb200h_segment* seg = nullptr;
  int rc = pb200h_segment_load_dir(c->ctx, index_dir, &seg);
  if (rc == PB200_E_NOMEM && make_room(c, c->budget - c->resident_bytes + 1)) {  // the hint was too small: free one more victim and retry once
    rc = pb200h_segment_load_dir(c->ctx, index_dir, &seg);
  }
  if (rc) return rc;
  pb200h_cache::Entry e;
  e.name = name; e.crc = crc; e.seg = seg; e.pins = 1; e.last_use = ++c->clock;
  e.bytes = pb200_segment_device_bytes(pb200h_segment_device(seg));
  c->resident_bytes += e.bytes;
  c->entries.push_back(e);
  make_room(c, 0);  // the real size may exceed the hint: trim other unpinned segments back under the budget
  *out = seg;
  return PB200_OK;
}

extern "C" int32_t pb200h_cache_release(pb200h_cache* c, pb200h_segment* seg) {
  if (!c || !seg) { set_error("null argument"); return PB200_E_INVALID; }
  std::lock_guard<std::mutex> g(c->mu);
  for (auto it = c->entries.begin(); it != c->entries.end(); ++it) {
    if (it->seg != seg) continue;
    if (it->pins <= 0) { set_error("segment %s released more often than acquired", it->name.c_str()); return PB200_E_INVALID; }
    if (--it->pins == 0 && it->doomed) drop(c, it);
    return PB200_OK;
  }
  set_error("segment is not managed by this cache");
  return PB200_E_INVALID;
}

extern "C" int32_t pb200h_cache_evict(pb200h_cache* c, const char* name, uint64_t crc) {
  if (!c || !name) { set_error("null argument"); return PB200_E_INVALID; }
  std::lock_guard<std::mutex> g(c->mu);
  for (auto it = c->entries.begin(); it != c->entries.end(); ++it) {
    if (it->name != name || it->crc != crc) continue;
    if (it->pins == 0) drop(c, it); else it->doomed = true;
    return PB200_OK;
  }
  return PB200_OK;  // not resident: nothing to do (offloadSegment of a segment that never reached the device)
}

extern "C" int32_t pb200h_cache_stats(pb200h_cache* c, int64_t out[6]) {
  if (!c || !out) { set_error("null argument"); return PB200_E_INVALID; }
  std::lock_guard<std::mutex> g(c->mu);
  refresh_bytes(c);
  out[0] = (int64_t)c->entries.size(); out[1] = c->resident_bytes; out[2] = c->budget;
  out[3] = c->hits; out[4] = c->misses; out[5] = c->evictions;
  return PB200_OK;
}

extern "C" int32_t pb200h_cache_destroy(pb200h_cache* c) {
  if (!c) return PB200_OK;
  {
    std::lock_guard<std::mutex> g(c->mu);
    for (auto& e : c->entries) pb200h_segment_destroy(e.seg);
    c->entries.clear();
  }
  delete c;
  return PB200_OK;
}
