// selection_probe.cpp -- TEST shim: pb200::plan_selection / selection_rescan (pinot_b200/csrc/pb200_plan.cpp) on segments
// made of column metadata alone, without a GPU.  Built by tests/test_selection_cpu.py with g++ against the in-tree library.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../pinot_b200/csrc/pb200_plan.h"

extern "C" {

typedef struct {
  int32_t fwd_kind, stored_type, bits, cardinality;
  int32_t dict_native;  // 1: the column has a device dictionary (a sentinel pointer, never dereferenced)
  int32_t reserved;
} sel_probe_col;

enum { SP_SEG = 40, SP_COL = 8, SP_CHUNK = 4 };
typedef struct {  // every field int64: tests/test_selection_cpu.py mirrors this list
  int64_t tile_rows, prefix, mask_words, num_chunks, limit, num_rescan;
  int64_t kinds[SP_COL];
  int64_t chunk_word_off[SP_CHUNK], chunk_total_tiles[SP_CHUNK];
  int64_t mask_word_off[SP_SEG], scan_docs[SP_SEG], num_tiles[SP_SEG], first_tile[SP_SEG], in_filter[SP_SEG], rescan[SP_SEG];
} sel_probe_plan;

int64_t sel_probe_plan_size(void) { return (int64_t)sizeof(sel_probe_plan); }

// cols: nseg x ncols; matches: per segment the matched docs of the prefix pass (for selection_rescan), may be NULL.
int32_t sel_probe_plan_selection(int32_t sm_count, int32_t max_smem_optin, const pb200_query* filter_only,
                                 const pb200_selection* sel, const sel_probe_col* cols, int32_t ncols, const int32_t* num_docs,
                                 int32_t nseg, int32_t prefix, const int64_t* matches, sel_probe_plan* out) {
  using namespace pb200;
  pb200_ctx ctx;
  static uint32_t sentinel[4];
  std::vector<pb200_segment> segs(nseg);
  std::vector<pb200_segment*> ptrs(nseg);
  for (int s = 0; s < nseg; s++) {
    segs[s].num_docs = num_docs[s];
    segs[s].cols.resize(ncols);
    for (int k = 0; k < ncols; k++) {
      const sel_probe_col& p = cols[(size_t)s * ncols + k];
      DeviceColumn& c = segs[s].cols[k];
      c.fwd_kind = p.fwd_kind; c.stored_type = p.stored_type; c.bits = p.bits; c.cardinality = p.cardinality;
      c.fwd = sentinel;
      c.dict_native = p.dict_native ? sentinel : nullptr;
    }
    ptrs[s] = &segs[s];
  }
  SelectionPlan plan;
  memset(out, 0, sizeof *out);
  const int rc = plan_selection(ctx.tune, DeviceLimits{sm_count, max_smem_optin}, filter_only, sel, ptrs.data(), nseg, prefix != 0, &plan);
  if (rc) return rc;
  sel_probe_plan& o = *out;
  o.tile_rows = plan.scan.q.tile_rows; o.prefix = plan.prefix; o.mask_words = plan.mask_words; o.limit = plan.limit;
  o.num_chunks = (int64_t)plan.scan.chunks.size();
  for (size_t k = 0; k < plan.kinds.size() && k < SP_COL; k++) o.kinds[k] = plan.kinds[k];
  for (size_t c = 0; c < plan.scan.chunks.size() && c < SP_CHUNK; c++) {
    o.chunk_word_off[c] = plan.chunk_word_off[c];
    o.chunk_total_tiles[c] = plan.scan.chunks[c].total_tiles;
  }
  for (int s = 0; s < nseg && s < SP_SEG; s++) {
    o.mask_word_off[s] = plan.mask_word_off[s]; o.scan_docs[s] = plan.scan_docs[s];
    o.num_tiles[s] = plan.scan.segs[s].num_tiles; o.first_tile[s] = plan.scan.segs[s].first_tile;
    o.in_filter[s] = plan.scan.in_filter[s];
  }
  if (matches) {
    const std::vector<long long> m(matches, matches + nseg);
    const std::vector<int> r = selection_rescan(plan, ptrs.data(), m);
    o.num_rescan = (int64_t)r.size();
    for (size_t i = 0; i < r.size() && i < SP_SEG; i++) o.rescan[i] = r[i];
  }
  return PB200_OK;
}

}  // extern "C"
