// star_tree.cpp -- star-tree support of the native host layer (include/pinot_b200_host.h).
//
// Restates the DECISIONS of
//   seglocal/startree/OffHeapStarTree.java:39-82, OffHeapStarTreeNode.java:30-47      on-disk tree (little-endian)
//   seglocal/startree/v2/store/StarTreeLoaderUtils.java:54-88                            which buffers make a StarTreeV2
//   core/startree/StarTreeUtils.java + AggregationFunctionUtils.buildAggregationInfo :285-310   when a query fits
//   core/startree/operator/StarTreeFilterOperator.java:217-370                           the BFS traversal
// The pre-aggregated docs live in HBM as a segment of their own and are scanned by the SAME kernel as raw segments:
// dimensions are fixed-bit dictId columns (shared dictionaries); the raw 64-bit metric columns are dictionary-encoded
// once at attach time (sorted distinct LONG / DOUBLE values + fixed-bit ids) so that SUM / MIN / MAX over them are
// the kernel's dictionary-gather / dictId-order paths.  The traversal result reaches the device as a doc mask
// (PB200_F_DOC_MASK), i.e. the BitmapBasedFilterOperator the reference builds from the matched doc ids.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "host_internal.h"
#include "../pb200_order.h"
#include "../pb200_startree_build.h"

using pb200::set_error;

namespace pb200h {

static inline uint32_t le32(const unsigned char* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
static inline uint64_t le64(const unsigned char* p) { return (uint64_t)le32(p) | (uint64_t)le32(p + 4) << 32; }
static inline uint32_t be32(const unsigned char* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
static inline uint64_t be64(const unsigned char* p) { return (uint64_t)be32(p) << 32 | be32(p + 4); }

bool StarTree::parse(const unsigned char* b, uint64_t len) {
  if (len < 24 || le64(b) != 0xBADDA55B00DAD00Dull || le32(b + 8) != 1) return false;
  const uint64_t root = le32(b + 12);
  const int nd = (int)le32(b + 16);
  if (nd < 0 || nd > 32) return false;  // dimensions are addressed by bits of a 32-bit mask
  uint64_t off = 20;
  dim_names.assign(nd, "");
  for (int i = 0; i < nd; i++) {
    if (off + 8 > len) return false;
    int id = (int)le32(b + off), n = (int)le32(b + off + 4);
    off += 8;
    if (id < 0 || id >= nd || n < 0 || off + (uint64_t)n > len) return false;
    dim_names[id] = std::string((const char*)b + off, n);
    off += n;
  }
  if (off + 4 > len) return false;
  num_nodes = (int)le32(b + off);
  off += 4;
  if (num_nodes <= 0 || off != root || off + 28ull * (uint64_t)num_nodes != len) return false;
  bytes.assign(b, b + len);
  nodes = bytes.data() + off;
  // a malformed buffer must not send the traversal out of bounds or in circles: children lie behind their parent
  // (OffHeapStarTreeBuilder writes nodes breadth first), inside the node array, first <= last; doc ranges are ordered
  for (int n = 0; n < num_nodes; n++) {
    const int fc = first_child(n), lc = last_child(n);
    if (fc == -1) continue;
    if (fc <= n || lc < fc || lc >= num_nodes) { nodes = nullptr; num_nodes = 0; return false; }
  }
  for (int n = 0; n < num_nodes; n++)
    if ((!(start(n) == -1 && end(n) == -1) && (start(n) < 0 || end(n) < start(n))) || dim_id(n) >= nd) { nodes = nullptr; num_nodes = 0; return false; }  // (-1, -1): the root
  return true;
}

int StarTree::child_for_value(int n, int value) const {
  if (is_leaf(n)) return -1;
  int lo = first_child(n), hi = last_child(n);
  while (lo <= hi) {
    int mid = (lo + hi) >> 1, v = dim_value(mid);
    if (v == value) return mid;
    if (v < value) lo = mid + 1; else hi = mid - 1;
  }
  return -1;
}

// StarTreeFilterOperator.traverseStarTree.  preds[d] == nullptr: no predicate on dimension d.
// Returns false when some predicate matches no dictId (EmptyFilterOperator).
// Matching docs come back as [start, end) ranges (adjacent ones coalesced): a star-tree node IS a doc range, and the
// device consumes them as a doc mask, so single doc ids are never materialised.
bool StarTree::traverse(const std::vector<const std::vector<int32_t>*>& preds, uint32_t group_by_mask,
                        std::vector<std::pair<int32_t, int32_t>>& docs, uint32_t& remaining_out) const {
  auto add = [&](int32_t s, int32_t e) {
    if (!docs.empty() && docs.back().second == s) docs.back().second = e;
    else docs.emplace_back(s, e);
  };
  constexpr int kAll = -1;
  uint32_t remaining_pred = 0, remaining_gb = group_by_mask;
  for (size_t d = 0; d < preds.size(); d++) if (preds[d]) remaining_pred |= 1u << d;
  bool found_leaf = is_leaf(0), have_global = false;
  uint32_t global_remaining = 0;
  if (found_leaf) { global_remaining = remaining_pred; have_global = true; }
  std::vector<int> queue{0};
  size_t head = 0;
  int current_dim = -1;
  const std::vector<int32_t>* matching = nullptr;
  docs.clear();
  while (head < queue.size()) {
    const int node = queue[head++];
    const int dim = dim_id(node);
    if (dim > current_dim) {
      remaining_pred &= ~(1u << dim);
      remaining_gb &= ~(1u << dim);
      if (found_leaf && !have_global) { global_remaining = remaining_pred; have_global = true; }
      matching = nullptr;
      current_dim = dim;
    }
    if (remaining_pred == 0 && remaining_gb == 0) { add(agg_doc(node), agg_doc(node) + 1); continue; }
    if (is_leaf(node)) { add(start(node), end(node)); continue; }
    const int child_dim = dim + 1;
    int star_node = -1;
    if ((!have_global || !((global_remaining >> child_dim) & 1)) && !((remaining_gb >> child_dim) & 1))
      star_node = child_for_value(node, kAll);
    const int first = first_child(node), nchild = num_children(node);
    if ((remaining_pred >> child_dim) & 1) {
      if (!matching) {
        matching = preds[child_dim];
        if (matching->empty()) return false;
      }
      auto contains = [&](int v) { return std::binary_search(matching->begin(), matching->end(), v); };
      if ((long long)matching->size() * 10 > nchild) {  // USE_SCAN_TO_TRAVERSE_NODES_THRESHOLD
        if (star_node >= 0 && (int)matching->size() >= nchild - 1) {
          std::vector<int> hit;
          bool leaf_child = false;
          for (int c = first; c < first + nchild; c++) if (contains(dim_value(c))) { hit.push_back(c); leaf_child |= is_leaf(c); }
          if ((int)hit.size() == nchild - 1) { queue.push_back(star_node); found_leaf |= is_leaf(star_node); }
          else { for (int c : hit) queue.push_back(c); found_leaf |= leaf_child; }
        } else {
          for (int c = first; c < first + nchild; c++) if (contains(dim_value(c))) { queue.push_back(c); found_leaf |= is_leaf(c); }
        }
      } else {
        for (int32_t id : *matching) {
          int c = child_for_value(node, id);
          if (c >= 0) { queue.push_back(c); found_leaf |= is_leaf(c); }
        }
      }
    } else if (star_node >= 0) {
      queue.push_back(star_node);
      found_leaf |= is_leaf(star_node);
    } else {
      for (int c = first; c < first + nchild; c++) if (dim_value(c) != kAll) { queue.push_back(c); found_leaf |= is_leaf(c); }
    }
  }
  remaining_out = have_global ? global_remaining : 0u;
  return true;
}

// raw PASS_THROUGH chunk file -> 64-bit values (BaseChunkForwardIndexReader header :60-106)
static bool read_raw64(const unsigned char* p, uint64_t len, int n, std::vector<uint64_t>& out) {
  if (len < 28) return false;
  const int version = (int)be32(p), nchunks = (int)be32(p + 4), entry = (int)be32(p + 12);
  if (version < 2 || be32(p + 20) != 0 || entry != 8) return false;
  const uint64_t start = be32(p + 24) + (uint64_t)nchunks * (version <= 2 ? 4 : 8);
  if (len < start + 8ull * n) return false;
  out.resize(n);
  for (int i = 0; i < n; i++) out[i] = be64(p + start + 8ull * i);
  return true;
}

static void pack_bits(const std::vector<int32_t>& ids, int bits, std::vector<unsigned char>& out) {
  out.assign(((uint64_t)ids.size() * bits + 7) / 8 + 8, 0);
  uint64_t bit = 0;
  for (int32_t id : ids)
    for (int b = bits - 1; b >= 0; b--, bit++)
      if ((id >> b) & 1) out[bit >> 3] |= (unsigned char)(0x80 >> (bit & 7));
  out.resize(((uint64_t)ids.size() * bits + 7) / 8);
}

}  // namespace pb200h

using namespace pb200h;

extern "C" int32_t pb200h_startree_attach(pb200_ctx* ctx, pb200h_segment* seg, const void* tree, uint64_t tree_bytes,
                                          int32_t num_star_docs, int32_t ndims, const char* const* dim_names,
                                          const void* const* dim_fwd, const uint64_t* dim_fwd_bytes, int32_t nmetrics,
                                          const pb200h_star_metric* metrics) {
  if (!ctx || !seg || !tree || ndims <= 0 || ndims > 30 || nmetrics <= 0 || num_star_docs <= 0) { set_error("invalid argument to pb200h_startree_attach"); return PB200_E_INVALID; }
  if (seg->dev && seg->dev->domain) { set_error("segment is bound to a dictionary domain: star-tree dimension ids would not match"); return PB200_E_UNSUPPORTED; }
  std::unique_ptr<StarTreeIndex> st(new StarTreeIndex());
  if (!st->tree.parse((const unsigned char*)tree, tree_bytes)) { set_error("malformed star-tree buffer (magic / version / size)"); return PB200_E_INVALID; }
  if ((int)st->tree.dim_names.size() != ndims) { set_error("star-tree has %zu dimensions, %d given", st->tree.dim_names.size(), ndims); return PB200_E_INVALID; }
  // star-tree docs as a segment: dimensions first (same names, dictionaries, bits as the base columns), then metrics
  std::vector<pb200h_column> cols;
  std::vector<std::string> names;
  std::vector<std::vector<unsigned char>> bufs;  // packed metric ids + metric dictionaries
  bufs.reserve(2 * nmetrics);
  names.reserve(ndims + nmetrics);
  for (int d = 0; d < ndims; d++) {
    if (st->tree.dim_names[d] != dim_names[d]) { set_error("dimension %d is '%s' in the tree but '%s' was given", d, st->tree.dim_names[d].c_str(), dim_names[d]); return PB200_E_INVALID; }
    const int bc = seg->column_index(dim_names[d]);
    if (bc < 0 || !seg->cols[bc].has_dictionary) { set_error("star-tree dimension '%s' is not a dictionary column of the segment", dim_names[d]); return PB200_E_INVALID; }
    const HostColumn& base = seg->cols[bc];
    st->dim_base_col.push_back(bc);
    pb200h_column c;
    memset(&c, 0, sizeof c);
    names.push_back(dim_names[d]);
    c.data_type = base.data_type; c.has_dictionary = 1; c.bits_per_value = base.bits; c.cardinality = base.cardinality;
    c.dict_entry_bytes = base.entry_bytes;
    c.fwd = dim_fwd[d]; c.fwd_bytes = dim_fwd_bytes[d];
    c.dict = base.dict.data(); c.dict_bytes = base.dict.size();
    cols.push_back(c);
  }
  for (int m = 0; m < nmetrics; m++) {
    const pb200h_star_metric& sm = metrics[m];
    if (sm.function != PB200_AGG_COUNT && sm.function != PB200_AGG_SUM && sm.function != PB200_AGG_MIN && sm.function != PB200_AGG_MAX) {
      set_error("function-column pair %d: function %d not accelerated", m, sm.function); return PB200_E_UNSUPPORTED;
    }
    int bc = -1;
    if (sm.function != PB200_AGG_COUNT) {
      bc = seg->column_index(sm.column);
      if (bc < 0) { set_error("function-column pair %d: unknown column '%s'", m, sm.column ? sm.column : "(null)"); return PB200_E_INVALID; }
    }
    std::vector<uint64_t> raw;
    if (!read_raw64((const unsigned char*)sm.fwd, sm.fwd_bytes, num_star_docs, raw)) { set_error("function-column pair %d: not an uncompressed 8-byte raw forward index", m); return PB200_E_UNSUPPORTED; }
    // dictionary-encode: sorted distinct values (LONG for count__*, DOUBLE otherwise) + ids
    const bool is_long = sm.function == PB200_AGG_COUNT;
    std::vector<int32_t> ids(num_star_docs);
    std::vector<unsigned char> dict;
    int card = 0;
    if (is_long) {
      std::vector<int64_t> v(raw.begin(), raw.end()), u;
      u = v; std::sort(u.begin(), u.end()); u.erase(std::unique(u.begin(), u.end()), u.end());
      card = (int)u.size();
      for (int i = 0; i < num_star_docs; i++) ids[i] = (int32_t)(std::lower_bound(u.begin(), u.end(), v[i]) - u.begin());
      dict.resize(8ull * card);
      for (int i = 0; i < card; i++) { uint64_t x = (uint64_t)u[i]; for (int b = 0; b < 8; b++) dict[8ull * i + b] = (unsigned char)(x >> (56 - 8 * b)); }
    } else {
      // sorted and made unique by Double.compare order keys: a pre-aggregated SUM may be NaN (one value, last) or -0.0
      std::vector<uint64_t> v(num_star_docs), u;
      for (int i = 0; i < num_star_docs; i++) { double d; memcpy(&d, &raw[i], 8); v[i] = pb200::double_order_bits(d); }
      u = v; std::sort(u.begin(), u.end()); u.erase(std::unique(u.begin(), u.end()), u.end());
      card = (int)u.size();
      for (int i = 0; i < num_star_docs; i++) ids[i] = (int32_t)(std::lower_bound(u.begin(), u.end(), v[i]) - u.begin());
      dict.resize(8ull * card);
      for (int i = 0; i < card; i++) {
        const uint64_t x = (u[i] >> 63) ? (u[i] & 0x7FFFFFFFFFFFFFFFull) : ~u[i];   // the key back to the double's bits
        for (int b = 0; b < 8; b++) dict[8ull * i + b] = (unsigned char)(x >> (56 - 8 * b));
      }
    }
    int bits = 1;
    while (bits < 31 && (1ll << bits) < card) bits++;
    std::vector<unsigned char> packed;
    pack_bits(ids, bits, packed);
    bufs.push_back(std::move(packed));
    bufs.push_back(std::move(dict));
    names.push_back(lower_fn_name(sm.function) + "__" + (sm.column ? sm.column : "*"));
    pb200h_column c;
    memset(&c, 0, sizeof c);
    c.data_type = is_long ? PB200_LONG : PB200_DOUBLE; c.has_dictionary = 1; c.bits_per_value = bits; c.cardinality = card; c.dict_entry_bytes = 8;
    c.fwd = bufs[bufs.size() - 2].data(); c.fwd_bytes = bufs[bufs.size() - 2].size();
    c.dict = bufs.back().data(); c.dict_bytes = bufs.back().size();
    cols.push_back(c);
    st->metric_fn.push_back(sm.function);
    st->metric_base_col.push_back(bc);
  }
  for (size_t i = 0; i < cols.size(); i++) cols[i].name = names[i].c_str();
  st->num_docs = num_star_docs;
  pb200h_segment* star = nullptr;
  int rc = pb200h_segment_create(ctx, (seg->name + "$startree").c_str(), num_star_docs, (int)cols.size(), cols.data(), &star);
  if (rc) return rc;
  st->star_segment = star;
  seg->star_trees.push_back(std::move(st));
  return PB200_OK;
}

extern "C" int32_t pb200h_startree_build(pb200_ctx* ctx, pb200h_segment* seg, const pb200h_startree_config* cfg,
                                         pb200h_startree_build_info* info) {
  // the configuration first: these refusals need no segment
  if (!cfg || cfg->num_dimensions < 1 || !cfg->dimensions) { set_error("star-tree config: empty dimensionsSplitOrder"); return PB200_E_INVALID; }
  const int D = cfg->num_dimensions, M = cfg->num_pairs;
  if (D > 30) { set_error("star-tree config: %d dimensions, at most 30 are supported", D); return PB200_E_UNSUPPORTED; }
  std::set<std::string> split;
  for (int j = 0; j < D; j++) {
    if (!cfg->dimensions[j]) { set_error("star-tree config: dimension %d has no name", j); return PB200_E_INVALID; }
    if (!split.insert(cfg->dimensions[j]).second) { set_error("star-tree config: dimension '%s' repeated in the split order", cfg->dimensions[j]); return PB200_E_INVALID; }
  }
  std::vector<char> skip(D, 0);
  if (cfg->num_skip_star < 0 || (cfg->num_skip_star > 0 && !cfg->skip_star)) { set_error("star-tree config: bad skipStarNodeCreationForDimensions"); return PB200_E_INVALID; }
  for (int s = 0; s < cfg->num_skip_star; s++) {
    int j = 0;
    while (j < D && !(cfg->skip_star[s] && strcmp(cfg->skip_star[s], cfg->dimensions[j]) == 0)) j++;
    if (j == D) { set_error("star-tree config: skip-star dimension '%s' is not in the split order", cfg->skip_star[s] ? cfg->skip_star[s] : "(null)"); return PB200_E_INVALID; }
    skip[j] = 1;
  }
  if (cfg->max_leaf_records < 1) { set_error("star-tree config: maxLeafRecords %d < 1", cfg->max_leaf_records); return PB200_E_INVALID; }
  if (M < 1 || !cfg->pairs) { set_error("star-tree config: no function-column pairs"); return PB200_E_INVALID; }
  for (int m = 0; m < M; m++) {
    const pb200h_agg& p = cfg->pairs[m];
    if (p.function != PB200_AGG_COUNT && p.function != PB200_AGG_SUM && p.function != PB200_AGG_MIN && p.function != PB200_AGG_MAX) {
      set_error("function-column pair %d: function %d has no star-tree metric here (COUNT, SUM, MIN, MAX)", m, p.function); return PB200_E_UNSUPPORTED;
    }
    if (p.function == PB200_AGG_COUNT ? (p.column && strcmp(p.column, "*") != 0) : !p.column) {
      set_error("function-column pair %d: COUNT takes '*', SUM / MIN / MAX a column", m); return PB200_E_INVALID;
    }
  }
  if (!ctx || !seg || !seg->dev) { set_error("invalid argument to pb200h_startree_build"); return PB200_E_INVALID; }
  if (seg->dev->domain) { set_error("segment is bound to a dictionary domain: star-tree dimension ids would not match"); return PB200_E_UNSUPPORTED; }
  if (seg->num_docs <= 0) { set_error("segment '%s' has no docs", seg->name.c_str()); return PB200_E_UNSUPPORTED; }
  pb200::StarBuildSpec spec;
  spec.skip_star = skip;
  spec.max_leaf_records = cfg->max_leaf_records;
  std::unique_ptr<StarTreeIndex> st(new StarTreeIndex());
  for (int j = 0; j < D; j++) {
    const int bc = seg->column_index(cfg->dimensions[j]);
    if (bc < 0) { set_error("star-tree dimension '%s': no such column", cfg->dimensions[j]); return PB200_E_INVALID; }
    if (seg->cols[bc].derived) { set_error("star-tree dimension '%s' is a derived column", cfg->dimensions[j]); return PB200_E_UNSUPPORTED; }
    const pb200::DeviceColumn& dc = seg->dev->cols[bc];
    if (!seg->cols[bc].has_dictionary || dc.fwd_kind != PB200_FWD_DICT_FIXEDBIT || dc.bits > 31) {
      set_error("star-tree dimension '%s' has no dictIds (a raw column streamed as 32-bit values)", cfg->dimensions[j]); return PB200_E_UNSUPPORTED;
    }
    spec.dim_cols.push_back(bc);
    st->dim_base_col.push_back(bc);
  }
  std::vector<std::string> metric_names;
  for (int m = 0; m < M; m++) {
    const pb200h_agg& p = cfg->pairs[m];
    int bc = -1;
    if (p.function != PB200_AGG_COUNT) {
      bc = seg->column_index(p.column);
      if (bc < 0) { set_error("function-column pair %d: no column '%s'", m, p.column); return PB200_E_INVALID; }
      if (seg->cols[bc].derived) { set_error("function-column pair %d: '%s' is a derived column", m, p.column); return PB200_E_UNSUPPORTED; }
      if (seg->cols[bc].data_type == PB200_STRING) { set_error("function-column pair %d: '%s' is a STRING column", m, p.column); return PB200_E_UNSUPPORTED; }
    }
    spec.metric_fn.push_back(p.function);
    spec.metric_col.push_back(bc);
    st->metric_fn.push_back(p.function);
    st->metric_base_col.push_back(bc);
    metric_names.push_back(lower_fn_name(p.function) + "__" + (bc < 0 ? "*" : p.column));
  }
  pb200::StarBuildResult res;
  if (int rc = pb200::startree_build(ctx, seg->dev, spec, &res)) return rc;
  // the star docs: the host side of their segment (dimensions keep the base columns' dictionaries)
  std::unique_ptr<pb200h_segment> docs(new pb200h_segment());
  docs->ctx = ctx; docs->dev = res.docs; docs->name = seg->name + "$startree"; docs->num_docs = res.docs->num_docs;
  docs->cols.reserve((size_t)D + M + PB200_MAX_DERIVED_COLUMNS);
  for (int j = 0; j < D; j++) {
    HostColumn h = seg->cols[spec.dim_cols[j]];
    h.bits = res.docs->cols[j].bits; h.is_sorted = 0; h.has_inverted = false; h.sorted_idx.clear();
    docs->cols.push_back(std::move(h));
  }
  for (int m = 0; m < M; m++) {
    const pb200::DeviceColumn& dc = res.docs->cols[D + m];
    HostColumn h;
    h.name = metric_names[m];
    h.data_type = dc.stored_type; h.has_dictionary = 1; h.bits = dc.bits; h.cardinality = dc.cardinality; h.entry_bytes = 8;
    h.dict = dc.dict_be;
    docs->cols.push_back(std::move(h));
  }
  docs->num_stored = D + M;
  docs->published.store(D + M, std::memory_order_release);
  st->star_segment = docs.release();
  st->num_docs = st->star_segment->num_docs;
  st->metric_limb_col = res.limb_col;
  // the tree: OffHeapStarTree layout, read back by the same parser as an attached tree
  std::vector<unsigned char> b(20);
  auto put32 = [&](size_t at, uint32_t v) { for (int k = 0; k < 4; k++) b[at + k] = (unsigned char)(v >> (8 * k)); };
  auto app32 = [&](uint32_t v) { b.resize(b.size() + 4); put32(b.size() - 4, v); };
  const uint64_t magic = 0xBADDA55B00DAD00Dull;
  put32(0, (uint32_t)magic); put32(4, (uint32_t)(magic >> 32)); put32(8, 1); put32(16, (uint32_t)D);
  for (int j = 0; j < D; j++) {
    const size_t len = strlen(cfg->dimensions[j]);
    app32((uint32_t)j); app32((uint32_t)len);
    b.insert(b.end(), cfg->dimensions[j], cfg->dimensions[j] + len);
  }
  const int num_nodes = (int)(res.nodes.size() / 7);
  app32((uint32_t)num_nodes);
  put32(12, (uint32_t)b.size());
  for (int32_t v : res.nodes) app32((uint32_t)v);
  if (!st->tree.parse(b.data(), b.size())) { set_error("star-tree build produced a tree the reader refuses"); return PB200_E_INVALID; }
  if (info) {
    memset(info, 0, sizeof *info);
    info->num_star_docs = st->num_docs; info->num_base_docs = res.num_base_docs; info->num_nodes = num_nodes;
    for (int p = 0; p < 4; p++) info->phase_ms[p] = res.ms[p];
  }
  seg->star_trees.push_back(std::move(st));
  return PB200_OK;
}

extern "C" int32_t pb200h_startree_get(const pb200h_segment* seg, int32_t index, const void** tree, uint64_t* tree_bytes,
                                       pb200h_segment** star_docs) {
  if (!seg || index < 0 || index >= (int)seg->star_trees.size()) { set_error("segment has no star-tree %d", index); return PB200_E_INVALID; }
  const StarTreeIndex& st = *seg->star_trees[index];
  if (tree) *tree = st.tree.bytes.data();
  if (tree_bytes) *tree_bytes = st.tree.bytes.size();
  if (star_docs) *star_docs = st.star_segment;
  return PB200_OK;
}

namespace pb200h {

StarTreeIndex::~StarTreeIndex() { if (star_segment) pb200h_segment_destroy(star_segment); }

// Fit test + execution.  Returns 1 when the star-tree answered (result set), 0 when the query does not fit, < 0 on error.
int try_star_tree(pb200_ctx* ctx, const pb200h_segment& seg, const StarTreeIndex& st, const pb200h_query& q,
                  pb200_result** out) {
  const int ndims = (int)st.dim_base_col.size();
  auto star_dim_of = [&](int base_col) { for (int d = 0; d < ndims; d++) if (st.dim_base_col[d] == base_col) return d; return -1; };
  // ---- filter: a single predicate or a flat AND of predicates, all on star-tree dimensions (StarTreeUtils) ----
  std::vector<int> leaves;
  if (q.num_filter_nodes > 0) {
    const pb200h_filter_node& root = q.filter[q.num_filter_nodes - 1];
    if (root.type >= PB200H_EQ) { if (q.num_filter_nodes != 1) return 0; leaves.push_back(0); }
    else if (root.type == PB200H_AND && root.num_children == q.num_filter_nodes - 1) {
      for (int i = 0; i + 1 < q.num_filter_nodes; i++) { if (q.filter[i].type < PB200H_EQ) return 0; leaves.push_back(i); }
    } else return 0;
  }
  std::vector<std::unique_ptr<std::vector<int32_t>>> owned(ndims);
  std::vector<const std::vector<int32_t>*> preds(ndims, nullptr);
  for (int li : leaves) {
    const pb200h_filter_node& n = q.filter[li];
    const int bc = seg.column_index(n.column);
    const int d = bc < 0 ? -1 : star_dim_of(bc);
    if (d < 0) return 0;
    std::vector<int32_t> ids = matching_dict_ids(seg.cols[bc], n, q.literals);
    if (!owned[d]) owned[d].reset(new std::vector<int32_t>(std::move(ids)));
    else {
      std::vector<int32_t> both;
      std::set_intersection(owned[d]->begin(), owned[d]->end(), ids.begin(), ids.end(), std::back_inserter(both));
      *owned[d] = std::move(both);
    }
    preds[d] = owned[d].get();
  }
  uint32_t gb_mask = 0;
  std::vector<int32_t> gb_cols;
  for (int g = 0; g < q.num_group_by; g++) {
    const int bc = seg.column_index(q.group_by[g]);
    const int d = bc < 0 ? -1 : star_dim_of(bc);
    if (d < 0) return 0;
    gb_mask |= 1u << d;
    gb_cols.push_back(d);  // star segment column index == dimension index
  }
  // ---- aggregations -> function-column pairs ----
  auto metric_of = [&](int fn, int base_col) { for (size_t m = 0; m < st.metric_fn.size(); m++) if (st.metric_fn[m] == fn && st.metric_base_col[m] == base_col) return (int)m; return -1; };
  // internal aggregations over star segment columns, each once however many of the query's aggregations read it
  std::vector<pb200_agg> star_aggs;
  auto internal = [&](int fn, int col) {
    for (size_t i = 0; i < star_aggs.size(); i++) if (star_aggs[i].function == fn && star_aggs[i].column == col) return (int)i;
    star_aggs.push_back({fn, col});
    return (int)star_aggs.size() - 1;
  };
  // a0: the value (MIN / MAX / a SUM of the metric's column), a1: AVG's count, limb: the first of three consecutive
  // limb sums that replace a0 for a built tree's INT SUM (the exact sum, rounded once)
  struct Map { int fn; int a0, a1, limb; };
  std::vector<Map> mapping;
  for (int a = 0; a < q.num_aggs; a++) {
    const int fn = q.aggs[a].function;
    Map m{fn, -1, -1, -1};
    if (fn == PB200_AGG_COUNT) {
      const int c = metric_of(PB200_AGG_COUNT, -1);
      if (c < 0) return 0;
      m.a0 = internal(PB200_AGG_SUM, ndims + c);
    } else if (fn == PB200_AGG_SUM || fn == PB200_AGG_MIN || fn == PB200_AGG_MAX || fn == PB200_AGG_AVG) {
      const int bc = seg.column_index(q.aggs[a].column);
      const int sfn = fn == PB200_AGG_AVG ? PB200_AGG_SUM : fn;
      const int c = bc < 0 ? -1 : metric_of(sfn, bc);
      if (c < 0) return 0;
      const int limb = sfn == PB200_AGG_SUM && c < (int)st.metric_limb_col.size() ? st.metric_limb_col[c] : -1;
      if (limb >= 0) {   // the three are only ever added together, so they stay consecutive
        m.limb = internal(PB200_AGG_SUM, limb);
        internal(PB200_AGG_SUM, limb + 1);
        internal(PB200_AGG_SUM, limb + 2);
      } else {
        m.a0 = internal(sfn, ndims + c);
      }
      if (fn == PB200_AGG_AVG) {
        const int cc = metric_of(PB200_AGG_COUNT, -1);
        if (cc < 0) return 0;
        m.a1 = internal(PB200_AGG_SUM, ndims + cc);
      }
    } else return 0;
    mapping.push_back(m);
  }
  if ((int)star_aggs.size() > 6) return 0;
  // a limb-summed INT SUM: l2 * 2^42 + l1 * 2^21 + l0 in 128 bits (each limb sum is an integer below 2^52, exact in
  // double).  The total is the rows' exact sum, |S| <= 2^31 rows x 2^31, so it fits int64 and is rounded to double
  // once: float(exact sum), as the scan returns it
  auto limb_sum = [](const double* l0, const double* l1, const double* l2, size_t r) {
    const __int128 s = (__int128)(long long)l2[r] * ((__int128)1 << 42) + (__int128)(long long)l1[r] * (1 << 21) + (long long)l0[r];
    return (double)(long long)s;
  };

  // ---- traversal -> doc mask (cached per predicate set) ----
  const int sdocs = st.num_docs;
  std::string key(reinterpret_cast<const char*>(&gb_mask), sizeof gb_mask);
  for (int d = 0; d < ndims; d++) {
    const int32_t n = preds[d] ? (int32_t)preds[d]->size() : -1;
    key.append(reinterpret_cast<const char*>(&n), sizeof n);
    if (n > 0) key.append(reinterpret_cast<const char*>(preds[d]->data()), (size_t)n * 4);
  }
  std::shared_ptr<const StarTreeIndex::Traversal> tr;
  {
    std::lock_guard<std::mutex> g(st.cache_mu);
    for (auto& e : st.cache) if (e->key == key) { tr = e; break; }
  }
  if (!tr) {
    auto fresh = std::make_shared<StarTreeIndex::Traversal>();
    fresh->key = std::move(key);
    std::vector<std::pair<int32_t, int32_t>> docs;
    const bool non_empty = st.tree.traverse(preds, gb_mask, docs, fresh->remaining);
    fresh->mask.assign(((size_t)sdocs + 31) / 32 + 1, 0u);
    std::vector<uint32_t>& mask = fresh->mask;
    if (non_empty) {
      for (auto [s, e] : docs) {  // word-wise fill of [s, e)
        s = std::max(s, 0); e = std::min(e, sdocs);
        if (s >= e) continue;
        const int ws = s >> 5, we = (e - 1) >> 5;
        const uint32_t first = 0xFFFFFFFFu << (s & 31), last = 0xFFFFFFFFu >> (31 - ((e - 1) & 31));
        if (ws == we) mask[ws] |= first & last;
        else { mask[ws] |= first; for (int w = ws + 1; w < we; w++) mask[w] = 0xFFFFFFFFu; mask[we] |= last; }
      }
    }
    if (pb200_doc_mask_upload(ctx, sdocs, fresh->mask.data(), (int64_t)fresh->mask.size(), &fresh->dev_mask) == PB200_OK) fresh->ctx = ctx;
    else fresh->dev_mask = nullptr;  // the per-query upload still works
    tr = fresh;
    std::lock_guard<std::mutex> g(st.cache_mu);
    st.cache.push_back(tr);
    if (st.cache.size() > 8) st.cache.pop_front();
  }
  const std::vector<uint32_t>& mask = tr->mask;
  const uint32_t remaining = tr->remaining;

  // ---- device query on the star-tree segment: DOC_MASK AND remaining predicates ----
  std::vector<pb200_filter_node> nodes;
  SegmentFilterStore store;
  pb200_filter_node mn;
  memset(&mn, 0, sizeof mn);
  mn.op = PB200_F_DOC_MASK; mn.column = -1; mn.ids = (const int32_t*)mask.data(); mn.num_ids = (int32_t)mask.size();
  if (tr->dev_mask) { mn.ids = (const int32_t*)tr->dev_mask; mn.reserved = PB200_NODE_IDS_ON_DEVICE; }
  nodes.push_back(mn);
  int extra = 0;
  for (int li : leaves) {
    const pb200h_filter_node& n = q.filter[li];
    const int d = star_dim_of(seg.column_index(n.column));
    if (!((remaining >> d) & 1)) continue;
    pb200_filter_node dn;
    if (n.type == PB200H_REGEXP_LIKE)   // the star docs' dimension shares the base column's dictionary, so its ids
      pattern_alias(seg.cols[seg.column_index(n.column)], st.star_segment->cols[d], q.literals[n.values_offset].s);
    int rc = leaf_to_device(*st.star_segment, d, n, q.literals, store, dn);
    if (rc) return rc;
    nodes.push_back(dn);
    extra++;
  }
  if (extra) { pb200_filter_node an; memset(&an, 0, sizeof an); an.op = PB200_F_AND; an.num_children = extra + 1; nodes.push_back(an); }
  pb200_query dq;
  memset(&dq, 0, sizeof dq);
  dq.num_filter_nodes = (int)nodes.size();
  dq.num_group_by = q.num_group_by;
  dq.num_aggs = (int)star_aggs.size();
  dq.num_groups_limit = q.num_groups_limit > 0 ? q.num_groups_limit : 100000;
  dq.max_initial_result_holder_capacity = q.max_initial_result_holder_capacity > 0 ? q.max_initial_result_holder_capacity : 10000;
  dq.filter = nodes.data(); dq.group_by_columns = gb_cols.data(); dq.aggs = star_aggs.data();
  pb200_segment* dev = st.star_segment->dev;
  pb200_result* sr = nullptr;
  int rc = pb200_execute(ctx, &dq, &dev, 1, &sr);
  if (rc == PB200_E_UNSUPPORTED) return 0;   // the star docs' row is too wide for the scan (limb columns): scan the base
  if (rc) return rc;
  // ---- back to the query's own aggregation list ----
  std::unique_ptr<pb200_result> R(new pb200_result());
  R->meta = sr->meta;
  R->meta.num_aggs = q.num_aggs;
  R->meta.num_total_docs = seg.num_docs;
  const size_t rows = sr->meta.num_groups < 0 ? 1 : (size_t)sr->meta.num_groups;
  R->dbl.resize(q.num_aggs); R->lng.resize(q.num_aggs); R->ids.resize(q.num_aggs); R->distinct.resize(q.num_aggs);
  if (sr->view.block) {
    // extracted groups sit in a pinned block in their final column layout: the remap is a re-pointing of columns that
    // shares the block (no 2 x rows x 20 B copy per aggregation -- at 1 M groups that copy cost more than the scan);
    // only the COUNT / AVG row counts (star-tree COUNT metric sums, exact in double) get a column of their own
    const pb200_result::View& sv = sr->view;
    pb200_result::View& v = R->view;
    v.block = sv.block; v.rows = sv.rows; v.keys = sv.keys;
    std::vector<double> zeros;
    for (int a = 0; a < q.num_aggs; a++) {
      const Map& m = mapping[a];
      if (m.limb >= 0) {   // a column of its own, owned by the result
        const double* l[3];
        for (int k = 0; k < 3; k++) {
          l[k] = sv.dbl[m.limb + k];
          if (!l[k]) { zeros.assign(rows, 0.0); l[k] = zeros.data(); }
        }
        R->dbl[a].resize(rows);
        for (size_t r = 0; r < rows; r++) R->dbl[a][r] = limb_sum(l[0], l[1], l[2], r);
        v.dbl[a] = R->dbl[a].data();
      } else {
        v.dbl[a] = sv.dbl[m.a0];
      }
      v.ids[a] = nullptr;   // all -1: star-tree metrics are raw values
      const int src = m.fn == PB200_AGG_COUNT ? m.a0 : m.fn == PB200_AGG_AVG ? m.a1 : -1;
      if (src >= 0 && sv.dbl[src]) {
        // row counts = sums of the star-tree COUNT metric: non-negative integers, exact in double.  The SUM's own (unused)
        // long column inside the pinned block takes them -- no allocation, no libm call per row
        const double* d = sv.dbl[src];
        int64_t* l = const_cast<int64_t*>(sv.lng[src]);
        if (!l) { R->lng[a].resize(rows); l = R->lng[a].data(); }
        for (size_t r = 0; r < rows; r++) l[r] = (int64_t)(d[r] + 0.5);
        v.lng[a] = l;
      }
    }
  } else {
    R->keys = sr->keys;
    for (int a = 0; a < q.num_aggs; a++) {
      const Map& m = mapping[a];
      if (m.limb >= 0) {
        R->dbl[a].resize(rows);
        for (size_t r = 0; r < rows; r++) R->dbl[a][r] = limb_sum(sr->dbl[m.limb].data(), sr->dbl[m.limb + 1].data(), sr->dbl[m.limb + 2].data(), r);
      } else {
        R->dbl[a] = sr->dbl[m.a0];
      }
      R->lng[a].assign(rows, 0);
      R->ids[a].assign(rows, -1);
      for (size_t r = 0; r < rows; r++) {
        if (m.fn == PB200_AGG_COUNT) { R->lng[a][r] = (int64_t)std::llround(sr->dbl[m.a0][r]); R->dbl[a][r] = (double)R->lng[a][r]; }
        else if (m.fn == PB200_AGG_AVG) R->lng[a][r] = (int64_t)std::llround(sr->dbl[m.a1][r]);
      }
    }
  }
  pb200_result_free(sr);
  *out = R.release();
  return 1;
}

}  // namespace pb200h
