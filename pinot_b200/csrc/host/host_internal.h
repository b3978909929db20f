// host_internal.h -- shared declarations of the native host layer (plan_maker.cpp, star_tree.cpp).
#pragma once
#include <cmath>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../../include/pinot_b200_host.h"
#include "../pb200_internal.h"

namespace pb200h {
using pb200::set_error;

inline uint32_t hbe32(const unsigned char* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
inline uint64_t hbe64(const unsigned char* p) { return (uint64_t)hbe32(p) << 32 | hbe32(p + 4); }

// Stored INT / LONG value vs a predicate literal, by exact numeric value (-1, 0, 1).  `d` is the literal rounded to
// double; when it is an int64, `i` holds it exactly and (double)i == d.  Otherwise a fractional `d` is the literal
// itself (it equals no integer) and an integral or infinite one lies beyond the int64 range on its side.  This is what
// the reference's broker (NumericalFilterOptimizer) makes of `intCol >= 2.5` or `longCol < 1e19` before a server sees
// them.
inline int compare_integral(int64_t v, const pb200h_literal& l) {
  if ((double)l.i == l.d) return v < l.i ? -1 : v > l.i;
  if (std::isfinite(l.d) && l.d != std::floor(l.d)) return (double)v < l.d ? -1 : 1;   // |d| < 2^52: rounding v keeps its side
  return l.d > 0 ? -1 : 1;
}

struct HostColumn {
  std::string name;
  int data_type = 0, has_dictionary = 0, bits = 0, cardinality = 0, is_sorted = 0, entry_bytes = 0;
  bool has_inverted = false;
  bool synthesized_dictionary = false;    // the segment stores this column raw: `dict` was built from its values at load (raw_forward.cpp)
  std::vector<unsigned char> dict;        // big-endian values or padded strings (host copy): the SEGMENT's own dictionary
  std::vector<unsigned char> sorted_idx;  // (start,end) BE pairs when is_sorted
  // Bound to a table-wide dictionary domain (pb200h_segment_bind_domain): predicates are still resolved against the
  // segment's own dictionary above (same alwaysTrue / alwaysFalse / index decisions as the reference), then ids are
  // translated with local_ids; everything the device returns for this column is a DOMAIN id, decoded through `global`.
  std::vector<int32_t> local_ids;               // local dictId -> domain id (ascending); empty = unbound
  std::shared_ptr<const HostColumn> global;     // the domain's dictionary as a column (dict, cardinality, bits, entry_bytes)
  int to_device_id(int local) const { return local_ids.empty() ? local : local_ids[local]; }
  const HostColumn& decode_column() const { return global ? *global : *this; }

  int32_t get_int(int id) const { return (int32_t)hbe32(dict.data() + 4ull * id); }
  int64_t get_long(int id) const { return (int64_t)hbe64(dict.data() + 8ull * id); }
  float get_float(int id) const { uint32_t u = hbe32(dict.data() + 4ull * id); float f; memcpy(&f, &u, 4); return f; }
  double get_double(int id) const { uint64_t u = hbe64(dict.data() + 8ull * id); double d; memcpy(&d, &u, 8); return d; }
  std::string get_string(int id) const {
    const char* p = (const char*)dict.data() + (size_t)entry_bytes * id;
    size_t n = 0;
    while (n < (size_t)entry_bytes && p[n]) n++;
    return std::string(p, n);
  }
  double as_double(int id) const {
    switch (data_type) {
      case PB200_INT: return get_int(id);
      case PB200_LONG: return (double)get_long(id);
      case PB200_FLOAT: return get_float(id);
      case PB200_DOUBLE: return get_double(id);
      default: return NAN;
    }
  }
  // Dictionary.insertionIndexOf (BaseImmutableDictionary.java:124-139): >= 0 found, else -(insertion point) - 1
  int insertion_index_of(const pb200h_literal& l) const {
    int lo = 0, hi = cardinality - 1;
    while (lo <= hi) {
      int mid = (lo + hi) >> 1, cmp;
      switch (data_type) {
        case PB200_INT: cmp = compare_integral(get_int(mid), l); break;
        case PB200_LONG: cmp = compare_integral(get_long(mid), l); break;
        case PB200_FLOAT: { float v = get_float(mid), t = (float)l.d; cmp = v < t ? -1 : v > t; break; }
        case PB200_DOUBLE: { double v = get_double(mid); cmp = v < l.d ? -1 : v > l.d; break; }
        default: { int r = get_string(mid).compare(l.s ? l.s : ""); cmp = r < 0 ? -1 : r > 0; }
      }
      if (cmp < 0) lo = mid + 1; else if (cmp > 0) hi = mid - 1; else return mid;
    }
    return -(lo + 1);
  }
  int sorted_start(int id) const { return (int)hbe32(sorted_idx.data() + 8ull * id); }
  int sorted_end(int id) const { return (int)hbe32(sorted_idx.data() + 8ull * id + 4); }
};

// OffHeapStarTree: parsed header + node accessors (7 little-endian ints per node)
struct StarTree {
  std::vector<unsigned char> bytes;
  std::vector<std::string> dim_names;
  const unsigned char* nodes = nullptr;
  int num_nodes = 0;
  bool parse(const unsigned char* b, uint64_t len);
  int field(int n, int f) const { const unsigned char* p = nodes + 28ll * n + 4 * f; return (int)((uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24); }
  int dim_id(int n) const { return field(n, 0); }
  int dim_value(int n) const { return field(n, 1); }
  int start(int n) const { return field(n, 2); }
  int end(int n) const { return field(n, 3); }
  int agg_doc(int n) const { return field(n, 4); }
  int first_child(int n) const { return field(n, 5); }
  int last_child(int n) const { return field(n, 6); }
  bool is_leaf(int n) const { return first_child(n) == -1; }
  int num_children(int n) const { return is_leaf(n) ? 0 : last_child(n) - first_child(n) + 1; }
  int child_for_value(int n, int value) const;
  bool traverse(const std::vector<const std::vector<int32_t>*>& preds, uint32_t group_by_mask,
                std::vector<std::pair<int32_t, int32_t>>& docs,
                uint32_t& remaining_out) const;
};

}  // namespace pb200h

struct pb200h_segment;
namespace pb200h {
struct StarTreeIndex {
  StarTree tree;
  std::vector<int> dim_base_col;     // star dimension -> column index in the base segment
  std::vector<int> metric_fn;        // function of each function-column pair
  std::vector<int> metric_base_col;  // its column in the base segment (-1 for count__*)
  int num_docs = 0;
  pb200h_segment* star_segment = nullptr;  // columns: dimensions..., metrics...
  // Traversal results by (predicate dictId sets per dimension, group-by mask): the BFS over a tree with 10^5..10^6 nodes
  // costs more host time than the device scan of the docs it selects, and dashboards repeat their predicates.  The
  // tree is immutable, so an entry never goes stale; a handful of entries, oldest evicted first.
  struct Traversal {
    std::string key; std::vector<uint32_t> mask; uint32_t remaining = 0;
    pb200_ctx* ctx = nullptr; uint32_t* dev_mask = nullptr;   // the mask resident in HBM (pb200_doc_mask_upload): no per-query copy
    ~Traversal() { if (dev_mask) pb200_doc_mask_free(ctx, dev_mask); }
  };
  mutable std::mutex cache_mu;
  mutable std::deque<std::shared_ptr<const Traversal>> cache;
  ~StarTreeIndex();
};
}  // namespace pb200h

struct pb200h_segment {
  pb200_ctx* ctx = nullptr;
  pb200_segment* dev = nullptr;
  std::string name;
  int num_docs = 0;
  std::vector<pb200h::HostColumn> cols;
  std::vector<std::unique_ptr<pb200h::StarTreeIndex>> star_trees;
  int column_index(const char* n) const {
    if (!n) return -1;
    for (size_t i = 0; i < cols.size(); i++) if (cols[i].name == n) return (int)i;
    return -1;
  }
};

namespace pb200h {
// raw_forward.cpp: no-dictionary fixed-width SV forward indexes at load time
int raw_value_width(int data_type);
int decode_fixed_byte_forward(const unsigned char* file, uint64_t len, int width, int64_t num_docs, std::vector<unsigned char>& values_be);
void wrap_pass_through(const std::vector<unsigned char>& values_be, int width, int64_t num_docs, std::vector<unsigned char>& file);
bool synthesize_dictionary(const std::vector<unsigned char>& values_be, int data_type, int64_t num_docs, int max_cardinality,
                           std::vector<unsigned char>& dict_be, std::vector<unsigned char>& fwd_packed, int* cardinality, int* bits);
// filtered_agg.cpp: FILTER (WHERE ...) clauses = one device submission per distinct clause, aligned by group key
int execute_filtered(pb200_ctx* ctx, const pb200h_query& q, const pb200_order_by* order, pb200h_segment* const* segs, int nseg,
                     pb200_result** results, int32_t* kinds);
// ids[] storage that must outlive the pb200_execute call
struct SegmentFilterStore { std::vector<std::unique_ptr<std::vector<int32_t>>> ids; };
// PredicateEvaluator.getMatchingDictIds (sorted) of one predicate on a dictionary column
std::vector<int32_t> matching_dict_ids(const HostColumn& c, const pb200h_filter_node& n, const pb200h_literal* lits);
// one value-space predicate -> the device leaf FilterOperatorUtils.getLeafFilterOperator would build on `seg`.column
int leaf_to_device(const pb200h_segment& seg, int column, const pb200h_filter_node& n, const pb200h_literal* lits,
                   SegmentFilterStore& store, pb200_filter_node& out);
int try_star_tree(pb200_ctx* ctx, const pb200h_segment& seg, const StarTreeIndex& st, const pb200h_query& q,
                  pb200_result** out);
}  // namespace pb200h
