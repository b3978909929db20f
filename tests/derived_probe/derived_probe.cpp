// derived_probe.cpp -- TEST shim: predicate resolution (pb200h::matching_dict_ids / leaf_to_device) on a column marked
// as transform.cpp marks a derived column (derived = true, synthesized_dictionary = false), or as a stored / synthesised
// dictionary column for comparison, without a GPU.
// Built by tests/test_transform_edges_cpu.py with g++ against the in-tree library; nothing here ships.
#include <cstdint>
#include <vector>

#include "../../pinot_b200/csrc/host/host_internal.h"

extern "C" {

// derived / synthesized: the column's flags.  leaf = 0: matching_dict_ids -> ids (returns their count); leaf = 1:
// leaf_to_device -> out4 = {op, column, lo, hi} and ids = its payload (returns num_ids or a negative status)
int64_t probe_derived_leaf(int32_t data_type, int32_t derived, int32_t synthesized, const unsigned char* dict_be,
                           int32_t cardinality, int32_t num_docs, int32_t leaf, const pb200h_filter_node* node,
                           const pb200h_literal* literals, int32_t* out4, int32_t* ids, int64_t cap) {
  pb200h_segment seg;
  seg.num_docs = num_docs;
  pb200h::HostColumn h;
  h.name = node->column ? node->column : "";
  h.data_type = data_type; h.has_dictionary = 1; h.cardinality = cardinality;
  h.derived = derived != 0; h.synthesized_dictionary = synthesized != 0;
  h.entry_bytes = pb200h::raw_value_width(data_type);
  h.dict.assign(dict_be, dict_be + (size_t)cardinality * h.entry_bytes);
  if (!leaf) {
    std::vector<int32_t> m = pb200h::matching_dict_ids(h, *node, literals);
    for (size_t i = 0; i < m.size() && (int64_t)i < cap; i++) ids[i] = m[i];
    return (int64_t)m.size();
  }
  seg.cols.push_back(std::move(h));
  pb200h::SegmentFilterStore store;
  pb200_filter_node d;
  int rc = pb200h::leaf_to_device(seg, 0, *node, literals, store, d);
  if (rc) return rc;
  out4[0] = d.op; out4[1] = d.column; out4[2] = d.lo; out4[3] = d.hi;
  for (int i = 0; i < d.num_ids && i < cap; i++) ids[i] = d.ids[i];
  return d.num_ids;
}

}  // extern "C"
