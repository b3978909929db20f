// expr_filter_probe.cpp -- TEST shim for predicates on multi-column expressions (DESIGN.md section 3.16): the
// __host__ __device__ comparison the doc-mask pass runs (pinot_b200/csrc/pb200_expr.h) and pb200h_explain over a host-only
// segment, without a GPU.  Built by tests/test_expr_filter_cpu.py with g++ against the in-tree library.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../pinot_b200/csrc/host/host_internal.h"
#include "../../pinot_b200/csrc/pb200_expr.h"

extern "C" {

// pb200::expr_matches on n values of x: out[k] = 1 when x[k] matches
void efp_matches(int32_t op, int32_t flags, double lo, double hi, const double* values, int32_t nvalues, const double* x, int32_t n,
                 uint8_t* out) {
  for (int k = 0; k < n; k++) out[k] = pb200::expr_matches(op, flags, lo, hi, values, nvalues, x[k]) ? 1 : 0;
}

// 1 when a filter leaf on `text` is evaluated per row (an expression over two or more distinct columns)
int32_t efp_is_expression_filter(const char* text) { return pb200h::is_expression_filter(text) ? 1 : 0; }

// pb200h_explain over a HOST-ONLY segment (no device registration), as tests/host_probe does
int32_t efp_explain(const pb200h_column* cols, int32_t ncols, int32_t num_docs, const pb200h_query* q, char* out, int32_t cap) {
  pb200h_segment seg;
  seg.num_docs = num_docs;
  seg.num_stored = ncols;
  for (int i = 0; i < ncols; i++) {
    const pb200h_column& c = cols[i];
    pb200h::HostColumn h;
    h.name = c.name ? c.name : "";
    h.data_type = c.data_type; h.has_dictionary = c.has_dictionary; h.bits = c.bits_per_value;
    h.cardinality = c.cardinality; h.is_sorted = c.is_sorted; h.entry_bytes = c.dict_entry_bytes;
    h.has_inverted = c.inv != nullptr && c.inv_bytes > 0 && !c.is_sorted;
    if (c.dict && c.dict_bytes) h.dict.assign((const unsigned char*)c.dict, (const unsigned char*)c.dict + c.dict_bytes);
    if (c.is_sorted && c.fwd) h.sorted_idx.assign((const unsigned char*)c.fwd, (const unsigned char*)c.fwd + c.fwd_bytes);
    seg.cols.push_back(std::move(h));
  }
  return pb200h_explain(nullptr, q, &seg, out, cap);
}

}  // extern "C"
