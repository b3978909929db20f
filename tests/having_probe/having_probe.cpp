// having_probe.cpp -- TEST shim: the HAVING predicate of pinot_b200/csrc/pb200_having.h (the code the device keep kernel
// and the host filter run) compiled with g++, so that CPU tests can hold it to a Python reference.  Built by
// tests/test_having_cpu.py; nothing here ships.
#include <cstdint>

#include "../../pinot_b200/csrc/pb200_having.h"

extern "C" {

// 0 when the tree is well formed over num_aggs aggregations, 1 otherwise
int32_t probe_having_validate(const pb200_having* h, int32_t num_aggs) { return pb200::having_validate(h, num_aggs) ? 1 : 0; }

// out[r] = the tree's outcome for row r; dv / lv = the rows' double and long columns, [rows x num_aggs]
void probe_having_eval(const pb200_having* h, int32_t num_aggs, const int32_t* fns, const double* dv, const int64_t* lv,
                       int64_t rows, uint8_t* out) {
  for (int64_t r = 0; r < rows; r++)
    out[r] = pb200::having_eval(*h, [&](int a) { return pb200::having_value(fns[a], dv[r * num_aggs + a], lv[r * num_aggs + a]); });
}

}  // extern "C"
