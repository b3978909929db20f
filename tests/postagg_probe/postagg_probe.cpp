// postagg_probe.cpp -- TEST shim: the post-aggregation evaluator of pinot_b200/csrc/pb200_postagg.h (the code the device
// order pass and the host order run) compiled with g++, so that CPU tests can hold it to Python floats.  Built by
// tests/test_postagg_cpu.py; nothing here ships.
#include <cstdint>

#include "../../pinot_b200/csrc/pb200_having.h"
#include "../../pinot_b200/csrc/pb200_postagg.h"

extern "C" {

// 0 when the program is well formed over num_aggs aggregations, 1 otherwise
int32_t probe_postagg_validate(const pb200_post_program* p, int32_t num_aggs) { return pb200::postagg_validate(p, num_aggs) ? 1 : 0; }

// out[r] = the program's value for row r; dv / lv = the rows' double and long columns, [rows x num_aggs]
void probe_postagg_eval(const pb200_post_program* p, int32_t num_aggs, const int32_t* fns, const double* dv, const int64_t* lv,
                        int64_t rows, double* out) {
  for (int64_t r = 0; r < rows; r++)
    out[r] = pb200::postagg_eval(*p, [&](int a) { return pb200::having_value(fns[a], dv[r * num_aggs + a], lv[r * num_aggs + a]); });
}

}  // extern "C"
