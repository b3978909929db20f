// The descriptors of pinot_b200/csrc/pb200_aggfn.h, one field per call, for tests/test_aggfn_cpu.py.
#include "../../pinot_b200/csrc/pb200_aggfn.h"

extern "C" {
int ap_known(int fn) { return pb200::agg_fn(fn) != nullptr; }
const char* ap_name(int fn) { return pb200::agg_fn(fn)->name; }
const char* ap_family(int fn) { return pb200::agg_fn(fn)->family; }
int ap_arg(int fn) { return pb200::agg_fn(fn)->arg; }
int ap_dict_ids(int fn) { return pb200::agg_fn(fn)->dict_ids; }
}
