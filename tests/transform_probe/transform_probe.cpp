// transform_probe.cpp -- TEST shim: the host layer's expression compiler (pinot_b200/csrc/host/transform.cpp) and the
// __host__ __device__ evaluator the derivation kernel runs (pinot_b200/csrc/pb200_transform.h), without a GPU.  Built by
// tests/test_transform_cpu.py with g++ against the in-tree library.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../pinot_b200/csrc/host/host_internal.h"
#include "../../pinot_b200/csrc/pb200_transform.h"

extern "C" {

// text -> canonical text (into `canonical`, NUL terminated) and the number of program ops; < 0: the PB200_E_* code
int32_t tp_compile(const char* text, char* canonical, int32_t cap) {
  std::string c, col;
  std::vector<pb200_transform_op> ops;
  const int rc = pb200h::compile_expression(text, &c, &ops, &col);
  if (rc) return rc;
  snprintf(canonical, (size_t)cap, "%s", c.c_str());
  return (int32_t)ops.size();
}

// Compiles `text` for a source column of `source_type`, checks the program and evaluates it on n values (integral
// sources read si, floating ones sd).  kind: the result's PB200_* type.  ok[k] = 0 where the value is refused (beyond
// +-2^53 ms).  Returns 0 or the PB200_E_* code of the compile / check.
int32_t tp_eval(const char* text, int32_t source_type, int32_t n, const int64_t* si, const double* sd, int32_t* kind,
                int64_t* oi, double* od, uint64_t* key, int32_t* ok) {
  std::string c, col;
  std::vector<pb200_transform_op> ops;
  int rc = pb200h::compile_expression(text, &c, &ops, &col);
  if (rc) return rc;
  const char* why = "";
  rc = pb200::transform_check(ops.data(), (int)ops.size(), source_type, kind, &why);
  if (rc) return rc;
  for (int k = 0; k < n; k++) {
    oi[k] = 0;
    od[k] = 0.0;
    ok[k] = pb200::transform_eval(ops.data(), (int)ops.size(), source_type, si ? si[k] : 0, sd ? sd[k] : 0.0, &oi[k], &od[k]);
    key[k] = pb200::transform_key(*kind, oi[k], od[k]);
  }
  return 0;
}

}  // extern "C"
