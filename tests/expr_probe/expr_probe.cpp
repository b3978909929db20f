// expr_probe.cpp -- TEST shim: the host layer's multi-column expression compiler (pinot_b200/csrc/host/transform.cpp)
// and the __host__ __device__ evaluator the expression pass runs (pinot_b200/csrc/pb200_expr.h), without a GPU.  Built
// by tests/test_expr_cpu.py with g++ against the in-tree library.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../pinot_b200/csrc/host/host_internal.h"
#include "../../pinot_b200/csrc/pb200_expr.h"

extern "C" {

// text -> canonical text, the leaf column names joined by ',' and the number of ops; < 0: the PB200_E_* code
int32_t ep_compile(const char* text, char* canonical, char* leaves, int32_t cap) {
  std::string c;
  std::vector<pb200_transform_op> ops;
  std::vector<std::string> names;
  const int rc = pb200h::compile_multi_expression(text, &c, &ops, &names);
  if (rc) return rc;
  std::string joined;
  for (size_t k = 0; k < names.size(); k++) joined += (k ? "," : "") + names[k];
  snprintf(canonical, (size_t)cap, "%s", c.c_str());
  snprintf(leaves, (size_t)cap, "%s", joined.c_str());
  return (int32_t)ops.size();
}

// 1 when `text` takes the per-row route (a multi-column expression), else 0
int32_t ep_is_multi(const char* text) { return pb200h::is_multi_column_expression(text) ? 1 : 0; }

// the single-column compiler, to show it keeps its refusals
int32_t ep_compile_single(const char* text) {
  std::string c, col;
  std::vector<pb200_transform_op> ops;
  return pb200h::compile_expression(text, &c, &ops, &col);
}

// Compiles `text`, checks the program and evaluates it on n rows.  Leaf k of row r is ints[r * nleaves + k] converted to
// double when integral[k], else dbls[r * nleaves + k].  Returns 0 or the PB200_E_* code of the compile / check.
int32_t ep_eval(const char* text, int32_t n, int32_t nleaves, const int32_t* integral, const int64_t* ints, const double* dbls,
                double* out) {
  std::string c;
  std::vector<pb200_transform_op> ops;
  std::vector<std::string> names;
  int rc = pb200h::compile_multi_expression(text, &c, &ops, &names);
  if (rc) return rc;
  const char* why = "";
  int leaves = 0;
  if ((rc = pb200::expr_check(ops.data(), (int)ops.size(), &leaves, &why))) return rc;
  if (leaves != nleaves) return PB200_E_INVALID;
  std::vector<double> v((size_t)nleaves);
  for (int r = 0; r < n; r++) {
    for (int k = 0; k < nleaves; k++) v[k] = integral[k] ? (double)ints[(size_t)r * nleaves + k] : dbls[(size_t)r * nleaves + k];
    out[r] = pb200::expr_eval(ops.data(), (int)ops.size(), v.data());
  }
  return 0;
}

// expr_check on a raw program: returns its code, the number of leaves in *leaves
int32_t ep_check(const pb200_transform_op* ops, int32_t n, int32_t* leaves) {
  const char* why = "";
  int l = 0;
  const int rc = pb200::expr_check(ops, n, &l, &why);
  *leaves = l;
  return rc;
}

// the MIN / MAX accumulator's key of a double and the value a final key decodes to
uint64_t ep_key(double x) { return pb200::transform_key(pb200::TK_DOUBLE, 0, x); }
double ep_key_value(int32_t fn, uint64_t key) { return pb200::expr_key_value(fn, key); }

}  // extern "C"
