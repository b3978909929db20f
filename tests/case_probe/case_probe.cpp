// case_probe.cpp -- TEST shim: CASE WHEN (DESIGN.md section 3.19) without a GPU -- the host compiler of
// pinot_b200/csrc/host/transform.cpp, the condition resolution of host/case_expr.cpp over a dictionary built here, and
// the __host__ __device__ check and evaluator of pinot_b200/csrc/pb200_expr.h.  Built by tests/test_case_cpu.py with g++
// against the in-tree library.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../pinot_b200/csrc/host/host_internal.h"
#include "../../pinot_b200/csrc/pb200_expr.h"

extern "C" {

// text -> canonical text; returns the number of program entries (< 0: the PB200_E_* code), the value leaves and the
// conditions in *nleaves / *nconds
int32_t cp_compile(const char* text, char* canonical, int32_t cap, int32_t* nleaves, int32_t* nconds) {
  std::string c;
  std::vector<pb200_transform_op> ops;
  std::vector<std::string> names;
  std::vector<pb200h::CaseCond> conds;
  const int rc = pb200h::compile_multi_expression(text, &c, &ops, &names, &conds);
  if (rc) return rc;
  snprintf(canonical, (size_t)cap, "%s", c.c_str());
  *nleaves = (int32_t)names.size();
  *nconds = (int32_t)conds.size();
  return (int32_t)ops.size();
}

// compile_multi_expression without a condition list (the callers that refuse CASE)
int32_t cp_compile_plain(const char* text) {
  std::string c;
  std::vector<pb200_transform_op> ops;
  std::vector<std::string> names;
  return pb200h::compile_multi_expression(text, &c, &ops, &names);
}

int32_t cp_is_multi(const char* text) { return pb200h::is_multi_column_expression(text) ? 1 : 0; }
int32_t cp_is_filter(const char* text) { return pb200h::is_expression_filter(text) ? 1 : 0; }

// Compiles `text`, checks it and evaluates it on n rows.  Value leaf k of row r is ints[r * nleaves + k] (as a double)
// when integral[k], else dbls[r * nleaves + k]; row r's condition word is cond[r].  0 or the PB200_E_* code.
int32_t cp_eval(const char* text, int32_t n, int32_t nleaves, const int32_t* integral, const int64_t* ints, const double* dbls,
                const uint32_t* cond, double* out) {
  std::string c;
  std::vector<pb200_transform_op> ops;
  std::vector<std::string> names;
  std::vector<pb200h::CaseCond> conds;
  int rc = pb200h::compile_multi_expression(text, &c, &ops, &names, &conds);
  if (rc) return rc;
  const char* why = "";
  int leaves = 0;
  if ((rc = pb200::expr_check(ops.data(), (int)ops.size(), &leaves, &why, (int)conds.size()))) return rc;
  if ((int)names.size() != nleaves) return PB200_E_INVALID;
  std::vector<double> v((size_t)nleaves + 1);
  for (int r = 0; r < n; r++) {
    for (int k = 0; k < nleaves; k++) v[k] = integral[k] ? (double)ints[(size_t)r * nleaves + k] : dbls[(size_t)r * nleaves + k];
    out[r] = pb200::expr_eval<true>(ops.data(), (int)ops.size(), v.data(), cond[r]);
  }
  return 0;
}

// expr_check on a raw program with `nconds` conditions; its code, the leaves in *leaves
int32_t cp_check(const pb200_transform_op* ops, int32_t n, int32_t nconds, int32_t* leaves) {
  const char* why = "";
  int l = 0;
  const int rc = pb200::expr_check(ops, n, &l, &why, nconds);
  *leaves = l;
  return rc;
}

// The local dictIds the first condition of `text` matches on a dictionary column of `type` whose sorted values are
// ints / dbls / strs[0 .. card); `flags` bit0: synthesised at load, bit1: no dictionary.  Returns the count (ids in out) or
// the PB200_E_* code.
int32_t cp_ids(const char* text, int32_t type, int32_t card, const int64_t* ints, const double* dbls, const char* const* strs,
               int32_t flags, int32_t* out) {
  std::string canon;
  std::vector<pb200_transform_op> ops;
  std::vector<std::string> names;
  std::vector<pb200h::CaseCond> conds;
  if (int rc = pb200h::compile_multi_expression(text, &canon, &ops, &names, &conds)) return rc;
  if (conds.empty()) return PB200_E_INVALID;
  pb200h::HostColumn c;
  c.name = conds[0].column;
  c.data_type = type; c.cardinality = card; c.has_dictionary = !(flags & 2); c.synthesized_dictionary = flags & 1;
  c.entry_bytes = type == PB200_STRING ? 16 : (type == PB200_LONG || type == PB200_DOUBLE) ? 8 : 4;
  c.dict.assign((size_t)card * c.entry_bytes, 0);
  for (int k = 0; k < card; k++) {
    unsigned char* p = c.dict.data() + (size_t)k * c.entry_bytes;
    uint64_t u = 0;
    switch (type) {
      case PB200_INT: u = (uint32_t)(int32_t)ints[k]; break;
      case PB200_LONG: u = (uint64_t)ints[k]; break;
      case PB200_FLOAT: { const float f = (float)dbls[k]; uint32_t w; memcpy(&w, &f, 4); u = w; break; }
      case PB200_DOUBLE: memcpy(&u, &dbls[k], 8); break;
      default: strncpy((char*)p, strs[k], 16); continue;
    }
    for (int b = 0; b < c.entry_bytes; b++) p[b] = (unsigned char)(u >> (8 * (c.entry_bytes - 1 - b)));
  }
  std::vector<int32_t> ids;
  if (int rc = pb200h::case_condition_ids(c, conds[0], &ids)) return rc;
  std::copy(ids.begin(), ids.end(), out);
  return (int32_t)ids.size();
}

// the REGEXP_LIKE pattern of like(x,'<like>'); -1 for a refused pattern
int32_t cp_like(const char* like, char* out, int32_t cap) {
  pb200h::CaseCond cc;
  cc.fn = "like";
  cc.literals.push_back(like);
  std::string re;
  if (!pb200h::case_pattern(cc, &re)) return -1;
  snprintf(out, (size_t)cap, "%s", re.c_str());
  return 0;
}

}  // extern "C"
