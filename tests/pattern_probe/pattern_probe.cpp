// pattern_probe.cpp -- TEST shim: the REGEXP_LIKE compiler and matcher of pinot_b200/csrc/pb200_pattern.h (the code the
// device kernel runs) compiled with g++, so that CPU tests can hold them to a Python reference.  Built by
// tests/test_pattern_cpu.py; nothing here ships.
#include <cstdint>
#include <cstring>
#include <string>

#include "../../pinot_b200/csrc/pb200_pattern.h"

extern "C" {

// PATTERN_OK / _UNSUPPORTED / _INVALID; the reason of a refusal in why (NUL terminated, at most cap bytes)
int32_t probe_pattern_compile(const char* pattern, char* why, int32_t cap) {
  static pb200::PatternAutomaton a;
  std::string w;
  const int rc = pb200::pattern_compile(pattern, &a, &w);
  if (why && cap > 0) { const size_t n = std::min<size_t>(w.size(), (size_t)cap - 1); memcpy(why, w.data(), n); why[n] = 0; }
  return rc;
}

// out[k] = 1 iff entry k (bytes [offsets[k], offsets[k + 1]) of data, up to its first NUL as the device's compact copy of
// a dictionary holds it) matches; returns the compile status
int32_t probe_pattern_match(const char* pattern, const unsigned char* data, const int64_t* offsets, int64_t n, uint8_t* out) {
  static pb200::PatternAutomaton a;
  const int rc = pb200::pattern_compile(pattern, &a, nullptr);
  if (rc != pb200::PATTERN_OK) return rc;
  for (int64_t k = 0; k < n; k++) {
    int len = 0;
    while (offsets[k] + len < offsets[k + 1] && data[offsets[k] + len]) len++;
    out[k] = pb200::pattern_match(a, data + offsets[k], len) ? 1 : 0;
  }
  return rc;
}

}  // extern "C"
