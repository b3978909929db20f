// hll_probe.cpp -- TEST shim: the DISTINCTCOUNTHLL hash, offer step and estimate (pinot_b200/csrc/pb200_hll.h, the same
// code the device runs) on the CPU.  Built by tests/test_hll_cpu.py with g++.
#include <cstdint>
#include <vector>

#include "../../pinot_b200/csrc/pb200_hll.h"

extern "C" {

uint32_t hp_hash_long(uint64_t v) { return pb200::hll_hash_long(v); }
uint32_t hp_hash_bytes(const unsigned char* b, int32_t len, uint32_t seed) { return pb200::hll_hash_bytes(b, len, seed); }
uint32_t hp_hash_value(int32_t stored_type, uint64_t raw) { return pb200::hll_hash_value(stored_type, raw); }
int32_t hp_utf8_valid(const unsigned char* b, int32_t len) { return pb200::hll_utf8_valid(b, len) ? 1 : 0; }
double hp_alpha_mm(int32_t p) { return pb200::hll_alpha_mm(p); }
void hp_linear_table(int32_t p, long long* out) { pb200::hll_linear_table(p, out); }

// the estimate of the registers the hashes give, through the finalize's steps: offer, scaled sum and zeros, estimate
int64_t hp_estimate(const uint32_t* hashes, int64_t n, int32_t p) {
  std::vector<uint32_t> reg((size_t)1 << p, 0);
  for (int64_t i = 0; i < n; i++) {
    const uint32_t j = pb200::hll_index(hashes[i], p), r = pb200::hll_rank(hashes[i], p);
    if (r > reg[j]) reg[j] = r;
  }
  unsigned long long s = 0;
  uint32_t z = 0;
  for (uint32_t r : reg) { s += pb200::hll_term(r, p); z += r == 0; }
  std::vector<long long> linear(reg.size() + 1);
  pb200::hll_linear_table(p, linear.data());
  return pb200::hll_estimate(s, z, p, pb200::hll_alpha_mm(p), linear.data());
}

}  // extern "C"
