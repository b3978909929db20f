// probe: `sub.cc.u32 t,a,b; addc.u32 m,m,m` yields m = 2m + (a >= b) on sm_90a (CF = hardware carry = no borrow)
#include <cstdint>
#include <cstdio>
#include <vector>
__device__ __forceinline__ void borrow_into(uint32_t& m, uint32_t a, uint32_t b) {
  asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\taddc.u32 %0, %0, %0;\n\t}" : "+r"(m) : "r"(a), "r"(b));
}
__global__ void k(const uint32_t* a, const uint32_t* b, uint32_t* out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t m = 0;
  borrow_into(m, a[i], b[i]);
  borrow_into(m, a[i] ^ 0x80000000u, b[i]);
  borrow_into(m, a[i], b[i] ^ 0x80000000u);
  out[i] = m;
}
int main() {
  std::vector<uint32_t> a, b;
  uint32_t edge[] = {0u, 1u, 2u, 0x7FFFFFFFu, 0x80000000u, 0x80000001u, 0xFFFFFFFEu, 0xFFFFFFFFu, 0x1000u, 0xFFFFF000u};
  for (uint32_t x : edge) for (uint32_t y : edge) { a.push_back(x); b.push_back(y); }
  uint64_t s = 88172645463325252ull;
  for (int i = 0; i < 1 << 20; i++) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; a.push_back((uint32_t)s); b.push_back((uint32_t)(s >> 32)); }
  int n = (int)a.size();
  uint32_t *da, *db, *dout;
  cudaMalloc(&da, n * 4); cudaMalloc(&db, n * 4); cudaMalloc(&dout, n * 4);
  cudaMemcpy(da, a.data(), n * 4, cudaMemcpyHostToDevice); cudaMemcpy(db, b.data(), n * 4, cudaMemcpyHostToDevice);
  k<<<(n + 255) / 256, 256>>>(da, db, dout, n);
  std::vector<uint32_t> out(n);
  if (cudaMemcpy(out.data(), dout, n * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { printf("cuda error\n"); return 2; }
  long bad = 0;
  for (int i = 0; i < n; i++) {
    uint32_t want = ((a[i] >= b[i]) << 2) | (((a[i] ^ 0x80000000u) >= b[i]) << 1) | (a[i] >= (b[i] ^ 0x80000000u));
    if (out[i] != want) { if (bad < 10) printf("a=%08x b=%08x got=%u want=%u\n", a[i], b[i], out[i], want); bad++; }
  }
  printf("n=%d bad=%ld\n", n, bad);
  return bad != 0;
}
