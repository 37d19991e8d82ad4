// Where do the warps of 1024 two-warp CTAs land?  Records (%smid, %warpid) of both warps of every CTA while all CTAs
// are co-resident, then prints CTAs per SM and, per scheduler (warpid % 4), how many "folder" warps the hash kernel's
// role rule would place there.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/slot_map tools/micro/slot_map.cu
#include <cstdio>
#include <cstdint>
#include <vector>
#include <map>
#include <algorithm>
__global__ void k(uint32_t* out) {
  uint32_t sm, wid;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
  asm volatile("mov.u32 %0, %%warpid;" : "=r"(wid));
  if ((threadIdx.x & 31) == 0) out[blockIdx.x * 2 + (threadIdx.x >> 5)] = (sm << 16) | wid;
  const long long t0 = clock64();
  while (clock64() - t0 < 60000) {}
}
int main(int argc, char** argv) {
  const int n = argc > 1 ? atoi(argv[1]) : 1024;
  uint32_t* d; cudaMalloc(&d, n * 8);
  k<<<n, 64>>>(d); cudaDeviceSynchronize();
  std::vector<uint32_t> h(n * 2); cudaMemcpy(h.data(), d, n * 8, cudaMemcpyDeviceToHost);
  std::map<int, int> per_sm; std::map<int, std::vector<int>> fold_sched;
  int aligned = 0;
  for (int c = 0; c < n; ++c) {
    const uint32_t a = h[2 * c] & 0xffff, b = h[2 * c + 1] & 0xffff; const int sm = h[2 * c] >> 16;
    per_sm[sm]++;
    aligned += (b == a + 1 && (a & 1) == 0);
    const bool fa = ((a >> 2) & 1) == (a & 1), fb = ((b >> 2) & 1) == (b & 1);
    const uint32_t folder = (fa != fb) ? (fa ? a : b) : b;
    auto& v = fold_sched[sm]; if (v.empty()) v.assign(4, 0); v[folder & 3]++;
  }
  int mn = 1 << 30, mx = 0; for (auto& kv : per_sm) { mn = std::min(mn, kv.second); mx = std::max(mx, kv.second); }
  printf("%d CTAs on %zu SMs: %d..%d per SM; warp pairs on aligned slots (2j, 2j+1): %d of %d\n", n, per_sm.size(), mn, mx, aligned, n);
  int worst = 0; std::map<int, int> hist;
  for (auto& kv : fold_sched) for (int s = 0; s < 4; ++s) { worst = std::max(worst, kv.second[s]); hist[kv.second[s]]++; }
  printf("folder warps per scheduler: worst %d; histogram:", worst);
  for (auto& kv : hist) printf("  %d folders x %d schedulers", kv.first, kv.second);
  printf("\nfirst CTAs (sm, warpid0, warpid1):");
  for (int c = 0; c < 12 && c < n; ++c) printf(" (%u,%u,%u)", h[2 * c] >> 16, h[2 * c] & 0xffff, h[2 * c + 1] & 0xffff);
  printf("\n%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
