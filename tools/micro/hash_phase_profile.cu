// Per-phase cycle counts of the two-warp hash kernel (clock64 around each phase, CTA 0, lane 0).
// (without -DKVB_HASH_PROFILE the same program only times the production kernel: tools/micro/hash_time)
// nvcc -DKVB_HASH_PROFILE -gencode arch=compute_90a,code=sm_90a -O3 -I include -I llm-d-kv-cache_b200/csrc \
//      -o tools/micro/hash_phase_profile tools/micro/hash_phase_profile.cu llm-d-kv-cache_b200/csrc/pool_api.cu llm-d-kv-cache_b200/csrc/copy_kernels.cu
#include "../../llm-d-kv-cache_b200/csrc/hash_kernels.cu"
#include <vector>
int main(int argc, char** argv) {
  const int n = argc > 1 ? atoi(argv[1]) : 1024, L = 1000, BS = 16;  // KVB_HASH_KERNEL=lanes profiles the two-warp kernel
  std::vector<uint32_t> tok((size_t)n * L);
  uint64_t x = 88172645463325252ull;
  for (auto& t : tok) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; t = (uint32_t)(x % 128256); }
  std::vector<int64_t> off(n + 1), koff(n + 1);
  for (int i = 0; i <= n; ++i) { off[i] = (int64_t)i * L; koff[i] = (int64_t)i * (L / BS); }
  std::vector<uint64_t> par(n, 0x1234567890abcdefull);
  uint32_t* dt; int64_t *dof, *dk; uint64_t *dp, *dout;
  cudaMalloc(&dt, tok.size() * 4); cudaMalloc(&dof, (n + 1) * 8); cudaMalloc(&dk, (n + 1) * 8);
  cudaMalloc(&dp, n * 8); cudaMalloc(&dout, (size_t)n * (L / BS) * 8);
  cudaMemcpy(dt, tok.data(), tok.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(dof, off.data(), (n + 1) * 8, cudaMemcpyHostToDevice);
  cudaMemcpy(dk, koff.data(), (n + 1) * 8, cudaMemcpyHostToDevice);
  cudaMemcpy(dp, par.data(), n * 8, cudaMemcpyHostToDevice);
  for (int it = 0; it < 3; ++it) kvb::launch_hash_blocks(dt, dof, dp, n, BS, nullptr, nullptr, dout, dk, 0);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  for (int it = 0; it < 20; ++it) kvb::launch_hash_blocks(dt, dof, dp, n, BS, nullptr, nullptr, dout, dk, 0);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
#ifndef KVB_HASH_PROFILE
  printf("prompts %d: %.1f us per launch (production build, 20 back-to-back launches)\n", n, ms * 1000 / 20);
  return 0;
#else
  printf("prompts %d: %.1f us per launch (clock64 instrumented build)\n", n, ms * 1000 / 20);
  long long h[16];
  cudaMemcpyFromSymbol(h, kvb::g_hash_prof, sizeof(h));
  const double nb = (double)h[10];
  printf("blocks per chain: %.0f\n", nb);
  if (n <= kvb::kWpcMaxPrompts && getenv("KVB_HASH_KERNEL") == nullptr) {
    printf("chain v2 folder : wait+loads %.0f  bits-0/1 %.0f  rounds(6) %.0f  reduce %.0f  tail %.0f  cycles/block (sum %.0f)\n",
           h[5] / nb, h[6] / nb, h[7] / nb, h[8] / nb, h[9] / nb, (h[5] + h[6] + h[7] + h[8] + h[9]) / nb);
  } else if (n <= kvb::kWpcMaxPrompts && getenv("KVB_HASH_KERNEL") != nullptr && !strcmp(getenv("KVB_HASH_KERNEL"), "wpc")) {
    printf("warp-per-chain  stager : work %.0f  barrier-wait %.0f  cycles/block\n", h[0] / nb, h[4] / nb);
    printf("warp-per-chain  folder : rounds %.0f  reduce+combine %.0f  rest %.0f  barrier-wait %.0f  cycles/block\n", h[6] / nb, h[7] / nb, h[8] / nb, h[9] / nb);
  } else {
    printf("stager : work %.0f  barrier-wait %.0f  cycles/block\n", h[0] / nb, h[4] / nb);
    printf("folder : prefix %.0f  staged-fold %.0f  rest %.0f  barrier-wait %.0f  cycles/block\n", h[6] / nb, h[7] / nb, h[8] / nb, h[9] / nb);
  }
  printf("status %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
#endif
}
