// Phase clocks of the table ("spec") hash kernel, CTA 0 (clock64 on one SM): start | own tables done | all tables seen |
// first rows staged | chain start | chain end.
// nvcc -DKVB_HASH_PROFILE -gencode arch=compute_90a,code=sm_90a -O3 -I include -I llm-d-kv-cache_b200/csrc \
//      -o tools/micro/spec_phase_profile tools/micro/spec_phase_profile.cu llm-d-kv-cache_b200/csrc/pool_api.cu llm-d-kv-cache_b200/csrc/copy_kernels.cu
#include "../../llm-d-kv-cache_b200/csrc/hash_kernels.cu"
#include <vector>
int main(int argc, char** argv) {
  const int n = argc > 1 ? atoi(argv[1]) : 1, L = 1000, BS = 16;
  const bool pinned = argc > 2 && atoi(argv[2]) != 0;  // tokens in pinned host memory, read in place
  const bool score = argc > 3 && atoi(argv[3]) != 0;   // fused form: every key is in a table with one pod entry
  std::vector<uint32_t> tok((size_t)n * L);
  uint64_t x = 88172645463325252ull;
  for (auto& t : tok) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; t = (uint32_t)(x % 128256); }
  std::vector<int64_t> off(n + 1), koff(n + 1);
  for (int i = 0; i <= n; ++i) { off[i] = (int64_t)i * L; koff[i] = (int64_t)i * (L / BS); }
  std::vector<uint64_t> par(n, 0x1234567890abcdefull);
  uint32_t* dt; int64_t *dof, *dk; uint64_t *dp, *dout;
  if (pinned) { cudaHostAlloc(&dt, tok.size() * 4, cudaHostAllocMapped); memcpy(dt, tok.data(), tok.size() * 4); }
  else { cudaMalloc(&dt, tok.size() * 4); cudaMemcpy(dt, tok.data(), tok.size() * 4, cudaMemcpyHostToDevice); }
  cudaMalloc(&dof, (n + 1) * 8); cudaMalloc(&dk, (n + 1) * 8);
  cudaMalloc(&dp, n * 8); cudaMalloc(&dout, (size_t)n * (L / BS) * 8);
  cudaMemcpy(dof, off.data(), (n + 1) * 8, cudaMemcpyHostToDevice);
  cudaMemcpy(dk, koff.data(), (n + 1) * 8, cudaMemcpyHostToDevice);
  cudaMemcpy(dp, par.data(), n * 8, cudaMemcpyHostToDevice);
  setenv("KVB_HASH_KERNEL", "spec", 1);
  const int64_t total = (int64_t)n * (L / BS);
  for (int it = 0; it < 5; ++it) kvb::launch_hash_blocks(dt, dof, dp, n, BS, nullptr, nullptr, dout, dk, 0, total);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  for (int it = 0; it < 20; ++it) kvb::launch_hash_blocks(dt, dof, dp, n, BS, nullptr, nullptr, dout, dk, 0, total);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
  printf("prompts %d (%s tokens): %.1f us per launch\n", n, pinned ? "pinned host" : "device", ms * 1000 / 20);
#ifdef KVB_HASH_PROFILE
  long long h[16];
  cudaMemcpyFromSymbol(h, kvb::g_hash_prof, sizeof(h));
  int clk = 0; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
  const double us = 1000.0 / clk;
  printf("CTA 0 (cycles -> us at %d MHz): own tables %.2f | all tables seen %.2f | first rows staged %.2f | chain start %.2f | chain end %.2f"
         "  (chain: %.0f cycles per block)\n", clk / 1000,
         (h[1] - h[0]) * us, (h[2] - h[0]) * us, (h[3] - h[0]) * us, (h[4] - h[0]) * us, (h[5] - h[0]) * us,
         (double)(h[5] - h[4]) / (L / BS));
#endif
  if (score) {
    std::vector<uint64_t> keys((size_t)total);
    cudaMemcpy(keys.data(), dout, total * 8, cudaMemcpyDeviceToHost);
    const uint64_t slots = 1ull << 20, mask = slots - 1;
    std::vector<kvb::Bucket> tab(slots);
    memset(tab.data(), 0, slots * sizeof(kvb::Bucket));
    for (uint64_t k : keys) {
      uint64_t sl = kvb::mix64(k) & mask;
      while ((tab[sl].meta & 3u) == kvb::kFull) sl = (sl + 1) & mask;
      tab[sl].key = k; tab[sl].meta = kvb::kFull | (1u << 8); tab[sl].ent[0] = kvb::pack_entry(3, 0, 0);
    }
    kvb::Bucket* dtab; cudaMalloc(&dtab, slots * sizeof(kvb::Bucket));
    cudaMemcpy(dtab, tab.data(), slots * sizeof(kvb::Bucket), cudaMemcpyHostToDevice);
    double* dw; std::vector<double> w(256, 1.0); cudaMalloc(&dw, 256 * 8); cudaMemcpy(dw, w.data(), 256 * 8, cudaMemcpyHostToDevice);
    int32_t* on; uint16_t* op; double* os;
    cudaHostAlloc(&on, n * 4, cudaHostAllocMapped); cudaHostAlloc(&op, n * 13 * 2, cudaHostAllocMapped); cudaHostAlloc(&os, n * 13 * 8, cudaHostAllocMapped);
    unsigned long long* ts; cudaMalloc(&ts, slots * 8); cudaMemset(ts, 0, slots * 8);
    unsigned* dcnt; cudaMalloc(&dcnt, 4); cudaMemset(dcnt, 0, 4);
    unsigned long long* hflag; cudaHostAlloc(&hflag, 8, cudaHostAllocMapped); *hflag = 0;
    kvb::ChainArgs a{};
    a.tokens = dt; a.tokens_lo = dt; a.tokens_hi = dt + tok.size();
    a.single = n == 1; a.single_tokens = L; a.single_parent = par[0];
    a.prompt_off = dof; a.parents = dp; a.key_off = dk;
    a.table = dtab; a.mask = mask; a.tier_w = dw; a.out_n = on; a.out_pods = op; a.out_scores = os;
    a.ts = ts; a.stamp_base = 1000; a.score_min_batch = argc > 4 ? atoi(argv[4]) : 32;
    a.done_counter = dcnt; a.done_target = (unsigned)n; a.done_flag_host = hflag;
    int rc = 0;
    for (int it = 0; it < 5; ++it) { a.done_value = it + 1; kvb::launch_spec(a, true, n, BS, total, 0, &rc); }
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    for (int it = 0; it < 20; ++it) { a.done_value = 100 + it; kvb::launch_spec(a, true, n, BS, total, 0, &rc); }
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    printf("fused (score batch %d): %.1f us per launch; prompt 0: %d pods, score %.1f\n", a.score_min_batch, ms * 1000 / 20, on[0], os[0]);
#ifdef KVB_HASH_PROFILE
    cudaMemcpyFromSymbol(h, kvb::g_hash_prof, sizeof(h));
    printf("CTA 0 us: own tables %.2f | all tables %.2f | rows staged %.2f | chain start %.2f | chain end %.2f | scorer: first tile start %.2f end %.2f | last tile end %.2f | results written %.2f | signalled %.2f\n",
           (h[1] - h[0]) * us, (h[2] - h[0]) * us, (h[3] - h[0]) * us, (h[4] - h[0]) * us, (h[5] - h[0]) * us,
           (h[7] - h[0]) * us, (h[8] - h[0]) * us, (h[9] - h[0]) * us, (h[10] - h[0]) * us, (h[6] - h[0]) * us);
#endif
  }
  printf("status %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
