// Dependent-chain latencies of the warp-level instructions the warp-per-chain hash kernel is built from
// (one warp, one CTA; clock64 around N dependent iterations).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/warp_chain_latency tools/micro/warp_chain_latency.cu
#include <cstdio>
#include <cstdint>
constexpr int N = 4096;
__global__ void k(long long* out, uint32_t seed) {
  const uint32_t lane = threadIdx.x, lt = (1u << lane) - 1u;
  uint32_t x = seed + lane, y = seed * 3 + 1, acc = 0;
  long long t0, t1;
  // A: vote -> and -> popc -> lop3+setp -> vote
  uint32_t before = lane & 1;
  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < N; ++i) {
    const uint32_t v = __ballot_sync(0xffffffffu, ((before & x) ^ y) & 1u);
    before = __popc(v & lt);
    y ^= 1u;
  }
  t1 = clock64();
  acc += before;
  if (lane == 0) out[0] = t1 - t0;
  // B: dependent REDUX.SUM
  uint32_t s = x & 0xffffu;
  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < N; ++i) s = __reduce_add_sync(0xffffffffu, (s & 0xffu) + lane);
  t1 = clock64();
  acc += s;
  if (lane == 0) out[1] = t1 - t0;
  // C: 4 independent REDUX per step, combined, dependent across steps
  uint32_t c = x;
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; ++i) {
    const uint32_t a0 = __reduce_add_sync(0xffffffffu, c & 0xffu), a1 = __reduce_add_sync(0xffffffffu, (c >> 8) & 0xffu),
                   a2 = __reduce_add_sync(0xffffffffu, (c >> 16) & 0xffu), a3 = __reduce_add_sync(0xffffffffu, c >> 24);
    c = (a0 + (a1 << 8) + (a2 << 16) + (a3 << 24)) ^ lane;
  }
  t1 = clock64();
  acc += c;
  if (lane == 0) out[2] = t1 - t0;
  // D: dependent SHFL
  uint32_t d = x;
  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < N; ++i) d = __shfl_xor_sync(0xffffffffu, d, 1) + 1u;
  t1 = clock64();
  acc += d;
  if (lane == 0) out[3] = t1 - t0;
  // E: vote alone (predicate from a LOP3 on the previous mask)
  uint32_t e = x;
  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < N; ++i) e = __ballot_sync(0xffffffffu, (e ^ lane) & 1u);
  t1 = clock64();
  acc += e;
  if (lane == 0) out[4] = t1 - t0;
  // F: popc alone
  uint32_t f = x;
  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < N; ++i) f = __popc(f ^ lt) + lane;
  t1 = clock64();
  acc += f;
  if (lane == 0) out[5] = t1 - t0;
  // G: LOP3 -> IMAD (calibration, ~10)
  uint32_t g = x;
  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < N; ++i) g = (g ^ lane) * 0xb3u;
  t1 = clock64();
  acc += g;
  if (lane == 0) out[6] = t1 - t0;
  // H: shared-memory round trip (STS -> syncwarp -> LDS of the neighbour's word)
  __shared__ uint32_t sm[32];
  uint32_t h = x;
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; ++i) {
    sm[lane] = h;
    __syncwarp();
    h = sm[(lane + 1) & 31] + 1u;
    __syncwarp();
  }
  t1 = clock64();
  acc += h;
  if (lane == 0) out[7] = t1 - t0;
  if (acc == 0x12345u) out[15] = acc;
}
int main() {
  long long* d; cudaMalloc(&d, 16 * 8);
  k<<<1, 32>>>(d, 7); k<<<1, 32>>>(d, 7);
  long long h[16]; cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost);
  const char* names[] = {"vote->and->popc->lop3.p->vote", "redux.sum (dependent)", "4x redux.sum + recombine", "shfl (dependent, +iadd)",
                         "vote (dependent, +lop3/setp)", "popc (dependent, +lop3/iadd)", "lop3->imad", "sts->syncwarp->lds->syncwarp"};
  for (int i = 0; i < 8; ++i) printf("%-36s %.1f cycles per step\n", names[i], (double)h[i] / N);
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
