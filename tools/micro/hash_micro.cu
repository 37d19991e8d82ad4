// Micro-benchmark of the hash kernel's building blocks on one lone warp (cycles from clock64).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/hash_micro tools/micro/hash_micro.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

struct Fnv { uint32_t lo, hi; };
__device__ __forceinline__ void fold_wide(Fnv& h, uint32_t byte) {
  const uint32_t x = h.lo ^ byte;
  uint32_t lo2, carry;
  asm("{\n\t.reg .u64 t;\n\tmul.wide.u32 t, %2, 435;\n\tmov.b64 {%0, %1}, t;\n\t}" : "=r"(lo2), "=r"(carry) : "r"(x));
  h.hi = h.hi * 0x1b3u + (carry + (x << 8));
  h.lo = lo2;
}
__device__ __forceinline__ void fold_split(Fnv& h, uint32_t byte) {  // mul.lo on the chain, mul.hi beside it
  const uint32_t x = h.lo ^ byte;
  const uint32_t carry = __umulhi(x, 0x1b3u);
  h.hi = h.hi * 0x1b3u + (carry + (x << 8));
  h.lo = x * 0x1b3u;
}
__device__ __forceinline__ uint64_t fold64(uint64_t h, uint32_t b) { return (h ^ b) * 0x100000001b3ull; }

__device__ __forceinline__ int stage_token(uint8_t* buf, int n, uint32_t t) {
  const bool ge24 = t >= 24u, ge256 = t >= 0x100u, ge64k = t >= 0x10000u;
  const uint32_t head = ge64k ? 0x1au : (ge256 ? 0x19u : (ge24 ? 0x18u : t));
  const uint32_t pay = ge64k ? t : (ge256 ? (t << 16) : (t << 24));
  buf[n] = (uint8_t)head; buf[n + 1] = (uint8_t)(pay >> 24); buf[n + 2] = (uint8_t)(pay >> 16);
  buf[n + 3] = (uint8_t)(pay >> 8); buf[n + 4] = (uint8_t)pay;
  return n + (ge64k ? 5 : (ge256 ? 3 : (ge24 ? 2 : 1)));
}

__global__ void micro(const uint32_t* __restrict__ data, long long* out, uint64_t* sink) {
  __shared__ uint32_t strips[32 * 23];
  uint8_t* buf = reinterpret_cast<uint8_t*>(strips + threadIdx.x * 23);
  const int lane = threadIdx.x;
  uint32_t w[16];
  for (int i = 0; i < 16; ++i) w[i] = data[lane * 16 + i];
  const int R = 256;
  // A: fold from registers, wide form (64 bytes per rep)
  Fnv h{0x84222325u ^ lane, 0xcbf29ce4u};
  long long t0 = clock64();
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int i = 0; i < 16; ++i) { fold_wide(h, w[i] & 0xff); fold_wide(h, (w[i] >> 8) & 0xff); fold_wide(h, (w[i] >> 16) & 0xff); fold_wide(h, w[i] >> 24); }
  long long t1 = clock64();
  // B: split mul.lo / mul.hi
  Fnv g{0x84222325u ^ lane, 0xcbf29ce4u};
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int i = 0; i < 16; ++i) { fold_split(g, w[i] & 0xff); fold_split(g, (w[i] >> 8) & 0xff); fold_split(g, (w[i] >> 16) & 0xff); fold_split(g, w[i] >> 24); }
  long long t2 = clock64();
  // C: plain 64-bit multiply
  uint64_t q = 0xcbf29ce484222325ull ^ lane;
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int i = 0; i < 16; ++i) { q = fold64(q, w[i] & 0xff); q = fold64(q, (w[i] >> 8) & 0xff); q = fold64(q, (w[i] >> 16) & 0xff); q = fold64(q, w[i] >> 24); }
  long long t3 = clock64();
  // D: stage 16 tokens
  int n = 0;
  for (int r = 0; r < R; ++r) { n = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) n = stage_token(buf, n, w[i] % 128256u); }
  long long t4 = clock64();
  // E: fold the staged strip from shared memory (n bytes)
  Fnv e{0x84222325u ^ lane, 0xcbf29ce4u};
  const uint32_t* sw = reinterpret_cast<const uint32_t*>(buf);
  for (int r = 0; r < R; ++r) {
    int k = 0;
#pragma unroll 2
    for (; k + 4 <= n; k += 4) { const uint32_t v = sw[k >> 2]; fold_wide(e, v & 0xff); fold_wide(e, (v >> 8) & 0xff); fold_wide(e, (v >> 16) & 0xff); fold_wide(e, v >> 24); }
    for (; k < n; ++k) fold_wide(e, buf[k]);
  }
  long long t5 = clock64();
  // F: pure low-half chain (LOP3 -> IMAD.WIDE), nothing else
  uint32_t lo = 0x84222325u ^ lane, acc = 0;
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t x = lo ^ ((w[i] >> (8 * j)) & 0xff);
        uint32_t carry;
        asm("{\n\t.reg .u64 t;\n\tmul.wide.u32 t, %2, 435;\n\tmov.b64 {%0, %1}, t;\n\t}" : "=r"(lo), "=r"(carry) : "r"(x));
        acc += carry;
      }
  long long t6 = clock64();
  // G: pure low-half chain with a plain 32-bit multiply (LOP3 -> IMAD)
  uint32_t lo2 = 0x84222325u ^ lane;
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) lo2 = (lo2 ^ ((w[i] >> (8 * j)) & 0xff)) * 435u;
  long long t7 = clock64();
  // H: word-at-a-time with a runtime length and a branch per word (the kernel's shape), from registers
  Fnv k{0x84222325u ^ lane, 0xcbf29ce4u};
  int nn = n;  // runtime value
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      if (4 * i + 4 > nn) break;
      fold_wide(k, w[i] & 0xff); fold_wide(k, (w[i] >> 8) & 0xff); fold_wide(k, (w[i] >> 16) & 0xff); fold_wide(k, w[i] >> 24);
    }
  long long t8 = clock64();
  if (lane == 0) { out[6] = t6 - t5; out[7] = t7 - t6; out[8] = t8 - t7; }
  sink[32 + lane] = lo + acc + lo2 + k.lo + k.hi;
  if (lane == 0) { out[0] = t1 - t0; out[1] = t2 - t1; out[2] = t3 - t2; out[3] = t4 - t3; out[4] = t5 - t4; out[5] = n; }
  sink[lane] = ((uint64_t)h.hi << 32 | h.lo) ^ ((uint64_t)g.hi << 32 | g.lo) ^ q ^ ((uint64_t)e.hi << 32 | e.lo);
}

int main() {
  uint32_t hdata[512];
  for (int i = 0; i < 512; ++i) hdata[i] = 1103515245u * (i + 7) + 12345u;
  uint32_t* d; long long* o; uint64_t* s;
  cudaMalloc(&d, sizeof(hdata)); cudaMalloc(&o, 128); cudaMalloc(&s, 1024);
  cudaMemcpy(d, hdata, sizeof(hdata), cudaMemcpyHostToDevice);
  for (int it = 0; it < 3; ++it) micro<<<1, 32>>>(d, o, s);
  long long h[9]; cudaMemcpy(h, o, 72, cudaMemcpyDeviceToHost);
  const double R = 256;
  printf("fold wide (regs)   : %.2f cycles/byte\n", h[0] / (R * 64));
  printf("fold split (regs)  : %.2f cycles/byte\n", h[1] / (R * 64));
  printf("fold u64 mul (regs): %.2f cycles/byte\n", h[2] / (R * 64));
  printf("stage_token        : %.2f cycles/token\n", h[3] / (R * 16));
  printf("fold staged (smem) : %.2f cycles/byte (n=%lld bytes)\n", h[4] / (R * (double)h[5]), h[5]);
  printf("lo chain LOP3->WIDE : %.2f cycles/byte\n", h[6] / (R * 64));
  printf("lo chain LOP3->IMAD : %.2f cycles/byte\n", h[7] / (R * 64));
  printf("fold wide, branch per word, runtime n: %.2f cycles/byte\n", h[8] / (R * (double)(h[5] / 4 * 4 < 64 ? h[5] / 4 * 4 : 64)));
  printf("cuda status: %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
