// How fast can SMs read pinned HOST memory in place?  4 MB (the config #5 token array), three access paths:
//   ldg  : 16 B per lane, a warp covers 512 B per instruction, ITEMS chunks per CTA
//   cpas : cp.async.cg 16 B per lane into shared memory (what chain_kernel's stager does)
//   bulk : cp.async.bulk (TMA, 1-D) of CHUNK bytes per elected thread into shared memory, mbarrier completion
// against cudaMemcpyAsync (copy engine).   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/pinned_read_bw tools/micro/pinned_read_bw.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

__global__ void k_ldg(const uint4* __restrict__ src, size_t n16, unsigned long long* sink) {
  uint32_t acc = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i));
    acc ^= v.x ^ v.y ^ v.z ^ v.w;
  }
  if (acc == 0x12345u) *sink = acc;
}

template <int DEPTH>
__global__ void k_cpas(const uint4* __restrict__ src, size_t n16, unsigned long long* sink) {
  extern __shared__ uint4 sm[];
  uint32_t acc = 0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int inflight = 0;
  for (; i < n16; i += stride) {
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(sm + (inflight % DEPTH) * blockDim.x + threadIdx.x);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src + i) : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
    if (++inflight >= DEPTH) asm volatile("cp.async.wait_group %0;" ::"n"(DEPTH - 1) : "memory");
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  acc = sm[threadIdx.x].x;
  if (acc == 0x12345u) *sink = acc;
}

template <int CHUNK, int STAGES>
__global__ void k_bulk(const uint8_t* __restrict__ src, size_t bytes, unsigned long long* sink) {
  extern __shared__ __align__(128) uint8_t smb[];
  __shared__ __align__(8) unsigned long long bar[STAGES];
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      const uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar[s]);
      asm volatile("mbarrier.init.shared.b64 [%0], 1;" ::"r"(b));
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const size_t nchunks = bytes / CHUNK;
    uint32_t phase[STAGES] = {};
    size_t issued = 0, done = 0;
    for (size_t c = blockIdx.x; c < nchunks || done < issued; c += gridDim.x) {
      if (c < nchunks) {
        const int s = (int)(issued % STAGES);
        if (issued >= STAGES) {  // wait for the stage's previous copy
          const uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar[s]);
          uint32_t ok = 0;
          while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(b), "r"(phase[s]) : "memory");
          phase[s] ^= 1u;
          ++done;
        }
        const uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar[s]);
        const uint32_t d = (uint32_t)__cvta_generic_to_shared(smb + (size_t)s * CHUNK);
        asm volatile("mbarrier.arrive.expect_tx.shared.b64 _, [%0], %1;" ::"r"(b), "r"(CHUNK) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(d), "l"(src + c * CHUNK), "r"(CHUNK), "r"(b) : "memory");
        ++issued;
      } else {
        const int s = (int)(done % STAGES);
        const uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar[s]);
        uint32_t ok = 0;
        while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(b), "r"(phase[s]) : "memory");
        phase[s] ^= 1u;
        ++done;
      }
    }
    if (smb[0] == 0x77 && smb[1] == 0x78 && bytes == 1) *sink = 1;
  }
}

// one CTA (one warp) per prompt, as chain_kernel's stager reads: the prompt's 4000 B in 512 B chunks (16 B per lane), DEPTH
// chunks in flight, optionally with the chunk grid aligned to 128 B lines (the first chunk is then shorter)
template <int DEPTH, bool ALIGN, int DELAY>
__global__ void k_prompt(const uint8_t* __restrict__ src, int prompt_bytes, unsigned long long* sink) {
  __shared__ uint4 ring[DEPTH][32];
  const uint8_t* b0 = src + (size_t)blockIdx.x * prompt_bytes;
  const uint8_t* b1 = b0 + prompt_bytes;
  const uint8_t* c = ALIGN ? (const uint8_t*)((uintptr_t)b0 & ~(uintptr_t)127) : b0;
  int inflight = 0;
  for (; c < b1; c += 512) {
    const uint8_t* a = c + threadIdx.x * 16;
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&ring[inflight % DEPTH][threadIdx.x]);
    if (a >= b0 && a + 16 <= b1) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(a) : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
    if (++inflight >= DEPTH) {
      asm volatile("cp.async.wait_group %0;" ::"n"(DEPTH - 1) : "memory");
      if (DELAY) __nanosleep(DELAY);  // the folder consuming a chunk
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  if (ring[0][threadIdx.x].x == 0x12345u) *sink = 1;
}

int main() {
  const size_t bytes = 4096000;  // 1024 prompts x 1000 tokens x 4 B
  uint8_t* h; CK(cudaHostAlloc(&h, bytes, cudaHostAllocMapped));
  for (size_t i = 0; i < bytes; ++i) h[i] = (uint8_t)(i * 131u);
  uint8_t* d; CK(cudaMalloc(&d, bytes));
  unsigned long long* sink; CK(cudaMalloc(&sink, 8));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  auto time = [&](const char* name, auto fn) {
    for (int i = 0; i < 3; ++i) fn();
    CK(cudaDeviceSynchronize());
    float best = 1e9f;
    for (int r = 0; r < 10; ++r) {
      CK(cudaEventRecord(e0)); fn(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
    }
    CK(cudaGetLastError());
    printf("%-44s %7.1f us  %6.1f GB/s\n", name, best * 1e3, bytes / (best * 1e-3) / 1e9);
  };
  time("cudaMemcpyAsync H2D (copy engine)", [&] { CK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, 0)); });
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  for (int grid : {sms, 2 * sms, 1024}) for (int thr : {128, 256}) {
    char nm[96]; snprintf(nm, sizeof nm, "ldg 16 B/lane, grid %d x %d", grid, thr);
    time(nm, [&] { k_ldg<<<grid, thr>>>((const uint4*)h, bytes / 16, sink); });
  }
  for (int grid : {sms, 1024}) {
    char nm[96]; snprintf(nm, sizeof nm, "cp.async 16 B/lane depth 8, grid %d x 128", grid);
    time(nm, [&] { k_cpas<8><<<grid, 128, 8 * 128 * 16>>>((const uint4*)h, bytes / 16, sink); });
  }
  for (int grid : {sms, 2 * sms, 4 * sms}) {
    char nm[96]; snprintf(nm, sizeof nm, "cp.async.bulk 4000 B x 4 stages, grid %d", grid);
    time(nm, [&] { k_bulk<4000, 4><<<grid, 32, 4 * 4000>>>(h, bytes, sink); });
  }
  for (int grid : {sms, 2 * sms}) {
    char nm[96]; snprintf(nm, sizeof nm, "cp.async.bulk 16000 B x 4 stages, grid %d", grid);
    CK(cudaFuncSetAttribute(k_bulk<16000, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 16000));
    time(nm, [&] { k_bulk<16000, 4><<<grid, 32, 4 * 16000>>>(h, bytes, sink); });
  }
  time("per-prompt 512 B chunks, 3 in flight          ", [&] { k_prompt<3, false, 0><<<1024, 32>>>(h, 4000, sink); });
  time("per-prompt 512 B chunks, 3 in flight, 128 B grid", [&] { k_prompt<3, true, 0><<<1024, 32>>>(h, 4000, sink); });
  time("per-prompt 512 B chunks, 6 in flight          ", [&] { k_prompt<6, false, 0><<<1024, 32>>>(h, 4000, sink); });
  time("per-prompt 512 B chunks, 6 in flight, 128 B grid", [&] { k_prompt<6, true, 0><<<1024, 32>>>(h, 4000, sink); });
  time("per-prompt, 3 in flight, 6 us per chunk consumed", [&] { k_prompt<3, false, 6000><<<1024, 32>>>(h, 4000, sink); });
  time("same, 128 B grid                               ", [&] { k_prompt<3, true, 6000><<<1024, 32>>>(h, 4000, sink); });
  time("per-prompt, 6 in flight, 6 us per chunk consumed", [&] { k_prompt<6, false, 6000><<<1024, 32>>>(h, 4000, sink); });
  return 0;
}
