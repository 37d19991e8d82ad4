// hash_kernels.cu — chained kvblock prefix hash on the device.
//
// Replaces chunkedTokenDatabase.{hash,prefixHashes,TokensToKVBlockKeys}
// (pkg/kvcache/kvblock/token_processor.go:123-205):
//     key_i = FNV64a( 0x83 | U(parent) | ARR(chunk_i) | X(extra_i) ),  parent = key_{i-1}
// with U/ARR the RFC 8949 shortest-form heads the reference gets from fxamacker/cbor v2.7.0
// CanonicalEncOptions (token_processor.go:97).  The payload never reaches global memory: token bytes
// are staged in a per-lane strip of shared memory and folded from registers.
//
// Parallelism: keys chain across blocks, so one prompt is one serial chain of blocks.  Two kernel families:
//   lane per prompt (32 chains per warp; the byte chain xor -> multiply runs serially in each lane)
//     hash_chain_kernel_2w<BS<=16>  two warps per 32 chains: warp 0 encodes block i+1, warp 1 folds block i
//     hash_chain_kernel<BS>         one warp does both (any block size; A/B switch KVB_HASH_ONE_WARP)
//   warp per prompt, batches <= kWpcPromptsPerSm x SMs and block size 4/8/16 (KVB_HASH_KERNEL=lanes disables it)
//     hash_chain_kernel_wpc<BS>     the 32 lanes resolve one block's byte stream together: FNV-1a is a T-function,
//                                   so its low byte is 8 prefix-XOR rounds (warp votes) and the 64-bit state a dot
//                                   product with powers of P^-1 (see the comment above the kernel)
// Bound: issue/latency of dependent warp instructions (xor -> wide multiply >= 10-12 cycles per payload byte for the
// lane kernels, ~75 cycles per vote round for the warp kernel; tools/micro/), NOT HBM: the only memory traffic is
// 4 B/token in and 8 B/key out.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include "kvb_internal.h"
#include "index_device.cuh"

namespace kvb {

constexpr uint64_t kFnvOffset = 0xcbf29ce484222325ull;
constexpr uint64_t kFnvPrime = 0x100000001b3ull;

// FNV-1a state kept as two 32-bit halves.  h * 0x100000001b3 = h * 0x1b3 + (h << 40), so per byte:
//   x = lo ^ b;  lo' = x * 0x1b3 (low half);  hi' = hi * 0x1b3 + mulhi(x, 0x1b3) + (x << 8)
// The serial dependency is xor -> mul.lo on the low half (2 ops per byte); the high half trails it with one
// multiply-add per byte.  (A plain 64-bit multiply compiles to ~5 dependent IMADs + selects per byte.)
struct Fnv {
  uint32_t lo, hi;
};
__device__ __forceinline__ void fold(Fnv& h, uint32_t byte) {
  const uint32_t x = h.lo ^ byte;
  // one IMAD.WIDE gives both halves of x * 0x1b3 with a ZERO addend: written as PTX so the compiler cannot fold the
  // high-half accumulation into the wide multiply's addend, which would chain lo' behind the hi update
  // (LOP3 -> SHL -> IMAD -> IMAD.WIDE per byte instead of LOP3 -> IMAD.WIDE: a three times longer dependent chain)
  uint32_t lo2, carry;
  asm("{\n\t.reg .u64 t;\n\tmul.wide.u32 t, %2, 435;\n\tmov.b64 {%0, %1}, t;\n\t}" : "=r"(lo2), "=r"(carry) : "r"(x));
  h.hi = h.hi * 0x1b3u + (carry + (x << 8));
  h.lo = lo2;
}
// Four bytes (one little-endian word of the byte stream).  The low half is the serial chain (LOP3 -> IMAD.WIDE per
// byte).  The high half is  hi' = hi*M^4 + c0*M^3 + c1*M^2 + c2*M + c3  with c_j = carry_j + (x_j << 8): evaluated
// as (hi*M^2 + (c0*M + c1))*M^2 + (c2*M + c3), i.e. only TWO multiply-adds depend on the previous hi instead of four
// — an in-order lone warp otherwise stalls ~20 cycles per word on that tail (tools/micro/hash_phase_profile.cu).
__device__ __forceinline__ void fold4(Fnv& h, uint32_t word) {
  constexpr uint32_t M = 0x1b3u, M2 = M * M;
  uint32_t lo = h.lo, c[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t x = lo ^ ((word >> (8 * j)) & 0xffu);
    uint32_t carry;
    asm("{\n\t.reg .u64 t;\n\tmul.wide.u32 t, %2, 435;\n\tmov.b64 {%0, %1}, t;\n\t}" : "=r"(lo), "=r"(carry) : "r"(x));
    c[j] = carry + (x << 8);
  }
  h.hi = (h.hi * M2 + (c[0] * M + c[1])) * M2 + (c[2] * M + c[3]);
  h.lo = lo;
}
__device__ __forceinline__ Fnv fnv_init();
__device__ __forceinline__ void fold_head64(Fnv& h, uint32_t major, uint64_t n);
__device__ __forceinline__ void fold(Fnv& h, uint32_t byte);

// Block prefix  0x83 | U(parent) | array-head(bs)  for the common shape (parent >= 2^32 so U(parent) is the 9-byte
// form, bs < 24 so the array head is one byte): 11 bytes packed into words and folded with fold4.
__device__ __forceinline__ void fold_prefix(Fnv& h, uint64_t parent, uint32_t bs) {
  if (parent >= 0x100000000ull && bs < 24u) {
    const uint32_t ph = (uint32_t)(parent >> 32), pl = (uint32_t)parent;
    // stream: 83 1b P7 P6 | P5 P4 P3 P2 | P1 P0 (80+bs)          (P7 = most significant byte of parent)
    fold4(h, 0x83u | (0x1bu << 8) | ((ph >> 24) << 16) | (((ph >> 16) & 0xffu) << 24));
    fold4(h, ((ph >> 8) & 0xffu) | ((ph & 0xffu) << 8) | ((pl >> 24) << 16) | (((pl >> 16) & 0xffu) << 24));
    fold(h, (pl >> 8) & 0xffu);
    fold(h, pl & 0xffu);
    fold(h, 0x80u | bs);
  } else {
    fold(h, 0x83u);
    fold_head64(h, 0x00u, parent);
    fold_head64(h, 0x80u, (uint64_t)bs);
  }
}
__device__ __forceinline__ Fnv fnv_init() { return Fnv{(uint32_t)kFnvOffset, (uint32_t)(kFnvOffset >> 32)}; }
__device__ __forceinline__ uint64_t fnv_value(const Fnv& h) { return ((uint64_t)h.hi << 32) | h.lo; }

// CBOR head for major type `major` (already shifted <<5) with argument n, shortest form.
__device__ __forceinline__ void fold_head64(Fnv& h, uint32_t major, uint64_t n) {
  if (n < 24) {
    fold(h, major | (uint32_t)n);
  } else if (n < 0x100ull) {
    fold(h, major | 24);
    fold(h, (uint32_t)n);
  } else if (n < 0x10000ull) {
    fold(h, major | 25);
    fold(h, (uint32_t)(n >> 8));
    fold(h, (uint32_t)n & 0xff);
  } else if (n < 0x100000000ull) {
    fold(h, major | 26);
#pragma unroll
    for (int s = 24; s >= 0; s -= 8) fold(h, (uint32_t)(n >> s) & 0xff);
  } else {
    fold(h, major | 27);
#pragma unroll
    for (int s = 56; s >= 0; s -= 8) fold(h, (uint32_t)(n >> s) & 0xff);
  }
}

// Token bytes are produced in two passes per block so that a lone warp (one chain per lane, nothing else on its
// scheduler to hide latency) issues as few instructions as possible:
//   pass 1 (independent across tokens, full ILP): every token's CBOR unsigned-int encoding (1, 2, 3 or 5 bytes) is
//           written to the lane's private strip of shared memory with five unconditional byte stores — bytes past
//           the encoding's length are overwritten by the next token, so there is no branch on the token width;
//   pass 2 (the serial chain): the strip is read back a word at a time and folded byte by byte.
#ifdef KVB_HASH_PROFILE
__device__ long long g_hash_prof[16];
#endif
constexpr int kStageTokens = 16;  // tokens staged per pass
constexpr int kStageWords = 28;   // 112 B strip (16 x 5 B + slack), 16 B aligned so it is read back with 128-bit loads

__device__ __forceinline__ int stage_token(uint8_t* buf, int n, uint32_t t) {
  const bool ge24 = t >= 24u, ge256 = t >= 0x100u, ge64k = t >= 0x10000u;
  const uint32_t head = ge64k ? 0x1au : (ge256 ? 0x19u : (ge24 ? 0x18u : t));
  // payload, left-aligned big-endian: 4 bytes (>= 65536), 2 bytes (>= 256) or 1 byte (>= 24)
  const uint32_t pay = ge64k ? t : (ge256 ? (t << 16) : (t << 24));
  buf[n] = (uint8_t)head;
  buf[n + 1] = (uint8_t)(pay >> 24);
  buf[n + 2] = (uint8_t)(pay >> 16);
  buf[n + 3] = (uint8_t)(pay >> 8);
  buf[n + 4] = (uint8_t)pay;
  return n + (ge64k ? 5 : (ge256 ? 3 : (ge24 ? 2 : 1)));
}

template <bool BRANCH_FREE>
__device__ __forceinline__ void fold_staged(Fnv& h, const uint8_t* buf, int n) {
  // Pull the whole strip into registers first (five 128-bit LDS, one shared-memory latency in total), then fold
  // from registers: folding out of shared memory word by word exposes the LDS latency on every word to the in-order
  // issue of a lone warp (29 vs 14 cycles/byte, tools/micro/hash_micro.cu).  asm volatile pins the loads up front.
  constexpr int kWords = (kStageTokens * 5 + 3) / 4;  // 20
  uint32_t v[kWords];
  const uint32_t saddr = (uint32_t)__cvta_generic_to_shared(buf);
#pragma unroll
  for (int q = 0; q < kWords / 4; ++q)
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v[4 * q]), "=r"(v[4 * q + 1]), "=r"(v[4 * q + 2]), "=r"(v[4 * q + 3])
                 : "r"(saddr + 16 * q));  // words past n hold stale bytes and are never folded
  // Whole words, branch-free: every lane runs the same straight-line code (a branch per word costs a lone warp
  // ~4 cycles/byte, tools/micro/hash_micro.cu) and keeps the folded state only for the words it really has.
  // The first 12 words (48 B = 16 three-byte tokens, the minimum for real vocabularies) are usually all present.
  // Large batches have many warps per scheduler: there the issue slots, not the latency, are scarce, and skipping
  // absent words (a branch per word) wins — BRANCH_FREE = false.
  const int nwords = n >> 2;
#pragma unroll
  for (int i = 0; i < kWords; ++i) {
    if (BRANCH_FREE) {
      Fnv t = h;
      fold4(t, v[i]);
      const bool take = i < nwords;
      h.lo = take ? t.lo : h.lo;
      h.hi = take ? t.hi : h.hi;
    } else {
      if (i >= nwords) break;
      fold4(h, v[i]);
    }
  }
  const int tail = n & 3;  // 0..3 trailing bytes live in word n/4 (dynamic index: re-read it from the strip)
  if (tail) {
    const uint32_t tw = reinterpret_cast<const uint32_t*>(buf)[n >> 2];
    fold(h, tw & 0xffu);
    if (tail > 1) fold(h, (tw >> 8) & 0xffu);
    if (tail > 2) fold(h, (tw >> 16) & 0xffu);
  }
}

template <int BS>
__global__ void __launch_bounds__(128) hash_chain_kernel(const uint32_t* __restrict__ tokens,
                                                         const int64_t* __restrict__ prompt_off,
                                                         const uint64_t* __restrict__ parents, int32_t n_prompts,
                                                         int32_t block_size_rt, const uint8_t* __restrict__ extra,
                                                         const int64_t* __restrict__ extra_off,
                                                         uint64_t* __restrict__ out_keys,
                                                         const int64_t* __restrict__ key_off) {
  __shared__ __align__(16) uint32_t strips[128 * kStageWords];
  uint8_t* buf = reinterpret_cast<uint8_t*>(strips + threadIdx.x * kStageWords);
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_prompts) return;
  const int bs = BS > 0 ? BS : block_size_rt;
  const int64_t t0 = prompt_off[p];
  const int64_t nblk = (prompt_off[p + 1] - t0) / bs;  // tail tokens dropped (token_processor.go:166-168)
  const int64_t k0 = key_off[p];
  const uint32_t* tk = tokens + t0;
  uint64_t parent = parents[p];

  uint32_t cur[BS > 0 ? BS : 1];
  if (BS > 0 && nblk > 0) {
#pragma unroll
    for (int j = 0; j < BS; ++j) cur[j] = __ldg(tk + j);
  }
  for (int64_t i = 0; i < nblk; ++i) {
    uint32_t nxt[BS > 0 ? BS : 1];
    if (BS > 0 && i + 1 < nblk) {  // prefetch the next block's tokens under this block's fold chain
#pragma unroll
      for (int j = 0; j < BS; ++j) nxt[j] = __ldg(tk + (i + 1) * BS + j);
    }
    Fnv h = fnv_init();
    fold_prefix(h, parent, (uint32_t)bs);           // array(3) | parent | array(bs)
    if (BS > 0 && BS <= kStageTokens) {
      int n = 0;
#pragma unroll
      for (int j = 0; j < BS; ++j) n = stage_token(buf, n, cur[j]);
      fold_staged<true>(h, buf, n);
    } else {
      for (int j0 = 0; j0 < bs; j0 += kStageTokens) {
        const int m = min(kStageTokens, bs - j0);
        int n = 0;
        for (int j = 0; j < m; ++j) n = stage_token(buf, n, __ldg(tk + i * bs + j0 + j));
        fold_staged<true>(h, buf, n);
      }
    }
    bool text = true;
    if (extra_off != nullptr) {                     // pre-encoded X(extra_i), host-built (extra_keys.go)
      const int64_t e0 = extra_off[k0 + i], e1 = extra_off[k0 + i + 1];
      if (e1 > e0) {
        text = false;
        for (int64_t e = e0; e < e1; ++e) fold(h, extra[e]);
      }
    }
    if (text) fold(h, 0xf6u);                       // nil extra -> CBOR null
    parent = fnv_value(h);
    out_keys[k0 + i] = parent;
    if (BS > 0) {
#pragma unroll
      for (int j = 0; j < BS; ++j) cur[j] = nxt[j];
    }
  }
}

// Two-warp variant for block sizes <= 16 (the vLLM default is 16): 32 chains per CTA, warp 0 STAGES block i+1 of
// every chain (pass 1) while warp 1 FOLDS block i (pass 2), double-buffered strips, one CTA barrier per block.
// The two warps sit on different SM sub-partitions, so the encode work leaves the serial chain's issue stream: the
// one-warp kernel is issue-bound (a lone in-order warp retires about one instruction per three cycles).
template <int BS, bool BRANCH_FREE>
__global__ void __launch_bounds__(64) hash_chain_kernel_2w(const uint32_t* __restrict__ tokens,
                                                           const int64_t* __restrict__ prompt_off,
                                                           const uint64_t* __restrict__ parents, int32_t n_prompts,
                                                           const uint8_t* __restrict__ extra,
                                                           const int64_t* __restrict__ extra_off,
                                                           uint64_t* __restrict__ out_keys,
                                                           const int64_t* __restrict__ key_off) {
  static_assert(BS > 0 && BS <= kStageTokens, "two-warp kernel stages one whole block per strip");
  __shared__ __align__(16) uint32_t strips[2][32 * kStageWords];
  __shared__ int nbytes[2][32];
  const int lane = threadIdx.x & 31;
  const bool stager = threadIdx.x < 32;
  const int p = blockIdx.x * 32 + lane;
  const bool live = p < n_prompts;
  int64_t t0 = 0, nblk = 0, k0 = 0;
  if (live) {
    t0 = prompt_off[p];
    nblk = (prompt_off[p + 1] - t0) / BS;
    k0 = key_off[p];
  }
  // both warps must run the same number of barriers: longest chain in this CTA
  int64_t nmax = nblk;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
  const uint32_t* tk = tokens + t0;
  uint64_t parent = (!stager && live) ? parents[p] : 0;

  uint32_t cur[BS];  // stager: tokens of the next block to stage, loaded one barrier interval ahead
  auto load_block = [&](int64_t i) {
    if (i < nblk) {
#pragma unroll
      for (int j = 0; j < BS; ++j) cur[j] = __ldg(tk + i * BS + j);
    }
  };
  auto stage_block = [&](int64_t i) {  // stages `cur` as block i, then starts loading block i+1
    uint8_t* buf = reinterpret_cast<uint8_t*>(strips[i & 1] + lane * kStageWords);
    int n = 0;
#pragma unroll
    for (int j = 0; j < BS; ++j) n = stage_token(buf, n, cur[j]);
    nbytes[i & 1][lane] = n;
    load_block(i + 1);
  };
  if (stager) {
    load_block(0);
    if (nblk > 0) stage_block(0);
  }
  __syncthreads();
#ifdef KVB_HASH_PROFILE
  long long pc[5] = {0, 0, 0, 0, 0};  // stager work, folder prefix, folder staged, folder rest, barrier wait
#define PROF(slot, t_begin) pc[slot] += clock64() - (t_begin)
#else
#define PROF(slot, t_begin)
#endif
  for (int64_t i = 0; i < nmax; ++i) {
#ifdef KVB_HASH_PROFILE
    long long tb = clock64();
#endif
    if (stager) {
      if (i + 1 < nblk) stage_block(i + 1);
      PROF(0, tb);
    } else if (i < nblk) {
      Fnv h = fnv_init();
      fold_prefix(h, parent, (uint32_t)BS);
      PROF(1, tb);
#ifdef KVB_HASH_PROFILE
      long long ts = clock64();
#endif
      fold_staged<BRANCH_FREE>(h, reinterpret_cast<const uint8_t*>(strips[i & 1] + lane * kStageWords), nbytes[i & 1][lane]);
      PROF(2, ts);
#ifdef KVB_HASH_PROFILE
      long long tr = clock64();
#endif
      bool text = true;
      if (extra_off != nullptr) {
        const int64_t e0 = extra_off[k0 + i], e1 = extra_off[k0 + i + 1];
        if (e1 > e0) {
          text = false;
          for (int64_t e = e0; e < e1; ++e) fold(h, extra[e]);
        }
      }
      if (text) fold(h, 0xf6u);
      parent = fnv_value(h);
      out_keys[k0 + i] = parent;
      PROF(3, tr);
    }
#ifdef KVB_HASH_PROFILE
    long long tw = clock64();
#endif
    __syncthreads();
    PROF(4, tw);
  }
#ifdef KVB_HASH_PROFILE
  if (blockIdx.x == 0 && lane == 0) {
    long long* dst = g_hash_prof + (stager ? 0 : 5);
    for (int q = 0; q < 5; ++q) dst[q] = pc[q];
    g_hash_prof[10] = nmax;
  }
#endif
}

// ---------------------------------------------------------------------------------------------------------------
// Warp-per-chain kernel for small batches (one CTA per prompt): the 32 lanes of a warp fold ONE block's byte stream
// together, so the serial cost per block is ~8 warp votes instead of ~75 dependent xor->multiply steps.
//
// FNV-1a is a T-function: bit k of (h ^ b) * P depends only on bits <= k of h and b.  With l_i = low byte of the
// state before stream byte b_i and z_i = l_i ^ b_i:
//   (1) l_{i+1} = low8(z_i * 0xb3)               (0xb3 = low byte of P): an 8-bit chain, and for every bit k
//       l_{i+1,k} = l_{i,k} ^ b_{i,k} ^ c_{i,k},  c_{i,k} = bit k of ((z_i mod 2^k) * 0xb3)
//       — linear in bit k once the lower bits are known, so bit k of EVERY position is one prefix-XOR over the stream:
//       a warp vote + popc per bit, 8 rounds per block, each lane owning 3 consecutive stream positions;
//   (2) h ^ b = h + e with e_i = z_i - l_i in [-255, 255], so  h_m = P^m * (h_0 + sum_i e_i * Q^i),  Q = P^-1 mod 2^64:
//       once the l_i are known the 64-bit state is a dot product with per-position constants, summed over the warp
//       in four 16-bit limbs (redux.sync.add).
// Stream of one block (block sizes < 24, parent >= 2^32):  83 1b P7..P0 (80+BS) | token bytes | f6   (<= 92 bytes).
// Warp 0 of the CTA stages blocks two ahead (token widths -> exclusive scan -> byte scatter -> per-lane 3-byte words),
// warp 1 runs the rounds; the rare block whose parent is < 2^32 (a caller-supplied root) and multimodal extras fall back
// to the byte-serial fold.  Measured against the lane-per-prompt kernels in DESIGN.md section 4.
constexpr uint64_t inv_mod_2_64(uint64_t a) {  // Newton: the correct low bits double every step (a * a == 1 mod 8)
  uint64_t x = a;
  for (int i = 0; i < 6; ++i) x *= 2 - a * x;
  return x;
}
constexpr uint64_t kFnvPrimeInv = inv_mod_2_64(kFnvPrime);
static_assert(kFnvPrimeInv * kFnvPrime == 1ull, "P^-1 mod 2^64");
constexpr int kWpcPositions = 96;  // 32 lanes x 3 stream positions
constexpr int kWpcPrefix = 11;     // 83 1b P7..P0 (80+BS)
// The warp-per-prompt kernel takes batches of up to kWpcPromptsPerSm prompts per SM; past that the SMs are full and the
// lane-per-prompt kernels win (H100, 132 SMs, tests/bench_hash.py: 58 vs 63 us at 1320 prompts, even at 1408, 65 vs
// 62 us at 1536)
constexpr int kWpcPromptsPerSm = 10;
constexpr int kChainMaxPrompts = 1536; // round-2 chain kernel; the round-1 warp kernel stays available (KVB_HASH_KERNEL=wpc)

__device__ __forceinline__ uint64_t pow_u64(uint64_t base, uint32_t e) {  // e < 128
  uint64_t r = 1;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    if (e & 1u) r *= base;
    base *= base;
    e >>= 1;
  }
  return r;
}

template <int BS>
__global__ void __launch_bounds__(64) hash_chain_kernel_wpc(const uint32_t* __restrict__ tokens,
                                                            const int64_t* __restrict__ prompt_off,
                                                            const uint64_t* __restrict__ parents,
                                                            const uint8_t* __restrict__ extra,
                                                            const int64_t* __restrict__ extra_off,
                                                            uint64_t* __restrict__ out_keys,
                                                            const int64_t* __restrict__ key_off) {
  static_assert(BS > 0 && BS < 24 && kWpcPrefix + 5 * BS + 1 <= kWpcPositions, "stream must fit 96 positions");
  constexpr uint32_t kFull = 0xffffffffu;
  __shared__ uint32_t bw[3][32];                          // per lane: its 3 stream bytes (parent bytes left zero)
  __shared__ uint8_t raw[3][kWpcPositions];               // token bytes (+ f6); the byte-serial fallback reads it too
  // per staged block, one 16 B load: .x/.y = P^(stream length), .z = bytes after the prefix, .w = 1 if nil extra (f6 in)
  __shared__ uint4 meta[3];
  __shared__ uint32_t tring[4][BS];                       // token ring (cp.async landing buffer)
  __shared__ uint64_t pw[kWpcPositions];                  // P^m
  __shared__ uint32_t slot_id[2];
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x;
  const int64_t t0 = prompt_off[p];
  const int nblk = (int)((prompt_off[p + 1] - t0) / BS);  // tail tokens dropped (token_processor.go:166-168)
  if (nblk == 0) return;
  const int64_t k0 = key_off[p];
  for (int t = threadIdx.x; t < kWpcPositions; t += 64) pw[t] = pow_u64(kFnvPrime, (uint32_t)t);
  // Which warp folds: a warp's scheduler (SM sub-partition) is its hardware slot % 4 and a CTA's two warps take
  // consecutive slots, so "warp 1 folds" would put every folder of an SM on sub-partitions 1 and 3.  Pick by slot so
  // that successive CTAs' folders land on 0, 2, 1, 3, ...; fall back to warp 1 if the slots are not an aligned pair.
  if (lane == 0) {
    uint32_t wid;
    asm volatile("mov.u32 %0, %%warpid;" : "=r"(wid));
    slot_id[threadIdx.x >> 5] = wid;
  }
  __syncthreads();  // also publishes pw[]
  const uint32_t sa = slot_id[0], sb = slot_id[1];
  const bool fa = ((sa >> 2) & 1u) == (sa & 1u), fb = ((sb >> 2) & 1u) == (sb & 1u);
  const int folder_warp = (fa != fb) ? (fa ? 0 : 1) : 1;
  const bool stager = (int)(threadIdx.x >> 5) != folder_warp;

  // ---- stager: tokens land in a 4-slot shared-memory ring by cp.async, three blocks ahead of their use (an L2/HBM
  // round trip is longer than one block interval; a register destination would stall the warp on the rotation moves)
  const uint32_t lt = (1u << lane) - 1u;
  auto fetch_tokens = [&](int i) {  // one commit group per block, empty past the end so the group count stays uniform
    if (lane < BS && i < nblk) {
      const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&tring[i & 3][lane]);
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(tokens + t0 + (int64_t)i * BS + lane));
    }
    asm volatile("cp.async.commit_group;");
  };
  int sbuf = 0;              // buffer of the next block to stage (i % 3 without the division)
  auto stage = [&](int i) {  // block i -> buffer i % 3
    const int buf = sbuf;
    sbuf = sbuf == 2 ? 0 : sbuf + 1;
    fetch_tokens(i + 3);
    asm volatile("cp.async.wait_group 3;" ::: "memory");  // all but the three newest groups: block i has landed
    const uint32_t t = lane < BS ? tring[i & 3][lane] : 0u;  // each lane reads back its own copy
    const bool ge24 = t >= 24u, ge256 = t >= 0x100u, ge64k = t >= 0x10000u;
    const uint32_t head = ge64k ? 0x1au : (ge256 ? 0x19u : (ge24 ? 0x18u : t));
    const uint32_t pay = ge64k ? t : (ge256 ? (t << 16) : (t << 24));  // payload, left-aligned big-endian
    // width = 1 + [>=24] + [>=256] + 2*[>=65536]: the exclusive scan over the block is three votes and popcounts
    // (lanes >= BS hold token 0 and vote false everywhere)
    const uint32_t v24 = __ballot_sync(kFull, ge24), v256 = __ballot_sync(kFull, ge256),
                   v64k = __ballot_sync(kFull, ge64k);
    const int w = 1 + (ge24 ? 1 : 0) + (ge256 ? 1 : 0) + (ge64k ? 2 : 0);
    const int off = lane + __popc(v24 & lt) + __popc(v256 & lt) + 2 * __popc(v64k & lt);
    const int n_tok = BS + __popc(v24) + __popc(v256) + 2 * __popc(v64k);
    bool text = true;
    if (extra_off != nullptr) text = extra_off[k0 + i + 1] <= extra_off[k0 + i];
    {  // exactly w bytes per token (neighbouring lanes' ranges must not overlap); lane BS appends f6 for a nil extra;
       // predicated stores, no divergent branches
      const uint32_t d = (uint32_t)__cvta_generic_to_shared(raw[buf]) + (lane < BS ? off : n_tok);
      const uint32_t first = lane < BS ? head : 0xf6u;
      const int nst = lane < BS ? w : ((lane == BS && text) ? 1 : 0);
      asm volatile(
          "{\n\t.reg .pred p1, p2, p3, p4;\n\t"
          "setp.gt.s32 p1, %2, 0;\n\tsetp.gt.s32 p2, %2, 1;\n\tsetp.gt.s32 p3, %2, 2;\n\tsetp.gt.s32 p4, %2, 3;\n\t"
          "@p1 st.shared.u8 [%0], %1;\n\t@p2 st.shared.u8 [%0+1], %3;\n\t@p3 st.shared.u8 [%0+2], %4;\n\t"
          "@p4 st.shared.u8 [%0+3], %5;\n\t@p4 st.shared.u8 [%0+4], %6;\n\t}"
          :
          : "r"(d), "r"(first), "r"(nst), "r"(pay >> 24), "r"((pay >> 16) & 0xffu), "r"((pay >> 8) & 0xffu), "r"(pay & 0xffu)
          : "memory");
    }
    __syncwarp();
    const int n_tot = n_tok + (text ? 1 : 0);
    uint32_t word = 0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {  // unconditional loads from a clamped index, then selects
      const int pos = 3 * lane + j, idx = pos - kWpcPrefix;
      const uint32_t ld = raw[buf][idx < 0 ? 0 : idx];
      const uint32_t fixed = pos == 0 ? 0x83u : (pos == 1 ? 0x1bu : (pos == kWpcPrefix - 1 ? (0x80u | BS) : 0u));
      const uint32_t byte = (idx >= 0 && idx < n_tot) ? ld : fixed;
      word |= byte << (8 * j);
    }
    bw[buf][lane] = word;
    if (lane == 0) {
      const uint64_t pm = pw[kWpcPrefix + n_tot];
      meta[buf] = make_uint4((uint32_t)pm, (uint32_t)(pm >> 32), (uint32_t)n_tot, text ? 1u : 0u);
    }
  };

  // ---- folder constants: where the parent's bytes land in this lane's word, and Q^(3*lane + j)
  uint32_t psel = 0, pmask = 0;
  int32_t qlo[3];
  uint32_t qhi[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int pos = 3 * lane + j;
    if (pos >= 2 && pos <= 9) {  // stream position 2 + k carries parent byte 7 - k
      psel |= (uint32_t)(9 - pos) << (4 * j);
      pmask |= 0xffu << (8 * j);
    }
    const uint64_t q = pow_u64(kFnvPrimeInv, (uint32_t)pos);
    qlo[j] = (int32_t)(uint32_t)q;  // q = (qhi + [qlo < 0]) * 2^32 + (signed) qlo
    qhi[j] = (uint32_t)(q >> 32) + (qlo[j] < 0 ? 1u : 0u);
  }

  if (stager) {
    fetch_tokens(0);
    fetch_tokens(1);
    fetch_tokens(2);
  }
  if (stager) {
    stage(0);
    if (nblk > 1) stage(1);
  }
  __syncthreads();

  uint64_t parent = parents[p];
  uint32_t w_cur = 0;
  int n_cur = 0, text_cur = 1, cbuf = 0, nbuf = 1;  // buffers of block i and i + 1 (i % 3 without the division)
  uint64_t pw_cur = 0;
  if (!stager) {
    w_cur = bw[0][lane];
    const uint4 m = meta[0];
    pw_cur = ((uint64_t)m.y << 32) | m.x;
    n_cur = (int)m.z;
    text_cur = (int)m.w;
  }
#ifdef KVB_HASH_PROFILE
  long long wp[5] = {0, 0, 0, 0, 0};  // stager: work | folder: rounds, reduce+combine, rest | both: barrier wait
#define WPROF(slot, t_begin) wp[slot] += clock64() - (t_begin)
#else
#define WPROF(slot, t_begin)
#endif
  for (int i = 0; i < nblk; ++i) {
#ifdef KVB_HASH_PROFILE
    long long tb = clock64();
#endif
    if (stager) {
      if (i + 2 < nblk) stage(i + 2);
      WPROF(0, tb);
    } else {
      uint32_t w_nxt = 0;
      int n_nxt = 0, text_nxt = 1;
      uint64_t pw_nxt = 0;
      if (i + 1 < nblk) {  // staged during the previous interval, published by its barrier
        const int nb = nbuf;
        w_nxt = bw[nb][lane];
        const uint4 m = meta[nb];
        pw_nxt = ((uint64_t)m.y << 32) | m.x;
        n_nxt = (int)m.z;
        text_nxt = (int)m.w;
      }
      uint64_t key;
      if (parent >= 0x100000000ull) {
        const uint32_t w = w_cur | (__byte_perm((uint32_t)parent, (uint32_t)(parent >> 32), psel) & pmask);
        const uint32_t b0 = __byte_perm(w, 0u, 0x4440u), b1 = __byte_perm(w, 0u, 0x4441u), b2 = __byte_perm(w, 0u, 0x4442u);
        // z_j starts as b_j: bit k of z_j * 0xb3 is then exactly b_{j,k} ^ c_{j,k}; resolved l bits are xor-ed in.
        // Serial part of a round: IMAD -> LOP3 (xor3) -> LOP3.P -> VOTE -> LOP3 -> POPC -> SHL -> LOP3, ~61 cycles
        // (tools/micro/warp_chain_latency.cu); everything else is prepared while the vote is in flight.
        uint32_t z0 = b0, z1 = b1, z2 = b2;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          constexpr uint32_t kL0 = (uint32_t)(kFnvOffset & 0xffu);
          const uint32_t mask = 1u << k;
          const uint32_t p0 = z0 * 0xb3u, p1 = z1 * 0xb3u, p2 = z2 * 0xb3u;
          uint32_t votes;
          asm volatile(
              "{\n\t.reg .pred q;\n\t.reg .b32 g;\n\tlop3.b32 g, %1, %2, %3, 0x96;\n\tand.b32 g, g, %4;\n\t"
              "setp.ne.u32 q, g, 0;\n\tvote.sync.ballot.b32 %0, q, 0xffffffff;\n\t}"
              : "=r"(votes)
              : "r"(p0), "r"(p1), "r"(p2), "r"(mask));
          // l bit k at the lane's positions = l0 bit ^ parity(earlier lanes) ^ {0, t0, t0 ^ t1}: the local part now
          const uint32_t m0 = (kL0 & mask) ? mask : 0u;
          uint32_t zc0 = z0 ^ m0, zc1 = z1 ^ m0 ^ (p0 & mask), zc2 = z2 ^ m0 ^ ((p0 ^ p1) & mask);
          asm volatile("" : "+r"(zc0), "+r"(zc1), "+r"(zc2));  // keep them off the vote -> popc chain (no re-association)
          const uint32_t sh = (uint32_t)__popc(votes & lt) << k;  // parity of all earlier positions' toggles -> bit k
          // z = zc ^ (sh & mask) as ONE LOP3 each (the compiler would share sh & mask and add a level to the chain)
          asm("lop3.b32 %0, %1, %2, %3, 0x78;" : "=r"(z0) : "r"(zc0), "r"(sh), "r"(mask));
          asm("lop3.b32 %0, %1, %2, %3, 0x78;" : "=r"(z1) : "r"(zc1), "r"(sh), "r"(mask));
          asm("lop3.b32 %0, %1, %2, %3, 0x78;" : "=r"(z2) : "r"(zc2), "r"(sh), "r"(mask));
        }
        WPROF(1, tb);
#ifdef KVB_HASH_PROFILE
        tb = clock64();
#endif
        // e = z - l with l = z ^ b
        const int32_t e0 = (int32_t)z0 - (int32_t)(z0 ^ b0), e1 = (int32_t)z1 - (int32_t)(z1 ^ b1),
                      e2 = (int32_t)z2 - (int32_t)(z2 ^ b2);
        int64_t acc;  // three signed IMAD.WIDE (plain C++ widens both operands and emulates the 64-bit product)
        asm("{\n\t.reg .s64 t;\n\tmul.wide.s32 t, %1, %2;\n\tmad.wide.s32 t, %3, %4, t;\n\tmad.wide.s32 %0, %5, %6, t;\n\t}"
            : "=l"(acc)
            : "r"(e0), "r"(qlo[0]), "r"(e1), "r"(qlo[1]), "r"(e2), "r"(qlo[2]));
        const uint32_t hi = (uint32_t)e0 * qhi[0] + (uint32_t)e1 * qhi[1] + (uint32_t)e2 * qhi[2];
        // lane 0 carries the FNV offset basis into the sum
        const uint64_t tl = (uint64_t)acc + ((uint64_t)hi << 32) + (lane == 0 ? kFnvOffset : 0ull);
        const uint32_t tlo = (uint32_t)tl, thi = (uint32_t)(tl >> 32);
        const uint64_t s0 = __reduce_add_sync(kFull, tlo & 0xffffu), s1 = __reduce_add_sync(kFull, tlo >> 16),
                       s2 = __reduce_add_sync(kFull, thi & 0xffffu), s3 = __reduce_add_sync(kFull, thi >> 16);
        key = pw_cur * (s0 + (s1 << 16) + (s2 << 32) + (s3 << 48));
#ifdef KVB_HASH_PROFILE
        if (key == 0x1234u) wp[3] = 1;  // keep `key` live up to the clock read
#endif
        WPROF(2, tb);
#ifdef KVB_HASH_PROFILE
        tb = clock64();
#endif
      } else {  // short parent head: byte-serial fold, every lane the same
        Fnv h = fnv_init();
        fold_prefix(h, parent, (uint32_t)BS);
        const uint8_t* src = raw[cbuf];
        for (int k = 0; k < n_cur; ++k) fold(h, src[k]);
        key = fnv_value(h);
      }
      if (!text_cur) {  // pre-encoded X(extra_i) follows the tokens (extra_keys.go)
        Fnv h{(uint32_t)key, (uint32_t)(key >> 32)};
        for (int64_t e = extra_off[k0 + i]; e < extra_off[k0 + i + 1]; ++e) fold(h, extra[e]);
        key = fnv_value(h);
      }
      if (lane == 0) out_keys[k0 + i] = key;
      parent = key;
      w_cur = w_nxt;
      n_cur = n_nxt;
      text_cur = text_nxt;
      pw_cur = pw_nxt;
      cbuf = nbuf;
      nbuf = nbuf == 2 ? 0 : nbuf + 1;
      WPROF(3, tb);
    }
#ifdef KVB_HASH_PROFILE
    long long tw = clock64();
#endif
    __syncthreads();
    WPROF(4, tw);
  }
#ifdef KVB_HASH_PROFILE
  if (blockIdx.x == 0 && lane == 0) {
    long long* dst = g_hash_prof + (stager ? 0 : 5);
    for (int q = 0; q < 5; ++q) dst[q] = wp[q];
    g_hash_prof[10] = nblk;
  }
#endif
#undef WPROF
}

// ---------------------------------------------------------------------------------------------------------------
// chain kernel (round 2): one CTA per prompt, warp 0 FOLDS the chain, warps 1..NST STAGE blocks ahead of it, and — in
// the fused tokens -> scores form — one more warp SCORES the keys as they appear (probes and the longest-prefix walk run
// under the hash chain; only the last tile of keys is left when the chain ends).  Same T-function rounds as
// hash_chain_kernel_wpc, with these differences:
//   * no CTA barrier per block: staged blocks sit in a ring of S slots, the warps exchange progress counters in shared
//     memory (stagers publish with release, the folder reads the counter one block ahead of its use, so no memory
//     latency sits on the chain), tokens are fetched TR blocks ahead with cp.async;
//   * key = sum_i e_i * P^(m - i) + P^m * H0: the per-position constants are table entries indexed by (stream length -
//     position), looked up by the stager; the offset-basis term rides on position 0, whose byte (0x83) and therefore
//     e_0 = 129 are constant: c_0' = P^m * (1 + H0 * 129^-1).  Nothing is multiplied after the warp reduction;
//   * the 64-bit warp sum is three REDUX instead of four: low words mod 2^32, the EXACT sum of their upper halves
//     (21 bits, which recovers the carry), high words mod 2^32;
//   * one staged block is ONE 32 B record per lane (two 128-bit shared loads for the folder);
//   * MERGED (A/B): bits 0 and 1 of every z byte without a vote.  Mod 4, x -> 0xb3 * x is the GF(2)-linear map
//     (z1, z0) -> (z1 ^ z0, z0), so bits 0/1 of the running low byte are XOR prefixes of bits 0/1 of the stream; the
//     stager resolves them for the stream with the parent bytes ZEROED (six ballots, off the chain) and the folder adds
//     the parent's contribution with two 64-bit masks per position and one popcount each: six vote rounds instead of
//     eight, at the price of more instructions in both warps.
// A lone in-order warp retires about one instruction per three cycles (tools/micro/hash_phase_profile.cu), so the
// folder's INSTRUCTION COUNT is on the chain as much as its dependency depth: everything that does not depend on the
// parent key is done by the stagers.  The arithmetic is restated on the CPU in tests/test_wpc_math.py.
constexpr int kV2Slots = 4;    // staged blocks the stagers may run ahead
constexpr int kV2TokRing = 8;  // token blocks in flight (cp.async commit groups), power of two
constexpr uint64_t kInv129 = inv_mod_2_64(129);
static_assert(kInv129 * 129ull == 1ull, "129^-1 mod 2^64");
constexpr uint64_t kBasisOnPos0 = 1ull + kFnvOffset * kInv129;  // c_0' = P^m * kBasisOnPos0

__device__ __forceinline__ int ld_acquire_cta(const int* p) {
  int v;
  asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(v) : "r"((uint32_t)__cvta_generic_to_shared(p)) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_cta(int* p, int v) {
  asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(p)), "r"(v) : "memory");
}

// fused form: the last prompt to finish tells the host through a word in pinned memory, so the caller can watch that word
// instead of paying a stream synchronisation after the kernel has already ended
__device__ __forceinline__ void chain_signal_done(const ChainArgs& A) {
  if (A.done_counter == nullptr) return;
  __threadfence_system();  // this prompt's results (possibly written to pinned host memory) before the count
  if (A.done_target == 1u) {  // one prompt: nobody to count
    *reinterpret_cast<volatile unsigned long long*>(A.done_flag_host) = A.done_value;
    return;
  }
  const unsigned prev = atomicAdd(A.done_counter, 1u);
  if (prev + 1u == A.done_target) {
    *A.done_counter = 0u;  // ready for the next call (stream order: no other launch touches it before this one ends)
    __threadfence_system();
    *reinterpret_cast<volatile unsigned long long*>(A.done_flag_host) = A.done_value;
  }
}

template <int BS, bool MERGED, bool SCORE, int CHUNK_TOK = 128, int LOOKAHEAD = 2>
__global__ void __launch_bounds__(32 * (2 + (SCORE ? 1 : 0))) chain_kernel(const ChainArgs A) {
  static_assert(BS > 0 && BS < 24 && kWpcPrefix + 5 * BS + 1 <= kWpcPositions, "stream must fit 96 positions");
  constexpr uint32_t kFull = 0xffffffffu;
  constexpr int NST = 1;  // one stager warp keeps up (a second one gains nothing: tests/bench_hash.py)
  constexpr int S = kV2Slots, NT = 32 * (1 + NST + (SCORE ? 1 : 0));
  // token chunks: CHUNK_TOK tokens each (CHUNK_TOK / 128 16-byte granules per lane), LOOKAHEAD chunks in flight beyond
  // the one being consumed, ring of the next power of two >= LOOKAHEAD + 2 chunks
  constexpr int kChunkTok = CHUNK_TOK, kLookahead = LOOKAHEAD, kGran = CHUNK_TOK / 128;
  constexpr int kChunks = (LOOKAHEAD + 2) <= 4 ? 4 : 8, kRingTok = kChunkTok * kChunks;
  static_assert(CHUNK_TOK % 128 == 0 && LOOKAHEAD + 2 <= kChunks, "chunk geometry");
  constexpr int kKeyRing = 64;
  // per staged block and lane: {w, c0.lo, c0.hi', c1.lo} {c1.hi', c2.lo, c2.hi', n_tot | text << 31}; w = the lane's 3
  // stream bytes (parent bytes zero) [+ static z bits 0/1 in bits 24..29 when MERGED]; c_j = P^(m - position), split for
  // signed 32 x 32 products; raw = the token bytes for the byte-serial fallback
  __shared__ uint4 rec[S][2][32];
  __shared__ uint8_t raw[S][kWpcPositions];
  __shared__ __align__(16) uint32_t tring[kRingTok];  // token ring: chunks of 128 tokens, fetched 16 B per lane
  __shared__ uint64_t pw[kWpcPositions + 1];  // P^t
  __shared__ int staged, folded, scored;      // blocks published by the stager / folded / consumed by the scorer
  __shared__ uint64_t skeys[SCORE ? kKeyRing : 1];
  __shared__ Bucket tile[SCORE ? 32 : 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int p = blockIdx.x;
  // a single prompt travels in the kernel arguments: no array to read before the chain can start
  const int64_t t0 = A.single ? 0 : A.prompt_off[p];
  const int64_t t1 = A.single ? A.single_tokens : A.prompt_off[p + 1];
  const int nblk = (int)((t1 - t0) / BS);  // tail tokens dropped (token_processor.go:166-168)
  if (nblk == 0) {
    if (SCORE && threadIdx.x == 0) {
      A.out_n[p] = 0;
      chain_signal_done(A);
    }
    return;
  }
  const int64_t k0 = A.single ? 0 : A.key_off[p];
  for (int t = threadIdx.x; t <= kWpcPositions; t += NT) pw[t] = pow_u64(kFnvPrime, (uint32_t)t);
  if (threadIdx.x == 0) {
    staged = 0;
    folded = 0;
    scored = 0;
  }
  __syncthreads();  // the only CTA barrier: publishes pw[] and the counters
  const uint32_t lt = (1u << lane) - 1u, self = 1u << lane;

  if (warp >= 1 && warp <= NST) {
    // ------------------------------------------------------------------------------------------------ stager
    uint32_t le[3][3], lso[3][3];  // MERGED: lanes whose slot-j' position is <= / < (opposite parity) position j
    if (MERGED) {
#pragma unroll
      for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int jp = 0; jp < 3; ++jp) {
          le[j][jp] = lt | (jp <= j ? self : 0u);
          const uint32_t opp = ((3 * lane + j + jp) & 1) ? 0x55555555u : 0xaaaaaaaau;  // position 3L+j has parity (L+j)&1
          lso[j][jp] = (lt | (jp < j ? self : 0u)) & opp;
        }
    }
    constexpr uint32_t l00 = (uint32_t)(kFnvOffset & 1u), l01 = (uint32_t)((kFnvOffset >> 1) & 1u);
    // tokens arrive in chunks of 128 (one 16 B granule per lane: a single warp instruction moves 512 B, which matters
    // when the source is pinned HOST memory read in place over PCIe); the prompt need not start on a granule boundary —
    // the granules are taken from the aligned superset, and granules that stick out of the caller's array fall back to
    // 4 B copies of the tokens that are inside it
    const uint32_t* tk = A.tokens + t0;
    // The chunk grid is aligned to 128 B lines, not just to the 16 B granule: sysmem is read a line at a time, and a chunk
    // that straddles lines makes the link fetch its boundary lines twice (tools/micro/pinned_read_bw.cu compares the
    // grids with a plain streaming read)
    const int mis = (int)((reinterpret_cast<uintptr_t>(tk) >> 2) & 31u);  // tokens between the 128 B boundary and tk
    const uint32_t* tka = tk - mis;
    const int need_hi = mis + nblk * BS;                                  // aligned token indices [mis, need_hi) are needed
    auto fetch_chunk = [&](int c) {  // one commit group per chunk, empty past the end so the group count stays uniform
#pragma unroll
      for (int g = 0; g < kGran; ++g) {
        const int a0 = c * kChunkTok + (g * 32 + lane) * 4;
        if (a0 + 3 >= mis && a0 < need_hi) {
          const uint32_t* src = tka + a0;
          const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&tring[a0 & (kRingTok - 1)]);
          if (src >= A.tokens_lo && src + 4 <= A.tokens_hi) {
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src));
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q)
              if (src + q >= A.tokens_lo && src + q < A.tokens_hi)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst + 4 * q), "l"(src + q));
          }
        }
      }
      asm volatile("cp.async.commit_group;");
    };
    int committed = 0;
    for (int i = 0; i < nblk; ++i) {
      const int buf = i % S;
      const int c_need = (mis + i * BS + BS - 1) / kChunkTok;
      while (committed <= c_need + kLookahead) fetch_chunk(committed++);
      asm volatile("cp.async.wait_group %0;" ::"n"(kLookahead) : "memory");  // all but the newest chunks: block i landed
      if (i >= S)
        while (ld_acquire_cta(&folded) < i - S + 1) __nanosleep(64);  // until the slot's previous block is consumed
      // (waiting warps sleep instead of spinning: at 1024 prompts five warps share a scheduler and a spinning one takes
      //  issue slots from a folding one, and most of the kernel's instructions become polls)
      __syncwarp();  // a chunk is written by all lanes and read by others
      const uint32_t t = lane < BS ? tring[(mis + i * BS + lane) & (kRingTok - 1)] : 0u;
      const bool ge24 = t >= 24u, ge256 = t >= 0x100u, ge64k = t >= 0x10000u;
      const uint32_t head = ge64k ? 0x1au : (ge256 ? 0x19u : (ge24 ? 0x18u : t));
      const uint32_t pay = ge64k ? t : (ge256 ? (t << 16) : (t << 24));  // payload, left-aligned big-endian
      const uint32_t v24 = __ballot_sync(kFull, ge24), v256 = __ballot_sync(kFull, ge256),
                     v64k = __ballot_sync(kFull, ge64k);
      const int w = 1 + (ge24 ? 1 : 0) + (ge256 ? 1 : 0) + (ge64k ? 2 : 0);
      const int off = lane + __popc(v24 & lt) + __popc(v256 & lt) + 2 * __popc(v64k & lt);
      const int n_tok = BS + __popc(v24) + __popc(v256) + 2 * __popc(v64k);
      bool text = true;
      if (A.extra_off != nullptr) text = A.extra_off[k0 + i + 1] <= A.extra_off[k0 + i];
      {  // exactly w bytes per token; lane BS appends f6 for a nil extra; predicated stores, no divergent branches
        const uint32_t d = (uint32_t)__cvta_generic_to_shared(raw[buf]) + (lane < BS ? off : n_tok);
        const uint32_t first_b = lane < BS ? head : 0xf6u;
        const int nst = lane < BS ? w : ((lane == BS && text) ? 1 : 0);
        asm volatile(
            "{\n\t.reg .pred p1, p2, p3, p4;\n\t"
            "setp.gt.s32 p1, %2, 0;\n\tsetp.gt.s32 p2, %2, 1;\n\tsetp.gt.s32 p3, %2, 2;\n\tsetp.gt.s32 p4, %2, 3;\n\t"
            "@p1 st.shared.u8 [%0], %1;\n\t@p2 st.shared.u8 [%0+1], %3;\n\t@p3 st.shared.u8 [%0+2], %4;\n\t"
            "@p4 st.shared.u8 [%0+3], %5;\n\t@p4 st.shared.u8 [%0+4], %6;\n\t}"
            :
            : "r"(d), "r"(first_b), "r"(nst), "r"(pay >> 24), "r"((pay >> 16) & 0xffu), "r"((pay >> 8) & 0xffu), "r"(pay & 0xffu)
            : "memory");
      }
      __syncwarp();
      const int n_tot = n_tok + (text ? 1 : 0);
      uint32_t word = 0;
#pragma unroll
      for (int j = 0; j < 3; ++j) {  // unconditional loads from a clamped index, then selects
        const int pos = 3 * lane + j, idx = pos - kWpcPrefix;
        const uint32_t ld = raw[buf][idx < 0 ? 0 : idx];
        const uint32_t fixed = pos == 0 ? 0x83u : (pos == 1 ? 0x1bu : (pos == kWpcPrefix - 1 ? (0x80u | BS) : 0u));
        const uint32_t byte = (idx >= 0 && idx < n_tot) ? ld : fixed;
        word |= byte << (8 * j);
      }
      if (MERGED) {  // static bits 0/1 of z at this lane's three positions, parent bytes taken as zero
        uint32_t v0[3], v1[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          v0[j] = __ballot_sync(kFull, (word >> (8 * j)) & 1u);
          v1[j] = __ballot_sync(kFull, (word >> (8 * j + 1)) & 1u);
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const uint32_t x0 = (v0[0] & le[j][0]) ^ (v0[1] & le[j][1]) ^ (v0[2] & le[j][2]);
          const uint32_t x1 = (v1[0] & le[j][0]) ^ (v1[1] & le[j][1]) ^ (v1[2] & le[j][2]);
          const uint32_t xa = (v0[0] & lso[j][0]) ^ (v0[1] & lso[j][1]) ^ (v0[2] & lso[j][2]);
          const uint32_t z0 = (l00 ^ (uint32_t)__popc(x0)) & 1u;
          const uint32_t z1 = (l01 ^ (((3 * lane + j) & 1) ? l00 : 0u) ^ (uint32_t)(__popc(x1) + __popc(xa))) & 1u;
          word |= (z0 | (z1 << 1)) << (24 + 2 * j);
        }
      }
      // per-position constants P^(m - position); position 0 also carries the offset-basis term
      const int m = kWpcPrefix + n_tot;
      uint32_t clo[3], chi[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int d = m - (3 * lane + j);
        uint64_t c = pw[d < 0 ? 0 : d];
        if (j == 0 && lane == 0) c *= kBasisOnPos0;
        const int32_t lo = (int32_t)(uint32_t)c;  // c = (hi' ) * 2^32 + (signed) lo with hi' = hi + [lo < 0]
        clo[j] = (uint32_t)lo;
        chi[j] = (uint32_t)(c >> 32) + (lo < 0 ? 1u : 0u);
      }
      rec[buf][0][lane] = make_uint4(word, clo[0], chi[0], clo[1]);
      rec[buf][1][lane] = make_uint4(chi[1], clo[2], chi[2], (uint32_t)n_tot | (text ? 0x80000000u : 0u));
      // Publish with a plain store after the warp barrier — NOT st.release: a release compiles to MEMBAR.ALL.CTA, and the
      // membar waits for every memory operation this warp has in flight, i.e. for the token chunks being prefetched from
      // host memory.  That serialised each block behind a PCIe round trip.  Ordering still holds: the record stores of all lanes precede the barrier, the
      // counter store follows it, and one SM's shared-memory pipeline performs them in that order; readers poll the
      // counter before they load the record.
      __syncwarp();
      if (lane == 0) *reinterpret_cast<volatile int*>(&staged) = i + 1;
    }
    return;
  }

  if (SCORE && warp == 1 + NST) {
    // ------------------------------------------------------------------------------------------------ scorer
    ScoreWalker wk;
    // keys are taken as they appear: at least `score_min_batch` at a time (a probe costs a DRAM round trip whatever the
    // batch, so a lone prompt is followed a few keys behind and only those are left when its chain ends; a large batch
    // waits for full tiles, fewer instructions), never more than 32
    for (int base = 0; base < nblk;) {
      const int want = min(A.score_min_batch, nblk - base);
      int avail;
      while ((avail = ld_acquire_cta(&folded) - base) < want) __nanosleep(A.score_min_batch >= 32 ? 400 : 40);
      const int in_tile = min(avail, 32);
      const uint64_t key = lane < in_tile ? skeys[(base + lane) & (kKeyRing - 1)] : 0ull;
      __syncwarp();
      if (lane == 0) *reinterpret_cast<volatile int*>(&scored) = base + in_tile;  // the ring slots may be reused
      if (wk.chain_alive || A.ts != nullptr)  // else: nothing left to add and nothing to stamp
        wk.tile(A.table, A.mask, tile, key, lane < in_tile, base, in_tile, A.filter_bits, A.tier_w, A.ts,
                A.stamp_base + (unsigned long long)(k0 + base + lane));
      base += in_tile;
    }
    wk.finish(p, A.out_n, A.out_pods, A.out_scores);
    __syncwarp();
    if (lane == 0) chain_signal_done(A);
    return;
  }

  // -------------------------------------------------------------------------------------------------- folder
  // where the parent's bytes land in this lane's word (stream position 2 + k carries parent byte 7 - k)
  uint32_t psel = 0, pmask = 0;
  uint32_t m0lo[3], m0hi[3], m1lo[3], m1hi[3];  // MERGED: z0 ^= parity(parent & m0), z1 ^= parity(parent & m1)
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int pos = 3 * lane + j;
    if (pos >= 2 && pos <= 9) {
      psel |= (uint32_t)(9 - pos) << (4 * j);
      pmask |= 0xffu << (8 * j);
    }
    // m0 = bit 0 of the parent bytes at positions <= pos; m1 = their bit 1, plus bit 0 of those at positions < pos of
    // the opposite position parity (the cross term of the mod-4 map)
    uint64_t mle = 0, mopp = 0;
    for (int q = 2; q <= 9; ++q) {
      if (q <= pos) mle |= 1ull << (8 * (9 - q));
      if (q < pos && ((pos - q) & 1)) mopp |= 1ull << (8 * (9 - q));
    }
    const uint64_t m1 = (mle << 1) | mopp;
    m0lo[j] = (uint32_t)mle;
    m0hi[j] = (uint32_t)(mle >> 32);
    m1lo[j] = (uint32_t)m1;
    m1hi[j] = (uint32_t)(m1 >> 32);
  }
#ifdef KVB_HASH_PROFILE
  // clock reads that cannot issue before `dep` is ready: they sit ON the dependent chain, like the next real instruction
  long long vp[6] = {0, 0, 0, 0, 0, 0};  // top (check + loads) | prefix / bits 0,1 | rounds | reduce | tail
  auto clk = [](uint32_t dep) {
    long long t;
    asm volatile("{\n\t.reg .b32 d;\n\tmov.b32 d, %1;\n\tmov.u64 %0, %%clock64;\n\t}" : "=l"(t) : "r"(dep) : "memory");
    return t;
  };
#define VPROF(slot, t_begin, dep)  \
  {                                \
    const long long _n = clk(dep); \
    vp[slot] += _n - (t_begin);    \
    (t_begin) = _n;                \
  }
#else
#define VPROF(slot, t_begin, dep)
#endif
  uint64_t parent = A.single ? A.single_parent : A.parents[p];
  int seen = 0;  // last value read from `staged`: the stagers run ahead, so the check below rarely has to look again
  while ((seen = ld_acquire_cta(&staged)) < 1) __nanosleep(20);
  uint4 ra = rec[0][0][lane], rb = rec[0][1][lane];
  int cbuf = 0, nbuf = 1, scored_seen = 0;
#ifdef KVB_HASH_PROFILE
  long long tb = clk((uint32_t)parent);
#endif
  for (int i = 0; i < nblk; ++i) {
    uint4 ra_n = make_uint4(0, 0, 0, 0), rb_n = make_uint4(0, 0, 0, 0x80000000u);
    int seen_nxt = seen;
    if (i + 1 < nblk) {
      // block i + 1 was normally published long ago and `seen` (read an iteration ago) already says so: the compare is
      // on a register, the loads are issued at once and consumed only when the next block starts
      while (seen < i + 2) {
        seen = ld_acquire_cta(&staged);
        if (seen < i + 2) __nanosleep(40);  // the stager is waiting for tokens (host memory read in place): do not spin
      }
      ra_n = rec[nbuf][0][lane];
      rb_n = rec[nbuf][1][lane];
      seen_nxt = *reinterpret_cast<volatile int*>(&staged);  // for the next iteration's check; not waited for here
    }
    VPROF(0, tb, (uint32_t)parent);
    const uint32_t w_cur = ra.x;
    uint64_t key;
    if (parent >= 0x100000000ull) {
      const uint32_t klo = (uint32_t)parent, khi = (uint32_t)(parent >> 32);
      const uint32_t w = (w_cur & 0x00ffffffu) | (__byte_perm(klo, khi, psel) & pmask);
      const uint32_t b0 = __byte_perm(w, 0u, 0x4440u), b1 = __byte_perm(w, 0u, 0x4441u), b2 = __byte_perm(w, 0u, 0x4442u);
      uint32_t z0, z1, z2;
      if (MERGED) {  // bits 0/1: static part from the stager, parent part from two masked popcounts per position
        const uint32_t q00 = (uint32_t)__popc((klo & m0lo[0]) ^ (khi & m0hi[0])), q10 = (uint32_t)__popc((klo & m1lo[0]) ^ (khi & m1hi[0]));
        const uint32_t q01 = (uint32_t)__popc((klo & m0lo[1]) ^ (khi & m0hi[1])), q11 = (uint32_t)__popc((klo & m1lo[1]) ^ (khi & m1hi[1]));
        const uint32_t q02 = (uint32_t)__popc((klo & m0lo[2]) ^ (khi & m0hi[2])), q12 = (uint32_t)__popc((klo & m1lo[2]) ^ (khi & m1hi[2]));
        const uint32_t s0 = w_cur >> 24, s1 = w_cur >> 26, s2 = w_cur >> 28;
        z0 = (b0 & 0xfcu) | ((s0 ^ (q00 & 1u) ^ ((q10 & 1u) << 1)) & 3u);
        z1 = (b1 & 0xfcu) | ((s1 ^ (q01 & 1u) ^ ((q11 & 1u) << 1)) & 3u);
        z2 = (b2 & 0xfcu) | ((s2 ^ (q02 & 1u) ^ ((q12 & 1u) << 1)) & 3u);
      } else {  // z starts as b: bit k of z * 0xb3 is then exactly b_k ^ c_k
        z0 = b0;
        z1 = b1;
        z2 = b2;
      }
      VPROF(1, tb, z0 ^ z1 ^ z2);
      // the dependent rounds (IMAD -> LOP3 -> LOP3.P -> VOTE -> LOP3 -> POPC -> SHL -> LOP3 each)
#pragma unroll
      for (int k = MERGED ? 2 : 0; k < 8; ++k) {
        constexpr uint32_t kL0 = (uint32_t)(kFnvOffset & 0xffu);
        const uint32_t mask = 1u << k;
        const uint32_t p0 = z0 * 0xb3u, p1 = z1 * 0xb3u, p2 = z2 * 0xb3u;
        uint32_t votes;
        asm volatile(
            "{\n\t.reg .pred q;\n\t.reg .b32 g;\n\tlop3.b32 g, %1, %2, %3, 0x96;\n\tand.b32 g, g, %4;\n\t"
            "setp.ne.u32 q, g, 0;\n\tvote.sync.ballot.b32 %0, q, 0xffffffff;\n\t}"
            : "=r"(votes)
            : "r"(p0), "r"(p1), "r"(p2), "r"(mask));
        const uint32_t mm = (kL0 & mask) ? mask : 0u;
        uint32_t zc0 = z0 ^ mm, zc1 = z1 ^ mm ^ (p0 & mask), zc2 = z2 ^ mm ^ ((p0 ^ p1) & mask);
        asm volatile("" : "+r"(zc0), "+r"(zc1), "+r"(zc2));  // keep them off the vote -> popc chain (no re-association)
        const uint32_t sh = (uint32_t)__popc(votes & lt) << k;  // parity of all earlier positions' toggles -> bit k
        asm("lop3.b32 %0, %1, %2, %3, 0x78;" : "=r"(z0) : "r"(zc0), "r"(sh), "r"(mask));
        asm("lop3.b32 %0, %1, %2, %3, 0x78;" : "=r"(z1) : "r"(zc1), "r"(sh), "r"(mask));
        asm("lop3.b32 %0, %1, %2, %3, 0x78;" : "=r"(z2) : "r"(zc2), "r"(sh), "r"(mask));
      }
      VPROF(2, tb, z0 ^ z1 ^ z2);
      // e = z - l with l = z ^ b;  key = sum_i e_i * c_i (the offset-basis term rides on position 0)
      const int32_t e0 = (int32_t)z0 - (int32_t)(z0 ^ b0), e1 = (int32_t)z1 - (int32_t)(z1 ^ b1),
                    e2 = (int32_t)z2 - (int32_t)(z2 ^ b2);
      int64_t acc;  // three signed IMAD.WIDE
      asm("{\n\t.reg .s64 t;\n\tmul.wide.s32 t, %1, %2;\n\tmad.wide.s32 t, %3, %4, t;\n\tmad.wide.s32 %0, %5, %6, t;\n\t}"
          : "=l"(acc)
          : "r"(e0), "r"((int32_t)ra.y), "r"(e1), "r"((int32_t)ra.w), "r"(e2), "r"((int32_t)rb.y));
      const uint32_t hi = (uint32_t)e0 * ra.z + (uint32_t)e1 * rb.x + (uint32_t)e2 * rb.z;
      const uint32_t tlo = (uint32_t)acc, thi = (uint32_t)((uint64_t)acc >> 32) + hi;
      const uint32_t r1 = __reduce_add_sync(kFull, tlo), r2 = __reduce_add_sync(kFull, tlo >> 16),
                     r3 = __reduce_add_sync(kFull, thi);
      const uint32_t a = r2 << 16;  // exact low sum = (r2 << 16) + B with B < 2^21, and its low word is r1
      const uint32_t carry = (r2 >> 16) + (r1 < a ? 1u : 0u);
      key = ((uint64_t)(r3 + carry) << 32) | r1;
    } else {  // short parent head (a caller-supplied root below 2^32): byte-serial fold, every lane the same
      Fnv h = fnv_init();
      fold_prefix(h, parent, (uint32_t)BS);
      const uint8_t* src = raw[cbuf];
      const int n_cur = (int)(rb.w & 0x7fffffffu);
      for (int k = 0; k < n_cur; ++k) fold(h, src[k]);
      key = fnv_value(h);
    }
    if (!(rb.w & 0x80000000u)) {  // pre-encoded X(extra_i) follows the tokens (extra_keys.go)
      Fnv h{(uint32_t)key, (uint32_t)(key >> 32)};
      for (int64_t e = A.extra_off[k0 + i]; e < A.extra_off[k0 + i + 1]; ++e) fold(h, A.extra[e]);
      key = fnv_value(h);
    }
    VPROF(3, tb, (uint32_t)key ^ (uint32_t)(key >> 32));
    if (SCORE) {  // the key ring is 64 deep and the scorer consumes 32 at a time: it is normally far ahead of this check
      while (i - scored_seen >= kKeyRing) {
        scored_seen = ld_acquire_cta(&scored);
        if (i - scored_seen >= kKeyRing) __nanosleep(64);
      }
    }
    if (lane == 0) {
      if (SCORE) skeys[i & (kKeyRing - 1)] = key;
      // slot i may be restaged: its record is in registers and raw[] has been read — every value the key depends on has
      // arrived, so a relaxed store is enough (a release here would put a MEMBAR, and the wait for the global store
      // below, on the chain).  The key store above and this counter store come from the same thread, in order.
      *reinterpret_cast<volatile int*>(&folded) = i + 1;
      if (A.out_keys != nullptr) A.out_keys[k0 + i] = key;
    }
    parent = key;
    ra = ra_n;
    rb = rb_n;
    seen = seen_nxt > seen ? seen_nxt : seen;
    if (SCORE) {
      const int sc = *reinterpret_cast<volatile int*>(&scored);
      scored_seen = sc > scored_seen ? sc : scored_seen;
    }
    cbuf = nbuf;
    nbuf = nbuf == S - 1 ? 0 : nbuf + 1;
    VPROF(4, tb, (uint32_t)parent);
  }
#ifdef KVB_HASH_PROFILE
  if (blockIdx.x == 0 && lane == 0) {
    for (int q = 0; q < 5; ++q) g_hash_prof[5 + q] = vp[q];
    g_hash_prof[10] = nblk;
  }
#endif
#undef VPROF
}

template <int BS, bool SCORE>
static void launch_chain_bs(const ChainArgs& a, int n_prompts, cudaStream_t s) {
  // MERGED (bits 0/1 without votes) shortens a lone chain but costs instructions in both warps: it pays while every
  // folder has a scheduler to itself and loses when they share one.  On H100 the two measure the same from 16 to 2048
  // prompts (tests/bench_hash.py), so the switch point is kept.  A/B: KVB_HASH_MERGED
  const char* e2 = std::getenv("KVB_HASH_MERGED");
  const bool merged = e2 ? std::atoi(e2) != 0 : n_prompts <= 512;
  // token fetch geometry (A/B: KVB_CHAIN_FETCH = 128x2 | 256x2 | 256x4 | 128x6): chunk size in tokens x chunks ahead
  const char* e3 = std::getenv("KVB_CHAIN_FETCH");
  const int geo = !e3 ? 0 : (!std::strcmp(e3, "256x2") ? 1 : (!std::strcmp(e3, "256x4") ? 2 : (!std::strcmp(e3, "128x6") ? 3 : 0)));
  const int threads = 32 * (2 + (SCORE ? 1 : 0));
  if (merged) {
    chain_kernel<BS, true, SCORE><<<n_prompts, threads, 0, s>>>(a);
    return;
  }
  switch (geo) {
    case 1: chain_kernel<BS, false, SCORE, 256, 2><<<n_prompts, threads, 0, s>>>(a); break;
    case 2: chain_kernel<BS, false, SCORE, 256, 4><<<n_prompts, threads, 0, s>>>(a); break;
    case 3: chain_kernel<BS, false, SCORE, 128, 6><<<n_prompts, threads, 0, s>>>(a); break;
    default: chain_kernel<BS, false, SCORE><<<n_prompts, threads, 0, s>>>(a);
  }
}

static bool chain_kernel_supports(int32_t block_size) { return block_size == 16 || block_size == 8 || block_size == 4; }

// fused tokens -> keys -> lookup -> scores, one launch (kvb_index_score_tokens_batch); false if this block size has no
// chain kernel (the caller then hashes and scores with two launches)
bool launch_chain_score(const ChainArgs& a, int32_t n_prompts, int32_t block_size, cudaStream_t s) {
  if (!chain_kernel_supports(block_size)) return false;
  if (block_size == 16) launch_chain_bs<16, true>(a, n_prompts, s);
  else if (block_size == 8) launch_chain_bs<8, true>(a, n_prompts, s);
  else launch_chain_bs<4, true>(a, n_prompts, s);
  count_launch();
  return true;
}

// ------------------------------------------------------------------------------------------------------------------
// "Spec" kernel for small batches: take the token bytes OFF the chain.
//
// FNV-1a is  h <- (h ^ b) * P.  The xor touches only the low byte, and the low byte of a product depends only on the
// low bytes of its factors, so with h = u + l (l = low byte, u = the rest):
//     fold(h, bytes[0..m)) = u * P^m + fold(l, bytes[0..m))                                    (mod 2^64, exactly)
// A block's byte stream is  83 | U(parent) | tail  where  tail = array-head(bs) | tokens | extra  does not depend on
// the chain.  So fold(v, tail) is tabulated for all 256 values of v — 256 independent plain FNV runs per block, in
// parallel over every block of every prompt (phase A: one 128-thread CTA per block, two start values per thread) —
// and the serial chain per block shrinks to the 10 prefix bytes plus one table look-up and one multiply by P^m (phase B:
// one thread per prompt): about a third of the cycles per block of the vote rounds.  The price is 256x the byte
// work, which idle SMs absorb for small batches only (the vote kernels stay the choice from a few dozen prompts up).
constexpr int kSpecThreads = 128;   // each thread folds TWO start values (two independent chains: the warp's issue slots
                                    // are half empty with one), so a 128-thread CTA tabulates a block
constexpr int kSpecPassRows = 8;    // table rows (blocks) per staging buffer; two buffers: 2 x 8 x 2 KiB — small, so that
                                    // six CTAs fit an SM while the tables are being built
constexpr int kSpecChunk = 640;     // tail bytes staged per round (128 tokens x 5 B)
constexpr int kSpecMaxPrompts = 64;
constexpr int kSpecAutoPrompts = 16;  // the small argument block holds this many prompts
constexpr int kSpecDefaultPrompts = 32;  // chosen without being asked for up to this many prompts (H100 fused call,
                                          // tests/bench_small_batches.py: 47 vs 53 us at 32 prompts, 62 vs 55 us at 64)
constexpr int kSpecKeyRing = 64;

struct SpecArgs {
  int32_t n_prompts, block_size;
  int64_t total_keys;
  uint64_t* table;  // [total_keys][256]  fold(v, tail_k)
  uint64_t* pm;     // [total_keys]       P^len(tail_k)
  unsigned* done;   // [n_prompts] tables finished per prompt; zero at launch, reset by the prompt's CTA
  unsigned* next_task;  // task counter: a launch with T tasks advances it by exactly T (one fetch per executed task)
  unsigned task_base;   // its value at launch
  int32_t inl;      // offsets / parents are in the SpecInline argument (else in the ChainArgs arrays)
};
// Prompt offsets, key offsets and parents in the launch arguments: no array to fetch before the first table can start (the
// fused call otherwise keeps them in pinned HOST memory, a PCIe round trip per dependent read).  Two sizes, because the
// argument block is copied at every launch: 16 prompts (0.4 KiB) for the common case, 64 (1.5 KiB) above.
template <int N>
struct SpecInline {
  int64_t koff[N + 1], poff[N + 1];
  uint64_t par[N];
};

__device__ __forceinline__ uint64_t pow_prime(uint32_t e) {
  uint64_t r = 1, b = kFnvPrime;
  while (e) {
    if (e & 1u) r *= b;
    b *= b;
    e >>= 1;
  }
  return r;
}

// all threads fold the n staged bytes into both of their states (same bytes for every thread: shared-memory broadcasts)
__device__ __forceinline__ void spec_fold_chunk(Fnv& h, Fnv& g, const uint32_t* words, int n) {
  const int nw = n >> 2;
  int i = 0;
  for (; i + 4 <= nw; i += 4) {
    const uint4 q = *reinterpret_cast<const uint4*>(words + i);
    fold4(h, q.x);
    fold4(g, q.x);
    fold4(h, q.y);
    fold4(g, q.y);
    fold4(h, q.z);
    fold4(g, q.z);
    fold4(h, q.w);
    fold4(g, q.w);
  }
  for (; i < nw; ++i) {
    fold4(h, words[i]);
    fold4(g, words[i]);
  }
  const int tail = n & 3;
  if (tail) {
    const uint32_t tw = words[nw];
    fold(h, tw & 0xffu);
    fold(g, tw & 0xffu);
    if (tail > 1) {
      fold(h, (tw >> 8) & 0xffu);
      fold(g, (tw >> 8) & 0xffu);
    }
    if (tail > 2) {
      fold(h, (tw >> 16) & 0xffu);
      fold(g, (tw >> 16) & 0xffu);
    }
  }
}

constexpr uint64_t kSpecAfter831b = (((kFnvOffset ^ 0x83ull) * kFnvPrime) ^ 0x1bull) * kFnvPrime;  // state after 83 1b

__device__ __forceinline__ void spec_wait_ge(const int* p, int v) {
  while (ld_acquire_cta(p) < v) __nanosleep(20);
}

// A: the chain kernel's arguments (tokens may be pinned host memory read in place; `single` = one prompt whose offsets
// travel in the arguments; SCORE adds lookup + longest-prefix scores by a scorer warp that follows the chain)
template <bool SCORE, int NIN>
__global__ void __launch_bounds__(kSpecThreads) hash_spec_kernel(const ChainArgs A, const SpecArgs X, const SpecInline<NIN> I) {
  extern __shared__ __align__(16) uint8_t spec_smem[];
  __shared__ int s_scan[kSpecThreads / 32];
  __shared__ int s_n;
  __shared__ int loaded, chained, folded, scored;  // passes staged / passes consumed / keys produced / keys consumed
  __shared__ uint64_t skeys[SCORE ? kSpecKeyRing : 1];
  __shared__ Bucket tile[SCORE ? 32 : 1];
  __shared__ int64_t s_koff[kSpecMaxPrompts + 1], s_poff[kSpecMaxPrompts + 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bs = X.block_size;
  if (!A.single) {  // prompt and key offsets: one parallel fetch (launch arguments, or one read of the arrays)
    for (int i = tid; i <= X.n_prompts; i += kSpecThreads) {
      s_koff[i] = X.inl ? I.koff[i] : A.key_off[i];
      s_poff[i] = X.inl ? I.poff[i] : A.prompt_off[i];
    }
    __syncthreads();
  }
#ifdef KVB_HASH_PROFILE
#define SPROF(slot) do { if (blockIdx.x == 0) g_hash_prof[slot] = clock64(); } while (0)
  if (tid == 0) SPROF(0);
#else
#define SPROF(slot) do { } while (0)
#endif

  // ---- phase A: tables.  Task k = key k of the batch (prompt p, block i).  A CTA's first task is its own index, the
  // rest come from a counter (fetched while the current task runs).  Whoever is resident drains the queue, the prompts'
  // own CTAs included, so the chains below never wait for a CTA that has not been scheduled — whatever else holds SMs.
  __shared__ unsigned s_next;
  uint8_t* stage = spec_smem;  // <= 5 + kSpecChunk bytes
  const int64_t first_round = min((int64_t)gridDim.x, X.total_keys);
  for (int64_t k = blockIdx.x; k < X.total_keys;) {
    if (tid == 0) s_next = atomicAdd(X.next_task, 1u) - X.task_base;  // read after the barriers inside the task
    int p = 0;
    int64_t i = k, tok0 = 0;
    if (!A.single) {
      int lo = 0, hi = X.n_prompts;  // p = last prompt with key_off[p] <= k
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_koff[mid] <= k) lo = mid;
        else hi = mid;
      }
      p = lo;
      i = k - s_koff[p];
      tok0 = s_poff[p];
    }
    const uint32_t* tk = A.tokens + tok0 + i * bs;
    Fnv h{(uint32_t)tid, 0u}, g{(uint32_t)tid + 128u, 0u};  // start values tid and tid + 128
    uint32_t m = 0;
    for (int t0 = 0; t0 < bs; t0 += 128) {
      // stage: [array head, first round only] + up to 128 tokens, compacted by a CTA-wide prefix sum of the lengths
      const int nt = min(128, bs - t0);
      int len = 0;
      uint32_t head = 0, pay = 0;
      if (tid < nt) {
        const uint32_t t = __ldg(tk + t0 + tid);
        const bool ge24 = t >= 24u, ge256 = t >= 0x100u, ge64k = t >= 0x10000u;
        head = ge64k ? 0x1au : (ge256 ? 0x19u : (ge24 ? 0x18u : t));
        pay = ge64k ? t : (ge256 ? (t << 16) : (t << 24));
        len = ge64k ? 5 : (ge256 ? 3 : (ge24 ? 2 : 1));
      }
      int incl = len;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
      }
      if (lane == 31) s_scan[warp] = incl;
      __syncthreads();
      int base = 0;
      for (int w = 0; w < warp; ++w) base += s_scan[w];
      int hl = 0;  // array head in front of the first round's tokens
      if (t0 == 0) hl = bs < 24 ? 1 : (bs < 256 ? 2 : (bs < 65536 ? 3 : 5));
      const int at = hl + base + incl - len;
      if (tid < nt) {
        stage[at] = (uint8_t)head;
        if (len > 1) stage[at + 1] = (uint8_t)(pay >> 24);
        if (len > 2) stage[at + 2] = (uint8_t)(pay >> 16);
        if (len > 3) {
          stage[at + 3] = (uint8_t)(pay >> 8);
          stage[at + 4] = (uint8_t)pay;
        }
      }
      if (tid == 0) {
        if (t0 == 0) {
          if (bs < 24) {
            stage[0] = (uint8_t)(0x80u | bs);
          } else if (bs < 256) {
            stage[0] = 0x98u;
            stage[1] = (uint8_t)bs;
          } else if (bs < 65536) {
            stage[0] = 0x99u;
            stage[1] = (uint8_t)(bs >> 8);
            stage[2] = (uint8_t)bs;
          } else {
            stage[0] = 0x9au;
            stage[1] = (uint8_t)(bs >> 24);
            stage[2] = (uint8_t)(bs >> 16);
            stage[3] = (uint8_t)(bs >> 8);
            stage[4] = (uint8_t)bs;
          }
        }
        int total = hl;
        for (int w = 0; w < kSpecThreads / 32; ++w) total += s_scan[w];
        s_n = total;
      }
      __syncthreads();
      const int n = s_n;
      spec_fold_chunk(h, g, reinterpret_cast<const uint32_t*>(stage), n);
      m += (uint32_t)n;
      __syncthreads();
    }
    // extra: pre-encoded X(extra_k) (extra_keys.go) or CBOR null
    int64_t e0 = 0, e1 = 0;
    if (A.extra_off != nullptr) {
      e0 = A.extra_off[k];
      e1 = A.extra_off[k + 1];
    }
    if (e1 > e0) {
      for (int64_t e = e0; e < e1; e += kSpecChunk) {
        const int n = (int)min((int64_t)kSpecChunk, e1 - e);
        for (int j = tid; j < n; j += kSpecThreads) stage[j] = A.extra[e + j];
        __syncthreads();
        spec_fold_chunk(h, g, reinterpret_cast<const uint32_t*>(stage), n);
        m += (uint32_t)n;
        __syncthreads();
      }
    } else {
      fold(h, 0xf6u);
      fold(g, 0xf6u);
      m += 1;
    }
    X.table[k * 256 + tid] = fnv_value(h);
    X.table[k * 256 + 128 + tid] = fnv_value(g);
    if (tid == 0) X.pm[k] = pow_prime(m);
    __threadfence();
    __syncthreads();
    if (tid == 0) atomicAdd(&X.done[p], 1u);
    k = first_round + (int64_t)s_next;
    __syncthreads();  // everybody has read s_next before thread 0 fetches again
  }

  if (tid == 0) SPROF(1);
  // ---- phase B: CTA p follows prompt p.  The queue is empty, so every table this CTA waits for is done or being computed
  // by a running CTA.  Lane 0 of warp 0 walks the chain, warp 1 scores behind it, warps 2..3
  // stage the table rows (two buffers of kSpecPassRows rows, cp.async) ahead of it.
  const int p = blockIdx.x;
  if (p >= X.n_prompts) return;
  const int64_t k0 = A.single ? 0 : s_koff[p];
  const int nblk = A.single ? (int)(A.single_tokens / bs) : (int)(s_koff[p + 1] - k0);
  if (nblk == 0) {
    if (SCORE && tid == 0) {
      A.out_n[p] = 0;
      chain_signal_done(A);
    }
    return;
  }
  if (tid == 0) {
    loaded = 0;
    chained = 0;
    folded = 0;
    scored = 0;
  }
  __syncthreads();
  uint64_t* rows = reinterpret_cast<uint64_t*>(spec_smem);                    // [2][kSpecPassRows][256]
  uint64_t* pms = rows + (size_t)2 * kSpecPassRows * 256;                      // [2][kSpecPassRows]
  const int npass = (nblk + kSpecPassRows - 1) / kSpecPassRows;

  if (warp >= 2) {
    // ------------------------------------------------------------------------------------------------ loaders
    const int lt = tid - 64;
    constexpr int kLoaders = kSpecThreads - 64;
    if (lt == 0) {
      const volatile unsigned* d = X.done + p;
      unsigned long long t_wait0 = 0, t_now = 0;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_wait0));
      while (*d < (unsigned)nblk) {
        __nanosleep(50);
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_now));
        if (t_now - t_wait0 > 2000000000ull) __trap();  // the only wait on OTHER CTAs: fail the launch rather than hang the GPU
      }
      __threadfence();
      SPROF(2);
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kLoaders));
    for (int q = 0; q < npass; ++q) {
      if (q >= 2) {
        if (lt == 0) spec_wait_ge(&chained, q - 1);  // buffer q & 1 was last used by pass q - 2
        asm volatile("bar.sync 1, %0;" ::"n"(kLoaders));
      }
      const int b0 = q * kSpecPassRows, cnt = min(kSpecPassRows, nblk - b0);
      const uint4* src = reinterpret_cast<const uint4*>(X.table + (k0 + b0) * 256);
      uint64_t* buf = rows + (size_t)(q & 1) * kSpecPassRows * 256;
      const uint32_t dst = (uint32_t)__cvta_generic_to_shared(buf);
      for (int j = lt; j < cnt * 128; j += kLoaders)  // .cg: the rows were written by other SMs (L2, never this SM's L1)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16u * j), "l"(src + j) : "memory");
      if (lt < cnt) pms[(q & 1) * kSpecPassRows + lt] = __ldcg(X.pm + k0 + b0 + lt);
      asm volatile("cp.async.wait_all;" ::: "memory");
      __threadfence_block();
      asm volatile("bar.sync 1, %0;" ::"n"(kLoaders));
      if (lt == 0) st_release_cta(&loaded, q + 1);
      if (lt == 0 && q == 0) SPROF(3);
    }
    if (lt == 0) X.done[p] = 0u;  // ready for the next launch
    return;
  }

  if (warp == 1) {
    if (!SCORE) return;
    // ------------------------------------------------------------------------------------------------ scorer
    ScoreWalker wk;
    for (int base = 0; base < nblk;) {
      const int want = min(A.score_min_batch, nblk - base);
      int avail;
      while ((avail = ld_acquire_cta(&folded) - base) < want) __nanosleep(40);
      const int in_tile = min(avail, 32);
      const uint64_t key = lane < in_tile ? skeys[(base + lane) & (kSpecKeyRing - 1)] : 0ull;
      __syncwarp();
      if (lane == 0) *reinterpret_cast<volatile int*>(&scored) = base + in_tile;  // the ring slots may be reused
      if (lane == 0 && base == 0) SPROF(7);
      if (wk.chain_alive || A.ts != nullptr)
        wk.tile(A.table, A.mask, tile, key, lane < in_tile, base, in_tile, A.filter_bits, A.tier_w, A.ts,
                A.stamp_base + (unsigned long long)(k0 + base + lane));
      if (lane == 0 && base == 0) SPROF(8);
      base += in_tile;
    }
    if (lane == 0) SPROF(9);
    wk.finish(p, A.out_n, A.out_pods, A.out_scores);
    __syncwarp();
    if (lane == 0) SPROF(10);
    if (lane == 0) chain_signal_done(A);
    if (lane == 0) SPROF(6);
    return;
  }

  // ---------------------------------------------------------------------------------------------------- chain
  if (lane != 0) return;
  uint64_t parent = A.single ? A.single_parent : (X.inl ? I.par[p] : A.parents[p]);
  for (int q = 0; q < npass; ++q) {
    spec_wait_ge(&loaded, q + 1);
    if (q == 0) SPROF(4);
    const int b0 = q * kSpecPassRows, cnt = min(kSpecPassRows, nblk - b0);
    const uint64_t* rowp = rows + (size_t)(q & 1) * kSpecPassRows * 256;
    const uint64_t* pq = pms + (q & 1) * kSpecPassRows;
    uint64_t pm_next = pq[0];
    for (int b = 0; b < cnt; ++b, rowp += 256) {
      const uint64_t pm = pm_next;
      if (b + 1 < cnt) pm_next = pq[b + 1];  // off the chain: fetched a block early
      Fnv h;
      if (parent >= 0x100000000ull) {  // U(parent) is the 9-byte form: 83 1b are constants, 8 bytes to fold
        h = Fnv{(uint32_t)kSpecAfter831b, (uint32_t)(kSpecAfter831b >> 32)};
        fold4(h, __byte_perm((uint32_t)(parent >> 32), 0u, 0x0123));  // most significant byte first
        fold4(h, __byte_perm((uint32_t)parent, 0u, 0x0123));
      } else {
        h = fnv_init();
        fold(h, 0x83u);
        fold_head64(h, 0x00u, parent);
      }
      const uint32_t l = h.lo & 0xffu;
      const uint64_t u = ((uint64_t)h.hi << 32) | (h.lo ^ l);  // the state with its low byte cleared
      parent = u * pm + rowp[l];
      const int kb = b0 + b;
      if (A.out_keys != nullptr) A.out_keys[k0 + kb] = parent;
      if (SCORE) {
        if (kb >= kSpecKeyRing) spec_wait_ge(&scored, kb - kSpecKeyRing + 1);
        skeys[kb & (kSpecKeyRing - 1)] = parent;
        // plain store behind the key's (one thread, shared memory: performed in order); a release would put a CTA-wide
        // memory barrier on the chain for every block
        *reinterpret_cast<volatile int*>(&folded) = kb + 1;
      }
    }
    st_release_cta(&chained, q + 1);
  }
  SPROF(5);
#undef SPROF
}

// Scratch of the table kernel (2 KiB of table per key + the counters).  Launches that share one are stream-ordered: the
// next launch reuses the tables.  An index and the host hash entry point own theirs (created on first use, released with
// the owner); callers of the device-resident entry point get one per (device, stream) that lives as long as the process.
struct SpecScratch {
  std::mutex mu;
  uint8_t* d = nullptr;
  size_t cap = 0;
  unsigned* done = nullptr;   // kSpecMaxPrompts counters + the task counter
  unsigned task_base = 0;
  int max_grid = 0;
};
SpecScratch* spec_scratch_create() { return new SpecScratch(); }
void spec_scratch_destroy(SpecScratch* sc) {
  if (!sc) return;
  if (sc->d) cudaFree(sc->d);
  if (sc->done) cudaFree(sc->done);
  delete sc;
}
static SpecScratch& spec_scratch_shared(int device, cudaStream_t s) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, std::unique_ptr<SpecScratch>> all;
  std::lock_guard<std::mutex> lk(mu);
  auto& p = all[std::make_pair(device, s)];
  if (!p) p.reset(new SpecScratch());
  return *p;
}
constexpr size_t kSpecSmem = (size_t)2 * kSpecPassRows * 256 * 8 + (size_t)2 * kSpecPassRows * 8;
constexpr int64_t kSpecMaxKeys = 16384;  // 32 MiB of tables

// true if the batch was handed to the spec kernel (*rc_out tells how that went); false = not applicable, the caller
// picks another kernel.
static bool launch_spec(const ChainArgs& ca, bool score, int32_t n_prompts, int32_t block_size, int64_t total_keys,
                        cudaStream_t s, int* rc_out, const int64_t* h_prompt_off = nullptr,
                        const int64_t* h_key_off = nullptr, const uint64_t* h_parents = nullptr,
                        SpecScratch* own = nullptr) {
  *rc_out = KVB_OK;
  if (n_prompts > kSpecMaxPrompts || total_keys <= 0 || total_keys > kSpecMaxKeys) return false;
  int dev = 0;
  cudaGetDevice(&dev);
  SpecScratch& sc = own ? *own : spec_scratch_shared(dev, s);
  std::lock_guard<std::mutex> lk(sc.mu);
  auto fail = [&](const char* what, cudaError_t e) {
    set_error("hash (spec kernel): %s: %s", what, cudaGetErrorString(e));
    *rc_out = KVB_ERR_CUDA;
    return true;
  };
  if (sc.max_grid == 0) {
    int per_sm = 1 << 30;
    cudaError_t e = cudaSuccess;
    auto prep = [&](auto kernel) {
      if (e != cudaSuccess) return;
      e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSpecSmem);
      int n = 0;
      if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, kSpecThreads, kSpecSmem);
      if (e == cudaSuccess) per_sm = std::min(per_sm, n);
    };
    prep(hash_spec_kernel<false, kSpecAutoPrompts>);
    prep(hash_spec_kernel<true, kSpecAutoPrompts>);
    prep(hash_spec_kernel<false, kSpecMaxPrompts>);
    prep(hash_spec_kernel<true, kSpecMaxPrompts>);
    if (e != cudaSuccess || per_sm < 1) return fail("kernel attributes / occupancy query", e);
    e = cudaMalloc(&sc.done, (kSpecMaxPrompts + 1) * sizeof(unsigned));
    if (e != cudaSuccess) return fail("counters", e);
    cudaMemset(sc.done, 0, (kSpecMaxPrompts + 1) * sizeof(unsigned));
    sc.max_grid = per_sm * sm_count(dev);  // one wave when the GPU is ours; not needed for progress
  }
  const size_t need = (size_t)total_keys * (256 + 1) * 8;
  if (need > sc.cap) {
    cudaStreamSynchronize(s);  // an earlier launch may still read the old tables
    if (sc.d) cudaFree(sc.d);
    sc.d = nullptr;
    sc.cap = 0;
    const size_t cap = std::max<size_t>(need * 3 / 2, 4 << 20);
    cudaError_t e = cudaMalloc(&sc.d, cap);
    if (e != cudaSuccess) return fail("table scratch", e);
    sc.cap = cap;
  }
  SpecArgs x{};
  x.n_prompts = n_prompts;
  x.block_size = block_size;
  x.total_keys = total_keys;
  x.table = reinterpret_cast<uint64_t*>(sc.d);
  x.pm = x.table + (size_t)total_keys * 256;
  x.done = sc.done;
  x.next_task = sc.done + kSpecMaxPrompts;
  x.task_base = sc.task_base;
  const int grid = (int)std::min<int64_t>(std::max<int64_t>(total_keys, n_prompts), sc.max_grid);
  const bool inl = h_prompt_off && h_key_off && h_parents;  // host copies at hand: they go into the arguments
  x.inl = inl ? 1 : 0;
  auto go = [&](auto tag) {
    constexpr int N = decltype(tag)::value;
    SpecInline<N> in{};
    if (inl) {
      for (int i = 0; i <= n_prompts; ++i) {
        in.koff[i] = h_key_off[i];
        in.poff[i] = h_prompt_off[i];
      }
      for (int i = 0; i < n_prompts; ++i) in.par[i] = h_parents[i];
    }
    if (score) hash_spec_kernel<true, N><<<grid, kSpecThreads, kSpecSmem, s>>>(ca, x, in);
    else hash_spec_kernel<false, N><<<grid, kSpecThreads, kSpecSmem, s>>>(ca, x, in);
  };
  if (n_prompts <= kSpecAutoPrompts) go(std::integral_constant<int, kSpecAutoPrompts>{});
  else go(std::integral_constant<int, kSpecMaxPrompts>{});
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("launch", e);  // nothing ran: the task counter has not moved either
  sc.task_base += (unsigned)total_keys;            // the launch advances the counter by exactly one per task (wraps with it)
  count_launch();
  return true;
}

static bool spec_wanted(int32_t n_prompts) {
  // KVB_HASH_KERNEL=spec forces the table kernel for every batch it can take; any other forced family or KVB_HASH_SPEC=0
  // keeps it out; by default it takes the batches it wins on
  const char* f0 = std::getenv("KVB_HASH_KERNEL");
  const char* s0 = std::getenv("KVB_HASH_SPEC");
  if (f0 != nullptr) return std::strcmp(f0, "spec") == 0;
  return !(s0 && s0[0] == '0') && n_prompts <= kSpecDefaultPrompts;
}

// fused tokens -> scores for small batches (see launch_chain_score); false = not applicable
bool launch_spec_score(const ChainArgs& a, int32_t n_prompts, int32_t block_size, int64_t total_keys, cudaStream_t s,
                       int* rc_out, const int64_t* h_prompt_off, const int64_t* h_key_off, const uint64_t* h_parents,
                       SpecScratch* scratch) {
  *rc_out = KVB_OK;
  if (!spec_wanted(n_prompts)) return false;
  // this chain hands over keys far faster than a probe round completes, whatever the round's size: the scorer takes
  // full tiles (with the slower vote-round chain, small tiles keep it closer behind)
  ChainArgs b = a;
  const char* e = std::getenv("KVB_SPEC_SCORE_BATCH");
  b.score_min_batch = e ? std::max(1, std::min(32, std::atoi(e))) : 32;
  return launch_spec(b, true, n_prompts, block_size, total_keys, s, rc_out, h_prompt_off, h_key_off, h_parents, scratch);
}

// getInitHash: H(seed_hash, nil, model_name) = FNV64a(83 | U(seed) | f6 | text(model))
__global__ void init_hash_kernel(uint64_t seed_hash, const uint8_t* __restrict__ name, uint32_t len,
                                 uint64_t* __restrict__ out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  Fnv h = fnv_init();
  fold(h, 0x83u);
  fold_head64(h, 0x00u, seed_hash);
  fold(h, 0xf6u);
  fold_head64(h, 0x60u, len);
  for (uint32_t i = 0; i < len; ++i) fold(h, name[i]);
  *out = fnv_value(h);
}

int launch_hash_blocks(const uint32_t* tokens, const int64_t* prompt_off, const uint64_t* parents, int32_t n_prompts,
                       int32_t block_size, const uint8_t* extra, const int64_t* extra_off, uint64_t* out_keys,
                       const int64_t* key_off, cudaStream_t s, int64_t total_keys, const int64_t* h_prompt_off,
                       const int64_t* h_key_off, const uint64_t* h_parents, SpecScratch* scratch) {
  if (n_prompts <= 0) return KVB_OK;
  if (total_keys > 0 && spec_wanted(n_prompts)) {  // small batches whose key count the caller knows: tables off the chain
    ChainArgs a{};
    a.tokens = tokens;
    a.prompt_off = prompt_off;
    a.parents = parents;
    a.extra = extra;
    a.extra_off = extra_off;
    a.out_keys = out_keys;
    a.key_off = key_off;
    int rc = KVB_OK;
    if (launch_spec(a, false, n_prompts, block_size, total_keys, s, &rc, h_prompt_off, h_key_off, h_parents, scratch)) return rc;
  }
  // small batches: 32-thread CTAs so the chains spread over the SMs; large: 128
  int dev = 0;
  cudaGetDevice(&dev);
  const int threads = n_prompts >= sm_count(dev) * 128 ? 128 : 32;
  const int grid = (n_prompts + threads - 1) / threads;
  static const bool one_warp = std::getenv("KVB_HASH_ONE_WARP") != nullptr;  // A/B switch for profiling
  // KVB_HASH_KERNEL=lanes forces the lane-per-prompt kernels (A/B and parity tests of both families); read per call
  const char* force = std::getenv("KVB_HASH_KERNEL");
  const bool lanes_only = force != nullptr && std::strcmp(force, "lanes") == 0;
  const bool wpc_v1 = force != nullptr && std::strcmp(force, "wpc") == 0;  // round-1 warp kernel, kept for A/B
  // the round-2 chain kernel in its hash-only form is no faster than round 1's warp kernel (tests/bench_hash.py), so it
  // hashes alone only on request; its value is the fused tokens -> scores launch
  const bool chain_only = force != nullptr && std::strcmp(force, "chain") == 0;
  if (chain_only && n_prompts <= kChainMaxPrompts && chain_kernel_supports(block_size)) {
    ChainArgs a{};
    a.tokens = tokens;
    a.tokens_lo = tokens;
    a.tokens_hi = tokens + (1ll << 40);  // device-resident tokens: the caller's array bounds are not known here
    a.prompt_off = prompt_off;
    a.parents = parents;
    a.extra = extra;
    a.extra_off = extra_off;
    a.out_keys = out_keys;
    a.key_off = key_off;
    if (block_size == 16) launch_chain_bs<16, false>(a, n_prompts, s);
    else if (block_size == 8) launch_chain_bs<8, false>(a, n_prompts, s);
    else launch_chain_bs<4, false>(a, n_prompts, s);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_error("hash kernel launch failed: %s", cudaGetErrorString(e));
      return KVB_ERR_CUDA;
    }
    count_launch();
    return KVB_OK;
  }
  if (!one_warp && !lanes_only && n_prompts <= kWpcPromptsPerSm * sm_count(dev) && (block_size == 16 || block_size == 8 || block_size == 4)) {
    if (block_size == 16)
      hash_chain_kernel_wpc<16><<<n_prompts, 64, 0, s>>>(tokens, prompt_off, parents, extra, extra_off, out_keys, key_off);
    else if (block_size == 8)
      hash_chain_kernel_wpc<8><<<n_prompts, 64, 0, s>>>(tokens, prompt_off, parents, extra, extra_off, out_keys, key_off);
    else
      hash_chain_kernel_wpc<4><<<n_prompts, 64, 0, s>>>(tokens, prompt_off, parents, extra, extra_off, out_keys, key_off);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_error("hash kernel launch failed: %s", cudaGetErrorString(e));
      return KVB_ERR_CUDA;
    }
    count_launch();
    return KVB_OK;
  }
  const int grid2 = (n_prompts + 31) / 32;
  // fewer CTAs than ~2 per SM sub-partition: every warp is alone on its scheduler -> optimise latency, else issue slots
  const bool latency_bound = grid2 <= 4 * sm_count(dev);
  switch (one_warp ? -1 : block_size) {
#define KVB_LAUNCH_2W(BSV)                                                                                          \
  if (latency_bound)                                                                                                \
    hash_chain_kernel_2w<BSV, true><<<grid2, 64, 0, s>>>(tokens, prompt_off, parents, n_prompts, extra, extra_off,  \
                                                         out_keys, key_off);                                        \
  else                                                                                                              \
    hash_chain_kernel_2w<BSV, false><<<grid2, 64, 0, s>>>(tokens, prompt_off, parents, n_prompts, extra, extra_off, \
                                                          out_keys, key_off)
    case 16:
      KVB_LAUNCH_2W(16);
      break;
    case 8:
      KVB_LAUNCH_2W(8);
      break;
    case 4:
      KVB_LAUNCH_2W(4);
      break;
#undef KVB_LAUNCH_2W
    case -1:
      if (block_size == 16) {
        hash_chain_kernel<16><<<grid, threads, 0, s>>>(tokens, prompt_off, parents, n_prompts, block_size, extra,
                                                       extra_off, out_keys, key_off);
        break;
      }
      [[fallthrough]];
    default:
      hash_chain_kernel<0><<<grid, threads, 0, s>>>(tokens, prompt_off, parents, n_prompts, block_size, extra,
                                                    extra_off, out_keys, key_off);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("hash kernel launch failed: %s", cudaGetErrorString(e));
    return KVB_ERR_CUDA;
  }
  count_launch();
  return KVB_OK;
}

// Device + pinned-host scratch of kvb_hash_token_blocks, one per device, kept for the life of the process.
struct HashScratch {
  std::mutex mu;
  uint8_t* d = nullptr;
  size_t d_cap = 0;
  uint8_t* h = nullptr;  // pinned on the GPU's NUMA node; holds everything but the keys
  size_t h_cap = 0;
  cudaStream_t stream = nullptr;  // for callers that pass no stream
  SpecScratch* spec = nullptr;    // tables of the table kernel (small batches)
  int ensure(int device, size_t dev_bytes, size_t host_bytes) {
    if (!spec) spec = spec_scratch_create();
    if (!stream) KVB_CUDA_TRY(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    if (dev_bytes > d_cap) {
      if (d) cudaFree(d);
      d = nullptr;
      d_cap = 0;
      const size_t cap = (std::max<size_t>(dev_bytes, 1 << 20) * 3 / 2 + 255) & ~size_t(255);
      KVB_CUDA_TRY(cudaMalloc(&d, cap));
      d_cap = cap;
    }
    if (host_bytes > h_cap) {
      if (h) cudaFreeHost(h);
      h = nullptr;
      h_cap = 0;
      const size_t cap = (std::max<size_t>(host_bytes, 1 << 20) * 3 / 2 + 255) & ~size_t(255);
      KVB_CUDA_TRY(host_alloc_near(device, reinterpret_cast<void**>(&h), cap, cudaHostAllocDefault));
      h_cap = cap;
    }
    return KVB_OK;
  }
};
static HashScratch& hash_scratch(int device) {
  static std::mutex mu;
  static std::map<int, std::unique_ptr<HashScratch>> all;
  std::lock_guard<std::mutex> lk(mu);
  auto& p = all[device];
  if (!p) p.reset(new HashScratch());
  return *p;
}

}  // namespace kvb

using namespace kvb;

extern "C" {

uint64_t kvb_fnv64a(const void* data, size_t len) {
  // seed hash only (token_processor.go:90-95): once per processor, a handful of bytes
  const uint8_t* p = static_cast<const uint8_t*>(data);
  uint64_t h = kFnvOffset;
  for (size_t i = 0; i < len; ++i) h = (h ^ p[i]) * kFnvPrime;
  return h;
}

int kvb_init_hash(int device, uint64_t seed_hash, const char* model_name, size_t model_len, uint64_t* out) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(out != nullptr, "out is NULL");
    KVB_REQUIRE(model_name != nullptr || model_len == 0, "model_name is NULL");
    KVB_REQUIRE(model_len < (1u << 31), "model name too long");
    DeviceGuard g(device);
    if (!g.ok) {
      set_error("cannot select CUDA device %d", device);
      return KVB_ERR_CUDA;
    }
    uint8_t* d = nullptr;
    KVB_CUDA_TRY(cudaMalloc(&d, model_len + 8 + 8));
    uint64_t* d_out = reinterpret_cast<uint64_t*>(d);
    uint8_t* d_name = d + 8;
    cudaError_t e = cudaSuccess;
    if (model_len) e = cudaMemcpy(d_name, model_name, model_len, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
      init_hash_kernel<<<1, 32>>>(seed_hash, d_name, (uint32_t)model_len, d_out);
      count_launch();
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, 8, cudaMemcpyDeviceToHost);
    cudaFree(d);
    KVB_CUDA_TRY(e);
    return KVB_OK;
  });
}

int kvb_hash_token_blocks_dev(int device, const uint32_t* tokens, const int64_t* prompt_off, const uint64_t* parents,
                              int32_t n_prompts, int32_t block_size, const uint8_t* extra, const int64_t* extra_off,
                              uint64_t* out_keys, const int64_t* key_off, int64_t total_keys, void* stream) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(block_size > 0, "blockSize must be greater than 0, got %d", block_size);  // token_processor.go:86-88
    KVB_REQUIRE(n_prompts >= 0, "negative prompt count");
    if (n_prompts == 0) return KVB_OK;
    KVB_REQUIRE(tokens && prompt_off && parents && out_keys && key_off, "NULL argument");
    DeviceGuard g(device);
    return launch_hash_blocks(tokens, prompt_off, parents, n_prompts, block_size, extra, extra_off, out_keys, key_off,
                              static_cast<cudaStream_t>(stream), total_keys);
  });
}

int kvb_hash_token_blocks(int device, const uint32_t* tokens, const int64_t* prompt_off, const uint64_t* parents,
                          int32_t n_prompts, int32_t block_size, const uint8_t* extra, const int64_t* extra_off,
                          uint64_t* out_keys, int64_t* out_key_off, void* stream) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(block_size > 0, "blockSize must be greater than 0, got %d", block_size);
    KVB_REQUIRE(n_prompts >= 0, "negative prompt count");
    KVB_REQUIRE(out_key_off != nullptr, "out_key_off is NULL");
    out_key_off[0] = 0;
    if (n_prompts == 0) return KVB_OK;
    KVB_REQUIRE(prompt_off && parents, "NULL argument");
    for (int32_t p = 0; p < n_prompts; ++p) {
      KVB_REQUIRE(prompt_off[p + 1] >= prompt_off[p], "prompt_off not monotonic at %d", p);
      out_key_off[p + 1] = out_key_off[p] + (prompt_off[p + 1] - prompt_off[p]) / block_size;
    }
    const int64_t total_keys = out_key_off[n_prompts];
    const int64_t total_tok = prompt_off[n_prompts] - prompt_off[0];
    if (total_keys == 0) return KVB_OK;
    KVB_REQUIRE(tokens && out_keys, "NULL argument");
    DeviceGuard g(device);
    if (!g.ok) {
      set_error("cannot select CUDA device %d", device);
      return KVB_ERR_CUDA;
    }
    const int64_t extra_bytes = extra_off ? extra_off[total_keys] : 0;
    // per-device scratch kept for the life of the process (device + pinned host, same offsets on both sides):
    // [tokens | prompt_off | key_off | parents | extra_off | extra | keys]; calls on one device serialise on it
    HashScratch& sc = hash_scratch(device);
    std::lock_guard<std::mutex> lk(sc.mu);
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t o_tok = 0;
    const size_t o_poff = o_tok + al((size_t)total_tok * 4);
    const size_t o_koff = o_poff + al(((size_t)n_prompts + 1) * 8);
    const size_t o_par = o_koff + al(((size_t)n_prompts + 1) * 8);
    const size_t small_end = o_par + (size_t)n_prompts * 8;
    const size_t o_eoff = al(small_end);
    const size_t o_ext = o_eoff + (extra_off ? al(((size_t)total_keys + 1) * 8) : 0);
    const size_t o_keys = o_ext + (extra_off ? al((size_t)extra_bytes) : 0);
    const size_t total = o_keys + al((size_t)total_keys * 8);
    int rc = sc.ensure(device, total, o_keys);
    if (rc) return rc;
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : sc.stream;
    uint8_t *H = sc.h, *D = sc.d;
    int64_t* h_poff = reinterpret_cast<int64_t*>(H + o_poff);
    for (int32_t p = 0; p <= n_prompts; ++p) h_poff[p] = prompt_off[p] - prompt_off[0];
    std::memcpy(H + o_koff, out_key_off, ((size_t)n_prompts + 1) * 8);
    std::memcpy(H + o_par, parents, (size_t)n_prompts * 8);
    // tokens go straight from the caller's buffer: pinned memory is read by the copy engine in place, pageable memory
    // is staged by the driver (faster than staging it here: tools/ab_stage.py compares the two)
    KVB_CUDA_TRY(cudaMemcpyAsync(D + o_tok, tokens + prompt_off[0], (size_t)total_tok * 4, cudaMemcpyHostToDevice, s));
    KVB_CUDA_TRY(cudaMemcpyAsync(D + o_poff, H + o_poff, small_end - o_poff, cudaMemcpyHostToDevice, s));
    if (extra_off) {
      std::memcpy(H + o_eoff, extra_off, ((size_t)total_keys + 1) * 8);
      if (extra_bytes) std::memcpy(H + o_ext, extra, (size_t)extra_bytes);
      KVB_CUDA_TRY(cudaMemcpyAsync(D + o_eoff, H + o_eoff, (o_ext + (size_t)extra_bytes) - o_eoff, cudaMemcpyHostToDevice, s));
    }
    rc = launch_hash_blocks(reinterpret_cast<uint32_t*>(D + o_tok), reinterpret_cast<int64_t*>(D + o_poff),
                            reinterpret_cast<uint64_t*>(D + o_par), n_prompts, block_size,
                            extra_off ? D + o_ext : nullptr, extra_off ? reinterpret_cast<int64_t*>(D + o_eoff) : nullptr,
                            reinterpret_cast<uint64_t*>(D + o_keys), reinterpret_cast<int64_t*>(D + o_koff), s, total_keys,
                            h_poff, out_key_off, parents, sc.spec);
    cudaError_t e = cudaSuccess;
    if (rc == KVB_OK) e = cudaMemcpyAsync(out_keys, D + o_keys, (size_t)total_keys * 8, cudaMemcpyDeviceToHost, s);
    const cudaError_t e2 = cudaStreamSynchronize(s);  // the scratch and the caller's buffers must outlive the copies
    if (rc != KVB_OK) return rc;
    KVB_CUDA_TRY(e);
    KVB_CUDA_TRY(e2);
    return KVB_OK;
  });
}

}  // extern "C"
