// copy_kernels.cu — paged-KV gather / scatter / page->page migration kernels for sm_90a (H100).
//
// Replaces the reference's per-(block x tensor) cudaMemcpyAsync loop
// (kv_connectors/llmd_fs_backend/csrc/storage/tensor_copier.cu:78-96) and its opt-in
// 1-byte-per-thread copy kernel launched once per tensor (tensor_copier_kernels.cu:54-143)
// with ONE launch that moves every fragment of every listed block.
//
// Work decomposition: a KV block is T fragments (one per canonical tensor) of frag_bytes each;
// a fragment is cut into pieces of PIECE bytes.  item = (block b, tensor t, piece p), numbered so that
// consecutive items are consecutive bytes of the packed buffer [block][tensor][fragment].
// A persistent grid (multiple of the SM count) strides over items.
//
// Two data movers, selected by KVB_COPY_*:
//   LDG  : 16 B ld.global.nc / st.global per thread, UNROLL independent loads in flight per thread.
//   BULK : TMA bulk copies, global -> shared (cp.async.bulk + mbarrier complete_tx) -> global
//          (cp.async.bulk ... bulk_group), a ring of STAGES x PIECE bytes per CTA driven by one thread.
// HBM traffic is exactly 2 x payload (read once, write once); nothing is re-read.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "kvb_internal.h"

namespace kvb {

enum Mode : int { kGather = 0, kScatter = 1, kMigrate = 2 };

struct CopyArgs {
  const uint8_t* const* tensors;   // paged side (gather: source, scatter: destination, migrate: source)
  const uint8_t* const* tensors2;  // migrate: destination pool tensors
  const int64_t* ids;              // paged-side block ids
  const int64_t* ids2;             // migrate: destination block ids
  uint8_t* packed;                 // gather: destination, scatter: source
  int64_t frag;                    // bytes per fragment
  int64_t stride;                  // paged-side block stride
  int64_t stride2;                 // migrate: destination block stride
  uint32_t T;
  uint32_t ppf;                    // pieces per fragment
  uint32_t piece;                  // bytes per piece (last piece of a fragment may be shorter)
  uint64_t total_items;            // n * T * ppf
};

__device__ __forceinline__ const uint8_t* ldg_ptr(const uint8_t* const* p) {
  return reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(p)));
}

template <int MODE>
__device__ __forceinline__ void item_addresses(const CopyArgs& a, uint64_t item, const uint8_t*& src, uint8_t*& dst,
                                               uint32_t& bytes) {
  // item -> (f = b*T + t, p); 32-bit math when it fits (the usual case), 64-bit otherwise
  uint64_t f;
  uint32_t p;
  if (a.total_items <= 0xffffffffull) {
    uint32_t it = (uint32_t)item;
    uint32_t f32 = it / a.ppf;
    p = it - f32 * a.ppf;
    f = f32;
  } else {
    f = item / a.ppf;
    p = (uint32_t)(item - f * a.ppf);
  }
  uint64_t b;
  uint32_t t;
  if (f <= 0xffffffffull) {
    uint32_t b32 = (uint32_t)f / a.T;
    t = (uint32_t)f - b32 * a.T;
    b = b32;
  } else {
    b = f / a.T;
    t = (uint32_t)(f - b * a.T);
  }
  const uint64_t off = (uint64_t)p * a.piece;
  const uint64_t rem = (uint64_t)a.frag - off;
  bytes = rem < a.piece ? (uint32_t)rem : a.piece;
  const int64_t id = __ldg(a.ids + b);
  const uint8_t* paged = ldg_ptr(a.tensors + t) + id * a.stride + off;
  if (MODE == kGather) {
    src = paged;
    dst = a.packed + f * (uint64_t)a.frag + off;
  } else if (MODE == kScatter) {
    src = a.packed + f * (uint64_t)a.frag + off;
    dst = const_cast<uint8_t*>(paged);
  } else {
    const int64_t id2 = __ldg(a.ids2 + b);
    src = paged;
    dst = const_cast<uint8_t*>(ldg_ptr(a.tensors2 + t)) + id2 * a.stride2 + off;
  }
}

// ------------------------------------------------------------------------------------------
// LDG / STG mover
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int4 ld_stream(const int4* p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(int4* p, const int4& v) {
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
template <typename V>
__device__ __forceinline__ V ld_any(const V* p) {
  return *p;
}
template <>
__device__ __forceinline__ int4 ld_any<int4>(const int4* p) {
  return ld_stream(p);
}
template <typename V>
__device__ __forceinline__ void st_any(V* p, const V& v) {
  *p = v;
}
template <>
__device__ __forceinline__ void st_any<int4>(int4* p, const int4& v) {
  st_stream(p, v);
}

constexpr int kLdgThreads = 256;

template <int MODE, typename V, int UNROLL>
__global__ void __launch_bounds__(kLdgThreads) paged_copy_ldg_kernel(const CopyArgs a) {
  for (uint64_t item = blockIdx.x; item < a.total_items; item += gridDim.x) {
    const uint8_t* src;
    uint8_t* dst;
    uint32_t bytes;
    item_addresses<MODE>(a, item, src, dst, bytes);
    const V* s = reinterpret_cast<const V*>(src);
    V* d = reinterpret_cast<V*>(dst);
    const uint32_t nvec = bytes / (uint32_t)sizeof(V);
    for (uint32_t base = 0; base < nvec; base += kLdgThreads * UNROLL) {
      V v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const uint32_t i = base + threadIdx.x + u * kLdgThreads;
        if (i < nvec) v[u] = ld_any<V>(s + i);
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const uint32_t i = base + threadIdx.x + u * kLdgThreads;
        if (i < nvec) st_any<V>(d + i, v[u]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// TMA bulk mover: global -> smem ring -> global, one issuing thread per CTA
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// STAGES ring slots of a.piece bytes; LOOKAHEAD loads kept in flight, STAGES-LOOKAHEAD stores draining.
template <int MODE, int STAGES, int LOOKAHEAD>
__global__ void __launch_bounds__(32) paged_copy_bulk_kernel(const CopyArgs a) {
  extern __shared__ __align__(128) uint8_t ring[];
  __shared__ __align__(8) uint64_t full[STAGES];
  if (threadIdx.x != 0) return;
  static_assert(LOOKAHEAD >= 1 && LOOKAHEAD < STAGES, "need at least one draining slot");
#pragma unroll
  for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");

  const uint64_t first = blockIdx.x, step = gridDim.x;
  if (first >= a.total_items) return;
  const uint64_t my_n = (a.total_items - first + step - 1) / step;

  // addresses of item k of this CTA, and its load
  auto issue_load = [&](uint64_t k) {
    const uint8_t* src;
    uint8_t* dst;
    uint32_t bytes;
    item_addresses<MODE>(a, first + k * step, src, dst, bytes);
    const int s = (int)(k % STAGES);
    mbar_expect_tx(&full[s], bytes);
    bulk_g2s(ring + (size_t)s * a.piece, src, bytes, &full[s]);
  };

  const uint64_t pre = my_n < (uint64_t)LOOKAHEAD ? my_n : (uint64_t)LOOKAHEAD;
  for (uint64_t k = 0; k < pre; ++k) issue_load(k);

  for (uint64_t k = 0; k < my_n; ++k) {
    const int s = (int)(k % STAGES);
    const uint8_t* src;
    uint8_t* dst;
    uint32_t bytes;
    item_addresses<MODE>(a, first + k * step, src, dst, bytes);  // recomputed: keeps no per-stage state in registers
    mbar_wait(&full[s], (uint32_t)((k / STAGES) & 1));
    bulk_s2g(dst, ring + (size_t)s * a.piece, bytes);
    bulk_commit();
    if (k + LOOKAHEAD < my_n) {
      // slot of item k+LOOKAHEAD was last read by the store of item k+LOOKAHEAD-STAGES:
      // all but the newest STAGES-LOOKAHEAD store groups must have finished reading shared memory
      bulk_wait_read<STAGES - LOOKAHEAD>();
      issue_load(k + LOOKAHEAD);
    }
  }
  bulk_wait_all();
}

// ------------------------------------------------------------------------------------------
// launch logic
// ------------------------------------------------------------------------------------------
static int env_int(const char* name, int dflt) {
  const char* v = std::getenv(name);
  return (v && *v) ? std::atoi(v) : dflt;
}

struct Tuning {
  int default_variant;  // KVB_COPY_LDG / KVB_COPY_BULK
  int ldg_unroll;       // 2 / 4 / 8
  int ldg_ctas_per_sm;
  int bulk_piece;       // bytes
  int bulk_ctas_per_sm;
  int bulk_deep;        // 0: 6 stages / 3 lookahead, 1: 8 / 4, 2: 12 / 6
};
static const Tuning& tuning() {
  static Tuning t = [] {
    Tuning x;
    x.default_variant = env_int("KVB_COPY_VARIANT", KVB_COPY_BULK);
    x.ldg_unroll = env_int("KVB_LDG_UNROLL", 4);
    x.ldg_ctas_per_sm = env_int("KVB_LDG_CTAS_PER_SM", 8);
    x.bulk_piece = env_int("KVB_BULK_PIECE", 8192);
    x.bulk_ctas_per_sm = env_int("KVB_BULK_CTAS_PER_SM", 2);
    x.bulk_deep = env_int("KVB_BULK_DEEP", 0);
    return x;
  }();
  return t;
}

template <int MODE, typename V>
static cudaError_t launch_ldg_v(const CopyArgs& a, int grid, int unroll, cudaStream_t s) {
  switch (unroll) {
    case 2: paged_copy_ldg_kernel<MODE, V, 2><<<grid, kLdgThreads, 0, s>>>(a); break;
    case 8: paged_copy_ldg_kernel<MODE, V, 8><<<grid, kLdgThreads, 0, s>>>(a); break;
    default: paged_copy_ldg_kernel<MODE, V, 4><<<grid, kLdgThreads, 0, s>>>(a); break;
  }
  return cudaGetLastError();
}

// flags layout (debug / tuning sweeps; 0 everywhere = library defaults):
//   bits 0-7  KVB_COPY_* variant      bits 8-11  LDG unroll (2/4/8) or BULK depth code+1 (1..3)
//   bits 12-19 CTAs per SM            bits 20-23 BULK piece = 1 KiB << code (code 1..6)
template <int MODE>
static cudaError_t launch_ldg(CopyArgs a, int vec, int device, cudaStream_t s, int flags) {
  Tuning t = tuning();
  if ((flags >> 8) & 0xf) t.ldg_unroll = (flags >> 8) & 0xf;
  if ((flags >> 12) & 0xff) t.ldg_ctas_per_sm = (flags >> 12) & 0xff;
  int unroll = (t.ldg_unroll == 2 || t.ldg_unroll == 8) ? t.ldg_unroll : 4;
  a.piece = (uint32_t)(kLdgThreads * unroll * vec);
  a.ppf = (uint32_t)((a.frag + a.piece - 1) / a.piece);
  const uint64_t frags = a.total_items;  // caller passes n*T here
  a.total_items = frags * a.ppf;
  uint64_t cap = (uint64_t)sm_count(device) * (uint64_t)std::max(1, t.ldg_ctas_per_sm);
  int grid = (int)std::min<uint64_t>(a.total_items, cap);
  if (grid < 1) grid = 1;
  switch (vec) {
    case 16: return launch_ldg_v<MODE, int4>(a, grid, unroll, s);
    case 8: return launch_ldg_v<MODE, uint2>(a, grid, unroll, s);
    case 4: return launch_ldg_v<MODE, uint32_t>(a, grid, unroll, s);
    default: return launch_ldg_v<MODE, uint8_t>(a, grid, unroll, s);
  }
}

template <int MODE, int STAGES, int LOOKAHEAD>
static cudaError_t launch_bulk_cfg(const CopyArgs& a, int grid, size_t smem, cudaStream_t s) {
  auto k = paged_copy_bulk_kernel<MODE, STAGES, LOOKAHEAD>;
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k<<<grid, 32, smem, s>>>(a);
  return cudaGetLastError();
}

template <int MODE>
static cudaError_t launch_bulk(CopyArgs a, int device, cudaStream_t s, int flags) {
  Tuning t = tuning();
  if ((flags >> 8) & 0xf) t.bulk_deep = ((flags >> 8) & 0xf) - 1;
  if ((flags >> 12) & 0xff) t.bulk_ctas_per_sm = (flags >> 12) & 0xff;
  if ((flags >> 20) & 0xf) t.bulk_piece = 1024 << ((flags >> 20) & 0xf);
  int piece = t.bulk_piece;
  if (piece < 1024 || piece % 16) piece = 16384;
  const int stages = t.bulk_deep == 2 ? 12 : (t.bulk_deep == 1 ? 8 : 6);
  const int ctas = std::max(1, t.bulk_ctas_per_sm);
  // the rings of all resident CTAs must fit the SM's 227 KB of shared memory
  while (piece > 1024 && (size_t)piece * stages * ctas > 224u * 1024u) piece >>= 1;
  if ((int64_t)piece > a.frag) piece = (int)a.frag;  // frag is a multiple of 16 here
  a.piece = (uint32_t)piece;
  a.ppf = (uint32_t)((a.frag + a.piece - 1) / a.piece);
  const uint64_t frags = a.total_items;
  a.total_items = frags * a.ppf;
  size_t smem = (size_t)stages * a.piece;
  uint64_t cap = (uint64_t)sm_count(device) * (uint64_t)ctas;
  int grid = (int)std::min<uint64_t>(a.total_items, cap);
  if (grid < 1) grid = 1;
  switch (stages) {
    case 12: return launch_bulk_cfg<MODE, 12, 6>(a, grid, smem, s);
    case 8: return launch_bulk_cfg<MODE, 8, 4>(a, grid, smem, s);
    default: return launch_bulk_cfg<MODE, 6, 3>(a, grid, smem, s);
  }
}

template <int MODE>
static int launch_copy(CopyArgs a, int vec, int device, cudaStream_t s, int flags) {
  if (a.total_items == 0) return KVB_OK;
  int variant = flags & 0xff;
  if (variant == KVB_COPY_DEFAULT) variant = tuning().default_variant;
  // TMA bulk copies need 16 B aligned addresses and sizes; other shapes take the vector mover
  if (variant == KVB_COPY_BULK && vec != 16) variant = KVB_COPY_LDG;
  cudaError_t e = (variant == KVB_COPY_BULK) ? launch_bulk<MODE>(a, device, s, flags)
                                             : launch_ldg<MODE>(a, vec, device, s, flags);
  if (e != cudaSuccess) {
    set_error("paged copy launch failed: %s", cudaGetErrorString(e));
    return KVB_ERR_CUDA;
  }
  count_launch();
  return KVB_OK;
}

int launch_gather(const kvb_pool* pool, const int64_t* ids_dev, int64_t n, void* packed, cudaStream_t s, int flags) {
  CopyArgs a{};
  a.tensors = pool->d_tensor_ptrs;
  a.ids = ids_dev;
  a.packed = static_cast<uint8_t*>(packed);
  a.frag = pool->frag_bytes;
  a.stride = pool->stride_bytes;
  a.T = (uint32_t)pool->num_tensors;
  a.total_items = (uint64_t)n * (uint64_t)pool->num_tensors;
  int vec = pool->vec_bytes;
  while (vec > 1 && (reinterpret_cast<uintptr_t>(packed) % vec)) vec >>= 1;
  return launch_copy<kGather>(a, vec, pool->device, s, flags);
}

int launch_scatter(const kvb_pool* pool, const int64_t* ids_dev, int64_t n, const void* packed, cudaStream_t s,
                   int flags) {
  CopyArgs a{};
  a.tensors = pool->d_tensor_ptrs;
  a.ids = ids_dev;
  a.packed = const_cast<uint8_t*>(static_cast<const uint8_t*>(packed));
  a.frag = pool->frag_bytes;
  a.stride = pool->stride_bytes;
  a.T = (uint32_t)pool->num_tensors;
  a.total_items = (uint64_t)n * (uint64_t)pool->num_tensors;
  int vec = pool->vec_bytes;
  while (vec > 1 && (reinterpret_cast<uintptr_t>(packed) % vec)) vec >>= 1;
  return launch_copy<kScatter>(a, vec, pool->device, s, flags);
}

int launch_migrate(const kvb_pool* src, const kvb_pool* dst, const int64_t* src_ids_dev, const int64_t* dst_ids_dev,
                   int64_t n, cudaStream_t s, int flags) {
  CopyArgs a{};
  a.tensors = src->d_tensor_ptrs;
  a.tensors2 = dst->d_tensor_ptrs;  // must be addressable from src->device (same device, peer-mapped or IPC)
  a.ids = src_ids_dev;
  a.ids2 = dst_ids_dev;
  a.frag = src->frag_bytes;
  a.stride = src->stride_bytes;
  a.stride2 = dst->stride_bytes;
  a.T = (uint32_t)src->num_tensors;
  a.total_items = (uint64_t)n * (uint64_t)src->num_tensors;
  int vec = std::min(src->vec_bytes, dst->vec_bytes);
  // NVLink peer stores default to the 16 B LDG/STG mover (unroll 4, 8 CTAs/SM): registers keep more stores in flight
  // than the bulk ring's shared memory.  Not yet swept on H100 (tools/tune_migrate.py needs two GPUs); local HBM keeps bulk
  if ((flags & 0xff) == KVB_COPY_DEFAULT && dst->peer && vec == 16) flags = KVB_COPY_LDG | (4 << 8) | (8 << 12);
  return launch_copy<kMigrate>(a, vec, src->device, s, flags);
}

}  // namespace kvb
