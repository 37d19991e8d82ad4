// kvb_internal.h — shared helpers for libkvb.so (not part of the ABI).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <exception>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "kvb.h"

namespace kvb {

// ---- error plumbing: thread-local message, integer status across the C ABI ----
void set_error(const char* fmt, ...);
const char* get_error();

#define KVB_CUDA_TRY(expr)                                                                       \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      ::kvb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return KVB_ERR_CUDA;                                                                       \
    }                                                                                            \
  } while (0)

#define KVB_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) {                        \
      ::kvb::set_error(__VA_ARGS__);      \
      return KVB_ERR_INVALID;             \
    }                                     \
  } while (0)

// No C++ exception may cross the C ABI: every int-returning entry point runs its body through this.
template <class F>
static inline int guarded(F&& f) noexcept {
  try {
    return f();
  } catch (const std::bad_alloc&) {
    set_error("out of host memory");
    return KVB_ERR_NOMEM;
  } catch (const std::exception& e) {
    set_error("unexpected exception: %s", e.what());
    return KVB_ERR_INVALID;
  } catch (...) {
    set_error("unexpected exception");
    return KVB_ERR_INVALID;
  }
}

// NUMA placement (pool_api.cu): CPUs of the GPU's node (empty: unknown or KVB_NO_NUMA_BIND), thread binding, and
// pinned host memory first-touched on that node.
std::vector<int> gpu_local_cpus(int device);
std::vector<int> gpu_remote_cpus(int device);  // CPUs of the other NUMA nodes
void bind_this_thread(const std::vector<int>& cpus);
cudaError_t host_alloc_near(int device, void** out, size_t bytes, unsigned flags);
int host_alloc_mode(int device, size_t bytes, int mode, void** out);  // KVB_HOST_ALLOC_*; release with host_free_any
int host_free_any(void* p);

// Set the device for the duration of a scope and restore the caller's on exit
// (the caller is typically a torch process that owns "current device").
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; }
    if (prev != dev) ok = (cudaSetDevice(dev) == cudaSuccess);
  }
  ~DeviceGuard() {
    int cur = -1;
    if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
  }
};

extern std::atomic<int64_t> g_launches;  // kernels launched by this library
inline void count_launch(int64_t n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count(int device);

}  // namespace kvb

// ---- pool (section 1 of kvb.h) ----
struct kvb_pool {
  int device = 0;
  int32_t num_tensors = 0;
  int64_t num_blocks = 0;
  int64_t frag_bytes = 0;
  int64_t stride_bytes = 0;
  const uint8_t** d_tensor_ptrs = nullptr;  // device array [T]
  const uint8_t** h_tensor_ptrs = nullptr;  // host copy [T]
  int vec_bytes = 16;                        // widest aligned vector usable for every fragment (16/8/4/1)
  bool peer = false;                         // tensors live on another GPU (peer / CUDA-IPC mapping)
  // ring of pinned + device scratch slots for uploading block ids: a slot is rewritten only after the kernel that
  // read it has finished (event), and calls on different streams use different slots, so they do not serialise
  static constexpr int kIdSlots = 8;
  struct IdSlot {
    int64_t* h_ids = nullptr;
    int64_t* d_ids = nullptr;
    int64_t cap = 0;
    cudaEvent_t free_ev = nullptr;
  } id_slots[kIdSlots];
  int next_slot = 0;
  // held by a host-id call from taking its slot until it has recorded the slot's event: calls from several host
  // threads must neither share a slot nor let the ring come round to a slot before its release is recorded
  std::mutex ids_mu;
  // how each fragment holds its KV heads (kvb_pool_set_geometry); kvb_migrate_heads and kvb_migrate_tokens refuse pools
  // without one
  bool has_geom = false;
  kvb_kv_geometry_t geom{};
};

namespace kvb {
// Launch the paged copy.  ids_dev: device int64[n].  dst_ids_dev != nullptr => page->page migration
// (packed unused, dst_pool required).
int launch_gather(const kvb_pool* pool, const int64_t* ids_dev, int64_t n, void* packed, cudaStream_t s, int flags);
int launch_scatter(const kvb_pool* pool, const int64_t* ids_dev, int64_t n, const void* packed, cudaStream_t s,
                   int flags);
int launch_migrate(const kvb_pool* src, const kvb_pool* dst, const int64_t* src_ids_dev, const int64_t* dst_ids_dev,
                   int64_t n, cudaStream_t s, int flags);
// heads [src_head0, +n_heads) of src's fragments -> heads [dst_head0, +n_heads) of dst's (both pools carry a geometry,
// arguments already checked); the whole fragment in the same layout goes to launch_migrate
int launch_migrate_heads(const kvb_pool* src, const kvb_pool* dst, const int64_t* src_ids_dev,
                         const int64_t* dst_ids_dev, int64_t n, int src_head0, int dst_head0, int n_heads,
                         cudaStream_t s, int flags);
// token segments segs_dev[0, n) of src -> dst with heads [src_head0, +n_heads) -> [dst_head0, +n_heads) (arguments
// already checked; whole-block calls are routed to launch_migrate_heads by the caller); max_n: largest n_tokens
int launch_migrate_tokens(const kvb_pool* src, const kvb_pool* dst, const kvb_token_segment_t* segs_dev, int64_t n,
                          int32_t max_n, int src_head0, int dst_head0, int n_heads, cudaStream_t s, int flags);
// copies ids into a free scratch slot and enqueues the H2D on s; after launching the kernel that reads *out_dev the
// caller records *done_ev on s (release of the slot).  The caller holds pool->ids_mu from before this call until that
// record.
int upload_ids(kvb_pool* pool, const int64_t* ids_host, int64_t n, cudaStream_t s, const int64_t** out_dev,
               cudaEvent_t* done_ev);
int validate_ids(const kvb_pool* pool, const int64_t* ids_host, int64_t n);

// hashing (device-resident arguments)
struct SpecScratch;  // tables of the table kernel (hash_kernels.cu), owned by the caller
SpecScratch* spec_scratch_create();
void spec_scratch_destroy(SpecScratch* sc);
int launch_hash_blocks(const uint32_t* tokens, const int64_t* prompt_off, const uint64_t* parents, int32_t n_prompts,
                       int32_t block_size, const uint8_t* extra, const int64_t* extra_off, uint64_t* out_keys,
                       const int64_t* key_off, cudaStream_t s, int64_t total_keys = -1,
                       const int64_t* h_prompt_off = nullptr, const int64_t* h_key_off = nullptr,
                       const uint64_t* h_parents = nullptr, SpecScratch* scratch = nullptr);
// total_keys: key_off[n_prompts] if the caller knows it; h_*: host-readable copies of the three small arrays, if at hand
// (a handful of prompts then travels in the launch arguments); scratch: the caller's table-kernel scratch (else a shared
// one per device and stream)
}  // namespace kvb
