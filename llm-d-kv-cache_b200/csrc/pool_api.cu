// pool_api.cu — error plumbing, pool objects and the gather/scatter/migrate C entry points.
#include <pthread.h>
#include <sched.h>
#include <sys/mman.h>

#include <algorithm>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "kvb_internal.h"

namespace kvb {

static thread_local char t_err[1024] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_err, sizeof(t_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return t_err; }

int sm_count(int device) {
  static std::mutex mu;
  static int cache[64];
  static bool have[64];
  std::lock_guard<std::mutex> lk(mu);
  if (device >= 0 && device < 64 && have[device]) return cache[device];
  int n = 132;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 132;
  if (device >= 0 && device < 64) {
    cache[device] = n;
    have[device] = true;
  }
  return n;
}

int validate_ids(const kvb_pool* pool, const int64_t* ids, int64_t n) {
  for (int64_t i = 0; i < n; ++i) {
    if (ids[i] < 0 || ids[i] >= pool->num_blocks) {
      set_error("block id %lld at position %lld out of range [0,%lld)", (long long)ids[i], (long long)i,
                (long long)pool->num_blocks);
      return KVB_ERR_INVALID;
    }
  }
  return KVB_OK;
}

// Upload ids through one slot of the pool's scratch ring (see kvb_internal.h).
int upload_ids(kvb_pool* pool, const int64_t* ids_host, int64_t n, cudaStream_t s, const int64_t** out_dev,
               cudaEvent_t* done_ev) {
  kvb_pool::IdSlot& sl = pool->id_slots[pool->next_slot];
  pool->next_slot = (pool->next_slot + 1) % kvb_pool::kIdSlots;
  if (!sl.free_ev) KVB_CUDA_TRY(cudaEventCreateWithFlags(&sl.free_ev, cudaEventDisableTiming));
  // previous user of this slot (pinned source AND device copy) must be done
  KVB_CUDA_TRY(cudaEventSynchronize(sl.free_ev));
  if (n > sl.cap) {
    if (sl.h_ids) cudaFreeHost(sl.h_ids);
    if (sl.d_ids) cudaFree(sl.d_ids);
    sl.h_ids = nullptr;
    sl.d_ids = nullptr;
    sl.cap = 0;
    int64_t cap = 1024;
    while (cap < n) cap <<= 1;
    KVB_CUDA_TRY(cudaHostAlloc(&sl.h_ids, cap * sizeof(int64_t), cudaHostAllocDefault));
    KVB_CUDA_TRY(cudaMalloc(&sl.d_ids, cap * sizeof(int64_t)));
    sl.cap = cap;
  }
  std::memcpy(sl.h_ids, ids_host, n * sizeof(int64_t));
  KVB_CUDA_TRY(cudaMemcpyAsync(sl.d_ids, sl.h_ids, n * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  *out_dev = sl.d_ids;
  *done_ev = sl.free_ev;
  return KVB_OK;
}

// ---------------------------------------------------------------------------------- NUMA placement
// The reference pins its I/O threads to the GPU-local NUMA node and prefers that node for staging memory
// (thread_pool.cpp:73-131, numa_utils.cpp).  Same intent without libnuma: read the GPU's node from sysfs and set the
// affinity of the threads that allocate (first touch => local pages) and drive the copies.
static int gpu_numa_node(int device) {
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
  std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
  FILE* f = fopen(path.c_str(), "r");
  if (!f) return -1;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  return node;
}
static std::vector<int> cpus_of_node(int node) {
  std::vector<int> cpus;
  if (node < 0) return cpus;
  std::string path = "/sys/devices/system/node/node" + std::to_string(node) + "/cpulist";
  FILE* f = fopen(path.c_str(), "r");
  if (!f) return cpus;
  char buf[4096] = {0};
  if (!fgets(buf, sizeof(buf), f)) buf[0] = 0;
  fclose(f);
  char* save = nullptr;
  for (char* tok = strtok_r(buf, ",\n", &save); tok; tok = strtok_r(nullptr, ",\n", &save)) {  // "0-31,64-95"
    int a = 0, b = 0;
    if (sscanf(tok, "%d-%d", &a, &b) == 2) {
      for (int c = a; c <= b; ++c) cpus.push_back(c);
    } else if (sscanf(tok, "%d", &a) == 1) {
      cpus.push_back(a);
    }
  }
  return cpus;
}
void bind_this_thread(const std::vector<int>& cpus) {
  if (cpus.empty()) return;
  cpu_set_t set;
  CPU_ZERO(&set);
  for (int c : cpus)
    if (c >= 0 && c < CPU_SETSIZE) CPU_SET(c, &set);
  pthread_setaffinity_np(pthread_self(), sizeof(set), &set);  // best effort
}


std::vector<int> gpu_local_cpus(int device) {
  if (std::getenv("KVB_NO_NUMA_BIND")) return {};
  static std::mutex mu;
  static std::map<int, std::vector<int>> cache;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(device);
  if (it == cache.end()) it = cache.emplace(device, cpus_of_node(gpu_numa_node(device))).first;
  return it->second;
}

// CPUs of every OTHER NUMA node (empty on a single-node box or with KVB_NO_NUMA_BIND): the file tier spreads its writer
// threads over all nodes, because what bounds it on tmpfs is page-cache insertion per node, not the copy
std::vector<int> gpu_remote_cpus(int device) {
  if (std::getenv("KVB_NO_NUMA_BIND")) return {};
  const int mine = gpu_numa_node(device);
  if (mine < 0) return {};
  std::vector<int> cpus;
  for (int node = 0; node < 64; ++node) {
    if (node == mine) continue;
    const std::vector<int> c = cpus_of_node(node);
    cpus.insert(cpus.end(), c.begin(), c.end());
  }
  return cpus;
}

// Pinned host memory placed on the GPU's NUMA node: allocated (pinning touches every page) from a short-lived thread
// bound to that node, so the caller's own affinity is left alone.
cudaError_t host_alloc_near(int device, void** out, size_t bytes, unsigned flags) {
  const std::vector<int> cpus = gpu_local_cpus(device);
  if (cpus.empty()) return cudaHostAlloc(out, bytes, flags);
  cudaError_t e = cudaSuccess;
  std::thread t([&] {
    bind_this_thread(cpus);
    cudaSetDevice(device);
    e = cudaHostAlloc(out, bytes, flags);
  });
  t.join();
  return e;
}

}  // namespace kvb

using namespace kvb;

extern "C" {

int kvb_abi_version(void) { return KVB_ABI_VERSION; }
const char* kvb_last_error(void) { return get_error(); }
int64_t kvb_launch_count(void) { return g_launches.load(); }

int kvb_device_count(void) {
  return kvb::guarded([&]() -> int {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
      cudaGetLastError();
      return 0;
    }
    return n;
  });
}

int kvb_pool_create(int device, const void* const* tensor_ptrs, int32_t num_tensors, int64_t num_blocks,
                    int64_t frag_bytes, int64_t block_stride_bytes, kvb_pool_t** out) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(out != nullptr, "kvb_pool_create: out is NULL");
    *out = nullptr;
    KVB_REQUIRE(tensor_ptrs != nullptr && num_tensors > 0, "kvb_pool_create: tensors is empty");  // tensor_copier.cu:34
    KVB_REQUIRE(num_blocks > 0 && frag_bytes > 0, "kvb_pool_create: num_blocks and frag_bytes must be > 0");
    if (block_stride_bytes == 0) block_stride_bytes = frag_bytes;
    KVB_REQUIRE(block_stride_bytes >= frag_bytes, "kvb_pool_create: block stride smaller than fragment");
    DeviceGuard g(device);
    if (!g.ok) {
      set_error("kvb_pool_create: cannot select CUDA device %d", device);
      return KVB_ERR_CUDA;
    }
    kvb_pool* p = new kvb_pool();
    p->device = device;
    p->num_tensors = num_tensors;
    p->num_blocks = num_blocks;
    p->frag_bytes = frag_bytes;
    p->stride_bytes = block_stride_bytes;
    int vec = 16;
    while (vec > 1 && ((frag_bytes % vec) || (block_stride_bytes % vec))) vec >>= 1;
    p->h_tensor_ptrs = new const uint8_t*[num_tensors];
    for (int i = 0; i < num_tensors; ++i) {
      if (!tensor_ptrs[i]) {
        set_error("kvb_pool_create: tensor %d is NULL", i);
        delete[] p->h_tensor_ptrs;
        delete p;
        return KVB_ERR_INVALID;
      }
      p->h_tensor_ptrs[i] = static_cast<const uint8_t*>(tensor_ptrs[i]);
      while (vec > 1 && (reinterpret_cast<uintptr_t>(tensor_ptrs[i]) % vec)) vec >>= 1;
    }
    p->vec_bytes = vec;
    {  // tensors that live on another GPU (peer-enabled or CUDA-IPC mapped): remember it for kernel selection
      cudaPointerAttributes attr;
      if (cudaPointerGetAttributes(&attr, tensor_ptrs[0]) == cudaSuccess) {
        p->peer = attr.type == cudaMemoryTypeDevice && attr.device != device;
      } else {
        cudaGetLastError();
      }
    }
    cudaError_t e = cudaMalloc(&p->d_tensor_ptrs, sizeof(void*) * num_tensors);
    if (e == cudaSuccess)
      e = cudaMemcpy(p->d_tensor_ptrs, p->h_tensor_ptrs, sizeof(void*) * num_tensors, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      set_error("kvb_pool_create: %s", cudaGetErrorString(e));
      if (p->d_tensor_ptrs) cudaFree(p->d_tensor_ptrs);
      delete[] p->h_tensor_ptrs;
      delete p;
      return KVB_ERR_CUDA;
    }
    *out = p;
    return KVB_OK;
  });
}

void kvb_pool_destroy(kvb_pool_t* p) {
  if (!p) return;
  DeviceGuard g(p->device);
  cudaDeviceSynchronize();
  if (p->d_tensor_ptrs) cudaFree(p->d_tensor_ptrs);
  for (auto& sl : p->id_slots) {
    if (sl.d_ids) cudaFree(sl.d_ids);
    if (sl.h_ids) cudaFreeHost(sl.h_ids);
    if (sl.free_ev) cudaEventDestroy(sl.free_ev);
  }
  delete[] p->h_tensor_ptrs;
  delete p;
}

int64_t kvb_pool_block_bytes(const kvb_pool_t* p) { return p ? p->frag_bytes * p->num_tensors : 0; }

int kvb_pool_mark_peer(kvb_pool_t* p, int is_peer) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(p != nullptr, "pool is NULL");
    p->peer = is_peer != 0;
    return KVB_OK;
  });
}

static int gs_host(kvb_pool_t* pool, const int64_t* ids, int64_t n, void* packed, void* stream, int flags,
                   bool gather) {
  KVB_REQUIRE(pool != nullptr, "pool is NULL");
  KVB_REQUIRE(n >= 0, "negative block count");
  if (n == 0) return KVB_OK;
  KVB_REQUIRE(ids != nullptr && packed != nullptr, "block_ids / packed is NULL");
  int rc = validate_ids(pool, ids, n);
  if (rc) return rc;
  DeviceGuard g(pool->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t* d = nullptr;
  cudaEvent_t done = nullptr;
  std::lock_guard<std::mutex> lk(pool->ids_mu);
  rc = upload_ids(pool, ids, n, s, &d, &done);
  if (rc) return rc;
  rc = gather ? launch_gather(pool, d, n, packed, s, flags) : launch_scatter(pool, d, n, packed, s, flags);
  cudaEventRecord(done, s);
  return rc;
}

int kvb_gather_blocks(kvb_pool_t* pool, const int64_t* ids, int64_t n, void* packed, void* stream, int flags) {
  return kvb::guarded([&]() -> int {
    return gs_host(pool, ids, n, packed, stream, flags, true);
  });
}
int kvb_scatter_blocks(kvb_pool_t* pool, const int64_t* ids, int64_t n, const void* packed, void* stream,
                       int flags) {
  return kvb::guarded([&]() -> int {
    return gs_host(pool, ids, n, const_cast<void*>(packed), stream, flags, false);
  });
}
int kvb_gather_blocks_dev(kvb_pool_t* pool, const int64_t* ids_dev, int64_t n, void* packed, void* stream,
                          int flags) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(pool && (n == 0 || (ids_dev && packed)), "NULL argument");
    KVB_REQUIRE(n >= 0, "negative block count");
    DeviceGuard g(pool->device);
    return launch_gather(pool, ids_dev, n, packed, static_cast<cudaStream_t>(stream), flags);
  });
}
int kvb_scatter_blocks_dev(kvb_pool_t* pool, const int64_t* ids_dev, int64_t n, const void* packed, void* stream,
                           int flags) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(pool && (n == 0 || (ids_dev && packed)), "NULL argument");
    KVB_REQUIRE(n >= 0, "negative block count");
    DeviceGuard g(pool->device);
    return launch_scatter(pool, ids_dev, n, packed, static_cast<cudaStream_t>(stream), flags);
  });
}

// pinned host memory for callers that want zero staging copies (token buffers, host-tier staging)
// mode KVB_HOST_ALLOC_THP buffers: anonymous memory advised to transparent huge pages, first-touched on the GPU's NUMA
// node, then registered with CUDA; remembered here so that kvb_host_free knows how to release them
static std::mutex g_thp_mu;
static std::map<void*, size_t> g_thp_regions;

}  // extern "C"

namespace kvb {
// pinned host memory for `device`, placed on its NUMA node; mode = KVB_HOST_ALLOC_*.  Released with host_free_any.
int host_alloc_mode(int device, size_t bytes, int mode, void** out) {
  if (mode == KVB_HOST_ALLOC_DEFAULT) {
    KVB_CUDA_TRY(host_alloc_near(device, out, bytes, cudaHostAllocPortable));
    return KVB_OK;
  }
  const size_t len = (bytes + (2u << 20) - 1) & ~(size_t)((2u << 20) - 1);
  void* p = ::mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  if (p == MAP_FAILED) {
    set_error("mmap of %zu bytes failed", len);
    return KVB_ERR_NOMEM;
  }
  ::madvise(p, len, MADV_HUGEPAGE);  // best effort: without THP these are ordinary pages
  const std::vector<int> cpus = gpu_local_cpus(device);
  {  // first touch from the GPU's node (a few threads: page faults of a multi-GB region on one thread take seconds)
    const int nt = 8;
    std::vector<std::thread> th;
    const size_t part = ((len / nt) + (2u << 20) - 1) & ~(size_t)((2u << 20) - 1);
    for (int k = 0; k < nt; ++k) {
      const size_t lo = (size_t)k * part;
      if (lo >= len) break;
      const size_t n = std::min(part, len - lo);
      th.emplace_back([=, &cpus] {
        bind_this_thread(cpus);
        std::memset(static_cast<uint8_t*>(p) + lo, 0, n);
      });
    }
    for (auto& t : th) t.join();
  }
  cudaError_t e = cudaSuccess;
  {
    DeviceGuard g(device);
    e = cudaHostRegister(p, len, cudaHostRegisterPortable | cudaHostRegisterMapped);
  }
  if (e != cudaSuccess) {
    ::munmap(p, len);
    set_error("cudaHostRegister of %zu bytes failed: %s", len, cudaGetErrorString(e));
    return KVB_ERR_CUDA;
  }
  {
    std::lock_guard<std::mutex> lk(g_thp_mu);
    g_thp_regions[p] = len;
  }
  *out = p;
  return KVB_OK;
}
int host_free_any(void* p) {
  if (!p) return KVB_OK;
  size_t len = 0;
  {
    std::lock_guard<std::mutex> lk(g_thp_mu);
    auto it = g_thp_regions.find(p);
    if (it != g_thp_regions.end()) {
      len = it->second;
      g_thp_regions.erase(it);
    }
  }
  if (len) {
    KVB_CUDA_TRY(cudaHostUnregister(p));
    ::munmap(p, len);
    return KVB_OK;
  }
  KVB_CUDA_TRY(cudaFreeHost(p));
  return KVB_OK;
}
}  // namespace kvb

extern "C" {

int kvb_host_alloc_mode(size_t bytes, int mode, void** out) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(out != nullptr && bytes > 0, "bad argument");
    KVB_REQUIRE(mode == KVB_HOST_ALLOC_DEFAULT || mode == KVB_HOST_ALLOC_THP, "unknown host allocation mode %d", mode);
    int dev = 0;
    KVB_CUDA_TRY(cudaGetDevice(&dev));  // placed on the NUMA node of the caller's current device
    return kvb::host_alloc_mode(dev, bytes, mode, out);
  });
}
int kvb_host_alloc(size_t bytes, void** out) { return kvb_host_alloc_mode(bytes, KVB_HOST_ALLOC_DEFAULT, out); }
int kvb_host_free(void* p) {
  return kvb::guarded([&]() -> int { return kvb::host_free_any(p); });
}

// ------------------------------------------------------------------------------- migration / IPC
int kvb_ipc_export(int device, const void* dev_ptr, kvb_ipc_mem_t* out) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(dev_ptr && out, "NULL argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == KVB_IPC_HANDLE_BYTES, "handle size");
    DeviceGuard g(device);
    // cudaIpcGetMemHandle returns the handle of the containing allocation; find its base for the offset
    void* base = nullptr;
    size_t size = 0;
    cudaPointerAttributes attr;
    KVB_CUDA_TRY(cudaPointerGetAttributes(&attr, dev_ptr));
    typedef int (*cuMemGetAddressRange_t)(unsigned long long*, size_t*, unsigned long long);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    KVB_CUDA_TRY(cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess) {
      set_error("cuMemGetAddressRange entry point unavailable");
      return KVB_ERR_CUDA;
    }
    unsigned long long b = 0;
    int dr = reinterpret_cast<cuMemGetAddressRange_t>(fn)(&b, &size, (unsigned long long)(uintptr_t)dev_ptr);
    if (dr != 0) {
      set_error("cuMemGetAddressRange failed (%d)", dr);
      return KVB_ERR_CUDA;
    }
    base = reinterpret_cast<void*>((uintptr_t)b);
    cudaIpcMemHandle_t h;
    KVB_CUDA_TRY(cudaIpcGetMemHandle(&h, base));
    std::memcpy(out->handle, &h, sizeof(h));
    out->offset = (int64_t)((const uint8_t*)dev_ptr - (const uint8_t*)base);
    return KVB_OK;
  });
}

int kvb_ipc_import(int device, const kvb_ipc_mem_t* mem, void** out_ptr) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(mem && out_ptr, "NULL argument");
    DeviceGuard g(device);
    cudaIpcMemHandle_t h;
    std::memcpy(&h, mem->handle, sizeof(h));
    void* base = nullptr;
    KVB_CUDA_TRY(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    *out_ptr = static_cast<uint8_t*>(base) + mem->offset;
    return KVB_OK;
  });
}

int kvb_ipc_close(int device, void* imported_ptr, int64_t offset) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(imported_ptr, "NULL argument");
    DeviceGuard g(device);
    KVB_CUDA_TRY(cudaIpcCloseMemHandle(static_cast<uint8_t*>(imported_ptr) - offset));
    return KVB_OK;
  });
}

int kvb_enable_peer_access(int device, int peer) {
  return kvb::guarded([&]() -> int {
    DeviceGuard g(device);
    int can = 0;
    KVB_CUDA_TRY(cudaDeviceCanAccessPeer(&can, device, peer));
    if (!can) {
      set_error("device %d cannot access peer %d", device, peer);
      return KVB_ERR_UNSUPPORTED;
    }
    cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) {
      cudaGetLastError();
      return KVB_OK;
    }
    KVB_CUDA_TRY(e);
    return KVB_OK;
  });
}

int kvb_migrate_blocks(kvb_pool_t* src, kvb_pool_t* dst, const int64_t* src_ids, const int64_t* dst_ids, int64_t n,
                       void* stream, int flags) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(src && dst, "pool is NULL");
    KVB_REQUIRE(n >= 0, "negative block count");
    if (n == 0) return KVB_OK;
    KVB_REQUIRE(src_ids && dst_ids, "ids NULL");
    KVB_REQUIRE(src->num_tensors == dst->num_tensors && src->frag_bytes == dst->frag_bytes,
                "migrate: pools differ in shape (T %d vs %d, frag %lld vs %lld)", src->num_tensors, dst->num_tensors,
                (long long)src->frag_bytes, (long long)dst->frag_bytes);
    KVB_REQUIRE(dst->device == src->device,
                "migrate: describe the destination pool on the source device (peer/IPC pointers)");
    int rc = validate_ids(src, src_ids, n);
    if (rc) return rc;
    rc = validate_ids(dst, dst_ids, n);
    if (rc) return rc;
    DeviceGuard g(src->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    // both id lists go through one scratch upload: [src ids | dst ids]
    std::vector<int64_t> both(2 * n);
    std::memcpy(both.data(), src_ids, n * sizeof(int64_t));
    std::memcpy(both.data() + n, dst_ids, n * sizeof(int64_t));
    const int64_t* d = nullptr;
    cudaEvent_t done = nullptr;
    std::lock_guard<std::mutex> lk(src->ids_mu);
    rc = upload_ids(src, both.data(), 2 * n, s, &d, &done);
    if (rc) return rc;
    rc = launch_migrate(src, dst, d, d + n, n, s, flags);
    cudaEventRecord(done, s);
    return rc;
  });
}

int kvb_pool_set_geometry(kvb_pool_t* p, const kvb_kv_geometry_t* g) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(p && g, "NULL argument");
    KVB_REQUIRE(g->planes >= 1 && g->tokens >= 1 && g->heads >= 1 && g->head_bytes >= 1,
                "geometry: planes, tokens, heads and head_bytes must be >= 1 (got %d, %d, %d, %d)", g->planes,
                g->tokens, g->heads, g->head_bytes);
    KVB_REQUIRE(g->layout == KVB_KV_LAYOUT_NHD || g->layout == KVB_KV_LAYOUT_HND, "geometry: unknown layout %d",
                g->layout);
    const int64_t bytes = (int64_t)g->planes * g->tokens * g->heads * g->head_bytes;
    KVB_REQUIRE(bytes == p->frag_bytes, "geometry: planes x tokens x heads x head_bytes = %lld, fragment is %lld B",
                (long long)bytes, (long long)p->frag_bytes);
    KVB_REQUIRE(bytes <= 0xffffffffll, "geometry: fragments of 4 GiB or more are not supported");
    p->geom = *g;
    p->geom.pad = 0;
    p->has_geom = true;
    return KVB_OK;
  });
}

int kvb_migrate_heads(kvb_pool_t* src, kvb_pool_t* dst, const int64_t* src_ids, const int64_t* dst_ids, int64_t n,
                      int32_t src_head0, int32_t dst_head0, int32_t n_heads, void* stream, int flags) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(src && dst, "pool is NULL");
    KVB_REQUIRE(n >= 0, "negative block count");
    KVB_REQUIRE(src->has_geom && dst->has_geom, "migrate_heads: the %s pool has no KV geometry",
                src->has_geom ? "destination" : "source");
    const kvb_kv_geometry_t &gs = src->geom, &gd = dst->geom;
    KVB_REQUIRE(src->num_tensors == dst->num_tensors && gs.planes == gd.planes && gs.tokens == gd.tokens &&
                    gs.head_bytes == gd.head_bytes,
                "migrate_heads: pools differ in shape (T %d vs %d, planes %d vs %d, tokens %d vs %d, head_bytes %d vs %d)",
                src->num_tensors, dst->num_tensors, gs.planes, gd.planes, gs.tokens, gd.tokens, gs.head_bytes,
                gd.head_bytes);
    KVB_REQUIRE(n_heads >= 1 && src_head0 >= 0 && dst_head0 >= 0 && (int64_t)src_head0 + n_heads <= gs.heads &&
                    (int64_t)dst_head0 + n_heads <= gd.heads,
                "migrate_heads: heads [%d, +%d) -> [%d, +%d) out of range (source holds %d, destination %d)", src_head0,
                n_heads, dst_head0, n_heads, gs.heads, gd.heads);
    KVB_REQUIRE(dst->device == src->device,
                "migrate_heads: describe the destination pool on the source device (peer/IPC pointers)");
    if (n == 0) return KVB_OK;
    KVB_REQUIRE(src_ids && dst_ids, "ids NULL");
    int rc = validate_ids(src, src_ids, n);
    if (rc) return rc;
    rc = validate_ids(dst, dst_ids, n);
    if (rc) return rc;
    DeviceGuard g(src->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    std::vector<int64_t> both(2 * n);  // one scratch upload: [src ids | dst ids]
    std::memcpy(both.data(), src_ids, n * sizeof(int64_t));
    std::memcpy(both.data() + n, dst_ids, n * sizeof(int64_t));
    const int64_t* d = nullptr;
    cudaEvent_t done = nullptr;
    std::lock_guard<std::mutex> lk(src->ids_mu);
    rc = upload_ids(src, both.data(), 2 * n, s, &d, &done);
    if (rc) return rc;
    rc = launch_migrate_heads(src, dst, d, d + n, n, src_head0, dst_head0, n_heads, s, flags);
    cudaEventRecord(done, s);
    return rc;
  });
}

int kvb_migrate_tokens(kvb_pool_t* src, kvb_pool_t* dst, const kvb_token_segment_t* segs, int64_t n_segs,
                       int32_t src_head0, int32_t dst_head0, int32_t n_heads, void* stream, int flags) {
  static_assert(sizeof(kvb_token_segment_t) == 4 * sizeof(int64_t), "a segment travels as 4 id words");
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(src && dst, "pool is NULL");
    KVB_REQUIRE(n_segs >= 0, "negative segment count");
    KVB_REQUIRE(src->has_geom && dst->has_geom, "migrate_tokens: the %s pool has no KV geometry",
                src->has_geom ? "destination" : "source");
    const kvb_kv_geometry_t &gs = src->geom, &gd = dst->geom;
    KVB_REQUIRE(src->num_tensors == dst->num_tensors && gs.planes == gd.planes && gs.head_bytes == gd.head_bytes,
                "migrate_tokens: pools differ in shape (T %d vs %d, planes %d vs %d, head_bytes %d vs %d)",
                src->num_tensors, dst->num_tensors, gs.planes, gd.planes, gs.head_bytes, gd.head_bytes);
    KVB_REQUIRE(n_heads >= 1 && src_head0 >= 0 && dst_head0 >= 0 && (int64_t)src_head0 + n_heads <= gs.heads &&
                    (int64_t)dst_head0 + n_heads <= gd.heads,
                "migrate_tokens: heads [%d, +%d) -> [%d, +%d) out of range (source holds %d, destination %d)",
                src_head0, n_heads, dst_head0, n_heads, gs.heads, gd.heads);
    KVB_REQUIRE(dst->device == src->device,
                "migrate_tokens: describe the destination pool on the source device (peer/IPC pointers)");
    if (n_segs == 0) return KVB_OK;
    KVB_REQUIRE(segs, "segments NULL");
    int32_t max_n = 0;
    bool whole = true;  // every segment covers a whole block on both sides
    for (int64_t i = 0; i < n_segs; ++i) {
      const kvb_token_segment_t& g = segs[i];
      KVB_REQUIRE(g.n_tokens >= 1 && g.src_tok0 >= 0 && g.dst_tok0 >= 0 &&
                      (int64_t)g.src_tok0 + g.n_tokens <= gs.tokens && (int64_t)g.dst_tok0 + g.n_tokens <= gd.tokens,
                  "migrate_tokens: segment %lld tokens [%d, +%d) -> [%d, +%d) out of range (blocks of %d and %d tokens)",
                  (long long)i, g.src_tok0, g.n_tokens, g.dst_tok0, g.n_tokens, gs.tokens, gd.tokens);
      KVB_REQUIRE(g.src_block >= 0 && g.src_block < src->num_blocks && g.dst_block >= 0 &&
                      g.dst_block < dst->num_blocks,
                  "migrate_tokens: segment %lld blocks %lld -> %lld out of range [0,%lld) -> [0,%lld)", (long long)i,
                  (long long)g.src_block, (long long)g.dst_block, (long long)src->num_blocks,
                  (long long)dst->num_blocks);
      max_n = std::max(max_n, g.n_tokens);
      whole = whole && g.src_tok0 == 0 && g.dst_tok0 == 0 && g.n_tokens == gs.tokens && g.n_tokens == gd.tokens;
    }
    {  // no destination token is written twice: sorted by (block, first token), each range ends before the next starts
      std::vector<int64_t> order(n_segs);
      for (int64_t i = 0; i < n_segs; ++i) order[i] = i;
      std::sort(order.begin(), order.end(), [&](int64_t a, int64_t b) {
        return segs[a].dst_block != segs[b].dst_block ? segs[a].dst_block < segs[b].dst_block
                                                      : segs[a].dst_tok0 < segs[b].dst_tok0;
      });
      for (int64_t k = 1; k < n_segs; ++k) {
        const kvb_token_segment_t &a = segs[order[k - 1]], &b = segs[order[k]];
        KVB_REQUIRE(a.dst_block != b.dst_block || a.dst_tok0 + a.n_tokens <= b.dst_tok0,
                    "migrate_tokens: segments %lld and %lld overlap in destination block %lld",
                    (long long)order[k - 1], (long long)order[k], (long long)b.dst_block);
      }
    }
    DeviceGuard g(src->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int64_t* d = nullptr;
    cudaEvent_t done = nullptr;
    int rc;
    if (whole) {  // whole blocks on both sides: exactly kvb_migrate_heads on the two id lists
      std::vector<int64_t> both(2 * n_segs);
      for (int64_t i = 0; i < n_segs; ++i) {
        both[i] = segs[i].src_block;
        both[n_segs + i] = segs[i].dst_block;
      }
      std::lock_guard<std::mutex> lk(src->ids_mu);
      rc = upload_ids(src, both.data(), 2 * n_segs, s, &d, &done);
      if (rc) return rc;
      rc = launch_migrate_heads(src, dst, d, d + n_segs, n_segs, src_head0, dst_head0, n_heads, s, flags);
      cudaEventRecord(done, s);
      return rc;
    }
    std::lock_guard<std::mutex> lk(src->ids_mu);  // the segments travel through the id ring as 4 words each
    rc = upload_ids(src, reinterpret_cast<const int64_t*>(segs), 4 * n_segs, s, &d, &done);
    if (rc) return rc;
    rc = launch_migrate_tokens(src, dst, reinterpret_cast<const kvb_token_segment_t*>(d), n_segs, max_n, src_head0,
                               dst_head0, n_heads, s, flags);
    cudaEventRecord(done, s);
    return rc;
  });
}

}  // extern "C"
