// engine.cu — asynchronous offload engine: save_blocks / load_blocks behind the reference's
// StorageOffloadEngine surface (kv_connectors/llmd_fs_backend/csrc/storage/storage_offload.cpp).
//
// What is kept from the reference (so the vLLM plugin sees the same behaviour):
//   * submit-only store/load, get_finished() draining (job_id, ok), wait_job() cancelling queued work
//     (storage_offload.cpp:185-233,249-423);
//   * two FIFO queues, loads (high) before stores (normal) with per-worker preference (thread_pool.cpp:169-190);
//   * store skips files that already exist and bumps atime (storage_offload.cpp:299-304, file_io.cpp:144-149);
//   * EMA-based dynamic write-queue limit that drops stores (storage_offload.cpp:80-108,272-288);
//   * on-disk format of the CPU path: file of max(bpf*block_bytes, 16 MiB), blocks tail-aligned, written to a
//     temp name and renamed (file_io.cpp:50-101, tensor_copier.cu:75-76).
// What is different (GPU-first):
//   * the unit of GPU work is a CHUNK of whole files (tens of MiB), not one (block x tensor) fragment:
//     one gather kernel packs the chunk in HBM, ONE large pinned-async D2H moves it (the reference issues
//     blocks x tensors cudaMemcpyAsync calls of 16-64 KiB); loads are the inverse H2D -> scatter;
//   * a host tier in pinned DRAM (KVB_TIER_HOST_ARENA) addressed by the same path strings, D2H lands
//     directly in its final place (no staging copy on the host).
#include <cufile.h>  // types only: the library is loaded at run time (the reference does the same, cufile_loader.hpp)
#include <dlfcn.h>
#include <fcntl.h>
#include <pthread.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/types.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cerrno>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <future>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "kvb_internal.h"

namespace kvb {

constexpr int64_t kMinFileBytes = 16ll * 1024 * 1024;  // thread_pool.cpp:35 MIN_STAGING_BUFFER_SIZE
constexpr double kEmaAlpha = 0.05;                       // storage_offload.cpp:78

struct JobState {
  int64_t id = 0;
  std::atomic<int> completed{0};
  int total = 0;
  std::atomic<bool> ok{true};
  std::atomic<bool> cancelled{false};
};

struct FilePart {
  std::string path;
  std::vector<int64_t> ids;
};

struct ChunkTask {
  std::shared_ptr<JobState> job;
  bool is_store = false;
  std::vector<FilePart> files;  // whole files, total blocks <= blocks_per_chunk
  int64_t n_blocks = 0;
  int io_parts = 1;             // >1: nothing else was queued when the task started -> split file I/O for latency
  cudaEvent_t ready = nullptr;  // caller-stream event (shared by the job's chunks, owned by last user)
  std::shared_ptr<void> ready_owner;
};

// ---------------------------------------------------------------------------------- host arena
class Arena {
 public:
  struct Entry {
    int64_t off = 0;
    int64_t n_blocks = 0;
    int pins = 0;
    bool valid = false;  // data landed
    std::list<std::string>::iterator lru;
  };
  uint8_t* base = nullptr;
  int64_t cap = 0;
  std::mutex mu;
  std::map<int64_t, int64_t> free_;  // offset -> size
  std::unordered_map<std::string, Entry> entries;
  std::list<std::string> lru;  // front = oldest

  int init(int device, int64_t bytes, int alloc_mode) {
    cap = bytes;
    void* p = nullptr;
    if (host_alloc_mode(device, (size_t)bytes, alloc_mode, &p) != KVB_OK) {
      const std::string why = get_error();
      set_error("host arena of %lld bytes: %s", (long long)bytes, why.c_str());
      base = nullptr;
      return KVB_ERR_NOMEM;
    }
    base = static_cast<uint8_t*>(p);
    free_[0] = bytes;
    return KVB_OK;
  }
  void destroy() {
    if (base) host_free_any(base);
    base = nullptr;
  }
  bool exists(const std::string& k) {
    std::lock_guard<std::mutex> lk(mu);
    auto it = entries.find(k);
    return it != entries.end() && it->second.valid;
  }
  int32_t count_prefix(const char* const* keys, int32_t n) {  // consecutive valid entries from the start, one lock
    std::lock_guard<std::mutex> lk(mu);
    int32_t hits = 0;
    for (; hits < n; ++hits) {
      if (!keys[hits]) break;
      auto it = entries.find(keys[hits]);
      if (it == entries.end() || !it->second.valid) break;
    }
    return hits;
  }
  void clear() {  // drops every entry that is not pinned by an in-flight store or load
    std::lock_guard<std::mutex> lk(mu);
    for (auto it = entries.begin(); it != entries.end();) {
      auto cur = it++;
      if (cur->second.pins == 0) erase_locked(cur);
    }
  }
  // reserve space for a new entry (pinned for writing); evicts unpinned LRU entries when full.
  // returns nullptr if the key exists already (*existed=true) or no space can be made.
  uint8_t* reserve(const std::string& k, int64_t n_blocks, int64_t bytes, bool* existed) {
    std::lock_guard<std::mutex> lk(mu);
    *existed = false;
    if (entries.count(k)) {
      *existed = true;
      touch_locked(k);
      return nullptr;
    }
    int64_t off = alloc_locked(bytes);
    while (off < 0) {
      if (!evict_one_locked()) return nullptr;
      off = alloc_locked(bytes);
    }
    Entry e;
    e.off = off;
    e.n_blocks = n_blocks;
    e.pins = 1;
    e.valid = false;
    lru.push_back(k);
    e.lru = std::prev(lru.end());
    entries.emplace(k, e);
    bytes_of_[k] = bytes;
    return base + off;
  }
  void commit(const std::string& k, bool ok) {
    std::lock_guard<std::mutex> lk(mu);
    auto it = entries.find(k);
    if (it == entries.end()) return;
    it->second.pins--;
    if (ok) {
      it->second.valid = true;
    } else {
      erase_locked(it);
    }
  }
  // pin an entry for reading the LAST n_blocks blocks of it (tail-aligned, like the file format)
  const uint8_t* pin_read(const std::string& k, int64_t n_blocks, int64_t block_bytes) {
    std::lock_guard<std::mutex> lk(mu);
    auto it = entries.find(k);
    if (it == entries.end() || !it->second.valid || it->second.n_blocks < n_blocks) return nullptr;
    it->second.pins++;
    touch_locked(k);
    return base + it->second.off + (it->second.n_blocks - n_blocks) * block_bytes;
  }
  void unpin(const std::string& k) {
    std::lock_guard<std::mutex> lk(mu);
    auto it = entries.find(k);
    if (it != entries.end()) it->second.pins--;
  }

 private:
  std::unordered_map<std::string, int64_t> bytes_of_;
  void touch_locked(const std::string& k) {
    auto it = entries.find(k);
    if (it == entries.end()) return;
    lru.erase(it->second.lru);
    lru.push_back(k);
    it->second.lru = std::prev(lru.end());
  }
  int64_t alloc_locked(int64_t bytes) {
    for (auto it = free_.begin(); it != free_.end(); ++it) {
      if (it->second >= bytes) {
        int64_t off = it->first, sz = it->second;
        free_.erase(it);
        if (sz > bytes) free_[off + bytes] = sz - bytes;
        return off;
      }
    }
    return -1;
  }
  void free_locked(int64_t off, int64_t bytes) {
    auto nx = free_.lower_bound(off);
    if (nx != free_.begin()) {
      auto pv = std::prev(nx);
      if (pv->first + pv->second == off) {
        off = pv->first;
        bytes += pv->second;
        free_.erase(pv);
      }
    }
    if (nx != free_.end() && off + bytes == nx->first) {
      bytes += nx->second;
      free_.erase(nx);
    }
    free_[off] = bytes;
  }
  void erase_locked(std::unordered_map<std::string, Entry>::iterator it) {
    free_locked(it->second.off, bytes_of_[it->first]);
    lru.erase(it->second.lru);
    bytes_of_.erase(it->first);
    entries.erase(it);
  }
  bool evict_one_locked() {
    for (auto li = lru.begin(); li != lru.end(); ++li) {
      auto it = entries.find(*li);
      if (it != entries.end() && it->second.pins == 0) {
        erase_locked(it);
        return true;
      }
    }
    return false;
  }
};

// ---------------------------------------------------------------------------------- file helpers
static bool file_exists(const std::string& p) {
  struct stat st;
  return ::stat(p.c_str(), &st) == 0;
}
static void touch_atime(const std::string& p) {  // file_io.cpp:144-149
  struct timespec times[2];
  times[0].tv_sec = 0;
  times[0].tv_nsec = UTIME_NOW;
  times[1].tv_sec = 0;
  times[1].tv_nsec = UTIME_OMIT;
  ::utimensat(AT_FDCWD, p.c_str(), times, 0);
}
static bool mkdirs(const std::string& dir) {
  if (dir.empty()) return true;
  struct stat st;
  if (::stat(dir.c_str(), &st) == 0) return S_ISDIR(st.st_mode);
  size_t pos = dir.find_last_of('/');
  if (pos != std::string::npos && pos > 0 && !mkdirs(dir.substr(0, pos))) return false;
  if (::mkdir(dir.c_str(), 0777) != 0 && errno != EEXIST) return false;
  return true;
}
static bool write_all(int fd, const uint8_t* p, int64_t n, int64_t off) {
  while (n > 0) {
    ssize_t w = ::pwrite(fd, p, (size_t)std::min<int64_t>(n, 1ll << 30), off);
    if (w < 0) {
      if (errno == EINTR) continue;
      return false;
    }
    p += w;
    n -= w;
    off += w;
  }
  return true;
}
static bool read_all(int fd, uint8_t* p, int64_t n, int64_t off) {
  while (n > 0) {
    ssize_t r = ::pread(fd, p, (size_t)std::min<int64_t>(n, 1ll << 30), off);
    if (r < 0) {
      if (errno == EINTR) continue;
      return false;
    }
    if (r == 0) return false;  // short file
    p += r;
    n -= r;
    off += r;
  }
  return true;
}

// One file's payload through the page cache.  With parts > 1 the byte range is split over short-lived helper threads
// (pread with explicit offsets is thread-safe on one descriptor): a lone multi-MiB load finishes sooner on tmpfs.
// Only reads are split — writes to ONE file serialise on the inode lock (measured: no gain) — and only when no other
// task is queued, so the throughput regime keeps one I/O thread per worker.
static bool file_rw(int fd, uint8_t* p, int64_t n, int64_t off, bool is_write, int parts) {
  if (parts <= 1 || n < (8ll << 20)) return is_write ? write_all(fd, p, n, off) : read_all(fd, p, n, off);
  const int64_t chunk = ((n + parts - 1) / parts + 4095) & ~4095ll;
  std::atomic<bool> ok{true};
  std::vector<std::thread> th;
  for (int k = 0; k < parts; ++k) {
    const int64_t lo = (int64_t)k * chunk, len = std::min(chunk, n - lo);
    if (len <= 0) break;
    th.emplace_back([=, &ok] {
      if (!(is_write ? write_all(fd, p + lo, len, off + lo) : read_all(fd, p + lo, len, off + lo))) ok = false;
    });
  }
  for (auto& t : th) t.join();
  return ok.load();
}

// A lone store has nothing to overlap with, so its one file should not be written by one thread: pwrite() calls on ONE
// file serialise on the inode lock, but page faults on a shared mapping do not — map the (already sized) file and let a
// few short-lived threads copy disjoint ranges into the page cache.  Used only when nothing else is queued (latency
// regime) or when KVB_FILE_WRITE=mmap forces it for A/B; the throughput regime keeps one pwrite per worker.
static bool mmap_write(int fd, const uint8_t* p, int64_t n, int64_t off, int64_t file_bytes, int parts) {
  void* m = ::mmap(nullptr, (size_t)file_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  if (m == MAP_FAILED) return false;
  uint8_t* dst = static_cast<uint8_t*>(m) + off;
  if (parts <= 1) {
    std::memcpy(dst, p, (size_t)n);
  } else {
    const int64_t chunk = ((n + parts - 1) / parts + 4095) & ~4095ll;
    std::vector<std::thread> th;
    for (int k = 0; k < parts; ++k) {
      const int64_t lo = (int64_t)k * chunk, len = std::min(chunk, n - lo);
      if (len <= 0) break;
      th.emplace_back([=] { std::memcpy(dst + lo, p + lo, (size_t)len); });
    }
    for (auto& t : th) t.join();
  }
  return ::munmap(m, (size_t)file_bytes) == 0;
}
static int lone_io_parts() {  // helper threads of a lone file job (KVB_FILE_LONE_PARTS, default 8)
  static const int parts = [] {
    const char* e = std::getenv("KVB_FILE_LONE_PARTS");
    const int v = e ? std::atoi(e) : 8;
    return v < 1 ? 1 : (v > 32 ? 32 : v);
  }();
  return parts;
}
static int file_write_mode() {  // 0 = auto (mmap only for lone stores), 1 = always pwrite, 2 = always mmap
  static const int mode = [] {
    const char* e = std::getenv("KVB_FILE_WRITE");
    if (!e) return 0;
    return std::strcmp(e, "pwrite") == 0 ? 1 : (std::strcmp(e, "mmap") == 0 ? 2 : 0);
  }();
  return mode;
}

// ---------------------------------------------------------------------------------- cuFile (GDS tier)
// libcufile is resolved with dlopen so that libkvb.so has no hard dependency on it; the driver is opened once per
// process and left open.  Without the nvidia-fs kernel module cuFile runs in its compatibility mode (POSIX I/O through
// its own bounce buffers) — same calls, same file bytes.
struct CuFile {
  bool ok = false;
  bool stalled = false;  // cuFileDriverOpen did not return in kOpenWait: cuFile is never called again in this process
  CUfileError_t (*DriverOpen)() = nullptr;
  CUfileError_t (*HandleRegister)(CUfileHandle_t*, CUfileDescr_t*) = nullptr;
  void (*HandleDeregister)(CUfileHandle_t) = nullptr;
  CUfileError_t (*BufRegister)(const void*, size_t, int) = nullptr;
  CUfileError_t (*BufDeregister)(const void*) = nullptr;
  ssize_t (*Read)(CUfileHandle_t, void*, size_t, off_t, off_t) = nullptr;
  ssize_t (*Write)(CUfileHandle_t, const void*, size_t, off_t, off_t) = nullptr;
  std::string why;

  static CuFile& get() {
    static CuFile c;
    static std::once_flag once;
    std::call_once(once, [] { c.load(); });
    return c;
  }

 private:
  void load() {
    void* lib = nullptr;
    for (const char* name : {"libcufile.so.0", "libcufile.so", "/usr/local/cuda/lib64/libcufile.so.0"}) {
      lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (lib) break;
    }
    if (!lib) {
      why = "libcufile not found";
      return;
    }
    auto sym = [&](const char* n) { return dlsym(lib, n); };
    DriverOpen = reinterpret_cast<decltype(DriverOpen)>(sym("cuFileDriverOpen"));
    HandleRegister = reinterpret_cast<decltype(HandleRegister)>(sym("cuFileHandleRegister"));
    HandleDeregister = reinterpret_cast<decltype(HandleDeregister)>(sym("cuFileHandleDeregister"));
    BufRegister = reinterpret_cast<decltype(BufRegister)>(sym("cuFileBufRegister"));
    BufDeregister = reinterpret_cast<decltype(BufDeregister)>(sym("cuFileBufDeregister"));
    Read = reinterpret_cast<decltype(Read)>(sym("cuFileRead"));
    Write = reinterpret_cast<decltype(Write)>(sym("cuFileWrite"));
    if (!DriverOpen || !HandleRegister || !HandleDeregister || !Read || !Write) {
      why = "libcufile lacks a required symbol";
      return;
    }
    // Where nvidia-fs is absent the driver open can log that it runs in compatibility mode and then not return at all
    // (an H100 host: no answer within 400 s).  It runs on a helper thread; one that has not answered in 15 s is left
    // behind, detached, and the engine treats the driver as stalled (DESIGN.md section 4).
    constexpr auto kOpenWait = std::chrono::seconds(15);
    auto done = std::make_shared<std::promise<CUfileError_t>>();
    std::future<CUfileError_t> answer = done->get_future();
    std::thread([done, open = DriverOpen] { done->set_value(open()); }).detach();
    if (answer.wait_for(kOpenWait) != std::future_status::ready) {
      why = "cuFileDriverOpen did not return within 15 s";
      stalled = true;
      return;
    }
    const CUfileError_t st = answer.get();
    if (st.err != CU_FILE_SUCCESS) {
      why = "cuFileDriverOpen failed (" + std::to_string((int)st.err) + ")";
      return;
    }
    ok = true;
  }
};

}  // namespace kvb

using namespace kvb;

// ---------------------------------------------------------------------------------- engine object
struct kvb_engine {
  kvb_pool* pool = nullptr;
  kvb_engine_opts_t opts{};
  int device = 0;
  int64_t block_bytes = 0;
  int64_t blocks_per_chunk = 0;
  int64_t file_bytes = 0;  // on-disk size of every file

  struct Worker {
    std::thread th;
    bool high_first = false;
    bool remote_cpu = false;  // file tier: this worker's page-cache copies run on another NUMA node's CPUs
    cudaStream_t stream = nullptr;
    uint8_t* d_packed = nullptr;
    uint8_t* h_stage = nullptr;  // file tier only
    bool packed_registered = false;  // d_packed registered with cuFile
    int64_t* d_ids = nullptr;
    int64_t* h_ids = nullptr;
    bool ready = false;
  };
  std::vector<std::unique_ptr<Worker>> workers;
  // every worker allocates its stream / staging when its thread starts; kvb_engine_create waits for all of them, so an
  // allocation failure is a constructor error and never a silently failing load later
  std::mutex init_mu;
  std::condition_variable init_cv;
  int init_done = 0;
  bool init_failed = false;
  std::string init_error;

  std::mutex qmu;
  std::condition_variable qcv;
  std::deque<std::unique_ptr<ChunkTask>> q_high, q_normal;
  bool stop = false;
  std::atomic<int64_t> queued_store_files{0};

  std::mutex jmu;
  std::condition_variable jcv;
  std::map<int64_t, std::shared_ptr<JobState>> jobs;

  Arena arena;
  std::vector<int> local_cpus;   // CPUs of the GPU's NUMA node (empty: unknown, no binding)
  std::vector<int> remote_cpus;  // CPUs of the other nodes (file tier: every second worker runs there)
  std::atomic<uint64_t> avg_write_us{0};
  std::string tmp_suffix;

  // stats
  std::atomic<int64_t> bytes_stored{0}, bytes_loaded{0}, files_stored{0}, files_loaded{0}, files_skipped{0},
      writes_dropped{0}, load_failures{0}, kernels{0}, h2d{0}, d2h{0};

  void task_done(const std::shared_ptr<JobState>& job, bool ok) {
    if (!ok) job->ok = false;
    job->completed.fetch_add(1);
    std::lock_guard<std::mutex> lk(jmu);
    jcv.notify_all();
  }

  void update_write_duration(uint64_t us) {  // storage_offload.cpp:81-95
    if (us == 0) us = 1;
    uint64_t old_val = avg_write_us.load(), new_val;
    do {
      new_val = old_val == 0 ? us : (uint64_t)(old_val * (1.0 - kEmaAlpha) + us * kEmaAlpha);
    } while (!avg_write_us.compare_exchange_weak(old_val, new_val));
  }
  size_t dynamic_write_queue_limit() const {  // storage_offload.cpp:98-106
    uint64_t avg = avg_write_us.load();
    if (avg == 0 || opts.max_write_queued_seconds <= 0) return 0;
    return (size_t)(workers.size() * opts.max_write_queued_seconds / (avg / 1e6));
  }

  bool worker_init(Worker& w);
  void worker_release(Worker& w);
  void worker_loop(Worker* w);
  bool run_store(Worker& w, ChunkTask& t);
  // load outcome: only kSoft (a file that is missing / short / unreadable) may be reported as success, and only in the
  // file tier without strict_load_errors — that is the reference's swallow (storage_offload.cpp:378-383).  An arena
  // miss, a CUDA error or a failed kernel launch always fails the job: nothing was restored.
  enum LoadResult { kLoaded = 0, kSoft = 1, kHard = 2 };
  LoadResult run_load(Worker& w, ChunkTask& t);
  bool write_file(const FilePart& f, const uint8_t* payload, int parts);
  bool read_file(const FilePart& f, uint8_t* payload, int parts);
  // GDS tier: the reference's GDS file format (gds_file_io.cpp:238-418: n x block_bytes, head-aligned, tmp + rename),
  // ONE cuFile call per file between the file and the worker's packed HBM chunk
  // When cuFile cannot register a file (seen on overlay and tmpfs mounts: CU_FILE_INTERNAL_ERROR),
  // the same file format moves through the worker's pinned staging buffer instead; cufile_broken makes that sticky.
  bool gds_read = false, gds_write = false;
  std::atomic<bool> cufile_broken{false};
  std::atomic<int64_t> cufile_files{0}, gds_staged_files{0};
  bool gds_write_file(Worker& w, const FilePart& f, int64_t dev_off);
  bool gds_read_file(Worker& w, const FilePart& f, int64_t dev_off);
  int submit(int64_t job_id, int32_t n_files, const char* const* files, const int64_t* ids, const int64_t* off,
             void* caller_stream, bool is_store);
};

bool kvb_engine::worker_init(Worker& w) {
  if (cudaSetDevice(device) != cudaSuccess) return false;
  const size_t chunk = (size_t)(blocks_per_chunk * block_bytes);
  if (cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking) != cudaSuccess) return false;
  if (cudaMalloc(&w.d_packed, chunk) != cudaSuccess) return false;
  if (cudaMalloc(&w.d_ids, blocks_per_chunk * sizeof(int64_t)) != cudaSuccess) return false;
  if (cudaHostAlloc(&w.h_ids, blocks_per_chunk * sizeof(int64_t), cudaHostAllocDefault) != cudaSuccess) return false;
  // the pinned staging buffer stays on the GPU's node (the DMA side) whichever node this worker's CPU is on
  if (opts.tier == KVB_TIER_FILE &&
      host_alloc_near(device, reinterpret_cast<void**>(&w.h_stage), chunk, cudaHostAllocDefault) != cudaSuccess)
    return false;
  // optional: unregistered buffers go through cuFile's own bounce buffers
  if ((gds_read || gds_write) && CuFile::get().ok && CuFile::get().BufRegister)
    w.packed_registered = CuFile::get().BufRegister(w.d_packed, chunk, 0).err == CU_FILE_SUCCESS;
  w.ready = true;
  return true;
}

static int open_direct(const std::string& path, int flags, mode_t mode) {
  int fd = ::open(path.c_str(), flags | O_DIRECT, mode);  // gds_file_io.cpp:262,352 open with O_DIRECT
  if (fd < 0 && errno == EINVAL) fd = ::open(path.c_str(), flags, mode);  // file systems without O_DIRECT
  return fd;
}

bool kvb_engine::gds_write_file(Worker& w, const FilePart& f, int64_t dev_off) {
  CuFile& cf = CuFile::get();
  const std::string& target = f.path;
  size_t pos = target.find_last_of('/');
  if (pos != std::string::npos && !mkdirs(target.substr(0, pos))) return false;
  const std::string tmp = target + tmp_suffix + std::to_string((uintptr_t)(w.d_packed + dev_off) & 0xffffff);
  int fd = open_direct(tmp, O_RDWR | O_CREAT | O_TRUNC, 0644);  // O_RDWR: cuFile needs it even to write (:260-262)
  if (fd < 0) return false;
  const int64_t bytes = (int64_t)f.ids.size() * block_bytes;
  bool ok = false, via_cufile = false;
  if (!cufile_broken.load()) {
    CUfileDescr_t descr;
    std::memset(&descr, 0, sizeof(descr));
    descr.handle.fd = fd;
    descr.type = CU_FILE_HANDLE_TYPE_OPAQUE_FD;
    CUfileHandle_t h;
    if (cf.HandleRegister(&h, &descr).err == CU_FILE_SUCCESS) {
      via_cufile = ok = true;
      int64_t done = 0;
      while (ok && done < bytes) {  // one call in practice; the loop only covers short writes
        const ssize_t n = cf.Write(h, w.d_packed, (size_t)(bytes - done), (off_t)done, (off_t)(dev_off + done));
        if (n <= 0) ok = false;
        else done += n;
      }
      cf.HandleDeregister(h);
    } else {
      cufile_broken = true;
    }
  }
  if (!via_cufile) {  // same bytes through the pinned staging buffer (O_DIRECT wants aligned I/O: reopen buffered)
    ::close(fd);
    fd = ::open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
    ok = fd >= 0 &&
         cudaMemcpyAsync(w.h_stage + dev_off, w.d_packed + dev_off, (size_t)bytes, cudaMemcpyDeviceToHost, w.stream) ==
             cudaSuccess &&
         cudaStreamSynchronize(w.stream) == cudaSuccess && write_all(fd, w.h_stage + dev_off, bytes, 0);
    d2h += bytes;
    gds_staged_files++;
  } else {
    cufile_files++;
  }
  if (fd >= 0) ok = (::close(fd) == 0) && ok;
  if (ok && ::rename(tmp.c_str(), target.c_str()) != 0) ok = false;
  if (!ok) ::unlink(tmp.c_str());
  return ok;
}

bool kvb_engine::gds_read_file(Worker& w, const FilePart& f, int64_t dev_off) {
  CuFile& cf = CuFile::get();
  const int64_t bytes = (int64_t)f.ids.size() * block_bytes;  // the FIRST n blocks of the file (:386-414)
  if (!cufile_broken.load()) {
    int fd = open_direct(f.path, O_RDONLY, 0);
    if (fd < 0) return false;
    CUfileDescr_t descr;
    std::memset(&descr, 0, sizeof(descr));
    descr.handle.fd = fd;
    descr.type = CU_FILE_HANDLE_TYPE_OPAQUE_FD;
    CUfileHandle_t h;
    if (cf.HandleRegister(&h, &descr).err == CU_FILE_SUCCESS) {
      bool ok = true;
      int64_t done = 0;
      while (ok && done < bytes) {
        const ssize_t n = cf.Read(h, w.d_packed, (size_t)(bytes - done), (off_t)done, (off_t)(dev_off + done));
        if (n <= 0) ok = false;  // 0 = short file
        else done += n;
      }
      cf.HandleDeregister(h);
      ::close(fd);
      cufile_files++;
      return ok;
    }
    ::close(fd);
    cufile_broken = true;
  }
  int fd = ::open(f.path.c_str(), O_RDONLY);
  if (fd < 0) return false;
  bool ok = read_all(fd, w.h_stage + dev_off, bytes, 0);
  ::close(fd);
  if (ok)
    ok = cudaMemcpyAsync(w.d_packed + dev_off, w.h_stage + dev_off, (size_t)bytes, cudaMemcpyHostToDevice, w.stream) ==
         cudaSuccess;  // ordered before the scatter on the same stream
  h2d += bytes;
  gds_staged_files++;
  return ok;
}

// reference on-disk format, CPU path: full-size file, payload tail-aligned inside the bpf slots
bool kvb_engine::write_file(const FilePart& f, const uint8_t* payload, int parts) {
  const std::string& target = f.path;
  size_t pos = target.find_last_of('/');
  if (pos != std::string::npos && !mkdirs(target.substr(0, pos))) return false;
  std::string tmp = target + tmp_suffix + std::to_string((uintptr_t)payload & 0xffffff);
  int fd = ::open(tmp.c_str(), O_CREAT | O_TRUNC | O_RDWR, 0644);  // O_RDWR: the lone-store path maps the file
  if (fd < 0) return false;
  const int64_t n = (int64_t)f.ids.size();
  const int64_t off = ((int64_t)opts.gpu_blocks_per_file - n) * block_bytes;
  const int mode = file_write_mode();
  const bool use_mmap = mode == 2 || (mode == 0 && parts > 1 && n * block_bytes >= (8ll << 20));
  bool ok = ::ftruncate(fd, file_bytes) == 0 &&
            (use_mmap ? mmap_write(fd, payload, n * block_bytes, off, file_bytes, parts)
                      : file_rw(fd, const_cast<uint8_t*>(payload), n * block_bytes, off, true, 1));
  ok = (::close(fd) == 0) && ok;
  if (ok && ::rename(tmp.c_str(), target.c_str()) != 0) ok = false;
  if (!ok) ::unlink(tmp.c_str());
  return ok;
}

bool kvb_engine::read_file(const FilePart& f, uint8_t* payload, int parts) {
  int fd = ::open(f.path.c_str(), O_RDONLY);
  if (fd < 0) return false;
  const int64_t n = (int64_t)f.ids.size();
  const int64_t off = ((int64_t)opts.gpu_blocks_per_file - n) * block_bytes;
  bool ok = file_rw(fd, payload, n * block_bytes, off, false, parts);
  ::close(fd);
  return ok;
}

bool kvb_engine::run_store(Worker& w, ChunkTask& t) {
  // cancelled before start: nothing to do (storage_offload.cpp:294-297)
  if (t.job->cancelled.load()) return true;
  // drop files that already exist (storage_offload.cpp:299-304) and, in the arena tier, reserve their space
  struct Dest {
    const FilePart* f;
    uint8_t* host;  // arena destination (arena tier) or offset into h_stage (file tier)
    int64_t first_block;
  };
  std::vector<Dest> dests;
  int64_t n = 0;
  for (auto& f : t.files) {
    const int64_t nb = (int64_t)f.ids.size();
    if (nb == 0) continue;
    if (opts.tier == KVB_TIER_HOST_ARENA) {
      bool existed = false;
      uint8_t* dst = arena.reserve(f.path, nb, nb * block_bytes, &existed);
      if (existed) {
        files_skipped++;
        continue;
      }
      if (!dst) {
        set_error("host arena full storing %s", f.path.c_str());
        for (auto& d : dests) arena.commit(d.f->path, false);
        return false;
      }
      dests.push_back({&f, dst, n});
    } else {
      if (file_exists(f.path)) {
        touch_atime(f.path);
        files_skipped++;
        continue;
      }
      dests.push_back({&f, w.h_stage + n * block_bytes, n});
    }
    std::memcpy(w.h_ids + n, f.ids.data(), nb * sizeof(int64_t));
    n += nb;
  }
  if (n == 0) return true;
  auto t0 = std::chrono::steady_clock::now();
  bool ok = true;
  cudaError_t e = cudaSuccess;
  const bool gds_w = opts.tier == KVB_TIER_FILE && gds_write;  // files leave from the packed HBM chunk, no host leg
  const bool direct = opts.direct_host_io && !gds_w;
  if (t.ready) e = cudaStreamWaitEvent(w.stream, t.ready, 0);  // KV produced on the caller's stream
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(w.d_ids, w.h_ids, n * sizeof(int64_t), cudaMemcpyHostToDevice, w.stream);
  if (e == cudaSuccess && !direct) {
    ok = launch_gather(pool, w.d_ids, n, w.d_packed, w.stream, opts.copy_flags) == KVB_OK;
    kernels++;
  }
  if (e == cudaSuccess && ok && !gds_w) {
    // merge destinations that are contiguous on the host into one run
    size_t i = 0;
    while (i < dests.size() && e == cudaSuccess && ok) {
      size_t j = i;
      int64_t bytes = (int64_t)dests[i].f->ids.size() * block_bytes;
      while (j + 1 < dests.size() && dests[j + 1].host == dests[i].host + bytes) {
        ++j;
        bytes += (int64_t)dests[j].f->ids.size() * block_bytes;
      }
      if (direct) {
        // fused gather + D2H: the kernel's bulk stores land in the pinned host run (UVA), no HBM staging, no memcpy
        ok = launch_gather(pool, w.d_ids + dests[i].first_block, bytes / block_bytes, dests[i].host, w.stream,
                           opts.copy_flags) == KVB_OK;
        kernels++;
      } else {
        e = cudaMemcpyAsync(dests[i].host, w.d_packed + dests[i].first_block * block_bytes, (size_t)bytes,
                            cudaMemcpyDeviceToHost, w.stream);
      }
      d2h += bytes;
      i = j + 1;
    }
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(w.stream);
  if (e != cudaSuccess) {
    set_error("store chunk: %s", cudaGetErrorString(e));
    cudaGetLastError();
    ok = false;
  }
  if (opts.tier == KVB_TIER_HOST_ARENA) {
    for (auto& d : dests) arena.commit(d.f->path, ok);
  } else if (ok) {
    for (auto& d : dests) {
      if (t.job->cancelled.load()) break;  // in-flight cancelled job skips the file write (storage_offload.cpp:228-229)
      const bool wrote = gds_w ? gds_write_file(w, *d.f, d.first_block * block_bytes)
                               : write_file(*d.f, d.host, t.io_parts);
      if (!wrote) {
        set_error("store: writing %s failed: %s", d.f->path.c_str(), std::strerror(errno));
        ok = false;
      }
    }
  }
  if (ok) {
    bytes_stored += n * block_bytes;
    files_stored += (int64_t)dests.size();
  }
  auto us = std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count();
  if (!dests.empty()) update_write_duration((uint64_t)(us / (int64_t)dests.size()));
  return ok;
}

kvb_engine::LoadResult kvb_engine::run_load(Worker& w, ChunkTask& t) {
  struct Src {
    const FilePart* f;
    const uint8_t* host;
    int64_t first_block;
  };
  std::vector<Src> srcs;
  int64_t n = 0;
  bool soft = false, hard = false;
  const bool gds_r = opts.tier == KVB_TIER_FILE && gds_read;  // files land in the packed HBM chunk, no host leg
  const bool direct = opts.direct_host_io && !gds_r;
  for (auto& f : t.files) {
    const int64_t nb = (int64_t)f.ids.size();
    if (nb == 0) continue;
    if (opts.tier == KVB_TIER_HOST_ARENA) {
      const uint8_t* src = arena.pin_read(f.path, nb, block_bytes);
      if (!src) {
        // the arena's own LRU may have dropped the entry between the scheduler's lookup and this load: the pages were
        // NOT restored, so the job must say so (the reference's swallow covers a vanished FILE, not this)
        set_error("load: %s not in host arena (or holds fewer than %lld blocks)", f.path.c_str(), (long long)nb);
        hard = true;
        continue;
      }
      srcs.push_back({&f, src, n});
    } else {
      uint8_t* dst = w.h_stage + n * block_bytes;
      if (gds_r ? !gds_read_file(w, f, n * block_bytes) : !read_file(f, dst, t.io_parts)) {
        // the reference runs one task per file: a missing file fails alone, the others still load
        set_error("load: reading %s failed", f.path.c_str());
        soft = true;
        continue;
      }
      srcs.push_back({&f, dst, n});
    }
    std::memcpy(w.h_ids + n, f.ids.data(), nb * sizeof(int64_t));
    n += nb;
  }
  cudaError_t e = cudaSuccess;
  if (n > 0) {
    if (t.ready) e = cudaStreamWaitEvent(w.stream, t.ready, 0);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(w.d_ids, w.h_ids, n * sizeof(int64_t), cudaMemcpyHostToDevice, w.stream);
    size_t i = gds_r ? srcs.size() : 0;  // GDS: the bytes are in d_packed already
    bool moved = true;
    while (i < srcs.size() && e == cudaSuccess) {
      size_t j = i;
      int64_t bytes = (int64_t)srcs[i].f->ids.size() * block_bytes;
      while (j + 1 < srcs.size() && srcs[j + 1].host == srcs[i].host + bytes) {
        ++j;
        bytes += (int64_t)srcs[j].f->ids.size() * block_bytes;
      }
      if (direct) {
        // fused H2D + scatter: the kernel's bulk loads read the pinned host run directly
        if (launch_scatter(pool, w.d_ids + srcs[i].first_block, bytes / block_bytes, srcs[i].host, w.stream,
                           opts.copy_flags) != KVB_OK)
          moved = false;
        kernels++;
      } else {
        e = cudaMemcpyAsync(w.d_packed + srcs[i].first_block * block_bytes, srcs[i].host, (size_t)bytes,
                            cudaMemcpyHostToDevice, w.stream);
      }
      h2d += bytes;
      i = j + 1;
    }
    if (e == cudaSuccess && !direct) {
      moved = launch_scatter(pool, w.d_ids, n, w.d_packed, w.stream, opts.copy_flags) == KVB_OK && moved;
      kernels++;
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(w.stream);
    if (e != cudaSuccess) {
      set_error("load chunk: %s", cudaGetErrorString(e));
      cudaGetLastError();
      moved = false;
    }
    if (moved) {  // the files that were found did load, whatever happened to the missing ones
      bytes_loaded += n * block_bytes;
      files_loaded += (int64_t)srcs.size();
    } else {
      hard = true;
    }
  }
  if (opts.tier == KVB_TIER_HOST_ARENA)
    for (auto& s : srcs) arena.unpin(s.f->path);
  if (soft || hard) load_failures++;
  return hard ? kHard : (soft ? kSoft : kLoaded);
}

void kvb_engine::worker_loop(Worker* w) {
  bind_this_thread(w->remote_cpu && !remote_cpus.empty() ? remote_cpus : local_cpus);
  const bool inited = worker_init(*w);
  {
    std::lock_guard<std::mutex> lk(init_mu);
    ++init_done;
    if (!inited) {
      init_failed = true;
      init_error = "engine worker: CUDA resource allocation failed (stream / packed HBM chunk / pinned staging)";
    }
  }
  init_cv.notify_all();
  if (!inited) {  // kvb_engine_create reports the failure and tears the engine down; this thread takes no task
    worker_release(*w);
    return;
  }
  for (;;) {
    std::unique_ptr<ChunkTask> task;
    {
      std::unique_lock<std::mutex> lk(qmu);
      qcv.wait(lk, [&] { return stop || !q_high.empty() || !q_normal.empty(); });
      if (stop && q_high.empty() && q_normal.empty()) break;
      auto& first = w->high_first ? q_high : q_normal;
      auto& second = w->high_first ? q_normal : q_high;
      auto& q = !first.empty() ? first : second;
      task = std::move(q.front());
      q.pop_front();
      if (q_high.empty() && q_normal.empty() && opts.tier == KVB_TIER_FILE) task->io_parts = lone_io_parts();
    }
    bool ok = false;
    try {
      if (task->is_store) {
        ok = run_store(*w, *task);
      } else {
        const LoadResult r = run_load(*w, *task);
        // reference parity (storage_offload.cpp:378-383): a FILE that could not be read is logged and the job still
        // reports success — unless strict_load_errors; everything else that kept the pages from being restored fails
        ok = r == kLoaded || (r == kSoft && !opts.strict_load_errors);
        if (r != kLoaded)
          fprintf(stderr, "[kvb][ERROR] load chunk of job %lld failed%s: %s\n", (long long)task->job->id,
                  ok ? " (reported as success, reference parity)" : "", get_error());
      }
    } catch (...) {
      set_error("exception in engine worker");
      ok = false;
    }
    if (!ok && task->is_store)  // reference logs failures at ERROR level (storage_offload.cpp:330-346)
      fprintf(stderr, "[kvb][ERROR] store chunk of job %lld failed: %s\n", (long long)task->job->id, get_error());
    if (task->is_store) queued_store_files -= (int64_t)task->files.size();
    task_done(task->job, ok);
  }
  worker_release(*w);
}

void kvb_engine::worker_release(Worker& w) {
  cudaSetDevice(device);
  if (w.stream) cudaStreamSynchronize(w.stream);
  if (w.packed_registered && CuFile::get().BufDeregister) CuFile::get().BufDeregister(w.d_packed);
  w.packed_registered = false;
  if (w.d_packed) cudaFree(w.d_packed);
  if (w.d_ids) cudaFree(w.d_ids);
  if (w.h_ids) cudaFreeHost(w.h_ids);
  if (w.h_stage) cudaFreeHost(w.h_stage);
  if (w.stream) cudaStreamDestroy(w.stream);
  w.d_packed = w.h_stage = nullptr;
  w.d_ids = w.h_ids = nullptr;
  w.stream = nullptr;
  cudaGetLastError();
}

int kvb_engine::submit(int64_t job_id, int32_t n_files, const char* const* files, const int64_t* ids,
                       const int64_t* off, void* caller_stream, bool is_store) {
  KVB_REQUIRE(n_files >= 0, "negative file count");
  KVB_REQUIRE(n_files == 0 || (files && ids && off), "NULL argument");
  for (int32_t i = 0; i < n_files; ++i) {
    const int64_t nb = off[i + 1] - off[i];
    KVB_REQUIRE(nb >= 0 && nb <= opts.gpu_blocks_per_file, "file %d holds %lld blocks, gpu_blocks_per_file is %d", i,
                (long long)nb, opts.gpu_blocks_per_file);
    KVB_REQUIRE(files[i] != nullptr, "file %d is NULL", i);
    int rc = validate_ids(pool, ids + off[i], nb);
    if (rc) return rc;
  }
  auto job = std::make_shared<JobState>();
  job->id = job_id;

  // order after the caller's stream (storage_offload.cpp:259-265)
  cudaEvent_t ev = nullptr;
  std::shared_ptr<void> ev_owner;
  {
    DeviceGuard g(device);
    KVB_CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    ev_owner = std::shared_ptr<void>(ev, [](void* e) { cudaEventDestroy(static_cast<cudaEvent_t>(e)); });
    KVB_CUDA_TRY(cudaEventRecord(ev, static_cast<cudaStream_t>(caller_stream)));
  }

  std::vector<std::unique_ptr<ChunkTask>> tasks;
  std::unique_ptr<ChunkTask> cur;
  int dropped = 0;
  for (int32_t i = 0; i < n_files; ++i) {
    const int64_t nb = off[i + 1] - off[i];
    if (is_store) {
      // dynamic write-queue limit (storage_offload.cpp:272-288): dropped files count as done + success
      size_t limit = dynamic_write_queue_limit();
      if (limit > 0 && (size_t)queued_store_files.load() >= limit) {
        ++dropped;
        writes_dropped++;
        continue;
      }
      queued_store_files++;
    }
    if (!cur || cur->n_blocks + nb > blocks_per_chunk) {
      if (cur) tasks.push_back(std::move(cur));
      cur.reset(new ChunkTask());
      cur->job = job;
      cur->is_store = is_store;
      cur->ready = ev;
      cur->ready_owner = ev_owner;
    }
    FilePart fp;
    fp.path = files[i];
    fp.ids.assign(ids + off[i], ids + off[i + 1]);
    cur->files.push_back(std::move(fp));
    cur->n_blocks += nb;
  }
  if (cur) tasks.push_back(std::move(cur));
  job->total = (int)tasks.size();
  {
    std::lock_guard<std::mutex> lk(jmu);
    jobs[job_id] = job;
  }
  {
    std::lock_guard<std::mutex> lk(qmu);
    for (auto& t : tasks) (is_store ? q_normal : q_high).push_back(std::move(t));
  }
  qcv.notify_all();
  (void)dropped;
  return KVB_OK;
}

extern "C" {

void kvb_engine_default_opts(kvb_engine_opts_t* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  o->io_threads = 4;
  o->gpu_blocks_per_file = 16;
  o->read_preferring_workers = 3;
  o->max_write_queued_seconds = 10.0f;  // worker.py:61 DEFAULT_MAX_WRITE_QUEUED_SECONDS
  o->tier = KVB_TIER_FILE;
  o->copy_flags = KVB_COPY_DEFAULT;
  o->host_arena_bytes = 0;
  o->chunk_bytes = 64ll << 20;
  o->direct_host_io = 0;
  o->strict_load_errors = 0;
  o->gds_mode = KVB_GDS_DISABLED;
  o->arena_alloc_mode = KVB_HOST_ALLOC_DEFAULT;
}

int kvb_engine_create(kvb_pool_t* pool, const kvb_engine_opts_t* opts, kvb_engine_t** out) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(out != nullptr, "out is NULL");
    *out = nullptr;
    KVB_REQUIRE(pool != nullptr && opts != nullptr, "NULL argument");
    KVB_REQUIRE(opts->gpu_blocks_per_file > 0, "gpu_blocks_per_file must be > 0");  // tensor_copier.cu:35-36
    KVB_REQUIRE(opts->io_threads > 0 && opts->io_threads <= 256, "io_threads out of range");
    KVB_REQUIRE(opts->tier == KVB_TIER_FILE || opts->tier == KVB_TIER_HOST_ARENA, "unknown tier %d", opts->tier);
    std::unique_ptr<kvb_engine> e(new kvb_engine());
    e->pool = pool;
    e->opts = *opts;
    e->device = pool->device;
    e->block_bytes = pool->frag_bytes * pool->num_tensors;
    int64_t chunk = opts->chunk_bytes > 0 ? opts->chunk_bytes : (64ll << 20);
    int64_t bpc = chunk / e->block_bytes;
    if (bpc < opts->gpu_blocks_per_file) bpc = opts->gpu_blocks_per_file;  // a chunk always holds whole files
    e->blocks_per_chunk = bpc;
    e->file_bytes = std::max<int64_t>((int64_t)opts->gpu_blocks_per_file * e->block_bytes, kMinFileBytes);
    e->tmp_suffix = "_" + std::to_string((long long)::getpid()) + "_" +
                    std::to_string((unsigned long long)(uintptr_t)e.get() & 0xffffff) + ".tmp";
    DeviceGuard g(e->device);
    if (!g.ok) {
      set_error("cannot select CUDA device %d", e->device);
      return KVB_ERR_CUDA;
    }
    e->local_cpus = gpu_local_cpus(e->device);
    // KVB_FILE_SPREAD=1 (A/B, off by default): every second file-tier worker runs on the OTHER NUMA node's CPUs, so that its
    // page-cache pages land there while its pinned staging buffer stays next to the GPU.  On tmpfs the limit is the
    // kernel's page-cache insertion path, which more threads or more nodes do not widen (tools/probe_file_tier.py).
    const char* spread = std::getenv("KVB_FILE_SPREAD");
    if (opts->tier == KVB_TIER_FILE && spread && spread[0] == '1') e->remote_cpus = gpu_remote_cpus(e->device);
    if (opts->tier == KVB_TIER_FILE && (opts->gds_mode & (KVB_GDS_READ | KVB_GDS_WRITE))) {
      cudaFree(nullptr);  // cuFileDriverOpen wants a CUDA context
      if (CuFile::get().ok || CuFile::get().stalled) {
        e->gds_read = (opts->gds_mode & KVB_GDS_READ) != 0;
        e->gds_write = (opts->gds_mode & KVB_GDS_WRITE) != 0;
        if (!CuFile::get().ok) {  // a stalled driver: the GDS file format moves through the pinned staging buffers
          e->cufile_broken = true;
          fprintf(stderr, "[kvb][WARN] %s: GDS-format files go through pinned staging\n", CuFile::get().why.c_str());
        }
      } else {  // storage_offload.cpp:129-134: warn and use CPU staging for both directions
        fprintf(stderr, "[kvb][WARN] GDS requested but unavailable (%s): falling back to CPU staging\n",
                CuFile::get().why.c_str());
      }
    }
    if (opts->tier == KVB_TIER_HOST_ARENA) {
      KVB_REQUIRE(opts->host_arena_bytes >= e->block_bytes, "host_arena_bytes too small");
      KVB_REQUIRE(opts->arena_alloc_mode == KVB_HOST_ALLOC_DEFAULT || opts->arena_alloc_mode == KVB_HOST_ALLOC_THP,
                  "unknown arena_alloc_mode %d", opts->arena_alloc_mode);
      int rc = e->arena.init(e->device, opts->host_arena_bytes, opts->arena_alloc_mode);  // pinned, on the GPU-local node
      if (rc) return rc;
    }
    const int n_high = std::min(std::max(opts->read_preferring_workers, 0), opts->io_threads);
    for (int i = 0; i < opts->io_threads; ++i) {
      auto w = std::make_unique<kvb_engine::Worker>();
      w->high_first = i < n_high;  // thread_pool.cpp:52-57
      w->remote_cpu = (i & 1) != 0;
      e->workers.push_back(std::move(w));
    }
    for (auto& w : e->workers) w->th = std::thread([eng = e.get(), wp = w.get()] { eng->worker_loop(wp); });
    {  // worker resources (io_threads x chunk_bytes of HBM, the same again pinned in the file tier) are part of
       // construction: if they do not fit, say so HERE, not through loads that quietly restore nothing
      std::unique_lock<std::mutex> lk(e->init_mu);
      e->init_cv.wait(lk, [&] { return e->init_done == (int)e->workers.size(); });
      if (e->init_failed) {
        const std::string why = e->init_error;
        const long long per_worker = (long long)(e->blocks_per_chunk * e->block_bytes);
        lk.unlock();
        kvb_engine_destroy(e.release());
        set_error("%s: %d workers x %lld bytes per worker do not fit; lower io_threads or chunk_bytes", why.c_str(),
                  opts->io_threads, per_worker);
        return KVB_ERR_NOMEM;
      }
    }
    *out = e.release();
    return KVB_OK;
  });
}

void kvb_engine_destroy(kvb_engine_t* e) {
  if (!e) return;
  {
    std::lock_guard<std::mutex> lk(e->qmu);
    e->stop = true;
  }
  e->qcv.notify_all();
  for (auto& w : e->workers)
    if (w->th.joinable()) w->th.join();
  e->arena.destroy();
  delete e;
}

int kvb_engine_store(kvb_engine_t* e, int64_t job_id, int32_t n_files, const char* const* files,
                     const int64_t* block_ids, const int64_t* file_off, void* caller_stream) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(e != nullptr, "engine is NULL");
    return e->submit(job_id, n_files, files, block_ids, file_off, caller_stream, true);
  });
}
int kvb_engine_load(kvb_engine_t* e, int64_t job_id, int32_t n_files, const char* const* files,
                    const int64_t* block_ids, const int64_t* file_off, void* caller_stream) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(e != nullptr, "engine is NULL");
    return e->submit(job_id, n_files, files, block_ids, file_off, caller_stream, false);
  });
}

int kvb_engine_poll(kvb_engine_t* e, int64_t* job_ids, int32_t* ok, int32_t cap) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(e != nullptr, "engine is NULL");
    KVB_REQUIRE(cap >= 0 && (cap == 0 || (job_ids && ok)), "bad output buffers");
    std::lock_guard<std::mutex> lk(e->jmu);
    int n = 0;
    for (auto it = e->jobs.begin(); it != e->jobs.end() && n < cap;) {
      if (it->second->completed.load() == it->second->total) {  // storage_offload.cpp:196-201
        job_ids[n] = it->first;
        ok[n] = it->second->ok.load() ? 1 : 0;
        ++n;
        it = e->jobs.erase(it);
      } else {
        ++it;
      }
    }
    return n;
  });
}

int kvb_engine_wait(kvb_engine_t* e, int64_t job_id) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(e != nullptr, "engine is NULL");
    std::shared_ptr<JobState> job;
    {
      std::lock_guard<std::mutex> lk(e->jmu);
      auto it = e->jobs.find(job_id);
      if (it == e->jobs.end()) return KVB_OK;  // storage_offload.cpp:221: unknown job returns
      job = it->second;
    }
    job->cancelled = true;  // queued tasks bail early (storage_offload.cpp:226-229)
    std::unique_lock<std::mutex> lk(e->jmu);
    e->jcv.wait(lk, [&] { return job->completed.load() == job->total; });
    return KVB_OK;
  });
}

int kvb_engine_exists(kvb_engine_t* e, const char* file) {
  return kvb::guarded([&]() -> int {
    if (!e || !file) return 0;
    if (e->opts.tier == KVB_TIER_HOST_ARENA) return e->arena.exists(file) ? 1 : 0;
    return file_exists(file) ? 1 : 0;
  });
}

int kvb_engine_lookup_prefix(kvb_engine_t* e, int32_t n_files, const char* const* files, int32_t* out_hits) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(e && out_hits, "NULL argument");
    KVB_REQUIRE(n_files >= 0 && (n_files == 0 || files), "bad file list");
    *out_hits = 0;
    if (e->opts.tier == KVB_TIER_HOST_ARENA) {
      *out_hits = e->arena.count_prefix(files, n_files);
      return KVB_OK;
    }
    int32_t hits = 0;
    for (; hits < n_files; ++hits) {  // manager.py:49-53: stop at the first block that is not offloaded
      if (!files[hits]) break;
      struct statx sx;
      if (::statx(AT_FDCWD, files[hits], AT_STATX_DONT_SYNC, 0, &sx) != 0) break;  // existence only: no attributes asked
    }
    *out_hits = hits;
    return KVB_OK;
  });
}

int kvb_engine_lookup_prefix_hashes(kvb_engine_t* e, const char* base_path, const uint64_t* hashes, int32_t n,
                                    int32_t* out_hits) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(e && out_hits && base_path, "NULL argument");
    KVB_REQUIRE(n >= 0 && (n == 0 || hashes), "bad hash list");
    *out_hits = 0;
    // FileMapper.get_file_name (file_mapper.py:69-87): <base>/<hhh>/<hh>/<016x>.bin, built here so that the caller
    // hands over 8 bytes per block instead of a path string
    std::string path(base_path);
    const size_t base_len = path.size();
    path.resize(base_len + 1 + 3 + 1 + 2 + 1 + 16 + 4);
    static const char* hex = "0123456789abcdef";
    auto fill = [&](uint64_t h) {
      char name[16];
      for (int i = 0; i < 16; ++i) name[i] = hex[(h >> (60 - 4 * i)) & 0xf];
      char* q = &path[base_len];
      *q++ = '/';
      std::memcpy(q, name, 3);
      q += 3;
      *q++ = '/';
      std::memcpy(q, name + 3, 2);
      q += 2;
      *q++ = '/';
      std::memcpy(q, name, 16);
      q += 16;
      std::memcpy(q, ".bin", 4);
    };
    int32_t hits = 0;
    if (e->opts.tier == KVB_TIER_HOST_ARENA) {
      std::lock_guard<std::mutex> lk(e->arena.mu);
      for (; hits < n; ++hits) {
        fill(hashes[hits]);
        auto it = e->arena.entries.find(path);
        if (it == e->arena.entries.end() || !it->second.valid) break;
      }
    } else {
      for (; hits < n; ++hits) {  // manager.py:49-53: stop at the first block that is not offloaded
        fill(hashes[hits]);
        struct statx sx;
        if (::statx(AT_FDCWD, path.c_str(), AT_STATX_DONT_SYNC, 0, &sx) != 0) break;
      }
    }
    *out_hits = hits;
    return KVB_OK;
  });
}

int kvb_engine_arena_clear(kvb_engine_t* e) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(e != nullptr, "engine is NULL");
    if (e->opts.tier == KVB_TIER_HOST_ARENA) e->arena.clear();
    return KVB_OK;
  });
}

int kvb_engine_get_stats(kvb_engine_t* e, kvb_engine_stats_t* s) {
  return kvb::guarded([&]() -> int {
    KVB_REQUIRE(e && s, "NULL argument");
    s->bytes_stored = e->bytes_stored;
    s->bytes_loaded = e->bytes_loaded;
    s->files_stored = e->files_stored;
    s->files_loaded = e->files_loaded;
    s->files_skipped_existing = e->files_skipped;
    s->writes_dropped = e->writes_dropped;
    s->load_failures = e->load_failures;
    s->kernels_launched = e->kernels;
    s->h2d_bytes = e->h2d;
    s->d2h_bytes = e->d2h;
    return KVB_OK;
  });
}

}  // extern "C"
