// CUDA runtime side of backend.h: allocation, streams, error handling, launch
// accounting and optional per-kernel CUDA-event timing (product build only).
#include <cuda_runtime.h>

#include <atomic>
#include <map>
#include <string.h>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "backend.h"
#include "pipeline.h"
#include "tma.cuh"

namespace gb200 {

void cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  char buf[512];
  snprintf(buf, sizeof(buf), "CUDA error %d (%s) at %s:%d: %s", static_cast<int>(e), cudaGetErrorString(e),
           file, line, what);
  throw std::runtime_error(buf);
}

// Caching device allocator.  cudaMalloc takes a process-wide lock and cudaFree
// synchronises the whole device; with one image context per host thread (dozens of
// planes each, created and destroyed per image) that serialises the threads and
// stalls every stream.  Freed blocks are kept in per-(device, size) free lists and
// handed out again; callers only free memory whose stream work has completed
// (contexts synchronise their stream before releasing anything).
namespace {
struct DevCache {
  std::mutex mu;
  std::map<std::pair<int, size_t>, std::vector<void*> > free_list;
  std::map<void*, std::pair<int, size_t> > live;
};
DevCache& dev_cache() {
  static DevCache c;
  return c;
}
}  // namespace

void* dev_alloc(size_t bytes) {
  const size_t size = ((bytes ? bytes : 1) + 511) & ~static_cast<size_t>(511);
  int dev = 0;
  GB_CUDA(cudaGetDevice(&dev));
  DevCache& c = dev_cache();
  {
    std::lock_guard<std::mutex> lock(c.mu);
    std::vector<void*>& fl = c.free_list[std::make_pair(dev, size)];
    if (!fl.empty()) {
      void* p = fl.back();
      fl.pop_back();
      c.live[p] = std::make_pair(dev, size);
      return p;
    }
  }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, size);
  if (e != cudaSuccess) {
    // out of memory: drop the cache and retry once
    cudaGetLastError();
    {
      std::lock_guard<std::mutex> lock(c.mu);
      for (std::map<std::pair<int, size_t>, std::vector<void*> >::iterator it = c.free_list.begin();
           it != c.free_list.end(); ++it) {
        if (it->first.first != dev) continue;
        for (size_t i = 0; i < it->second.size(); ++i) cudaFree(it->second[i]);
        it->second.clear();
      }
    }
    GB_CUDA(cudaMalloc(&p, size));
  }
  std::lock_guard<std::mutex> lock(c.mu);
  c.live[p] = std::make_pair(dev, size);
  return p;
}

// Returns every cached (currently unused) block of all devices to the driver.
void dev_trim() {
  DevCache& c = dev_cache();
  std::lock_guard<std::mutex> lock(c.mu);
  int cur = 0;
  cudaGetDevice(&cur);
  for (std::map<std::pair<int, size_t>, std::vector<void*> >::iterator it = c.free_list.begin();
       it != c.free_list.end(); ++it) {
    cudaSetDevice(it->first.first);
    for (size_t i = 0; i < it->second.size(); ++i) cudaFree(it->second[i]);
    it->second.clear();
  }
  cudaSetDevice(cur);
}

void dev_free(void* p) {
  if (!p) return;
  DevCache& c = dev_cache();
  std::lock_guard<std::mutex> lock(c.mu);
  std::map<void*, std::pair<int, size_t> >::iterator it = c.live.find(p);
  if (it == c.live.end()) return;
  c.free_list[it->second].push_back(p);
  c.live.erase(it);
}

// Tensor map of a float plane group (tma.cuh).  cuTensorMapEncodeTiled is a driver-API
// entry point; it is fetched through the runtime so that the library does not link libcuda.
CUtensorMap make_plane_map(const float* base, int w, int h, int pitch, size_t plane_floats, int nplanes, int box_w,
                           int box_h) {
  typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeTiled encode = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    GB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    if (q != cudaDriverEntryPointSuccess || fn == nullptr)
      throw std::runtime_error("guetzli_b200: the CUDA driver does not provide cuTensorMapEncodeTiled");
    return reinterpret_cast<EncodeTiled>(fn);
  }();
  if (box_w % 4 != 0 || box_w > 256 || box_h > 256 || box_w < 1 || box_h < 1)
    throw std::runtime_error("make_plane_map: illegal box");
  CUtensorMap m;
  const cuuint64_t dims[3] = {static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(h), static_cast<cuuint64_t>(nplanes)};
  const cuuint64_t strides[2] = {static_cast<cuuint64_t>(pitch) * 4, static_cast<cuuint64_t>(plane_floats) * 4};
  const cuuint32_t box[3] = {static_cast<cuuint32_t>(box_w), static_cast<cuuint32_t>(box_h), 1};
  const cuuint32_t elem[3] = {1, 1, 1};
  const CUresult rc = encode(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, elem,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (%d) for %dx%dx%d pitch %d box %dx%d", static_cast<int>(rc),
             w, h, nplanes, pitch, box_w, box_h);
    throw std::runtime_error(buf);
  }
  return m;
}

static std::atomic<long long> g_h2d_bytes(0), g_d2h_bytes(0);
long long h2d_bytes_total() { return g_h2d_bytes.load(); }
long long d2h_bytes_total() { return g_d2h_bytes.load(); }

void h2d(void* dst, const void* src, size_t n, Stream s) {
  g_h2d_bytes += static_cast<long long>(n);
  GB_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, s));
}
// Waiting for a stream.  cudaStreamSynchronize spins on the host; that is the lowest latency
// for one image, but with many image contexts in flight (batch mode: one host thread per
// image, times one process per GPU) the spinning threads take the cores that the other
// threads' selection walks need.  With more than two live streams in the process the wait
// therefore sleeps on a blocking event instead.  GB200_SYNC=spin|block forces either.
static std::atomic<int> g_live_streams(0);
static void wait_stream(Stream s) {
  static const int forced = [] {
    const char* e = getenv("GB200_SYNC");
    return e == nullptr ? 0 : (e[0] == 'b' ? 2 : 1);
  }();
  const bool block = forced ? forced == 2 : g_live_streams.load(std::memory_order_relaxed) > 2;
  if (!block) {
    GB_CUDA(cudaStreamSynchronize(s));
    return;
  }
  thread_local std::map<int, cudaEvent_t> events;  // one per device this thread has used
  int dev = 0;
  GB_CUDA(cudaGetDevice(&dev));
  cudaEvent_t& ev = events[dev];
  if (ev == nullptr) GB_CUDA(cudaEventCreateWithFlags(&ev, cudaEventBlockingSync | cudaEventDisableTiming));
  GB_CUDA(cudaEventRecord(ev, s));
  GB_CUDA(cudaEventSynchronize(ev));
}

// Small results (sums, counters, the window's block states: ≈7 per iteration of the search) come
// back through a pinned per-thread mailbox: a copy into pageable memory is staged by the driver
// and waits on its own; the pinned copy is a plain DMA followed by the stream wait.
namespace {
constexpr size_t kMailboxBytes = 64 << 10;
struct Mailbox {
  void* p = nullptr;
  bool tried = false;
  ~Mailbox() {
    if (p) cudaFreeHost(p);
  }
};
void* mailbox() {
  thread_local Mailbox m;
  if (!m.tried) {
    m.tried = true;
    if (cudaHostAlloc(&m.p, kMailboxBytes, cudaHostAllocPortable) != cudaSuccess) {
      m.p = nullptr;
      cudaGetLastError();  // pageable copies then
    }
  }
  return m.p;
}
}  // namespace

void d2h(void* dst, const void* src, size_t n, Stream s) {
  g_d2h_bytes += static_cast<long long>(n);
  void* pin = n <= kMailboxBytes ? mailbox() : nullptr;
  if (pin != nullptr) {
    GB_CUDA(cudaMemcpyAsync(pin, src, n, cudaMemcpyDeviceToHost, s));
    wait_stream(s);
    memcpy(dst, pin, n);
    return;
  }
  GB_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, s));
  wait_stream(s);
}
void d2d(void* dst, const void* src, size_t n, Stream s) {
  GB_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, s));
}
void dev_zero(void* dst, size_t n, Stream s) { GB_CUDA(cudaMemsetAsync(dst, 0, n, s)); }
void stream_sync(Stream s) { wait_stream(s); }

int cuda_device_count() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

void select_device(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    throw std::runtime_error(
        "guetzli_b200: no CUDA device visible. This library has no CPU fallback; it needs an H100 (sm_90a).");
  }
  GB_CUDA(cudaSetDevice(device));
}

Stream make_stream() {
  cudaStream_t s;
  GB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  ++g_live_streams;
  return s;
}

void destroy_stream(Stream s) {
  --g_live_streams;
  cudaStreamDestroy(s);
}

namespace {
struct Prof {
  std::mutex mu;
  bool on = false;
  long launches = 0;
  struct Entry {
    long launches = 0;
    double ms = 0;
    double elements = 0;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t> > pending;
  };
  std::map<std::string, Entry> by_name;
};
thread_local cudaEvent_t t_cur_start = nullptr;
Prof& prof() {
  static Prof p;
  return p;
}

void drain(Prof::Entry& e) {
  for (size_t i = 0; i < e.pending.size(); ++i) {
    float ms = 0;
    cudaEventSynchronize(e.pending[i].second);
    cudaEventElapsedTime(&ms, e.pending[i].first, e.pending[i].second);
    e.ms += ms;
    cudaEventDestroy(e.pending[i].first);
    cudaEventDestroy(e.pending[i].second);
  }
  e.pending.clear();
}
}  // namespace

void note_launch(const char* name, Stream s, double elements) {
  Prof& p = prof();
  std::lock_guard<std::mutex> lock(p.mu);
  ++p.launches;
  Prof::Entry& e = p.by_name[name];
  ++e.launches;
  e.elements += elements;
  if (p.on) {
    cudaEvent_t a;
    cudaEventCreate(&a);
    cudaEventRecord(a, s);
    t_cur_start = a;
  }
}

void note_launch_end(const char* name, Stream s) {
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) cuda_fail(err, name, __FILE__, __LINE__);
  Prof& p = prof();
  std::lock_guard<std::mutex> lock(p.mu);
  if (p.on && t_cur_start) {
    cudaEvent_t b;
    cudaEventCreate(&b);
    cudaEventRecord(b, s);
    Prof::Entry& e = p.by_name[name];
    e.pending.push_back(std::make_pair(t_cur_start, b));
    t_cur_start = nullptr;
    if (e.pending.size() > 256) drain(e);
  }
}

bool profiling_on() {
  Prof& p = prof();
  std::lock_guard<std::mutex> lock(p.mu);
  return p.on;
}

// kernels executed by a CUDA graph launch (or, negative, recorded during a capture without running)
void add_launches(long n) {
  Prof& p = prof();
  std::lock_guard<std::mutex> lock(p.mu);
  p.launches += n;
}

long total_launches() {
  Prof& p = prof();
  std::lock_guard<std::mutex> lock(p.mu);
  return p.launches;
}

void profiling_enable(bool on) {
  Prof& p = prof();
  std::lock_guard<std::mutex> lock(p.mu);
  p.on = on;
}

std::vector<KernelStat> profiling_snapshot() {
  Prof& p = prof();
  std::lock_guard<std::mutex> lock(p.mu);
  std::vector<KernelStat> out;
  for (std::map<std::string, Prof::Entry>::iterator it = p.by_name.begin(); it != p.by_name.end(); ++it) {
    drain(it->second);
    KernelStat k;
    k.name = it->first;
    k.launches = it->second.launches;
    k.ms = it->second.ms;
    k.elements = it->second.elements;
    out.push_back(k);
  }
  return out;
}

void profiling_reset() {
  Prof& p = prof();
  std::lock_guard<std::mutex> lock(p.mu);
  for (std::map<std::string, Prof::Entry>::iterator it = p.by_name.begin(); it != p.by_name.end(); ++it)
    drain(it->second);
  p.by_name.clear();
  p.launches = 0;
}

}  // namespace gb200
