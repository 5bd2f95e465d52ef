// Launch / memory abstraction shared by the product (CUDA, sm_90a) and the
// CPU restatement (oracle/port, -DGB200_HOSTSIM).  See hd.h.
//
//   launch_2d(stream, f, w, h)  : f(x, y) for every 0<=x<w, 0<=y<h
//   launch_1d(stream, f, n)     : f(i)    for every 0<=i<n
//
// Functors must be trivially copyable, write only to locations no other
// invocation touches, and read only data produced by earlier launches.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <stdexcept>

#include "hd.h"

#if defined(GB200_HOSTSIM)

namespace gb200 {

typedef int Stream;  // unused

inline void* dev_alloc(size_t bytes) { return calloc(bytes ? bytes : 1, 1); }
inline void dev_free(void* p) { free(p); }
inline void h2d(void* dst, const void* src, size_t n, Stream = 0) { memcpy(dst, src, n); }
inline void d2h(void* dst, const void* src, size_t n, Stream = 0) { memcpy(dst, src, n); }
inline void d2d(void* dst, const void* src, size_t n, Stream = 0) { memcpy(dst, src, n); }
inline void dev_zero(void* dst, size_t n, Stream = 0) { memset(dst, 0, n); }
inline void stream_sync(Stream = 0) {}
inline const char* backend_name() { return "hostsim"; }
// caller-owned device memory and streams exist only on a GPU
inline int pointer_device(const void*) { throw std::runtime_error("the CPU port has no device memory"); }
inline void stream_wait(Stream, Stream) { throw std::runtime_error("the CPU port has no streams"); }
inline void d2d_2d(void*, size_t, const void*, size_t, size_t, size_t, Stream) {
  throw std::runtime_error("the CPU port has no device memory");
}
inline void copy_3d(void* dst, size_t dpitch, size_t drows, const void* src, size_t spitch, size_t srows, size_t width,
                    size_t rows, size_t depth, Stream) {
  for (size_t z = 0; z < depth; ++z)
    for (size_t r = 0; r < rows; ++r)
      memcpy(static_cast<char*>(dst) + (z * drows + r) * dpitch, static_cast<const char*>(src) + (z * srows + r) * spitch,
             width);
}

template <class F>
inline void launch_2d(Stream, const F& f, int w, int h, const char* = nullptr) {
#pragma omp parallel for schedule(static)
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) f(x, y);
}

template <class F>
inline void launch_1d(Stream, const F& f, int n, const char* = nullptr) {
#pragma omp parallel for schedule(dynamic, 16)
  for (int i = 0; i < n; ++i) f(i);
}

}  // namespace gb200

#else  // CUDA product build (there is no CPU fallback in the product)

struct CUstream_st;

namespace gb200 {

typedef CUstream_st* Stream;  // == cudaStream_t

// implemented in backend_cuda.cu; throw std::runtime_error on CUDA failures
void* dev_alloc(size_t bytes);
void dev_free(void* p);
void h2d(void* dst, const void* src, size_t n, Stream s);
void d2h(void* dst, const void* src, size_t n, Stream s);  // synchronous
void d2d(void* dst, const void* src, size_t n, Stream s);
void dev_zero(void* dst, size_t n, Stream s);
void stream_sync(Stream s);
// device ordinal of device memory (cudaPointerGetAttributes); -1 for host, managed or unknown pointers
int pointer_device(const void* p);
// work queued on `waiter` from now on runs after the work queued so far on `signaller` (an event)
void stream_wait(Stream waiter, Stream signaller);
// rows of `width` bytes between device pitches (cudaMemcpy2DAsync)
void d2d_2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t rows, Stream s);
// `depth` slices of `rows` rows of `width` bytes; a slice is drows (srows) rows of dpitch (spitch)
// bytes; host or device memory on either side (one cudaMemcpy3DAsync)
void copy_3d(void* dst, size_t dpitch, size_t drows, const void* src, size_t spitch, size_t srows, size_t width,
             size_t rows, size_t depth, Stream s);
inline const char* backend_name() { return "cuda-sm_90a"; }
// streaming multiprocessors of the target (H100 SXM); caps grid-stride launches
constexpr int kTargetSMs = 132;

// launch accounting (gpu_launches in bench.py; per-kernel-name CUDA-event timing)
void note_launch(const char* name, Stream s, double elements);
void note_launch_end(const char* name, Stream s);

}  // namespace gb200

#if defined(__CUDACC__)
#include <cuda_runtime.h>

namespace gb200 {

void cuda_fail(cudaError_t e, const char* what, const char* file, int line);
#define GB_CUDA(x)                                            \
  do {                                                        \
    cudaError_t e__ = (x);                                    \
    if (e__ != cudaSuccess) ::gb200::cuda_fail(e__, #x, __FILE__, __LINE__); \
  } while (0)

template <class F>
__global__ void __launch_bounds__(256) k_launch_2d(F f, int w, int h) {
  // 32x8 thread tile: a warp covers 32 consecutive x of one row (coalesced).
  int x = blockIdx.x * 32 + threadIdx.x;
  int y = blockIdx.y * 8 + threadIdx.y;
  if (x < w && y < h) f(x, y);
}

template <class F>
__global__ void __launch_bounds__(128) k_launch_1d(F f, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) f(i);
}

template <class F>
inline void launch_2d(Stream s, const F& f, int w, int h, const char* name = "px2d") {
  if (w <= 0 || h <= 0) return;
  dim3 block(32, 8), grid((w + 31) / 32, (h + 7) / 8);
  note_launch(name, s, static_cast<double>(w) * h);
  k_launch_2d<F><<<grid, block, 0, s>>>(f, w, h);
  note_launch_end(name, s);
}

template <class F>
inline void launch_1d(Stream s, const F& f, int n, const char* name = "px1d") {
  if (n <= 0) return;
  note_launch(name, s, n);
  k_launch_1d<F><<<(n + 127) / 128, 128, 0, s>>>(f, n);
  note_launch_end(name, s);
}

}  // namespace gb200
#endif  // __CUDACC__
#endif
