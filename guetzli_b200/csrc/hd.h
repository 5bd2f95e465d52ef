// Host/device portability shims for the single-source kernel bodies.
//
// Every arithmetic body of the hot path is written once, as a functor whose
// operator() is GB_HD.  The product compiles these with nvcc for sm_90a and
// launches them as CUDA kernels (backend_cuda.cuh).  The CPU restatement under
// oracle/port compiles the very same bodies with g++ (-DGB200_HOSTSIM) and
// runs them in plain loops; that build is test infrastructure and is never
// linked into the product library.
//
// Bit-exactness contract (SURVEY.md §0.4): no FMA contraction (nvcc
// --fmad=false, g++ -ffp-contract=off), IEEE div/sqrt, no flush-to-zero, and
// every float/double promotion written out explicitly.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define GB_HD __host__ __device__ __forceinline__
#define GB_D __device__ __forceinline__
#else
#define GB_HD inline
#define GB_D inline
#endif

namespace gb200 {

// std::min / std::max semantics (return first argument on ties / unordered).
template <typename T>
GB_HD T hd_min(T a, T b) { return (b < a) ? b : a; }
template <typename T>
GB_HD T hd_max(T a, T b) { return (a < b) ? b : a; }

GB_HD float hd_fabsf(float x) { return ::fabsf(x); }
GB_HD double hd_fabs(double x) { return ::fabs(x); }

// Relaxed atomics usable from kernel bodies on both backends.
GB_HD unsigned int hd_atomic_add(unsigned int* p, unsigned int v) {
#if defined(__CUDA_ARCH__)
  return atomicAdd(p, v);
#else
  return __atomic_fetch_add(p, v, __ATOMIC_RELAXED);
#endif
}
GB_HD unsigned int hd_atomic_or(unsigned int* p, unsigned int v) {
#if defined(__CUDA_ARCH__)
  return atomicOr(p, v);
#else
  return __atomic_fetch_or(p, v, __ATOMIC_RELAXED);
#endif
}
GB_HD unsigned int hd_atomic_min(unsigned int* p, unsigned int v) {
#if defined(__CUDA_ARCH__)
  return atomicMin(p, v);
#else
  unsigned int old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {
  }
  return old;
#endif
}
GB_HD unsigned int hd_float_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  unsigned int u;
  __builtin_memcpy(&u, &f, 4);
  return u;
#endif
}
// Monotone map float -> uint32 (total order; -0 sorts just below +0).
GB_HD unsigned int hd_float_sortable(float f) {
  const unsigned int u = hd_float_bits(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

}  // namespace gb200
