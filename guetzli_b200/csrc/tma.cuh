// TMA (cp.async.bulk.tensor) plumbing for the image-plane kernels: tensor maps over
// float plane groups and the mbarrier / bulk-copy PTX of sm_90a.
//
// A plane group [n][h][pitch] is described to the TMA unit as a rank-3 tensor with
// extents {w, h, n}: the TRUE width w, so that a box reaching past the image (x < 0,
// x >= w, y < 0, y >= h) is zero-filled by the hardware.  That is exactly the padding
// the stencils need: Malta reads zeros outside the image (b/butteraugli.cc:1429) and a
// border sum of the blur over the clipped support equals the sum over the full support
// with zero samples (0 * tap adds +0 to a sum that starts at +0).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdexcept>

namespace gb200 {

// host: rank-3 float tensor map, box {box_w, box_h, 1}; no swizzle, no interleave
CUtensorMap make_plane_map(const float* base, int w, int h, int pitch, size_t plane_floats, int nplanes, int box_w,
                           int box_h);

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// makes the initialised barrier visible to the async (TMA) proxy
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t a = smem_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(a), "r"(parity)
        : "memory");
  } while (!done);
}
// one box {x.., y.., plane} of a plane group -> shared memory; completes `bar` with the box bytes
__device__ __forceinline__ void tma_load_box(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int x, int y,
                                             int plane) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(plane)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_map(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

}  // namespace gb200
