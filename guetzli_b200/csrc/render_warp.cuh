// a7 + a9 on sm_90a, one warp per 8x8 block: dequantised coefficients -> IDCT (the
// integer transform of g/idct.cc, shared with the zeroing kernel) -> YCbCr to RGB ->
// linear light, two pixels per lane.  Same arithmetic as the RenderBlocks functor in
// kernels.h (one thread per block), which stays the CPU port's version; the dirty-block
// lists of the search are a few thousand blocks, too few threads for that shape.
#pragma once
#include <cuda_runtime.h>

#include "zeroing_warp.cuh"

namespace gb200 {

struct RenderWarpArgs {
  const int16_t* cand;
  float* lin;
  const int* list;  // block indices, or nullptr: blocks b0 .. b0 + n - 1
  int b0, n;
  Geom g;
  Tables t;
};

__global__ void __launch_bounds__(256) k_render_blocks_warp(RenderWarpArgs a) {
  __shared__ int16_t s_blk[8][64];
  __shared__ int16_t s_col[8][64];
  __shared__ uint8_t s_px[8][3][64];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * 8 + warp;
  if (i >= a.n) return;
  const int b = a.list ? a.list[i] : a.b0 + i;
  const Geom& g = a.g;
  const Tables& t = a.t;
  for (int c = 0; c < 3; ++c) {
    const int16_t* src = a.cand + (static_cast<size_t>(c) * g.nblocks + b) * 64;
    reinterpret_cast<int*>(s_blk[warp])[lane] = reinterpret_cast<const int*>(src)[lane];  // 2 coefficients per lane
    __syncwarp();
    warp_idct(t.idct, s_blk[warp], s_col[warp], s_px[warp][c], lane);
  }
  const int bx = b % g.bw, by = b / g.bw;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int p = lane + 32 * k, iy = p >> 3, ix = p & 7;
    const int y = 8 * by + iy, x = 8 * bx + ix;
    if (y >= g.h || x >= g.w) continue;
    int r, gg, bb;
    ycc_to_rgb(t.cr_r, t.cb_b, t.cr_g, t.cb_g, s_px[warp][0][p], s_px[warp][1][p], s_px[warp][2][p], &r, &gg, &bb);
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    a.lin[o] = t.srgb_lin[r];
    a.lin[g.plane + o] = t.srgb_lin[gg];
    a.lin[2 * g.plane + o] = t.srgb_lin[bb];
  }
}

inline void launch_render_blocks_warp(Stream s, const RenderWarpArgs& a) {
  if (a.n <= 0) return;
  note_launch("render_blocks", s, a.n);
  k_render_blocks_warp<<<(a.n + 7) / 8, 256, 0, s>>>(a);
  note_launch_end("render_blocks", s);
}

}  // namespace gb200
