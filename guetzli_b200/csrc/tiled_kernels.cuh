// Hand-tiled sm_90a kernels of the STAGED Compare chain (round 1: one kernel per stage).  The
// product runs the TMA-staged fused chain of fused_kernels.cuh; this chain stays in the library
// behind GB200_COMPARE=staged as the second implementation that the fused one is checked
// against on the GPU (tests/test_gpu_parity.py::test_fused_matches_staged), and it shares the
// Malta line-sum window code, the JPEG histogram and the order-select kernels with it.
// Original note: hand-tiled kernels for the stages that dominate Compare (a10).  They
// compute exactly what the generic per-pixel functors in kernels.h compute (same
// helper arithmetic from ba_math.h, same tap order) but stage tiles in shared
// memory and keep partial results in registers instead of round-tripping planes
// through HBM.  CUDA only; the CPU port keeps the generic functors.
#pragma once
#include <cuda_runtime.h>

#include <cstdlib>
#include <stdexcept>

#include "ba_math.h"
#include "jpeg_dev.h"
#include "kernels.h"
#include "malta_unrolled.inc"

namespace gb200 {

// ---------------------------------------------------------------------------
// S7 Malta, one colour channel per launch (b/butteraugli.cc:829-871,1461-1568).
// For each of the three bands (uhf: 9-tap lines; hf, mf: 5-tap lines) the CTA
// builds the "diffs" tile (pre-pass, malta_diff) with a 4-pixel zero-padded halo
// in shared memory, every thread evaluates the 16 line sums of its two pixels from
// shared memory, and the three results are accumulated in registers in the
// reference's call order: ac = ((0 + uhf) + hf) + mf.   Replaces 3x(malta_pre +
// malta_acc): 6 plane reads + 1 write per pixel instead of 9 reads + 6 writes.
struct MaltaChannelArgs {
  const float* lum0[3];  // original:  uhf, hf, mf plane of this channel
  const float* lum1[3];  // candidate
  MaltaParams mp[3];
  float* acc;            // block_diff_ac plane of this channel (overwritten)
  Geom g;
  int y0, nrows;         // rows [y0, y0 + nrows) are produced
};

// Tile 64 x 32 outputs per CTA (256 threads = 16 column groups x 16
// rows); a thread makes 4 ADJACENT pixels of a row, for rows ty and ty + 16.  Its 9 x 12
// sample window comes from shared memory as 27 float4 loads and then lives in registers:
// every sample is loaded once per 4 pixels instead of once per line-sum term.
#define GB_MALTA_TILE_W 64
#define GB_MALTA_TILE_H 32
#define GB_MALTA_SW (GB_MALTA_TILE_W + 8)
#define GB_MALTA_SH (GB_MALTA_TILE_H + 8)

// Line sums of the thread's 2 x 4 pixels for one band from the diffs tile; r += sums.
__device__ __forceinline__ void malta_window_sums(const float* tile, int tx, int ty, bool hf, float r[2][4]) {
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    // window rows ty + 16k .. +8, columns 4tx .. 4tx + 11 of the tile (pixel p of the
    // thread is at window column 4 + p, window row 4)
    float win[9][12];
    const float4* src = reinterpret_cast<const float4*>(tile + (ty + 16 * k) * GB_MALTA_SW + 4 * tx);
#pragma unroll
    for (int wy = 0; wy < 9; ++wy) {
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const float4 v = src[wy * (GB_MALTA_SW / 4) + q];
        win[wy][4 * q + 0] = v.x;
        win[wy][4 * q + 1] = v.y;
        win[wy][4 * q + 2] = v.z;
        win[wy][4 * q + 3] = v.w;
      }
    }
    float u0 = 0.0f, u1 = 0.0f, u2 = 0.0f, u3 = 0.0f;
#define GB_T0(dx, dy) win[(dy) + 4][(dx) + 4]
#define GB_T1(dx, dy) win[(dy) + 4][(dx) + 5]
#define GB_T2(dx, dy) win[(dy) + 4][(dx) + 6]
#define GB_T3(dx, dy) win[(dy) + 4][(dx) + 7]
    if (hf) {
      GB_MALTA_HF_SUMS(GB_T0, u0)
      GB_MALTA_HF_SUMS(GB_T1, u1)
      GB_MALTA_HF_SUMS(GB_T2, u2)
      GB_MALTA_HF_SUMS(GB_T3, u3)
    } else {
      GB_MALTA_LF_SUMS(GB_T0, u0)
      GB_MALTA_LF_SUMS(GB_T1, u1)
      GB_MALTA_LF_SUMS(GB_T2, u2)
      GB_MALTA_LF_SUMS(GB_T3, u3)
    }
#undef GB_T0
#undef GB_T1
#undef GB_T2
#undef GB_T3
    r[k][0] = r[k][0] + u0;
    r[k][1] = r[k][1] + u1;
    r[k][2] = r[k][2] + u2;
    r[k][3] = r[k][3] + u3;
  }
}

__device__ __forceinline__ void malta_store(const MaltaChannelArgs& a, int x0, int y0, int y_end, int tx, int ty,
                                            const float r[2][4]) {
  const int xb = x0 + 4 * tx;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int y = y0 + ty + 16 * k;
    if (y >= y_end || xb >= a.g.w) continue;
    float* orow = a.acc + static_cast<size_t>(y) * a.g.pitch + xb;
    if (xb + 3 < a.g.w) {
      *reinterpret_cast<float4*>(orow) = make_float4(r[k][0], r[k][1], r[k][2], r[k][3]);
    } else {
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (xb + p < a.g.w) orow[p] = r[k][p];
    }
  }
}

// The pre-pass is its own elementwise kernel (three diffs planes, zero in
// the pad columns), and the line-sum kernel only copies tiles (cp.async, double
// buffered over the bands, zero fill outside the plane).
__global__ void __launch_bounds__(256) k_malta_pre3(MaltaChannelArgs a, float* diffs, int r0) {
  const int x = blockIdx.x * 256 + threadIdx.x;
  if (x >= a.g.pitch) return;
  const int y = r0 + blockIdx.y, band = blockIdx.z;
  const size_t o = static_cast<size_t>(y) * a.g.pitch + x;
  float v = 0.0f;
  if (x < a.g.w) v = malta_diff(a.lum0[band][o], a.lum1[band][o], a.mp[band]);
  diffs[band * a.g.plane + o] = v;
}

__device__ __forceinline__ void cp_async16_zfill(float* smem, const float* gmem, bool valid) {
  const unsigned int sa = static_cast<unsigned int>(__cvta_generic_to_shared(smem));
  const int bytes = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(sa), "l"(gmem), "r"(bytes));
}

__device__ __forceinline__ void malta_stage_async(float* tile, const float* plane, const Geom& g, int x0, int y0,
                                                  int tid) {
  constexpr int Q = GB_MALTA_SW / 4;
  for (int i = tid; i < GB_MALTA_SH * Q; i += 256) {
    const int sy = i / Q, q = i - sy * Q;
    const int x = x0 - 4 + 4 * q, y = y0 + sy - 4;
    const bool valid = x >= 0 && x < g.pitch && y >= 0 && y < g.h;
    const float* src = valid ? plane + static_cast<size_t>(y) * g.pitch + x : plane;
    cp_async16_zfill(tile + sy * GB_MALTA_SW + 4 * q, src, valid);
  }
  asm volatile("cp.async.commit_group;\n" ::);
}

__global__ void __launch_bounds__(256, 2) k_malta_sums(MaltaChannelArgs a, const float* diffs) {
  __shared__ __align__(16) float tile[2][GB_MALTA_SH * GB_MALTA_SW];
  const int tx = threadIdx.x, ty = threadIdx.y;  // 16 x 16
  const int x0 = blockIdx.x * GB_MALTA_TILE_W, y0 = a.y0 + blockIdx.y * GB_MALTA_TILE_H;
  const int y_end = a.y0 + a.nrows < a.g.h ? a.y0 + a.nrows : a.g.h;
  const int tid = ty * 16 + tx;
  float r[2][4];
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int p = 0; p < 4; ++p) r[k][p] = 0.0f;
  malta_stage_async(tile[0], diffs, a.g, x0, y0, tid);
#pragma unroll 1
  for (int band = 0; band < 3; ++band) {
    if (band + 1 < 3) {
      malta_stage_async(tile[(band + 1) & 1], diffs + (band + 1) * a.g.plane, a.g, x0, y0, tid);
      asm volatile("cp.async.wait_group 1;\n" ::);
    } else {
      asm volatile("cp.async.wait_group 0;\n" ::);
    }
    __syncthreads();
    malta_window_sums(tile[band & 1], tx, ty, band == 0, r);
    __syncthreads();  // the buffer is refilled two bands later
  }
  malta_store(a, x0, y0, y_end, tx, ty, r);
}

inline void launch_malta_channel(Stream s, const MaltaChannelArgs& a, float* scratch3) {
  note_launch("malta_channel", s, static_cast<double>(a.g.w) * a.nrows);
  dim3 block(16, 16), grid((a.g.w + GB_MALTA_TILE_W - 1) / GB_MALTA_TILE_W, (a.nrows + GB_MALTA_TILE_H - 1) / GB_MALTA_TILE_H);
  const int r0 = a.y0 - 4 > 0 ? a.y0 - 4 : 0;
  const int r1 = a.y0 + a.nrows + 4 < a.g.h ? a.y0 + a.nrows + 4 : a.g.h;
  dim3 pgrid((a.g.pitch + 255) / 256, r1 - r0, 3);
  k_malta_pre3<<<pgrid, 256, 0, s>>>(a, scratch3, r0);
  k_malta_sums<<<grid, block, 0, s>>>(a, scratch3);
  note_launch_end("malta_channel", s);
}

// ---------------------------------------------------------------------------
// Separable blur (b/butteraugli.cc:184-233), register-blocked, radius known at
// compile time.  The interior taps travel as a kernel argument, i.e. they sit in
// the constant bank and every multiply takes its tap as an immediate constant
// operand (fully unrolled loops): per multiply-add the SM issues one FMUL and one
// FADD (no FMA: bit-exactness, DESIGN.md §3) and per input sample one load.
// For every output the products are added in ascending tap order, exactly the
// reference's sequence.  Border outputs (p < r or p + r >= n) take the raw-tap /
// per-position-scale path of ConvolveBorderColumn.
#define GB_BLUR_MAX_R 24

struct BlurArgs {
  const float* in;
  float* out;
  BlurTab tab;
  Geom g;
  int rows;   // rows to produce = nplanes * nrows
  int y0;     // first row of every plane
  int nrows;  // rows per plane
};

template <int R>
struct BlurTaps {
  float n[2 * R + 1];  // taps * (1/sum)
};

// x pass: a warp owns one row segment of 256 outputs.  It stages the 256 + 2R input
// samples in shared memory (its private row: only __syncwarp), then every lane makes 8
// ADJACENT outputs, streaming its 8 + 2R samples once through registers into eight
// accumulators (one shared-memory load per sample instead of one per product).  The
// row is stored with one pad word per 8 samples, so lane l reads word 9l + const:
// conflict-free for a fixed stream position.
#define GB_BLURX_TW 256
#define GB_BLURX_PT 8
template <int R>
__global__ void __launch_bounds__(256) k_blur_x(BlurArgs a, BlurTaps<R> taps) {
  constexpr int LEN = 2 * R + 1;
  constexpr int SPAN = GB_BLURX_TW + 2 * R;
  constexpr int SROW = SPAN + SPAN / 8 + 1;
  __shared__ float tile[8][SROW];
  const int lane = threadIdx.x;
  const int x0 = blockIdx.x * GB_BLURX_TW;
  const int row = blockIdx.y * 8 + threadIdx.y;
  if (row >= a.rows) return;  // whole warp; no block-wide barrier below
  const int w = a.g.w;
  const int pl = row / a.nrows;
  const size_t grow = (static_cast<size_t>(pl) * a.g.h + a.y0 + (row - pl * a.nrows)) * a.g.pitch;
  const float* irow = a.in + grow;
  float* orow = a.out + grow;
  float* srow = tile[threadIdx.y];
#pragma unroll 4
  for (int sx = lane; sx < SPAN; sx += 32) {
    const int x = x0 - R + sx;
    srow[sx + (sx >> 3)] = (x >= 0 && x < w) ? irow[x] : 0.0f;
  }
  __syncwarp();
  // outputs x0 + 8*lane + o, o < 8; sample t of the lane sits at tile column 8*lane + t
  float acc[GB_BLURX_PT];
#pragma unroll
  for (int o = 0; o < GB_BLURX_PT; ++o) acc[o] = 0.0f;
  const float* sl = srow + 9 * lane;
#pragma unroll
  for (int t = 0; t < LEN + GB_BLURX_PT - 1; ++t) {
    const float v = sl[t + (t >> 3)];
#pragma unroll
    for (int o = 0; o < GB_BLURX_PT; ++o) {
      const int j = t - o;  // compile-time after unrolling; ascending for every output
      if (j >= 0 && j < LEN) acc[o] += v * taps.n[j];
    }
  }
  const int xb = x0 + 8 * lane;
  if (x0 >= R && x0 + GB_BLURX_TW - 1 + R < w) {  // whole tile interior (all but the first / last tile of a row)
    float4* o4 = reinterpret_cast<float4*>(orow + xb);  // pitch, x0 multiples of 32 floats; 256-byte aligned planes
    o4[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    o4[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    return;
  }
#pragma unroll
  for (int o = 0; o < GB_BLURX_PT; ++o) {
    const int x = xb + o;
    if (x < w && x >= R && x + R < w) orow[x] = acc[o];
  }
  // border rule (blur_tap_sum's clamped window and per-column scale): at most R outputs at
  // either end of the row, one per lane so that their serial sums run side by side
#pragma unroll 1
  for (int side = 0; side < 2; ++side) {
    const int x = side == 0 ? lane : w - R + lane;
    if (lane >= R || x < x0 || x >= x0 + GB_BLURX_TW || x >= w || (side == 1 && x < R)) continue;
    const int lo = x < R ? 0 : x - R;
    const int hi = (x + R < w - 1) ? x + R : w - 1;
    const float* tp = a.tab.taps + (R - x);
    float sum = 0.0f;
#pragma unroll 4
    for (int j = lo; j <= hi; ++j) {
      const int c = j - x0 + R;
      sum += srow[c + (c >> 3)] * tp[j];
    }
    orow[x] = sum * a.tab.scale_x[x];
  }
}

// y pass: a thread owns one column and makes GB_BLURY_R consecutive rows, streaming the
// GB_BLURY_R + 2R input rows once (coalesced across the warp) into that many accumulators.
#define GB_BLURY_R 8
#define GB_BLURY_CH 16
template <int R>
__global__ void __launch_bounds__(128) k_blur_y(BlurArgs a, BlurTaps<R> taps) {
  constexpr int LEN = 2 * R + 1;
  const int x = blockIdx.x * 128 + threadIdx.x;
  if (x >= a.g.w) return;
  const int h = a.g.h;
  const int y_end = a.y0 + a.nrows < h ? a.y0 + a.nrows : h;
  const int strips = (a.nrows + GB_BLURY_R - 1) / GB_BLURY_R;
  const int pl = blockIdx.y / strips;
  const int yb = a.y0 + (blockIdx.y - pl * strips) * GB_BLURY_R;
  const float* col = a.in + static_cast<size_t>(pl) * a.g.plane + x;
  float* ocol = a.out + static_cast<size_t>(pl) * a.g.plane + x;
  const size_t pitch = a.g.pitch;
  const bool interior = (yb >= R) && (yb + GB_BLURY_R - 1 + R < h) && (yb + GB_BLURY_R <= y_end);
  if (interior) {
    // The GB_BLURY_R + 2R input rows are fetched in batches of GB_BLURY_CH loads that are
    // all in flight together, one batch ahead of the arithmetic (register double buffer).
    constexpr int NT = LEN + GB_BLURY_R - 1;
    constexpr int NCH = (NT + GB_BLURY_CH - 1) / GB_BLURY_CH;
    float acc[GB_BLURY_R];
#pragma unroll
    for (int o = 0; o < GB_BLURY_R; ++o) acc[o] = 0.0f;
    const float* p = col + static_cast<size_t>(yb - R) * pitch;
    float buf[2][GB_BLURY_CH];
#pragma unroll
    for (int i = 0; i < GB_BLURY_CH; ++i) {
      if (i < NT) buf[0][i] = *p;
      p += pitch;
    }
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      if (c + 1 < NCH) {
#pragma unroll
        for (int i = 0; i < GB_BLURY_CH; ++i) {
          if ((c + 1) * GB_BLURY_CH + i < NT) buf[(c + 1) & 1][i] = *p;
          p += pitch;
        }
      }
#pragma unroll
      for (int i = 0; i < GB_BLURY_CH; ++i) {
        const int t = c * GB_BLURY_CH + i;
        if (t < NT) {
          const float v = buf[c & 1][i];
#pragma unroll
          for (int o = 0; o < GB_BLURY_R; ++o) {
            const int j = t - o;  // compile-time after unrolling
            if (j >= 0 && j < LEN) acc[o] += v * taps.n[j];
          }
        }
      }
    }
#pragma unroll
    for (int o = 0; o < GB_BLURY_R; ++o) ocol[static_cast<size_t>(yb + o) * pitch] = acc[o];
  } else {
    // strip that touches the top / bottom of the plane (or the end of the row range):
    // same streaming pass with rows outside the plane read as zero -- exact for every
    // row whose 2R+1 taps lie inside the plane -- then the border rows are recomputed
    // with the border rule, all (up to 8) of them in one pass over the column so that
    // their serial sums overlap.
    float acc[GB_BLURY_R];
#pragma unroll
    for (int o = 0; o < GB_BLURY_R; ++o) acc[o] = 0.0f;
#pragma unroll
    for (int t = 0; t < LEN + GB_BLURY_R - 1; ++t) {
      const int yi = yb - R + t;
      const float v = (yi >= 0 && yi < h) ? col[static_cast<size_t>(yi) * pitch] : 0.0f;
#pragma unroll
      for (int o = 0; o < GB_BLURY_R; ++o) {
        const int j = t - o;
        if (j >= 0 && j < LEN) acc[o] += v * taps.n[j];
      }
    }
    bool any_border = false;
#pragma unroll
    for (int o = 0; o < GB_BLURY_R; ++o) {
      const int y = yb + o;
      const bool border = y < R || y + R >= h;
      any_border = any_border || (border && y < y_end);
      if (y < y_end && !border) ocol[static_cast<size_t>(y) * pitch] = acc[o];
    }
    if (any_border) {  // uniform over the CTA
#pragma unroll
      for (int o = 0; o < GB_BLURY_R; ++o) acc[o] = 0.0f;
      const int j_lo = yb - R > 0 ? yb - R : 0;
      const int j_hi = yb + GB_BLURY_R - 1 + R < h - 1 ? yb + GB_BLURY_R - 1 + R : h - 1;
      const float* raw = a.tab.taps;
#pragma unroll 2
      for (int j = j_lo; j <= j_hi; ++j) {
        const float v = col[static_cast<size_t>(j) * pitch];
#pragma unroll
        for (int o = 0; o < GB_BLURY_R; ++o) {
          const int k = j - (yb + o) + R;  // ascending with j for every output, as in blur_tap_sum
          if (k >= 0 && k < LEN) acc[o] += v * raw[k];
        }
      }
#pragma unroll
      for (int o = 0; o < GB_BLURY_R; ++o) {
        const int y = yb + o;
        if (y < y_end && (y < R || y + R >= h)) ocol[static_cast<size_t>(y) * pitch] = acc[o] * a.tab.scale_y[y];
      }
    }
  }
}

template <int R>
inline void launch_blur_r(Stream s, const float* in, float* tmp, float* out, int nplanes, const BlurTab& tab,
                          const float* host_taps_n, const Geom& g, int y0, int nrows) {
  BlurTaps<R> taps;
  for (int j = 0; j < 2 * R + 1; ++j) taps.n[j] = host_taps_n[j];
  // strip mode: the y pass reads x-pass rows outside [y0, y0+nrows) that are stale; the
  // outputs they reach lie in the halo margin that the next stage no longer needs
  const int xy0 = y0, xy1 = y0 + nrows;
  BlurArgs ax{in, tmp, tab, g, nplanes * (xy1 - xy0), xy0, xy1 - xy0};
  dim3 bx(32, 8), gx((g.w + GB_BLURX_TW - 1) / GB_BLURX_TW, (nplanes * (xy1 - xy0) + 7) / 8);
  note_launch("blur_x", s, static_cast<double>(g.w) * (xy1 - xy0) * nplanes);
  k_blur_x<R><<<gx, bx, 0, s>>>(ax, taps);
  note_launch_end("blur_x", s);
  BlurArgs ay{tmp, out, tab, g, nplanes * nrows, y0, nrows};
  const int strips = (nrows + GB_BLURY_R - 1) / GB_BLURY_R;
  dim3 gy((g.w + 127) / 128, strips * nplanes);
  note_launch("blur_y", s, static_cast<double>(g.w) * nrows * nplanes);
  k_blur_y<R><<<gy, 128, 0, s>>>(ay, taps);
  note_launch_end("blur_y", s);
}

// host_taps_n: the interior kernel (taps * 1/sum) as built by tables.cc.
inline void launch_blur_tiled(Stream s, const float* in, float* tmp, float* out, int nplanes, const BlurTab& tab,
                              const float* host_taps_n, const Geom& g, int y0, int nrows) {
  switch (tab.r) {
    case 2: launch_blur_r<2>(s, in, tmp, out, nplanes, tab, host_taps_n, g, y0, nrows); break;
    case 3: launch_blur_r<3>(s, in, tmp, out, nplanes, tab, host_taps_n, g, y0, nrows); break;
    case 4: launch_blur_r<4>(s, in, tmp, out, nplanes, tab, host_taps_n, g, y0, nrows); break;
    case 5: launch_blur_r<5>(s, in, tmp, out, nplanes, tab, host_taps_n, g, y0, nrows); break;
    case 8: launch_blur_r<8>(s, in, tmp, out, nplanes, tab, host_taps_n, g, y0, nrows); break;
    case 16: launch_blur_r<16>(s, in, tmp, out, nplanes, tab, host_taps_n, g, y0, nrows); break;
    case 20: launch_blur_r<20>(s, in, tmp, out, nplanes, tab, host_taps_n, g, y0, nrows); break;
    case 23: launch_blur_r<23>(s, in, tmp, out, nplanes, tab, host_taps_n, g, y0, nrows); break;
    case 24: launch_blur_r<24>(s, in, tmp, out, nplanes, tab, host_taps_n, g, y0, nrows); break;
    default: throw std::runtime_error("blur radius without a compiled kernel");
  }
}

// ---------------------------------------------------------------------------
// a11 symbol histograms with a per-CTA shared-memory histogram (same counts as
// JpegHistAcc + JpegHistSum in jpeg_dev.h): out[6][257] = dc0 dc1 dc2 ac0 ac1 ac2.
__global__ void __launch_bounds__(256) k_jpeg_hist(const int16_t* cand, const int* q, const int* zigzag,
                                                   unsigned int* out, unsigned int* chroma_nonzero, int nblocks) {
  __shared__ unsigned int sh[kHistStride];
  __shared__ int sq[192];
  __shared__ int szz[64];
  for (int i = threadIdx.x; i < kHistStride; i += 256) sh[i] = 0;
  if (threadIdx.x < 192) sq[threadIdx.x] = q[threadIdx.x];
  if (threadIdx.x < 64) szz[threadIdx.x] = zigzag[threadIdx.x];
  __syncthreads();
  const int units = 3 * nblocks;
  bool chroma = false;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < units; i += gridDim.x * 256) {
    const int c = i / nblocks, b = i - c * nblocks;
    const int16_t* blk = cand + static_cast<size_t>(i) * 64;
    const int* qc = sq + 64 * c;
    const int prev = b > 0 ? div_exact_multiple((blk - 64)[0], qc[0]) : 0;
    JpegHistAcc::Visitor v{sh + c * 257, sh + (3 + c) * 257};
    visit_block_symbols(blk, qc, prev, szz, v);
    if (c > 0) {
      for (int k = 0; k < 64; ++k) chroma = chroma || (blk[k] != 0);
    }
  }
  if (chroma) *chroma_nonzero = 1u;
  __syncthreads();
  for (int i = threadIdx.x; i < kHistStride; i += 256) {
    const unsigned int n = sh[i];
    if (n) atomicAdd(&out[i], n);
  }
}

inline void launch_jpeg_hist(Stream s, const int16_t* cand, const int* q, const int* zigzag, unsigned int* out,
                             unsigned int* chroma_nonzero, int nblocks) {
  int ctas = (3 * nblocks + 255) / 256;
  if (ctas > 4 * kTargetSMs) ctas = 4 * kTargetSMs;
  note_launch("jpeg_hist", s, 3.0 * nblocks);
  k_jpeg_hist<<<ctas, 256, 0, s>>>(cand, q, zigzag, out, chroma_nonzero, nblocks);
  note_launch_end("jpeg_hist", s);
}

// ---------------------------------------------------------------------------
// a16 key histograms with a per-CTA shared-memory histogram (keys cluster in a few
// bins: global atomics would serialise), flushed once per CTA; and the matching
// single-CTA bin search.  Same results as OrderKeyHist / OrderSelectBin (kernels.h).
__global__ void __launch_bounds__(256) k_order_hist(OrderKeyCommon c, unsigned int* hist, const OrderSelectState* st,
                                                    int level, int entries) {
  __shared__ unsigned int sh[kOrderBins];
  for (int i = threadIdx.x; i < kOrderBins; i += 256) sh[i] = 0;
  __syncthreads();
  for (int e = blockIdx.x * 256 + threadIdx.x; e < entries; e += gridDim.x * 256) {
    float v;
    int b;
    if (!c.key(e, &b, &v)) continue;
    unsigned int bin;
    if (order_bin(st, level, hd_float_sortable(v), &bin)) atomicAdd(&sh[bin], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kOrderBins; i += 256) {
    const unsigned int n = sh[i];
    if (n) atomicAdd(&hist[i], n);
  }
}

__global__ void __launch_bounds__(1024) k_order_select_bin(const unsigned int* hist, OrderSelectState* st, int level) {
  __shared__ unsigned int warp_tot[32];
  const int t = threadIdx.x;
  const unsigned int h0 = hist[2 * t], h1 = hist[2 * t + 1];
  const unsigned int local = h0 + h1;
  unsigned int incl = local;
  const int lane = t & 31, warp = t >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  unsigned int base = 0, total = 0;
  for (int k = 0; k < 32; ++k) {
    if (k < warp) base += warp_tot[k];
    total += warp_tot[k];
  }
  const unsigned int excl = base + incl - local;
  const unsigned int want = level == 0 ? st->want : (st->want > st->below0 ? st->want - st->below0 : 0u);
  // serial semantics: first bin i with cum_before(i) + hist[i] >= want; none -> last bin
  unsigned int bin = 0xffffffffu, at = 0;
  if (excl + h0 >= want) {
    if (t == 0 || excl < want || want == 0) {
      // candidate: bin 2t, valid only if no earlier bin qualifies
      bin = 2 * t;
      at = excl;
    }
  } else if (excl + local >= want) {
    bin = 2 * t + 1;
    at = excl + h0;
  }
  // the first qualifying bin overall = minimum candidate
  __shared__ unsigned int best_bin;
  if (t == 0) best_bin = 0xffffffffu;
  __syncthreads();
  if (bin != 0xffffffffu) atomicMin(&best_bin, bin);
  __syncthreads();
  const unsigned int chosen = best_bin;
  if (chosen == 0xffffffffu) {
    if (t == 0) {
      const unsigned int last = kOrderBins - 1;
      const unsigned int before = total - hist[last];
      if (level == 0) {
        st->bin0 = last;
        st->below0 = before;
        st->total = total;
      } else {
        st->threshold = (st->bin0 << 21) | (last << 10) | 0x3ffu;
        st->kept = st->below0 + before + hist[last];
        st->counter = 0;
      }
    }
    return;
  }
  if (bin == chosen) {
    if (level == 0) {
      st->bin0 = chosen;
      st->below0 = at;
      st->total = total;
    } else {
      st->threshold = (st->bin0 << 21) | (chosen << 10) | 0x3ffu;
      st->kept = st->below0 + at + hist[chosen];
      st->counter = 0;
    }
  }
}

inline void launch_order_hist(Stream s, const OrderKeyCommon& c, unsigned int* hist, const OrderSelectState* st,
                              int level, int entries) {
  int ctas = (entries + 256 * 8 - 1) / (256 * 8);
  if (ctas < 1) ctas = 1;
  if (ctas > 8 * kTargetSMs) ctas = 8 * kTargetSMs;  // 8 resident CTAs per SM
  note_launch("order_key_hist", s, entries);
  k_order_hist<<<ctas, 256, 0, s>>>(c, hist, st, level, entries);
  note_launch_end("order_key_hist", s);
}

inline void launch_order_select_bin(Stream s, const unsigned int* hist, OrderSelectState* st, int level) {
  note_launch("order_select_bin", s, kOrderBins);
  k_order_select_bin<<<1, 1024, 0, s>>>(hist, st, level);
  note_launch_end("order_select_bin", s);
}

}  // namespace gb200
