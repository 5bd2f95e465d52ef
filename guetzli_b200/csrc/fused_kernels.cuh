// TMA-staged, fused kernels of ButteraugliComparator::Compare (a10) for sm_90a.
//
// Every image-plane stage of the metric is a separable Gaussian blur followed by
// point-wise arithmetic (b/butteraugli.cc:324-366 opsin, :489-622 frequency split,
// :624-714 noise / asymmetric L2, :718-751 diffmap, :753-782,1699-1817 mask,
// :1597-1621 combine).  With FMA contraction forbidden (DESIGN.md §3) the blurs cost one
// FMUL + one FADD per tap and the chain is bound by instruction issue, not by HBM; so
// the kernels here are built to spend issue slots on those two instructions only:
//
//  * tiles (with their halo) are brought into shared memory by the TMA unit
//    (cp.async.bulk.tensor, one elected thread, mbarrier completion): no address
//    arithmetic, no load instructions, and the out-of-image zero fill is free;
//  * a thread keeps 4 (x pass) or 16 (y pass) accumulators and streams its window
//    through them: one shared-memory load per 4 samples (x, LDS.128) or per sample with
//    an immediate offset (y); taps are kernel parameters, i.e. constant-bank immediates;
//  * the point-wise stage that consumes a blur runs in the y pass's epilogue on the
//    values still in registers (Epi functors below), instead of as its own kernel
//    over planes in HBM;
//  * blurs of radius <= 5 do x and y in one kernel from one tile;
//  * the lf and mf blurs roll a window down a column strip (k_roll_blur): the x pass goes
//    to a shared-memory ring of rows instead of a plane in HBM.
//
// Border outputs (fewer than r samples to an image edge) use the raw taps and the
// per-position scale of ConvolveBorderColumn (b/butteraugli.cc:156-181); tiles that
// contain such outputs run a second streaming pass with the raw taps.
// All results are bit-identical to the generic functors in kernels.h (same products, same
// order of additions), which remain the CPU port's version and the reference for
// tests/test_gpu_parity.py::test_fused_matches_staged.
#pragma once
#include <cuda_runtime.h>

#include "ba_math.h"
#include "kernels.h"
#include "tma.cuh"

namespace gb200 {

template <int R>
struct BlurK {
  float n[2 * R + 1];    // taps * (1/sum): interior kernel
  float raw[2 * R + 1];  // raw taps: border rule
};

// Mixed-size launches (kernel template argument B = 2): the images of a pass have sizes of their own,
// each at most the batch's, in arena slots n0 .. n0 + m - 1 at the batch's pitch and plane size.
// The grid is one-dimensional over (image, tile) work items: image j owns items
// [tile0[j], tile0[j + 1]), its tiles in x-major, then y, then single-image z order.
#define GB_MIX_SHAPES 16  // distinct sizes per pass: tensor maps of each in the kernel parameters
struct MixImage {
  int w, h;
  int shape;   // index of its tensor maps in the pass's map sets
  int sx, sy;  // offsets of its border scales (x, y) in the pass's scale table of a blur
  int seg;       // rows of a rolling-blur segment (launch_roll's rule for h rows)
  int channels;  // bytes per pixel of an 8-bit image (k_mix_srgb); 3 for float planes
  int pad;       // 32 bytes
};
struct MixGeom {
  const MixImage* img;  // [m]
  const int* tile0;     // [m + 1] first work item of each image, for the launch's tile shape
  int m, n0;
};

struct PlaneGeom {
  int w, h, pitch;
  size_t plane;   // floats per plane
  int y0, y_end;  // rows [y0, y_end) are produced (strip mode computes a sub-range)
  // Batched launches (kernel template argument B): image n keeps its planes in arena slot n,
  // kslot planes (kslot * plane floats) after slot 0, so every pointer moves by n * kslot * plane
  // and every TMA plane coordinate by n * kslot.  The grid's z is n * zimg + (the single-image z).
  // The original's planes (ps0, sup0) move by kslot0 planes per image instead: kslot0 = kslot
  // when every image has its own original, 0 when all images are scored against one.
  // Single-image instantiations (B = 0) read none of these fields.
  int kslot, zimg, kslot0;
};
// the geometry argument of a mixed launch: the batch's, and the pass's images
struct PlaneGeomMix : PlaneGeom {
  MixGeom mix;
};
template <int B>
struct GeomArg {
  typedef PlaneGeom type;
};
template <>
struct GeomArg<2> {
  typedef PlaneGeomMix type;
};

// image index and single-image z of a block of a batched launch; (0, blockIdx.z) when B is 0
template <int B>
__device__ __forceinline__ int batch_image(const PlaneGeom& g) {
  return B ? static_cast<int>(blockIdx.z) / g.zimg : 0;
}

// A block's work item: arena slot, tile column, tile row, single-image z.
struct Item {
  int n;
  unsigned x, y, z;  // unsigned as blockIdx, so that B < 2 computes what it computed before
};
// the j with t0[j] <= v < t0[j + 1], for a non-decreasing t0[0 .. m] with t0[0] <= v < t0[m]
__device__ __forceinline__ int mix_find(const int* t0, int m, int v) {
  int lo = 0, hi = m;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(t0 + mid) <= v) {
      lo = mid;
    } else {
      hi = mid;
    }
  }
  return lo;
}
// Mixed launch: the item of this block, with g's w, h and rows made the image's; th = 0 takes the
// image's rolling-blur segment as the tile height.
__device__ __forceinline__ MixImage mix_item(PlaneGeomMix& g, int tw, int th, Item& it) {
  const int lin = blockIdx.x;
  const int* t0 = g.mix.tile0;
  const int lo = mix_find(t0, g.mix.m, lin);
  const MixImage im = g.mix.img[lo];
  const int tx = (im.w + tw - 1) / tw, tyh = th ? th : im.seg, ty = (im.h + tyh - 1) / tyh;
  int local = lin - __ldg(t0 + lo);
  it.n = g.mix.n0 + lo;
  it.x = local % tx;
  local /= tx;
  it.y = local % ty;
  it.z = local / ty;
  g.w = im.w;
  g.h = im.h;
  g.y0 = 0;
  g.y_end = im.h;
  return im;
}

// Tensor maps of a launch: one (B < 2), or one per distinct size of a mixed pass, with that size's
// true dims so that the TMA unit zero-fills at each image's own border.
struct MixMaps {
  CUtensorMap m[GB_MIX_SHAPES];
};
template <int B>
struct MapArg {
  typedef CUtensorMap type;
};
template <>
struct MapArg<2> {
  typedef MixMaps type;
};
__device__ __forceinline__ const CUtensorMap* map_of(const CUtensorMap& m, int) { return &m; }
__device__ __forceinline__ const CUtensorMap* map_of(const MixMaps& m, int shape) { return &m.m[shape]; }
__device__ __forceinline__ size_t slot_offset(const PlaneGeom& g, int n) {
  return static_cast<size_t>(n) * g.kslot * g.plane;
}
__device__ __forceinline__ size_t slot_offset0(const PlaneGeom& g, int n) {  // the original's planes
  return static_cast<size_t>(n) * g.kslot0 * g.plane;
}

// ---------------------------------------------------------------------------
// Streaming inner loops.  `acc` must be zero on entry.
//
// x: 4 adjacent outputs from an aligned run of float4 chunks.  The tile column of the
// thread's first chunk is 4*lane; output o uses samples at chunk-relative columns
// OFF + o + j, j = 0..2R.
template <int R, bool RAW>
__device__ __forceinline__ void stream_x4(const float* s, const BlurK<R>& k, float acc[4]) {
  constexpr int RP = (R + 3) & ~3, OFF = RP - R, NQ = (OFF + 2 * R + 3) / 4 + 1;
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const float4 v4 = *reinterpret_cast<const float4*>(s + 4 * q);
    const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
#pragma unroll
      for (int o = 0; o < 4; ++o) {
        const int j = 4 * q + e - OFF - o;  // compile-time after unrolling; ascending for every output
        if (j >= 0 && j <= 2 * R) acc[o] += v[e] * (RAW ? k.raw[j] : k.n[j]);
      }
    }
  }
}

// y: G consecutive rows of one column from a tile with row stride TW.
template <int R, int G, int TW, bool RAW>
__device__ __forceinline__ void stream_y(const float* s, const BlurK<R>& k, float acc[G]) {
#pragma unroll
  for (int t = 0; t < G + 2 * R; ++t) {
    const float v = s[t * TW];
#pragma unroll
    for (int o = 0; o < G; ++o) {
      const int j = t - o;
      if (j >= 0 && j <= 2 * R) acc[o] += v * (RAW ? k.raw[j] : k.n[j]);
    }
  }
}

template <int R>
struct XTile {
  static constexpr int RP = (R + 3) & ~3;
  static constexpr int OFF = RP - R;
  static constexpr int NQ = (OFF + 2 * R + 3) / 4 + 1;
};

// ---------------------------------------------------------------------------
// x pass: tile of GBX_TW x GBX_TH outputs, 128 threads; lane -> 4 adjacent columns,
// warp -> rows warp, warp + 4, ...   grid (ceil(w / TW), ceil(rows / TH), planes).
#define GBX_TW 128
#define GBX_TH 16
template <int R>
struct BlurXCfg {
  static constexpr int SW = GBX_TW - 4 + 4 * XTile<R>::NQ;  // tile row length (box width), multiple of 4
};

// body of the x pass for one tile; `tile` holds GBX_TH * BlurXCfg<R>::SW floats, `bar` one mbarrier
template <int R>
__device__ __forceinline__ void blur_x_tile(float* tile, uint64_t* bar, const CUtensorMap* in_map, float* out,
                                            const float* scale_x, const PlaneGeom& g, const BlurK<R>& k, int pl,
                                            int bx, int by) {
  constexpr int SW = BlurXCfg<R>::SW, RP = XTile<R>::RP;
  const int x0 = bx * GBX_TW, yb = g.y0 + by * GBX_TH;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, GBX_TH * SW * 4);
    tma_load_box(tile, in_map, bar, x0 - RP, yb, pl);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool edge = (x0 < R) || (x0 + GBX_TW + R > g.w);  // some output of this tile takes the border rule
  const int xb = x0 + 4 * lane;
  float* oplane = out + static_cast<size_t>(pl) * g.plane;
  mbar_wait(bar, 0);
#pragma unroll 1
  for (int r = warp; r < GBX_TH; r += 4) {
    const int y = yb + r;
    if (y >= g.y_end) break;
    const float* s = tile + r * SW + 4 * lane;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    stream_x4<R, false>(s, k, acc);
    float* orow = oplane + static_cast<size_t>(y) * g.pitch;
    if (!edge) {
      *reinterpret_cast<float4*>(orow + xb) = make_float4(acc[0], acc[1], acc[2], acc[3]);
      continue;
    }
    float raw[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    stream_x4<R, true>(s, k, raw);
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      const int x = xb + o;
      if (x >= g.w) continue;
      orow[x] = (x < R || x + R >= g.w) ? raw[o] * scale_x[x] : acc[o];
    }
  }
}

// Four single-plane x passes with different kernels in one launch (blockIdx.z picks the blur;
// batched: z = n * 4 + blur): the noise blur and the three mask blurs all become ready after
// hf_fused / mask_pre, and each alone is a one-wave launch whose ramp and tail cost as much as its
// arithmetic.
template <int R0, int R1, int R2, int R3>
struct BlurX4Args {
  float* out[4];
  const float* scale_x[4];
  BlurK<R0> k0;
  BlurK<R1> k1;
  BlurK<R2> k2;
  BlurK<R3> k3;
};

template <int B, int R0, int R1, int R2, int R3>
__global__ void __launch_bounds__(128) k_tma_blur_x4(const __grid_constant__ typename MapArg<B>::type m0,
                                                     const __grid_constant__ typename MapArg<B>::type m1,
                                                     const __grid_constant__ typename MapArg<B>::type m2,
                                                     const __grid_constant__ typename MapArg<B>::type m3,
                                                     typename GeomArg<B>::type g,
                                                     const __grid_constant__ BlurX4Args<R0, R1, R2, R3> a) {
  constexpr int RMAX = R0 > R1 ? (R0 > R2 ? (R0 > R3 ? R0 : R3) : (R2 > R3 ? R2 : R3))
                               : (R1 > R2 ? (R1 > R3 ? R1 : R3) : (R2 > R3 ? R2 : R3));
  __shared__ __align__(128) float tile[GBX_TH * BlurXCfg<RMAX>::SW];
  __shared__ __align__(8) uint64_t bar;
  Item it;
  int shape = 0, sx = 0;
  if constexpr (B == 2) {
    const MixImage im = mix_item(g, GBX_TW, GBX_TH, it);
    shape = im.shape;
    sx = im.sx;
  } else {
    it = Item{B ? static_cast<int>(blockIdx.z) >> 2 : 0, blockIdx.x, blockIdx.y,
              B ? blockIdx.z & 3 : blockIdx.z};
  }
  // the image's first plane: blur_x_tile takes it as the TMA plane and as the output plane
  const int pl = it.n * g.kslot;
  switch (it.z) {  // uniform per CTA
    case 0: blur_x_tile<R0>(tile, &bar, map_of(m0, shape), a.out[0], a.scale_x[0] + sx, g, a.k0, pl, it.x, it.y); break;
    case 1: blur_x_tile<R1>(tile, &bar, map_of(m1, shape), a.out[1], a.scale_x[1] + sx, g, a.k1, pl, it.x, it.y); break;
    case 2: blur_x_tile<R2>(tile, &bar, map_of(m2, shape), a.out[2], a.scale_x[2] + sx, g, a.k2, pl, it.x, it.y); break;
    default: blur_x_tile<R3>(tile, &bar, map_of(m3, shape), a.out[3], a.scale_x[3] + sx, g, a.k3, pl, it.x, it.y); break;
  }
}

// ---------------------------------------------------------------------------
// y pass with epilogue: tile of GBY_TW x GBY_TH outputs, 256 threads = 128 columns x
// 2 groups of 16 rows.  NP planes are blurred by the same thread (their tiles arrive
// together) and handed to the epilogue as v[NP] per pixel.
// grid (ceil(w / TW), ceil(rows / TH), NP == 1 ? planes : 1), times the images of a batched launch.
#define GBY_TW 128
#define GBY_TH 32
#define GBY_G 16

template <int B, int R, int NP, class Epi>
__global__ void __launch_bounds__(256, NP == 1 ? 3 : 2) k_tma_blur_y(const __grid_constant__ typename MapArg<B>::type in_map, const float* scale_y,
                                                    typename GeomArg<B>::type g, BlurK<R> k, Epi epi) {
  constexpr int HI = GBY_TH + 2 * R;
  extern __shared__ __align__(128) float dyn_smem[];
  float* tile = dyn_smem;                                                     // [NP][HI][TW]
  uint64_t* bar = reinterpret_cast<uint64_t*>(dyn_smem + NP * HI * GBY_TW);  // 8-byte aligned: sizes are multiples of 128 B
  Item it;
  int shape = 0;
  if constexpr (B == 2) {
    const MixImage im = mix_item(g, GBY_TW, GBY_TH, it);
    shape = im.shape;
    scale_y += im.sy;
  } else {
    const int n = batch_image<B>(g);
    it = Item{n, blockIdx.x, blockIdx.y, blockIdx.z - n * g.zimg};
  }
  const int n = it.n, pz = it.z;
  const int x0 = it.x * GBY_TW, yb = g.y0 + it.y * GBY_TH;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, NP * HI * GBY_TW * 4);
#pragma unroll
    for (int p = 0; p < NP; ++p)
      tma_load_box(tile + p * HI * GBY_TW, map_of(in_map, shape), bar, x0, yb - R, n * g.kslot + (NP == 1 ? pz : p));
  }
  const int c = threadIdx.x & (GBY_TW - 1), grp = threadIdx.x >> 7;
  const int x = x0 + c, yg = yb + GBY_G * grp;
  const bool edge = (yb < R) || (yb + GBY_TH + R > g.h);
  float res[NP][GBY_G];
  mbar_wait(bar, 0);
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    const float* s = tile + p * HI * GBY_TW + (GBY_G * grp) * GBY_TW + c;
#pragma unroll
    for (int o = 0; o < GBY_G; ++o) res[p][o] = 0.0f;
    stream_y<R, GBY_G, GBY_TW, false>(s, k, res[p]);
    if (edge) {
      float raw[GBY_G];
#pragma unroll
      for (int o = 0; o < GBY_G; ++o) raw[o] = 0.0f;
      stream_y<R, GBY_G, GBY_TW, true>(s, k, raw);
#pragma unroll
      for (int o = 0; o < GBY_G; ++o) {
        const int y = yg + o;
        if (y < g.h && (y < R || y + R >= g.h)) res[p][o] = raw[o] * scale_y[y];
      }
    }
  }
  constexpr int CH = Epi::kChunk;
  if (x >= g.w) return;
  // Epilogue in chunks: first every global operand of the chunk's pixels (read-only path,
  // all loads in flight together), then the arithmetic and the stores.
#pragma unroll
  for (int o0 = 0; o0 < GBY_G; o0 += CH) {
    typename Epi::Pre pre[CH];
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int y = yg + o0 + i;
      if (y < g.y_end) epi.load(x, y, n, pz, pre[i]);
    }
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int y = yg + o0 + i;
      if (y >= g.y_end) continue;
      float v[NP];
#pragma unroll
      for (int p = 0; p < NP; ++p) v[p] = res[p][o0 + i];
      epi.apply(x, y, n, pz, v, pre[i]);
    }
  }
}

// ---------------------------------------------------------------------------
// Rolling-window separable blur (large radii): x and y pass in one kernel, the x pass
// never leaves shared memory.  A CTA (128 threads) owns a GBR_TW-column strip of a
// segment of `seg` output rows [ys, ye) and walks it top to bottom in steps of GBR_CH rows:
//
//   chunk c   = input rows [ys - R + c*CH, +CH) with their x halo, one TMA box per plane,
//               in NS stages (one mbarrier each; the load of chunk c + NS is issued as soon
//               as the x pass of chunk c is done)
//   x pass    of chunk c -> ring position c % (RING / CH) of the x-output ring, with rows
//               0 .. 2R-1 of the ring also written at RING + i, so that every window of
//               CH + 2R ring rows is contiguous (stream_y's immediate-offset loads)
//   y pass    of step b = c - D (output rows [ys + b*CH, +CH)) from the ring; warp w owns
//               rows w*G .. w*G + G-1, lane = column; then the epilogue on the registers.
//
// D = ceil(2R / CH) chunks of look-ahead.  A ring of D + 2 chunks means the x pass of chunk
// c + 1 never overwrites rows the y pass of step c - D reads (one barrier per step); a ring of
// D + 1 chunks needs a second barrier (RollCfg::kLean).  The only recomputation is the D
// chunks of x rows above each segment.  Rows outside the image are zero-filled by the TMA
// unit (or, for chunks wholly below the image, written as zeros), so their x outputs are +0,
// as the y kernels' zero fill made them.
#define GBR_TW 32
#define GBR_CH 32
#define GBR_G 8    // 4 warps x 8 rows = GBR_CH
#define GBR_SEG 288  // target segment length: 4 segments of 1080 rows, recompute D*CH rows each

template <int R, int NP>
struct RollCfg {
  static constexpr int SW = GBR_TW - 4 + 4 * XTile<R>::NQ;  // input box width
  static constexpr int D = (2 * R + GBR_CH - 1) / GBR_CH;
  // Multi-plane (lean): one input stage and a ring of D + 1 chunks, so that four CTAs fit on
  // an SM; paid with a second barrier per step (the next x pass overwrites the rows the
  // current y pass reads).  Single plane: two stages, D + 2 chunks, one barrier per step.
  static constexpr bool kLean = NP > 1;
  static constexpr int NS = kLean ? 1 : 2;
  static constexpr int RING = (D + (kLean ? 1 : 2)) * GBR_CH;
  static constexpr int RBUF = RING + 2 * R;  // ring rows incl. the wrap copy
  static constexpr int kStageFloats = NP * GBR_CH * SW;
  static constexpr int kRingFloats = NP * RBUF * GBR_TW;
  static constexpr size_t kSmemBytes = (NS * kStageFloats + kRingFloats) * sizeof(float) + 16;
  static_assert(SW <= 256 && SW % 4 == 0, "TMA box width");
  static_assert((GBR_CH * SW * 4) % 128 == 0, "TMA destinations must be 128-byte aligned");
};

// x pass of one staged chunk (NP planes of CH rows) into ring rows [row0, row0 + CH) of each plane
template <int R, int NP>
__device__ __forceinline__ void roll_x_chunk(const float* st, float* ring, int row0, bool live, bool edge_x, int x0,
                                             const float* scale_x, int w, const BlurK<R>& k) {
  typedef RollCfg<R, NP> C;
  constexpr int SLOTS = GBR_TW / 4;
#pragma unroll 1
  for (int i = threadIdx.x; i < NP * GBR_CH * SLOTS; i += 128) {
    const int slot = i % SLOTS, prow = i / SLOTS;  // prow = p * CH + r
    const int p = prow / GBR_CH, r = prow % GBR_CH;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (live) {
      const float* s = st + prow * C::SW + 4 * slot;
      stream_x4<R, false>(s, k, acc);
      if (edge_x) {
        float raw[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        stream_x4<R, true>(s, k, raw);
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const int x = x0 + 4 * slot + o;
          // columns beyond the image only feed outputs that are never stored
          if (x < w && (x < R || x + R >= w)) acc[o] = raw[o] * scale_x[x];
        }
      }
    }
    const int rr = row0 + r;
    float* d = ring + (p * C::RBUF + rr) * GBR_TW + 4 * slot;
    const float4 v = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(d) = v;
    if (rr < 2 * R) *reinterpret_cast<float4*>(d + C::RING * GBR_TW) = v;
  }
}

// y pass of G rows of one column from the ring; s points at the window's first row
template <int R>
__device__ __forceinline__ void roll_y(const float* s, const BlurK<R>& k, const float* scale_y, int yg, int h,
                                       float res[GBR_G]) {
#pragma unroll
  for (int o = 0; o < GBR_G; ++o) res[o] = 0.0f;
  stream_y<R, GBR_G, GBR_TW, false>(s, k, res);
  if ((yg < R) || (yg + GBR_G + R > h)) {  // warp-uniform: some row of this group takes the border rule
    float raw[GBR_G];
#pragma unroll
    for (int o = 0; o < GBR_G; ++o) raw[o] = 0.0f;
    stream_y<R, GBR_G, GBR_TW, true>(s, k, raw);
#pragma unroll
    for (int o = 0; o < GBR_G; ++o) {
      const int y = yg + o;
      if (y < h && (y < R || y + R >= h)) res[o] = raw[o] * scale_y[y];
    }
  }
}

// NP planes blurred by the same thread and handed to the epilogue as v[NP] per pixel
// (NP == 1: blockIdx.z picks the plane).  grid (ceil(w / TW), ceil(rows / seg), NP == 1 ? planes : 1),
// times the images of a batched launch.
template <int B, int R, int NP, class Epi>
__global__ void __launch_bounds__(128) k_roll_blur(const __grid_constant__ typename MapArg<B>::type in_map_arg,
                                                   const float* scale_x, const float* scale_y, typename GeomArg<B>::type g, int seg,
                                                   BlurK<R> k, Epi epi) {
  typedef RollCfg<R, NP> C;
  constexpr int D = C::D, RP = XTile<R>::RP, NS = C::NS, NPOS = C::RING / GBR_CH;
  extern __shared__ __align__(128) float dyn_smem[];
  float* stage = dyn_smem;                        // [NS][NP][CH][SW]
  float* ring = dyn_smem + NS * C::kStageFloats;  // [NP][RBUF][TW]
  uint64_t* bar = reinterpret_cast<uint64_t*>(ring + C::kRingFloats);
  Item it;
  int shape = 0;
  if constexpr (B == 2) {
    const MixImage im = mix_item(g, GBR_TW, 0, it);
    shape = im.shape;
    seg = im.seg;
    scale_x += im.sx;
    scale_y += im.sy;
  } else {
    const int n = batch_image<B>(g);
    it = Item{n, blockIdx.x, blockIdx.y, blockIdx.z - n * g.zimg};
  }
  const CUtensorMap& in_map = *map_of(in_map_arg, shape);
  const int n = it.n, pl0 = n * g.kslot;  // image, its first TMA plane
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, pz = it.z;
  const int x0 = it.x * GBR_TW, x = x0 + lane;
  const int ys = g.y0 + it.y * seg;
  const int ye = min(ys + seg, g.y_end);
  const int nsteps = (ye - ys + GBR_CH - 1) / GBR_CH, nchunks = nsteps + D;
  const int yin = ys - R;  // first input row of chunk 0
  // chunks that start below the image are not loaded (their rows are zeros)
  const int nlive = min(nchunks, (g.h - yin + GBR_CH - 1) / GBR_CH);
  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    for (int c = 0; c < NS && c < nlive; ++c) {
      mbar_expect_tx(&bar[c], C::kStageFloats * 4);
#pragma unroll
      for (int p = 0; p < NP; ++p)
        tma_load_box(stage + c * C::kStageFloats + p * GBR_CH * C::SW, &in_map, &bar[c], x0 - RP, yin + c * GBR_CH,
                     pl0 + (NP == 1 ? pz : p));
    }
  }
  const bool edge_x = (x0 < R) || (x0 + GBR_TW + R > g.w);
#pragma unroll 1
  for (int c = 0; c < nchunks; ++c) {
    const int sidx = c % NS;
    const bool live = c < nlive;
    if (C::kLean && c > 0) __syncthreads();  // the y pass of the previous step is done with its rows
    if (live) mbar_wait(&bar[sidx], (c / NS) & 1);
    roll_x_chunk<R, NP>(stage + sidx * C::kStageFloats, ring, (c % NPOS) * GBR_CH, live, edge_x, x0, scale_x, g.w, k);
    __syncthreads();  // ring rows of chunk c complete; stage sidx free
    if (tid == 0 && c + NS < nlive) {
      mbar_expect_tx(&bar[sidx], C::kStageFloats * 4);
#pragma unroll
      for (int p = 0; p < NP; ++p)
        tma_load_box(stage + sidx * C::kStageFloats + p * GBR_CH * C::SW, &in_map, &bar[sidx], x0 - RP,
                     yin + (c + NS) * GBR_CH, pl0 + (NP == 1 ? pz : p));
    }
    if (c < D) continue;
    const int b = c - D;
    const int yg = ys + b * GBR_CH + GBR_G * warp;
    const float* win = ring + ((b % NPOS) * GBR_CH + GBR_G * warp) * GBR_TW + lane;
    float res[NP][GBR_G];
#pragma unroll
    for (int p = 0; p < NP; ++p) roll_y<R>(win + p * C::RBUF * GBR_TW, k, scale_y, yg, g.h, res[p]);
    if (x >= g.w) continue;
    // Epilogue: first every global operand of the G pixels (read-only path, all loads in
    // flight together), then the arithmetic and the stores.  One copy of G = 8 pixels is in
    // the instruction stream, inside the rolled step loop: as small as the rolled 8-pixel
    // chunks of the former multi-plane y kernel, so EpiMf's long epilogue fits the cache.
    static_assert(Epi::kChunk >= GBR_G, "the epilogue takes the G pixels of a thread in one chunk");
    typename Epi::Pre pre[GBR_G];
#pragma unroll
    for (int o = 0; o < GBR_G; ++o) {
      const int y = yg + o;
      if (y < ye) epi.load(x, y, n, pz, pre[o]);
    }
#pragma unroll
    for (int o = 0; o < GBR_G; ++o) {
      const int y = yg + o;
      if (y >= ye) continue;
      float v[NP];
#pragma unroll
      for (int p = 0; p < NP; ++p) v[p] = res[p][o];
      epi.apply(x, y, n, pz, v, pre[o]);
    }
  }
}

// ---------------------------------------------------------------------------
// Small radius (<= 5): x and y pass of NP planes in one kernel from one tile, epilogue
// on the registers.  Tile GB2_TW x GB2_TH outputs, 256 threads.
//   phase 1  x pass of all NP * (TH + 2R) tile rows -> tmp (shared), 4 outputs per item
//   phase 2  thread = column x group of 8 rows: y pass from tmp, then the epilogue, which
//            also sees the un-blurred samples of its pixel (`sharp`, from the input tile).
// grid (ceil(w / TW), ceil(rows / TH), 1), or (..., images) batched.
#define GB2_TW 64
#define GB2_TH 32
#define GB2_G 8

template <int R, int NP>
struct Blur2dCfg {
  static constexpr int SWI = GB2_TW - 4 + 4 * XTile<R>::NQ;  // input tile row length
  static constexpr int HI = GB2_TH + 2 * R;
  static constexpr int kInFloats = NP * HI * SWI;
  static constexpr int kTmpFloats = NP * HI * GB2_TW;
  static constexpr size_t kSmemBytes = (kInFloats + kTmpFloats) * sizeof(float) + 16;
  static_assert(NP == 1 || (HI * SWI * 4) % 128 == 0, "TMA destinations must be 128-byte aligned");
};

template <int B, int R, int NP, class Epi>
__global__ void __launch_bounds__(256) k_tma_blur_2d(const __grid_constant__ typename MapArg<B>::type in_map,
                                                     const float* scale_x, const float* scale_y, typename GeomArg<B>::type g,
                                                     BlurK<R> k, Epi epi) {
  typedef Blur2dCfg<R, NP> C;
  constexpr int SWI = C::SWI, HI = C::HI, RP = XTile<R>::RP;
  extern __shared__ __align__(128) float dyn_smem[];
  float* in = dyn_smem;                 // [NP][HI][SWI]
  float* tmp = dyn_smem + C::kInFloats;  // [NP][HI][TW]
  uint64_t* bar = reinterpret_cast<uint64_t*>(dyn_smem + C::kInFloats + C::kTmpFloats);
  Item it;
  int shape = 0;
  if constexpr (B == 2) {
    const MixImage im = mix_item(g, GB2_TW, GB2_TH, it);
    shape = im.shape;
    scale_x += im.sx;
    scale_y += im.sy;
  } else {
    it = Item{batch_image<B>(g), blockIdx.x, blockIdx.y, 0};
  }
  const int x0 = it.x * GB2_TW, yb = g.y0 + it.y * GB2_TH;
  const int tid = threadIdx.x, n = it.n;
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(bar, C::kInFloats * 4);
#pragma unroll
    for (int p = 0; p < NP; ++p)
      tma_load_box(in + p * HI * SWI, map_of(in_map, shape), bar, x0 - RP, yb - R, n * g.kslot + p);
  }
  const bool edge_x = (x0 < R) || (x0 + GB2_TW + R > g.w);
  const bool edge_y = (yb < R) || (yb + GB2_TH + R > g.h);
  mbar_wait(bar, 0);
  // phase 1
#pragma unroll 1
  for (int i = tid; i < NP * HI * (GB2_TW / 4); i += 256) {
    const int slot = i & (GB2_TW / 4 - 1), prow = i / (GB2_TW / 4);  // prow = p * HI + row
    const float* s = in + prow * SWI + 4 * slot;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    stream_x4<R, false>(s, k, acc);
    if (edge_x) {
      float raw[4] = {0.0f, 0.0f, 0.0f, 0.0f};
      stream_x4<R, true>(s, k, raw);
#pragma unroll
      for (int o = 0; o < 4; ++o) {
        const int x = x0 + 4 * slot + o;
        // columns beyond the image only feed outputs that are never stored
        if (x < g.w && (x < R || x + R >= g.w)) acc[o] = raw[o] * scale_x[x];
      }
    }
    *reinterpret_cast<float4*>(tmp + prow * GB2_TW + 4 * slot) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  }
  __syncthreads();
  // phase 2
  const int c = tid & (GB2_TW - 1), grp = tid >> 6;  // 4 groups of 8 rows
  const int x = x0 + c, yg = yb + GB2_G * grp;
  float res[NP][GB2_G];
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    const float* s = tmp + p * HI * GB2_TW + (GB2_G * grp) * GB2_TW + c;
#pragma unroll
    for (int o = 0; o < GB2_G; ++o) res[p][o] = 0.0f;
    stream_y<R, GB2_G, GB2_TW, false>(s, k, res[p]);
    if (edge_y) {
      float raw[GB2_G];
#pragma unroll
      for (int o = 0; o < GB2_G; ++o) raw[o] = 0.0f;
      stream_y<R, GB2_G, GB2_TW, true>(s, k, raw);
#pragma unroll
      for (int o = 0; o < GB2_G; ++o) {
        const int y = yg + o;
        if (y < g.h && (y < R || y + R >= g.h)) res[p][o] = raw[o] * scale_y[y];
      }
    }
  }
  const bool live_col = x < g.w;
  float carry = 0.0f;  // per-thread state of the epilogue across its 8 rows (EpiFinal: running block maximum)
  constexpr int CH = Epi::kChunk;
#pragma unroll
  for (int o0 = 0; o0 < GB2_G; o0 += CH) {
    typename Epi::Pre pre[CH];
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int y = yg + o0 + i;
      if (live_col && y < g.y_end) epi.load(x, y, n, pre[i]);
    }
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int o = o0 + i, y = yg + o;
      float v[NP], sharp[NP];
#pragma unroll
      for (int p = 0; p < NP; ++p) {
        v[p] = res[p][o];
        sharp[p] = in[(p * HI + R + GB2_G * grp + o) * SWI + RP + c];
      }
      // every thread calls the epilogue (it may contain warp-wide reductions); `live` tells
      // whether (x, y) is a pixel this launch must produce
      epi.apply(x, y, n, live_col && y < g.y_end, sharp, v, pre[i], carry);
    }
  }
}

// ---------------------------------------------------------------------------
// Epilogues.  Plane groups are addressed as base + n * slot + plane_index * g.plane + y * pitch + x,
// where n is the image of a batched launch (0 otherwise) and slot the floats per arena slot; the
// original's planes (ps0) as ps0 + n * slot0 + ..., slot0 = slot or 0 (PlaneGeom::kslot0).

// Each epilogue has two halves: load() fetches the pixel's global operands through the
// read-only path into a Pre, apply() does the arithmetic and the stores.  The kernels call
// load() for a chunk of kChunk pixels before the first apply(), so that the chunk's loads are
// in flight together instead of queueing behind one another's dependent stores.
struct NoPre {};

// plain store (stand-alone blur: tests, the one-time mask of the original); single image only
struct EpiStore {
  float* out;
  int pitch;
  size_t plane;
  typedef NoPre Pre;
  static constexpr int kChunk = 16;
  __device__ __forceinline__ void load(int, int, int, int, Pre&) const {}
  __device__ __forceinline__ void apply(int x, int y, int, int pz, const float v[1], const Pre&) const {
    out[pz * plane + static_cast<size_t>(y) * pitch + x] = v[0];
  }
};

// S2 (b/butteraugli.cc:509-513): lf = Blur(xyb); mf = xyb - lf, per plane.
struct EpiLf {
  const float* xyb;
  float* lf;
  float* mf_in;
  int pitch;
  size_t plane, slot;
  struct Pre {
    float a;
  };
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int x, int y, int n, int pz, Pre& p) const {
    p.a = __ldg(xyb + n * slot + pz * plane + static_cast<size_t>(y) * pitch + x);
  }
  __device__ __forceinline__ void apply(int x, int y, int n, int pz, const float v[1], const Pre& p) const {
    const size_t o = n * slot + pz * plane + static_cast<size_t>(y) * pitch + x;
    lf[o] = v[0];
    mf_in[o] = p.a - v[0];
  }
};

// S3 + S4 (SplitMfHf in kernels.h) on the three blurred mf planes of a pixel, plus the
// Malta pre-pass of the two mf bands (b/butteraugli.cc:1476-1529) when the PsychoImage
// of the original is given.
struct EpiMf {
  const float* mf_in;  // [3]
  float* ps;           // PsychoImage group being built
  float* hf_raw;       // [2]
  const float* ps0;    // original's PsychoImage, or nullptr (no Malta pre-pass)
  float* diffs;        // [6]: X uhf, hf, mf; Y uhf, hf, mf
  MaltaParams mp_x, mp_y;
  int pitch;
  size_t plane, slot, slot0;
  struct Pre {
    float inx, iny, p0x, p0y;
  };
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int x, int y, int n, int, Pre& p) const {
    const size_t r = static_cast<size_t>(y) * pitch + x, o = n * slot + r;
    p.inx = __ldg(mf_in + o);
    p.iny = __ldg(mf_in + plane + o);
    if (ps0 != nullptr) {
      const size_t o0 = n * slot0 + r;
      p.p0x = __ldg(ps0 + kMfX * plane + o0);
      p.p0y = __ldg(ps0 + kMfY * plane + o0);
    }
  }
  __device__ __forceinline__ void apply(int x, int y, int n, int, const float v[3], const Pre& p) const {
    const size_t o = n * slot + static_cast<size_t>(y) * pitch + x;
    const float mbx = v[0], mby = v[1];
    const float hx = p.inx - mbx;
    const float hy = p.iny - mby;
    const float mfx = remove_range_around_zero(static_cast<float>(0.120079806822), mbx);
    const float mfy = amplify_range_around_zero(static_cast<float>(0.03430529365), mby);
    hf_raw[o] = suppress_x_by_y(hx, hy);
    hf_raw[plane + o] = hy;
    // the candidate's mf planes are consumed here (Malta pre-pass) and nowhere else: stored
    // only when building a full PsychoImage
    if (ps0 == nullptr) {
      ps[kMfX * plane + o] = mfx;
      ps[kMfY * plane + o] = mfy;
      ps[kMfB * plane + o] = v[2];
    } else {
      diffs[2 * plane + o] = malta_diff(p.p0x, mfx, mp_x);
      diffs[5 * plane + o] = malta_diff(p.p0y, mfy, mp_y);
    }
  }
};

// S1 (b/butteraugli.cc:337-362): sensitivity from the blurred pixel, applied to the sharp one.
struct EpiOpsin {
  float* xyb;
  int pitch;
  size_t plane, slot;
  typedef NoPre Pre;
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int, int, int, Pre&) const {}
  __device__ __forceinline__ void apply(int x, int y, int n, bool live, const float sharp[3], const float v[3], const Pre&,
                                        float&) const {
    if (!live) return;
    const size_t o = n * slot + static_cast<size_t>(y) * pitch + x;
    opsin_pixel(sharp[0], sharp[1], sharp[2], v[0], v[1], v[2], &xyb[o], &xyb[plane + o], &xyb[2 * plane + o]);
  }
};

// S5 + S6 (SplitHfUhf in kernels.h) on the two blurred hf planes, plus -- against the
// original's PsychoImage -- the Malta pre-pass of the uhf and hf bands of both channels and
// the SameNoiseLevels difference (b/butteraugli.cc:624-640, NoisePre in kernels.h).
struct EpiHf {
  const float* lf_raw;  // [3] blurred xyb
  float* ps;
  const float* ps0;     // or nullptr
  float* diffs;         // [6]
  float* noise;         // [1]
  MaltaParams mp_uhf_x, mp_uhf_y, mp_hf_x, mp_hf_y;
  int pitch;
  size_t plane, slot, slot0;
  struct Pre {
    float lfx, lfy, lfb, u0x, h0x, u0y, h0y;
  };
  static constexpr int kChunk = 4;
  __device__ __forceinline__ void load(int x, int y, int n, Pre& p) const {
    const size_t r = static_cast<size_t>(y) * pitch + x, o = n * slot + r;
    p.lfx = __ldg(lf_raw + o);
    p.lfy = __ldg(lf_raw + plane + o);
    p.lfb = __ldg(lf_raw + 2 * plane + o);
    if (ps0 != nullptr) {
      const size_t o0 = n * slot0 + r;
      p.u0x = __ldg(ps0 + kUhfX * plane + o0);
      p.h0x = __ldg(ps0 + kHfX * plane + o0);
      p.u0y = __ldg(ps0 + kUhfY * plane + o0);
      p.h0y = __ldg(ps0 + kHfY * plane + o0);
    }
  }
  __device__ __forceinline__ void apply(int x, int y, int n, bool live, const float sharp[2], const float v[2],
                                        const Pre& p, float&) const {
    if (!live) return;
    const size_t o = n * slot + static_cast<size_t>(y) * pitch + x;
    const float uhfx = sharp[0] - v[0];
    const float hfx = remove_range_around_zero(static_cast<float>(0.0287615200377), v[0]);
    const float lfx = p.lfx, lfy = p.lfy, lfb = p.lfb;
    const float kMulSuppressHf = static_cast<float>(1.10684769012);
    const float kMulRegHf = static_cast<float>(0.478741530298);
    const float kRegHf = 2000 * kMulRegHf;
    const float kMulSuppressUhf = static_cast<float>(1.76905001176);
    const float kMulRegUhf = static_cast<float>(0.310148420674);
    const float kRegUhf = 2000 * kMulRegUhf;
    float uhfy = sharp[1] - v[1];
    float hfy = maximum_clamp(v[1], static_cast<float>(78.8223237675));
    uhfy = maximum_clamp(uhfy, static_cast<float>(5.8907152736));
    uhfy = suppress_in_bright_areas(uhfy, lfy, kMulSuppressUhf, kRegUhf);
    hfy = suppress_in_bright_areas(hfy, lfy, kMulSuppressHf, kRegHf);
    // against the original (ps0 given), uhf[X] and lf[Y] of the candidate are consumed here
    // only; k_mask_pre reads hf[X], uhf[Y], hf[Y], the noise epilogue hf[Y], the combine lf[X], lf[B]
    ps[kHfX * plane + o] = hfx;
    ps[kUhfY * plane + o] = uhfy;
    ps[kHfY * plane + o] = hfy;
    const float xmul = static_cast<float>(5.57547552483);
    const float ymul = static_cast<float>(1.20828034498);
    const float bmul = static_cast<float>(6.08319517575);
    const float y_to_b_mul = static_cast<float>(-0.628811683685);
    const float bb = lfb + y_to_b_mul * lfy;
    ps[kLfB * plane + o] = bb * bmul;
    ps[kLfX * plane + o] = lfx * xmul;
    if (ps0 == nullptr) {
      ps[kUhfX * plane + o] = uhfx;
      ps[kLfY * plane + o] = lfy * ymul;
    } else {
      const float h0y = p.h0y;
      diffs[0 * plane + o] = malta_diff(p.u0x, uhfx, mp_uhf_x);
      diffs[1 * plane + o] = malta_diff(p.h0x, hfx, mp_hf_x);
      diffs[3 * plane + o] = malta_diff(p.u0y, uhfy, mp_uhf_y);
      diffs[4 * plane + o] = malta_diff(h0y, hfy, mp_hf_y);
      const double maxclamp = 85.7047444518;
      double v0 = hd_fabsf(h0y);
      double v1 = hd_fabsf(hfy);
      if (v0 > maxclamp) v0 = maxclamp;
      if (v1 > maxclamp) v1 = maxclamp;
      noise[o] = static_cast<float>(v0 - v1);
    }
  }
};

// S8 tail + S9 (NoiseAndAsymAcc in kernels.h) on the blurred noise difference.
struct EpiNoise {
  const float* hf0;  // pi0.hf[Y]
  const float* hf1;  // pi1.hf[Y]
  float* acc;        // block_diff_ac[Y], read-modify-write (each pixel by exactly one thread)
  double w_0gt1, w_0lt1;
  int pitch;
  size_t slot, slot0;
  struct Pre {
    float r0, r1, a;
  };
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int x, int y, int n, int, Pre& p) const {
    const size_t r = static_cast<size_t>(y) * pitch + x, o = n * slot + r;
    p.r0 = __ldg(hf0 + n * slot0 + r);
    p.r1 = __ldg(hf1 + o);
    p.a = acc[o];  // plain load: this launch writes the location later (same thread)
  }
  __device__ __forceinline__ void apply(int x, int y, int n, int, const float v[1], const Pre& p) const {
    const size_t o = n * slot + static_cast<size_t>(y) * pitch + x;
    float a = p.a;
    {
      const double w = 884.809801415;
      const double diff = v[0];
      a = static_cast<float>(static_cast<double>(a) + w * diff * diff);
    }
    const float r0 = p.r0, r1f = p.r1;
    const double diff = r0 - r1f;  // float subtraction, then widened
    a = static_cast<float>(static_cast<double>(a) + w_0gt1 * diff * diff);
    const double fabs0 = hd_fabsf(r0);
    const double too_small = 0.4 * fabs0;
    const double too_big = 1.0 * fabs0;
    const double r1 = r1f;
    if (r0 < 0) {
      if (r1 > -too_small) {
        const double t = r1 + too_small;
        a = static_cast<float>(static_cast<double>(a) + w_0lt1 * t * t);
      } else if (r1 < -too_big) {
        const double t = -r1 - too_big;
        a = static_cast<float>(static_cast<double>(a) + w_0lt1 * t * t);
      }
    } else {
      if (r1 < too_small) {
        const double t = too_small - r1;
        a = static_cast<float>(static_cast<double>(a) + w_0lt1 * t * t);
      } else if (r1 > too_big) {
        const double t = r1 - too_big;
        a = static_cast<float>(static_cast<double>(a) + w_0lt1 * t * t);
      }
    }
    acc[o] = a;
  }
};

// S12 second half + S13 (DiffmapMix, BlockMax in kernels.h): the blurred sqrt-diffmap is
// mixed with the sharp one; the lanes of an 8x8 block reduce their maximum with warp
// shuffles (a thread holds 8 rows of one column, 8 adjacent lanes hold the block's
// columns), and one lane per block stores it and folds it into the global maximum
// (non-negative floats order like their bit patterns).  Image n of a batch has its own
// block_max (n * nblocks on) and global maximum (gmax[n]).
struct EpiFinal {
  float* distmap;
  float* block_max;     // [nblocks], written for block rows [by_lo, by_hi)
  unsigned int* gmax;   // global maximum (float bits), or nullptr
  int pitch, bw, by_lo, by_hi;
  size_t slot;
  int nblocks;
  typedef NoPre Pre;
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int, int, int, Pre&) const {}
  // m: running maximum of the thread's pixels of the current block row (one block column)
  __device__ __forceinline__ void apply(int x, int y, int n, bool live, const float sharp[1], const float v[1],
                                        const Pre&, float& m) const {
    if (live) {
      const double mul1 = 0.458794906198;
      const float scale = static_cast<float>(1.0f / (1.0f + mul1));
      float d = static_cast<float>(static_cast<double>(sharp[0]) + mul1 * v[0]);
      d *= scale;
      distmap[n * slot + static_cast<size_t>(y) * pitch + x] = d;
      m = (y & 7) == 0 ? hd_max(0.0f, d) : hd_max(m, d);
    } else if ((y & 7) == 0) {
      m = 0.0f;
    }
    if ((y & 7) == 7) {
      float b = m;
      b = hd_max(b, __shfl_xor_sync(0xffffffffu, b, 1));
      b = hd_max(b, __shfl_xor_sync(0xffffffffu, b, 2));
      b = hd_max(b, __shfl_xor_sync(0xffffffffu, b, 4));
      const int by = y >> 3, bx = x >> 3;
      if ((x & 7) == 0 && bx < bw && by >= by_lo && by < by_hi) {
        (block_max + static_cast<size_t>(n) * nblocks)[by * bw + bx] = b;
        if (gmax != nullptr) atomicMax(gmax + n, __float_as_uint(b));
      }
    }
  }
};

// ---------------------------------------------------------------------------
// S10 y passes + S11 + first half of S12: the three mask blurs (X with r = RA, Y with
// r = RB and r = RC) finish in one kernel whose epilogue is CombineAndSqrt (kernels.h).
template <int RA, int RB, int RC>
struct MaskYCfg {
  static constexpr int HA = GBY_TH + 2 * RA, HB = GBY_TH + 2 * RB, HC = GBY_TH + 2 * RC;
  static constexpr size_t kSmemBytes = static_cast<size_t>(HA + HB + HC) * GBY_TW * sizeof(float) + 16;
};

template <int R, bool RAW_PASS>
__device__ __forceinline__ void mask_y_plane(const float* s, const BlurK<R>& k, const float* scale_y, int yg, int h,
                                             bool edge, float res[GBY_G]) {
#pragma unroll
  for (int o = 0; o < GBY_G; ++o) res[o] = 0.0f;
  stream_y<R, GBY_G, GBY_TW, false>(s, k, res);
  if (edge) {
    float raw[GBY_G];
#pragma unroll
    for (int o = 0; o < GBY_G; ++o) raw[o] = 0.0f;
    stream_y<R, GBY_G, GBY_TW, true>(s, k, raw);
#pragma unroll
    for (int o = 0; o < GBY_G; ++o) {
      const int y = yg + o;
      if (y < h && (y < R || y + R >= h)) res[o] = raw[o] * scale_y[y];
    }
  }
}

struct CombineArgs {
  const float* ps0;
  const float* ps1;
  const float* ac;  // [2]
  float* out;       // sqrt-diffmap
  const double* luts;
  int pitch;
  size_t plane;
};

// grid (ceil(w / TW), ceil(rows / TH), 1), or (..., images) batched.
template <int B, int RA, int RB, int RC>
__global__ void __launch_bounds__(256) k_tma_mask_y(const __grid_constant__ typename MapArg<B>::type map_a,
                                                    const __grid_constant__ typename MapArg<B>::type map_b,
                                                    const __grid_constant__ typename MapArg<B>::type map_c,
                                                    const float* sya, const float* syb, const float* syc, typename GeomArg<B>::type g,
                                                    BlurK<RA> ka, BlurK<RB> kb, BlurK<RC> kc, CombineArgs ca) {
  typedef MaskYCfg<RA, RB, RC> C;
  extern __shared__ __align__(128) float dyn_smem[];
  float* ta = dyn_smem;
  float* tb = ta + C::HA * GBY_TW;
  float* tc = tb + C::HB * GBY_TW;
  uint64_t* bar = reinterpret_cast<uint64_t*>(tc + C::HC * GBY_TW);
  Item it;
  int shape = 0;
  if constexpr (B == 2) {
    const MixImage im = mix_item(g, GBY_TW, GBY_TH, it);
    shape = im.shape;
    sya += im.sy;
    syb += im.sy;
    syc += im.sy;
  } else {
    it = Item{batch_image<B>(g), blockIdx.x, blockIdx.y, 0};
  }
  const int x0 = it.x * GBY_TW, yb = g.y0 + it.y * GBY_TH;
  const int n = it.n;
  const size_t so = slot_offset(g, n), so0 = slot_offset0(g, n);
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, (C::HA + C::HB + C::HC) * GBY_TW * 4);
    tma_load_box(ta, map_of(map_a, shape), bar, x0, yb - RA, n * g.kslot);
    tma_load_box(tb, map_of(map_b, shape), bar, x0, yb - RB, n * g.kslot);
    tma_load_box(tc, map_of(map_c, shape), bar, x0, yb - RC, n * g.kslot);
  }
  const int c = threadIdx.x & (GBY_TW - 1), grp = threadIdx.x >> 7;
  const int x = x0 + c, yg = yb + GBY_G * grp;
  float sx[GBY_G], sy1[GBY_G], sy2[GBY_G];
  mbar_wait(bar, 0);
  mask_y_plane<RA, false>(ta + (GBY_G * grp) * GBY_TW + c, ka, sya, yg, g.h, (yb < RA) || (yb + GBY_TH + RA > g.h), sx);
  mask_y_plane<RB, false>(tb + (GBY_G * grp) * GBY_TW + c, kb, syb, yg, g.h, (yb < RB) || (yb + GBY_TH + RB > g.h), sy1);
  mask_y_plane<RC, false>(tc + (GBY_G * grp) * GBY_TW + c, kc, syc, yg, g.h, (yb < RC) || (yb + GBY_TH + RC > g.h), sy2);
  // The three activities go back to shared memory (over the input tiles, which are dead once
  // every thread has finished its passes), each thread into slots only it reads again: the
  // epilogue below can then be a rolled loop instead of 16 unrolled copies of the LUT code.
  __syncthreads();
  float* stash = dyn_smem + threadIdx.x;  // [3][GBY_G][256]
#pragma unroll
  for (int o = 0; o < GBY_G; ++o) {
    stash[(0 * GBY_G + o) * 256] = sx[o];
    stash[(1 * GBY_G + o) * 256] = sy1[o];
    stash[(2 * GBY_G + o) * 256] = sy2[o];
  }
  if (x >= g.w) return;
  CombineAndSqrt comb;
  comb.ps0 = ca.ps0 + so0;
  comb.ps1 = ca.ps1 + so;
  comb.ac = ca.ac + so;
  comb.out = ca.out + so;
  comb.luts = ca.luts;
  comb.g.pitch = ca.pitch;
  comb.g.plane = ca.plane;
  constexpr int CH = 4;
#pragma unroll 1
  for (int o0 = 0; o0 < GBY_G; o0 += CH) {
    float l0x[CH], l0b[CH], l1x[CH], l1b[CH], acx[CH], acy[CH];
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int y = yg + o0 + i;
      if (y >= g.y_end) continue;
      const size_t r = static_cast<size_t>(y) * ca.pitch + x, o = so + r, o0 = so0 + r;
      l0x[i] = __ldg(ca.ps0 + kLfX * ca.plane + o0);
      l0b[i] = __ldg(ca.ps0 + kLfB * ca.plane + o0);
      l1x[i] = __ldg(ca.ps1 + kLfX * ca.plane + o);
      l1b[i] = __ldg(ca.ps1 + kLfB * ca.plane + o);
      acx[i] = __ldg(ca.ac + o);
      acy[i] = __ldg(ca.ac + ca.plane + o);
    }
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int y = yg + o0 + i;
      if (y >= g.y_end) continue;
      comb.pixel_with(x, y, stash[(0 * GBY_G + o0 + i) * 256], stash[(1 * GBY_G + o0 + i) * 256],
                      stash[(2 * GBY_G + o0 + i) * 256], l0x[i], l0b[i], l1x[i], l1b[i], acx[i], acy[i]);
    }
  }
}

// ---------------------------------------------------------------------------
// S7 Malta line sums of both colour channels in one launch (b/butteraugli.cc:1429-1568;
// MaltaUnit :914, :1146).  The "diffs" planes (pre-pass, written by EpiMf / EpiHf) are
// copied as 72 x 40 boxes by the TMA unit, double-buffered over the three bands; the zero
// fill outside the image is PaddedMaltaUnit's padding.  Line sums as in k_malta_sums
// (tiled_kernels.cuh): a thread evaluates 2 x 4 pixels from a 9 x 12 register window.
// grid (ceil(w / 64), ceil(rows / 32), 2 channels), times the images of a batched launch; 256 threads.
template <int B>
__global__ void __launch_bounds__(256, 2) k_tma_malta_sums(const __grid_constant__ typename MapArg<B>::type diffs_map_arg,
                                                           float* acc, typename GeomArg<B>::type g) {
  __shared__ __align__(128) float tile[2][GB_MALTA_SH * GB_MALTA_SW];
  __shared__ __align__(8) uint64_t bar[2];
  const int tx = threadIdx.x, ty = threadIdx.y;  // 16 x 16
  const int tid = ty * 16 + tx;
  Item it;
  int shape = 0;
  if constexpr (B == 2) {
    shape = mix_item(g, GB_MALTA_TILE_W, GB_MALTA_TILE_H, it).shape;
  } else {
    it = Item{B ? static_cast<int>(blockIdx.z) >> 1 : 0, blockIdx.x, blockIdx.y,
              B ? blockIdx.z & 1 : blockIdx.z};
  }
  const CUtensorMap& diffs_map = *map_of(diffs_map_arg, shape);
  const int n = it.n;
  const int x0 = it.x * GB_MALTA_TILE_W, y0 = g.y0 + it.y * GB_MALTA_TILE_H;
  const int ch = it.z, pl = n * g.kslot + 3 * ch;  // first plane of the channel's bands
  constexpr uint32_t kBytes = GB_MALTA_SH * GB_MALTA_SW * 4;
  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(&bar[0], kBytes);
    tma_load_box(tile[0], &diffs_map, &bar[0], x0 - 4, y0 - 4, pl + 0);
    mbar_expect_tx(&bar[1], kBytes);
    tma_load_box(tile[1], &diffs_map, &bar[1], x0 - 4, y0 - 4, pl + 1);
  }
  float r[2][4];
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int p = 0; p < 4; ++p) r[k][p] = 0.0f;
  // band 0 (uhf, 9-tap lines) from buffer 0
  mbar_wait(&bar[0], 0);
  malta_window_sums(tile[0], tx, ty, true, r);
  __syncthreads();  // everybody is done with buffer 0
  if (tid == 0) {
    mbar_expect_tx(&bar[0], kBytes);
    tma_load_box(tile[0], &diffs_map, &bar[0], x0 - 4, y0 - 4, pl + 2);
  }
  // band 1 (hf) from buffer 1, band 2 (mf) from buffer 0 again
  mbar_wait(&bar[1], 0);
  malta_window_sums(tile[1], tx, ty, false, r);
  mbar_wait(&bar[0], 1);
  malta_window_sums(tile[0], tx, ty, false, r);
  const int xb = x0 + 4 * tx;
  float* aplane = acc + slot_offset(g, n) + static_cast<size_t>(ch) * g.plane;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int y = y0 + ty + 16 * k;
    if (y >= g.y_end || xb >= g.w) continue;
    float* orow = aplane + static_cast<size_t>(y) * g.pitch + xb;
    if (xb + 3 < g.w) {
      *reinterpret_cast<float4*>(orow) = make_float4(r[k][0], r[k][1], r[k][2], r[k][3]);
    } else {
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (xb + p < g.w) orow[p] = r[k][p];
    }
  }
}

// ---------------------------------------------------------------------------
// S10 DiffPrecompute (b/butteraugli.cc:1699-1739; MaskDiffPre in kernels.h).  The
// original's half of the min() does not change during the search: sup0 is computed once
// per image (k_mask_sup, which also serves Mask(xyb0, xyb0) of StartBlockComparisons) and
// only the candidate's neighbour differences are formed per Compare.
// X combines (0 * uhf + b * hf): the uhf term only contributes a signed zero that the
// differences below cannot see, so the X channel reads hf alone.
__device__ __forceinline__ float mask_combo_x(float hf) { return static_cast<float>(0.0 * 0.0 + 1.64178305129 * hf); }
__device__ __forceinline__ float mask_combo_y(float uhf, float hf) {
  return static_cast<float>(0.831081703362 * uhf + 3.23680933546 * hf);
}

// sup = |v - v_right| + |v - v_down| (float magnitudes, float sum, widened by the consumer),
// neighbours mirrored at the last column / row; one plane per channel: sup[0] = X, sup[1] = Y.
// grid (ceil(w / 32), ceil(rows / 8), 1), or (..., images) batched; 32 x 8 threads.
// 32 x 8 tiles of k_mask_sup / k_mask_pre; B < 2 leaves the image to image_of (after the kernel's early exit)
template <int B>
__device__ __forceinline__ Item px_item(typename GeomArg<B>::type& g) {
  Item it;
  if constexpr (B == 2) {
    mix_item(g, 32, 8, it);
  } else {
    it = Item{0, blockIdx.x, blockIdx.y, 0};
  }
  return it;
}
template <int B>
__device__ __forceinline__ int image_of(const Item& it, const typename GeomArg<B>::type& g) {
  return B == 2 ? it.n : batch_image<B>(g);
}

template <int B>
__global__ void __launch_bounds__(256) k_mask_sup(const float* ps, float* sup, typename GeomArg<B>::type g) {
  const Item it = px_item<B>(g);
  const int x = it.x * 32 + threadIdx.x, y = g.y0 + it.y * 8 + threadIdx.y;
  if (x >= g.w || y >= g.y_end) return;
  const size_t so = slot_offset(g, image_of<B>(it, g));
  ps += so;
  sup += so;
  const int x2 = (x + 1 < g.w) ? x + 1 : (x > 0 ? x - 1 : x);
  const int y2 = (y + 1 < g.h) ? y + 1 : (y > 0 ? y - 1 : y);
  const size_t o = static_cast<size_t>(y) * g.pitch + x;
  const size_t ox = static_cast<size_t>(y) * g.pitch + x2;
  const size_t oy = static_cast<size_t>(y2) * g.pitch + x;
  const float* hx = ps + kHfX * g.plane;
  const float* uy = ps + kUhfY * g.plane;
  const float* hy = ps + kHfY * g.plane;
  const float a = mask_combo_x(hx[o]), ax = mask_combo_x(hx[ox]), ay = mask_combo_x(hx[oy]);
  const float b = mask_combo_y(uy[o], hy[o]), bx = mask_combo_y(uy[ox], hy[ox]), by = mask_combo_y(uy[oy], hy[oy]);
  sup[o] = hd_fabsf(a - ax) + hd_fabsf(a - ay);
  sup[g.plane + o] = hd_fabsf(b - bx) + hd_fabsf(b - by);
}

// mpre[c] = min(cutoff, mul0 * min(sup0_c, sup1_c)) for c = X, Y.  Grid as k_mask_sup.
template <int B>
__global__ void __launch_bounds__(256) k_mask_pre(const float* ps1, const float* sup0, float* mpre, typename GeomArg<B>::type g) {
  const Item it = px_item<B>(g);
  const int x = it.x * 32 + threadIdx.x, y = g.y0 + it.y * 8 + threadIdx.y;
  if (x >= g.w || y >= g.y_end) return;
  const int n = image_of<B>(it, g);
  const size_t so = slot_offset(g, n);
  ps1 += so;
  sup0 += slot_offset0(g, n);
  mpre += so;
  const int x2 = (x + 1 < g.w) ? x + 1 : (x > 0 ? x - 1 : x);
  const int y2 = (y + 1 < g.h) ? y + 1 : (y > 0 ? y - 1 : y);
  const size_t o = static_cast<size_t>(y) * g.pitch + x;
  const size_t ox = static_cast<size_t>(y) * g.pitch + x2;
  const size_t oy = static_cast<size_t>(y2) * g.pitch + x;
  const float* hx = ps1 + kHfX * g.plane;
  const float* uy = ps1 + kUhfY * g.plane;
  const float* hy = ps1 + kHfY * g.plane;
  const double mul0 = 0.918416534734;
  const double cutoff = 55.0184555849;
  {
    const float a = mask_combo_x(hx[o]), ax = mask_combo_x(hx[ox]), ay = mask_combo_x(hx[oy]);
    const double sup1 = hd_fabsf(a - ax) + hd_fabsf(a - ay);
    const double s0 = sup0[o];
    float v = static_cast<float>(mul0 * hd_min(s0, sup1));
    if (v >= cutoff) v = static_cast<float>(cutoff);
    mpre[o] = v;
  }
  {
    const float b = mask_combo_y(uy[o], hy[o]), bx = mask_combo_y(uy[ox], hy[ox]), by = mask_combo_y(uy[oy], hy[oy]);
    const double sup1 = hd_fabsf(b - bx) + hd_fabsf(b - by);
    const double s0 = sup0[g.plane + o];
    float v = static_cast<float>(mul0 * hd_min(s0, sup1));
    if (v >= cutoff) v = static_cast<float>(cutoff);
    mpre[g.plane + o] = v;
  }
}

// ---------------------------------------------------------------------------
// Mixed-size calls: rows between the caller's packed images and the arena, all images of a pass in
// one launch.  Image j has rows [row0[j], row0[j + 1]) of w floats at ext[j] (3h of its RGB planes,
// or h of its diffmap); row r of it is row r % h of plane r / h of arena slot n0 + j.  A warp per
// row, 8 rows per block.
template <bool TO_ARENA>
__global__ void __launch_bounds__(256) k_mix_rows(float* const* ext, const int* row0, float* arena, PlaneGeomMix g) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= __ldg(row0 + g.mix.m)) return;
  const int j = mix_find(row0, g.mix.m, row);
  const int w = g.mix.img[j].w, h = g.mix.img[j].h;
  const int r = row - __ldg(row0 + j), c = r / h, y = r - c * h;
  float* a = arena + slot_offset(g, g.mix.n0 + j) + c * g.plane + static_cast<size_t>(y) * g.pitch;
  float* e = ext[j] + static_cast<size_t>(r) * w;
  for (int x = lane; x < w; x += 32) {
    if (TO_ARENA) {
      a[x] = e[x];
    } else {
      e[x] = a[x];
    }
  }
}

// The same packing for 8-bit images, converted on the way (srgb_over_linear, over `background`): image j
// has rows [row0[j], row0[j + 1]), h of them, of w pixels of MixImage::channels bytes at src[j].  Row y
// is read once and written to row y of all three planes of arena slot n0 + j.  A warp per row, 8 rows
// per block.
__global__ void __launch_bounds__(256) k_mix_srgb(const uint8_t* const* src, const int* row0, int background,
                                                  const float* lut, float* arena, PlaneGeomMix g) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= __ldg(row0 + g.mix.m)) return;
  const int j = mix_find(row0, g.mix.m, row);
  const int w = g.mix.img[j].w, C = g.mix.img[j].channels;
  const int y = row - __ldg(row0 + j);
  float* a = arena + slot_offset(g, g.mix.n0 + j) + static_cast<size_t>(y) * g.pitch;
  const uint8_t* s = src[j] + static_cast<size_t>(y) * w * C;
  for (int x = lane; x < w; x += 32) srgb_over_linear(s + x * C, C, background, lut, a + x, g.plane);
}

// Comparator sets: an original's analysis between the set's store and arena slot n0 + j, all images of a
// pass in one launch.  Image j has rows [row0[j], row0[j + 1]), kStoredPlanes * h of them, of w floats at
// store[j]; row r is row r % h of stored plane r / h.  The stored planes are the eight of ps0 that the
// Compare chain reads (EpiMf: mf X, Y; EpiHf: uhf, hf of X and Y; EpiNoise: hf Y; CombineArgs: lf X, B),
// then sup0's two.  TO_ARENA: the gather before a Compare; else the store after the analysis.  A warp per
// row, 8 rows per block; float4 where the row is 16-byte aligned on both sides (arena rows always are: the
// pitch is a multiple of 32 floats; store rows are where w is a multiple of 4).
static_assert(kUhfX == 0 && kUhfY == 1 && kHfX == 2 && kHfY == 3 && kMfX == 4 && kMfY == 5 && kLfX == 7 &&
                  kLfB == 9,
              "stored plane c < 6 is ps0 plane c, 6 and 7 are lf X and lf B");
template <bool TO_ARENA>
__global__ void __launch_bounds__(256) k_mix_original(float* const* store, const int* row0, float* ps0, float* sup0,
                                                      PlaneGeomMix g) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= __ldg(row0 + g.mix.m)) return;
  const int j = mix_find(row0, g.mix.m, row);
  const int w = g.mix.img[j].w, h = g.mix.img[j].h;
  const int r = row - __ldg(row0 + j), c = r / h, y = r - c * h;
  const int pl = c < 6 ? c : c < 8 ? 2 * c - 5 : c - 8;
  float* a = (c < 8 ? ps0 : sup0) + slot_offset(g, g.mix.n0 + j) + pl * g.plane + static_cast<size_t>(y) * g.pitch;
  float* e = store[j] + static_cast<size_t>(r) * w;
  if (((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(e)) & 15) == 0 && (w & 3) == 0) {
    float4* a4 = reinterpret_cast<float4*>(a);
    float4* e4 = reinterpret_cast<float4*>(e);
    for (int x = lane; x < (w >> 2); x += 32) {
      if (TO_ARENA) {
        a4[x] = e4[x];
      } else {
        e4[x] = a4[x];
      }
    }
    return;
  }
  for (int x = lane; x < w; x += 32) {
    if (TO_ARENA) {
      a[x] = e[x];
    } else {
      e[x] = a[x];
    }
  }
}

}  // namespace gb200
