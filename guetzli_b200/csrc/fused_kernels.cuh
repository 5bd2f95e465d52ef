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

struct PlaneGeom {
  int w, h, pitch;
  size_t plane;   // floats per plane
  int y0, y_end;  // rows [y0, y_end) are produced (strip mode computes a sub-range)
};

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
                                            const float* scale_x, const PlaneGeom& g, const BlurK<R>& k, int pl) {
  constexpr int SW = BlurXCfg<R>::SW, RP = XTile<R>::RP;
  const int x0 = blockIdx.x * GBX_TW, yb = g.y0 + blockIdx.y * GBX_TH;
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

// Four single-plane x passes with different kernels in one launch (blockIdx.z picks the blur):
// the noise blur and the three mask blurs all become ready after hf_fused / mask_pre, and each
// alone is a one-wave launch whose ramp and tail cost as much as its arithmetic.
template <int R0, int R1, int R2, int R3>
struct BlurX4Args {
  float* out[4];
  const float* scale_x[4];
  BlurK<R0> k0;
  BlurK<R1> k1;
  BlurK<R2> k2;
  BlurK<R3> k3;
};

template <int R0, int R1, int R2, int R3>
__global__ void __launch_bounds__(128) k_tma_blur_x4(const __grid_constant__ CUtensorMap m0,
                                                     const __grid_constant__ CUtensorMap m1,
                                                     const __grid_constant__ CUtensorMap m2,
                                                     const __grid_constant__ CUtensorMap m3, PlaneGeom g,
                                                     const __grid_constant__ BlurX4Args<R0, R1, R2, R3> a) {
  constexpr int RMAX = R0 > R1 ? (R0 > R2 ? (R0 > R3 ? R0 : R3) : (R2 > R3 ? R2 : R3))
                               : (R1 > R2 ? (R1 > R3 ? R1 : R3) : (R2 > R3 ? R2 : R3));
  __shared__ __align__(128) float tile[GBX_TH * BlurXCfg<RMAX>::SW];
  __shared__ __align__(8) uint64_t bar;
  switch (blockIdx.z) {  // uniform per CTA
    case 0: blur_x_tile<R0>(tile, &bar, &m0, a.out[0], a.scale_x[0], g, a.k0, 0); break;
    case 1: blur_x_tile<R1>(tile, &bar, &m1, a.out[1], a.scale_x[1], g, a.k1, 0); break;
    case 2: blur_x_tile<R2>(tile, &bar, &m2, a.out[2], a.scale_x[2], g, a.k2, 0); break;
    default: blur_x_tile<R3>(tile, &bar, &m3, a.out[3], a.scale_x[3], g, a.k3, 0); break;
  }
}

// ---------------------------------------------------------------------------
// y pass with epilogue: tile of GBY_TW x GBY_TH outputs, 256 threads = 128 columns x
// 2 groups of 16 rows.  NP planes are blurred by the same thread (their tiles arrive
// together) and handed to the epilogue as v[NP] per pixel.
// grid (ceil(w / TW), ceil(rows / TH), NP == 1 ? planes : 1).
#define GBY_TW 128
#define GBY_TH 32
#define GBY_G 16

template <int R, int NP, class Epi>
__global__ void __launch_bounds__(256, NP == 1 ? 3 : 2) k_tma_blur_y(const __grid_constant__ CUtensorMap in_map, const float* scale_y,
                                                    PlaneGeom g, BlurK<R> k, Epi epi) {
  constexpr int HI = GBY_TH + 2 * R;
  extern __shared__ __align__(128) float dyn_smem[];
  float* tile = dyn_smem;                                                     // [NP][HI][TW]
  uint64_t* bar = reinterpret_cast<uint64_t*>(dyn_smem + NP * HI * GBY_TW);  // 8-byte aligned: sizes are multiples of 128 B
  const int x0 = blockIdx.x * GBY_TW, yb = g.y0 + blockIdx.y * GBY_TH, pz = blockIdx.z;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, NP * HI * GBY_TW * 4);
#pragma unroll
    for (int p = 0; p < NP; ++p) tma_load_box(tile + p * HI * GBY_TW, &in_map, bar, x0, yb - R, NP == 1 ? pz : p);
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
      if (y < g.y_end) epi.load(x, y, pz, pre[i]);
    }
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int y = yg + o0 + i;
      if (y >= g.y_end) continue;
      float v[NP];
#pragma unroll
      for (int p = 0; p < NP; ++p) v[p] = res[p][o0 + i];
      epi.apply(x, y, pz, v, pre[i]);
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
// (NP == 1: blockIdx.z picks the plane).  grid (ceil(w / TW), ceil(rows / seg), NP == 1 ? planes : 1).
template <int R, int NP, class Epi>
__global__ void __launch_bounds__(128) k_roll_blur(const __grid_constant__ CUtensorMap in_map, const float* scale_x,
                                                   const float* scale_y, PlaneGeom g, int seg, BlurK<R> k, Epi epi) {
  typedef RollCfg<R, NP> C;
  constexpr int D = C::D, RP = XTile<R>::RP, NS = C::NS, NPOS = C::RING / GBR_CH;
  extern __shared__ __align__(128) float dyn_smem[];
  float* stage = dyn_smem;                        // [NS][NP][CH][SW]
  float* ring = dyn_smem + NS * C::kStageFloats;  // [NP][RBUF][TW]
  uint64_t* bar = reinterpret_cast<uint64_t*>(ring + C::kRingFloats);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, pz = blockIdx.z;
  const int x0 = blockIdx.x * GBR_TW, x = x0 + lane;
  const int ys = g.y0 + blockIdx.y * seg;
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
                     NP == 1 ? pz : p);
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
                     yin + (c + NS) * GBR_CH, NP == 1 ? pz : p);
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
      if (y < ye) epi.load(x, y, pz, pre[o]);
    }
#pragma unroll
    for (int o = 0; o < GBR_G; ++o) {
      const int y = yg + o;
      if (y >= ye) continue;
      float v[NP];
#pragma unroll
      for (int p = 0; p < NP; ++p) v[p] = res[p][o];
      epi.apply(x, y, pz, v, pre[o]);
    }
  }
}

// ---------------------------------------------------------------------------
// Small radius (<= 5): x and y pass of NP planes in one kernel from one tile, epilogue
// on the registers.  Tile GB2_TW x GB2_TH outputs, 256 threads.
//   phase 1  x pass of all NP * (TH + 2R) tile rows -> tmp (shared), 4 outputs per item
//   phase 2  thread = column x group of 8 rows: y pass from tmp, then the epilogue, which
//            also sees the un-blurred samples of its pixel (`sharp`, from the input tile).
// grid (ceil(w / TW), ceil(rows / TH), 1).
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

template <int R, int NP, class Epi>
__global__ void __launch_bounds__(256) k_tma_blur_2d(const __grid_constant__ CUtensorMap in_map, const float* scale_x,
                                                     const float* scale_y, PlaneGeom g, BlurK<R> k, Epi epi) {
  typedef Blur2dCfg<R, NP> C;
  constexpr int SWI = C::SWI, HI = C::HI, RP = XTile<R>::RP;
  extern __shared__ __align__(128) float dyn_smem[];
  float* in = dyn_smem;                 // [NP][HI][SWI]
  float* tmp = dyn_smem + C::kInFloats;  // [NP][HI][TW]
  uint64_t* bar = reinterpret_cast<uint64_t*>(dyn_smem + C::kInFloats + C::kTmpFloats);
  const int x0 = blockIdx.x * GB2_TW, yb = g.y0 + blockIdx.y * GB2_TH;
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(bar, C::kInFloats * 4);
#pragma unroll
    for (int p = 0; p < NP; ++p) tma_load_box(in + p * HI * SWI, &in_map, bar, x0 - RP, yb - R, p);
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
      if (live_col && y < g.y_end) epi.load(x, y, pre[i]);
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
      epi.apply(x, y, live_col && y < g.y_end, sharp, v, pre[i], carry);
    }
  }
}

// ---------------------------------------------------------------------------
// Epilogues.  Plane groups are addressed as base + plane_index * g.plane + y * pitch + x.

// Each epilogue has two halves: load() fetches the pixel's global operands through the
// read-only path into a Pre, apply() does the arithmetic and the stores.  The kernels call
// load() for a chunk of kChunk pixels before the first apply(), so that the chunk's loads are
// in flight together instead of queueing behind one another's dependent stores.
struct NoPre {};

// plain store (stand-alone blur: tests, the one-time mask of the original)
struct EpiStore {
  float* out;
  int pitch;
  size_t plane;
  typedef NoPre Pre;
  static constexpr int kChunk = 16;
  __device__ __forceinline__ void load(int, int, int, Pre&) const {}
  __device__ __forceinline__ void apply(int x, int y, int pz, const float v[1], const Pre&) const {
    out[pz * plane + static_cast<size_t>(y) * pitch + x] = v[0];
  }
};

// S2 (b/butteraugli.cc:509-513): lf = Blur(xyb); mf = xyb - lf, per plane.
struct EpiLf {
  const float* xyb;
  float* lf;
  float* mf_in;
  int pitch;
  size_t plane;
  struct Pre {
    float a;
  };
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int x, int y, int pz, Pre& p) const {
    p.a = __ldg(xyb + pz * plane + static_cast<size_t>(y) * pitch + x);
  }
  __device__ __forceinline__ void apply(int x, int y, int pz, const float v[1], const Pre& p) const {
    const size_t o = pz * plane + static_cast<size_t>(y) * pitch + x;
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
  size_t plane;
  struct Pre {
    float inx, iny, p0x, p0y;
  };
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int x, int y, int, Pre& p) const {
    const size_t o = static_cast<size_t>(y) * pitch + x;
    p.inx = __ldg(mf_in + o);
    p.iny = __ldg(mf_in + plane + o);
    if (ps0 != nullptr) {
      p.p0x = __ldg(ps0 + kMfX * plane + o);
      p.p0y = __ldg(ps0 + kMfY * plane + o);
    }
  }
  __device__ __forceinline__ void apply(int x, int y, int, const float v[3], const Pre& p) const {
    const size_t o = static_cast<size_t>(y) * pitch + x;
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
  size_t plane;
  typedef NoPre Pre;
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int, int, Pre&) const {}
  __device__ __forceinline__ void apply(int x, int y, bool live, const float sharp[3], const float v[3], const Pre&,
                                        float&) const {
    if (!live) return;
    const size_t o = static_cast<size_t>(y) * pitch + x;
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
  size_t plane;
  struct Pre {
    float lfx, lfy, lfb, u0x, h0x, u0y, h0y;
  };
  static constexpr int kChunk = 4;
  __device__ __forceinline__ void load(int x, int y, Pre& p) const {
    const size_t o = static_cast<size_t>(y) * pitch + x;
    p.lfx = __ldg(lf_raw + o);
    p.lfy = __ldg(lf_raw + plane + o);
    p.lfb = __ldg(lf_raw + 2 * plane + o);
    if (ps0 != nullptr) {
      p.u0x = __ldg(ps0 + kUhfX * plane + o);
      p.h0x = __ldg(ps0 + kHfX * plane + o);
      p.u0y = __ldg(ps0 + kUhfY * plane + o);
      p.h0y = __ldg(ps0 + kHfY * plane + o);
    }
  }
  __device__ __forceinline__ void apply(int x, int y, bool live, const float sharp[2], const float v[2], const Pre& p,
                                        float&) const {
    if (!live) return;
    const size_t o = static_cast<size_t>(y) * pitch + x;
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
  struct Pre {
    float r0, r1, a;
  };
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int x, int y, int, Pre& p) const {
    const size_t o = static_cast<size_t>(y) * pitch + x;
    p.r0 = __ldg(hf0 + o);
    p.r1 = __ldg(hf1 + o);
    p.a = acc[o];  // plain load: this launch writes the location later (same thread)
  }
  __device__ __forceinline__ void apply(int x, int y, int, const float v[1], const Pre& p) const {
    const size_t o = static_cast<size_t>(y) * pitch + x;
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
// (non-negative floats order like their bit patterns).
struct EpiFinal {
  float* distmap;
  float* block_max;     // [nblocks], written for block rows [by_lo, by_hi)
  unsigned int* gmax;   // global maximum (float bits), or nullptr
  int pitch, bw, by_lo, by_hi;
  typedef NoPre Pre;
  static constexpr int kChunk = 8;
  __device__ __forceinline__ void load(int, int, Pre&) const {}
  // m: running maximum of the thread's pixels of the current block row (one block column)
  __device__ __forceinline__ void apply(int x, int y, bool live, const float sharp[1], const float v[1], const Pre&,
                                        float& m) const {
    if (live) {
      const double mul1 = 0.458794906198;
      const float scale = static_cast<float>(1.0f / (1.0f + mul1));
      float d = static_cast<float>(static_cast<double>(sharp[0]) + mul1 * v[0]);
      d *= scale;
      distmap[static_cast<size_t>(y) * pitch + x] = d;
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
        block_max[by * bw + bx] = b;
        if (gmax != nullptr) atomicMax(gmax, __float_as_uint(b));
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

template <int RA, int RB, int RC>
__global__ void __launch_bounds__(256) k_tma_mask_y(const __grid_constant__ CUtensorMap map_a,
                                                    const __grid_constant__ CUtensorMap map_b,
                                                    const __grid_constant__ CUtensorMap map_c, const float* sya,
                                                    const float* syb, const float* syc, PlaneGeom g, BlurK<RA> ka,
                                                    BlurK<RB> kb, BlurK<RC> kc, CombineArgs ca) {
  typedef MaskYCfg<RA, RB, RC> C;
  extern __shared__ __align__(128) float dyn_smem[];
  float* ta = dyn_smem;
  float* tb = ta + C::HA * GBY_TW;
  float* tc = tb + C::HB * GBY_TW;
  uint64_t* bar = reinterpret_cast<uint64_t*>(tc + C::HC * GBY_TW);
  const int x0 = blockIdx.x * GBY_TW, yb = g.y0 + blockIdx.y * GBY_TH;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, (C::HA + C::HB + C::HC) * GBY_TW * 4);
    tma_load_box(ta, &map_a, bar, x0, yb - RA, 0);
    tma_load_box(tb, &map_b, bar, x0, yb - RB, 0);
    tma_load_box(tc, &map_c, bar, x0, yb - RC, 0);
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
  comb.ps0 = ca.ps0;
  comb.ps1 = ca.ps1;
  comb.ac = ca.ac;
  comb.out = ca.out;
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
      const size_t o = static_cast<size_t>(y) * ca.pitch + x;
      l0x[i] = __ldg(ca.ps0 + kLfX * ca.plane + o);
      l0b[i] = __ldg(ca.ps0 + kLfB * ca.plane + o);
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
// grid (ceil(w / 64), ceil(rows / 32), 2 channels), 256 threads.
__global__ void __launch_bounds__(256, 2) k_tma_malta_sums(const __grid_constant__ CUtensorMap diffs_map, float* acc,
                                                           PlaneGeom g) {
  __shared__ __align__(128) float tile[2][GB_MALTA_SH * GB_MALTA_SW];
  __shared__ __align__(8) uint64_t bar[2];
  const int tx = threadIdx.x, ty = threadIdx.y;  // 16 x 16
  const int tid = ty * 16 + tx;
  const int x0 = blockIdx.x * GB_MALTA_TILE_W, y0 = g.y0 + blockIdx.y * GB_MALTA_TILE_H, ch = blockIdx.z;
  constexpr uint32_t kBytes = GB_MALTA_SH * GB_MALTA_SW * 4;
  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(&bar[0], kBytes);
    tma_load_box(tile[0], &diffs_map, &bar[0], x0 - 4, y0 - 4, 3 * ch + 0);
    mbar_expect_tx(&bar[1], kBytes);
    tma_load_box(tile[1], &diffs_map, &bar[1], x0 - 4, y0 - 4, 3 * ch + 1);
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
    tma_load_box(tile[0], &diffs_map, &bar[0], x0 - 4, y0 - 4, 3 * ch + 2);
  }
  // band 1 (hf) from buffer 1, band 2 (mf) from buffer 0 again
  mbar_wait(&bar[1], 0);
  malta_window_sums(tile[1], tx, ty, false, r);
  mbar_wait(&bar[0], 1);
  malta_window_sums(tile[0], tx, ty, false, r);
  const int xb = x0 + 4 * tx;
  float* aplane = acc + static_cast<size_t>(ch) * g.plane;
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
__global__ void __launch_bounds__(256) k_mask_sup(const float* ps, float* sup, PlaneGeom g) {
  const int x = blockIdx.x * 32 + threadIdx.x, y = g.y0 + blockIdx.y * 8 + threadIdx.y;
  if (x >= g.w || y >= g.y_end) return;
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

// mpre[c] = min(cutoff, mul0 * min(sup0_c, sup1_c)) for c = X, Y.
__global__ void __launch_bounds__(256) k_mask_pre(const float* ps1, const float* sup0, float* mpre, PlaneGeom g) {
  const int x = blockIdx.x * 32 + threadIdx.x, y = g.y0 + blockIdx.y * 8 + threadIdx.y;
  if (x >= g.w || y >= g.y_end) return;
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

}  // namespace gb200
