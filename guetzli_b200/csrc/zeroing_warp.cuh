// a13/a14 on sm_90a: one warp per 8x8 block runs the whole greedy zeroing loop of
// Processor::ComputeBlockZeroingOrder (g/processor.cc:364-467) with every per-pixel /
// per-transform step of CompareBlock (g/butteraugli_comparator.cc:457-488) spread
// over the 32 lanes and all block state in shared memory.  Same helper arithmetic
// (idct_1d, ycc_to_rgb, blur_tap_sum, opsin_pixel, real_dft8, cplx_dft8) and the
// same ordered accumulations as the one-thread-per-block functor in block_math.h,
// which stays the CPU port's version; both are tested against the reference.
#pragma once
#include <cuda_runtime.h>

#include <stdexcept>

#include "block_math.h"

namespace gb200 {

// Per-warp block state in shared memory.  Arrays whose lifetimes do not overlap share
// storage (7.1 KB per warp instead of 11 KB: seven CTAs of four warps per SM instead of five):
//   sort   (only while the order is built)          over  f
//   d      (written after opsin_pixel has read lin) over  lin + tmp
//   pw     (written after the row transforms)       over  d
struct ZWarpState {
  uint8_t order_id[192];  // sorted candidate coefficients (component * 64 + natural index)
  int16_t blk[192];
  int16_t col[64];
  uint8_t px[3][64];
  uint8_t trial[64];
  float xyb0[3][64];
  union {
    struct {
      float lin[3][64];
      float tmp[3][64];
    };
    double d[3][64];
    double pw[3][40];
  };
  float blr[3][64];
  union {
    Cplx f[3][64];
    SortItem sort[192];
  };
};

#define GB_ZW_WARPS 4

struct SmemRow {
  const float* p;
  __device__ __forceinline__ float operator()(int j) const { return p[j]; }
};
struct SmemCol {
  const float* p;
  __device__ __forceinline__ float operator()(int j) const { return p[8 * j]; }
};

// IDCT of one component held in shared memory: blk (int16[64]) -> out (u8[64]).
__device__ __forceinline__ void warp_idct(const int* basis, const int16_t* blk, int16_t* col, uint8_t* out, int lane) {
  // column pass: output (y, x), two per lane
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int o = lane + 32 * k, y = o >> 3, x = o & 7;
    int acc = 0;
#pragma unroll
    for (int u = 0; u < 8; ++u) acc += basis[8 * y + u] * blk[8 * u + x];
    col[8 * y + x] = static_cast<int16_t>((acc + (1 << 10)) >> 11);
  }
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int o = lane + 32 * k, y = o >> 3, x = o & 7;
    int acc = 0;
#pragma unroll
    for (int u = 0; u < 8; ++u) acc += basis[8 * x + u] * col[8 * y + u];
    const int v = (acc + (257 << 17)) >> 18;
    out[8 * y + x] = static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
  }
  __syncwarp();
}

// The 8-wide opsin blur (sigma 1.2: radius 2) as a fixed 5-term sum.  For output
// position p the weights are the raw taps (border rule, p < 2 or p > 5), or the
// normalised taps (interior); terms whose sample lies outside 0..7 get weight 0 and a
// clamped (finite) sample: they add +-0 to a sum that starts at +0, which leaves every
// partial sum bit-identical to blur_tap_sum's shorter loop.  sc = 1/weight for border
// positions, 1 for interior ones (x * 1 == x).
struct Blur8W {
  float w[5];
  float sc;
};
__device__ __forceinline__ Blur8W blur8_weights(const BlurTab& tab, const float* scale8, int p) {
  Blur8W b;
  const bool border = p < 2 || p + 2 >= 8;
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const int q = p + j - 2;
    b.w[j] = (q < 0 || q > 7) ? 0.0f : (border ? tab.taps[j] : tab.taps_n[j]);
  }
  b.sc = border ? scale8[p] : 1.0f;
  return b;
}
// in[stride * q], q = 0..7, is the line through the output; p its position on the line.
__device__ __forceinline__ float blur8(const float* in, int stride, int p, const Blur8W& b) {
  float sum = 0.0f;
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    int q = p + j - 2;
    q = q < 0 ? 0 : (q > 7 ? 7 : q);
    sum += in[stride * q] * b.w[j];
  }
  return sum * b.sc;
}

// Both passes give a lane outputs at position lane & 7 of their line (the row pass
// x = lane & 7, the column pass y = lane & 7), so one weight set per lane serves both.
typedef Blur8W Blur8Lane;

// 8x8 linear RGB tile -> XYB (OpsinDynamicsImage on 8x8), two pixels per lane.
__device__ __forceinline__ void warp_opsin8(ZWarpState& s, const Blur8Lane& bw, int lane, float out[2][3]) {
  // row pass: 192 outputs, six per lane (x = lane & 7 for all of them)
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const int o = lane + 32 * k, c = o >> 6, i = o & 63, y = i >> 3, x = i & 7;
    s.tmp[c][i] = blur8(s.lin[c] + 8 * y, 1, x, bw);
  }
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const int c = k >> 1, y = lane & 7, x = (lane >> 3) + 4 * (k & 1);
    s.blr[c][8 * y + x] = blur8(s.tmp[c] + x, 8, y, bw);
  }
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int i = lane + 32 * k;
    opsin_pixel(s.lin[0][i], s.lin[1][i], s.lin[2][i], s.blr[0][i], s.blr[1][i], s.blr[2][i], &out[k][0],
                &out[k][1], &out[k][2]);
  }
  __syncwarp();  // lin / tmp are dead from here on: the caller may overwrite them (d shares their storage)
}

struct ZeroingWarpArgs {
  const int16_t* cand;
  const int16_t* orig;
  const uint8_t* rgb;
  const float* corner_mask;
  uint8_t* out_idx;
  float* out_err;
  int* out_count;
  Geom g;
  Tables t;
  int lookahead;
  float block_error_limit;
  int b0, nb;  // blocks [b0, b0 + nb) are processed
  int new_model;
};

// CompareBlock for the current pixel state: comp c uses `pc` (its trial pixels),
// the others s.px.  Returns the error in every lane.
__device__ __forceinline__ float warp_compare_block(ZWarpState& s, const ZeroingWarpArgs& a, const Blur8Lane& bw,
                                                    int c_changed, const uint8_t* pc, int xlast, int ylast,
                                                    const float* mask, int lane) {
  const Tables& t = a.t;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int i = lane + 32 * k, iy = i >> 3, ix = i & 7;
    const int sy = iy < ylast ? iy : ylast, sx = ix < xlast ? ix : xlast;
    const int sidx = 8 * sy + sx;
    const int yy = (c_changed == 0 ? pc : s.px[0])[sidx];
    const int cb = (c_changed == 1 ? pc : s.px[1])[sidx];
    const int cr = (c_changed == 2 ? pc : s.px[2])[sidx];
    int r, gg, bb;
    ycc_to_rgb(t.cr_r, t.cb_b, t.cr_g, t.cb_g, yy, cb, cr, &r, &gg, &bb);
    s.lin[0][i] = t.srgb_lin[r];
    s.lin[1][i] = t.srgb_lin[gg];
    s.lin[2][i] = t.srgb_lin[bb];
  }
  __syncwarp();
  float xyb1[2][3];
  warp_opsin8(s, bw, lane, xyb1);
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int i = lane + 32 * k;
#pragma unroll
    for (int c = 0; c < 3; ++c) s.d[c][i] = static_cast<double>(s.xyb0[c][i]) - static_cast<double>(xyb1[k][c]);
  }
  __syncwarp();
  // lanes 0..2: ordered sum of the 64 differences (avg term); lanes 8..31: the 24 row transforms
  double dc = 0.0;
  if (lane < 3) {
    double avg = 0.0;
    for (int i = 0; i < 64; ++i) avg += s.d[lane][i];
    const double avgdiff = avg / 64;
    dc += 4.0 * avgdiff * avgdiff;
  } else if (lane >= 8) {
    const int job = lane - 8, c = job >> 3, y = job & 7;
    Cplx row[8];
    real_dft8(&s.d[c][8 * y], row);
#pragma unroll
    for (int k = 0; k < 8; ++k) s.f[c][8 * k + y] = row[k];
  }
  __syncwarp();
  // column stage: per channel two real transforms (frequency rows 0 and 4) and three complex ones
  if (lane < 15) {
    const int c = lane / 5, job = lane - 5 * c;
    Cplx* f = s.f[c];
    if (job < 2) {
      double r[8];
#pragma unroll
      for (int x = 0; x < 8; ++x) r[x] = f[32 * job + x].re;
      Cplx o[8];
      real_dft8(r, o);
#pragma unroll
      for (int x = 0; x < 8; ++x) f[32 * job + x] = o[x];
    } else {
      Cplx v[8];
      Cplx* p = f + 8 * (job - 1);
#pragma unroll
      for (int x = 0; x < 8; ++x) v[x] = p[x];
      cplx_dft8(v);
#pragma unroll
      for (int x = 0; x < 8; ++x) p[x] = v[x];
    }
  }
  __syncwarp();
  // power spectrum bins 4..36 (99 values), then the ordered weighted sums on lanes 0..2
  for (int k = lane; k < 99; k += 32) {
    const int c = k / 33, i = 4 + (k - 33 * c);
    const Cplx z = s.f[c][i];
    double p = z.re * z.re + z.im * z.im;
    p *= 0.000064;
    s.pw[c][i] = p;
  }
  __syncwarp();
  if (lane < 3) {
    for (int i = 4; i < 37; ++i) dc += t.block_csf[i] * s.pw[lane][i];
  }
  const double d0 = __shfl_sync(0xffffffffu, dc, 0);
  const double d1 = __shfl_sync(0xffffffffu, dc, 1);
  const double d2 = __shfl_sync(0xffffffffu, dc, 2);
  double diff = 0.0;
  diff += d0 * mask[0];
  diff += d1 * mask[1];
  diff += d2 * mask[2];
  return static_cast<float>(sqrt(diff));
}

__global__ void __launch_bounds__(32 * GB_ZW_WARPS, 6) k_zeroing_orders_warp(ZeroingWarpArgs a) {
  __shared__ ZWarpState smem[GB_ZW_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int bl = blockIdx.x * GB_ZW_WARPS + warp;
  if (bl >= a.nb) return;
  const int b = a.b0 + bl;
  ZWarpState& s = smem[warp];
  const Geom& g = a.g;
  const Tables& t = a.t;
  const int bx = b % g.bw, by = b / g.bw;
  const int xlast = hd_min(7, g.w - 1 - 8 * bx), ylast = hd_min(7, g.h - 1 - 8 * by);

  // candidate coefficients
  for (int i = lane; i < 192; i += 32) {
    const int c = i >> 6, k = i & 63;
    s.blk[i] = a.cand[(static_cast<size_t>(c) * g.nblocks + b) * 64 + k];
  }
  __syncwarp();
  // nonzero AC coefficients in (component, natural index) order with their scores
  int n = 0;
  if (lane == 0) {
    for (int c = 0; c < 3; ++c) {
      const int16_t* ob = a.orig + (static_cast<size_t>(c) * g.nblocks + b) * 64;
      for (int k = 1; k < 64; ++k) {
        const int idx = 64 * c + k;
        if (s.blk[idx] != 0) {
          const int v = ob[k] < 0 ? -ob[k] : ob[k];
          s.sort[n].key = zeroing_score(v, idx, a.new_model != 0, t);
          s.sort[n].id = idx;
          ++n;
        }
      }
    }
    std_sort_replay(s.sort, n);
  }
  n = __shfl_sync(0xffffffffu, n, 0);
  __syncwarp();
  {
    int ids[6];
    for (int k = 0; k < 6; ++k) ids[k] = lane + 32 * k < n ? s.sort[lane + 32 * k].id : 0;
    __syncwarp();
    for (int k = 0; k < 6; ++k) s.order_id[lane + 32 * k] = static_cast<uint8_t>(ids[k]);
  }
  __syncwarp();
  // SwitchBlock: original tile (edge-replicated) -> linear -> opsin
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int i = lane + 32 * k, iy = i >> 3, ix = i & 7;
    const int y = hd_min(8 * by + iy, g.h - 1), x = hd_min(8 * bx + ix, g.w - 1);
    const uint8_t* p = a.rgb + 3 * (static_cast<size_t>(y) * g.w + x);
    s.lin[0][i] = t.srgb_lin[p[0]];
    s.lin[1][i] = t.srgb_lin[p[1]];
    s.lin[2][i] = t.srgb_lin[p[2]];
  }
  __syncwarp();
  const Blur8Lane bw = blur8_weights(t.blur[kBlurOpsin], t.opsin_scale8, lane & 7);
  {
    float x0[2][3];
    warp_opsin8(s, bw, lane, x0);
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int c = 0; c < 3; ++c) s.xyb0[c][lane + 32 * k] = x0[k][c];
  }
  const float mask[3] = {a.corner_mask[3 * b], a.corner_mask[3 * b + 1], a.corner_mask[3 * b + 2]};
  for (int c = 0; c < 3; ++c) warp_idct(t.idct, s.blk + 64 * c, s.col, s.px[c], lane);

  uint8_t* oi = a.out_idx + static_cast<size_t>(b) * 192;
  float* oe = a.out_err + static_cast<size_t>(b) * 192;
  int nout = 0;
  while (n > 0) {
    float best_err = 1e17f;
    int best_i = 0;
    const int tries = a.lookahead < n ? a.lookahead : n;
    for (int i = 0; i < tries; ++i) {
      const int idx = s.order_id[i];
      const int c = idx >> 6;
      const int16_t saved = s.blk[idx];
      __syncwarp();
      if (lane == 0) s.blk[idx] = 0;
      __syncwarp();
      warp_idct(t.idct, s.blk + 64 * c, s.col, s.trial, lane);
      const float err = warp_compare_block(s, a, bw, c, s.trial, xlast, ylast, mask, lane);
      float max_err = 0;
      max_err = hd_max(max_err, err);
      if (max_err < best_err) {
        best_err = max_err;
        best_i = i;
      }
      __syncwarp();
      if (lane == 0) s.blk[idx] = saved;
      __syncwarp();
    }
    const int idx = s.order_id[best_i];
    __syncwarp();
    if (lane == 0) s.blk[idx] = 0;
    __syncwarp();
    warp_idct(t.idct, s.blk + 64 * (idx >> 6), s.col, s.px[idx >> 6], lane);
    // erase order[best_i]
    uint8_t moved[6];
    int cnt = 0;
    for (int i = best_i + lane; i + 1 < n; i += 32) moved[cnt++] = s.order_id[i + 1];
    __syncwarp();
    cnt = 0;
    for (int i = best_i + lane; i + 1 < n; i += 32) s.order_id[i] = moved[cnt++];
    __syncwarp();
    --n;
    if (lane == 0) {
      oi[nout] = static_cast<uint8_t>(idx);
      oe[nout] = best_err;
    }
    ++nout;
  }
  __syncwarp();
  if (lane == 0) {
    // monotone suffix minimum, then cut at the block error limit (:447-459)
    float min_err = 1e10f;
    for (int i = nout - 1; i >= 0; --i) {
      min_err = hd_min(min_err, oe[i]);
      oe[i] = min_err;
    }
    int num = 0;
    while (num < nout && oe[num] <= a.block_error_limit) ++num;
    a.out_count[b] = num;
  }
}

inline void launch_zeroing_orders_warp(Stream s, const ZeroingWarpArgs& a) {
  if (a.t.blur[kBlurOpsin].r != 2) throw std::runtime_error("zeroing kernel: the opsin blur radius must be 2");
  const int ctas = (a.nb + GB_ZW_WARPS - 1) / GB_ZW_WARPS;
  if (ctas <= 0) return;
  note_launch("zeroing_orders", s, a.nb);
  k_zeroing_orders_warp<<<ctas, 32 * GB_ZW_WARPS, 0, s>>>(a);
  note_launch_end("zeroing_orders", s);
}

}  // namespace gb200
