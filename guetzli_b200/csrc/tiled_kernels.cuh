// Kernels of the search that count into a per-CTA shared-memory histogram: the symbol histograms
// of the JPEG size estimate (a11) and the key histogram and bin search of the order select (a16).
#pragma once
#include <cuda_runtime.h>

#include "jpeg_dev.h"
#include "kernels.h"

namespace gb200 {

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
