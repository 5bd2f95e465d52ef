// Device side of a11: entropy-coding of the candidate coefficients without
// moving them over PCIe.  Per iteration the search needs the exact size of the
// sequential JPEG (g/jpeg_data_writer.cc:455-536) and, a few times per image, its
// bytes.  Kernels:
//   JpegHistAcc    DC/AC symbol histograms (privatised global atomics)
//   JpegHistSum    reduction of the private copies
//   [host: cluster histograms, build canonical Huffman codes -- 1.5 KB of tables]
//   JpegUnitBits   code length of every unit (one block of one component) -> exclusive scan
//   JpegEmit       every unit ORs its bits into the scan at its bit offset
//   JpegCountFF    bytes equal to 0xFF (each needs a stuffed zero byte)
// All integer; bit-exact by construction against the host serialiser (jpeg_out.cc).
#pragma once
#include "hd.h"
#include "kernels.h"

namespace gb200 {

static const int kHistCopies = 256;   // private histogram copies (block index & 255)
static const int kHistStride = 6 * 257;  // [dc0 dc1 dc2 ac0 ac1 ac2][257]

GB_HD int hd_floor_log2_nz(unsigned int n) {
#if defined(__CUDA_ARCH__)
  return 31 - __clz(n);
#else
  return 31 ^ __builtin_clz(n);
#endif
}

// Quotient of a candidate coefficient by its quant step.  The candidate holds exact multiples of
// q (Quantize, g/quantize.h:24; coefficients of a JPEG input times their own step), |c| < 2^15, so
// on the device float(c) * rcp(float(q)) is off by less than 0.004 from the integer quotient and
// rounds to it: three instructions instead of an integer division per nonzero coefficient.
GB_HD int div_exact_multiple(int c, int q) {
#if defined(__CUDA_ARCH__)
  return __float2int_rn(__int2float_rn(c) * __frcp_rn(__int2float_rn(q)));
#else
  return c / q;
#endif
}

// Visits the entropy-coding symbols of one 8x8 block in scan order
// (EncodeDCTBlockSequential, g/jpeg_data_writer.cc:455): v.dc(nbits, extra),
// v.ac(symbol, nbits, extra).  dq = dequantised coefficients, q = quant table,
// prev_dc = quantised DC of the previous block of the same component.
template <class V>
GB_HD void visit_block_symbols(const int16_t* dq, const int* q, int prev_dc, const int* zigzag, V& v) {
  const int16_t dc = static_cast<int16_t>(div_exact_multiple(dq[0], q[0]));
  int16_t diff = static_cast<int16_t>(dc - prev_dc);
  int16_t low = diff;
  if (diff < 0) {
    diff = static_cast<int16_t>(-diff);
    --low;
  }
  const unsigned int mag = static_cast<unsigned int>(static_cast<int>(diff));
  const int nb = mag == 0 ? 0 : hd_floor_log2_nz(mag) + 1;
  v.dc(nb, static_cast<unsigned int>(low) & ((1u << nb) - 1u));
  int run = 0;
  for (int k = 1; k < 64; ++k) {
    const int nat = zigzag[k];
    int c = dq[nat];
    if (c == 0) {
      ++run;
      continue;
    }
    c = div_exact_multiple(c, q[nat]);
    int m = c, lo = c;
    if (c < 0) {
      m = -c;
      lo = ~m;
    }
    while (run > 15) {
      v.ac(0xf0, 0, 0u);
      run -= 16;
    }
    const int nbits = hd_floor_log2_nz(static_cast<unsigned int>(m)) + 1;
    v.ac((run << 4) + nbits, nbits, static_cast<unsigned int>(lo) & ((1u << nbits) - 1u));
    run = 0;
  }
  if (run > 0) v.ac(0, 0, 0u);
}

struct JpegHistAcc {  // 1D over 3*nblocks: i = c*nblocks + b
  const int16_t* cand;
  const int* q;          // [192]
  const int* zigzag;     // [64]
  unsigned int* hist;    // [kHistCopies][6][257]
  unsigned int* chroma_nonzero;
  int nblocks;
  struct Visitor {
    unsigned int* dc_h;
    unsigned int* ac_h;
    GB_HD void dc(int nbits, unsigned int) { hd_atomic_add(&dc_h[nbits], 1u); }
    GB_HD void ac(int symbol, int, unsigned int) { hd_atomic_add(&ac_h[symbol], 1u); }
  };
  GB_HD void operator()(int i) const {
    const int c = i / nblocks, b = i - c * nblocks;
    const int16_t* blk = cand + static_cast<size_t>(i) * 64;
    const int* qc = q + 64 * c;
    const int prev = b > 0 ? div_exact_multiple((blk - 64)[0], qc[0]) : 0;
    unsigned int* base = hist + static_cast<size_t>(b & (kHistCopies - 1)) * kHistStride;
    Visitor v{base + c * 257, base + (3 + c) * 257};
    visit_block_symbols(blk, qc, prev, zigzag, v);
    if (c > 0) {
      bool any = false;
      for (int k = 0; k < 64; ++k) any = any || (blk[k] != 0);
      if (any) *chroma_nonzero = 1u;
    }
  }
};

struct JpegHistSum {  // 1D over 6*257
  const unsigned int* hist;
  unsigned int* out;
  GB_HD void operator()(int i) const {
    unsigned int s = 0;
    for (int k = 0; k < kHistCopies; ++k) s += hist[static_cast<size_t>(k) * kHistStride + i];
    out[i] = s;
  }
};

struct JpegCodes {
  const uint8_t* depth;    // [6][256]  dc0 dc1 dc2 ac0 ac1 ac2
  const uint16_t* code;    // [6][256]
};

// One unit = one 8x8 block of one component; units are numbered in scan order
// u = b * ncomp + c (Y, Cb, Cr block of MCU b).
struct JpegUnitBits {  // 1D over nblocks * ncomp
  const int16_t* cand;
  const int* q;
  const int* zigzag;
  JpegCodes codes;
  unsigned int* bits;
  int nblocks, ncomp;
  struct Visitor {
    const uint8_t* dc_d;
    const uint8_t* ac_d;
    unsigned int n;
    GB_HD void dc(int nbits, unsigned int) { n += dc_d[nbits] + nbits; }
    GB_HD void ac(int symbol, int nbits, unsigned int) { n += ac_d[symbol] + nbits; }
  };
  GB_HD void operator()(int u) const {
    const int b = u / ncomp, c = u - b * ncomp;
    const int16_t* blk = cand + (static_cast<size_t>(c) * nblocks + b) * 64;
    const int* qc = q + 64 * c;
    const int prev = b > 0 ? div_exact_multiple((blk - 64)[0], qc[0]) : 0;
    Visitor v{codes.depth + c * 256, codes.depth + (3 + c) * 256, 0u};
    visit_block_symbols(blk, qc, prev, zigzag, v);
    bits[u] = v.n;
  }
};

// Bit sink writing MSB-first into big-endian 32-bit words.  Bits are gathered in a
// 64-bit register and leave as whole words with one atomic OR each (the first and
// last word of a unit are shared with its neighbours; the bits that belong to the
// neighbours are zero in our word, so OR-ing is safe).  Plain stores for the words in
// between were measured slower.
struct BitCursor {
  unsigned int* words;
  unsigned long long word;  // index of the next word to write
  unsigned long long acc;   // pending bits, right-aligned
  int nacc;                 // number of pending bits (< 32 between calls)
  GB_HD void start(unsigned int* w, unsigned long long bit_pos) {
    words = w;
    word = bit_pos >> 5;
    acc = 0;
    nacc = static_cast<int>(bit_pos & 31);  // leading zero bits stand in for the neighbour's bits
  }
  GB_HD void put(int n, unsigned int value) {  // n <= 27
    acc = (acc << n) | value;
    nacc += n;
    if (nacc >= 32) {
      nacc -= 32;
      hd_atomic_or(&words[word], static_cast<unsigned int>(acc >> nacc));
      ++word;
      acc &= (1ull << nacc) - 1ull;
    }
  }
  GB_HD void finish() {
    if (nacc > 0) hd_atomic_or(&words[word], static_cast<unsigned int>(acc << (32 - nacc)));
    nacc = 0;
  }
};

struct JpegEmit {  // 1D over nblocks * ncomp
  const int16_t* cand;
  const int* q;
  const int* zigzag;
  JpegCodes codes;
  const unsigned int* offset;  // exclusive scan of JpegUnitBits
  unsigned int* words;
  int nblocks, ncomp;
  struct Visitor {
    const uint8_t* dc_d;
    const uint16_t* dc_c;
    const uint8_t* ac_d;
    const uint16_t* ac_c;
    BitCursor cur;
    GB_HD void dc(int nbits, unsigned int extra) {
      cur.put(dc_d[nbits], dc_c[nbits]);
      if (nbits > 0) cur.put(nbits, extra);
    }
    GB_HD void ac(int symbol, int nbits, unsigned int extra) {
      cur.put(ac_d[symbol], ac_c[symbol]);
      if (nbits > 0) cur.put(nbits, extra);
    }
  };
  GB_HD void operator()(int u) const {
    const int b = u / ncomp, c = u - b * ncomp;
    const int16_t* blk = cand + (static_cast<size_t>(c) * nblocks + b) * 64;
    const int* qc = q + 64 * c;
    const int prev = b > 0 ? div_exact_multiple((blk - 64)[0], qc[0]) : 0;
    Visitor v{codes.depth + c * 256, codes.code + c * 256, codes.depth + (3 + c) * 256,
              codes.code + (3 + c) * 256, BitCursor()};
    v.cur.start(words, offset[u]);
    visit_block_symbols(blk, qc, prev, zigzag, v);
    v.cur.finish();
  }
};

// Pads the last byte with one-bits (JumpToByteBoundary, g/jpeg_bit_writer.h:90) and
// counts 0xFF bytes; 1D over the words of the scan.
struct JpegCountFF {
  unsigned int* words;
  unsigned long long total_bits;
  unsigned int* counter;
  GB_HD void operator()(int w) const {
    const unsigned long long nbytes = (total_bits + 7) >> 3;
    unsigned int v = words[w];
    const unsigned long long first_bit = static_cast<unsigned long long>(w) << 5;
    if (total_bits > first_bit && total_bits - first_bit < 32 && (total_bits & 7)) {
      // this word holds the final partial byte
      const int used = static_cast<int>(total_bits - first_bit);
      const int pad = 8 - (used & 7);
      v |= ((1u << pad) - 1u) << (32 - used - pad);
      words[w] = v;
    }
    unsigned int n = 0;
    for (int k = 0; k < 4; ++k) {
      const unsigned long long byte_index = (static_cast<unsigned long long>(w) << 2) + k;
      if (byte_index < nbytes && ((v >> (24 - 8 * k)) & 0xffu) == 0xffu) ++n;
    }
    if (n) hd_atomic_add(counter, n);
  }
};

// ---- f1: the complete file on the device ---------------------------------------------
// The scan leaves JpegEmit / JpegCountFF as padded, un-stuffed bytes in big-endian words.  The
// file is  prefix | stuffed scan | trailer  (g/jpeg_data_writer.cc:52-128,540-553; a zero byte
// after every 0xFF of the scan, g/jpeg_bit_writer.h:62-77).  JpegWordFF counts the 0xFF bytes
// of every word, an exclusive scan turns the counts into the shift of each word, JpegStuffBytes
// writes every byte to its final position.  1D over the words of the scan.
struct JpegWordFF {
  const unsigned int* words;
  unsigned long long nbytes;
  unsigned int* count;
  GB_HD void operator()(int w) const {
    const unsigned int v = words[w];
    unsigned int n = 0;
    for (int k = 0; k < 4; ++k) {
      const unsigned long long byte_index = (static_cast<unsigned long long>(w) << 2) + k;
      if (byte_index < nbytes && ((v >> (24 - 8 * k)) & 0xffu) == 0xffu) ++n;
    }
    count[w] = n;
  }
};

struct JpegStuffBytes {
  const unsigned int* words;
  const unsigned int* ff_before;  // exclusive scan of JpegWordFF
  unsigned long long nbytes;
  uint8_t* out;  // first byte of the scan inside the file buffer
  GB_HD void operator()(int w) const {
    const unsigned int v = words[w];
    unsigned long long pos = (static_cast<unsigned long long>(w) << 2) + ff_before[w];
    for (int k = 0; k < 4; ++k) {
      const unsigned long long byte_index = (static_cast<unsigned long long>(w) << 2) + k;
      if (byte_index >= nbytes) break;
      const unsigned int b = (v >> (24 - 8 * k)) & 0xffu;
      out[pos++] = static_cast<uint8_t>(b);
      if (b == 0xffu) out[pos++] = 0;
    }
  }
};

}  // namespace gb200
