// Kernel bodies (functors) of the full-image path: render (a7-a9), butteraugli
// Compare (a10), block maxima / weights (a15), one-time FDCT (a2).  Each functor
// is launched over pixels or blocks by backend.h.  Reference citations:
// g/ = /root/reference/guetzli/, b/ = .../third_party/butteraugli/butteraugli/.
//
// Layout: float planes are [h][pitch] with pitch = round_up(w, 32) floats (128 B
// rows: coalesced warps, TMA-legal strides); plane groups are contiguous
// ([n][h][pitch]) so a row pass can treat a group as one tall image.
// Coefficients are int16 [3][nblocks][64], block-major like JPEGComponent::coeffs.
#pragma once
#include "ba_math.h"
#include "jpeg_math.h"
#include "tables.h"

namespace gb200 {

struct Geom {
  int w, h, pitch, bw, bh, nblocks;
  size_t plane;  // floats per plane = h * pitch
};

inline Geom make_geom(int w, int h) {
  Geom g;
  g.w = w;
  g.h = h;
  g.pitch = (w + 31) & ~31;
  g.bw = (w + 7) / 8;
  g.bh = (h + 7) / 8;
  g.nblocks = g.bw * g.bh;
  g.plane = static_cast<size_t>(h) * g.pitch;
  return g;
}

// ---------------------------------------------------------------------------
// a2: RGB -> YCbCr -> FDCT -> descale, one block per invocation
// (g/jpeg_data_encoder.cc:84-113).  Edge blocks replicate the last row/column.
struct FdctBlocks {
  const uint8_t* rgb;  // interleaved [h][w][3]
  int16_t* coeffs;     // [3][nblocks][64]
  Geom g;
  GB_HD void operator()(int b) const {
    const int bx = b % g.bw, by = b / g.bw;
    int16_t blk[192];
    for (int iy = 0; iy < 8; ++iy) {
      const int y = hd_min(g.h - 1, 8 * by + iy);
      for (int ix = 0; ix < 8; ++ix) {
        const int x = hd_min(g.w - 1, 8 * bx + ix);
        const uint8_t* p = rgb + 3 * (static_cast<size_t>(y) * g.w + x);
        rgb_to_ycc16(p[0], p[1], p[2], &blk[8 * iy + ix], &blk[64 + 8 * iy + ix],
                     &blk[128 + 8 * iy + ix]);
      }
    }
    for (int c = 0; c < 3; ++c) {
      fdct_8x8(blk + 64 * c);
      int16_t* out = coeffs + (static_cast<size_t>(c) * g.nblocks + b) * 64;
      for (int k = 0; k < 64; ++k) out[k] = fdct_descale(blk[64 * c + k]);
    }
  }
};

// BlendOnBlack of the guetzli tool (g/guetzli.cc:43-45): an 8-bit sample under 8-bit alpha, laid over
// black in integers.  Not the butteraugli tool's rule (srgb_over_linear rounds with + 127, not + 128).
GB_HD int blend_on_black(int v, int a) { return (v * a + 128) / 255; }

// An 8-bit image of C = 1..4 channels in any strided layout -> packed sRGB [h][w][3], converted as the
// guetzli tool converts the PNG layouts before Process (ReadPNG, g/guetzli.cc:43-145): gray replicated
// (C = 1), gray + alpha blended on black and replicated (C = 2), RGB copied (C = 3), RGBA with each of
// R, G, B blended on black under the pixel's alpha (C = 4).  Sample (y, x, c) is at byte
// y rs + x ps + c cs of src; strides may be 0 (a broadcast view).  Launched over w x h.
struct IngestU8 {
  const uint8_t* src;
  long long rs, ps, cs;  // row, pixel and channel strides in bytes
  int C;
  uint8_t* rgb;  // [h][w][3]
  int w;
  GB_HD void operator()(int x, int y) const {
    const uint8_t* p = src + y * rs + x * ps;
    int r, g, b;
    if (C <= 2) {
      r = p[0];
      if (C == 2) r = blend_on_black(r, p[cs]);
      g = b = r;
    } else {
      r = p[0];
      g = p[cs];
      b = p[2 * cs];
      if (C == 4) {
        const int a = p[3 * cs];
        r = blend_on_black(r, a);
        g = blend_on_black(g, a);
        b = blend_on_black(b, a);
      }
    }
    uint8_t* o = rgb + 3 * (static_cast<size_t>(y) * w + x);
    o[0] = static_cast<uint8_t>(r);
    o[1] = static_cast<uint8_t>(g);
    o[2] = static_cast<uint8_t>(b);
  }
};

// ---------------------------------------------------------------------------
// JPEG decode as libjpeg-turbo decodes (jpeg_start_decompress with JDCT_ISLOW, fancy upsampling, RGB or
// gray output), N files of different sizes and samplings per launch.  Host side: jpeg_decode_rgb
// (pipeline.cu), which also lays out the buffers below.
//
// Every component of every file is one run of blocks of the call: coefficients [block][64] in natural
// order, and samples in a plane of 8 bw x 8 bh bytes (pitch 8 bw) that starts at byte 64 x its first block.
struct JpegDecFile {
  int w, h;          // image size
  int ncomp;         // 1 (gray) or 3
  int ycc;           // 3 components: 1 YCbCr, converted to RGB; 0 RGB, copied
  int hs, vs;        // the frame's maximum sampling (the first component's): 1x1, 2x1 or 2x2
  int blk0[4];       // first block of each component in the call; blk0[ncomp] ends the file's run
  int bw[3];         // blocks per row of each component
  int cw, ch;        // the chroma components' real size: ceil(w / hs) x ceil(h / vs)
  int row0;          // first output row of the file in the call's rows
  uint8_t* out;      // [h][w][3]
};

// the j with t0[j] <= v < t0[j + 1], for a non-decreasing t0[0 .. m] with t0[0] <= v < t0[m]
GB_HD int jpeg_find(const int* t0, int m, int v) {
  int lo = 0, hi = m;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (t0[mid] <= v) {
      lo = mid;
    } else {
      hi = mid;
    }
  }
  return lo;
}

// One 8x8 block per invocation, over all blocks of the call: jpeg_islow (jpeg_math.h) with the
// component's table (quant[3 f + c][64], natural order), into the component's plane.
struct JpegIdctIslow {
  const int16_t* coeffs;      // [blocks][64]
  const int* quant;           // [3 n][64]
  const JpegDecFile* files;   // [n]
  const int* file_blk0;       // [n + 1]: first block of each file, then the total
  int n;
  uint8_t* samples;           // 64 bytes per block
  GB_HD void operator()(int b) const {
    const int f = jpeg_find(file_blk0, n, b);
    const JpegDecFile& d = files[f];
    const int c = b >= d.blk0[1] ? (b >= d.blk0[2] ? 2 : 1) : 0;
    const int local = b - d.blk0[c], bw = d.bw[c];
    const int bx = local % bw, by = local / bw;
    uint8_t* out = samples + static_cast<size_t>(d.blk0[c]) * 64 + static_cast<size_t>(8 * by) * (8 * bw) + 8 * bx;
    jpeg_islow<false>(coeffs + static_cast<size_t>(b) * 64, quant + (3 * f + c) * 64, out, 8 * bw);
  }
};

// libjpeg's YCbCr -> RGB (jdcolor.c, build_ycc_rgb_table: SCALEBITS 16, ONE_HALF, FIX() of 1.40200,
// 1.77200, 0.71414 and 0.34414), clamped by the simple range-limit table.
GB_HD void jpeg_ycc_rgb(int y, int cb, int cr, uint8_t* o) {
  const int x_cb = cb - 128, x_cr = cr - 128, half = 1 << 15;
  const int r = y + ((91881 * x_cr + half) >> 16);
  const int g = y + ((-22554 * x_cb + half + -46802 * x_cr) >> 16);
  const int b = y + ((116130 * x_cb + half) >> 16);
  o[0] = static_cast<uint8_t>(r < 0 ? 0 : (r > 255 ? 255 : r));
  o[1] = static_cast<uint8_t>(g < 0 ? 0 : (g > 255 ? 255 : g));
  o[2] = static_cast<uint8_t>(b < 0 ? 0 : (b > 255 ? 255 : b));
}

// Output pixels of the call's rows: row yy of the call is row yy - row0 of file jpeg_find(file_row0, n,
// yy).  Invocation (lane, yy) writes pixels x = lane, lane + lanes, ... of that row.  Chroma is upsampled
// as jdsample.c does with do_fancy_upsampling: 2x1 by h2v1_fancy_upsample (3:1 weights, biases 1 and 2),
// 2x2 by h2v2_fancy_upsample (the 3:1 vertical sum, then 3:1 across with biases 8 and 7); the neighbour
// columns and rows beyond the chroma's real size cw x ch repeat its last one, and the row above the first
// is the first (jdmainct.c's context rows).  A chroma width of 1 or 2 is replicated instead
// (h2v1_upsample, h2v2_upsample), as libjpeg-turbo does at those widths.  Then jpeg_ycc_rgb, a copy for
// RGB files, or gray replicated.
struct JpegUpsampleYccRgb {
  const JpegDecFile* files;
  const int* file_row0;  // [n + 1]
  int n;
  const uint8_t* samples;
  int lanes;
  GB_HD int chroma(const JpegDecFile& d, const uint8_t* p, int x, int y) const {
    const int pitch = 8 * d.bw[1];
    const int j = x >> (d.hs - 1);
    if (d.hs == 1) return p[static_cast<size_t>(y) * pitch + x];
    if (d.cw <= 2) return p[static_cast<size_t>(y >> (d.vs - 1)) * pitch + j];
    const int jn = (x & 1) ? hd_min(j + 1, d.cw - 1) : hd_max(j - 1, 0);
    if (d.vs == 1) {
      const uint8_t* r = p + static_cast<size_t>(y) * pitch;
      return (3 * r[j] + r[jn] + 1 + (x & 1)) >> 2;
    }
    const int i = y >> 1, in = (y & 1) ? hd_min(i + 1, d.ch - 1) : hd_max(i - 1, 0);
    const uint8_t* r0 = p + static_cast<size_t>(i) * pitch;
    const uint8_t* r1 = p + static_cast<size_t>(in) * pitch;
    const int s = 3 * r0[j] + r1[j], sn = 3 * r0[jn] + r1[jn];
    return (3 * s + sn + ((x & 1) ? 7 : 8)) >> 4;
  }
  GB_HD void operator()(int lane, int yy) const {
    const int f = jpeg_find(file_row0, n, yy);
    const JpegDecFile& d = files[f];
    const int y = yy - d.row0;
    const uint8_t* yp = samples + static_cast<size_t>(d.blk0[0]) * 64 + static_cast<size_t>(y) * (8 * d.bw[0]);
    uint8_t* o = d.out + static_cast<size_t>(y) * d.w * 3;
    for (int x = lane; x < d.w; x += lanes) {
      const int v0 = yp[x];
      if (d.ncomp == 1) {
        o[3 * x] = o[3 * x + 1] = o[3 * x + 2] = static_cast<uint8_t>(v0);
        continue;
      }
      const int v1 = chroma(d, samples + static_cast<size_t>(d.blk0[1]) * 64, x, y);
      const int v2 = chroma(d, samples + static_cast<size_t>(d.blk0[2]) * 64, x, y);
      if (d.ycc) {
        jpeg_ycc_rgb(v0, v1, v2, o + 3 * x);
      } else {
        o[3 * x] = static_cast<uint8_t>(v0);
        o[3 * x + 1] = static_cast<uint8_t>(v1);
        o[3 * x + 2] = static_cast<uint8_t>(v2);
      }
    }
  }
};

// ---------------------------------------------------------------------------
// Entropy decoding of sequential scans on the device (jpeg_entropy_decode, pipeline.cu), for files whose
// first scan carries every component with Ss = 0, Se = 63, Ah = Al = 0.  Each functor restates a part of
// read_jpeg's scan() / first_pass() / ScanBits (jpeg_in.cc), so that a file decodes to read_jpeg's
// coefficients or is flagged in its status word and decoded on the host instead.
//
// Bytes: the call's scan bytes are one flat range, file f's readable ones (before len - 2, where
// ScanBits stops) at [byte0[f], byte0[f + 1]).  The segment pass compacts them, stuffed zeros and RSTn
// dropped, into one stream; restart interval I is bytes [cbyte, cbyte + nbytes) of it.

constexpr unsigned kJpegBadSegment = 1u;  // scan data does not end in EOI, or RSTn missing / out of order
constexpr unsigned kJpegBadCode = 2u;     // an error first_pass() / scan() raises, in the synchronised pass
constexpr unsigned kJpegBadRange = 4u;    // a block fails libjpeg_decodable's SIMD-range test
constexpr unsigned kJpegBadSync = 8u;     // the speculative decode did not converge within its rounds
constexpr int kJpegMaxSlots = 10;         // blocks per MCU

struct JpegScanFile {
  const uint8_t* data;  // the file
  long long len;
  int s0;               // first byte of entropy-coded data
  int int0, nint;       // the file's restart intervals in the call
  int R;                // restart interval in MCUs; 0 none
  int mcus, mcus_per_row;
  int nslot;            // blocks per MCU, in scan order
  int period;           // smallest p dividing nslot with slot s using slot s % p's tables: the decoder's states
                        // count slots modulo p, since the bits cannot tell slots with the same tables apart
  int slot_comp[kJpegMaxSlots], slot_ix[kJpegMaxSlots], slot_iy[kJpegMaxSlots];
  int slot_dc[kJpegMaxSlots], slot_ac[kJpegMaxSlots];  // lookup tables of the call
  int comp_h[3], comp_v[3], bw[3];  // MCU blocks per component (1 x 1 non-interleaved), blocks per row
  int blk0[3];                      // first block of each component in the coefficients
};

struct JpegInterval {
  long long cbyte;  // first compacted byte
  int nbytes;
  int file, mcu0, nmcu;
};

GB_HD bool jpeg_is_rst(int b) { return b >= 0xd0 && b <= 0xd7; }

// 4.1a: per scan byte, the first 0xFF followed by neither 0x00 nor RSTn ends the file's data (end[f] starts
// at len - 2, the file's last two bytes)
struct JpegSegEnd {
  const JpegScanFile* files;
  const int* byte0;  // [n + 1]
  int n;
  unsigned* end;
  GB_HD void operator()(int i) const {
    const int f = jpeg_find(byte0, n, i);
    const JpegScanFile& d = files[f];
    const long long p = d.s0 + (i - byte0[f]);
    if (d.data[p] != 0xff) return;
    const int nx = d.data[p + 1];
    if (nx != 0 && !jpeg_is_rst(nx)) hd_atomic_min(&end[f], static_cast<unsigned>(p));
  }
};

// 4.1b: per scan byte before the end: keep[i] = 1 for a data byte, rst[i] = 1 for the 0xFF of an RSTn
struct JpegSegFlags {
  const JpegScanFile* files;
  const int* byte0;
  int n;
  const unsigned* end;
  unsigned* keep;
  unsigned* rst;
  GB_HD void operator()(int i) const {
    const int f = jpeg_find(byte0, n, i);
    const JpegScanFile& d = files[f];
    const long long p = d.s0 + (i - byte0[f]);
    unsigned k = 0, r = 0;
    if (p < static_cast<long long>(end[f])) {
      const int b = d.data[p];
      const bool after_ff = p > d.s0 && d.data[p - 1] == 0xff;
      if (b == 0xff && jpeg_is_rst(d.data[p + 1])) {
        r = 1;
      } else if (!(after_ff && (b == 0 || jpeg_is_rst(b)))) {
        k = 1;
      }
    }
    keep[i] = k;
    rst[i] = r;
  }
};

// 4.1c: data bytes to their compacted place; RSTn to the start of the next interval, checked in order
struct JpegSegCompact {
  const JpegScanFile* files;
  const int* byte0;
  int n;
  const unsigned* keep;
  const unsigned* cpos;  // exclusive scan of keep
  const unsigned* rst;
  const unsigned* ridx;  // exclusive scan of rst
  uint8_t* comp;
  long long* istart;     // [intervals]: compacted start of each interval after the first
  unsigned* status;
  GB_HD void operator()(int i) const {
    const int f = jpeg_find(byte0, n, i);
    const JpegScanFile& d = files[f];
    const long long p = d.s0 + (i - byte0[f]);
    if (keep[i]) comp[cpos[i]] = d.data[p];
    if (rst[i]) {
      const unsigned r = ridx[i] - ridx[byte0[f]];
      if (static_cast<int>(r) + 1 < d.nint && d.data[p + 1] == 0xd0 + (r & 7)) {
        istart[d.int0 + r + 1] = cpos[i];
      } else {
        hd_atomic_or(&status[f], kJpegBadSegment);
      }
    }
  }
};

// 4.1d: per interval, its bytes and MCUs, and its number of subsequences of S bits; the first interval of
// a file also checks that the data ends in EOI with one RSTn between each two intervals
struct JpegIntervals {
  const JpegScanFile* files;
  const int* byte0;
  const int* int0;  // [n + 1]
  int n;
  const unsigned* end;
  const unsigned* cpos;
  const unsigned* ridx;
  const long long* istart;
  int S;
  JpegInterval* ivs;
  unsigned* nsub;
  unsigned* status;
  GB_HD void operator()(int I) const {
    const int f = jpeg_find(int0, n, I);
    const JpegScanFile& d = files[f];
    const int k = I - d.int0, nb = byte0[f + 1] - byte0[f];
    const long long e = end[f];
    const int at_end = static_cast<int>(hd_min(hd_max(e - d.s0, 0LL), static_cast<long long>(nb)));
    const long long fs = cpos[byte0[f]], fe = cpos[byte0[f] + at_end];
    long long a = k == 0 ? fs : istart[I];
    long long b = k == d.nint - 1 ? fe : istart[I + 1];
    a = hd_min(hd_max(a, fs), fe);
    b = hd_min(hd_max(b, a), fe);
    JpegInterval iv;
    iv.cbyte = a;
    iv.nbytes = static_cast<int>(b - a);
    iv.file = f;
    iv.mcu0 = d.R > 0 ? k * d.R : 0;
    iv.nmcu = d.R > 0 ? hd_min(d.R, d.mcus - k * d.R) : d.mcus;
    ivs[I] = iv;
    const long long bits = 8LL * iv.nbytes;
    nsub[I] = static_cast<unsigned>(hd_max(1LL, (bits + S - 1) / S));
    if (k == 0) {
      const bool eoi = nb > 0 && e + 1 < d.len && d.data[e] == 0xff && d.data[e + 1] == 0xd9;
      const unsigned rsts = ridx[byte0[f + 1]] - ridx[byte0[f]];
      if (!eoi || static_cast<int>(rsts) != d.nint - 1) hd_atomic_or(&status[f], kJpegBadSegment);
    }
  }
};

// Decoder state at a subsequence boundary: bit offset in the interval, block slot in the MCU modulo the
// file's period, zig-zag index in the block (0: the DC symbol is next), and an error mark.
GB_HD unsigned long long jpeg_state(unsigned pos, int slot, int zz) {
  return pos | (static_cast<unsigned long long>(slot) << 32) | (static_cast<unsigned long long>(zz) << 40);
}
constexpr unsigned long long kJpegStateError = 1ull << 48;

// One DHT table for the decoder: decode_symbol (jpeg_in.cc) on the first 9 bits of a window in `fast`, bit 15
// set for a symbol with its code length in bits 8..12 and the symbol in bits 0..7, bit 14 set where
// decode_symbol gives -1 within 9 bits, 0 where it reads on; from there on decode_symbol's own walk over
// lengths 10 to 16.
struct JpegHuffDev {
  uint16_t fast[512];
  int max_code[18], val_offset[18];
  int num_symbols;
  uint8_t symbols[256];
};

// decode_symbol on the 32 bits w (the first at bit 31): false for -1, else the symbol and its code length
GB_HD bool jpeg_decode_symbol(const JpegHuffDev& t, unsigned w, int* sym, int* len) {
  const uint16_t e = t.fast[w >> 23];
  if (e & 0x8000) {
    *len = (e >> 8) & 31;
    *sym = e & 255;
    return true;
  }
  if (e & 0x4000) return false;
  for (int l = 10; l <= 16; ++l) {
    const int code = static_cast<int>(w >> (32 - l));
    if (t.max_code[l] >= 0 && code <= t.max_code[l]) {
      const int idx = t.val_offset[l] + code;
      if (idx >= t.num_symbols) return false;
      *len = l;
      *sym = t.symbols[idx];
      return true;
    }
  }
  return false;
}

// Decodes subsequence bits [start, stop) of one interval from state `in`.  first_pass() for Ss = 0,
// Se = 63, Al = 0, symbol by symbol: with `coeffs`, blocks b0, b0 + 1, ... are written (DC as the
// difference) until block `total` is reached, and *end_bit is where that happened; without, only the
// exit state and the number of blocks completed are computed.  Returns the exit state.
struct JpegSubDecoder {
  const JpegScanFile& d;
  const JpegInterval& iv;
  const JpegHuffDev* luts;
  const uint8_t* comp;
  GB_HD unsigned peek32(unsigned pos) const {
    const uint8_t* p = comp + iv.cbyte;
    const unsigned nb = static_cast<unsigned>(iv.nbytes);
    const unsigned byte = pos >> 3;
    unsigned long long w = 0;
    for (unsigned k = 0; k < 5; ++k) w = (w << 8) | (byte + k < nb ? p[byte + k] : 0u);
    return static_cast<unsigned>((w << (24 + (pos & 7))) >> 32);
  }
  GB_HD unsigned long long run(unsigned long long in, unsigned stop, unsigned* blocks, int16_t* coeffs,
                               const uint8_t* zz_nat, int b0, int total, unsigned* end_bit, bool* bad) const {
    unsigned pos = static_cast<unsigned>(in);
    int slot = static_cast<int>((in >> 32) & 0xff), zz = static_cast<int>((in >> 40) & 0xff);
    const unsigned nbits = 8u * static_cast<unsigned>(iv.nbytes);
    int b = b0;
    unsigned done = 0;
    while (pos < stop) {
      if (coeffs && b >= total) break;
      const unsigned w = peek32(pos);
      int l = 0, sym = 0;
      if (!jpeg_decode_symbol(luts[zz == 0 ? d.slot_dc[slot] : d.slot_ac[slot]], w, &sym, &l)) goto fail;
      {
        const int sz = zz == 0 ? sym : (sym & 15);
        if (zz == 0 ? sz > 11 : (sz >= 12)) goto fail;
        const unsigned v = sz ? ((w << l) >> (32 - sz)) : 0u;
        pos += l + sz;
        if (pos > nbits) goto fail;
        const int val = sz ? (v < (1u << (sz - 1)) ? static_cast<int>(v) - (1 << sz) + 1 : static_cast<int>(v)) : 0;
        bool block_end = false;
        int16_t* blk = nullptr;
        if (coeffs) {
          // the block's own slot: b counts from the interval's start, where slot 0 is
          const int ts = b % d.nslot, m = iv.mcu0 + b / d.nslot, c = d.slot_comp[ts];
          const int mx = m % d.mcus_per_row, my = m / d.mcus_per_row;
          const size_t at = static_cast<size_t>(d.blk0[c]) +
                            static_cast<size_t>(my * d.comp_v[c] + d.slot_iy[ts]) * d.bw[c] + mx * d.comp_h[c] +
                            d.slot_ix[ts];
          blk = coeffs + at * 64;
        }
        if (zz == 0) {
          if (blk) blk[0] = static_cast<int16_t>(val);
          zz = 1;
        } else {
          const int run = sym >> 4;
          if (sz > 0) {
            const int k = zz + run;
            if (k > 63) goto fail;
            if (blk) blk[zz_nat[k]] = static_cast<int16_t>(val);
            zz = k + 1;
          } else if (run == 15) {
            zz += 16;
          } else if (run > 0) {
            goto fail;  // an end-of-block run in a sequential scan
          } else {
            block_end = true;
          }
          if (zz > 63) block_end = true;
        }
        if (block_end) {
          zz = 0;
          slot = slot + 1 == d.period ? 0 : slot + 1;
          ++b;
          ++done;
          if (coeffs && b == total) *end_bit = pos;
        }
      }
    }
    *blocks = done;
    return jpeg_state(pos, slot, zz);
  fail:
    *blocks = done;
    *bad = true;
    return jpeg_state(pos, slot, zz) | kJpegStateError;
  }
};

// The subsequences of the call: interval I has nsub[I] of them, from sub0[I] on; subsequence j of an
// interval covers bits [j S, (j + 1) S), the last one up to the interval's end.
struct JpegSubs {
  const JpegScanFile* files;
  const JpegInterval* ivs;
  int nint;
  const unsigned* sub0;  // [nint + 1]
  const JpegHuffDev* luts;
  const uint8_t* comp;
  int S;
  GB_HD bool locate(int t, int* I, int* j, unsigned* stop) const {
    if (static_cast<unsigned>(t) >= sub0[nint]) return false;
    *I = jpeg_find(reinterpret_cast<const int*>(sub0), nint, t);
    *j = t - static_cast<int>(sub0[*I]);
    const unsigned nbits = 8u * static_cast<unsigned>(ivs[*I].nbytes);
    const bool last = static_cast<unsigned>(t) + 1 == sub0[*I + 1];
    *stop = last ? nbits : static_cast<unsigned>(*j + 1) * static_cast<unsigned>(S);
    return true;
  }
};

// 4.2, one round of the speculative decode.  Round 0 decodes every subsequence from the interval's start
// (its first) or from a guess (an AC symbol of slot 0 at its first bit).  Each later round redoes
// subsequence j from the exit state subsequence j - 1 had in the round before (a guess again after an
// error), where that differs from what j started from last time.  States are read from one buffer and
// written to the other, so a round's result does not depend on the order its invocations run in.  Once a
// round changes no exit state, every subsequence started from the exact state; that holds file by file,
// so after the last round the pipeline allows (jpeg_max_sync_rounds), the files whose states still changed are flagged in
// `status` (null before) and decoded on the host.
struct JpegHuffSync {
  JpegSubs subs;
  int round;
  const unsigned long long* exit_in;
  unsigned long long* exit_out;
  unsigned long long* entry;  // the state each subsequence started from
  unsigned* count;            // blocks completed in each subsequence
  unsigned* changed;
  unsigned* status;
  GB_HD void operator()(int t) const {
    int I, j;
    unsigned stop;
    if (!subs.locate(t, &I, &j, &stop)) return;
    const JpegInterval& iv = subs.ivs[I];
    unsigned long long in = jpeg_state(0, 0, 0);
    if (j > 0) {
      in = round == 0 ? kJpegStateError : exit_in[t - 1];
      if (in & kJpegStateError) in = jpeg_state(static_cast<unsigned>(j) * subs.S, 0, 1);
    }
    if (round > 0 && in == entry[t]) {
      exit_out[t] = exit_in[t];
      return;
    }
    entry[t] = in;
    const JpegSubDecoder dec{subs.files[iv.file], iv, subs.luts, subs.comp};
    unsigned blocks = 0, end_bit = 0;
    bool bad = false;
    const unsigned long long out = dec.run(in, stop, &blocks, nullptr, nullptr, 0, 0, &end_bit, &bad);
    exit_out[t] = out;
    count[t] = blocks;
    if (round > 0 && out != exit_in[t]) {
      hd_atomic_or(changed, 1u);
      if (status) hd_atomic_or(&status[iv.file], kJpegBadSync);
    }
  }
};

// 4.2, the write pass: every subsequence from its exact state writes its blocks' coefficients (DC as the
// difference); an error in a block the interval needs, an interval that ends early, or one whose last
// block leaves whole bytes before its RSTn flags the file
struct JpegHuffWrite {
  JpegSubs subs;
  const unsigned long long* entry;
  const unsigned* bscan;  // exclusive scan of the blocks completed per subsequence
  const uint8_t* zz_nat;
  int16_t* coeffs;
  unsigned* status;
  GB_HD void operator()(int t) const {
    int I, j;
    unsigned stop;
    if (!subs.locate(t, &I, &j, &stop)) return;
    const JpegInterval& iv = subs.ivs[I];
    const JpegScanFile& d = subs.files[iv.file];
    const int total = iv.nmcu * d.nslot;
    const int b0 = static_cast<int>(bscan[t] - bscan[subs.sub0[I]]);
    if (b0 >= total) return;
    const JpegSubDecoder dec{d, iv, subs.luts, subs.comp};
    unsigned blocks = 0, end_bit = 0xffffffffu;
    bool bad = false;
    dec.run(entry[t], stop, &blocks, coeffs, zz_nat, b0, total, &end_bit, &bad);
    const bool last_sub = static_cast<unsigned>(t) + 1 == subs.sub0[I + 1];
    const bool last_interval = I == d.int0 + d.nint - 1;
    if (end_bit != 0xffffffffu) {
      // bytes consumed: the next RSTn must follow at once (read_jpeg: "Marker byte (0xff) expected")
      if (!last_interval && (end_bit + 7) / 8 != static_cast<unsigned>(iv.nbytes)) bad = true;
    } else if (last_sub && !bad) {
      bad = true;  // the interval's data ran out before its last block
    }
    if (bad) hd_atomic_or(&status[iv.file], kJpegBadCode);
  }
};

// DC differences -> values by a prefix sum per (interval, component), in chunks of kJpegDcChunk blocks:
// block k of a task is the k-th block of that component in the interval's MCUs
constexpr int kJpegDcChunk = 64;
struct JpegDcTask {
  int file, interval, c, nblk;
};
GB_HD int16_t* jpeg_dc_block(const JpegScanFile& d, const JpegInterval& iv, int c, int k, int16_t* coeffs) {
  const int per = d.comp_h[c] * d.comp_v[c];
  const int m = iv.mcu0 + k / per, w = k % per;
  const int mx = m % d.mcus_per_row, my = m / d.mcus_per_row;
  const size_t at = static_cast<size_t>(d.blk0[c]) + static_cast<size_t>(my * d.comp_v[c] + w / d.comp_h[c]) * d.bw[c] +
                    mx * d.comp_h[c] + w % d.comp_h[c];
  return coeffs + at * 64;
}
struct JpegDcChunkSum {
  const JpegScanFile* files;
  const JpegInterval* ivs;
  const JpegDcTask* tasks;
  const int* chunk0;  // [ntask + 1]
  int ntask;
  int16_t* coeffs;
  unsigned* sums;
  GB_HD void operator()(int g) const {
    const int t = jpeg_find(chunk0, ntask, g);
    const JpegDcTask& task = tasks[t];
    const int k0 = (g - chunk0[t]) * kJpegDcChunk, k1 = hd_min(k0 + kJpegDcChunk, task.nblk);
    unsigned s = 0;
    for (int k = k0; k < k1; ++k)
      s += static_cast<unsigned>(static_cast<int>(jpeg_dc_block(files[task.file], ivs[task.interval], task.c, k,
                                                                coeffs)[0]));
    sums[g] = s;
  }
};
// every running value checked against int16, as first_pass checks it
struct JpegDcChunkApply {
  const JpegScanFile* files;
  const JpegInterval* ivs;
  const JpegDcTask* tasks;
  const int* chunk0;
  int ntask;
  int16_t* coeffs;
  const unsigned* scan;  // exclusive scan of the chunk sums
  unsigned* status;
  GB_HD void operator()(int g) const {
    const int t = jpeg_find(chunk0, ntask, g);
    const JpegDcTask& task = tasks[t];
    const int k0 = (g - chunk0[t]) * kJpegDcChunk, k1 = hd_min(k0 + kJpegDcChunk, task.nblk);
    int v = static_cast<int>(scan[g] - scan[chunk0[t]]);
    bool bad = false;
    for (int k = k0; k < k1; ++k) {
      int16_t* blk = jpeg_dc_block(files[task.file], ivs[task.interval], task.c, k, coeffs);
      v += blk[0];
      if (!jpeg_fits16(v)) bad = true;
      blk[0] = static_cast<int16_t>(v);
    }
    if (bad) hd_atomic_or(&status[task.file], kJpegBadCode);
  }
};

// 3: libjpeg_decodable's SIMD-range test (jpeg_in.cc) on every block of the files marked in `check`
struct JpegRangeCheck {
  const int16_t* coeffs;
  const int* quant;          // [3 n][64]
  const JpegDecFile* files;
  const int* file_blk0;      // [n + 1]
  int n;
  const int* check;          // [n]
  unsigned* status;
  GB_HD void operator()(int b) const {
    const int f = jpeg_find(file_blk0, n, b);
    if (!check[f]) return;
    const JpegDecFile& d = files[f];
    const int c = b >= d.blk0[1] ? (b >= d.blk0[2] ? 2 : 1) : 0;
    const int16_t* blk = coeffs + static_cast<size_t>(b) * 64;
    const int* q = quant + (3 * f + c) * 64;
    long long t = 0;
    for (int k = 0; k < 64; ++k) t += static_cast<long long>(blk[k] < 0 ? -blk[k] : blk[k]) * q[k];
    if (t > 2040 && !jpeg_islow<true>(blk, q, nullptr, 0)) hd_atomic_or(&status[f], kJpegBadRange);
  }
};

// The encoder's JPEG input from one device-decoded 4:4:4 file, per coefficient of [3][nblocks][64]:
// RemoveOriginalQuantization (g/processor.cc:82), dq = coef * q, and CheckJpegSanity's bound (:106),
// |coef * q| <= 4096 as a 64-bit product, whose breach flags the file (kJpegBadSanity).  The int16 store
// is exact wherever the bound holds, and the encoder reads dq only then.
constexpr unsigned kJpegBadSanity = 16u;
struct JpegDequantSanity {
  const int16_t* coeffs;  // [3][nblocks][64], quantised, natural order
  const int* quant;       // [3][64], natural order
  int nblocks;
  int16_t* dq;
  unsigned* status;
  GB_HD void operator()(int i) const {
    const long long v = static_cast<long long>(coeffs[i]) * quant[(i / (64 * nblocks)) * 64 + (i & 63)];
    dq[i] = static_cast<int16_t>(v);
    if (v > 4096 || v < -4096) hd_atomic_or(status, kJpegBadSanity);
  }
};

// Original image u8 sRGB -> linear float planes (g/butteraugli_comparator.cc:33).
struct LinearizeRgb {
  const uint8_t* rgb;
  float* lin;  // [3][h][pitch]
  Geom g;
  const float* lut;
  GB_HD void operator()(int x, int y) const {
    const uint8_t* p = rgb + 3 * (static_cast<size_t>(y) * g.w + x);
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    lin[o] = lut[p[0]];
    lin[g.plane + o] = lut[p[1]];
    lin[2 * g.plane + o] = lut[p[2]];
  }
};

// The stand-alone `butteraugli` tool's input pixel (FromSrgbToLinear, b/butteraugli_main.cc:239-281):
// u8 p[0 .. C) -> linear o[0], o[plane], o[2 plane].  C = 4: the pixel is laid over `background` in sRGB
// space first, in integers: alpha 255 keeps it, alpha 0 gives the background, any other alpha
// (v a + background (255 - a) + 127) / 255.  lut: Tables::srgb_lin, which equals the tool's table once
// both are rounded to float.
GB_HD void srgb_over_linear(const uint8_t* p, int C, int background, const float* lut, float* o, size_t plane) {
  const int a = C == 4 ? p[3] : 255;
  for (int c = 0; c < 3; ++c) {
    int v = p[c];
    if (a == 0) {
      v = background;
    } else if (a != 255) {
      v = (v * a + background * (255 - a) + 127) / 255;
    }
    o[c * plane] = lut[v];
  }
}

// u8 sRGB images interleaved [n][h][w][C] -> linear planes [n][3][h][pitch], each pixel by
// srgb_over_linear.  Launched over w x n*h.
struct SrgbToLinear {
  const uint8_t* src;
  int C, background;
  float* dst;
  int w, h, pitch;
  const float* lut;
  GB_HD void operator()(int x, int yy) const {
    const int i = yy / h, y = yy - i * h;
    const size_t plane = static_cast<size_t>(h) * pitch;
    srgb_over_linear(src + (static_cast<size_t>(yy) * w + x) * C, C, background, lut,
                     dst + 3 * plane * i + static_cast<size_t>(y) * pitch + x, plane);
  }
};

// ScoreToRgb's colour table (b/butteraugli.cc:1940), rows 0..9 as halves (0, 1 or 2) of r, g and b, six bits
// a row; rows 10 and 11 are white
constexpr unsigned long long heat_row(int row, int r, int g, int b) {
  return static_cast<unsigned long long>(r | g << 2 | b << 4) << (6 * row);
}
constexpr unsigned long long kHeatHalves = heat_row(0, 0, 0, 0) | heat_row(1, 0, 0, 2) | heat_row(2, 0, 2, 2) |
                                           heat_row(3, 0, 2, 0) | heat_row(4, 2, 2, 0) | heat_row(5, 2, 0, 0) |
                                           heat_row(6, 2, 0, 2) | heat_row(7, 1, 1, 2) | heat_row(8, 2, 1, 1) |
                                           heat_row(9, 2, 2, 1);
GB_HD double heat_level(int row, int c) {
  return 0.5 * (row >= 10 ? 2 : static_cast<int>((kHeatHalves >> (6 * row + 2 * c)) & 3));
}

// ScoreToRgb (b/butteraugli.cc:1938) in its double arithmetic and order, up to v.  Its byte
// (uint8_t)(255 * pow(v, 0.5) + 0.5) is the largest k with steps[k] <= v, steps the host-pow table
// heat_byte_steps() (tables.h): IEEE sqrt differs from the host's pow in one byte (DESIGN.md §3).  NaN scores have
// no defined colour.
GB_HD void score_to_rgb(double score, double good, double bad, const double* steps, uint8_t* rgb) {
  if (score < good) {
    score = (score / good) * 0.3;
  } else if (score < bad) {
    score = 0.3 + (score - good) / (bad - good) * 0.15;
  } else {
    score = 0.45 + (score - bad) / (bad * 12) * 0.5;
  }
  score = hd_min<double>(hd_max<double>(score * 11, 0.0), 10);
  const int ix = static_cast<int>(score);
  const double mix = score - ix;
  for (int i = 0; i < 3; ++i) {
    const double v = mix * heat_level(ix + 1, i) + (1 - mix) * heat_level(ix, i);
    int k = 0;
    for (int step = 128; step > 0; step >>= 1)
      if (k + step <= 255 && steps[k + step] <= v) k += step;
    rgb[i] = static_cast<uint8_t>(k);
  }
}

// CreateHeatMapImage (b/butteraugli.cc:1979) of n diffmaps of sizes of their own, flat over all their pixels:
// pixel i of the call is pixel i - px0[f] of map f = jpeg_find(px0, n, i), map f [h][w] floats into rgb[f]
// [h][w][3] bytes.
struct HeatMap {
  const float* const* dm;
  uint8_t* const* rgb;
  const int* px0;        // [n + 1]
  const double* steps;   // [256] heat_byte_steps()
  int n;
  double good, bad;
  GB_HD void operator()(int i) const {
    const int f = jpeg_find(px0, n, i);
    const int p = i - px0[f];
    score_to_rgb(dm[f][p], good, bad, steps, rgb[f] + 3 * static_cast<size_t>(p));
  }
};

// a8: ApplyGlobalQuantization on top of CopyFromJpegData with unit quant
// (g/output_image.cc:211-243): cand = Quantize(orig, q[c][k]).
struct QuantizeCoeffs {
  const int16_t* orig;
  int16_t* cand;
  const int* q;  // [192] device
  int nblocks;
  GB_HD void operator()(int i) const {  // i over 3*nblocks*64
    const int k = i & 63;
    const int c = i / (nblocks * 64);
    cand[i] = static_cast<int16_t>(quantize_coeff(orig[i], q[c * 64 + k]));
  }
};

// Sparse coefficient edits produced by the selection walk (g/processor.cc:732-735).
struct ScatterCoeffs {
  const int* index;      // flat index into [3][nblocks][64]
  const int16_t* value;
  int16_t* cand;
  GB_HD void operator()(int i) const { cand[index[i]] = value[i]; }
};

// a7+a9: coefficients -> IDCT -> YCbCr u8 -> RGB u8 -> linear float planes, one
// 8x8 block per invocation (g/idct.cc:139, g/output_image.cc:134-145,411-436,
// g/color_transform.h:211).  Pixels outside the image are not stored.
struct RenderBlocks {
  const int16_t* cand;  // dequantised coefficients
  float* lin;           // [3][h][pitch]
  Geom g;
  Tables t;
  GB_HD void operator()(int b) const {
    const int bx = b % g.bw, by = b / g.bw;
    uint8_t px[3][64];
    for (int c = 0; c < 3; ++c)
      idct_8x8(t.idct, cand + (static_cast<size_t>(c) * g.nblocks + b) * 64, px[c]);
    for (int iy = 0; iy < 8; ++iy) {
      const int y = 8 * by + iy;
      if (y >= g.h) break;
      for (int ix = 0; ix < 8; ++ix) {
        const int x = 8 * bx + ix;
        if (x >= g.w) break;
        int r, gg, bb;
        ycc_to_rgb(t.cr_r, t.cb_b, t.cr_g, t.cb_g, px[0][8 * iy + ix], px[1][8 * iy + ix],
                   px[2][8 * iy + ix], &r, &gg, &bb);
        const size_t o = static_cast<size_t>(y) * g.pitch + x;
        lin[o] = t.srgb_lin[r];
        lin[g.plane + o] = t.srgb_lin[gg];
        lin[2 * g.plane + o] = t.srgb_lin[bb];
      }
    }
  }
};

// JPEG input: sRGB bytes of the decoded original (DecodeJpegToRGB for 4:4:4 input,
// g/jpeg_data_decoder.cc:45 -> OutputImage::ToSRGB): IDCT of the dequantised
// coefficients and the integer colour transform, image-sized interleaved u8.
struct RenderRgb8 {
  const int16_t* coeffs;
  uint8_t* rgb;  // [h][w][3]
  Geom g;
  Tables t;
  GB_HD void operator()(int b) const {
    const int bx = b % g.bw, by = b / g.bw;
    uint8_t px[3][64];
    for (int c = 0; c < 3; ++c)
      idct_8x8(t.idct, coeffs + (static_cast<size_t>(c) * g.nblocks + b) * 64, px[c]);
    for (int iy = 0; iy < 8; ++iy) {
      const int y = 8 * by + iy;
      if (y >= g.h) break;
      for (int ix = 0; ix < 8; ++ix) {
        const int x = 8 * bx + ix;
        if (x >= g.w) break;
        int r, gg, bb;
        ycc_to_rgb(t.cr_r, t.cb_b, t.cr_g, t.cb_g, px[0][8 * iy + ix], px[1][8 * iy + ix],
                   px[2][8 * iy + ix], &r, &gg, &bb);
        uint8_t* o = rgb + 3 * (static_cast<size_t>(y) * g.w + x);
        o[0] = static_cast<uint8_t>(r);
        o[1] = static_cast<uint8_t>(gg);
        o[2] = static_cast<uint8_t>(bb);
      }
    }
  }
};

// The same for a list of blocks (only blocks whose coefficients changed since the
// last render need new pixels: SetCoeffBlock's incremental update,
// g/output_image.cc:123-145).
struct RenderBlockList {
  RenderBlocks r;
  const int* list;
  GB_HD void operator()(int i) const { r(list[i]); }
};

// ---------------------------------------------------------------------------
// Separable blur (b/butteraugli.cc:184-233), split into an x pass and a y pass.
// Both take a group of `n` contiguous planes (launched over w x n*h).
struct BlurRowAt {
  const float* row;
  GB_HD float operator()(int j) const { return row[j]; }
};
struct BlurColAt {
  const float* col;
  int pitch;
  GB_HD float operator()(int j) const { return col[static_cast<size_t>(j) * pitch]; }
};

struct BlurX {
  const float* in;
  float* out;
  BlurTab tab;
  Geom g;
  GB_HD void operator()(int x, int yy) const {  // yy over n*h
    const size_t ro = static_cast<size_t>(yy) * g.pitch;
    BlurRowAt at{in + ro};
    out[ro + x] = blur_tap_sum(at, tab.taps, tab.taps_n, tab.scale_x, tab.r, x, g.w);
  }
};

struct BlurY {
  const float* in;
  float* out;
  BlurTab tab;
  Geom g;
  GB_HD void operator()(int x, int yy) const {
    const int pl = yy / g.h, y = yy - pl * g.h;
    const size_t base = static_cast<size_t>(pl) * g.plane + x;
    BlurColAt at{in + base, g.pitch};
    out[base + static_cast<size_t>(y) * g.pitch] =
        blur_tap_sum(at, tab.taps, tab.taps_n, tab.scale_y, tab.r, y, g.h);
  }
};

// OpsinDynamicsImage per pixel (b/butteraugli.cc:332-364).
struct OpsinPx {
  const float* rgb;      // [3] sharp
  const float* blurred;  // [3]
  float* xyb;            // [3]
  Geom g;
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    opsin_pixel(rgb[o], rgb[g.plane + o], rgb[2 * g.plane + o], blurred[o],
                blurred[g.plane + o], blurred[2 * g.plane + o], &xyb[o], &xyb[g.plane + o],
                &xyb[2 * g.plane + o]);
  }
};

// ---------------------------------------------------------------------------
// SeparateFrequencies (b/butteraugli.cc:489-622).  PsychoImage plane order in
// one contiguous group of 10: uhf[X,Y], hf[X,Y], mf[X,Y,B], lf[X,Y,B].
enum PsychoPlane { kUhfX = 0, kUhfY, kHfX, kHfY, kMfX, kMfY, kMfB, kLfX, kLfY, kLfB, kPsychoPlanes };
// planes of an original that a comparator set stores (k_mix_original): the Compare chain reads every
// plane of its PsychoImage but mf[B] and lf[Y], and its two DiffPrecompute neighbour sums
constexpr int kStoredPlanes = kPsychoPlanes - 2 + 2;

// mf = xyb - lf for 3 planes (:509-513); launched over w x 3h.
struct SubPlanes {
  const float* a;
  const float* b;
  float* out;
  Geom g;
  GB_HD void operator()(int x, int yy) const {
    const size_t o = static_cast<size_t>(yy) * g.pitch + x;
    out[o] = a[o] - b[o];
  }
};

// After mfb = Blur(mf): split into hf and mf with the range tweaks (:518-553),
// then SuppressXByY on hf[X] (:555-556).  Writes hf_raw[X,Y] (pre-blur hf) and
// the final mf[X,Y,B].
struct SplitMfHf {
  const float* mf_in;   // [3] xyb - lf
  const float* mf_blr;  // [3] blurred
  float* ps;            // PsychoImage group (writes mf*)
  float* hf_raw;        // [2] hf before the UHF split
  Geom g;
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    const float mbx = mf_blr[o], mby = mf_blr[g.plane + o];
    const float hx = mf_in[o] - mbx;
    const float hy = mf_in[g.plane + o] - mby;
    ps[kMfX * g.plane + o] = remove_range_around_zero(static_cast<float>(0.120079806822), mbx);
    ps[kMfY * g.plane + o] = amplify_range_around_zero(static_cast<float>(0.03430529365), mby);
    ps[kMfB * g.plane + o] = mf_blr[2 * g.plane + o];
    hf_raw[o] = suppress_x_by_y(hx, hy);
    hf_raw[g.plane + o] = hy;
  }
};

// After hfb = Blur(hf_raw): uhf/hf split and post-processing (:558-605), and the
// lf -> "vals" conversion (:610-621, XybLowFreqToVals :381).
struct SplitHfUhf {
  const float* hf_raw;  // [2]
  const float* hf_blr;  // [2]
  const float* lf_raw;  // [3] blurred xyb (before the vals conversion)
  float* ps;
  Geom g;
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    // X
    {
      const float hb = hf_blr[o];
      ps[kUhfX * g.plane + o] = hf_raw[o] - hb;
      ps[kHfX * g.plane + o] = remove_range_around_zero(static_cast<float>(0.0287615200377), hb);
    }
    const float lfx = lf_raw[o], lfy = lf_raw[g.plane + o], lfb = lf_raw[2 * g.plane + o];
    // Y
    {
      const float kMulSuppressHf = static_cast<float>(1.10684769012);
      const float kMulRegHf = static_cast<float>(0.478741530298);
      const float kRegHf = 2000 * kMulRegHf;
      const float kMulSuppressUhf = static_cast<float>(1.76905001176);
      const float kMulRegUhf = static_cast<float>(0.310148420674);
      const float kRegUhf = 2000 * kMulRegUhf;
      const float hb = hf_blr[g.plane + o];
      float uhf = hf_raw[g.plane + o] - hb;
      float hf = maximum_clamp(hb, static_cast<float>(78.8223237675));
      uhf = maximum_clamp(uhf, static_cast<float>(5.8907152736));
      uhf = suppress_in_bright_areas(uhf, lfy, kMulSuppressUhf, kRegUhf);
      hf = suppress_in_bright_areas(hf, lfy, kMulSuppressHf, kRegHf);
      ps[kUhfY * g.plane + o] = uhf;
      ps[kHfY * g.plane + o] = hf;
    }
    // lf -> vals
    {
      const float xmul = static_cast<float>(5.57547552483);
      const float ymul = static_cast<float>(1.20828034498);
      const float bmul = static_cast<float>(6.08319517575);
      const float y_to_b_mul = static_cast<float>(-0.628811683685);
      const float bb = lfb + y_to_b_mul * lfy;
      ps[kLfB * g.plane + o] = bb * bmul;
      ps[kLfX * g.plane + o] = lfx * xmul;
      ps[kLfY * g.plane + o] = lfy * ymul;
    }
  }
};

// ---------------------------------------------------------------------------
// Malta (b/butteraugli.cc:1461-1568).
struct MaltaPre {
  const float* lum0;
  const float* lum1;
  float* diffs;
  MaltaParams mp;
  Geom g;
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    diffs[o] = malta_diff(lum0[o], lum1[o], mp);
  }
};

// acc += sum over 16 line patterns of (sum of taps)^2, zero outside the image
// (PaddedMaltaUnit :1429).  LF: 5 taps per line; HF: 7..9.
struct MaltaAcc {
  const float* diffs;
  float* acc;
  const unsigned char* pat;      // [16][stride]
  const unsigned char* pat_len;  // [16] or null (=> stride taps)
  int stride;
  int first;  // 1 => acc = value (first term of the 0-initialised plane), else +=
  Geom g;
  GB_HD void operator()(int x, int y) const {
    float retval = 0;
    for (int p = 0; p < 16; ++p) {
      const int n = pat_len ? pat_len[p] : stride;
      float sum = 0.0f;
      for (int k = 0; k < n; ++k) {
        const int code = pat[p * stride + k];
        const int dy = code / 9 - 4, dx = code % 9 - 4;
        const int xx = x + dx, yy = y + dy;
        float v = 0.0f;
        if (xx >= 0 && xx < g.w && yy >= 0 && yy < g.h) v = diffs[static_cast<size_t>(yy) * g.pitch + xx];
        sum = (k == 0) ? v : sum + v;
      }
      retval += sum * sum;
    }
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    acc[o] = first ? (0.0f + retval) : (acc[o] + retval);
  }
};

// SameNoiseLevels (:624-652)
struct NoisePre {
  const float* i0;
  const float* i1;
  float* out;
  Geom g;
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    const double maxclamp = 85.7047444518;
    double v0 = hd_fabsf(i0[o]);
    double v1 = hd_fabsf(i1[o]);
    if (v0 > maxclamp) v0 = maxclamp;
    if (v1 > maxclamp) v1 = maxclamp;
    out[o] = static_cast<float>(v0 - v1);
  }
};

// ac[Y] += w*blurred^2 (SameNoiseLevels tail), then L2DiffAsymmetric(hf[Y])
// (:672-714, weights 32.4449876135*0.8 and /0.8 from :866,893).
struct NoiseAndAsymAcc {
  const float* blurred;
  const float* hf0;  // pi0.hf[Y]
  const float* hf1;  // pi1.hf[Y]
  float* acc;        // block_diff_ac[Y]
  double w_0gt1, w_0lt1;  // already multiplied by the inner 0.8
  Geom g;
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    float a = acc[o];
    {
      const double w = 884.809801415;
      const double diff = blurred[o];
      a = static_cast<float>(static_cast<double>(a) + w * diff * diff);
    }
    const float r0 = hf0[o], r1f = hf1[o];
    {
      const double diff = r0 - r1f;  // float subtraction, then widened
      a = static_cast<float>(static_cast<double>(a) + w_0gt1 * diff * diff);
      const double fabs0 = hd_fabsf(r0);
      const double too_small = 0.4 * fabs0;
      const double too_big = 1.0 * fabs0;
      const double r1 = r1f;
      if (r0 < 0) {
        if (r1 > -too_small) {
          const double v = r1 + too_small;
          a = static_cast<float>(static_cast<double>(a) + w_0lt1 * v * v);
        } else if (r1 < -too_big) {
          const double v = -r1 - too_big;
          a = static_cast<float>(static_cast<double>(a) + w_0lt1 * v * v);
        }
      } else {
        if (r1 < too_small) {
          const double v = too_small - r1;
          a = static_cast<float>(static_cast<double>(a) + w_0lt1 * v * v);
        } else if (r1 > too_big) {
          const double v = r1 - too_big;
          a = static_cast<float>(static_cast<double>(a) + w_0lt1 * v * v);
        }
      }
    }
    acc[o] = a;
  }
};

// ---------------------------------------------------------------------------
// Mask (b/butteraugli.cc:753-782, 1699-1817).
// The planes MaskPsychoImage hands to Mask (:768-781): m_c = a*uhf_c + b*hf_c in
// double, stored as float, c in {X,Y}.  a = 0 for X is multiplied as written.
struct MaskPsychoMix {
  const float* ps;  // PsychoImage group
  float* out;       // [2] X, Y
  Geom g;
  GB_HD static float mix(const float* ps, int c, size_t o, size_t plane) {
    // muls (:762-767): X: (0, 1.64178305129), Y: (0.831081703362, 3.23680933546)
    const double a = c == 0 ? 0.0 : 0.831081703362;
    const double b = c == 0 ? 1.64178305129 : 3.23680933546;
    const float uhf = ps[(kUhfX + c) * plane + o];
    const float hf = ps[(kHfX + c) * plane + o];
    return static_cast<float>(a * uhf + b * hf);
  }
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    out[o] = mix(ps, 0, o, g.plane);
    out[g.plane + o] = mix(ps, 1, o, g.plane);
  }
};

// DiffPrecompute of the combined planes m_c (MaskPsychoMix) for both images;
// neighbours mirror at the last column/row.
struct MaskDiffPre {
  const float* ps0;  // PsychoImage group of the original
  const float* ps1;  // candidate
  float* out;        // [2] X, Y
  Geom g;
  GB_HD float combo(const float* ps, int c, size_t o) const { return MaskPsychoMix::mix(ps, c, o, g.plane); }
  GB_HD void operator()(int x, int y) const {
    const int x2 = (x + 1 < g.w) ? x + 1 : (x > 0 ? x - 1 : x);
    const int y2 = (y + 1 < g.h) ? y + 1 : (y > 0 ? y - 1 : y);
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    const size_t ox = static_cast<size_t>(y) * g.pitch + x2;
    const size_t oy = static_cast<size_t>(y2) * g.pitch + x;
    for (int c = 0; c < 2; ++c) {
      const float a0 = combo(ps0, c, o), a0x = combo(ps0, c, ox), a0y = combo(ps0, c, oy);
      const float a1 = combo(ps1, c, o), a1x = combo(ps1, c, ox), a1y = combo(ps1, c, oy);
      const double sup0 = hd_fabsf(a0 - a0x) + hd_fabsf(a0 - a0y);
      const double sup1 = hd_fabsf(a1 - a1x) + hd_fabsf(a1 - a1y);
      const double mul0 = 0.918416534734;
      const double cutoff = 55.0184555849;
      float v = static_cast<float>(mul0 * hd_min(sup0, sup1));
      if (v >= cutoff) v = static_cast<float>(cutoff);
      out[c * g.plane + o] = v;
    }
  }
};

// Same as MaskDiffPre but on raw planes with xyb0 == xyb1 (StartBlockComparisons,
// g/butteraugli_comparator.cc:415: Mask(xyb0, xyb0)).
struct MaskDiffPreSelf {
  const float* xyb;  // [3]; X and Y used
  float* out;        // [2]
  Geom g;
  GB_HD void operator()(int x, int y) const {
    const int x2 = (x + 1 < g.w) ? x + 1 : (x > 0 ? x - 1 : x);
    const int y2 = (y + 1 < g.h) ? y + 1 : (y > 0 ? y - 1 : y);
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    const size_t ox = static_cast<size_t>(y) * g.pitch + x2;
    const size_t oy = static_cast<size_t>(y2) * g.pitch + x;
    for (int c = 0; c < 2; ++c) {
      const float* p = xyb + c * g.plane;
      const double sup0 = hd_fabsf(p[o] - p[ox]) + hd_fabsf(p[o] - p[oy]);
      const double mul0 = 0.918416534734;
      const double cutoff = 55.0184555849;
      float v = static_cast<float>(mul0 * hd_min(sup0, sup0));
      if (v >= cutoff) v = static_cast<float>(cutoff);
      out[c * g.plane + o] = v;
    }
  }
};

// Blurred activity of the Y channel (:1776-1785): normalizer*(m0*b1 + m1*b2).
GB_HD float mask_y_activity(float b1, float b2) {
  const double m0 = 0.207017089891, m1 = 0.267138152891;
  const double normalizer = 1.0 / (m0 + m1);
  return static_cast<float>(normalizer * (m0 * b1 + m1 * b2));
}

// Mask planes only at block corners (what CompareBlock reads,
// g/butteraugli_comparator.cc:485): out[b][3].
struct BlockCornerMask {
  const float* sx;   // blurred X activity
  const float* sy1;  // Y blurred with r0
  const float* sy2;  // Y blurred with r1
  float* out;        // [nblocks][3]
  Geom g;
  const double* luts;
  GB_HD void operator()(int b) const {
    const int bx = b % g.bw, by = b / g.bw;
    const size_t o = static_cast<size_t>(8 * by) * g.pitch + 8 * bx;
    float m[3], mdc[3];
    mask_from_activity(luts, sx[o], mask_y_activity(sy1[o], sy2[o]), m, mdc);
    out[3 * b + 0] = m[0];
    out[3 * b + 1] = m[1];
    out[3 * b + 2] = m[2];
  }
};

// The same at every pixel: the mask and mask_dc planes Mask returns (:1802-1815).
struct MaskPlanes {
  const float* sx;
  const float* sy1;
  const float* sy2;
  float* mask;     // [3]
  float* mask_dc;  // [3]
  Geom g;
  const double* luts;
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    float m[3], mdc[3];
    mask_from_activity(luts, sx[o], mask_y_activity(sy1[o], sy2[o]), m, mdc);
    for (int c = 0; c < 3; ++c) {
      mask[c * g.plane + o] = m[c];
      mask_dc[c * g.plane + o] = mdc[c];
    }
  }
};

// L2Diff of lf (:654, weights :873-883 -> dc[X] 1.01370836411, dc[B] 1.74566011615),
// the masks, CombineChannels (:1597) and the first half of CalculateDiffmap (:718-735).
struct CombineAndSqrt {
  const float* ps0;
  const float* ps1;
  const float* ac;   // [2] block_diff_ac X, Y (B is identically zero)
  const float* sx;
  const float* sy1;
  const float* sy2;
  float* out;
  Geom g;
  const double* luts;
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    pixel(x, y, sx[o], sy1[o], sy2[o]);
  }
  // the same with the three blurred activities of the pixel given by value (the fused
  // y pass of the mask blurs hands them over in registers)
  GB_HD void pixel(int x, int y, float s_x, float s_y1, float s_y2) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    pixel_with(x, y, s_x, s_y1, s_y2, ps0[kLfX * g.plane + o], ps0[kLfB * g.plane + o], ps1[kLfX * g.plane + o],
               ps1[kLfB * g.plane + o], ac[o], ac[g.plane + o]);
  }
  // ... and with the six plane samples of the pixel already loaded
  GB_HD void pixel_with(int x, int y, float s_x, float s_y1, float s_y2, float lf0x, float lf0b, float lf1x, float lf1b,
                        float ac_x, float ac_y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    float mask[3], dc_mask[3];
    mask_from_activity(luts, s_x, mask_y_activity(s_y1, s_y2), mask, dc_mask);
    float diff_dc[3], diff_ac[3];
    {
      const double d = lf0x - lf1x;
      diff_dc[0] = static_cast<float>(0.0 + 1.01370836411 * d * d);
      diff_dc[1] = 0.0f;
      const double e = lf0b - lf1b;
      diff_dc[2] = static_cast<float>(0.0 + 1.74566011615 * e * e);
    }
    diff_ac[0] = ac_x;
    diff_ac[1] = ac_y;
    diff_ac[2] = 0.0f;
    const float dot_dc = diff_dc[0] * dc_mask[0] + diff_dc[1] * dc_mask[1] + diff_dc[2] * dc_mask[2];
    const float dot_ac = diff_ac[0] * mask[0] + diff_ac[1] * mask[1] + diff_ac[2] * mask[2];
    const float v = dot_dc + dot_ac;
    const float kInitialSlope = 100.0f;
    out[o] = (v < (1.0f / (kInitialSlope * kInitialSlope))) ? kInitialSlope * v : sqrtf(v);
  }
};

// Second half of CalculateDiffmap (:737-749).
struct DiffmapMix {
  const float* blurred;
  float* diffmap;  // in/out
  Geom g;
  GB_HD void operator()(int x, int y) const {
    const size_t o = static_cast<size_t>(y) * g.pitch + x;
    const double mul1 = 0.458794906198;
    const float scale = static_cast<float>(1.0f / (1.0f + mul1));
    float v = static_cast<float>(static_cast<double>(diffmap[o]) + mul1 * blurred[o]);
    v *= scale;
    diffmap[o] = v;
  }
};

// ---------------------------------------------------------------------------
// a15 first half: per-block maximum of the distmap (g/butteraugli_comparator.cc:507-520).
struct BlockMax {
  const float* diffmap;
  float* block_max;
  Geom g;
  GB_HD void operator()(int b) const {
    const int bx = b % g.bw, by = b / g.bw;
    const int x1 = hd_min(g.w, 8 * (bx + 1)), y1 = hd_min(g.h, 8 * (by + 1));
    float m = 0.0f;
    for (int y = 8 * by; y < y1; ++y)
      for (int x = 8 * bx; x < x1; ++x) m = hd_max(m, diffmap[static_cast<size_t>(y) * g.pitch + x]);
    block_max[b] = m;
  }
};

// Partial maxima for the global score (b/butteraugli.cc:1623): lane i reduces
// elements i, i+lanes, ...
struct PartialMax {
  const float* in;
  float* out;
  int n, lanes;
  GB_HD void operator()(int i) const {
    float m = 0.0f;
    for (int j = i; j < n; j += lanes) m = hd_max(m, in[j]);
    out[i] = m;
  }
};

// a15 second half in gather form (g/butteraugli_comparator.cc:521-557).
// direction>0: weight 1 where own max <= target and neighbourhood max <= 1.1 target.
// direction<0: every block b' above its local threshold spreads 1/(d+1) to its
// (2r+1)^2 neighbourhood; weight[b] = max over such b'.
struct BlockWeights {
  const float* block_max;
  float* weight;
  Geom g;
  int direction, radius;
  double target_distance;
  GB_HD float local_max(int bx, int by) const {
    float m = static_cast<float>(target_distance);
    const int x0 = hd_max(0, bx - radius), y0 = hd_max(0, by - radius);
    const int x1 = hd_min(g.bw, bx + 1 + radius), y1 = hd_min(g.bh, by + 1 + radius);
    for (int y = y0; y < y1; ++y)
      for (int x = x0; x < x1; ++x) m = hd_max(m, block_max[y * g.bw + x]);
    return m;
  }
  GB_HD void operator()(int b) const {
    const int bx = b % g.bw, by = b / g.bw;
    if (direction > 0) {
      const float lm = local_max(bx, by);
      weight[b] = (block_max[b] <= target_distance && lm <= 1.1 * target_distance) ? 1.0f : 0.0f;
      return;
    }
    const double kLocalMaxWeight = 0.5;
    float wgt = 0.0f;
    const int x0 = hd_max(0, bx - radius), y0 = hd_max(0, by - radius);
    const int x1 = hd_min(g.bw, bx + 1 + radius), y1 = hd_min(g.bh, by + 1 + radius);
    for (int y = y0; y < y1; ++y) {
      for (int x = x0; x < x1; ++x) {
        const float lm = local_max(x, y);
        if (block_max[y * g.bw + x] <= (1 - kLocalMaxWeight) * target_distance + kLocalMaxWeight * lm)
          continue;
        const int dy = y > by ? y - by : by - y, dx = x > bx ? x - bx : bx - x;
        const int d = hd_max(dy, dx);
        wgt = hd_max(wgt, 1.0f / (d + 1.0f));
      }
    }
    weight[b] = wgt;
  }
};

// ---------------------------------------------------------------------------
// a16 ordering: keys of the selection walk, g/processor.cc:636-663.  Entry
// (block b, candidate slot i) has key (err_i - max_err_b)/w_b ("up", slots
// >= last_index) or (max_err_b - err_i)/w_b ("down", slots < last_index).
// Launched over the compact list of all candidates (entry -> block, slot).
// Pass 1 histograms the upper bits of the order-preserving integer image of the
// key; pass 2 compacts every entry whose bin is <= the threshold bin.
struct OrderKeyCommon {
  const float* err;        // [nblocks][192]
  const int* entry_block;  // [entries]
  const uint8_t* entry_slot;  // [entries]
  const int* last_index;   // [nblocks]
  const float* max_err;    // [nblocks]
  const float* weight;     // [nblocks]
  int direction;
  GB_HD bool key(int entry, int* block, float* val) const {
    const int b = entry_block[entry];
    const float w = weight[b];
    if (w == 0) return false;
    const int slot = entry_slot[entry];
    const int li = last_index[b];
    if (direction > 0 ? slot < li : slot >= li) return false;
    const float e = err[static_cast<size_t>(b) * 192 + slot];
    *val = direction > 0 ? (e - max_err[b]) / w : (max_err[b] - e) / w;
    *block = b;
    return true;
  }
};

// Device-resident state of the key selection: a two-level radix select on the
// order-preserving 32-bit image of the keys.  Level 0 bins bits 31..21 (sign,
// exponent, 2 mantissa bits), level 1 bins bits 20..10 of the keys that fell into the
// level-0 bin of the wanted rank; every entry with image <= threshold (22 significant
// bits) is kept -- a superset of the `want` smallest keys that is a prefix of the
// sorted order (equal keys are never separated).
static const int kOrderBins = 2048;

struct OrderSelectState {
  unsigned int want;       // rank wanted (number of smallest keys)
  unsigned int bin0;       // level-0 bin of that rank
  unsigned int below0;     // entries in level-0 bins < bin0
  unsigned int threshold;  // entries with sortable key <= threshold are kept
  unsigned int kept;       // number of such entries
  unsigned int total;      // all entries
  unsigned int counter;    // compaction cursor
};

GB_HD bool order_bin(const OrderSelectState* st, int level, unsigned int u, unsigned int* bin) {
  if (level == 0) {
    *bin = u >> 21;
    return true;
  }
  if ((u >> 21) != st->bin0) return false;
  *bin = (u >> 10) & 0x7ffu;
  return true;
}

struct OrderKeyHist {  // generic form (CPU port); the CUDA build uses k_order_hist
  OrderKeyCommon c;
  unsigned int* hist;  // [kOrderBins]
  const OrderSelectState* st;
  int level;
  GB_HD void operator()(int entry) const {
    float v;
    int b;
    if (!c.key(entry, &b, &v)) return;
    unsigned int bin;
    if (order_bin(st, level, hd_float_sortable(v), &bin)) hd_atomic_add(&hist[bin], 1u);
  }
};

// One invocation: scans the 2048-bin histogram for the bin where the cumulative
// count reaches the wanted rank (level 0), resp. the residual rank (level 1).
struct OrderSelectBin {
  const unsigned int* hist;
  OrderSelectState* st;
  int level;
  GB_HD void operator()(int) const {
    const unsigned int want = level == 0 ? st->want : (st->want > st->below0 ? st->want - st->below0 : 0u);
    unsigned int cum = 0, bin = kOrderBins - 1, at = 0;
    bool found = false;
    for (int i = 0; i < kOrderBins; ++i) {
      if (!found && cum + hist[i] >= want) {
        bin = static_cast<unsigned int>(i);
        at = cum;
        found = true;
      }
      cum += hist[i];
    }
    if (!found) at = cum - hist[kOrderBins - 1];
    if (level == 0) {
      st->bin0 = bin;
      st->below0 = at;
      st->total = cum;
    } else {
      st->threshold = (st->bin0 << 21) | (bin << 10) | 0x3ffu;
      st->kept = st->below0 + at + hist[bin];
      st->counter = 0;
    }
  }
};

struct OrderKeyCompact {
  OrderKeyCommon c;
  OrderSelectState* st;
  float* out_val;
  int* out_block;
  unsigned int cap;
  GB_HD void operator()(int entry) const {
    float v;
    int b;
    if (!c.key(entry, &b, &v)) return;
    if (hd_float_sortable(v) > st->threshold) return;
    const unsigned int at = hd_atomic_add(&st->counter, 1u);
    if (at < cap) {
      out_val[at] = v;
      out_block[at] = b;
    }
  }
};

}  // namespace gb200
