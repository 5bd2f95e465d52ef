// Integer JPEG arithmetic of the hot path, single source for device + CPU port.
// All of it is exact integer work: results must equal the reference bit for bit.
#pragma once
#include "hd.h"

namespace gb200 {

// ---------------------------------------------------------------------------
// Quantize (quantize.h:24): nearest multiple of q, C '%' semantics, ties to zero.
GB_HD int quantize_coeff(int raw, int q) {
  const int r = raw % q;
  const int delta = 2 * r > q ? q - r : (-2) * r > q ? -q - r : -r;
  return static_cast<int16_t>(raw + delta);
}

// ---------------------------------------------------------------------------
// 8-point inverse DCT as a dot product with the 13-bit basis (idct.cc:41):
// out[x] = sum_u basis[8x+u] * in[u].  int32 wrap-around like the reference.
GB_HD void idct_1d(const int* basis, const int in[8], int out[8]) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int x = 0; x < 8; ++x) {
    int acc = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int u = 0; u < 8; ++u) acc += basis[8 * x + u] * in[u];
    out[x] = acc;
  }
}

// ComputeBlockIDCT (idct.cc:139): column pass (+2^10 >> 11, stored as int16),
// row pass (+257*2^17 >> 18, includes the +128 level shift), clamp to u8.
GB_HD void idct_8x8(const int* basis, const int16_t* block, uint8_t* out) {
  int16_t col[64];
  for (int x = 0; x < 8; ++x) {
    int in[8], o[8];
    for (int u = 0; u < 8; ++u) in[u] = block[8 * u + x];
    idct_1d(basis, in, o);
    for (int y = 0; y < 8; ++y) col[8 * y + x] = static_cast<int16_t>((o[y] + (1 << 10)) >> 11);
  }
  for (int y = 0; y < 8; ++y) {
    int in[8], o[8];
    for (int u = 0; u < 8; ++u) in[u] = col[8 * y + u];
    idct_1d(basis, in, o);
    for (int x = 0; x < 8; ++x) {
      int v = (o[x] + (257 << 17)) >> 18;
      out[8 * y + x] = static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
  }
}

// ---------------------------------------------------------------------------
// YCbCr -> RGB (color_transform.h:211) with the range-limit table folded into a clamp.
GB_HD int clamp_u8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

GB_HD void ycc_to_rgb(const int* cr_r, const int* cb_b, const int* cr_g, const int* cb_g, int y,
                      int cb, int cr, int* r, int* g, int* b) {
  *r = clamp_u8(y + cr_r[cr]);
  *g = clamp_u8(y + ((cr_g[cr] + cb_g[cb]) >> 16));
  *b = clamp_u8(y + cb_b[cb]);
}

// ---------------------------------------------------------------------------
// RGB -> YCbCr, 16.16 fixed point, output centred on zero (jpeg_data_encoder.cc:40).
GB_HD void rgb_to_ycc16(int r, int g, int b, int16_t* y, int16_t* cb, int16_t* cr) {
  const int kHalf = 1 << 15;
  *y = static_cast<int16_t>((19595 * r + 38469 * g + 7471 * b - (128 << 16) + kHalf) >> 16);
  *cb = static_cast<int16_t>((-11059 * r - 21709 * g + 32768 * b + kHalf - 1) >> 16);
  *cr = static_cast<int16_t>((32768 * r - 27439 * g - 5329 * b + kHalf - 1) >> 16);
}

// Forward DCT (fdct.cc:160-240), output scaled by 16.  The fixed-point data
// flow (which products are truncated by >>16, what is narrowed to int16 between
// the passes) is what makes the result; additions are exact in int32.
GB_HD int mulhi16(int a, int b) { return (a * b) >> 16; }

// Vertical pass over one column (stride 8), in place.
GB_HD void fdct_column(int16_t* v) {
  const int kTan1 = 13036, kTan2 = 27146, kTan3m1 = -21746, k2Sqrt2 = 23170;
  // first butterfly stage: d = differences, s = sums of mirrored rows
  int d07 = v[0 * 8] - v[7 * 8], s07 = v[0 * 8] + v[7 * 8];
  int d25 = v[2 * 8] - v[5 * 8], s25 = v[2 * 8] + v[5 * 8];
  int d34 = v[3 * 8] - v[4 * 8], s34 = v[3 * 8] + v[4 * 8];
  int d16 = v[1 * 8] - v[6 * 8], s16 = v[1 * 8] + v[6 * 8];
  // even part
  int e_d = s07 - s34, e_s = s07 + s34;   // (m7, m4) after BUTTERFLY(m7, m4)
  int f_d = s16 - s25, f_s = s16 + s25;   // (m6, m5) after BUTTERFLY(m6, m5)
  int es = e_s << 3, fs = f_s << 3;
  v[0 * 8] = static_cast<int16_t>(es + fs);
  v[4 * 8] = static_cast<int16_t>(es - fs);
  int ed = e_d << 3, fd = f_d << 3;
  v[2 * 8] = static_cast<int16_t>(mulhi16(kTan2, fd) + ed);
  v[6 * 8] = static_cast<int16_t>(mulhi16(kTan2, ed) - fd);
  // odd part
  int a3 = d34 << 3, a0 = d07 << 3;
  int b2 = d25 << 4, b1 = d16 << 4;
  int p = mulhi16(b1 + b2, k2Sqrt2);   // m2 after BUTTERFLY(m1,m2); MULT
  int q = mulhi16(b1 - b2, k2Sqrt2);   // m1
  int t3 = a3 - q, t1 = a3 + q;        // BUTTERFLY(m3, m1): m3 = a3 - q, m1 = a3 + q
  int t0 = a0 - p, t2 = a0 + p;        // BUTTERFLY(m0, m2)
  int m3 = mulhi16(t3, kTan3m1) + t3;  // t3 * tan3
  int m1 = mulhi16(t1, kTan1) + t2;
  m1 += 1;                             // CORRECT_LSB
  m3 += 1;
  int m4 = mulhi16(kTan3m1, t0) + t0;  // t0 * tan3
  int m5 = mulhi16(kTan1, t2);
  v[1 * 8] = static_cast<int16_t>(m1);
  v[3 * 8] = static_cast<int16_t>(t0 - m3);
  v[5 * 8] = static_cast<int16_t>(t3 + m4);
  v[7 * 8] = static_cast<int16_t>(m5 - t1);
}

// Horizontal pass over one row with its 7-entry cosine table (fdct.cc:173).
GB_HD void fdct_row(int16_t* in, const int16_t* table) {
  const int a0 = in[0] + in[7], b0 = in[0] - in[7];
  const int a1 = in[1] + in[6], b1 = in[1] - in[6];
  const int a2 = in[2] + in[5], b2 = in[2] - in[5];
  const int a3 = in[3] + in[4], b3 = in[3] - in[4];
  const int C1 = table[0], C2 = table[1], C3 = table[2], C4 = table[3], C5 = table[4],
            C6 = table[5], C7 = table[6];
  const int c0 = a0 + a3, c1 = a0 - a3, c2 = a1 + a2, c3 = a1 - a2;
  in[0] = static_cast<int16_t>((C4 * (c0 + c2)) >> 16);
  in[4] = static_cast<int16_t>((C4 * (c0 - c2)) >> 16);
  in[2] = static_cast<int16_t>((C2 * c1 + C6 * c3) >> 16);
  in[6] = static_cast<int16_t>((C6 * c1 - C2 * c3) >> 16);
  in[1] = static_cast<int16_t>((C1 * b0 + C3 * b1 + C5 * b2 + C7 * b3) >> 16);
  in[3] = static_cast<int16_t>((C3 * b0 - C7 * b1 - C1 * b2 - C5 * b3) >> 16);
  in[5] = static_cast<int16_t>((C5 * b0 - C1 * b1 + C7 * b2 + C3 * b3) >> 16);
  in[7] = static_cast<int16_t>((C7 * b0 - C5 * b1 + C3 * b2 - C1 * b3) >> 16);
}

GB_HD void fdct_8x8(int16_t* c) {
  // cos(k*pi/16)/sqrt(2) in 15 bits; rows 1/7, 2/6, 3/5 pre-multiplied by
  // 2cos(pi/16), 2cos(2pi/16), 2cos(3pi/16) (fdct.cc:29-36)
  const int16_t t04[7] = {22725, 21407, 19266, 16384, 12873, 8867, 4520};
  const int16_t t17[7] = {31521, 29692, 26722, 22725, 17855, 12299, 6270};
  const int16_t t26[7] = {29692, 27969, 25172, 21407, 16819, 11585, 5906};
  const int16_t t35[7] = {26722, 25172, 22654, 19266, 15137, 10426, 5315};
  for (int x = 0; x < 8; ++x) fdct_column(c + x);
  fdct_row(c + 0 * 8, t04);
  fdct_row(c + 1 * 8, t17);
  fdct_row(c + 2 * 8, t26);
  fdct_row(c + 3 * 8, t35);
  fdct_row(c + 4 * 8, t04);
  fdct_row(c + 5 * 8, t35);
  fdct_row(c + 6 * 8, t26);
  fdct_row(c + 7 * 8, t17);
}

// Quantize by 1 after the x16 DCT scale (jpeg_data_encoder.cc:33 with iquant=65537).
GB_HD int16_t fdct_descale(int16_t v) {
  return static_cast<int16_t>((v * 65537 + (0x80 << 12)) >> 20);
}

// ---------------------------------------------------------------------------
// libjpeg's post-IDCT range limit: range_limit[x & RANGE_MASK] of the table of prepare_range_limit_table
// (jdmaster.c), x the descaled output without its +128 centring.  The mask keeps 10 bits, so sums out of
// [-512, 511] wrap before the clamp, as in libjpeg.
GB_HD int jpeg_idct_limit(long long x) {
  int v = static_cast<int>(x) & 1023;
  if (v >= 512) v -= 1024;
  v += 128;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

GB_HD bool jpeg_fits16(long long v) { return v >= -32768 && v <= 32767; }
GB_HD bool jpeg_fits32(long long v) { return v >= -2147483647LL - 1 && v <= 2147483647LL; }

// One 8-point pass of jpeg_islow: inputs in[0], in[s], .. in[7 s] (already dequantised), outputs
// DESCALE(., sh) into out[0], out[s], ..; CHECK: *ok is cleared where a quantity leaves the range of
// libjpeg-turbo's SIMD version (sums of inputs to 16 bits, products and sums to 32 bits).
template <bool CHECK>
GB_HD void jpeg_islow_pass(const long long* in, int s, int sh, long long* out, bool* ok) {
  const long long F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633,
                  F1501 = 12299, F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
  // even part
  long long z2 = in[2 * s], z3 = in[6 * s];
  long long z1 = (z2 + z3) * F0541;
  long long tmp2 = z1 + z3 * -F1847, tmp3 = z1 + z2 * F0765;
  const long long e0 = in[0] + in[4 * s], e1 = in[0] - in[4 * s];
  long long tmp0 = static_cast<long long>(static_cast<unsigned long long>(e0) << 13);
  long long tmp1 = static_cast<long long>(static_cast<unsigned long long>(e1) << 13);
  const long long t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  if (CHECK)
    *ok = *ok && jpeg_fits16(z2 + z3) && jpeg_fits16(e0) && jpeg_fits16(e1) && jpeg_fits32(t10) &&
          jpeg_fits32(t11) && jpeg_fits32(t12) && jpeg_fits32(t13) && jpeg_fits32(z1);
  // odd part: y7, y5, y3, y1
  tmp0 = in[7 * s];
  tmp1 = in[5 * s];
  tmp2 = in[3 * s];
  tmp3 = in[s];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * F1175;
  if (CHECK)
    *ok = *ok && jpeg_fits16(z1) && jpeg_fits16(z2) && jpeg_fits16(z3) && jpeg_fits16(z4) && jpeg_fits16(z3 + z4);
  tmp0 *= F0298;
  tmp1 *= F2053;
  tmp2 *= F3072;
  tmp3 *= F1501;
  z1 *= -F0899;
  z2 *= -F2562;
  z3 *= -F1961;
  z4 *= -F0390;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  const long long r = 1LL << (sh - 1);
  out[0] = (t10 + tmp3 + r) >> sh;
  out[7 * s] = (t10 - tmp3 + r) >> sh;
  out[s] = (t11 + tmp2 + r) >> sh;
  out[6 * s] = (t11 - tmp2 + r) >> sh;
  out[2 * s] = (t12 + tmp1 + r) >> sh;
  out[5 * s] = (t12 - tmp1 + r) >> sh;
  out[3 * s] = (t13 + tmp0 + r) >> sh;
  out[4 * s] = (t13 - tmp0 + r) >> sh;
  if (CHECK)
    *ok = *ok && jpeg_fits32(t10 + tmp3 + r) && jpeg_fits32(t10 - tmp3 + r) && jpeg_fits32(t11 + tmp2 + r) &&
          jpeg_fits32(t11 - tmp2 + r) && jpeg_fits32(t12 + tmp1 + r) && jpeg_fits32(t12 - tmp1 + r) &&
          jpeg_fits32(t13 + tmp0 + r) && jpeg_fits32(t13 - tmp0 + r);
}

// libjpeg's jpeg_idct_islow (jidctint.c) of one block: coefficients in natural order dequantised by q
// (the product an int), the two-pass LL&M with its constants, PASS1_BITS = 2, DESCALE rounding, an int
// workspace and 64-bit JLONG, its shortcuts for columns and rows whose AC terms are all zero, and
// jpeg_idct_limit; 8 rows of 8 samples at out, pitch bytes apart.
//
// libjpeg-turbo's SIMD IDCTs compute the same integers as long as its 16-bit lanes hold every
// dequantised value, pass-1 output and sum of them, and the output stays in [-512, 511] before the
// range limit; past that they saturate or wrap differently.  CHECK: nothing is written, and the result
// tells whether the block stays inside those ranges (on every quantity that could be 16 bits there).
template <bool CHECK>
GB_HD bool jpeg_islow(const int16_t* in, const int* q, uint8_t* out, int pitch) {
  bool ok = true;
  if (CHECK) {
    // a DC-only block takes both shortcuts here and the 16-bit DC shortcut there, which wraps 4 x DC to
    // 16 bits: the same output modulo 1024, so the same sample where that 16-bit output is in range
    bool ac = false;
    for (int k = 1; k < 64; ++k) ac = ac || in[k] != 0;
    if (!ac) {
      const long long dq = in[0] * q[0];
      const long long x = (static_cast<long long>(static_cast<int16_t>(static_cast<uint16_t>(4 * dq))) + 16) >> 5;
      return jpeg_fits16(dq) && x >= -512 && x <= 511;
    }
  }
  long long col[64], ws[64];
  int wsi[64];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int x = 0; x < 8; ++x) {
    for (int y = 0; y < 8; ++y) {
      col[8 * y + x] = in[8 * y + x] * q[8 * y + x];
      if (CHECK) ok = ok && jpeg_fits16(col[8 * y + x]);
    }
    if (in[8 + x] == 0 && in[16 + x] == 0 && in[24 + x] == 0 && in[32 + x] == 0 && in[40 + x] == 0 &&
        in[48 + x] == 0 && in[56 + x] == 0) {
      const int dc = static_cast<int>(static_cast<unsigned int>(in[x] * q[x]) << 2);
      if (CHECK) ok = ok && jpeg_fits16(4LL * col[x]);
      for (int y = 0; y < 8; ++y) wsi[8 * y + x] = dc;
      continue;
    }
    jpeg_islow_pass<CHECK>(col + x, 8, 11, ws + x, &ok);  // CONST_BITS - PASS1_BITS
    for (int y = 0; y < 8; ++y) {
      wsi[8 * y + x] = static_cast<int>(ws[8 * y + x]);
      if (CHECK) ok = ok && jpeg_fits16(ws[8 * y + x]);
    }
  }
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int y = 0; y < 8; ++y) {
    const int* w = wsi + 8 * y;
    long long row[8], o[8];
    if (w[1] == 0 && w[2] == 0 && w[3] == 0 && w[4] == 0 && w[5] == 0 && w[6] == 0 && w[7] == 0) {
      const long long v = (static_cast<long long>(w[0]) + 16) >> 5;  // PASS1_BITS + 3
      for (int x = 0; x < 8; ++x) o[x] = v;
    } else {
      for (int x = 0; x < 8; ++x) row[x] = w[x];
      jpeg_islow_pass<CHECK>(row, 1, 18, o, &ok);  // CONST_BITS + PASS1_BITS + 3
    }
    for (int x = 0; x < 8; ++x) {
      if (CHECK) {
        ok = ok && o[x] >= -512 && o[x] <= 511;
      } else {
        out[static_cast<size_t>(y) * pitch + x] = static_cast<uint8_t>(jpeg_idct_limit(o[x]));
      }
    }
  }
  return ok;
}

}  // namespace gb200
