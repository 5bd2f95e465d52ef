// Host construction of the constant tables (see tables.h).
#include "tables.h"

#include <math.h>

#include <algorithm>
#include <cmath>

namespace gb200 {

#include "tables_data.inc"

namespace {

struct ZigzagInit {
  int to_natural[64];
  int to_zigzag[64];
  ZigzagInit() {
    // Standard JPEG zig-zag walk over the anti-diagonals of the 8x8 block.
    int k = 0;
    for (int s = 0; s < 15; ++s) {
      if (s & 1) {
        for (int y = std::max(0, s - 7); y <= std::min(7, s); ++y) to_natural[k++] = 8 * y + (s - y);
      } else {
        for (int x = std::max(0, s - 7); x <= std::min(7, s); ++x) to_natural[k++] = 8 * (s - x) + x;
      }
    }
    for (int i = 0; i < 64; ++i) to_zigzag[to_natural[i]] = i;
  }
};

template <typename T>
const T* upload(const std::vector<T>& v, Stream s, std::vector<void*>* owned) {
  void* d = dev_alloc(v.size() * sizeof(T));
  h2d(d, v.data(), v.size() * sizeof(T), s);
  stream_sync(s);
  owned->push_back(d);
  return static_cast<const T*>(d);
}

// MakeMask (butteraugli.cc:1638): squared, floor-clamped hyperbola sampled at
// 512 points; kGlobalScale = 1/20.35 (butteraugli.cc:139-140).
void make_mask_lut(double extmul, double extoff, double mul, double offset, double scaler,
                   double* lut) {
  const double kInternalGoodQualityThreshold = 20.35;
  const double kGlobalScale = 1.0 / kInternalGoodQualityThreshold;
  for (int i = 0; i < 512; ++i) {
    const double c = mul / ((0.01 * scaler * i) + offset);
    double v = kGlobalScale * (1.0 + extmul * (c + extoff));
    if (v < 1e-5) v = 1e-5;
    lut[i] = v * v;
  }
}

}  // namespace

const int* zigzag_to_natural() {
  static const ZigzagInit zz;
  return zz.to_natural;
}
const int* natural_to_zigzag() {
  static const ZigzagInit zz;
  return zz.to_zigzag;
}

const std::vector<double>& heat_byte_steps() {
  static const std::vector<double> steps = [] {
    const auto byte_of = [](uint64_t bits) {
      double v;
      memcpy(&v, &bits, sizeof(v));
      return static_cast<uint8_t>(255 * pow(v, 0.5) + 0.5);
    };
    // bisection on the bit patterns, which order non-negative doubles as their values: byte_of(lo) < k <= byte_of(hi)
    uint64_t zero = 0, one;
    const double d1 = 1.0;
    memcpy(&one, &d1, sizeof(one));
    std::vector<double> t(256, 0.0);
    for (int k = 1; k <= 255; ++k) {
      uint64_t lo = zero, hi = one;
      while (hi - lo > 1) {
        const uint64_t mid = lo + (hi - lo) / 2;
        (byte_of(mid) >= k ? hi : lo) = mid;
      }
      memcpy(&t[k], &hi, sizeof(double));
    }
    return t;
  }();
  return steps;
}

double distance_for_quality(double quality) {
  // quality.cc:78 -- clamp to [70,110], linear interpolation between integers.
  if (quality < 70) quality = 70;
  if (quality > 110) quality = 110;
  const int index = static_cast<int>(quality);
  const double mix = quality - index;
  return kDistanceForQuality[index - 70] * (1 - mix) + kDistanceForQuality[index - 70 + 1] * mix;
}

void blur_spec(int id, float* sigma, float* border_ratio) {
  // Every call site passes doubles into Blur(const ImageF&, float, float).
  static const double kSpec[kNumBlurs][2] = {
      {1.2, 0.0},
      {7.46953768697, -0.00457628248637},
      {3.734768843485, -0.271277366628},
      {1.8673844217425, 0.147068973249},
      {10.6666499623, 0.0},
      {9.24456601467, -0.0724948220913},
      {2.3770330432, -0.0724948220913},
      {9.04353323561, -0.0724948220913},
      {1.72547472444, 1.0},
  };
  *sigma = static_cast<float>(kSpec[id][0]);
  *border_ratio = static_cast<float>(kSpec[id][1]);
}

std::vector<float> make_blur_taps(float sigma) {
  // ComputeKernel (butteraugli.cc:145): radius max(1, int(2.25f*|sigma|)),
  // weights exp(-i*i/(2 sigma^2)) with the exponent formed in float.
  const float m = 2.25;
  const float scaler = -1.0 / (2 * sigma * sigma);
  const int diff = std::max<int>(1, m * fabs(sigma));
  std::vector<float> kernel(2 * diff + 1);
  for (int i = -diff; i <= diff; ++i) {
    kernel[i + diff] = exp(scaler * i * i);
  }
  return kernel;
}

namespace {

// Border scale of ConvolveBorderColumn (butteraugli.cc:156-170) at position p of
// an axis of length n.
float border_scale(const std::vector<float>& taps, float weight_no_border, float border_ratio,
                   int p, int n) {
  const int r = static_cast<int>(taps.size() / 2);
  const int lo = p < r ? 0 : p - r;
  const int hi = std::min(n - 1, p + r);
  float weight = 0.0f;
  for (int j = lo; j <= hi; ++j) weight += taps[j - p + r];
  weight = (1.0f - border_ratio) * weight + border_ratio * weight_no_border;
  return 1.0f / weight;
}

}  // namespace

std::vector<float> blur_axis_scales(int id, int n) {
  float sigma, br;
  blur_spec(id, &sigma, &br);
  const std::vector<float> taps = make_blur_taps(sigma);
  const int len = static_cast<int>(taps.size()), r = len / 2;
  float weight_no_border = 0.0f;
  for (int j = 0; j < len; ++j) weight_no_border += taps[j];
  std::vector<float> sc(n, 0.0f);
  for (int p = 0; p < n; ++p)
    if (p < r || p + r >= n) sc[p] = border_scale(taps, weight_no_border, br, p, n);
  return sc;
}

const float* upload_srgb_lin(Stream s, std::vector<void*>* owned, HostTables* host) {
  HostTables local;
  HostTables& ht = host ? *host : local;
  // sRGB -> linear, gamma_correct.cc:23-33
  ht.srgb_lin_d.resize(256);
  ht.srgb_lin.resize(256);
  for (int i = 0; i < 256; ++i) {
    double v = i < 11 ? i / 12.92 : 255.0 * std::pow(((i / 255.0) + 0.055) / 1.055, 2.4);
    ht.srgb_lin_d[i] = v;
    ht.srgb_lin[i] = static_cast<float>(v);
  }
  return upload(ht.srgb_lin, s, owned);
}

Tables build_tables(int w, int h, Stream s, std::vector<void*>* owned, HostTables* host) {
  Tables t;
  HostTables local;
  HostTables& ht = host ? *host : local;

  t.srgb_lin = upload_srgb_lin(s, owned, &ht);

  // YCbCr -> RGB, the libjpeg 16.16 fixed-point tables (color_transform.h:22-140)
  ht.cr_r.resize(256); ht.cb_b.resize(256); ht.cr_g.resize(256); ht.cb_g.resize(256);
  const int kHalf = 1 << 15;
  for (int i = 0; i < 256; ++i) {
    const int x = i - 128;
    ht.cr_r[i] = (91881 * x + kHalf) >> 16;    // 1.40200
    ht.cb_b[i] = (116130 * x + kHalf) >> 16;   // 1.77200
    ht.cr_g[i] = -46802 * x;                   // 0.71414
    ht.cb_g[i] = -22554 * x + kHalf;           // 0.34414
  }
  t.cr_r = upload(ht.cr_r, s, owned);
  t.cb_b = upload(ht.cb_b, s, owned);
  t.cr_g = upload(ht.cr_g, s, owned);
  t.cb_g = upload(ht.cb_g, s, owned);

  t.idct = upload(std::vector<int>(kIdctBasis, kIdctBasis + 64), s, owned);
  t.zigzag = upload(std::vector<int>(zigzag_to_natural(), zigzag_to_natural() + 64), s, owned);

  std::vector<float> csf(192), bias(192);
  for (int i = 0; i < 192; ++i) {
    memcpy(&csf[i], &kOrderCsfBits[i], 4);
    memcpy(&bias[i], &kOrderBiasBits[i], 4);
  }
  t.order_csf = upload(csf, s, owned);
  t.order_bias = upload(bias, s, owned);
  t.order_old_csf = upload(std::vector<unsigned char>(kOrderOldCsf, kOrderOldCsf + 64), s, owned);
  t.nat2zz = upload(std::vector<int>(natural_to_zigzag(), natural_to_zigzag() + 64), s, owned);
  t.block_csf = upload(std::vector<double>(kBlockCsf, kBlockCsf + 37), s, owned);

  // MaskX / MaskY / MaskDcX / MaskDcY (butteraugli.cc:1655-1697)
  ht.mask_lut.resize(4 * 512);
  make_mask_lut(2.59885507073, 3.08805636789, 5.62939030582, 0.315424196682, 16.2770141832,
                &ht.mask_lut[0]);
  make_mask_lut(0.9613705131, -0.581933100068, 6.64307621174, 1.00846207765, 2.2342321176,
                &ht.mask_lut[512]);
  make_mask_lut(10.0470705878, 3.18472654033, 0.373092999662, 0.0551512255218, 70.0,
                &ht.mask_lut[1024]);
  make_mask_lut(0.0115640939227, 45.9483175519, 2.52611324247, 0.0142290066313, 5.0,
                &ht.mask_lut[1536]);
  t.mask_lut = upload(ht.mask_lut, s, owned);

  t.malta_lf = upload(std::vector<unsigned char>(&kMaltaLF[0][0], &kMaltaLF[0][0] + 80), s, owned);
  t.malta_hf = upload(std::vector<unsigned char>(&kMaltaHF[0][0], &kMaltaHF[0][0] + 144), s, owned);
  t.malta_hf_len = upload(std::vector<unsigned char>(kMaltaHFLen, kMaltaHFLen + 16), s, owned);

  for (int id = 0; id < kNumBlurs; ++id) {
    float sigma, br;
    blur_spec(id, &sigma, &br);
    std::vector<float> taps = make_blur_taps(sigma);
    ht.blur_taps[id] = taps;
    const int len = static_cast<int>(taps.size());
    const int r = len / 2;
    // Convolution (butteraugli.cc:190-200)
    float weight_no_border = 0.0f;
    for (int j = 0; j < len; ++j) weight_no_border += taps[j];
    const float scale_no_border = 1.0f / weight_no_border;
    std::vector<float> taps_n = taps;
    for (int j = 0; j < len; ++j) taps_n[j] *= scale_no_border;
    ht.blur_taps_n[id] = taps_n;
    const std::vector<float> sx = blur_axis_scales(id, w), sy = blur_axis_scales(id, h);
    t.blur[id].taps = upload(taps, s, owned);
    t.blur[id].taps_n = upload(taps_n, s, owned);
    t.blur[id].scale_x = upload(sx, s, owned);
    t.blur[id].scale_y = upload(sy, s, owned);
    t.blur[id].r = r;
    if (id == kBlurOpsin) {
      std::vector<float> s8(8, 0.0f);
      for (int p = 0; p < 8; ++p)
        if (p < r || p + r >= 8) s8[p] = border_scale(taps, weight_no_border, br, p, 8);
      t.opsin_scale8 = upload(s8, s, owned);
    }
  }
  return t;
}

namespace {
// MaltaDiffMapImpl prologue (butteraugli.cc:1470-1474)
MaltaParams malta_params(double w_0gt1, double w_0lt1, double norm1, double mulli) {
  const double len = 3.75;
  const float kWeight0 = 0.5;
  const float kWeight1 = 0.33;
  const double w_pre0gt1 = mulli * sqrt(kWeight0 * w_0gt1) / (len * 2 + 1);
  const double w_pre0lt1 = mulli * sqrt(kWeight1 * w_0lt1) / (len * 2 + 1);
  MaltaParams mp;
  mp.norm2_0gt1 = w_pre0gt1 * norm1;
  mp.norm2_0lt1 = w_pre0lt1 * norm1;
  mp.norm1 = static_cast<float>(norm1);
  return mp;
}
}  // namespace

void malta_call_params(MaltaParams out[6]) {
  const float hf_asymmetry = 0.8f;
  const double mulli_hf = 0.354191303559;  // MaltaDiffMap (9-tap), butteraugli.cc:1577
  const double mulli_lf = 0.405371989604;  // MaltaDiffMapLF, :1590
  const double wUhfMalta = 5.1409625726, norm1Uhf = 58.5001247061;
  const double wUhfMaltaX = 4.91743441556, norm1UhfX = 687196.39002;
  const double wHfMalta = 153.671655716, norm1Hf = 83150785.9592;
  const double wHfMaltaX = 668.358918152, norm1HfX = 0.882954368025;
  const double wMfMalta = 6841.81248144, norm1Mf = 0.0135134962487;
  const double wMfMaltaX = 813.901703816, norm1MfX = 16792.9322251;
  out[0] = malta_params(wUhfMalta * hf_asymmetry, wUhfMalta / hf_asymmetry, norm1Uhf, mulli_hf);
  out[1] = malta_params(wUhfMaltaX * hf_asymmetry, wUhfMaltaX / hf_asymmetry, norm1UhfX, mulli_hf);
  out[2] = malta_params(wHfMalta * sqrt(hf_asymmetry), wHfMalta / sqrt(hf_asymmetry), norm1Hf, mulli_lf);
  out[3] = malta_params(wHfMaltaX * sqrt(hf_asymmetry), wHfMaltaX / sqrt(hf_asymmetry), norm1HfX, mulli_lf);
  out[4] = malta_params(wMfMalta, wMfMalta, norm1Mf, mulli_lf);
  out[5] = malta_params(wMfMaltaX, wMfMaltaX, norm1MfX, mulli_lf);
}

void l2_asym_weights(double* w_0gt1, double* w_0lt1) {
  const float hf_asymmetry = 0.8f;
  const double wmul1 = 32.4449876135;
  double a = wmul1 * hf_asymmetry;
  double b = wmul1 / hf_asymmetry;
  a *= 0.8;
  b *= 0.8;
  *w_0gt1 = a;
  *w_0lt1 = b;
}

}  // namespace gb200
