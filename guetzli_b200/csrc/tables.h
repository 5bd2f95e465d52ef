// Constant tables of the hot path, built once on the host (with the host libm,
// exactly like the reference builds them) and kept resident in device memory.
#pragma once
#include <vector>

#include "backend.h"

namespace gb200 {

// One separable blur (butteraugli.cc:145-233): raw taps, taps pre-multiplied by
// 1/sum (interior path), and the per-position border scales of ConvolveBorderColumn
// for an axis of length w (x pass) and h (y pass).
struct BlurTab {
  const float* taps;     // 2r+1 raw weights exp(-i^2/(2 sigma^2)) (float)
  const float* taps_n;   // taps * (1/sum), the interior kernel
  const float* scale_x;  // [w] 1/weight for border columns (undefined elsewhere)
  const float* scale_y;  // [h]
  int r;
};

enum BlurId {
  kBlurOpsin = 0,   // sigma 1.2           br 0              butteraugli.cc:328
  kBlurLf,          // 7.46953768697       -0.00457628248637 :497,504
  kBlurMf,          // 3.734768843485      -0.271277366628   :498,505
  kBlurHf,          // 1.8673844217425     0.147068973249    :499,506
  kBlurNoise,       // 10.6666499623       0                 :881,645
  kBlurMaskX,       // 9.24456601467       -0.0724948220913  :1761,1762
  kBlurMaskY0,      // 2.3770330432        -0.0724948220913  :1759
  kBlurMaskY1,      // 9.04353323561       -0.0724948220913  :1760
  kBlurFinal,       // 1.72547472444       1.0               :738,741
  kNumBlurs
};

struct Tables {
  const float* srgb_lin;     // [256] float(Srgb8ToLinearTable()[v])  gamma_correct.cc:23
  const int* cr_r;           // [256] color_transform.h:22
  const int* cb_b;           // [256] :47
  const int* cr_g;           // [256] :72
  const int* cb_g;           // [256] :107
  const int* idct;           // [64]  idct.cc:29
  const int* zigzag;         // [64]  zig-zag scan position -> natural index
  const float* order_csf;    // [192] order.inc
  const float* order_bias;   // [192]
  const unsigned char* order_old_csf;  // [64] legacy zeroing model, processor.cc:369
  const int* nat2zz;         // [64] natural index -> zig-zag position
  const double* block_csf;   // [37]  butteraugli_comparator.cc:94
  const double* mask_lut;    // [4][512] MaskX, MaskY, MaskDcX, MaskDcY  butteraugli.cc:1655-1697
  const unsigned char* malta_lf;      // [16][5]
  const unsigned char* malta_hf;      // [16][9]
  const unsigned char* malta_hf_len;  // [16]
  BlurTab blur[kNumBlurs];
  const float* opsin_scale8;  // [8] border scales of the sigma-1.2 blur on an 8-long axis
};

// Malta pre-pass constants of one MaltaDiffMap call (butteraugli.cc:1470-1474).
struct MaltaParams {
  float norm2_0gt1;
  float norm2_0lt1;
  float norm1;  // static_cast<float>(norm1)
};
// The six calls of DiffmapPsychoImage (butteraugli.cc:829-871), in call order:
// uhf[Y], uhf[X] (9-tap lines), hf[Y], hf[X], mf[Y], mf[X] (5-tap lines).
void malta_call_params(MaltaParams out[6]);
// L2DiffAsymmetric weights for hf[Y] (butteraugli.cc:866,893,679-680).
void l2_asym_weights(double* w_0gt1, double* w_0lt1);

// Host-side copies (used by the host search driver and by tests).
struct HostTables {
  std::vector<double> srgb_lin_d;  // 256 doubles
  std::vector<float> srgb_lin;
  std::vector<int> cr_r, cb_b, cr_g, cb_g;
  std::vector<double> mask_lut;  // 4*512
  std::vector<float> blur_taps[kNumBlurs];
  std::vector<float> blur_taps_n[kNumBlurs];  // interior kernel: taps * (1/sum)
};

void blur_spec(int id, float* sigma, float* border_ratio);
std::vector<float> make_blur_taps(float sigma);
// BlurTab::scale_x / scale_y of blur `id` for an axis of length n (zero where the interior kernel applies)
std::vector<float> blur_axis_scales(int id, int n);

// Builds all tables for a w x h image and uploads them. Returns the device
// allocations in *owned so the caller can free them.
Tables build_tables(int w, int h, Stream s, std::vector<void*>* owned, HostTables* host);
// The sRGB table alone (Tables::srgb_lin), uploaded the same way.
const float* upload_srgb_lin(Stream s, std::vector<void*>* owned, HostTables* host);

const int* zigzag_to_natural();  // [64] JPEG zig-zag scan position -> natural index
const int* natural_to_zigzag();  // [64] inverse
double distance_for_quality(double quality);  // quality.cc:78

}  // namespace gb200
