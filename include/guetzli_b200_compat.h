// Source-level drop-in for the reference's public C++ API of the hot path
// (guetzli/processor.h:29-56, guetzli/stats.h:29-40, guetzli/quality.h:23):
// same namespace, names, argument meaning and error behaviour, implemented on
// top of the C ABI in guetzli_b200.h.  A caller of guetzli::Process(RGB) -- the
// CLI's PNG branch (guetzli/guetzli.cc:301) -- recompiles against this header
// and links libguetzli_b200.so instead of the reference's processor.o & co.
#ifndef GUETZLI_B200_COMPAT_H_
#define GUETZLI_B200_COMPAT_H_

#include <cstdio>
#include <cstdlib>
#include <map>
#include <string>
#include <vector>

#include "guetzli_b200.h"

namespace guetzli {

static const char* const kNumItersCnt = "number of iterations";
static const char* const kNumItersUpCnt = "number of iterations up";
static const char* const kNumItersDownCnt = "number of iterations down";

struct ProcessStats {
  ProcessStats() {}
  std::map<std::string, int> counters;
  std::string* debug_output = nullptr;
  FILE* debug_output_file = nullptr;
  std::string filename;
};

struct Params {
  float butteraugli_target = 1.0;
  bool clear_metadata = true;
  bool try_420 = false;
  bool force_420 = false;
  bool use_silver_screen = false;
  int zeroing_greedy_lookahead = 3;
  bool new_zeroing_model = true;
};

inline double ButteraugliScoreForQuality(double quality) {
  return gb200_butteraugli_score_for_quality(quality);
}

namespace b200_detail {
inline void LogSink(void* user, const char* text) {
  ProcessStats* stats = static_cast<ProcessStats*>(user);
  if (stats->debug_output) stats->debug_output->append(text);
  if (stats->debug_output_file) fprintf(stats->debug_output_file, "%s", text);
}
}  // namespace b200_detail

// Sets *out to a jpeg encoded string that will decode to an image that is
// visually indistinguishable from the input rgb image (processor.h:52-56).
// GUETZLI_B200_DEVICE (environment) selects the CUDA device, default 0.
inline bool Process(const Params& params, ProcessStats* stats, const std::vector<uint8_t>& rgb, int w,
                    int h, std::string* out) {
  if (w < 0 || h < 0 || rgb.size() != static_cast<size_t>(3) * w * h) {
    fprintf(stderr, "Could not create jpg data from rgb pixels\n");
    return false;
  }
  gb200_params p;
  gb200_params_default(&p);
  p.butteraugli_target = params.butteraugli_target;
  p.clear_metadata = params.clear_metadata;
  p.try_420 = params.try_420;
  p.force_420 = params.force_420;
  p.use_silver_screen = params.use_silver_screen;
  p.zeroing_greedy_lookahead = params.zeroing_greedy_lookahead;
  p.new_zeroing_model = params.new_zeroing_model;
  ProcessStats dummy;
  if (stats == nullptr) stats = &dummy;
  const bool want_log = stats->debug_output || stats->debug_output_file;
  int device = 0;
  if (const char* e = getenv("GUETZLI_B200_DEVICE")) device = atoi(e);
  uint8_t* buf = nullptr;
  size_t len = 0;
  gb200_stats st;
  const int ok = gb200_process_rgb(&p, rgb.data(), w, h, device, want_log ? b200_detail::LogSink : nullptr,
                                   stats, &buf, &len, &st);
  out->assign(reinterpret_cast<const char*>(buf), len);
  gb200_free(buf);
  if (ok) {
    stats->counters[kNumItersCnt] = st.iterations;
    stats->counters[kNumItersUpCnt] = st.iterations_up;
    stats->counters[kNumItersDownCnt] = st.iterations_down;
  } else if (*gb200_last_error() && len == 0) {
    // device-side failures (no GPU, CUDA error) are reported like any other failure
    fprintf(stderr, "%s\n", gb200_last_error());
  }
  return ok != 0;
}

// JPEG input (processor.h:39-41, processor.cc:890): 4:4:4 YCbCr files; the search starts
// from the file's coefficients and quant tables.
inline bool Process(const Params& params, ProcessStats* stats, const std::string& in_data, std::string* out) {
  gb200_params p;
  gb200_params_default(&p);
  p.butteraugli_target = params.butteraugli_target;
  p.clear_metadata = params.clear_metadata;
  p.try_420 = params.try_420;
  p.force_420 = params.force_420;
  p.use_silver_screen = params.use_silver_screen;
  p.zeroing_greedy_lookahead = params.zeroing_greedy_lookahead;
  p.new_zeroing_model = params.new_zeroing_model;
  ProcessStats dummy;
  if (stats == nullptr) stats = &dummy;
  const bool want_log = stats->debug_output || stats->debug_output_file;
  int device = 0;
  if (const char* e = getenv("GUETZLI_B200_DEVICE")) device = atoi(e);
  uint8_t* buf = nullptr;
  size_t len = 0;
  gb200_stats st;
  const int ok = gb200_process_jpeg(&p, reinterpret_cast<const uint8_t*>(in_data.data()), in_data.size(), device,
                                    want_log ? b200_detail::LogSink : nullptr, stats, &buf, &len, &st);
  out->assign(reinterpret_cast<const char*>(buf), len);
  gb200_free(buf);
  if (ok) {
    stats->counters[kNumItersCnt] = st.iterations;
    stats->counters[kNumItersUpCnt] = st.iterations_up;
    stats->counters[kNumItersDownCnt] = st.iterations_down;
  }
  return ok != 0;
}

}  // namespace guetzli

namespace guetzli_b200 {

// butteraugli::ButteraugliComparator (third_party/butteraugli/butteraugli/butteraugli.h:425) with
// the original resident on one GPU.  Images are three planes of linear RGB (nominally 0..255; values
// outside it are scored as the reference scores them, tested from -300 to 4500; no NaN or infinity),
// each w*h floats row by row, as ButteraugliAdaptiveQuantization takes them; outputs are laid out the
// same way.
// The methods return false on failure (gb200_last_error), where the reference's return nothing.
// One comparator is used by one thread at a time.
class ButteraugliComparator {
 public:
  ButteraugliComparator(const std::vector<std::vector<float> >& rgb0, int w, int h, int device = 0)
      : w_(w), h_(h) {
    if (Complete(rgb0)) {
      const std::vector<float> flat = Flat(rgb0);
      c_ = gb200_butteraugli_comparator_create(flat.data(), w, h, device);
    }
  }
  ~ButteraugliComparator() { gb200_butteraugli_comparator_destroy(c_); }
  ButteraugliComparator(const ButteraugliComparator&) = delete;
  ButteraugliComparator& operator=(const ButteraugliComparator&) = delete;

  // false when the original was refused (smaller than 8x8, no device, ...)
  bool ok() const { return c_ != nullptr; }

  // ButteraugliComparator::Diffmap (butteraugli.cc:799): result receives w*h floats.
  bool Diffmap(const std::vector<std::vector<float> >& rgb1, std::vector<float>& result) {
    if (!c_ || !Complete(rgb1)) return false;
    const std::vector<float> flat = Flat(rgb1);
    result.resize(static_cast<size_t>(w_) * h_);
    return gb200_butteraugli_comparator_diffmap(c_, flat.data(), result.data(), nullptr) != 0;
  }

  // ButteraugliComparator::Mask (butteraugli.cc:793): three planes each.
  bool Mask(std::vector<std::vector<float> >* mask, std::vector<std::vector<float> >* mask_dc) {
    if (!c_) return false;
    const size_t n = static_cast<size_t>(w_) * h_;
    std::vector<float> m(3 * n), mdc(3 * n);
    if (!gb200_butteraugli_comparator_mask(c_, m.data(), mdc.data())) return false;
    mask->assign(3, std::vector<float>());
    mask_dc->assign(3, std::vector<float>());
    for (int c = 0; c < 3; ++c) {
      (*mask)[c].assign(m.begin() + c * n, m.begin() + (c + 1) * n);
      (*mask_dc)[c].assign(mdc.begin() + c * n, mdc.begin() + (c + 1) * n);
    }
    return true;
  }

 private:
  bool Complete(const std::vector<std::vector<float> >& rgb) const {
    if (rgb.size() != 3 || w_ < 1 || h_ < 1) return false;
    for (int c = 0; c < 3; ++c)
      if (rgb[c].size() != static_cast<size_t>(w_) * h_) return false;
    return true;
  }
  static std::vector<float> Flat(const std::vector<std::vector<float> >& rgb) {
    std::vector<float> flat;
    for (int c = 0; c < 3; ++c) flat.insert(flat.end(), rgb[c].begin(), rgb[c].end());
    return flat;
  }
  gb200_butteraugli_comparator* c_ = nullptr;
  int w_, h_;
};

// butteraugli::ButteraugliAdaptiveQuantization (butteraugli.cc:1880), same signature; the device
// is GUETZLI_B200_DEVICE (environment), default 0.  False below 16x16, as the reference.
inline bool ButteraugliAdaptiveQuantization(size_t xsize, size_t ysize, const std::vector<std::vector<float> >& rgb,
                                            std::vector<float>& quant) {
  const size_t n = xsize * ysize;
  if (xsize < 16 || ysize < 16 || rgb.size() != 3 || xsize >= 65536 || ysize >= 65536) return false;
  std::vector<float> flat;
  for (int c = 0; c < 3; ++c) {
    if (rgb[c].size() != n) return false;
    flat.insert(flat.end(), rgb[c].begin(), rgb[c].end());
  }
  int device = 0;
  if (const char* e = getenv("GUETZLI_B200_DEVICE")) device = atoi(e);
  std::vector<float> q(n);
  if (!gb200_butteraugli_adaptive_quantization(flat.data(), static_cast<int>(xsize), static_cast<int>(ysize), device,
                                               q.data()))
    return false;
  quant.insert(quant.end(), q.begin(), q.end());  // the reference appends too
  return true;
}

}  // namespace guetzli_b200

#endif  // GUETZLI_B200_COMPAT_H_
