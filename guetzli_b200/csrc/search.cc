// See search.h.  Everything O(pixels) or O(blocks) runs in ImageContext kernels;
// this file is scalar control flow plus the (for now host-side) sequential
// selection walk and JPEG serialisation.
#include "search.h"
#include "jpeg_in.h"

#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <set>
#include <stdexcept>
#include <vector>

#include "exact_sort.h"
#include "jpeg_out.h"
#include "pipeline.h"
#include "tables.h"

namespace gb200 {

long total_launches();
long long h2d_bytes_total();
long long d2h_bytes_total();

double score_jpeg(double distance, int size, double target) {
  const double kScale = 50, kMaxExponent = 10, kLargeSize = 1e30;
  const double diff = distance - target;
  if (diff <= 0.0) return size;
  const double exponent = kScale * diff;
  if (exponent > kMaxExponent) return kLargeSize * std::exp(kMaxExponent) * diff + size;
  return std::exp(exponent) * size;
}

namespace {

typedef std::chrono::steady_clock Clock;
double ms_since(Clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(Clock::now() - t0).count();
}

struct QuantTrial {
  int q[3][64];
  size_t jpg_size;
  bool dist_ok;
};

// -1 / 0 / 1 when a <= b / a == b / a >= b coordinate-wise, 2 when incomparable
// (g/processor.cc:161).
int compare_quant(const int* a, const int* b) {
  int i = 0;
  while (i < 192 && a[i] == b[i]) ++i;
  if (i == 192) return 0;
  if (a[i] < b[i]) {
    for (++i; i < 192; ++i)
      if (a[i] > b[i]) return 2;
    return -1;
  }
  for (++i; i < 192; ++i)
    if (a[i] < b[i]) return 2;
  return 1;
}

double contrast_sensitivity(int k) { return 1.0 / (1.0 + natural_to_zigzag()[k] / 2.0); }

double quant_heuristic_score(const int q[3][64]) {
  double score = 0.0;
  for (int c = 0; c < 3; ++c)
    for (int k = 0; k < 64; ++k) score += 0.5 * (q[c][k] - 1.0) * contrast_sensitivity(k);
  return score;
}

// Bisection over a scalar "heuristic score" that indexes a one-parameter family
// of quant matrices (g/processor.cc:194-296).
class QuantBisection {
 public:
  // downsample: the generator of the YUV420 pass starts from score 0 (g/processor.cc:204)
  explicit QuantBisection(bool downsample) : downsample_(downsample), lo_(-1.0), hi_(-1.0), total_csf_(0.0) {
    for (int k = 0; k < 64; ++k) total_csf_ += 3.0 * contrast_sensitivity(k);
  }

  bool next(int q[3][64]) {
    for (int iter = 0; iter < 1000; ++iter) {
      double hscore;
      if (hi_ == -1.0) {
        if (lo_ == -1.0) {
          hscore = downsample_ ? 0.0 : total_csf_;
        } else if (lo_ < 5.0 * total_csf_) {
          hscore = lo_ + total_csf_;
        } else {
          hscore = 2 * (lo_ + total_csf_);
        }
        if (hscore > 100 * total_csf_) return false;
      } else if (hi_ == 0.0) {
        return false;
      } else if (lo_ == -1.0) {
        hscore = 0.0;
      } else {
        int lower_q[3][64], upper_q[3][64];
        const double kEps = 0.05;
        matrix_for_score((1 - kEps) * lo_ + kEps * 0.5 * (lo_ + hi_), lower_q);
        matrix_for_score((1 - kEps) * hi_ + kEps * 0.5 * (lo_ + hi_), upper_q);
        if (compare_quant(&lower_q[0][0], &upper_q[0][0]) == 0) return false;
        hscore = (lo_ + hi_) * 0.5;
      }
      matrix_for_score(hscore, q);
      bool retry = false;
      for (size_t i = 0; i < tried_.size(); ++i) {
        if (compare_quant(&q[0][0], &tried_[i].q[0][0]) == 0) {
          if (tried_[i].dist_ok) lo_ = hscore; else hi_ = hscore;
          retry = true;
          break;
        }
      }
      if (!retry) return true;
    }
    return false;
  }

  void add(const QuantTrial& t) {
    tried_.push_back(t);
    const double hscore = quant_heuristic_score(t.q);
    if (t.dist_ok) {
      lo_ = std::max(lo_, hscore);
    } else {
      hi_ = hi_ == -1.0 ? hscore : std::min(hi_, hscore);
    }
  }

 private:
  void matrix_for_score(double score, int q[3][64]) const {
    const int level = static_cast<int>(score / total_csf_);
    score -= level * total_csf_;
    const int* zz = zigzag_to_natural();
    for (int k = 63; k >= 0; --k) {
      for (int c = 0; c < 3; ++c) q[c][zz[k]] = 2 * level + (score > 0.0 ? 3 : 1);
      score -= 3.0 * contrast_sensitivity(zz[k]);
    }
  }
  bool downsample_;
  double lo_, hi_, total_csf_;
  std::vector<QuantTrial> tried_;
};

class Search {
 public:
  Search(const SearchParams& p, ImageContext* ctx, LogSink log, void* log_user, SearchStats* st)
      : params_(p), ctx_(ctx), log_(log), log_user_(log_user), st_(st), best_score_(-1.0), distance_(0.0f) {
    const Geom& g = ctx->geom();
    img_.w = g.w;
    img_.h = g.h;
    img_.bw = g.bw;
    img_.bh = g.bh;
    img_.nblocks = g.nblocks;
    cand_.assign(ctx->orig_coeffs().begin(), ctx->orig_coeffs().end());
    img_.coeffs = cand_.data();
    for (int c = 0; c < 3; ++c)
      for (int k = 0; k < 64; ++k) img_.q[c][k] = 1;
  }

  void set_meta(const JpegMeta* meta) { img_.meta = meta; }
  // Params::force_420 on a grayscale image: the reference's YUV420 pass finds nothing to downsample
  // (OutputImage::Downsample returns at once, g/output_image.cc:305) and runs, instead of the 4:4:4
  // pass, on the one-component JPEGData that SaveToJpegData leaves (g/processor.cc:855-877): quant
  // search from score 0, frequency masking of component 0 only with one AC histogram, and the
  // second masking call (comp_mask 6) returns at once (:577).
  void set_yuv420_gray() {
    yuv420_gray_ = true;
    sfm_ncomp_ = 1;
  }

  // JPEG input: the original's own quant tables (q_in of g/processor.cc:825), file
  // structure and metadata.  All pointers must outlive run().
  void set_jpeg_source(const int q_in[3][64], const JpegFileLayout* layout, const JpegMeta* meta) {
    memcpy(q_in_, q_in, sizeof(q_in_));
    layout_ = layout;
    img_.meta = meta;
    jpeg_source_ = true;
  }

  void run(std::string* best_out) {
    best_ = best_out;
    const float target = params_.butteraugli_target;
    // the input itself (RGB: its q=1 encoding; JPEG: the file re-serialised) is the
    // fallback output (g/processor.cc:826-846)
    if (jpeg_source_) {
      set_global_quant(q_in_);  // coefficients are multiples of q_in: values unchanged
      img_.as_read = layout_;
    } else {
      img_.as_encoded = true;
    }
    const size_t encoded = encoded_size();
    logf("Original Out[%7zd]", encoded);
    compare();
    maybe_output(encoded);
    img_.as_encoded = false;
    img_.as_read = nullptr;
    int best_q[3][64];
    for (int c = 0; c < 3; ++c)
      for (int k = 0; k < 64; ++k) best_q[c][k] = jpeg_source_ ? q_in_[c][k] : 1;
    if (!select_quant_matrix(best_q)) {
      for (int c = 0; c < 3; ++c)
        for (int k = 0; k < 64; ++k) best_q[c][k] = 1;
    }
    set_global_quant(best_q);
    try {
      select_frequency_masking(1.0);
    } catch (...) {
      try {
        finish_output();  // like the reference, leave the best output found so far
      } catch (...) {
      }
      throw;
    }
    finish_output();
    (void)target;
  }

 private:
  void logf(const char* fmt, ...) {
    if (!log_) return;
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    log_(log_user_, buf);
  }
  void log_quant(const int q[3][64]) {
    for (int y = 0; y < 8; ++y) {
      for (int c = 0; c < 3; ++c) {
        for (int x = 0; x < 8; ++x) logf(" %2d", q[c][8 * y + x]);
        logf("   ");
      }
      logf("\n");
    }
  }

  // a11 on the device: exact size of the candidate's JPEG; the bytes are fetched
  // only when the candidate becomes the best output.
  // host_ac != nullptr: the AC histograms the selection walk keeps up to date on the
  // host (exactly the candidate's, like the reference's own incremental bookkeeping,
  // g/processor.cc:471-495) replace the device histogram pass and its round trip; DC
  // symbols do not change during frequency masking (sfm_dc_hist_, captured at its start).
  size_t encoded_size(const SymbolHistogram* host_ac = nullptr) {
    Clock::time_point t0 = Clock::now();
    unsigned int hist[6][257];
    bool chroma = false;
    SymbolHistogram dc_h[3], ac_h[3];
    int ncomp;
    if (host_ac != nullptr) {
      chroma = chroma_nz_ > 0;  // kept incrementally: the host mirror of the candidate may be stale
      ncomp = chroma ? 3 : 1;
      for (int c = 0; c < ncomp; ++c) {
        for (int i = 0; i < 256; ++i) dc_h[c].counts[i] = 2 * sfm_dc_hist_[c][i];
        ac_h[c] = host_ac[c];
      }
      static const bool kCheck = getenv("GB200_CHECK_HOST_HIST") != nullptr;
      if (kCheck) {
        bool dev_chroma = false;
        ctx_->jpeg_histograms(&hist[0][0], &dev_chroma);
        bool same = dev_chroma == chroma;
        for (int c = 0; c < ncomp && same; ++c)
          for (int i = 0; i < 256 && same; ++i)
            same = 2 * hist[c][i] == dc_h[c].counts[i] && 2 * hist[3 + c][i] == ac_h[c].counts[i];
        if (!same) throw std::runtime_error("host symbol histograms differ from the device's");
      }
    } else {
      ctx_->jpeg_histograms(&hist[0][0], &chroma);
      ncomp = (img_.as_encoded || img_.as_read) ? 3 : (chroma ? 3 : 1);
      for (int c = 0; c < ncomp; ++c)
        for (int i = 0; i < 256; ++i) {
          dc_h[c].counts[i] = 2 * hist[c][i];
          ac_h[c].counts[i] = 2 * hist[3 + c][i];
        }
    }
    // symbol counts before the clustering merges them: with the final code lengths they give
    // the length of the scan (code + extra bits per symbol; extra bits = the DC category, the
    // low nibble of an AC symbol), so the device pass needs no round trip to size its buffers
    uint32_t raw[6][256];
    for (int c = 0; c < ncomp; ++c)
      for (int i = 0; i < 256; ++i) {
        raw[c][i] = dc_h[c].counts[i] / 2;
        raw[3 + c][i] = ac_h[c].counts[i] / 2;
      }
    plan_ = plan_jpeg(img_, ncomp, dc_h, ac_h);
    unsigned long long expected_bits = 0;
    for (int c = 0; c < ncomp; ++c)
      for (int i = 0; i < 256; ++i) {
        expected_bits += static_cast<unsigned long long>(raw[c][i]) * (plan_.depth[c][i] + (i & 15));
        expected_bits += static_cast<unsigned long long>(raw[3 + c][i]) * (plan_.depth[3 + c][i] + (i & 15));
      }
    size_t nbytes = 0, num_ff = 0;
    ctx_->jpeg_encode_scan(ncomp, &plan_.depth[0][0], &plan_.code[0][0], expected_bits, &nbytes, &num_ff);
    scan_bytes_ = nbytes;
    st_->ms_jpeg += ms_since(t0);
    return plan_.prefix.size() + nbytes + num_ff + plan_.trailer.size();
  }

  // DC symbol counts of the current candidate (device pass), for encoded_size(host_ac)
  void capture_dc_histograms() {
    unsigned int hist[6][257];
    bool chroma = false;
    ctx_->jpeg_histograms(&hist[0][0], &chroma);
    memcpy(sfm_dc_hist_, hist, sizeof(sfm_dc_hist_));
  }

  // the best candidate's bytes: kept scan + its headers (g/processor.cc:139-148 keeps the string)
  void finish_output() {
    if (!have_best_) return;
    Clock::time_point t0 = Clock::now();
    // headers (host-built: they hold the Huffman tables), byte stuffing and the trailer are put
    // together on the device; the file crosses PCIe once (scope row f1)
    ctx_->jpeg_fetch_kept_file(best_plan_.prefix, best_plan_.trailer, best_);
    have_best_ = false;
    st_->ms_jpeg += ms_since(t0);
    if (best_->size() != best_bytes_) throw std::runtime_error("device JPEG size mismatch");
  }

  std::string fetch_encoded() {
    Clock::time_point t0 = Clock::now();
    std::string s;
    ctx_->jpeg_fetch_file(plan_.prefix, plan_.trailer, &s);
    st_->ms_jpeg += ms_since(t0);
    return s;
  }

  void compare() {
    Clock::time_point t0 = Clock::now();
    distance_ = ctx_->compare();
    st_->ms_compare += ms_since(t0);
    ++st_->compares;
    logf(" BA[100.00%%] D[%6.4f]", distance_);
  }
  // the same around other work: the metric's kernels are queued first, the caller's JPEG size
  // pass (host code planning + its kernels) follows while they run
  void compare_begin() {
    Clock::time_point t0 = Clock::now();
    ctx_->compare_begin();
    st_->ms_compare += ms_since(t0);
  }
  void compare_end() {
    Clock::time_point t0 = Clock::now();
    distance_ = ctx_->compare_end();
    st_->ms_compare += ms_since(t0);
    ++st_->compares;
    logf(" BA[100.00%%] D[%6.4f]", distance_);
  }

  bool distance_ok(double target_mul) const {
    return distance_ <= target_mul * params_.butteraugli_target;
  }

  void maybe_output(size_t encoded_bytes) {
    const double score = score_jpeg(distance_, static_cast<int>(encoded_bytes), params_.butteraugli_target);
    logf(" Score[%.4f]", score);
    if (score < best_score_ || best_score_ < 0) {
      // the scan stays on the device (one device-to-device copy); it is fetched and wrapped
      // into the file once, by finish_output()
      ctx_->jpeg_keep_scan();
      best_plan_ = plan_;
      best_bytes_ = encoded_bytes;
      have_best_ = true;
      best_score_ = score;
      logf(" (*)");
    }
    logf("\n");
  }

  // candidate := Quantize(original, q) on the device; the host mirror of the candidate goes
  // stale (the host paths of the walk refresh it when they need it)
  void set_global_quant(const int q[3][64]) {
    memcpy(img_.q, q, sizeof(img_.q));
    ctx_->apply_global_quant(&q[0][0]);
    mirror_valid_ = false;
  }

  QuantTrial try_quant_matrix(const float target_mul, int q[3][64]) {
    QuantTrial data;
    memcpy(data.q, q, sizeof(data.q));
    set_global_quant(q);
    const size_t encoded = encoded_size();
    logf("Iter %2d: %s quantization matrix:\n", st_->iterations + 1, "f111111");
    log_quant(q);
    logf("Iter %2d: %s GQ[%5.2f] Out[%7zd]", st_->iterations + 1, "f111111", quant_heuristic_score(q),
         encoded);
    ++st_->iterations;
    compare();
    data.dist_ok = distance_ok(target_mul);
    data.jpg_size = encoded;
    maybe_output(encoded);
    return data;
  }

  static bool better(const QuantTrial& a, const QuantTrial& b) {
    if (a.dist_ok && !b.dist_ok) return true;
    if (!a.dist_ok && b.dist_ok) return false;
    return a.jpg_size < b.jpg_size;
  }

  bool select_quant_matrix(int best_q[3][64]) {
    QuantBisection gen(yuv420_gray_);
    const float target_mul_high = 0.97f, target_mul_low = 0.95f;
    QuantTrial best = try_quant_matrix(target_mul_high, best_q);
    for (;;) {
      int q_next[3][64];
      if (!gen.next(q_next)) break;
      QuantTrial data = try_quant_matrix(target_mul_high, q_next);
      gen.add(data);
      if (better(data, best)) {
        best = data;
        if (data.dist_ok && !distance_ok(target_mul_low)) break;
      }
    }
    memcpy(&best_q[0][0], &best.q[0][0], sizeof(best.q));
    logf("\n%s selected quantization matrix:\n", yuv420_gray_ ? "YUV420" : "YUV444");
    log_quant(best_q);
    return best.dist_ok;
  }

  // ---- a12/a16: frequency masking ----------------------------------------
  struct Sfm {
    std::vector<int> offsets;          // [nblocks+1] into cand_idx / cand_err
    std::vector<uint8_t> cand_idx;     // coefficient index (c*64+k) per candidate
    std::vector<float> cand_err;       // monotone block error per candidate
    SymbolHistogram ac_h[3];
    std::vector<uint8_t> ac_depths;
    int ac_histogram_size, header_size, dc_size;
    std::vector<float> max_block_error;
    std::vector<int> last_indexes;
    std::vector<char> block_changed;
    std::vector<int> edit_index;
    std::vector<int16_t> edit_value, edit_old;
  };

  struct WalkOutcome {
    size_t consumed = 0;       // entries applied
    bool stopped = false;      // stop test fired (else: ran out of entries)
    size_t changed_blocks = 0;
    float val_threshold = 0.0f;
    int est_jpg_size = 0;
    bool ambiguous = false;    // check_ties only: result depends on the order of equal keys
    int why = 0;               // diagnostic: which rule flagged the ambiguity
  };

  // The sequential selection walk (g/processor.cc:700-750) over `order`.
  // The walk only *reads* the size estimate in its stop test, and the stop test
  // cannot fire before min_coeffs_to_change entries are consumed; so the entropy
  // codes (refreshed at every 10th entry) and the estimate are evaluated only in
  // the 10-entry windows that can reach the test, or that contain the last entry.
  // Same integers as the reference's eager loop.
  // What consuming the next candidate of block_ix does (no side effects).
  struct Edit {
    int c, k, za, zb, newval;
    bool store;  // false: "precious" coefficient kept (g/processor.cc:722-733)
  };
  Edit plan_edit(const Sfm& m, int block_ix, int direction) const {
    const std::vector<int16_t>& orig = ctx_->orig_coeffs();
    const size_t per = static_cast<size_t>(img_.nblocks) * 64;
    const int* zz2nat = zigzag_to_natural();
    const int* nat2zz = natural_to_zigzag();
    Edit e;
    const int last_idx = m.last_indexes[block_ix];
    const uint8_t* candidates = &m.cand_idx[m.offsets[block_ix]];
    const int idx = candidates[last_idx + std::min(direction, 0)];
    e.c = idx / 64;
    e.k = idx % 64;
    const int* quant = img_.q[e.c];
    const int16_t* orig_block = &orig[e.c * per + static_cast<size_t>(block_ix) * 64];
    e.newval = direction > 0 ? 0 : quantize_coeff(orig_block[e.k], quant[e.k]);
    const int16_t* block = &cand_[e.c * per + static_cast<size_t>(block_ix) * 64];
    // only the symbols between the neighbouring nonzero coefficients (in zig-zag
    // order) can change
    const int zp = nat2zz[e.k];
    e.za = zp - 1;
    e.zb = zp + 1;
    while (e.za > 0 && block[zz2nat[e.za]] == 0) --e.za;
    while (e.zb < 64 && block[zz2nat[e.zb]] == 0) ++e.zb;
    bool precious = false;
    if (e.k == 1 || e.k == 8) {
      double sum_of_hf = 0;
      for (int ii = 3; ii < 64; ++ii) {
        if ((ii & 7) < 3 && ii < 3 * 8) continue;
        sum_of_hf += std::abs(orig_block[ii]);
      }
      const int limit = sum_of_hf < 60 ? 4 : 8;
      precious = std::abs(orig_block[e.k]) >= limit;
    }
    e.store = !precious || e.newval != 0;
    return e;
  }

  // The sequential selection walk (g/processor.cc:700-750) over `order`.
  // The walk only *reads* the size estimate in its stop test, and the stop test
  // cannot fire before min_coeffs_to_change entries are consumed; so the entropy
  // codes (refreshed at every 10th entry) and the estimate are evaluated only in
  // the 10-entry windows that can reach the test, or that contain the last entry.
  // Same integers as the reference's eager loop.
  //
  // check_ties: `order` is sorted by key but equal keys may be arranged differently
  // from the reference's std::sort.  Entries carry only a block index, so that
  // matters solely where two different blocks with equal keys straddle a point at
  // which the walk looks at its state: an entropy-code refresh or a stop test.  At
  // a stop test the alternative (the other block first) is evaluated as well; if
  // both arrangements decide "continue" the states coincide again one entry later.
  // Anything else sets out.ambiguous and the caller redoes the iteration with the
  // complete reference-ordered sort.
  // `order` may be only a prefix of the complete sorted order of n_total entries; the
  // caller must then discard the outcome unless the walk stopped inside the prefix.
  // `order` may also be a slice of the sorted order that starts at global position `base`
  // (device half of the walk, walk_dev.h): entries [start, end) of the slice are consumed,
  // the others only serve the tie analysis; fresh = false continues an iteration (edit lists
  // and changed-block flags are kept, changed0 blocks were already counted).
  WalkOutcome walk(Sfm& m, const std::vector<std::pair<int, float> >& order, size_t n_total, int direction,
                   int min_coeffs_to_change, double min_size_delta, int prev_size, bool check_ties, size_t base = 0,
                   size_t start = 0, size_t end = static_cast<size_t>(-1), bool fresh = true, size_t changed0 = 0) {
    const size_t per = static_cast<size_t>(img_.nblocks) * 64;
    const int16_t* orig_ = ctx_->orig_coeffs().data();
    WalkOutcome out;
    out.est_jpg_size = prev_size;
    out.changed_blocks = changed0;
    out.consumed = base + start;
    if (fresh) {
      std::fill(m.block_changed.begin(), m.block_changed.end(), 0);
      m.edit_index.clear();
      m.edit_value.clear();
      m.edit_old.clear();
    }
    const size_t n_avail = order.size();
    const size_t n_order = n_total;
    const size_t i_end = std::min(end, n_avail);
    for (size_t i = start; i < i_end; ++i) {
      const size_t gi = base + i;  // position in the complete order
      // every entry touches a different block: hide the cache misses
      if (i + 12 < n_avail) {
        const int pb = order[i + 12].first;
        __builtin_prefetch(&m.last_indexes[pb]);
        __builtin_prefetch(&m.offsets[pb]);
        __builtin_prefetch(&m.block_changed[pb]);
      }
      if (i + 6 < n_avail) {
        const int pb = order[i + 6].first;
        const int pli = m.last_indexes[pb] + std::min(direction, 0);
        const uint8_t* pc = &m.cand_idx[m.offsets[pb]];
        __builtin_prefetch(pc + (pli < 0 ? 0 : pli));
        for (int c = 0; c < 3; ++c) {
          __builtin_prefetch(&cand_[c * per + static_cast<size_t>(pb) * 64]);
          __builtin_prefetch(&cand_[c * per + static_cast<size_t>(pb) * 64 + 32]);
        }
      }
      if (i + 3 < n_avail) {
        // the candidate index is in cache by now: fetch the original coefficient it refers to
        const int pb = order[i + 3].first;
        const int pli = m.last_indexes[pb] + std::min(direction, 0);
        const int idx = m.cand_idx[m.offsets[pb] + (pli < 0 ? 0 : pli)];
        __builtin_prefetch(&orig_[(idx >> 6) * per + static_cast<size_t>(pb) * 64 + (idx & 63)]);
      }
      const int block_ix = order[i].first;
      const bool refresh_here =
          (gi % 10 == 0) && (static_cast<long long>(gi) + 9 >= min_coeffs_to_change || n_order - 1 <= gi + 9);
      const bool can_test = static_cast<long long>(gi) + 1 > min_coeffs_to_change;  // changed_coeffs == gi
      const bool eval_here = can_test || gi + 1 == n_order;
      // does a run of equal keys that contains two different blocks cross the boundary
      // i | i+1 ?  (then the set of entries applied so far depends on the arrangement)
      bool straddle = false, pair_only = false;
      if (check_ties && (refresh_here || eval_here) && i + 1 < n_avail &&
          !(order[i].second < order[i + 1].second)) {
        const float key = order[i].second;
        size_t lo = i, hi = i + 1;
        // a block has at most 189 entries: a run longer than that holds several blocks, no
        // need to walk to its ends (long runs are common on smooth images)
        const size_t kRunCap = 256;
        while (lo > 0 && i - lo < kRunCap && !(order[lo - 1].second < key)) --lo;
        while (hi + 1 < n_avail && hi - i < kRunCap && !(key < order[hi + 1].second)) ++hi;
        if (i - lo >= kRunCap || hi - i >= kRunCap) straddle = true;
        for (size_t j = lo + 1; j <= hi && !straddle; ++j)
          if (order[j].first != order[lo].first) straddle = true;
        // the run may continue beyond the fetched prefix, or begin before the fetched slice
        if (hi + 1 == n_avail && base + n_avail < n_order) straddle = true;
        if (lo == 0 && base > 0) straddle = true;
        pair_only = straddle && lo == i && hi == i + 1;
      }
      int alt_est = 0;
      bool have_alt = false;
      if (straddle) {
        // tractable case: a run of exactly two entries at a plain stop test
        if (!pair_only || refresh_here || !can_test) {
          out.ambiguous = true;
          out.why = !pair_only ? (refresh_here ? 1 : 2) : (refresh_here ? 3 : 4);
          return out;
        }
        const int other = order[i + 1].first;
        const Edit e2 = plan_edit(m, other, direction);
        SymbolHistogram alt[3] = {m.ac_h[0], m.ac_h[1], m.ac_h[2]};
        int16_t tmp[64];
        memcpy(tmp, &cand_[e2.c * per + static_cast<size_t>(other) * 64], sizeof(tmp));
        ac_symbols_of_range(tmp, img_.q[e2.c], e2.za, e2.zb, -1, &alt[e2.c]);
        if (e2.store) tmp[e2.k] = static_cast<int16_t>(e2.newval);
        ac_symbols_of_range(tmp, img_.q[e2.c], e2.za, e2.zb, 1, &alt[e2.c]);
        alt_est = m.header_size + m.dc_size + m.ac_histogram_size +
                  static_cast<int>(entropy_coded_bytes(alt, m.ac_depths.data()));
        have_alt = true;
      }
      const Edit e = plan_edit(m, block_ix, direction);
      const int* quant = img_.q[e.c];
      int16_t* block = &cand_[e.c * per + static_cast<size_t>(block_ix) * 64];
      ac_symbols_of_range(block, quant, e.za, e.zb, -1, &m.ac_h[e.c]);
      if (e.store) {
        m.edit_index.push_back(static_cast<int>(e.c * per + static_cast<size_t>(block_ix) * 64 + e.k));
        m.edit_value.push_back(static_cast<int16_t>(e.newval));
        m.edit_old.push_back(block[e.k]);
        block[e.k] = static_cast<int16_t>(e.newval);
      }
      ac_symbols_of_range(block, quant, e.za, e.zb, 1, &m.ac_h[e.c]);
      m.last_indexes[block_ix] += direction;
      if (!m.block_changed[block_ix]) {
        m.block_changed[block_ix] = 1;
        ++out.changed_blocks;
      }
      out.val_threshold = order[i].second;
      out.consumed = gi + 1;
      if (refresh_here)
        m.ac_histogram_size = static_cast<int>(compute_entropy_codes(m.ac_h, m.ac_depths.data(), sfm_ncomp_));
      if (eval_here) {
        out.est_jpg_size = m.header_size + m.dc_size + m.ac_histogram_size +
                           static_cast<int>(entropy_coded_bytes(m.ac_h, m.ac_depths.data()));
        const bool stop = can_test && std::abs(out.est_jpg_size - prev_size) > min_size_delta;
        if (have_alt) {
          const bool alt_stop = std::abs(alt_est - prev_size) > min_size_delta;
          if (stop || alt_stop) {
            out.ambiguous = true;
            out.why = 5;
            return out;
          }
        }
        if (stop) {
          out.stopped = true;
          break;
        }
      }
    }
    return out;
  }

  // Rolls the host state back to before walk() (used when the partial order turns
  // out to be insufficient or ambiguous).
  void unwalk(Sfm& m, const std::vector<std::pair<int, float> >& order, const WalkOutcome& out, int direction,
              const SymbolHistogram saved_h[3], int saved_hist_size, const std::vector<uint8_t>& saved_depths) {
    for (size_t i = m.edit_index.size(); i-- > 0;) cand_[m.edit_index[i]] = m.edit_old[i];
    for (size_t i = 0; i < out.consumed; ++i) m.last_indexes[order[i].first] -= direction;
    for (int c = 0; c < 3; ++c) m.ac_h[c] = saved_h[c];
    m.ac_histogram_size = saved_hist_size;
    m.ac_depths = saved_depths;
  }

  // One "down" iteration with the device half of the walk (walk_dev.h).  exact: the order is
  // the prefix of the reference-ordered std::sort (device replay, order_exact.h), else the
  // radix-selected smallest keys sorted on the device (tie analysis on).
  // -> 1 done (edits of the host window in m.edit_*), 0 ambiguous, -1 not applicable / ran
  // out of entries; in the last two cases everything is as before the call.
  int device_walk(Sfm& m, bool exact, size_t order_size, int direction, int min_coeffs_to_change, double min_size_delta,
                  int prev_size, size_t last_consumed, WalkOutcome* result) {
    // first entry after which the walk looks at its state: an entropy-code refresh needs
    // gi % 10 == 0 and gi + 9 >= min(min_coeffs, n - 1); the stop test gi >= min_coeffs, the final
    // estimate gi == n - 1
    const size_t x_first = std::min<size_t>(static_cast<size_t>(std::max(min_coeffs_to_change, 0)), order_size - 1);
    const size_t i0 = 10 * (x_first / 10);
    if (i0 < 256) return -1;
    Clock::time_point t0 = Clock::now();
    std::vector<std::pair<int, float> >& order = order_buf_;
    size_t base = 0, n_slice = 0, usable_end = 0;
    std::vector<int> bulk_blocks;
    bool split_count = false;  // the device already holds per-block counts of the entries before `base`
    if (exact) {
      Tick tk(&dt_[0]);
      size_t want = std::max(direction < 0 ? last_consumed : 0, i0) + std::min<size_t>(std::max<size_t>(i0 / 8, 1024), 16384),
             dev_total = 0;
      if (want > order_size) want = order_size;
      const size_t k_end = ctx_->exact_order_prefix_resident(direction, want, &order, &dev_total);
      if (dev_total != order_size) throw std::runtime_error("exact_order_prefix: entry count mismatch");
      if (k_end < i0 + 16 && k_end < order_size) return -1;
      n_slice = k_end;
      usable_end = k_end;
      bulk_blocks.resize(i0);
      for (size_t i = 0; i < i0; ++i) bulk_blocks[i] = order[i].first;
    } else {
      Tick tk(&dt_[1]);
      // two-rank select: everything certainly before position i0 - 64 is counted into the bulk
      // on the device right away; the entries from there up to the rank the window may reach
      // (the "middle") come back sorted -- their head completes the bulk, the rest is the window
      const size_t pre = 64;
      size_t total = 0, before = 0, n_mid = 0;
      // A long run of (nearly) equal keys just behind the window would drag all of its entries
      // into the middle list: shrink the upper rank until the middle is small.  (A run that
      // reaches position i0 itself cannot be avoided: the reference-ordered path then.)
      const size_t margins[3] = {std::min<size_t>(std::max<size_t>(i0 / 16, 1024), 8192), 256, 64};
      bool usable = false;
      for (int attempt = 0; attempt < 3 && !usable; ++attempt) {
        const size_t rank_hi =
            std::min(order_size, std::max(direction < 0 && attempt == 0 ? last_consumed : 0, i0) + margins[attempt]);
        n_mid = ctx_->walk_select_split(direction, i0 - pre, rank_hi, &before, &total);
        if (total != order_size) throw std::runtime_error("walk_select_split: entry count mismatch");
        dbg_n_[1] += n_mid;
        if (n_mid > dbg_mid_max_) dbg_mid_max_ = n_mid;
        if (n_mid > ImageContext::walk_middle_max()) {
          ctx_->walk_split_cancel();
        } else {
          usable = true;
        }
      }
      split_count = true;
      base = before;
      n_slice = n_mid;
      usable_end = n_slice;
      if (!usable) {
        st_->ms_sort += ms_since(t0);
        return 0;  // as if ambiguous: only the reference's own arrangement can split such a run
      }
      if (before + pre > i0 || (before + n_mid < i0 + 64 && before + n_mid < order_size)) {
        ctx_->walk_split_cancel();
        st_->ms_sort += ms_since(t0);
        return -1;
      }
    }
    ImageContext::BulkResult bulk;
    size_t pre_first = 0, pre_n = 0;
    {
      Tick tk(&dt_[2]);
      if (exact) {
        ctx_->walk_bulk_apply(direction, i0, &bulk, bulk_blocks.data());
      } else {
        // the window's first chunk: its block states are gathered right behind the bulk
        pre_first = i0 - base;
        pre_n = std::min<size_t>(64, usable_end > pre_first ? usable_end - pre_first : 0);
        ctx_->walk_bulk_apply(direction, i0 - base, &bulk, nullptr, split_count, pre_first, pre_n);
      }
    }
    if (!exact) {
      // the sorted middle comes back after the bulk's kernels were queued: one wait covers both
      Tick tk(&dt_[1]);
      order.resize(n_slice);
      ctx_->walk_fetch_pairs(n_slice, order.data());
    }
    st_->ms_sort += ms_since(t0);
    Clock::time_point tw = Clock::now();
    SymbolHistogram saved_h[3] = {m.ac_h[0], m.ac_h[1], m.ac_h[2]};
    const int saved_hist_size = m.ac_histogram_size;
    const std::vector<uint8_t> saved_depths = m.ac_depths;
    for (int c = 0; c < 3; ++c)
      for (int i = 0; i < 256; ++i) m.ac_h[c].counts[i] += static_cast<uint32_t>(2 * bulk.delta_hist[c][i]);
    mirror_valid_ = false;
    std::fill(m.block_changed.begin(), m.block_changed.end(), 0);
    m.edit_index.clear();
    m.edit_value.clear();
    m.edit_old.clear();
    for (size_t i = 0; i < fetched_list_.size(); ++i) fetched_[fetched_list_[i]] = 0;
    fetched_list_.clear();
    if (fetched_.size() != static_cast<size_t>(img_.nblocks)) fetched_.assign(img_.nblocks, 0);
    size_t pos = i0 - base, chunk = 64;  // the walk usually stops a few entries after i0
    size_t changed = static_cast<size_t>(bulk.touched);
    WalkOutcome out;
    bool ok = true;
    const size_t per = static_cast<size_t>(img_.nblocks) * 64;
    while (true) {
      const size_t end = std::min(usable_end, pos + chunk);
      // state of the blocks of this chunk that the host does not hold yet
      std::vector<int> need;
      std::vector<size_t> slot;  // where a needed block's state sits in the gathered arrays
      const bool pre = pre_n > 0 && pos == pre_first && end - pos == pre_n;
      for (size_t i = pos; i < end; ++i) {
        const int b = order[i].first;
        if (!fetched_[b]) {
          fetched_[b] = 1;
          fetched_list_.push_back(b);
          need.push_back(b);
          slot.push_back(pre ? i - pos : need.size() - 1);
        }
      }
      std::vector<int16_t> gc;
      std::vector<int> gcur, gin;
      {
        Tick tk(&dt_[3]);
        if (pre) {
          ctx_->walk_gather_selection_fetch(pre_n, &gc, &gcur, &gin);  // one slot per entry, queued with the bulk
        } else {
          ctx_->walk_gather(need, &gc, &gcur, &gin);
        }
      }
      Tick tk4(&dt_[4]);
      for (size_t k = 0; k < need.size(); ++k) {
        const int b = need[k];
        const size_t e = slot[k];
        for (int c = 0; c < 3; ++c)
          memcpy(&cand_[c * per + static_cast<size_t>(b) * 64], &gc[(e * 3 + c) * 64], 64 * sizeof(int16_t));
        m.last_indexes[b] = gcur[e];
        if (gin[e]) m.block_changed[b] = 1;  // already counted among the bulk's blocks
      }
      out = walk(m, order, order_size, direction, min_coeffs_to_change, min_size_delta, prev_size, !exact, base, pos, end,
                 false, changed);
      if (out.ambiguous) {
        ok = false;
        break;
      }
      changed = out.changed_blocks;
      if (out.stopped) break;
      pos = end;
      if (pos >= usable_end) {  // the entries ran out before the walk stopped
        ok = base + usable_end == order_size;
        break;
      }
      chunk *= 4;
    }
    // a stop on the very last fetched entry cannot be told from running out of them
    if (ok && out.stopped && base + usable_end < order_size && out.consumed >= base + usable_end) ok = false;
    st_->ms_walk += ms_since(tw);
    if (ok) {
      Tick tk(&dt_[5]);
      ++device_walks_;
      // device: cursors of the window's entries, the new max errors (the window's coefficient
      // edits follow with the common scatter)
      std::vector<int> consumed_blocks;
      for (size_t gi = i0; gi < out.consumed; ++gi) consumed_blocks.push_back(order[gi - base].first);
      ctx_->walk_advance(consumed_blocks, direction);
      ctx_->walk_add_max_err(out.val_threshold, direction);
      chroma_nz_ += bulk.chroma_delta;
      device_done_ = true;
      *result = out;
      return 1;
    }
    if (out.ambiguous) {
      ++tie_fallbacks_;
      ++tie_why_[out.why];
    }
    ctx_->walk_bulk_undo(direction);
    for (int c = 0; c < 3; ++c) m.ac_h[c] = saved_h[c];
    m.ac_histogram_size = saved_hist_size;
    m.ac_depths = saved_depths;
    m.edit_index.clear();
    m.edit_value.clear();
    m.edit_old.clear();
    // ambiguous, or the fetched entries ran out: worth another try on the reference-ordered
    // prefix (which fetches more); from there the host paths take over
    return exact ? -1 : 0;
  }

  void select_frequency_masking(const double target_mul) {
    const int num_blocks = img_.nblocks;
    Sfm m;
    // a13 + a14 on the device: per-block candidate lists
    m.offsets.resize(num_blocks + 1);
    std::vector<int> count;
    {
      Clock::time_point t0 = Clock::now();
      std::vector<uint8_t> idx;
      // the candidate errors stay on the device; only the host paths of the walk want them
      ctx_->zeroing_orders(params_.butteraugli_target, params_.zeroing_greedy_lookahead, params_.new_zeroing_model, &idx,
                           nullptr, &count);
      size_t total = 0;
      for (int b = 0; b < num_blocks; ++b) total += count[b];
      m.cand_idx.reserve(total);
      for (int b = 0; b < num_blocks; ++b) {
        m.offsets[b] = static_cast<int>(m.cand_idx.size());
        m.cand_idx.insert(m.cand_idx.end(), &idx[static_cast<size_t>(b) * 192], &idx[static_cast<size_t>(b) * 192] + count[b]);
      }
      m.offsets[num_blocks] = static_cast<int>(m.cand_idx.size());
      m.cand_err.clear();
      st_->ms_zeroing += ms_since(t0);
    }

    // symbol counts of the candidate from the device (no pass over the coefficients on the host):
    // header size, EstimateDCSize, the AC histograms the walk keeps up to date
    {
      unsigned int hist[6][257];
      bool chroma = false;
      ctx_->jpeg_histograms(&hist[0][0], &chroma);
      memcpy(sfm_dc_hist_, hist, sizeof(sfm_dc_hist_));
      const int ncomp0 = chroma ? 3 : 1;  // num_output_components (g/output_image.cc:357)
      m.header_size = static_cast<int>(jpeg_header_bytes(img_, ncomp0));
      SymbolHistogram dc_h[3];
      for (int c = 0; c < ncomp0; ++c)
        for (int i = 0; i < 256; ++i) dc_h[c].counts[i] = 2 * hist[c][i];
      m.dc_size = static_cast<int>(estimate_dc_bytes_of(dc_h, ncomp0));
      for (int c = 0; c < 3; ++c) m.ac_h[c].clear();
      for (int c = 0; c < ncomp0; ++c)
        for (int i = 0; i < 256; ++i) m.ac_h[c].counts[i] = 2 * hist[3 + c][i];
      chroma_nz_ = static_cast<long long>(ctx_->count_nonzero_chroma());
    }
    m.ac_depths.resize(3 * SymbolHistogram::kSize);
    m.ac_histogram_size = static_cast<int>(compute_entropy_codes(m.ac_h, m.ac_depths.data(), sfm_ncomp_));
    const int base_size = m.header_size + m.dc_size + m.ac_histogram_size +
                          static_cast<int>(entropy_coded_bytes(m.ac_h, m.ac_depths.data()));
    int prev_size = base_size;

    m.max_block_error.assign(num_blocks, 0.0f);
    m.last_indexes.assign(num_blocks, 0);
    m.block_changed.assign(num_blocks, 0);
    std::vector<float> block_weight(num_blocks);
    size_t last_consumed = 0;
    // The candidate cursors and max errors also live on the device (walk_dev.h); the host
    // copies above (and cand_) are a mirror that iterations on the device path leave stale.
    ctx_->walk_begin();
    weights_queued_ = false;
    fetched_.assign(num_blocks, 0);
    fetched_list_.clear();
    // GB200_WALK=host keeps every iteration on the host path, =device forces the device path.
    // Default: device in the product; host in the CPU port, whose emulated kernels make the
    // device path slow (tests/test_oracle_cpu.py::test_port_device_walk turns it on).
    const bool kDeviceWalk = [] {
      const char* e = getenv("GB200_WALK");
#if defined(GB200_HOSTSIM)
      return e != nullptr && e[0] == 'd';
#else
      return !(e != nullptr && e[0] == 'h');
#endif
    }();

    bool first_up_iter = true;
    const int directions[2] = {1, -1};
    for (int di = 0; di < 2; ++di) {
      const int direction = directions[di];
      for (;;) {
        // a15 on the device; entry counts from the per-block bookkeeping (:625-669)
        size_t order_size = 0;
        int blocks_to_change = 0;
        for (int rblock = 1; rblock <= 4; ++rblock) {
          unsigned long long n_entries = 0, n_blocks = 0;
          Tick tk(&dt_[6]);
          if (weights_queued_ && rblock == 1 && queued_direction_ == direction && !first_up_iter) {
            // queued behind the previous iteration's Compare: only the two sums are fetched
            ctx_->walk_weights_fetch(&n_entries, &n_blocks);
          } else {
            ctx_->walk_weights(direction, rblock, params_.butteraugli_target * target_mul, first_up_iter, &n_entries,
                               &n_blocks);
          }
          weights_queued_ = false;
          order_size = static_cast<size_t>(n_entries);
          blocks_to_change = static_cast<int>(n_blocks);
          if (order_size != 0) break;
        }
        if (order_size == 0) break;
        bool have_weights = false;  // block_weight[] is downloaded only by the host paths

        double rel_size_delta = direction > 0 ? 0.01 : 0.0005;
        if (direction > 0 && distance_ok(1.0)) rel_size_delta = 0.05;
        const double min_size_delta = base_size * rel_size_delta;
        const float coeffs_to_change_per_block = direction > 0 ? 2.0f : 1 * 1 * 0.2f;
        int min_coeffs_to_change = coeffs_to_change_per_block * blocks_to_change;

        std::vector<std::pair<int, float> >& order = order_buf_;  // capacity kept across iterations: no page faults
        order.clear();
        WalkOutcome out;
        bool done = false;
        device_done_ = false;
        // Device path (walk_dev.h): the entries before the first point at which the walk looks
        // at its state are applied on the device as a set; the host runs the sequential loop
        // only from there on, with the state of just the blocks involved.  First on the
        // radix-selected order (equal keys in arbitrary arrangement, tie analysis on); if that
        // is ambiguous, on the prefix of the reference-ordered sort (device replay of std::sort).
        bool skip_partial = false;
        if (kDeviceWalk && order_size > 16384) {
          int min_coeffs = min_coeffs_to_change;
          if (first_up_iter) {
            // partition_point of the sorted order (:690-698) == number of keys below the limit
            const size_t below = ctx_->walk_count_below(direction, 0.75f * params_.butteraugli_target);
            min_coeffs = std::max<int>(min_coeffs, static_cast<int>(below));
          }
          const int r = device_walk(m, false, order_size, direction, min_coeffs, min_size_delta, prev_size,
                                    last_consumed, &out);
          if (r == 1) {
            done = true;
            ++st_->order_partial;
          } else if (r == 0) {
            skip_partial = true;  // the host's partial order would stumble over the same equal keys
            const int r2 = device_walk(m, true, order_size, direction, min_coeffs, min_size_delta, prev_size,
                                       last_consumed, &out);
            if (r2 == 1) {
              done = true;
              ++st_->order_exact;
            }
          }
        }
        if (!done) {
          // host paths: they work on the host mirror of the candidate and of the cursors
          Tick tk(&dt_[8]);
          if (!mirror_valid_) {
            ctx_->download_candidate(cand_.data());
            ctx_->walk_download_state(&m.last_indexes, &m.max_block_error);
            mirror_valid_ = true;
          }
          ctx_->download_weights(block_weight.data());
          have_weights = true;
          if (m.cand_err.empty() && !m.cand_idx.empty()) {
            std::vector<float> err;
            ctx_->download_zeroing_err(&err);
            m.cand_err.reserve(m.cand_idx.size());
            for (int b = 0; b < num_blocks; ++b)
              m.cand_err.insert(m.cand_err.end(), &err[static_cast<size_t>(b) * 192],
                                &err[static_cast<size_t>(b) * 192] + (m.offsets[b + 1] - m.offsets[b]));
          }
        }
        const bool device_done = device_done_;
        // Fast path ("down" iterations consume a tiny prefix of the order): fetch only
        // the smallest keys from the device, sort those, and fall back to the complete
        // reference-ordered sort whenever the result could depend on how std::sort
        // places equal keys of different blocks, or the prefix runs out.
        if (!done && !skip_partial && direction < 0 && order_size > 16384) {
          // the walk usually stops right after min_coeffs_to_change entries
          size_t want = std::max<size_t>(last_consumed, static_cast<size_t>(min_coeffs_to_change)) * 5 / 4 + 512;
          while (!done && want < order_size / 2) {
            Clock::time_point t0 = Clock::now();
            std::vector<float> val;
            std::vector<int> blk;
            const size_t total = ctx_->order_smallest(direction, m.last_indexes, m.max_block_error, want, &val, &blk);
            dbg_ms_[0] += ms_since(t0);
            if (total != order_size) throw std::runtime_error("order_smallest: entry count mismatch");
            if (val.size() >= order_size) break;
            order.resize(val.size());
            for (size_t i = 0; i < val.size(); ++i) order[i] = std::make_pair(blk[i], val[i]);
#if defined(GB200_HOSTSIM)
            // test hook of the CPU port: the device compaction returns the entries in
            // arbitrary order; emulate that to exercise the tie analysis
            if (const char* sh = getenv("GB200_SHUFFLE_ORDER")) {
              unsigned int rng = static_cast<unsigned int>(atoi(sh)) * 2654435761u + static_cast<unsigned int>(st_->iterations);
              for (size_t i = order.size(); i > 1; --i) {
                rng = rng * 1664525u + 1013904223u;
                std::swap(order[i - 1], order[(rng >> 8) % i]);
              }
            }
#endif
            std::sort(order.begin(), order.end(), [](const std::pair<int, float>& a, const std::pair<int, float>& b) {
              return a.second < b.second;
            });
            st_->ms_sort += ms_since(t0);
            Clock::time_point tw = Clock::now();
            SymbolHistogram saved_h[3] = {m.ac_h[0], m.ac_h[1], m.ac_h[2]};
            const int saved_hist_size = m.ac_histogram_size;
            const std::vector<uint8_t> saved_depths = m.ac_depths;
            out = walk(m, order, order_size, direction, min_coeffs_to_change, min_size_delta, prev_size, true);
            st_->ms_walk += ms_since(tw);
            if (out.ambiguous) {
              ++tie_fallbacks_;
              ++tie_why_[out.why];
              unwalk(m, order, out, direction, saved_h, saved_hist_size, saved_depths);
              break;  // take the exact path
            }
            // usable only if the walk stopped strictly inside the fetched prefix
            if (out.stopped && out.consumed < order.size()) {
              ++st_->order_partial;
              done = true;
              break;
            }
            unwalk(m, order, out, direction, saved_h, saved_hist_size, saved_depths);
            want *= 4;
          }
        }
        if (!done) {
          ++st_->order_exact;
          // The reference's own order (:636-678): entries in block-raster / candidate
          // order, std::sort by key.  Only a prefix is consumed, and introsort never lets
          // a sub-range influence anything outside itself, so the replay in exact_sort.h
          // sorts just that prefix (element for element what std::sort would leave there).
          size_t want = direction > 0 ? order_size
                                      : std::max<size_t>(4 * static_cast<size_t>(min_coeffs_to_change) + 1024, 4096);
          // List and large partition passes on the device (order_exact.h); GB200_DEVICE_ORDER=check
          // runs the host replay as well and compares.
          // Default: on for lists of at least a million entries (1080p and larger), where the host
          // replay costs tens of milliseconds; GB200_DEVICE_ORDER=0 turns it off, =1 forces it for
          // every size.
          static const int kDeviceOrder = [] {
            const char* e = getenv("GB200_DEVICE_ORDER");
            return e == nullptr ? 3 : (e[0] == 'c' ? 2 : (e[0] == '1' ? 1 : 0));
          }();
          const bool device_order =
              direction < 0 && (kDeviceOrder == 1 || kDeviceOrder == 2 || (kDeviceOrder == 3 && order_size >= 1000000));
          for (;;) {
            Clock::time_point t0 = Clock::now();
            if (device_order && kDeviceOrder != 2) {
              size_t dev_total = 0;
              if (want > order_size) want = order_size;
              const size_t k_end = ctx_->exact_order_prefix(direction, m.last_indexes, m.max_block_error, want, &order,
                                                            &dev_total);
              if (dev_total != order_size) throw std::runtime_error("exact_order_prefix: entry count mismatch");
              st_->ms_sort += ms_since(t0);
              Clock::time_point tw = Clock::now();
              SymbolHistogram saved_h[3] = {m.ac_h[0], m.ac_h[1], m.ac_h[2]};
              const int saved_hist_size = m.ac_histogram_size;
              const std::vector<uint8_t> saved_depths = m.ac_depths;
              out = walk(m, order, order_size, direction, min_coeffs_to_change, min_size_delta, prev_size, false);
              st_->ms_walk += ms_since(tw);
              if (k_end == order_size || (out.stopped && out.consumed < k_end)) break;
              unwalk(m, order, out, direction, saved_h, saved_hist_size, saved_depths);
              want = std::min(order_size, want * 4);
              continue;
            }
            order.clear();
            order.reserve(order_size);
            for (int block_ix = 0; block_ix < num_blocks; ++block_ix) {
              if (block_weight[block_ix] == 0) continue;
              const int last_index = m.last_indexes[block_ix];
              const int offset = m.offsets[block_ix];
              const int num_candidates = m.offsets[block_ix + 1] - offset;
              const float* candidate_errors = &m.cand_err[offset];
              const float max_err = m.max_block_error[block_ix];
              if (direction > 0) {
                for (int i = last_index; i < num_candidates; ++i) {
                  const float val = (candidate_errors[i] - max_err) / block_weight[block_ix];
                  order.push_back(std::make_pair(block_ix, val));
                }
              } else {
                for (int i = last_index - 1; i >= 0; --i) {
                  const float val = (max_err - candidate_errors[i]) / block_weight[block_ix];
                  order.push_back(std::make_pair(block_ix, val));
                }
              }
            }
            int min_coeffs = min_coeffs_to_change;
            if (first_up_iter) {
              // partition_point of the sorted order (:690-698) == number of keys below the limit
              const float limit = 0.75f * params_.butteraugli_target;
              size_t below = 0;
              for (size_t i = 0; i < order.size(); ++i) below += order[i].second < limit ? 1 : 0;
              min_coeffs = std::max<int>(min_coeffs, static_cast<int>(below));
            }
            if (want > order.size()) want = order.size();
            dbg_ms_[1] += ms_since(t0);
            dbg_n_[0] += order.size();
            const size_t k_end = exact_sort::partial_std_sort(order.data(), order.size(), want);
            order.resize(k_end);
            if (device_order && kDeviceOrder == 2) {
              std::vector<std::pair<int, float> > dev;
              size_t dev_total = 0;
              const size_t dk = ctx_->exact_order_prefix(direction, m.last_indexes, m.max_block_error, want, &dev, &dev_total);
              if (dev_total != order_size || dk != k_end || dev != order)
                throw std::runtime_error("device order replay differs from the host replay");
              ++device_order_checked_;
            }
            st_->ms_sort += ms_since(t0);
            Clock::time_point tw = Clock::now();
            SymbolHistogram saved_h[3] = {m.ac_h[0], m.ac_h[1], m.ac_h[2]};
            const int saved_hist_size = m.ac_histogram_size;
            const std::vector<uint8_t> saved_depths = m.ac_depths;
            out = walk(m, order, order_size, direction, min_coeffs, min_size_delta, prev_size, false);
            st_->ms_walk += ms_since(tw);
            if (k_end == order_size || (out.stopped && out.consumed < k_end)) break;
            unwalk(m, order, out, direction, saved_h, saved_hist_size, saved_depths);
            want = std::min(order_size, want * 4);
          }
        }
        first_up_iter = false;
        last_consumed = out.consumed;
        order.clear();

        if (!device_done) {
          if (!have_weights) throw std::runtime_error("host path without block weights");
          for (int i = 0; i < num_blocks; ++i)
            m.max_block_error[i] += block_weight[i] * out.val_threshold * direction;
          // the device copies of the cursors and max errors follow the host's
          ctx_->walk_upload_state(m.last_indexes, m.max_block_error);
        }
        {
          const size_t per = static_cast<size_t>(img_.nblocks) * 64;
          for (size_t i = 0; i < m.edit_index.size(); ++i)
            if (static_cast<size_t>(m.edit_index[i]) >= per)
              chroma_nz_ += (m.edit_value[i] != 0 ? 1 : 0) - (m.edit_old[i] != 0 ? 1 : 0);
        }

        ++st_->iterations;
        if (direction > 0) ++st_->iterations_up; else ++st_->iterations_down;
        {
          Tick tk(&dt_[7]);
          ctx_->scatter_coeffs(m.edit_index, m.edit_value);
        }
        // GB200_OVERLAP=0 (A/B aid): size pass first, then the whole Compare, nothing queued ahead
        static const bool kOverlap = [] {
          const char* e = getenv("GB200_OVERLAP");
          return !(e != nullptr && e[0] == '0');
        }();
        if (kOverlap) {
          compare_begin();
          // a15 of the next iteration (same direction, radius 1) needs nothing from the host: its
          // kernels go behind the metric's, the sums are picked up at the top of the loop
          ctx_->walk_weights_launch(direction, 1, params_.butteraugli_target * target_mul, false);
          weights_queued_ = true;
          queued_direction_ = direction;
        }
        const size_t encoded = encoded_size(m.ac_h);
        logf("Iter %2d: %s(%d) %s Coeffs[%d/%zd] Blocks[%zd/%d/%d] ValThres[%.4f] Out[%7zd] EstErr[%.2f%%]",
             st_->iterations, "f111111", yuv420_gray_ ? 1 : 7, direction > 0 ? "up" : "down", static_cast<int>(out.consumed),
             order_size, out.changed_blocks, blocks_to_change, num_blocks, out.val_threshold, encoded,
             100.0 - (100.0 * out.est_jpg_size) / encoded);
        if (kOverlap) compare_end(); else compare();
        maybe_output(encoded);
        prev_size = out.est_jpg_size;
      }
    }
    if (getenv("GB200_TIE_DEBUG"))
      fprintf(stderr,
              "device walks %d; ms: exact prefix %.1f, select+sort+fetch %.1f, bulk %.1f, gather %.1f, window walk %.1f, "
              "advance %.1f, weights+stats %.1f, scatter %.1f, mirror sync %.1f; middle lists: %zu entries in all, largest %zu\n",
              device_walks_, dt_[0], dt_[1], dt_[2], dt_[3], dt_[4], dt_[5], dt_[6], dt_[7], dt_[8], dbg_n_[1], dbg_mid_max_);
    if (getenv("GB200_TIE_DEBUG"))
      fprintf(stderr, "tie fallbacks %d: run-at-refresh %d, run-at-test %d, pair-at-refresh %d, pair-untestable %d, pair-decides %d; exact %d partial %d\n",
              tie_fallbacks_, tie_why_[1], tie_why_[2], tie_why_[3], tie_why_[4], tie_why_[5], st_->order_exact,
              st_->order_partial);
    if (getenv("GB200_TIE_DEBUG") && device_order_checked_)
      fprintf(stderr, "device order replay checked against the host replay %d times\n", device_order_checked_);
    if (getenv("GB200_TIE_DEBUG"))
      fprintf(stderr, "order timing: device top-K fetch %.1f ms, exact-order build %.1f ms over %zu entries, sort total %.1f ms, walk %.1f ms\n",
              dbg_ms_[0], dbg_ms_[1], dbg_n_[0], st_->ms_sort, st_->ms_walk);
  }

  SearchParams params_;
  ImageContext* ctx_;
  LogSink log_;
  void* log_user_;
  SearchStats* st_;
  std::string* best_;
  double best_score_;
  float distance_;
  CoeffImage img_;
  std::vector<int16_t> cand_;
  JpegPlan plan_;
  JpegPlan best_plan_;
  size_t best_bytes_ = 0;
  bool have_best_ = false;
  size_t scan_bytes_ = 0;
  std::vector<std::pair<int, float> > order_buf_;
  int device_order_checked_ = 0;
  int device_walks_ = 0;
  double dt_[16] = {0};  // GB200_TIE_DEBUG: wall ms per phase, see the report at the end of select_frequency_masking
  struct Tick {
    double* acc;
    Clock::time_point t0;
    explicit Tick(double* a) : acc(a), t0(Clock::now()) {}
    ~Tick() { *acc += ms_since(t0); }
  };
  bool yuv420_gray_ = false;   // see set_yuv420_gray()
  int sfm_ncomp_ = 3;          // jpg.components.size() in SelectFrequencyMasking (g/processor.cc:583)
  bool device_done_ = false;   // the current iteration took the device path
  bool weights_queued_ = false;  // block weights + order statistics of the next iteration are on the device
  int queued_direction_ = 0;
  std::vector<char> fetched_;  // blocks whose state the host holds for the current iteration
  std::vector<int> fetched_list_;
  bool mirror_valid_ = true;   // cand_ / last_indexes / max_block_error equal the device's
  long long chroma_nz_ = 0;    // nonzero chroma coefficients of the candidate
  int tie_fallbacks_ = 0;
  int tie_why_[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  double dbg_ms_[4] = {0, 0, 0, 0};   // GB200_TIE_DEBUG: device top-K fetch, exact-order build
  size_t dbg_n_[2] = {0, 0};
  size_t dbg_mid_max_ = 0;
  unsigned int sfm_dc_hist_[3][257];
  bool jpeg_source_ = false;
  int q_in_[3][64];
  const JpegFileLayout* layout_ = nullptr;
};

}  // namespace

void device_save_jpeg(ImageContext* ctx, const int q[192], std::string* out) {
  const Geom& g = ctx->geom();
  CoeffImage img;
  img.w = g.w;
  img.h = g.h;
  img.bw = g.bw;
  img.bh = g.bh;
  img.nblocks = g.nblocks;
  img.coeffs = nullptr;  // the coefficients stay on the device
  memcpy(img.q, q, sizeof(img.q));
  ctx->set_quant(q);
  unsigned int hist[6][257];
  bool chroma = false;
  ctx->jpeg_histograms(&hist[0][0], &chroma);
  const int ncomp = chroma ? 3 : 1;  // num_output_components (g/output_image.cc:357)
  SymbolHistogram dc_h[3], ac_h[3];
  uint32_t raw[6][256];
  memset(raw, 0, sizeof(raw));
  for (int c = 0; c < ncomp; ++c)
    for (int i = 0; i < 256; ++i) {
      raw[c][i] = hist[c][i];
      raw[3 + c][i] = hist[3 + c][i];
      dc_h[c].counts[i] = 2 * hist[c][i];
      ac_h[c].counts[i] = 2 * hist[3 + c][i];
    }
  const JpegPlan plan = plan_jpeg(img, ncomp, dc_h, ac_h);
  unsigned long long expected_bits = 0;
  for (int c = 0; c < ncomp; ++c)
    for (int i = 0; i < 256; ++i) {
      expected_bits += static_cast<unsigned long long>(raw[c][i]) * (plan.depth[c][i] + (i & 15));
      expected_bits += static_cast<unsigned long long>(raw[3 + c][i]) * (plan.depth[3 + c][i] + (i & 15));
    }
  size_t nbytes = 0, num_ff = 0;
  ctx->jpeg_encode_scan(ncomp, &plan.depth[0][0], &plan.code[0][0], expected_bits, &nbytes, &num_ff);
  ctx->jpeg_fetch_file(plan.prefix, plan.trailer, out);
  if (out->size() != plan.prefix.size() + nbytes + num_ff + plan.trailer.size())
    throw std::runtime_error("device JPEG size mismatch");
}

// IsGrayscale (g/processor.cc:782): both chroma components of the input are all zero
static bool is_grayscale(ImageContext* ctx) {
  const std::vector<int16_t>& c = ctx->orig_coeffs();
  const size_t per = static_cast<size_t>(ctx->geom().nblocks) * 64;
  for (size_t i = per; i < 3 * per; ++i)
    if (c[i] != 0) return false;
  return true;
}

static bool check_params(const SearchParams& params, std::string* err) {
  if (params.butteraugli_target > 2.0f) {
    *err =
        "Guetzli should be called with quality >= 84, otherwise the\n"
        "output will have noticeable artifacts. If you want to\n"
        "proceed anyway, please edit the source code.\n";
    fputs(err->c_str(), stderr);
    return false;
  }
  return true;
}

// Flat coefficient indices and the candidate-list offsets are 32-bit: refuse larger images up
// front with a clear message instead of overflowing after all device memory is allocated.
// (The scan's 32-bit bit offsets are checked where the scan size is known, jpeg_encode_scan.)
bool image_size_supported(int w, int h, std::string* err) {
  const long long nblocks = static_cast<long long>((w + 7) / 8) * ((h + 7) / 8);
  if (nblocks * 192 >= (1ll << 31)) {
    char buf[160];
    snprintf(buf, sizeof(buf), "guetzli_b200: image too large (%d x %d): at most %lld 8x8 blocks are supported\n", w, h,
             (1ll << 31) / 192 - 1);
    *err = buf;
    fputs(buf, stderr);
    return false;
  }
  return true;
}

namespace {
// What process_jpeg knows about its input beyond the coefficients.
struct JpegSource {
  int q_in[3][64];
  JpegFileLayout layout;
  JpegMeta meta;
};
bool process_resident_impl(const SearchParams& params, ImageContext* ctx, const JpegSource* src, LogSink log,
                           void* log_user, std::string* jpeg_out, SearchStats* stats, std::string* err);
}  // namespace

bool process_resident(const SearchParams& params, ImageContext* ctx, LogSink log, void* log_user,
                      std::string* jpeg_out, SearchStats* stats, std::string* err) {
  return process_resident_impl(params, ctx, nullptr, log, log_user, jpeg_out, stats, err);
}

namespace {
bool process_resident_impl(const SearchParams& params, ImageContext* ctx, const JpegSource* src, LogSink log,
                           void* log_user, std::string* jpeg_out, SearchStats* stats, std::string* err) {
  SearchStats local;
  SearchStats* st = stats ? stats : &local;
  const double setup_ms = st->ms_device_setup;
  *st = SearchStats();
  st->ms_device_setup = setup_ms;
  jpeg_out->clear();
  Clock::time_point t_all = Clock::now();
  if (!check_params(params, err)) return false;
  const long launches0 = total_launches();
  const long long h2d0 = h2d_bytes_total(), d2h0 = d2h_bytes_total();
  ctx->prepare();
  const int w = ctx->width(), h = ctx->height();
  // YUV420 (g/processor.cc:847-877) is not built.  The reference only downsamples when the image is
  // large enough for Butteraugli (:832-838), not grayscale (IsGrayscale :782, OutputImage::Downsample
  // g/output_image.cc:305), and force_420 or try_420 is set.  A tiny image ignores the flags, a
  // grayscale image ignores try_420 and runs force_420 as a one-component pass (set_yuv420_gray).
  const bool gray = (params.force_420 || params.try_420) ? is_grayscale(ctx) : false;
  if (w >= 32 && h >= 32 && (params.force_420 || params.try_420) && !gray) {
    *err = "guetzli_b200: YUV420 is outside the GPU hot path (DESIGN.md)\n";
    fputs(err->c_str(), stderr);
    return false;
  }
  // RGB input: EncodeRGBToJpeg gives the JPEGData the same JFIF APP0 that stripping writes
  // (g/jpeg_data_encoder.cc:53-64,73), so Params::clear_metadata makes no difference there
  const JpegMeta* meta = src ? &src->meta : nullptr;
  if (w < 32 || h < 32) {
    // Butteraugli is skipped for tiny images (g/processor.cc:832-838,940)
    CoeffImage img;
    img.w = w;
    img.h = h;
    img.bw = ctx->geom().bw;
    img.bh = ctx->geom().bh;
    img.nblocks = ctx->geom().nblocks;
    img.coeffs = ctx->orig_coeffs().data();
    for (int c = 0; c < 3; ++c)
      for (int k = 0; k < 64; ++k) img.q[c][k] = src ? src->q_in[c][k] : 1;
    img.as_encoded = src == nullptr;
    img.as_read = src ? &src->layout : nullptr;
    img.meta = meta;
    *jpeg_out = write_jpeg(img);
    if (log) {
      char buf[128];
      snprintf(buf, sizeof(buf), "Original Out[%7zd] <image too small for Butteraugli>\n", jpeg_out->size());
      log(log_user, buf);
    }
  } else {
    Search search(params, ctx, log, log_user, st);
    if (params.force_420 && gray) search.set_yuv420_gray();
    if (src) {
      search.set_jpeg_source(src->q_in, &src->layout, meta);
    } else {
      search.set_meta(meta);
    }
    search.run(jpeg_out);
  }
  st->gpu_launches = total_launches() - launches0;
  st->h2d_bytes = h2d_bytes_total() - h2d0;
  st->d2h_bytes = d2h_bytes_total() - d2h0;
  st->ms_total = ms_since(t_all);
  return true;
}
}  // namespace

// Process(jpeg bytes), g/processor.cc:890-924.
bool process_jpeg(const SearchParams& params, const uint8_t* data, size_t len, int device, LogSink log,
                  void* log_user, std::string* jpeg_out, SearchStats* stats, std::string* err) {
  SearchStats local;
  SearchStats* st = stats ? stats : &local;
  *st = SearchStats();
  jpeg_out->clear();
  auto fail = [err](const char* msg) {
    *err = msg;
    fputs(msg, stderr);
    return false;
  };
  JpegInput jpg;
  std::string why;
  if (data == nullptr || !read_jpeg(data, len, &jpg, &why)) return fail("Can't read jpg data from input file\n");
  if (!check_jpeg_sanity(jpg)) return fail("Unsupported input JPEG (unexpectedly large coefficient values).\n");
  const size_t ncomp = jpg.components.size();
  const bool decodable = ncomp == 1 || (ncomp == 3 && has_ycbcr_color_space(jpg) && (jpg.is_420() || jpg.is_444()));
  if (!decodable)
    return fail(
        "Unsupported input JPEG file (e.g. unsupported downsampling mode).\nPlease provide the input image as a PNG "
        "file.\n");
  if (!check_params(params, err)) return false;
  if (ncomp != 3 || !has_ycbcr_color_space(jpg)) return fail("Only YUV color space input jpeg is supported\n");
  if (!jpg.is_444())
    return fail("guetzli_b200: YUV420 JPEG input is outside the GPU hot path (DESIGN.md); provide 4:4:4 or PNG\n");

  if (!image_size_supported(jpg.width, jpg.height, err)) return false;
  Clock::time_point t0 = Clock::now();
  const long long h2d0 = h2d_bytes_total();
  JpegSource src;
  const int w = jpg.width, h = jpg.height;
  const int nblocks = jpg.components[0].width_in_blocks * jpg.components[0].height_in_blocks;
  // RemoveOriginalQuantization (g/processor.cc:82): coefficients times their quant step
  std::vector<int16_t> dq(static_cast<size_t>(3) * nblocks * 64);
  for (int c = 0; c < 3; ++c) {
    const JpegComponent& comp = jpg.components[c];
    const int* q = jpg.quant[comp.quant_idx].values;
    memcpy(src.q_in[c], q, sizeof(src.q_in[c]));
    int16_t* dst = &dq[static_cast<size_t>(c) * nblocks * 64];
    for (size_t i = 0; i < comp.coeffs.size(); ++i) dst[i] = static_cast<int16_t>(comp.coeffs[i] * q[i & 63]);
    src.layout.comp_id[c] = comp.id;
    src.layout.comp_table[c] = comp.quant_idx;
  }
  src.layout.num_tables = static_cast<int>(jpg.quant.size());
  for (int i = 0; i < src.layout.num_tables; ++i) {
    memcpy(src.layout.table[i], jpg.quant[i].values, sizeof(src.layout.table[i]));
    src.layout.precision[i] = jpg.quant[i].precision;
    src.layout.index[i] = jpg.quant[i].index;
  }
  src.meta.strip = params.clear_metadata;
  src.meta.app_data = jpg.app_data;
  src.meta.com_data = jpg.com_data;
  src.meta.tail_data = jpg.tail_data;
  ImageContext ctx(dq.data(), w, h, device, false, nullptr);
  st->ms_device_setup = ms_since(t0);
  const bool ok = process_resident_impl(params, &ctx, &src, log, log_user, jpeg_out, st, err);
  st->h2d_bytes = h2d_bytes_total() - h2d0;
  st->ms_total = ms_since(t0);
  return ok;
}

bool process_rgb(const SearchParams& params, const uint8_t* rgb, int w, int h, int device, LogSink log,
                 void* log_user, std::string* jpeg_out, SearchStats* stats, std::string* err) {
  return process_rgb_tiled(params, rgb, w, h, device, nullptr, log, log_user, jpeg_out, stats, err);
}

bool process_rgb_tiled(const SearchParams& params, const uint8_t* rgb, int w, int h, int device, Comm* comm,
                       LogSink log, void* log_user, std::string* jpeg_out, SearchStats* stats, std::string* err) {
  SearchStats local;
  SearchStats* st = stats ? stats : &local;
  *st = SearchStats();
  jpeg_out->clear();
  if (rgb == nullptr || w < 0 || w >= 1 << 16 || h < 0 || h >= 1 << 16) {
    *err = "Could not create jpg data from rgb pixels\n";
    fputs(err->c_str(), stderr);
    return false;
  }
  if (!check_params(params, err)) return false;
  if (w == 0 || h == 0) {
    *err = "guetzli_b200: empty image\n";
    fputs(err->c_str(), stderr);
    return false;
  }
  if (!image_size_supported(w, h, err)) return false;
  Clock::time_point t0 = Clock::now();
  const long long h2d0 = h2d_bytes_total();
  ImageContext ctx(rgb, w, h, device, false, comm);
  st->ms_device_setup = ms_since(t0);
  const bool ok = process_resident(params, &ctx, log, log_user, jpeg_out, st, err);
  st->h2d_bytes = h2d_bytes_total() - h2d0;
  st->ms_total = ms_since(t0);
  return ok;
}

bool image_view(const uint8_t* img, int w, int channels, const int64_t* strides, ImageView* view, std::string* err) {
  char buf[192];
  if (channels < 1 || channels > 4) {
    snprintf(buf, sizeof(buf),
             "guetzli_b200: an image has 1 (gray), 2 (gray + alpha), 3 (RGB) or 4 (RGBA) channels, got %d\n",
             channels);
    *err = buf;
    fputs(buf, stderr);
    return false;
  }
  if (strides != nullptr && (strides[0] < 0 || strides[1] < 0 || strides[2] < 0)) {
    snprintf(buf, sizeof(buf), "guetzli_b200: image strides must not be negative, got row %lld, pixel %lld, channel %lld\n",
             static_cast<long long>(strides[0]), static_cast<long long>(strides[1]), static_cast<long long>(strides[2]));
    *err = buf;
    fputs(buf, stderr);
    return false;
  }
  view->data = img;
  view->channels = channels;
  view->stride[0] = strides ? strides[0] : static_cast<int64_t>(w) * channels;
  view->stride[1] = strides ? strides[1] : channels;
  view->stride[2] = strides ? strides[2] : 1;
  return true;
}

namespace {
// process_rgb_tiled's checks, messages and accounting (one GPU) on an image view
bool process_view(const SearchParams& params, const uint8_t* img, int w, int h, int channels, const int64_t* strides,
                  int device, bool on_device, Stream stream, LogSink log, void* log_user, std::string* jpeg_out,
                  SearchStats* stats, std::string* err) {
  SearchStats local;
  SearchStats* st = stats ? stats : &local;
  *st = SearchStats();
  jpeg_out->clear();
  if (img == nullptr || w < 0 || w >= 1 << 16 || h < 0 || h >= 1 << 16) {
    *err = "Could not create jpg data from rgb pixels\n";
    fputs(err->c_str(), stderr);
    return false;
  }
  ImageView view;
  if (!image_view(img, w, channels, strides, &view, err)) return false;
  view.device = on_device;
  view.stream = stream;
  if (!check_params(params, err)) return false;
  if (w == 0 || h == 0) {
    *err = "guetzli_b200: empty image\n";
    fputs(err->c_str(), stderr);
    return false;
  }
  if (!image_size_supported(w, h, err)) return false;
  Clock::time_point t0 = Clock::now();
  const long long h2d0 = h2d_bytes_total();
  ImageContext ctx(view, w, h, device, false);
  st->ms_device_setup = ms_since(t0);
  const bool ok = process_resident(params, &ctx, log, log_user, jpeg_out, st, err);
  st->h2d_bytes = h2d_bytes_total() - h2d0;
  st->ms_total = ms_since(t0);
  return ok;
}
}  // namespace

bool process_image(const SearchParams& params, const uint8_t* img, int w, int h, int channels, const int64_t* strides,
                   int device, LogSink log, void* log_user, std::string* jpeg_out, SearchStats* stats,
                   std::string* err) {
  return process_view(params, img, w, h, channels, strides, device, false, 0, log, log_user, jpeg_out, stats, err);
}

bool process_image_device(const SearchParams& params, const uint8_t* img, int w, int h, int channels,
                          const int64_t* strides, int device, Stream stream, LogSink log, void* log_user,
                          std::string* jpeg_out, SearchStats* stats, std::string* err) {
  return process_view(params, img, w, h, channels, strides, device, true, stream, log, log_user, jpeg_out, stats, err);
}

}  // namespace gb200
