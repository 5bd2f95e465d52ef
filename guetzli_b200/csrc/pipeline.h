// The encoder's device-resident state of one image and its kernel sequences: coefficients, render,
// zeroing orders, the device half of the selection walk, the order replay and the JPEG pass.  The
// metric that scores the candidate is a Butteraugli (butteraugli.h) held by the context.  One
// ImageContext = one image on one GPU, driven by one host thread on one stream, the metric's.
// See DESIGN.md for the HBM layout and the kernel list.
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

#include "butteraugli.h"

namespace gb200 {

struct OrderItem;
struct OrderSelectState;
struct JpegInput;

// libjpeg-turbo's pixels of n parsed files that libjpeg_decodable (jpeg_in.h) accepted, decoded on `device`
// with one launch of JpegIdctIslow and one of JpegUpsampleYccRgb (kernels.h) for all of them: out[i]
// receives file i as [h][w][3] bytes.  The coefficients of all files go up in one staging buffer, beside
// one per-file table.  Host outputs come back per file; with out_on_device, out[i] is memory of `device`,
// written after the work queued on `stream` so far.  Either way the outputs are written when this returns.
void jpeg_decode_rgb(const JpegInput* const* files, int n, int device, uint8_t* const* out, bool out_on_device,
                     Stream stream);

// An 8-bit image of 1 (gray), 2 (gray + alpha), 3 (RGB) or 4 (RGBA) channels in any layout with
// non-negative strides: sample (y, x, c) is at byte y * stride[0] + x * stride[1] + c * stride[2] of data.
struct ImageView {
  const uint8_t* data = nullptr;
  int channels = 3;
  int64_t stride[3] = {0, 0, 0};  // bytes: row, pixel, channel
  // data is memory of the context's device, read in place once the work queued on `stream` so far is
  // done; otherwise host memory
  bool device = false;
  Stream stream = 0;
  // bytes from data to the last sample of a w x h image, inclusive: the span a host view uploads
  size_t span(int w, int h) const {
    return static_cast<size_t>((h - 1) * stride[0] + (w - 1) * stride[1] + (channels - 1) * stride[2] + 1);
  }
};

class ImageContext {
 public:
  // Uploads the image, runs the one-time kernels (a2 FDCT, a3 PsychoImage of the
  // original, a13 block-corner masks).  rgb: interleaved sRGB u8, w*h*3.
  // comm != nullptr: row-strip mode, this context computes block rows strip_of(rank)
  // of the image-plane work and all-gathers the per-block results (comm.h).
  ImageContext(const uint8_t* rgb, int w, int h, int device, bool prepare_now = true, Comm* comm = nullptr);
  // JPEG input (4:4:4): the original is given as dequantised DCT coefficients
  // [3][nblocks][64]; its pixels (DecodeJpegToRGB) are rendered on the device.
  ImageContext(const int16_t* dq_coeffs, int w, int h, int device, bool prepare_now, Comm* comm);
  // An 8-bit view (ImageView) turned into the packed RGB of the first constructor on the device, as the
  // guetzli tool turns PNG layouts into RGB (IngestU8, kernels.h); everything after that is the RGB path.
  // A device view is read in place after the work queued on its stream; a host view's span is uploaded
  // into a staging buffer.  Either way the view has been read when the constructor returns.
  ImageContext(const ImageView& view, int w, int h, int device, bool prepare_now);
  // EXPERIMENTAL (order_exact.h, GB200_DEVICE_ORDER=1): the reference-ordered candidate list
  // and the introsort partition passes over large ranges on the device.  Returns k_end and the
  // first k_end entries exactly as std::sort would leave them (exact_sort.h semantics).
  size_t exact_order_prefix(int direction, const std::vector<int>& last_index, const std::vector<float>& max_err,
                            size_t want, std::vector<std::pair<int, float> >* out, size_t* order_size);
  // the same on the resident cursors / max errors (device half of the walk, walk_dev.h)
  size_t exact_order_prefix_resident(int direction, size_t want, std::vector<std::pair<int, float> >* out,
                                     size_t* order_size);
  // test hook: the same replay on caller-provided items
  size_t debug_device_partial_sort(std::pair<int, float>* items, size_t n, size_t want);
  // the one-time kernels (idempotent); split from the upload so that a caller can
  // time the job with the image already resident in HBM
  void prepare();
  // forgets the one-time results so that the next prepare() recomputes them (a resident
  // image encoded again must redo all of its work, bench.py)
  void reset_prepared() { prepared_ = false; }
  // sRGB bytes of the original as the metric sees it (tests)
  void download_rgb(uint8_t* rgb);
  // makes this context's device current for the calling host thread
  void bind() { ba_.bind(); }
  ~ImageContext();

  int width() const { return g_.w; }
  int height() const { return g_.h; }
  const Geom& geom() const { return g_; }

  // a2 result on the host: [3][nblocks][64] int16 (q = 1 coefficients).
  const std::vector<int16_t>& orig_coeffs() const { return orig_host_; }

  // a8: candidate := Quantize(original, q) for all coefficients. q: [3][64].
  void apply_global_quant(const int q[192]);
  void set_quant(const int q[192]);  // tables only (the candidate is given, upload_candidate)
  // Sparse edits of the candidate: flat indices into [3][nblocks][64].
  void scatter_coeffs(const std::vector<int>& index, const std::vector<int16_t>& value);
  // Whole candidate from the host (tests).
  void upload_candidate(const int16_t* coeffs);
  void download_candidate(int16_t* coeffs);

  // a7+a9+a10: renders the candidate and scores it against the original.
  // Leaves the distmap and per-block maxima on the device; returns distance_.
  float compare() {
    compare_render();
    return ba_.compare();
  }
  // the same in two halves: compare_begin() queues the kernels, compare_end() waits for the
  // distance; stream work queued in between runs behind the metric's kernels (where the
  // launches need a host round trip -- strip mode, the staged chain -- compare_begin() does it all)
  void compare_begin() {
    compare_render();
    ba_.compare_begin();
  }
  float compare_end() { return ba_.compare_end(); }
  void download_distmap(float* out) { ba_.download_distmap(out); }  // [h][w] packed
  void download_block_max(float* out) { d2h(out, ba_.block_max(), sizeof(float) * g_.nblocks, s_); }  // [nblocks]

  // a15: block weights for the current distmap (or an all-zero distmap when
  // zero_distmap is set, the reference's first "up" iteration).
  void block_weights(int direction, int radius, double target_distance, bool zero_distmap,
                     float* out);

  // a13+a14: greedy zeroing order of every block of the current candidate.
  // idx/err are [nblocks][192] slots, count[nblocks] valid entries each.
  // idx / err may be null: the lists then stay on the device (download_zeroing_err later)
  void zeroing_orders(float block_error_limit, int lookahead, bool new_model, std::vector<uint8_t>* idx,
                      std::vector<float>* err, std::vector<int>* count);
  void download_zeroing_err(std::vector<float>* err);

  // a16: the entries of the walk order whose keys are among (at least) the k
  // smallest, unsorted.  Needs zeroing_orders() and the weights of the latest
  // block_weights() call on the device.  Returns the total number of entries.
  size_t order_smallest(int direction, const std::vector<int>& last_index, const std::vector<float>& max_err,
                        size_t k, std::vector<float>* val, std::vector<int>* block);

  // ---- device-resident half of the selection walk (walk_dev.h) -----------------------
  // Candidate cursors (last_index) and max_block_error live on the device between
  // iterations; the host mirrors are refreshed only when an iteration takes the host path.
  void walk_begin();
  void walk_upload_state(const std::vector<int>& last_index, const std::vector<float>& max_err);
  void walk_download_state(std::vector<int>* last_index, std::vector<float>* max_err);
  // a15 without the download, plus the size of the order the weights imply
  void walk_weights(int direction, int radius, double target_distance, bool zero_distmap,
                    unsigned long long* order_size, unsigned long long* blocks_to_change);
  void walk_weights_launch(int direction, int radius, double target_distance, bool zero_distmap);
  void walk_weights_fetch(unsigned long long* order_size, unsigned long long* blocks_to_change);
  void download_weights(float* out);
  // nonzero coefficients of the candidate's two chroma components
  size_t count_nonzero_chroma();
  // entries of the order whose key is below `limit`
  size_t walk_count_below(int direction, float limit);
  // at least the `want` smallest keys of the order, sorted ascending, resident; -> how many
  size_t walk_select_sorted(int direction, size_t want, size_t* total);
  // Two-rank select: entries certainly among the first `rank_lo` are counted into the pending
  // bulk right away, the entries between the two ranks (the "middle") are left sorted in the
  // resident selection.  *before = entries already counted, -> size of the middle.
  size_t walk_select_split(int direction, size_t rank_lo, size_t rank_hi, size_t* before, size_t* total);
  static size_t walk_middle_max() { return 65536; }  // larger middles come back unsorted: cancel them
  void walk_split_cancel();
  void walk_fetch_sorted(size_t first, size_t n, float* val, int* block);
  void walk_fetch_pairs(size_t n, std::pair<int, float>* out);
  struct BulkResult {
    int touched, logged, chroma_delta;
    int delta_hist[3][256];
  };
  // consumes entries [0, nbulk) of the sorted selection on the device; host_blocks != nullptr:
  // the entries' blocks come from the host instead (prefix of the reference-ordered sort)
  // after_split: the counts of walk_select_split are pending and are consumed as well
  // gather_n > 0: the state of the blocks of selection entries [gather_first, gather_first + gather_n)
  // is gathered right behind the bulk's kernels (walk_gather_selection_fetch picks it up)
  void walk_bulk_apply(int direction, size_t nbulk, BulkResult* r, const int* host_blocks = nullptr,
                       bool after_split = false, size_t gather_first = 0, size_t gather_n = 0);
  // per entry of that range (a block may repeat): [n][3][64] coefficients, cursor, "touched by the bulk"
  void walk_gather_selection_fetch(size_t n, std::vector<int16_t>* coeffs, std::vector<int>* cursor,
                                   std::vector<int>* in_bulk);
  void walk_bulk_undo(int direction);
  void walk_gather(const std::vector<int>& blocks, std::vector<int16_t>* coeffs, std::vector<int>* cursor,
                   std::vector<int>* in_bulk);
  void walk_advance(const std::vector<int>& blocks, int direction);
  void walk_add_max_err(float val_threshold, int direction);

  // a11 on the device.  Symbol histograms of the candidate (raw counts):
  // hist[6][257] = dc0 dc1 dc2 ac0 ac1 ac2; *chroma_nonzero tells whether the
  // saved JPEG has 3 components (g/output_image.cc:357).
  void jpeg_histograms(unsigned int* hist, bool* chroma_nonzero);
  // Entropy-codes the scan with the given canonical codes (depth/code [6][256]).
  // Returns the number of scan bytes before 0xFF stuffing and the number of 0xFF
  // bytes among them; the bytes stay on the device until jpeg_fetch_file().
  // expected_bits: length of the scan as the caller's symbol counts give it (sum over the symbols of
  // count x (code length + extra bits)); sizes the buffers without a round trip and is checked
  // against the device's own total
  void jpeg_encode_scan(int ncomp, const uint8_t* depth, const uint16_t* code, unsigned long long expected_bits,
                        size_t* nbytes, size_t* num_ff);
  // keeps a device-side copy of the scan just encoded (the best output so far); the bytes
  // cross PCIe once, when the search is over
  void jpeg_keep_scan();
  // f1: the whole file = prefix | scan with a zero byte after every 0xFF | trailer, assembled on
  // the device from the current / the kept scan (jpeg_dev.h), one copy back
  void jpeg_fetch_file(const std::string& prefix, const std::string& trailer, std::string* file);
  void jpeg_fetch_kept_file(const std::string& prefix, const std::string& trailer, std::string* file);

  // test hooks: run single stages on caller-provided planes (packed [n][h][w]).
  void debug_blur(const float* in, float* out, int id) { ba_.debug_blur(in, out, id); }
  void debug_opsin(const float* rgb_lin, float* xyb) {
    render_all_ = true;  // the planes it overwrites are the render target
    ba_.debug_opsin(rgb_lin, xyb);
  }
  void debug_separate(const float* xyb, float* ps10) { ba_.debug_separate(xyb, ps10); }
  void debug_render(float* lin3);
  void debug_psycho0(float* ps10) { ba_.debug_psycho0(ps10); }
  void debug_corner_mask(float* out);  // [nblocks][3]

  long launches() const;
  void set_profiling(bool on);
  std::vector<KernelStat> kernel_stats() const;
  void reset_stats();
  Stream stream() const { return s_; }

 private:
  Butteraugli ba_;  // the metric; it owns the stream and the tables that the encoder's kernels use too
  const Region& r_ = ba_.region();
  const Geom& g_ = r_.g;
  const Stream s_ = r_.s;
  const Tables& t_ = ba_.tables();

  // device-resident walk state (walk_dev.h)
  unsigned int* w_cnt_ = nullptr;       // [nblocks]
  int* w_done_ = nullptr;               // [nblocks]
  int* w_stamp_ = nullptr;              // [nblocks]
  int* w_touched_ = nullptr;            // [nblocks]
  unsigned int* w_counters_ = nullptr;  // n_touched, n_log, chroma delta, pad, delta_hist[768]
  unsigned long long* w_stats_ = nullptr;  // [1024][2]
  int* w_log_index_ = nullptr;
  int16_t* w_log_old_ = nullptr;
  size_t w_log_cap_ = 0;
  int* w_gblocks_ = nullptr;
  int16_t* w_gcoeffs_ = nullptr;
  std::vector<char> gather_host_;
  void* d_sel_pairs_ = nullptr;  // the sorted selection as std::pair<int, float> (block, key)
  size_t pairs_cap_ = 0;
  size_t w_gcap_ = 0;
  int* w_ablocks_ = nullptr;
  size_t w_acap_ = 0;
  float* d_sel_val2_ = nullptr;
  int* d_sel_block2_ = nullptr;
  size_t sel2_cap_ = 0;
  size_t sel_sorted_ = 0;    // entries of the sorted resident selection
  unsigned int* w_keys_ = nullptr;  // order-preserving integer images of all order keys (two-rank select)
  size_t keys_cap_ = 0;
  unsigned int* w_sel2_ = nullptr;  // two-rank select: level-1 histogram pair + Select2State
  bool split_pending_ = false;      // walk_select_split has counted entries that no bulk has consumed yet
  size_t pending_bulk_extra_ = 0;   // ... how many
  int w_iter_ = 0;
  int w_last_touched_ = 0, w_last_logged_ = 0;
  int pending_touched_ = 0;  // blocks the last bulk changed and compare() has not rendered yet
  void select_keys(int direction, size_t k, OrderSelectState* got);
  void sort_selection(size_t n);
#if defined(__CUDACC__)
  int2* sel_pairs(size_t n);
#endif
  bool metric_;  // the image is large enough for the reference to run Butteraugli on it
  bool prepared_;
  std::vector<void*> owned_;
  void* own(size_t bytes) {  // device memory freed with the context
    owned_.push_back(dev_alloc(bytes));
    return owned_.back();
  }
  std::vector<int16_t> orig_host_;

  uint8_t* d_rgb_ = nullptr;
  int16_t* d_orig_ = nullptr;
  int16_t* d_cand_ = nullptr;
  int* d_q_ = nullptr;
  float* corner_mask_ = nullptr;  // [nblocks][3]
  // scratch of the device order replay (allocated on first use)
  OrderItem* x_items_ = nullptr;
  unsigned int* x_u32_ = nullptr;  // fl, sl, fr, sr
  int* x_i32_ = nullptr;           // llist, rlist
  unsigned int* x_small_ = nullptr;
  size_t x_cap_ = 0;
  void order_scratch(size_t n);
  size_t device_partial_sort_resident(size_t n, size_t want, std::vector<std::pair<int, float> >* out);
  void compare_render();
  std::vector<int> advance_host_;  // source of walk_advance's upload
  void gather_reserve(size_t n);
  void gather_fetch(size_t n, std::vector<int16_t>* coeffs, std::vector<int>* cursor, std::vector<int>* in_bulk);
  bool from_coeffs_ = false;  // original given as coefficients (JPEG input)
  void guarded_init(const uint8_t* rgb, const int16_t* dq_coeffs, bool prepare_now, const ImageView* view = nullptr);
  void init(const uint8_t* rgb, const int16_t* dq_coeffs, bool prepare_now, const ImageView* view);
  void ingest(const ImageView& view);
  void release();
  float* weights_ = nullptr;    // [nblocks]
  float* zero_block_max_ = nullptr;
  uint8_t* z_idx_ = nullptr;   // [nblocks][192] candidate coefficient index
  float* z_err_ = nullptr;     // [nblocks][192] candidate block error
  int* z_cnt_ = nullptr;       // [nblocks]
  int* d_last_index_ = nullptr;
  float* d_max_err_ = nullptr;
  unsigned int* d_hist_ = nullptr;  // [65536] + 1 counter
  float* d_sel_val_ = nullptr;
  int* d_sel_block_ = nullptr;
  size_t sel_cap_ = 0;
  int* e_block_ = nullptr;      // [entries] block of every candidate (compact list)
  uint8_t* e_slot_ = nullptr;   // [entries] its slot
  size_t num_entries_ = 0;
  size_t e_cap_ = 0;
  unsigned int* e_offset_ = nullptr;  // [nblocks] exclusive scan of z_cnt_
  int* d_edit_i_ = nullptr;
  int16_t* d_edit_v_ = nullptr;
  size_t edit_cap_ = 0;
  bool render_all_;
  int num_dirty_;
  int* d_dirty_ = nullptr;
  std::vector<char> dirty_flag_;
  std::vector<int> dirty_list_;
  unsigned int* j_hist_ = nullptr;      // [kHistCopies][6][257] + [6][257] + flag + ff counter
  unsigned int* j_bits_ = nullptr;      // [3*nblocks] unit bit lengths (scan order)
  unsigned int* j_offset_ = nullptr;    // [3*nblocks] exclusive scan
  unsigned int* j_sums_ = nullptr;      // scan scratch
  uint8_t* j_file_ = nullptr;           // the assembled file (jpeg_fetch_file)
  size_t j_file_cap_ = 0;
  unsigned int* j_file_scratch_ = nullptr;
  size_t j_file_scratch_cap_ = 0;
  uint8_t* j_depth_ = nullptr;          // [6][256]
  uint16_t* j_code_ = nullptr;          // [6][256]
  unsigned int* j_words_ = nullptr;     // scan bits, big-endian 32-bit words
  size_t j_words_cap_ = 0;
  size_t j_nbytes_ = 0;
  unsigned int* j_best_words_ = nullptr;
  size_t j_best_cap_ = 0;
  size_t j_best_nbytes_ = 0;
  void exclusive_scan(const unsigned int* in, unsigned int* out, int n, unsigned long long* total);
  void exclusive_scan_to(const unsigned int* in, unsigned int* out, int n, unsigned long long* d_total);
  // same with caller-provided scratch for the per-CTA sums (n / 1024 + 8 words)
  void exclusive_scan_with(const unsigned int* in, unsigned int* out, int n, unsigned long long* total,
                           unsigned int* scratch);
};

}  // namespace gb200
