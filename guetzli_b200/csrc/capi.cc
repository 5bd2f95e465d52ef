// C ABI (include/guetzli_b200.h) over the C++ implementation.
#include "guetzli_b200.h"

#include <stdlib.h>
#include <string.h>

#include <exception>
#include <memory>
#include <stdexcept>
#include <thread>
#include <string>
#include <vector>

#include <algorithm>

#include "comm.h"
#include "exact_sort.h"
#include "jpeg_out.h"
#include "pipeline.h"
#include "jpeg_in.h"
#include "search.h"
#include "tables.h"

namespace gb200 {
struct ThreadGroup;
ThreadGroup* thread_group_create(int world);
void thread_group_destroy(ThreadGroup* g);
void thread_group_abort(ThreadGroup* g);
Comm* thread_comm_create(ThreadGroup* g, int rank);
#if !defined(GB200_HOSTSIM)
void nccl_unique_id(uint8_t out[128]);
Comm* nccl_comm_create(const uint8_t id[128], int rank, int world);
void dev_trim();
int cuda_device_count();
#endif
}  // namespace gb200

namespace {
thread_local std::string g_err;

template <class F>
int guarded(F f) {
  try {
    f();
    return 1;
  } catch (const std::exception& e) {
    g_err = e.what();
  } catch (...) {
    g_err = "unknown error";
  }
  return 0;
}
}  // namespace

struct gb200_image {
  gb200::ImageContext* ctx;
};

struct gb200_butteraugli_comparator {
  gb200::Butteraugli* ba;
  // made from 8-bit images: their channels (3 or 4), and for RGBA the original laid over white (ba
  // holds it laid over black); 0 and null when made from float planes
  int channels = 0;
  gb200::Butteraugli* white = nullptr;
};

struct gb200_butteraugli_batch {
  gb200::Butteraugli* ba;
};

struct gb200_butteraugli_comparator_set {
  gb200::ComparatorSet* set;
};

namespace {
// A comparator (or set) made from float planes takes float images, one made from 8-bit images 8-bit images.
bool made_takes(const char* who, bool made_srgb, bool srgb) {
  if (made_srgb == srgb) return true;
  g_err = std::string(who) + (srgb ? ": made from float planes, it takes float images, not 8-bit ones"
                                   : ": made from 8-bit images, it takes 8-bit images, not float planes");
  return false;
}
bool comparator_takes(const gb200_butteraugli_comparator* c, bool srgb) {
  return made_takes("butteraugli comparator", c->channels != 0, srgb);
}

// device pointers of a *_device entry: memory of `device`, else a message naming the argument
void check_device_pointers(const char* who, int device, const void* const* ptrs, const char* const* what, int n) {
  for (int i = 0; i < n; ++i) {
    if (ptrs[i] == nullptr) continue;
    const int dev = gb200::pointer_device(ptrs[i]);
    if (dev != device)
      throw std::runtime_error(std::string(who) + ": " + what[i] + " is not device memory of device " +
                               std::to_string(device) +
                               (dev < 0 ? " (host or unknown memory)" : " (device " + std::to_string(dev) + ")"));
  }
}

// the same for the per-pair pointers of a mixed-size call, named rgb0[i], diffmap[i], ... (im0 null: a
// comparator set's call, whose originals are its own)
template <class T>
void check_pair_pointers(const gb200::Butteraugli& ba, const char* name0, const char* name1, const T* const* im0,
                         const T* const* im1, float* const* diffmap, int n, const char* who = "butteraugli batch") {
  for (int i = 0; i < n; ++i) {
    const void* ptrs[3] = {im0 != nullptr ? im0[i] : nullptr, im1[i], diffmap != nullptr ? diffmap[i] : nullptr};
    const std::string k = "[" + std::to_string(i) + "]";
    const std::string names[3] = {name0 + k, name1 + k, "diffmap" + k};
    const char* what[3] = {names[0].c_str(), names[1].c_str(), names[2].c_str()};
    check_device_pointers(who, ba.device(), ptrs, what, 3);
  }
}

// the caller's stream of a *_device entry (the host entries pass null and read no stream)
gb200::Stream caller_stream(void* stream) {
#if defined(GB200_HOSTSIM)
  (void)stream;  // the port has no device memory: its device entries refuse before they need a stream
  return 0;
#else
  return static_cast<gb200::Stream>(stream);
#endif
}

// sizes a metric is made for: the reference computes nothing below 8 pixels in a dimension
// (b/butteraugli.cc:788), and the batched Compare chain folds the image into blockIdx.z, four z per
// image in its widest launch
bool create_size_ok(int w, int h) { return w >= 8 && h >= 8 && w < 65536 && h < 65536; }
void check_capacity(const char* who, int capacity) {
  if (capacity < 1 || capacity > 16383) throw std::runtime_error(std::string(who) + ": the capacity must be in 1..16383");
}
void check_create(const char* who, const char* images, int w, int h, int capacity) {
  if (!create_size_ok(w, h))
    throw std::runtime_error(std::string(who) + ": the " + images + " must be at least 8x8 (and below 65536)");
  check_capacity(who, capacity);
}

// n of a batched call: `kind` is "batch" or "comparator", `items` "pairs" or "images"
bool n_ok(const char* kind, const char* items, int n, const gb200::Butteraugli& ba) {
  if (n >= 1 && n <= ba.capacity()) return true;
  g_err = std::string("butteraugli ") + kind + ": n = " + std::to_string(n) + " " + items + ", the " + kind +
          " takes 1.." + std::to_string(ba.capacity());
  return false;
}

// pair i of a mixed-size call: 8x8 up to the batch's size
bool pair_size_ok(const gb200::Butteraugli& ba, int i, int w, int h) {
  const int bw = ba.region().g.w, bh = ba.region().g.h;
  if (w >= 8 && h >= 8 && w <= bw && h <= bh) return true;
  g_err = "butteraugli batch: pair " + std::to_string(i) + " is " + std::to_string(w) + "x" + std::to_string(h) +
          ", the batch takes 8x8 up to " + std::to_string(bw) + "x" + std::to_string(bh);
  return false;
}

// a batched call: run(maxima) on ba's device, then the n maxima into score (if not null)
template <class Run>
int scored(gb200::Butteraugli* ba, int n, double* score, const Run& run) {
  return guarded([&]() {
    ba->bind();
    std::vector<float> m(n);
    run(m.data());
    if (score)
      for (int i = 0; i < n; ++i) score[i] = m[i];
  });
}

// Images below 8 pixels in a dimension are edge-replicated to 8 (b/butteraugli.cc:1825-1853), scored,
// and their diffmaps cropped back.  An image is `planes` planes of `per` elements per pixel: planar
// float RGB is 3 planes of 1, interleaved 8-bit RGB(A) 1 plane of 3 or 4.
struct Pad8 {
  int w, h, ws, hs, xb, yb;
  Pad8(int w_, int h_)
      : w(w_), h(h_), ws(std::max(w_, 8)), hs(std::max(h_, 8)), xb(w_ < 8 ? (8 - w_) / 2 : 0),
        yb(h_ < 8 ? (8 - h_) / 2 : 0) {}
  bool padded() const { return ws != w || hs != h; }
  // img padded into *buf, or img itself where no padding is needed
  template <class T>
  const T* pad(const T* img, int planes, int per, std::vector<T>* buf) const {
    if (!padded()) return img;
    buf->resize(static_cast<size_t>(planes) * ws * hs * per);
    for (int c = 0; c < planes; ++c)
      for (int y = 0; y < hs; ++y)
        for (int x = 0; x < ws; ++x) {
          const int x2 = std::min(w - 1, std::max(0, x - xb)), y2 = std::min(h - 1, std::max(0, y - yb));
          const size_t d = ((static_cast<size_t>(c) * hs + y) * ws + x) * per,
                       s = ((static_cast<size_t>(c) * h + y2) * w + x2) * per;
          memcpy(&(*buf)[d], img + s, sizeof(T) * per);
        }
    return buf->data();
  }
  // the image's w x h rows of a padded [hs][ws] diffmap -> out [h][w]
  void crop(const float* dm, float* out) const {
    for (int y = 0; y < h; ++y)
      memcpy(out + static_cast<size_t>(y) * w, dm + static_cast<size_t>(y + yb) * ws + xb, sizeof(float) * w);
  }
  float cropped_max(const float* dm) const {
    float m = 0.0f;
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) m = std::max(m, dm[static_cast<size_t>(y + yb) * ws + x + xb]);
    return m;
  }
};
}  // namespace

namespace {
gb200::SearchParams to_search_params(const gb200_params* params) {
  gb200::SearchParams sp;
  if (params) {
    sp.butteraugli_target = params->butteraugli_target;
    sp.clear_metadata = params->clear_metadata != 0;
    sp.try_420 = params->try_420 != 0;
    sp.force_420 = params->force_420 != 0;
    sp.use_silver_screen = params->use_silver_screen != 0;
    sp.zeroing_greedy_lookahead = params->zeroing_greedy_lookahead;
    sp.new_zeroing_model = params->new_zeroing_model != 0;
  }
  return sp;
}
void fill_stats(const gb200::SearchStats& st, gb200_stats* stats) {
  if (!stats) return;
  stats->iterations = st.iterations;
  stats->iterations_up = st.iterations_up;
  stats->iterations_down = st.iterations_down;
  stats->compares = st.compares;
  stats->gpu_launches = st.gpu_launches;
  stats->h2d_bytes = st.h2d_bytes;
  stats->d2h_bytes = st.d2h_bytes;
  stats->ms_total = st.ms_total;
  stats->ms_device_setup = st.ms_device_setup;
  stats->ms_compare = st.ms_compare;
  stats->ms_zeroing = st.ms_zeroing;
  stats->ms_jpeg = st.ms_jpeg;
  stats->ms_sort = st.ms_sort;
  stats->ms_walk = st.ms_walk;
  stats->order_partial = st.order_partial;
  stats->order_exact = st.order_exact;
}
}  // namespace

extern "C" {

void gb200_params_default(gb200_params* p) {
  p->butteraugli_target = 1.0f;
  p->clear_metadata = 1;
  p->try_420 = 0;
  p->force_420 = 0;
  p->use_silver_screen = 0;
  p->zeroing_greedy_lookahead = 3;
  p->new_zeroing_model = 1;
}

double gb200_butteraugli_score_for_quality(double quality) { return gb200::distance_for_quality(quality); }

int gb200_process_rgb(const gb200_params* params, const uint8_t* rgb, int w, int h, int device,
                      gb200_log_fn log, void* log_user, uint8_t** out, size_t* out_len,
                      gb200_stats* stats) {
  *out = nullptr;
  *out_len = 0;
  bool ok = false;
  int guarded_ok = guarded([&]() {
    gb200::SearchParams sp = to_search_params(params);
    gb200::SearchStats st;
    std::string jpeg, err;
    ok = gb200::process_rgb(sp, rgb, w, h, device, log, log_user, &jpeg, &st, &err);
    if (!ok) g_err = err;
    if (!jpeg.empty()) {
      *out = static_cast<uint8_t*>(malloc(jpeg.size()));
      memcpy(*out, jpeg.data(), jpeg.size());
      *out_len = jpeg.size();
    }
    fill_stats(st, stats);
  });
  return (guarded_ok && ok) ? 1 : 0;
}

namespace {
// the encoder's result and counters into the C outputs
void take_jpeg(const std::string& jpeg, const gb200::SearchStats& st, uint8_t** out, size_t* out_len,
               gb200_stats* stats) {
  if (!jpeg.empty()) {
    *out = static_cast<uint8_t*>(malloc(jpeg.size()));
    memcpy(*out, jpeg.data(), jpeg.size());
    *out_len = jpeg.size();
  }
  fill_stats(st, stats);
}
}  // namespace

int gb200_process_image(const gb200_params* params, const uint8_t* img, int w, int h, int channels,
                        const int64_t* strides, int device, gb200_log_fn log, void* log_user, uint8_t** out,
                        size_t* out_len, gb200_stats* stats) {
  *out = nullptr;
  *out_len = 0;
  bool ok = false;
  int guarded_ok = guarded([&]() {
    gb200::SearchStats st;
    std::string jpeg, err;
    ok = gb200::process_image(to_search_params(params), img, w, h, channels, strides, device, log, log_user, &jpeg,
                              &st, &err);
    if (!ok) g_err = err;
    take_jpeg(jpeg, st, out, out_len, stats);
  });
  return (guarded_ok && ok) ? 1 : 0;
}

int gb200_process_image_device(const gb200_params* params, const uint8_t* img_dev, int w, int h, int channels,
                               const int64_t* strides, int device, gb200_log_fn log, void* log_user, uint8_t** out,
                               size_t* out_len, gb200_stats* stats, void* stream) {
  *out = nullptr;
  *out_len = 0;
  bool ok = false;
  int guarded_ok = guarded([&]() {
    const void* ptrs[1] = {img_dev};
    const char* what[1] = {"img"};
    check_device_pointers("process_image_device", device, ptrs, what, 1);
    gb200::SearchStats st;
    std::string jpeg, err;
    ok = gb200::process_image_device(to_search_params(params), img_dev, w, h, channels, strides, device,
                                     caller_stream(stream), log, log_user, &jpeg, &st, &err);
    if (!ok) g_err = err;
    take_jpeg(jpeg, st, out, out_len, stats);
  });
  return (guarded_ok && ok) ? 1 : 0;
}

int gb200_process_jpeg(const gb200_params* params, const uint8_t* jpeg_in, size_t jpeg_len, int device,
                       gb200_log_fn log, void* log_user, uint8_t** out, size_t* out_len, gb200_stats* stats) {
  *out = nullptr;
  *out_len = 0;
  bool ok = false;
  int guarded_ok = guarded([&]() {
    gb200::SearchParams sp = to_search_params(params);
    gb200::SearchStats st;
    std::string jpeg, err;
    ok = gb200::process_jpeg(sp, jpeg_in, jpeg_len, device, log, log_user, &jpeg, &st, &err);
    if (!ok) g_err = err;
    if (!jpeg.empty()) {
      *out = static_cast<uint8_t*>(malloc(jpeg.size()));
      memcpy(*out, jpeg.data(), jpeg.size());
      *out_len = jpeg.size();
    }
    fill_stats(st, stats);
  });
  return (guarded_ok && ok) ? 1 : 0;
}

int gb200_process_jpeg_from_device(const gb200_params* params, const uint8_t* jpeg_dev, size_t jpeg_len, int device,
                                   gb200_log_fn log, void* log_user, uint8_t** out, size_t* out_len,
                                   gb200_stats* stats, void* stream) {
  *out = nullptr;
  *out_len = 0;
  bool ok = false;
  int guarded_ok = guarded([&]() {
    // an empty file may have no bytes at all; it is then refused as gb200_process_jpeg refuses it
    const void* ptrs[1] = {jpeg_len ? jpeg_dev : nullptr};
    const char* what[1] = {"jpeg"};
    check_device_pointers("process_jpeg_from_device", device, ptrs, what, 1);
    gb200::SearchStats st;
    std::string jpeg, err;
    ok = gb200::process_jpeg_from_device(to_search_params(params), jpeg_dev, jpeg_len, device, caller_stream(stream),
                                         log, log_user, &jpeg, &st, &err);
    if (!ok) g_err = err;
    take_jpeg(jpeg, st, out, out_len, stats);
  });
  return (guarded_ok && ok) ? 1 : 0;
}

// butteraugli::ButteraugliInterface (b/butteraugli.cc:1858) on the device kernels.
int gb200_butteraugli_diffmap(const float* rgb0, const float* rgb1, int w, int h, int device, float* diffmap,
                              double* score) {
  if (rgb0 == nullptr || rgb1 == nullptr || w < 1 || h < 1) {
    g_err = "butteraugli: no image";
    return 0;
  }
  return guarded([&]() {
    const Pad8 pad(w, h);
    std::vector<float> s0, s1;
    gb200::Butteraugli ba(pad.ws, pad.hs, device, nullptr);
    ba.analyse_original(pad.pad(rgb0, 3, 1, &s0));
    const float dmax = ba.compare_linear(pad.pad(rgb1, 3, 1, &s1));
    std::vector<float> dm(static_cast<size_t>(pad.ws) * pad.hs);
    if (diffmap != nullptr || pad.padded()) ba.download_distmap(dm.data());
    if (diffmap) pad.crop(dm.data(), diffmap);
    if (score) *score = pad.padded() ? pad.cropped_max(dm.data()) : dmax;
  });
}

// ---- butteraugli::ButteraugliComparator (b/butteraugli.h:425) ---------------------
// butteraugli::ButteraugliComparator::ButteraugliComparator (b/butteraugli.cc:784)
gb200_butteraugli_comparator* gb200_butteraugli_comparator_create(const float* rgb0, int w, int h, int device) {
  return gb200_butteraugli_comparator_create_batch(rgb0, w, h, 1, device);
}

void gb200_butteraugli_comparator_destroy(gb200_butteraugli_comparator* c) {
  if (!c) return;
  guarded([&]() {
    delete c->ba;
    delete c->white;
  });
  delete c;
}

// ButteraugliComparator::Diffmap (b/butteraugli.cc:799) + ButteraugliScoreFromDiffmap (:1623)
int gb200_butteraugli_comparator_diffmap(gb200_butteraugli_comparator* c, const float* rgb1, float* diffmap,
                                         double* score) {
  if (c == nullptr || rgb1 == nullptr) {
    g_err = "butteraugli comparator: no comparator or no image";
    return 0;
  }
  if (!comparator_takes(c, false)) return 0;
  return guarded([&]() {
    const float m = c->ba->compare_linear(rgb1);
    if (diffmap) c->ba->download_distmap(diffmap);
    if (score) *score = m;
  });
}

// The same with rgb1 and diffmap in device memory of the comparator's device.
int gb200_butteraugli_comparator_diffmap_device(gb200_butteraugli_comparator* c, const float* rgb1_dev,
                                                float* diffmap_dev, double* score, void* stream) {
  if (c == nullptr || rgb1_dev == nullptr) {
    g_err = "butteraugli comparator: no comparator or no image";
    return 0;
  }
  if (!comparator_takes(c, false)) return 0;
  return guarded([&]() {
    c->ba->bind();
    const void* ptrs[2] = {rgb1_dev, diffmap_dev};
    const char* what[2] = {"rgb1", "diffmap"};
    check_device_pointers("butteraugli comparator", c->ba->device(), ptrs, what, 2);
    const float m = c->ba->compare_linear_device(rgb1_dev, diffmap_dev, caller_stream(stream));
    if (score) *score = m;
  });
}

namespace {
// The comparator with `capacity` candidate slots: ButteraugliComparator::ButteraugliComparator(rgb0) once
// (capacity 1: the single-image metric); on_device: rgb0 in memory of `device`, read after `stream`'s work
gb200_butteraugli_comparator* comparator_create(const float* rgb0, int w, int h, int capacity, int device,
                                                bool on_device, void* stream) {
  gb200_butteraugli_comparator* c = nullptr;
  guarded([&]() {
    if (rgb0 == nullptr) throw std::runtime_error("butteraugli comparator: no image");
    check_create("butteraugli comparator", "image", w, h, capacity);
    if (on_device) {
      const void* ptrs[1] = {rgb0};
      const char* what[1] = {"rgb0"};
      check_device_pointers("butteraugli comparator", device, ptrs, what, 1);
    }
    std::unique_ptr<gb200::Butteraugli> ba(
        new gb200::Butteraugli(w, h, capacity, device, gb200::Butteraugli::Slots::kCandidates));
    ba->analyse_original(rgb0, on_device, caller_stream(stream));
    c = new gb200_butteraugli_comparator;
    c->ba = ba.release();
  });
  return c;
}
}  // namespace

gb200_butteraugli_comparator* gb200_butteraugli_comparator_create_batch(const float* rgb0, int w, int h, int capacity,
                                                                        int device) {
  return comparator_create(rgb0, w, h, capacity, device, false, nullptr);
}

gb200_butteraugli_comparator* gb200_butteraugli_comparator_create_device(const float* rgb0_dev, int w, int h,
                                                                         int capacity, int device, void* stream) {
  return comparator_create(rgb0_dev, w, h, capacity, device, true, stream);
}

namespace {
int comparator_diffmap_batch(gb200_butteraugli_comparator* c, const float* rgb1, int n, float* diffmap, double* score,
                             bool device, void* stream) {
  if (c == nullptr || rgb1 == nullptr) {
    g_err = "butteraugli comparator: no comparator or no images";
    return 0;
  }
  if (!comparator_takes(c, false)) return 0;
  if (!n_ok("comparator", "images", n, *c->ba)) return 0;
  return scored(c->ba, n, score, [&](float* m) {
    if (device) {
      const void* ptrs[2] = {rgb1, diffmap};
      const char* what[2] = {"rgb1", "diffmap"};
      check_device_pointers("butteraugli comparator", c->ba->device(), ptrs, what, 2);
    }
    c->ba->compare_many(rgb1, n, diffmap, m, device, caller_stream(stream));
  });
}
}  // namespace

int gb200_butteraugli_comparator_diffmap_batch(gb200_butteraugli_comparator* c, const float* rgb1, int n,
                                               float* diffmap, double* score) {
  return comparator_diffmap_batch(c, rgb1, n, diffmap, score, false, nullptr);
}

int gb200_butteraugli_comparator_diffmap_batch_device(gb200_butteraugli_comparator* c, const float* rgb1_dev, int n,
                                                      float* diffmap_dev, double* score, void* stream) {
  return comparator_diffmap_batch(c, rgb1_dev, n, diffmap_dev, score, true, stream);
}

// ---- butteraugli::ButteraugliInterface (b/butteraugli.cc:1858) on N pairs per call ----------
gb200_butteraugli_batch* gb200_butteraugli_batch_create(int w, int h, int capacity, int device) {
  gb200_butteraugli_batch* b = nullptr;
  guarded([&]() {
    check_create("butteraugli batch", "images", w, h, capacity);
    gb200::Butteraugli* ba = new gb200::Butteraugli(w, h, capacity, device);
    b = new gb200_butteraugli_batch;
    b->ba = ba;
  });
  return b;
}

void gb200_butteraugli_batch_destroy(gb200_butteraugli_batch* b) {
  if (!b) return;
  guarded([&]() { delete b->ba; });
  delete b;
}

namespace {
int batch_diffmap(gb200_butteraugli_batch* b, const float* rgb0, const float* rgb1, int n, float* diffmap,
                  double* score, bool device, void* stream) {
  if (b == nullptr || rgb0 == nullptr || rgb1 == nullptr) {
    g_err = "butteraugli batch: no batch or no images";
    return 0;
  }
  if (!n_ok("batch", "pairs", n, *b->ba)) return 0;
  return scored(b->ba, n, score, [&](float* m) {
    if (device) {
      const void* ptrs[3] = {rgb0, rgb1, diffmap};
      const char* what[3] = {"rgb0", "rgb1", "diffmap"};
      check_device_pointers("butteraugli batch", b->ba->device(), ptrs, what, 3);
    }
    b->ba->compare_batch(rgb0, rgb1, n, diffmap, m, device, caller_stream(stream));
  });
}
}  // namespace

int gb200_butteraugli_batch_diffmap(gb200_butteraugli_batch* b, const float* rgb0, const float* rgb1, int n,
                                    float* diffmap, double* score) {
  return batch_diffmap(b, rgb0, rgb1, n, diffmap, score, false, nullptr);
}

int gb200_butteraugli_batch_diffmap_device(gb200_butteraugli_batch* b, const float* rgb0_dev, const float* rgb1_dev,
                                           int n, float* diffmap_dev, double* score, void* stream) {
  return batch_diffmap(b, rgb0_dev, rgb1_dev, n, diffmap_dev, score, true, stream);
}

namespace {
// pairs of different sizes: every argument is checked before anything is queued
int batch_diffmap_sizes(gb200_butteraugli_batch* b, const int* w, const int* h, const float* const* rgb0,
                        const float* const* rgb1, int n, float* const* diffmap, double* score, bool device,
                        void* stream) {
  if (b == nullptr || w == nullptr || h == nullptr || rgb0 == nullptr || rgb1 == nullptr) {
    g_err = "butteraugli batch: no batch, no sizes or no images";
    return 0;
  }
  if (!n_ok("batch", "pairs", n, *b->ba)) return 0;
  for (int i = 0; i < n; ++i) {
    if (!pair_size_ok(*b->ba, i, w[i], h[i])) return 0;
    if (rgb0[i] == nullptr || rgb1[i] == nullptr || (diffmap != nullptr && diffmap[i] == nullptr)) {
      g_err = "butteraugli batch: pair " + std::to_string(i) + " has a null image or diffmap pointer";
      return 0;
    }
  }
  return scored(b->ba, n, score, [&](float* m) {
    if (device) check_pair_pointers(*b->ba, "rgb0", "rgb1", rgb0, rgb1, diffmap, n);
    b->ba->compare_batch_sizes(w, h, rgb0, rgb1, n, diffmap, m, device, caller_stream(stream));
  });
}
}  // namespace

int gb200_butteraugli_batch_diffmap_sizes(gb200_butteraugli_batch* b, const int* w, const int* h,
                                          const float* const* rgb0, const float* const* rgb1, int n,
                                          float* const* diffmap, double* score) {
  return batch_diffmap_sizes(b, w, h, rgb0, rgb1, n, diffmap, score, false, nullptr);
}

int gb200_butteraugli_batch_diffmap_sizes_device(gb200_butteraugli_batch* b, const int* w, const int* h,
                                                 const float* const* rgb0_dev, const float* const* rgb1_dev, int n,
                                                 float* const* diffmap_dev, double* score, void* stream) {
  return batch_diffmap_sizes(b, w, h, rgb0_dev, rgb1_dev, n, diffmap_dev, score, true, stream);
}

// ---- 8-bit sRGB input: the stand-alone tool's conversion and alpha rule (butteraugli_main.cc:239-281,
// :390-419) in front of the float entries above ----
namespace {
bool channels_ok(const char* who, int channels) {
  if (channels == 3 || channels == 4) return true;
  g_err = std::string(who) + ": channels = " + std::to_string(channels) + ", 8-bit images must have 3 (RGB) or 4 (RGBA)";
  return false;
}
}  // namespace

int gb200_butteraugli_diffmap_srgb(const uint8_t* img0, const uint8_t* img1, int w, int h, int channels, int device,
                                   float* diffmap, double* score) {
  if (img0 == nullptr || img1 == nullptr || w < 1 || h < 1) {
    g_err = "butteraugli: no image";
    return 0;
  }
  if (!channels_ok("butteraugli", channels)) return 0;
  return guarded([&]() {
    // padded as gb200_butteraugli_diffmap pads its planes; the conversion is per pixel, so replicating
    // bytes first gives the same planes
    const Pad8 pad(w, h);
    std::vector<uint8_t> s0, s1;
    const uint8_t* p0 = pad.pad(img0, 1, channels, &s0);
    const uint8_t* p1 = pad.pad(img1, 1, channels, &s1);
    gb200::Butteraugli ba(pad.ws, pad.hs, 1, device);  // a pair batch of one
    std::vector<float> dm(static_cast<size_t>(pad.ws) * pad.hs);
    // Each background is scored as ButteraugliInterface scores it, padded and then cropped, and the
    // tool chooses on those cropped scores (butteraugli_main.cc:390-419).  Padding can hold the maximum
    // of a padded diffmap, so the choice cannot be made on the padded maxima.
    float best = 0.0f;
    for (int k = 0; k < (channels == 4 ? 2 : 1); ++k) {
      float m = 0.0f;
      ba.compare_batch_srgb(p0, p1, 1, channels, dm.data(), &m, false, 0, k == 0 ? 0 : 255);
      if (pad.padded()) m = pad.cropped_max(dm.data());
      if (k == 1 && !gb200::white_wins(m, best)) continue;
      best = m;
      if (diffmap) pad.crop(dm.data(), diffmap);
    }
    if (score) *score = best;
  });
}

namespace {
int batch_diffmap_srgb(gb200_butteraugli_batch* b, const uint8_t* img0, const uint8_t* img1, int n, int channels,
                       float* diffmap, double* score, bool device, void* stream) {
  if (b == nullptr || img0 == nullptr || img1 == nullptr) {
    g_err = "butteraugli batch: no batch or no images";
    return 0;
  }
  if (!n_ok("batch", "pairs", n, *b->ba)) return 0;
  if (!channels_ok("butteraugli batch", channels)) return 0;
  return scored(b->ba, n, score, [&](float* m) {
    if (device) {
      const void* ptrs[3] = {img0, img1, diffmap};
      const char* what[3] = {"img0", "img1", "diffmap"};
      check_device_pointers("butteraugli batch", b->ba->device(), ptrs, what, 3);
    }
    b->ba->compare_batch_srgb(img0, img1, n, channels, diffmap, m, device, caller_stream(stream));
  });
}

// 8-bit pairs of different sizes: every argument is checked before anything is queued
int batch_diffmap_sizes_srgb(gb200_butteraugli_batch* b, const int* w, const int* h, const int* channels,
                             const uint8_t* const* img0, const uint8_t* const* img1, int n, float* const* diffmap,
                             double* score, bool device, void* stream) {
  if (b == nullptr || w == nullptr || h == nullptr || channels == nullptr || img0 == nullptr || img1 == nullptr) {
    g_err = "butteraugli batch: no batch, no sizes, no channels or no images";
    return 0;
  }
  if (!n_ok("batch", "pairs", n, *b->ba)) return 0;
  for (int i = 0; i < n; ++i) {
    const std::string pair = "butteraugli batch: pair " + std::to_string(i);
    if (!pair_size_ok(*b->ba, i, w[i], h[i])) {
      if (w[i] < 8 || h[i] < 8) g_err += " (gb200_butteraugli_diffmap_srgb scores smaller pairs)";
      return 0;
    }
    if (!channels_ok(pair.c_str(), channels[i])) return 0;
    if (img0[i] == nullptr || img1[i] == nullptr) {
      g_err = pair + " has a null image pointer";
      return 0;
    }
  }
  return scored(b->ba, n, score, [&](float* m) {
    if (device) check_pair_pointers(*b->ba, "img0", "img1", img0, img1, diffmap, n);
    b->ba->compare_batch_sizes_srgb(w, h, channels, img0, img1, n, diffmap, m, device, caller_stream(stream));
  });
}

int comparator_diffmap_srgb(gb200_butteraugli_comparator* c, const uint8_t* img1, int n, float* diffmap, double* score,
                            bool device, void* stream) {
  if (c == nullptr || img1 == nullptr) {
    g_err = "butteraugli comparator: no comparator or no images";
    return 0;
  }
  if (!comparator_takes(c, true)) return 0;
  if (!n_ok("comparator", "images", n, *c->ba)) return 0;
  return scored(c->ba, n, score, [&](float* m) {
    if (device) {
      const void* ptrs[2] = {img1, diffmap};
      const char* what[2] = {"img1", "diffmap"};
      check_device_pointers("butteraugli comparator", c->ba->device(), ptrs, what, 2);
    }
    c->ba->compare_many_srgb(img1, n, c->channels, c->white, diffmap, m, device, caller_stream(stream));
  });
}
}  // namespace

int gb200_butteraugli_batch_diffmap_srgb(gb200_butteraugli_batch* b, const uint8_t* img0, const uint8_t* img1, int n,
                                         int channels, float* diffmap, double* score) {
  return batch_diffmap_srgb(b, img0, img1, n, channels, diffmap, score, false, nullptr);
}

int gb200_butteraugli_batch_diffmap_srgb_device(gb200_butteraugli_batch* b, const uint8_t* img0_dev,
                                                const uint8_t* img1_dev, int n, int channels, float* diffmap_dev,
                                                double* score, void* stream) {
  return batch_diffmap_srgb(b, img0_dev, img1_dev, n, channels, diffmap_dev, score, true, stream);
}

int gb200_butteraugli_batch_diffmap_sizes_srgb(gb200_butteraugli_batch* b, const int* w, const int* h,
                                               const int* channels, const uint8_t* const* img0,
                                               const uint8_t* const* img1, int n, float* const* diffmap,
                                               double* score) {
  return batch_diffmap_sizes_srgb(b, w, h, channels, img0, img1, n, diffmap, score, false, nullptr);
}

int gb200_butteraugli_batch_diffmap_sizes_srgb_device(gb200_butteraugli_batch* b, const int* w, const int* h,
                                                      const int* channels, const uint8_t* const* img0_dev,
                                                      const uint8_t* const* img1_dev, int n,
                                                      float* const* diffmap_dev, double* score, void* stream) {
  return batch_diffmap_sizes_srgb(b, w, h, channels, img0_dev, img1_dev, n, diffmap_dev, score, true, stream);
}

namespace {
gb200_butteraugli_comparator* comparator_create_srgb(const uint8_t* img0, int w, int h, int channels, int capacity,
                                                     int device, bool on_device, void* stream) {
  gb200_butteraugli_comparator* c = nullptr;
  if (!channels_ok("butteraugli comparator", channels)) return nullptr;
  guarded([&]() {
    if (img0 == nullptr) throw std::runtime_error("butteraugli comparator: no image");
    check_create("butteraugli comparator", "image", w, h, capacity);
    if (on_device) {
      const void* ptrs[1] = {img0};
      const char* what[1] = {"img0"};
      check_device_pointers("butteraugli comparator", device, ptrs, what, 1);
    }
    const gb200::Stream caller = caller_stream(stream);
    const gb200::Butteraugli::Slots kind = gb200::Butteraugli::Slots::kCandidates;
    std::unique_ptr<gb200::Butteraugli> black(new gb200::Butteraugli(w, h, capacity, device, kind));
    black->analyse_original_srgb(img0, channels, 0, on_device, caller);
    std::unique_ptr<gb200::Butteraugli> white;
    if (channels == 4) {  // a second resident original, laid over white
      white.reset(new gb200::Butteraugli(w, h, capacity, device, kind));
      white->analyse_original_srgb(img0, channels, 255, on_device, caller);
    }
    c = new gb200_butteraugli_comparator;
    c->ba = black.release();
    c->white = white.release();
    c->channels = channels;
  });
  return c;
}
}  // namespace

gb200_butteraugli_comparator* gb200_butteraugli_comparator_create_srgb(const uint8_t* img0, int w, int h, int channels,
                                                                       int capacity, int device) {
  return comparator_create_srgb(img0, w, h, channels, capacity, device, false, nullptr);
}

gb200_butteraugli_comparator* gb200_butteraugli_comparator_create_srgb_device(const uint8_t* img0_dev, int w, int h,
                                                                              int channels, int capacity, int device,
                                                                              void* stream) {
  return comparator_create_srgb(img0_dev, w, h, channels, capacity, device, true, stream);
}

int gb200_butteraugli_comparator_diffmap_srgb(gb200_butteraugli_comparator* c, const uint8_t* img1, int n,
                                              float* diffmap, double* score) {
  return comparator_diffmap_srgb(c, img1, n, diffmap, score, false, nullptr);
}

int gb200_butteraugli_comparator_diffmap_srgb_device(gb200_butteraugli_comparator* c, const uint8_t* img1_dev, int n,
                                                     float* diffmap_dev, double* score, void* stream) {
  return comparator_diffmap_srgb(c, img1_dev, n, diffmap_dev, score, true, stream);
}

// ---- comparator sets: originals of sizes of their own, resident, each candidate scored against the
// original it names (ButteraugliInterface per pair) ----
namespace {
const char* const kSet = "butteraugli comparator set";

gb200_butteraugli_comparator_set* set_create(const int* w, const int* h, const int* channels, const void* const* img0,
                                             int count, int capacity, int device, bool srgb, bool on_device = false,
                                             void* stream = nullptr) {
  if (w == nullptr || h == nullptr || img0 == nullptr || (srgb && channels == nullptr)) {
    g_err = std::string(kSet) + (srgb ? ": no sizes, no channels or no images" : ": no sizes or no images");
    return nullptr;
  }
  if (count < 1) {
    g_err = std::string(kSet) + ": count = " + std::to_string(count) + ", a set holds at least 1 original";
    return nullptr;
  }
  for (int i = 0; i < count; ++i) {
    const std::string orig = std::string(kSet) + ": original " + std::to_string(i);
    if (!create_size_ok(w[i], h[i])) {
      g_err = orig + " is " + std::to_string(w[i]) + "x" + std::to_string(h[i]) +
              ", the originals must be at least 8x8 (and below 65536)";
      return nullptr;
    }
    if (srgb && !channels_ok(orig.c_str(), channels[i])) return nullptr;
    if (img0[i] == nullptr) {
      g_err = orig + " has a null image pointer";
      return nullptr;
    }
  }
  gb200_butteraugli_comparator_set* s = nullptr;
  guarded([&]() {
    check_capacity(kSet, capacity);
    if (on_device)
      for (int i = 0; i < count; ++i) {
        const std::string name = std::string(srgb ? "img0" : "rgb0") + "[" + std::to_string(i) + "]";
        const char* what[1] = {name.c_str()};
        check_device_pointers(kSet, device, &img0[i], what, 1);
      }
    std::unique_ptr<gb200::ComparatorSet> set(new gb200::ComparatorSet(
        w, h, srgb ? channels : nullptr, img0, count, capacity, device, on_device, caller_stream(stream)));
    s = new gb200_butteraugli_comparator_set;
    s->set = set.release();
  });
  return s;
}

// every argument is checked before anything is queued
int set_diffmap(gb200_butteraugli_comparator_set* s, const int* original, const void* const* img1, int n,
                float* const* diffmap, double* score, bool srgb, bool device, void* stream) {
  if (s == nullptr || original == nullptr || img1 == nullptr) {
    g_err = std::string(kSet) + ": no set, no indices or no images";
    return 0;
  }
  if (!made_takes(kSet, s->set->srgb(), srgb)) return 0;
  gb200::Butteraugli& ba = s->set->metric();
  if (!n_ok("comparator set", "images", n, ba)) return 0;
  const int count = s->set->count();
  for (int i = 0; i < n; ++i) {
    if (original[i] < 0 || original[i] >= count) {
      g_err = std::string(kSet) + ": original[" + std::to_string(i) + "] = " + std::to_string(original[i]) +
              ", the set holds originals 0.." + std::to_string(count - 1);
      return 0;
    }
    if (img1[i] == nullptr) {
      g_err = std::string(kSet) + ": image " + std::to_string(i) + " has a null pointer";
      return 0;
    }
  }
  return scored(&ba, n, score, [&](float* m) {
    if (device)
      check_pair_pointers<void>(ba, "", srgb ? "img1" : "rgb1", nullptr, img1, diffmap, n, kSet);
    s->set->compare(original, img1, n, diffmap, m, device, caller_stream(stream));
  });
}
}  // namespace

gb200_butteraugli_comparator_set* gb200_butteraugli_comparator_set_create(const int* w, const int* h,
                                                                          const float* const* rgb0, int count,
                                                                          int capacity, int device) {
  return set_create(w, h, nullptr, reinterpret_cast<const void* const*>(rgb0), count, capacity, device, false);
}

gb200_butteraugli_comparator_set* gb200_butteraugli_comparator_set_create_srgb(const int* w, const int* h,
                                                                               const int* channels,
                                                                               const uint8_t* const* img0, int count,
                                                                               int capacity, int device) {
  return set_create(w, h, channels, reinterpret_cast<const void* const*>(img0), count, capacity, device, true);
}

gb200_butteraugli_comparator_set* gb200_butteraugli_comparator_set_create_device(const int* w, const int* h,
                                                                                 const float* const* rgb0_dev,
                                                                                 int count, int capacity, int device,
                                                                                 void* stream) {
  return set_create(w, h, nullptr, reinterpret_cast<const void* const*>(rgb0_dev), count, capacity, device, false,
                    true, stream);
}

gb200_butteraugli_comparator_set* gb200_butteraugli_comparator_set_create_srgb_device(
    const int* w, const int* h, const int* channels, const uint8_t* const* img0_dev, int count, int capacity,
    int device, void* stream) {
  return set_create(w, h, channels, reinterpret_cast<const void* const*>(img0_dev), count, capacity, device, true,
                    true, stream);
}

int gb200_butteraugli_comparator_set_diffmap(gb200_butteraugli_comparator_set* s, const int* original,
                                             const float* const* rgb1, int n, float* const* diffmap, double* score) {
  return set_diffmap(s, original, reinterpret_cast<const void* const*>(rgb1), n, diffmap, score, false, false, nullptr);
}

int gb200_butteraugli_comparator_set_diffmap_device(gb200_butteraugli_comparator_set* s, const int* original,
                                                    const float* const* rgb1_dev, int n, float* const* diffmap_dev,
                                                    double* score, void* stream) {
  return set_diffmap(s, original, reinterpret_cast<const void* const*>(rgb1_dev), n, diffmap_dev, score, false, true,
                     stream);
}

int gb200_butteraugli_comparator_set_diffmap_srgb(gb200_butteraugli_comparator_set* s, const int* original,
                                                  const uint8_t* const* img1, int n, float* const* diffmap,
                                                  double* score) {
  return set_diffmap(s, original, reinterpret_cast<const void* const*>(img1), n, diffmap, score, true, false, nullptr);
}

int gb200_butteraugli_comparator_set_diffmap_srgb_device(gb200_butteraugli_comparator_set* s, const int* original,
                                                         const uint8_t* const* img1_dev, int n,
                                                         float* const* diffmap_dev, double* score, void* stream) {
  return set_diffmap(s, original, reinterpret_cast<const void* const*>(img1_dev), n, diffmap_dev, score, true, true,
                     stream);
}

void gb200_butteraugli_comparator_set_destroy(gb200_butteraugli_comparator_set* s) {
  if (!s) return;
  guarded([&]() { delete s->set; });
  delete s;
}

namespace {
// ButteraugliComparator::Mask (b/butteraugli.cc:793)
int comparator_mask(gb200_butteraugli_comparator* c, float* mask, float* mask_dc, bool device, void* stream) {
  if (c == nullptr || mask == nullptr || mask_dc == nullptr) {
    g_err = "butteraugli comparator: no comparator or no output";
    return 0;
  }
  if (c->channels == 4) {
    g_err = "butteraugli comparator: an RGBA comparator has two originals (over black and over white), no one mask";
    return 0;
  }
  return guarded([&]() {
    if (device) {
      const void* ptrs[2] = {mask, mask_dc};
      const char* what[2] = {"mask", "mask_dc"};
      check_device_pointers("butteraugli comparator", c->ba->device(), ptrs, what, 2);
    }
    c->ba->mask(mask, mask_dc, device, caller_stream(stream));
  });
}

// butteraugli::ButteraugliAdaptiveQuantization (b/butteraugli.cc:1880)
int adaptive_quantization(const float* rgb, int w, int h, int device, float* quant, bool on_device, void* stream) {
  if (rgb == nullptr || quant == nullptr) {
    g_err = "butteraugli adaptive quantization: no image or no output";
    return 0;
  }
  if (w < 16 || h < 16 || w >= 65536 || h >= 65536) {
    g_err = "butteraugli adaptive quantization: the image must be at least 16x16 (and below 65536)";
    return 0;
  }
  return guarded([&]() {
    if (on_device) {  // the quantization field depends on the image alone: no analysis of it is needed
      const void* ptrs[2] = {rgb, quant};
      const char* what[2] = {"rgb", "quant"};
      check_device_pointers("butteraugli adaptive quantization", device, ptrs, what, 2);
      gb200::Butteraugli ba(w, h, device, nullptr);
      ba.adaptive_quantization(rgb, quant, true, caller_stream(stream));
      return;
    }
    gb200::Butteraugli ba(w, h, device, nullptr);
    ba.analyse_original(rgb);
    ba.adaptive_quantization(rgb, quant);
  });
}

// CreateHeatMapImage (b/butteraugli.cc:1979) of n maps in one launch
int heatmap(const int* w, const int* h, const float* const* diffmap, int n, double good, double bad,
            uint8_t* const* rgb, int device, bool on_device, void* stream) {
  const char* const who = "butteraugli heatmap";
  if (w == nullptr || h == nullptr || diffmap == nullptr || rgb == nullptr) {
    g_err = std::string(who) + ": no sizes, no maps or no outputs";
    return 0;
  }
  if (n < 1) {
    g_err = std::string(who) + ": n = " + std::to_string(n) + ", a call takes at least 1 map";
    return 0;
  }
  if (!(good > 0) || !(bad > good)) {
    g_err = std::string(who) + ": the thresholds must satisfy 0 < good < bad, got good = " + std::to_string(good) +
            ", bad = " + std::to_string(bad);
    return 0;
  }
  for (int i = 0; i < n; ++i) {
    const std::string map = std::string(who) + ": map " + std::to_string(i);
    if (w[i] < 1 || h[i] < 1) {
      g_err = map + " is " + std::to_string(w[i]) + "x" + std::to_string(h[i]) + ", a map has at least 1x1 pixels";
      return 0;
    }
    if (diffmap[i] == nullptr || rgb[i] == nullptr) {
      g_err = map + " has a null pointer";
      return 0;
    }
  }
  return guarded([&]() {
    if (on_device)
      for (int i = 0; i < n; ++i) {
        const std::string k = "[" + std::to_string(i) + "]";
        const std::string names[2] = {"diffmap" + k, "rgb" + k};
        const void* ptrs[2] = {diffmap[i], rgb[i]};
        const char* what[2] = {names[0].c_str(), names[1].c_str()};
        check_device_pointers(who, device, ptrs, what, 2);
      }
    gb200::butteraugli_heatmap(w, h, diffmap, n, good, bad, rgb, on_device, device, caller_stream(stream));
  });
}
}  // namespace

int gb200_butteraugli_comparator_mask(gb200_butteraugli_comparator* c, float* mask, float* mask_dc) {
  return comparator_mask(c, mask, mask_dc, false, nullptr);
}

int gb200_butteraugli_comparator_mask_device(gb200_butteraugli_comparator* c, float* mask_dev, float* mask_dc_dev,
                                             void* stream) {
  return comparator_mask(c, mask_dev, mask_dc_dev, true, stream);
}

int gb200_butteraugli_adaptive_quantization(const float* rgb, int w, int h, int device, float* quant) {
  return adaptive_quantization(rgb, w, h, device, quant, false, nullptr);
}

int gb200_butteraugli_adaptive_quantization_device(const float* rgb_dev, int w, int h, int device, float* quant_dev,
                                                   void* stream) {
  return adaptive_quantization(rgb_dev, w, h, device, quant_dev, true, stream);
}

int gb200_butteraugli_heatmap(const int* w, const int* h, const float* const* diffmap, int n, double good, double bad,
                              uint8_t* const* rgb, int device) {
  return heatmap(w, h, diffmap, n, good, bad, rgb, device, false, nullptr);
}

int gb200_butteraugli_heatmap_device(const int* w, const int* h, const float* const* diffmap_dev, int n, double good,
                                     double bad, uint8_t* const* rgb_dev, int device, void* stream) {
  return heatmap(w, h, diffmap_dev, n, good, bad, rgb_dev, device, true, stream);
}

int gb200_jpeg_dimensions(const uint8_t* jpeg_in, size_t jpeg_len, int* width, int* height) {
  return gb200::read_jpeg_dimensions(jpeg_in, jpeg_len, width, height) ? 1 : 0;
}

namespace {
// gb200_jpeg_decode_rgb[_device]: every file parsed and checked, and every output pointer, before anything
// runs; a refusal names the file
int jpeg_decode(const char* who, const uint8_t* const* jpeg, const size_t* len, int n, int device,
                uint8_t* const* out, bool on_device, void* stream) {
  return guarded([&]() {
    if (n < 1) throw std::runtime_error(std::string(who) + ": n must be at least 1");
    if (jpeg == nullptr || len == nullptr || out == nullptr)
      throw std::runtime_error(std::string(who) + ": jpeg, len and out must not be null");
    for (int i = 0; i < n; ++i) {
      const std::string k = "[" + std::to_string(i) + "]";
      if (jpeg[i] == nullptr) throw std::runtime_error(std::string(who) + ": jpeg" + k + " is null");
      if (out[i] == nullptr) throw std::runtime_error(std::string(who) + ": out" + k + " is null");
      if (on_device) {
        const std::string name = "out" + k;
        const void* ptrs[1] = {out[i]};
        const char* what[1] = {name.c_str()};
        check_device_pointers(who, device, ptrs, what, 1);
      }
    }
    std::vector<gb200::JpegInput> files(n);
    std::vector<const gb200::JpegInput*> ptrs(n);
    for (int i = 0; i < n; ++i) {
      const std::string file = std::string(who) + ": file " + std::to_string(i) + ": ";
      std::string why;
      if (!gb200::read_jpeg(jpeg[i], len[i], &files[i], &why)) throw std::runtime_error(file + why);
      int w = 0, h = 0;
      if (!gb200::read_jpeg_dimensions(jpeg[i], len[i], &w, &h) || w != files[i].width || h != files[i].height)
        throw std::runtime_error(file + "the frame size differs from what gb200_jpeg_dimensions reads");
      if (!gb200::libjpeg_decodable(files[i], &why)) throw std::runtime_error(file + why);
      ptrs[i] = &files[i];
    }
    gb200::jpeg_decode_rgb(ptrs.data(), n, device, out, on_device, caller_stream(stream));
  });
}
}  // namespace

int gb200_jpeg_decode_rgb(const uint8_t* const* jpeg, const size_t* len, int n, int device, uint8_t* const* out) {
  return jpeg_decode("jpeg_decode_rgb", jpeg, len, n, device, out, false, nullptr);
}

int gb200_jpeg_decode_rgb_device(const uint8_t* const* jpeg, const size_t* len, int n, int device,
                                 uint8_t* const* out_dev, void* stream) {
  return jpeg_decode("jpeg_decode_rgb_device", jpeg, len, n, device, out_dev, true, stream);
}

namespace {
// the pointer checks of the *_from_device entries: every input and output pointer, before anything runs
void check_jpeg_device_args(const char* who, const uint8_t* const* jpeg, const size_t* len, int n, int device,
                            uint8_t* const* out) {
  if (n < 1) throw std::runtime_error(std::string(who) + ": n must be at least 1");
  if (jpeg == nullptr || len == nullptr) throw std::runtime_error(std::string(who) + ": jpeg and len must not be null");
  for (int i = 0; i < n; ++i) {
    const std::string k = "[" + std::to_string(i) + "]";
    // an empty file may have no bytes at all; the decode then refuses it with read_jpeg's reason
    if (jpeg[i] == nullptr && len[i] != 0) throw std::runtime_error(std::string(who) + ": jpeg" + k + " is null");
    if (out && out[i] == nullptr) throw std::runtime_error(std::string(who) + ": out" + k + " is null");
    const std::string nj = "jpeg" + k, no = "out" + k;
    const void* ptrs[2] = {len[i] ? jpeg[i] : nullptr, out ? out[i] : nullptr};
    const char* what[2] = {nj.c_str(), no.c_str()};
    check_device_pointers(who, device, ptrs, what, out ? 2 : 1);
  }
}
}  // namespace

int gb200_jpeg_dimensions_from_device(const uint8_t* const* jpeg_dev, const size_t* len, int n, int device,
                                      void* stream, int* width, int* height) {
  return guarded([&]() {
    const char* who = "jpeg_dimensions_from_device";
    if (width == nullptr || height == nullptr)
      throw std::runtime_error(std::string(who) + ": width and height must not be null");
    check_jpeg_device_args(who, jpeg_dev, len, n, device, nullptr);
    gb200::jpeg_dimensions_from_device(jpeg_dev, len, n, device, caller_stream(stream), width, height);
  });
}

int gb200_jpeg_decode_rgb_from_device(const uint8_t* const* jpeg_dev, const size_t* len, int n, int device,
                                      const int* width, const int* height, uint8_t* const* out_dev, void* stream) {
  return guarded([&]() {
    const char* who = "jpeg_decode_rgb_from_device";
    if (width == nullptr || height == nullptr || out_dev == nullptr)
      throw std::runtime_error(std::string(who) + ": width, height and out must not be null");
    check_jpeg_device_args(who, jpeg_dev, len, n, device, out_dev);
    gb200::jpeg_decode_rgb_from_device(who, jpeg_dev, len, n, device, width, height, out_dev, caller_stream(stream));
  });
}

int gb200_debug_entropy_decode(const uint8_t* jpeg_in, size_t jpeg_len, int S, int16_t* out, size_t out_cap,
                               int* status) {
  return guarded([&]() {
    if (jpeg_in == nullptr || status == nullptr) throw std::runtime_error("debug_entropy_decode: null argument");
    std::vector<int16_t> c;
    *status = gb200::jpeg_debug_entropy_decode(jpeg_in, jpeg_len, S, &c) ? 1 : 0;
    if (*status) {
      if (c.size() > out_cap) throw std::runtime_error("debug_entropy_decode: out is too small");
      memcpy(out, c.data(), c.size() * sizeof(int16_t));
    }
  });
}

int gb200_debug_entropy_decode_flags(const uint8_t* jpeg_in, size_t jpeg_len, int S, int16_t* out, size_t out_cap,
                                     int* taken, unsigned* flags, int* rounds) {
  return guarded([&]() {
    if (jpeg_in == nullptr || taken == nullptr || flags == nullptr || rounds == nullptr)
      throw std::runtime_error("debug_entropy_decode_flags: null argument");
    if (S < 8) throw std::runtime_error("debug_entropy_decode_flags: subsequences of fewer than 8 bits");
    std::vector<int16_t> c;
    gb200::JpegDebugDecode r;
    gb200::jpeg_debug_entropy_decode_flags(jpeg_in, jpeg_len, S, &c, &r);
    if (c.size() > out_cap) throw std::runtime_error("debug_entropy_decode_flags: out is too small");
    if (!c.empty()) memcpy(out, c.data(), c.size() * sizeof(int16_t));
    *taken = r.taken ? 1 : 0;
    *flags = r.flags;
    *rounds = r.rounds;
  });
}

int gb200_debug_jpeg_seed(const uint8_t* jpeg_in, size_t jpeg_len, int S, int16_t* dq, size_t dq_cap, int* status) {
  return guarded([&]() {
    if (jpeg_in == nullptr || dq == nullptr || status == nullptr)
      throw std::runtime_error("debug_jpeg_seed: null argument");
    if (S < 8) throw std::runtime_error("debug_jpeg_seed: subsequences of fewer than 8 bits");
    std::vector<int16_t> c;
    *status = gb200::jpeg_debug_seed_route(jpeg_in, jpeg_len, S, &c);
    if (c.size() > dq_cap) throw std::runtime_error("debug_jpeg_seed: dq is too small");
    memcpy(dq, c.data(), c.size() * sizeof(int16_t));
  });
}

int gb200_debug_read_jpeg(const uint8_t* jpeg_in, size_t jpeg_len, int* dims, int16_t* out, size_t out_cap) {
  gb200::JpegInput jpg;
  std::string err;
  if (!gb200::read_jpeg(jpeg_in, jpeg_len, &jpg, &err)) {
    g_err = err;
    return 0;
  }
  dims[0] = jpg.width;
  dims[1] = jpg.height;
  dims[2] = static_cast<int>(jpg.components.size());
  size_t pos = 0;
  for (size_t c = 0; c < jpg.components.size(); ++c) {
    dims[3 + 2 * c] = jpg.components[c].width_in_blocks;
    dims[4 + 2 * c] = jpg.components[c].height_in_blocks;
    for (size_t i = 0; i < jpg.components[c].coeffs.size(); ++i, ++pos)
      if (pos < out_cap) out[pos] = jpg.components[c].coeffs[i];
  }
  return pos <= out_cap ? 1 : 0;
}

int gb200_image_process(gb200_image* img, const gb200_params* params, gb200_log_fn log, void* log_user,
                        uint8_t** out, size_t* out_len, gb200_stats* stats) {
  *out = nullptr;
  *out_len = 0;
  bool ok = false;
  int guarded_ok = guarded([&]() {
    gb200::SearchParams sp = to_search_params(params);
    gb200::SearchStats st;
    std::string jpeg, err;
    ok = gb200::process_resident(sp, img->ctx, log, log_user, &jpeg, &st, &err);
    if (!ok) g_err = err;
    if (!jpeg.empty()) {
      *out = static_cast<uint8_t*>(malloc(jpeg.size()));
      memcpy(*out, jpeg.data(), jpeg.size());
      *out_len = jpeg.size();
    }
    fill_stats(st, stats);
  });
  return (guarded_ok && ok) ? 1 : 0;
}

// ---- row-strip mode -------------------------------------------------------
namespace {
gb200::Comm* g_comm = nullptr;
int g_comm_device = 0;
}  // namespace

int gb200_dist_unique_id(uint8_t* out128) {
#if defined(GB200_HOSTSIM)
  (void)out128;
  g_err = "the CPU port has no NCCL";
  return 0;
#else
  return guarded([&]() { gb200::nccl_unique_id(out128); });
#endif
}

int gb200_dist_init(const uint8_t* id128, int rank, int world, int device) {
#if defined(GB200_HOSTSIM)
  (void)id128; (void)rank; (void)world; (void)device;
  g_err = "the CPU port has no NCCL";
  return 0;
#else
  return guarded([&]() {
    gb200::select_device(device);
    delete g_comm;
    g_comm = gb200::nccl_comm_create(id128, rank, world);
    g_comm_device = device;
  });
#endif
}

void gb200_dist_shutdown(void) {
  guarded([&]() {
    delete g_comm;
    g_comm = nullptr;
  });
}

int gb200_process_rgb_tiled(const gb200_params* params, const uint8_t* rgb, int w, int h, gb200_log_fn log,
                            void* log_user, uint8_t** out, size_t* out_len, gb200_stats* stats) {
  *out = nullptr;
  *out_len = 0;
  bool ok = false;
  int guarded_ok = guarded([&]() {
    if (!g_comm) throw std::runtime_error("gb200_dist_init has not been called");
    gb200::SearchParams sp = to_search_params(params);
    gb200::SearchStats st;
    std::string jpeg, err;
    ok = gb200::process_rgb_tiled(sp, rgb, w, h, g_comm_device, g_comm, log, log_user, &jpeg, &st, &err);
    if (!ok) g_err = err;
    if (!jpeg.empty()) {
      *out = static_cast<uint8_t*>(malloc(jpeg.size()));
      memcpy(*out, jpeg.data(), jpeg.size());
      *out_len = jpeg.size();
    }
    fill_stats(st, stats);
  });
  return (guarded_ok && ok) ? 1 : 0;
}

// The same strip decomposition with `world` host threads of this process sharing one
// device (test entry: exercises the strip kernels and the exchange without NCCL).
int gb200_process_rgb_tiled_threads(const gb200_params* params, const uint8_t* rgb, int w, int h, int device,
                                    int world, uint8_t** out, size_t* out_len, gb200_stats* stats) {
  *out = nullptr;
  *out_len = 0;
  bool all_ok = true;
  int guarded_ok = guarded([&]() {
    if (world < 1 || world > 64) throw std::runtime_error("bad world size");
    gb200::ThreadGroup* group = gb200::thread_group_create(world);
    std::vector<std::string> jpegs(world), errs(world);
    std::vector<gb200::SearchStats> sts(world);
    std::vector<int> oks(world, 0);
    std::vector<std::string> what(world);
    std::vector<std::thread> threads;
    gb200::SearchParams sp = to_search_params(params);
    for (int r = 0; r < world; ++r) {
      threads.emplace_back([&, r]() {
        gb200::Comm* comm = gb200::thread_comm_create(group, r);
        try {
          oks[r] = gb200::process_rgb_tiled(sp, rgb, w, h, device, comm, nullptr, nullptr, &jpegs[r], &sts[r], &errs[r]);
        } catch (const std::exception& e) {
          what[r] = e.what();
          oks[r] = -1;
          gb200::thread_group_abort(group);  // the other ranks leave their barriers with an error
        }
        delete comm;
      });
    }
    for (auto& t : threads) t.join();
    gb200::thread_group_destroy(group);
    for (int r = 0; r < world; ++r) {
      if (oks[r] < 0) throw std::runtime_error("rank " + std::to_string(r) + ": " + what[r]);
      if (!oks[r]) {
        all_ok = false;
        g_err = errs[r];
      }
      if (jpegs[r] != jpegs[0]) throw std::runtime_error("ranks disagree on the output");
    }
    if (!jpegs[0].empty()) {
      *out = static_cast<uint8_t*>(malloc(jpegs[0].size()));
      memcpy(*out, jpegs[0].data(), jpegs[0].size());
      *out_len = jpegs[0].size();
    }
    fill_stats(sts[0], stats);
  });
  return (guarded_ok && all_ok) ? 1 : 0;
}

void gb200_free(void* p) { free(p); }
const char* gb200_last_error(void) { return g_err.c_str(); }
const char* gb200_backend_name(void) { return gb200::backend_name(); }

int gb200_device_count(void) {
#if defined(GB200_HOSTSIM)
  return 1;
#else
  return gb200::cuda_device_count();
#endif
}

gb200_image* gb200_image_create(const uint8_t* rgb, int w, int h, int device) {
  return gb200_image_create2(rgb, w, h, device, 1);
}

gb200_image* gb200_image_create2(const uint8_t* rgb, int w, int h, int device, int prepare) {
  gb200_image* img = nullptr;
  guarded([&]() {
    if (!rgb || w <= 0 || h <= 0 || w >= 65536 || h >= 65536) throw std::runtime_error("bad image size");
    std::string why;
    if (!gb200::image_size_supported(w, h, &why)) throw std::runtime_error(why);
    gb200::ImageContext* ctx = new gb200::ImageContext(rgb, w, h, device, prepare != 0);
    img = new gb200_image;
    img->ctx = ctx;
  });
  return img;
}

namespace {
// a resident image from an 8-bit view: create2's checks and messages, then the view's
gb200_image* image_from_view(const uint8_t* data, int w, int h, int channels, const int64_t* strides, int device,
                             int prepare, bool on_device, void* stream) {
  gb200_image* img = nullptr;
  guarded([&]() {
    if (on_device) {
      const void* ptrs[1] = {data};
      const char* what[1] = {"img"};
      check_device_pointers("image_create_device", device, ptrs, what, 1);
    }
    if (!data || w <= 0 || h <= 0 || w >= 65536 || h >= 65536) throw std::runtime_error("bad image size");
    std::string why;
    gb200::ImageView view;
    if (!gb200::image_view(data, w, channels, strides, &view, &why)) throw std::runtime_error(why);
    if (!gb200::image_size_supported(w, h, &why)) throw std::runtime_error(why);
    view.device = on_device;
    view.stream = caller_stream(stream);
    gb200::ImageContext* ctx = new gb200::ImageContext(view, w, h, device, prepare != 0);
    img = new gb200_image;
    img->ctx = ctx;
  });
  return img;
}
}  // namespace

gb200_image* gb200_image_create_strided(const uint8_t* img, int w, int h, int channels, const int64_t* strides,
                                        int device, int prepare) {
  return image_from_view(img, w, h, channels, strides, device, prepare, false, nullptr);
}

gb200_image* gb200_image_create_device(const uint8_t* img_dev, int w, int h, int channels, const int64_t* strides,
                                       int device, int prepare, void* stream) {
  return image_from_view(img_dev, w, h, channels, strides, device, prepare, true, stream);
}

int gb200_image_rgb(gb200_image* img, uint8_t* out) {
  return guarded([&]() { img->ctx->download_rgb(out); });
}

void gb200_image_destroy(gb200_image* img) {
  if (!img) return;
  guarded([&]() { img->ctx->bind(); delete img->ctx; });
  delete img;
}

int gb200_image_reset(gb200_image* img) {
  return guarded([&]() { img->ctx->reset_prepared(); });
}

int gb200_image_num_blocks(const gb200_image* img) { return img->ctx->geom().nblocks; }

int gb200_image_orig_coeffs(gb200_image* img, int16_t* out) {
  return guarded([&]() {
    img->ctx->bind();
    const std::vector<int16_t>& c = img->ctx->orig_coeffs();
    memcpy(out, c.data(), c.size() * sizeof(int16_t));
  });
}

int gb200_image_apply_global_quant(gb200_image* img, const int* q) {
  return guarded([&]() { img->ctx->bind(); img->ctx->apply_global_quant(q); });
}
int gb200_image_upload_candidate(gb200_image* img, const int16_t* coeffs) {
  return guarded([&]() { img->ctx->bind(); img->ctx->upload_candidate(coeffs); });
}
int gb200_image_download_candidate(gb200_image* img, int16_t* coeffs) {
  return guarded([&]() { img->ctx->bind(); img->ctx->download_candidate(coeffs); });
}
int gb200_image_scatter(gb200_image* img, const int* index, const int16_t* value, int n) {
  return guarded([&]() {
    img->ctx->bind();
    img->ctx->scatter_coeffs(std::vector<int>(index, index + n), std::vector<int16_t>(value, value + n));
  });
}
int gb200_image_compare(gb200_image* img, float* distance) {
  return guarded([&]() { *distance = img->ctx->compare(); });
}
int gb200_image_distmap(gb200_image* img, float* out) {
  return guarded([&]() { img->ctx->bind(); img->ctx->download_distmap(out); });
}
int gb200_image_block_weights(gb200_image* img, int direction, int radius, double target_distance,
                              int zero_distmap, float* out) {
  return guarded([&]() { img->ctx->bind(); img->ctx->block_weights(direction, radius, target_distance, zero_distmap != 0, out); });
}
int gb200_image_zeroing_orders(gb200_image* img, float block_error_limit, int lookahead, uint8_t* idx,
                               float* err, int* count) {
  return guarded([&]() {
    std::vector<uint8_t> vi;
    std::vector<float> ve;
    std::vector<int> vc;
    img->ctx->bind();
    img->ctx->zeroing_orders(block_error_limit, lookahead, true, &vi, &ve, &vc);
    memcpy(idx, vi.data(), vi.size());
    memcpy(err, ve.data(), ve.size() * sizeof(float));
    memcpy(count, vc.data(), vc.size() * sizeof(int));
  });
}
int gb200_image_debug_blur(gb200_image* img, const float* in, float* out, int blur_id) {
  return guarded([&]() { img->ctx->bind(); img->ctx->debug_blur(in, out, blur_id); });
}
int gb200_image_debug_opsin(gb200_image* img, const float* rgb_linear, float* xyb) {
  return guarded([&]() { img->ctx->bind(); img->ctx->debug_opsin(rgb_linear, xyb); });
}
int gb200_image_debug_separate(gb200_image* img, const float* xyb, float* psycho10) {
  return guarded([&]() { img->ctx->bind(); img->ctx->debug_separate(xyb, psycho10); });
}
int gb200_image_debug_render(gb200_image* img, float* linear_rgb) {
  return guarded([&]() { img->ctx->bind(); img->ctx->debug_render(linear_rgb); });
}
int gb200_image_debug_psycho0(gb200_image* img, float* psycho10) {
  return guarded([&]() { img->ctx->bind(); img->ctx->debug_psycho0(psycho10); });
}
int gb200_image_debug_corner_mask(gb200_image* img, float* out) {
  return guarded([&]() { img->ctx->bind(); img->ctx->debug_corner_mask(out); });
}

int gb200_write_jpeg(const int16_t* coeffs, int w, int h, const int* q, uint8_t** out, size_t* out_len) {
  return guarded([&]() {
    gb200::CoeffImage ci;
    ci.w = w;
    ci.h = h;
    ci.bw = (w + 7) / 8;
    ci.bh = (h + 7) / 8;
    ci.nblocks = ci.bw * ci.bh;
    ci.coeffs = coeffs;
    memcpy(ci.q, q, sizeof(ci.q));
    std::string s = gb200::write_jpeg(ci);
    *out = static_cast<uint8_t*>(malloc(s.size() + 1));
    memcpy(*out, s.data(), s.size());
    *out_len = s.size();
  });
}

int gb200_image_save_jpeg(gb200_image* img, const int* q, uint8_t** out, size_t* out_len) {
  return guarded([&]() {
    img->ctx->bind();
    std::string s;
    gb200::device_save_jpeg(img->ctx, q, &s);
    *out = static_cast<uint8_t*>(malloc(s.size() + 1));
    memcpy(*out, s.data(), s.size());
    *out_len = s.size();
  });
}

// test hooks for the prefix-exact std::sort replay (exact_sort.h)
size_t gb200_debug_partial_sort(int* block, float* key, size_t n, size_t want) {
  std::vector<gb200::exact_sort::Item> v(n);
  for (size_t i = 0; i < n; ++i) v[i] = std::make_pair(block[i], key[i]);
  const size_t k = gb200::exact_sort::partial_std_sort(v.data(), n, want);
  for (size_t i = 0; i < n; ++i) {
    block[i] = v[i].first;
    key[i] = v[i].second;
  }
  return k;
}
// the same replay with the large partition passes on the device (order_exact.h); needs an image
// context only for its stream and scratch
size_t gb200_debug_device_partial_sort(gb200_image* img, int* block, float* key, size_t n, size_t want) {
  size_t k = 0;
  guarded([&]() {
    std::vector<gb200::exact_sort::Item> v(n);
    for (size_t i = 0; i < n; ++i) v[i] = std::make_pair(block[i], key[i]);
    k = img->ctx->debug_device_partial_sort(v.data(), n, want);
    for (size_t i = 0; i < k; ++i) {
      block[i] = v[i].first;
      key[i] = v[i].second;
    }
  });
  return k;
}
void gb200_debug_std_sort(int* block, float* key, size_t n) {
  std::vector<std::pair<int, float> > v(n);
  for (size_t i = 0; i < n; ++i) v[i] = std::make_pair(block[i], key[i]);
  std::sort(v.begin(), v.end(),
            [](const std::pair<int, float>& a, const std::pair<int, float>& b) { return a.second < b.second; });
  for (size_t i = 0; i < n; ++i) {
    block[i] = v[i].first;
    key[i] = v[i].second;
  }
}

void gb200_debug_huffman_depths(const uint32_t* counts, int n, int limit, uint8_t* depth) {
  gb200::huffman_code_lengths(counts, n, limit, depth);
}

void gb200_trim_memory(void) {
#if !defined(GB200_HOSTSIM)
  guarded([&]() { gb200::dev_trim(); });
#endif
}

void gb200_counters(long* launches, long long* h2d_bytes, long long* d2h_bytes) {
  if (launches) *launches = gb200::total_launches();
  if (h2d_bytes) *h2d_bytes = gb200::h2d_bytes_total();
  if (d2h_bytes) *d2h_bytes = gb200::d2h_bytes_total();
}

void gb200_profile_enable(int on) { gb200::profiling_enable(on != 0); }
void gb200_profile_reset(void) { gb200::profiling_reset(); }
int gb200_profile_get(char (*names)[48], long* launches, double* ms, double* elements, int cap) {
  std::vector<gb200::KernelStat> s = gb200::profiling_snapshot();
  const int n = static_cast<int>(s.size());
  for (int i = 0; i < n && i < cap; ++i) {
    strncpy(names[i], s[i].name.c_str(), 47);
    names[i][47] = 0;
    launches[i] = s[i].launches;
    ms[i] = s[i].ms;
    elements[i] = s[i].elements;
  }
  return n;
}

}  // extern "C"
