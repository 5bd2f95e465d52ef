// The butteraugli metric (see butteraugli.h): its planes, their layout, its lifetime and its entry
// points.  The members that launch kernels are in pipeline.cu, which compiles every kernel of the
// library into one device module.  Compiled by nvcc for sm_90a in the product, and by g++
// -DGB200_HOSTSIM for the CPU port.
#include "butteraugli.h"

#include <string.h>

#include <algorithm>
#include <stdexcept>

namespace gb200 {

#if defined(GB200_HOSTSIM)
void Butteraugli::fused_sup0(int, int) {}
void Butteraugli::mixed_release() {}
#endif

void Region::gather_blocks(void* dev_buf, size_t elem_bytes_per_block) const {
  if (!strips()) return;
  const int W = comm->world();
  std::vector<size_t> off(W), cnt(W);
  for (int r = 0; r < W; ++r) {
    int lo, hi;
    strip_of(g.bh, r, W, &lo, &hi);
    off[r] = static_cast<size_t>(lo) * g.bw;
    cnt[r] = static_cast<size_t>(hi - lo) * g.bw;
  }
  comm->allgather_inplace(dev_buf, elem_bytes_per_block, off, cnt, s);
}

void Region::download_planes(const float* src, float* packed, int n) const {
  std::vector<float> buf(g.plane * n);
  d2h(buf.data(), src, sizeof(float) * g.plane * n, s);
  for (int c = 0; c < n; ++c)
    for (int y = 0; y < g.h; ++y)
      memcpy(packed + (static_cast<size_t>(c) * g.h + y) * g.w, &buf[c * g.plane + static_cast<size_t>(y) * g.pitch],
             sizeof(float) * g.w);
}

void Region::upload_planes(const float* packed, float* dst, int n) const {
  std::vector<float> buf(g.plane * n, 0.0f);
  for (int c = 0; c < n; ++c)
    for (int y = 0; y < g.h; ++y)
      memcpy(&buf[c * g.plane + static_cast<size_t>(y) * g.pitch], packed + (static_cast<size_t>(c) * g.h + y) * g.w,
             sizeof(float) * g.w);
  h2d(dst, buf.data(), sizeof(float) * g.plane * n, s);
  stream_sync(s);
}

Butteraugli::Butteraugli(int w, int h, int device, Comm* comm) : device_(device) { init(w, h, comm); }

Butteraugli::Butteraugli(int w, int h, int capacity, int device, Slots slots) : device_(device) {
  if (capacity < 1) throw std::runtime_error("butteraugli batch: the capacity must be at least 1");
  capacity_ = capacity;
  if (slots == Slots::kPairs) {
    kslot_ = kBatchSlotPlanes;
  } else if (capacity > 1) {  // capacity 1: the single-image layout
    one_original_ = true;
    kslot_ = kCandidateSlotPlanes;
  }
  init(w, h, nullptr);
}

// A constructor that throws never reaches the destructor: everything acquired so far (device
// buffers of owned_, the stream) is handed back here, so that an out-of-memory condition does not
// become permanent for the process.
void Butteraugli::init(int w, int h, Comm* comm) {
  r_.g = make_geom(w, h);
  r_.comm = comm;
  r_.by_lo = 0;
  r_.by_hi = g_.bh;
  if (r_.strips()) strip_of(g_.bh, comm->rank(), comm->world(), &r_.by_lo, &r_.by_hi);
  // rows whose distmap this rank must produce, widened by the metric's receptive field
  r_.cr_lo = std::max(0, 8 * r_.by_lo - 56);
  r_.cr_hi = std::min(g_.h, 8 * r_.by_hi + 56);
  try {
    select_device(device_);
    r_.s = make_stream();
    have_stream_ = true;
#if defined(GB200_HOSTSIM)
    // the CPU port has no batched launches: compare_many scores the candidates one by one on a
    // single-image layout, compare_batch the pairs through metrics of their own
    if (one_original_) kslot_ = 0;
    if (kslot_ != 0) return;
#endif
    t_ = build_tables(w, h, s_, &owned_, &ht_);
    malta_call_params(malta_);
    l2_asym_weights(&asym_w0_, &asym_w1_);
#if !defined(GB200_HOSTSIM)
    fused_ = new Fused();
    fused_->capacity = capacity_;
#endif
    alloc_planes();
    stream_sync(s_);
  } catch (...) {
    release();
    throw;
  }
}

float* Butteraugli::planes(size_t n) {
  void* p = dev_alloc(sizeof(float) * g_.plane * n);
  owned_.push_back(p);
  dev_zero(p, sizeof(float) * g_.plane * n, s_);
  return static_cast<float*>(p);
}

// The plane groups of all three shapes.  They lie in one arena of `slots` slots, each group at the
// same offset in every slot, so that slot n's copy of a group is the group plus n slots.  A batch
// slot holds only what the analysis of an original and the fused chain touch (DESIGN.md §4); the
// slot of one image adds the mask activity and, in the CPU port, the planes its chain blurs into.
// With one original for all slots, the original's groups lie once after the slots, with the planes
// of its mask activity (mask()), and a slot holds the rest.
void Butteraugli::alloc_planes() {
  struct Group {
    float** p;
    int single, batch;  // planes in the slot of one image / of a batch
    bool orig;          // the original's: outside the slots when they share one original
  };
#if defined(GB200_HOSTSIM)
  constexpr int kPort = 1;
#else
  constexpr int kPort = 0;
#endif
  const Group groups[] = {
      {&lin_, 3, 3, false},    {&xyb_, 3, 3, false},  {&lf_, 3, 3, false},  {&mf_in_, 3, 3, false},
      {&hf_raw_, 2, 2, false}, {&ps0_, kPsychoPlanes, kPsychoPlanes, true}, {&ps1_, kPsychoPlanes, kPsychoPlanes, false},
      {&sup0_, 2, 2, true},    {&diffs6_, 6, 6, false}, {&noise_, 1 + kPort, 1, false}, {&mpre_, 2, 2, false},
      {&tmp_, 3, 3, false},    {&blr_, 1 + 2 * kPort, 1, false}, {&ac_, 2, 2, false},  {&dm_, 2, 2, false},
      // the CPU port's blurred planes and the mask activity
      {&mf_blr_, 3 * kPort, 0, false}, {&hf_blr_, 2 * kPort, 0, false}, {&diffs_, kPort, 0, false},
      {&sact_, 3, 0, true}};
  const bool shared = one_original_ && kslot_ != 0;
  const int slots = kslot_ ? capacity_ : 1;
  int slot = 0, once = 0;
  for (const Group& gr : groups) {
    if (shared && gr.orig) {
      once += gr.single;
    } else {
      slot += kslot_ ? gr.batch : gr.single;
    }
  }
  if (kslot_ != 0 && slot != kslot_) throw std::logic_error("butteraugli batch: slot layout");
  float* a = planes(static_cast<size_t>(slot) * slots + once);
  int at = 0, at_once = slot * slots;
  for (const Group& gr : groups) {
    int& pos = shared && gr.orig ? at_once : at;
    const int n = shared && gr.orig ? gr.single : kslot_ ? gr.batch : gr.single;
    *gr.p = n ? a + static_cast<size_t>(pos) * g_.plane : nullptr;
    pos += n;
  }
  block_max_ = static_cast<float*>(dev_alloc(sizeof(float) * g_.nblocks * slots));
  owned_.push_back(block_max_);
  d_gmax_ = static_cast<unsigned int*>(dev_alloc(sizeof(unsigned int) * slots));
  owned_.push_back(d_gmax_);
  partial_ = static_cast<float*>(dev_alloc(sizeof(float) * 1024));
  owned_.push_back(partial_);
}

Butteraugli::~Butteraugli() { release(); }

void Butteraugli::release() {
  try {
    select_device(device_);
    if (have_stream_) stream_sync(s_);
  } catch (...) {
    // a failed device cannot be waited for; the blocks still go back to the cache
  }
  for (size_t i = 0; i < owned_.size(); ++i) dev_free(owned_[i]);
  owned_.clear();
  mixed_release();
#if !defined(GB200_HOSTSIM)
  delete fused_;
  fused_ = nullptr;
#endif
  if (have_stream_) destroy_stream(s_);
  have_stream_ = false;
}

void Butteraugli::lin_from_device(const float* linear_rgb, Stream caller) {
  const size_t row = sizeof(float) * g_.w, pitch = sizeof(float) * g_.pitch;
  stream_wait(s_, caller);
  // [3][h][w] -> [3][h][pitch]: a plane is h rows of pitch, so the three planes are 3h rows
  d2d_2d(lin_, pitch, linear_rgb, row, row, static_cast<size_t>(3) * g_.h, s_);
}

void Butteraugli::analyse_original(const float* linear_rgb, bool device, Stream caller) {
  if (linear_rgb != nullptr) {
    if (device) {
      lin_from_device(linear_rgb, caller);
    } else {
      r_.upload_planes(linear_rgb, lin_, 3);
    }
  }
  opsin(lin_, xyb_);
  separate(xyb_, ps0_);
  fused_sup0(1, 0);
  if (linear_rgb != nullptr) stream_sync(s_);  // a comparator is ready when its constructor returns
}

float Butteraugli::compare_linear(const float* linear_rgb) {
  bind();
  r_.upload_planes(linear_rgb, lin_, 3);
  return compare();
}

float Butteraugli::compare_linear_device(const float* linear_rgb, float* diffmap, Stream caller) {
  bind();
  lin_from_device(linear_rgb, caller);
  const float m = compare();
  if (diffmap != nullptr) {
    const size_t row = sizeof(float) * g_.w, pitch = sizeof(float) * g_.pitch;
    d2d_2d(diffmap, row, dm_, pitch, row, g_.h, s_);
    stream_sync(s_);
  }
  return m;
}

void Butteraugli::compare_batch(const float* rgb0, const float* rgb1, int n, float* diffmap, float* maxima, bool device,
                                Stream caller) {
  if (n < 1 || n > capacity_) throw std::runtime_error("butteraugli batch: n must be in 1..capacity");
  bind();
#if !defined(GB200_HOSTSIM)
  if (device) stream_wait(s_, caller);
  fused_compare_batch(rgb0, rgb1, n, diffmap, maxima);
#else
  // the CPU port: compare_batch_sizes with every pair at this batch's size
  const size_t img = static_cast<size_t>(3) * g_.w * g_.h, px = static_cast<size_t>(g_.w) * g_.h;
  const std::vector<int> w(n, g_.w), h(n, g_.h);
  std::vector<const float*> p0(n), p1(n);
  std::vector<float*> dm(n);
  for (int i = 0; i < n; ++i) {
    p0[i] = rgb0 + i * img;
    p1[i] = rgb1 + i * img;
    dm[i] = diffmap != nullptr ? diffmap + i * px : nullptr;
  }
  compare_batch_sizes(w.data(), h.data(), p0.data(), p1.data(), n, dm.data(), maxima, device, caller);
#endif
}

void Butteraugli::check_sizes(const int* w, const int* h, int n) const {
  if (n < 1 || n > capacity_) throw std::runtime_error("butteraugli batch: n must be in 1..capacity");
  for (int i = 0; i < n; ++i)
    if (w[i] < 8 || h[i] < 8 || w[i] > g_.w || h[i] > g_.h) throw std::runtime_error("butteraugli batch: pair size");
}

void Butteraugli::compare_batch_sizes(const int* w, const int* h, const float* const* rgb0, const float* const* rgb1,
                                      int n, float* const* diffmap, float* maxima, bool device, Stream caller) {
  check_sizes(w, h, n);
  bind();
#if !defined(GB200_HOSTSIM)
  if (device) stream_wait(s_, caller);
  const std::vector<const void*> in0(rgb0, rgb0 + n), in1(rgb1, rgb1 + n);
  fused_compare_sizes(w, h, nullptr, in0.data(), in1.data(), n, diffmap, maxima, device);
#else
  // the CPU port (host memory only): one single-image metric per pair, of the pair's size
  for (int i = 0; i < n; ++i) {
    Butteraugli pair(w[i], h[i], device_, nullptr);
    pair.analyse_original(rgb0[i]);
    maxima[i] = pair.compare_linear(rgb1[i]);
    if (diffmap != nullptr && diffmap[i] != nullptr) pair.download_distmap(diffmap[i]);
  }
#endif
}

void Butteraugli::compare_many(const float* rgb1, int n, float* diffmap, float* maxima, bool device, Stream caller) {
  if (n < 1 || n > capacity_) throw std::runtime_error("butteraugli comparator: n must be in 1..capacity");
  bind();
#if !defined(GB200_HOSTSIM)
  if (kslot_ != 0) {
    if (device) stream_wait(s_, caller);
    fused_compare_batch(nullptr, rgb1, n, diffmap, maxima);
    return;
  }
#endif
  // capacity 1 and the CPU port: one candidate at a time in slot 0
  const size_t img = static_cast<size_t>(3) * g_.w * g_.h, px = static_cast<size_t>(g_.w) * g_.h;
  for (int i = 0; i < n; ++i) {
    float* dm = diffmap != nullptr ? diffmap + i * px : nullptr;
    if (device) {
      maxima[i] = compare_linear_device(rgb1 + i * img, dm, caller);
    } else {
      maxima[i] = compare_linear(rgb1 + i * img);
      if (dm != nullptr) download_distmap(dm);
    }
  }
}

// ---- 8-bit sRGB input (butteraugli.h) ----
namespace {
// The converted planes are handed to the float entries as device memory.  The CPU port has no device
// memory (its dev_alloc is host memory, and its device entries refuse), so there they go in as host
// memory.
#if defined(GB200_HOSTSIM)
constexpr bool kScratchOnDevice = false;
#else
constexpr bool kScratchOnDevice = true;
#endif

void check_channels(int channels) {
  if (channels != 3 && channels != 4)
    throw std::runtime_error("butteraugli: channels = " + std::to_string(channels) +
                             ", 8-bit images must have 3 (RGB) or 4 (RGBA)");
}
}  // namespace

void Butteraugli::srgb_alloc(int per_slot) {
  if (srgb_lin_ != nullptr) return;
  // the CPU port's pair batch builds no tables of its own (its pairs go through metrics of their own);
  // the conversion needs only the sRGB table
  if (t_.srgb_lin == nullptr) t_.srgb_lin = upload_srgb_lin(s_, &owned_, nullptr);
  const size_t px = static_cast<size_t>(g_.w) * g_.h, imgs = static_cast<size_t>(per_slot) * capacity_;
  srgb_u8_ = static_cast<uint8_t*>(dev_alloc(4 * px * imgs));
  owned_.push_back(srgb_u8_);
  srgb_lin_ = static_cast<float*>(dev_alloc(sizeof(float) * 3 * px * imgs));
  owned_.push_back(srgb_lin_);
  for (float*& dm : srgb_dm_) {
    dm = static_cast<float*>(dev_alloc(sizeof(float) * px * capacity_));
    owned_.push_back(dm);
  }
}

template <class Score>
void Butteraugli::srgb_backgrounds(int n, int channels, int only, float* diffmap, float* maxima, bool device,
                                   const Score& score) {
  const size_t px = static_cast<size_t>(g_.w) * g_.h;
  const bool both = channels == 4 && only < 0;
  float* dm = diffmap == nullptr ? nullptr : device ? diffmap : srgb_dm_[0];
  score(only < 0 ? 0 : only, dm, maxima);
  if (both) {
    std::vector<float> white(n);
    score(255, dm != nullptr ? srgb_dm_[1] : nullptr, white.data());
    for (int i = 0; i < n; ++i) {
      if (!white_wins(white[i], maxima[i])) continue;
      maxima[i] = white[i];
      if (dm != nullptr) d2d(dm + i * px, srgb_dm_[1] + i * px, sizeof(float) * px, s_);
    }
  }
  if (dm != nullptr && !device) {
    d2h(diffmap, dm, sizeof(float) * px * n, s_);
  } else if (both) {
    stream_sync(s_);  // the white diffmaps copied into the caller's memory
  }
}

void Butteraugli::analyse_original_srgb(const uint8_t* img0, int channels, int background, bool device,
                                        Stream caller) {
  check_channels(channels);
  bind();
  if (device) {  // converted where it lies
    stream_wait(s_, caller);
    srgb_to_linear(img0, 1, channels, background, lin_, g_.pitch);
    analyse_original();
    stream_sync(s_);
    return;
  }
  const size_t bytes = static_cast<size_t>(g_.w) * g_.h * channels;
  uint8_t* u8 = static_cast<uint8_t*>(dev_alloc(bytes));
  try {
    h2d(u8, img0, bytes, s_);
    srgb_to_linear(u8, 1, channels, background, lin_, g_.pitch);
    analyse_original();
    stream_sync(s_);
  } catch (...) {
    dev_free(u8);
    throw;
  }
  dev_free(u8);
}

void Butteraugli::compare_batch_srgb(const uint8_t* img0, const uint8_t* img1, int n, int channels, float* diffmap,
                                     float* maxima, bool device, Stream caller, int background) {
  if (n < 1 || n > capacity_) throw std::runtime_error("butteraugli batch: n must be in 1..capacity");
  check_channels(channels);
  if (background != -1 && background != 0 && background != 255)
    throw std::logic_error("butteraugli batch: the background must be 0 or 255");
  bind();
  srgb_alloc(2);
  const size_t bytes = static_cast<size_t>(g_.w) * g_.h * channels * n;
  const size_t half = static_cast<size_t>(g_.w) * g_.h * capacity_;  // images of one side
  const uint8_t* in0 = img0;
  const uint8_t* in1 = img1;
  if (device) {
    stream_wait(s_, caller);
  } else {  // one upload of each side
    h2d(srgb_u8_, img0, bytes, s_);
    h2d(srgb_u8_ + 4 * half, img1, bytes, s_);
    in0 = srgb_u8_;
    in1 = srgb_u8_ + 4 * half;
  }
  float* lin0 = srgb_lin_;
  float* lin1 = srgb_lin_ + 3 * half;
  srgb_backgrounds(n, channels, background, diffmap, maxima, device, [&](int bg, float* dm, float* m) {
    srgb_to_linear(in0, n, channels, bg, lin0, g_.w);
    srgb_to_linear(in1, n, channels, bg, lin1, g_.w);
    compare_batch(lin0, lin1, n, dm, m, kScratchOnDevice, s_);
  });
}

void Butteraugli::compare_many_srgb(const uint8_t* img1, int n, int channels, Butteraugli* white, float* diffmap,
                                    float* maxima, bool device, Stream caller) {
  if (n < 1 || n > capacity_) throw std::runtime_error("butteraugli comparator: n must be in 1..capacity");
  check_channels(channels);
  if (channels == 4 && white == nullptr) throw std::logic_error("butteraugli comparator: RGBA needs the original over white");
  bind();
  srgb_alloc(1);
  const uint8_t* in = img1;
  if (device) {
    stream_wait(s_, caller);
  } else {
    h2d(srgb_u8_, img1, static_cast<size_t>(g_.w) * g_.h * channels * n, s_);
    in = srgb_u8_;
  }
  srgb_backgrounds(n, channels, -1, diffmap, maxima, device, [&](int background, float* dm, float* m) {
    srgb_to_linear(in, n, channels, background, srgb_lin_, g_.w);
    (background == 0 ? this : white)->compare_many(srgb_lin_, n, dm, m, kScratchOnDevice, s_);
  });
}

void Butteraugli::compare_batch_sizes_srgb(const int* w, const int* h, const int* channels,
                                           const uint8_t* const* img0, const uint8_t* const* img1, int n,
                                           float* const* diffmap, float* maxima, bool device, Stream caller) {
  check_sizes(w, h, n);
  for (int i = 0; i < n; ++i) check_channels(channels[i]);
  bind();
#if !defined(GB200_HOSTSIM)
  if (device) stream_wait(s_, caller);
  const std::vector<const void*> in0(img0, img0 + n), in1(img1, img1 + n);
  fused_compare_sizes(w, h, channels, in0.data(), in1.data(), n, diffmap, maxima, device);
#else
  // the CPU port: one pair batch per pair, of the pair's size
  for (int i = 0; i < n; ++i) {
    Butteraugli pair(w[i], h[i], 1, device_, Slots::kPairs);
    pair.compare_batch_srgb(img0[i], img1[i], 1, channels[i], diffmap != nullptr ? diffmap[i] : nullptr, &maxima[i],
                            device, caller);
  }
#endif
}

// ---- comparator sets (butteraugli.h) ----
ComparatorSet::ComparatorSet(const int* w, const int* h, const int* channels, const void* const* img0, int count,
                             int capacity, int device, bool on_device, Stream caller)
    : w_(w, w + count), h_(h, h + count) {
  if (channels != nullptr) {
    channels_.assign(channels, channels + count);
    for (int c : channels_) check_channels(c);
  }
  ba_.reset(new Butteraugli(*std::max_element(w_.begin(), w_.end()), *std::max_element(h_.begin(), h_.end()),
                            capacity, device, Butteraugli::Slots::kPairs));
#if defined(GB200_HOSTSIM)
  if (on_device) throw std::runtime_error("the CPU port has no device memory");
  for (int i = 0; i < count; ++i) {
    const size_t in = static_cast<size_t>(w[i]) * h[i] * (srgb() ? channels[i] : 3 * sizeof(float));
    const unsigned char* p = static_cast<const unsigned char*>(img0[i]);
    host_.emplace_back(p, p + in);
  }
#else
  // the store: each original's analyses, 16-byte aligned
  size_t bytes = 0;
  const auto take = [&](size_t n) {
    const size_t at = bytes;
    bytes = (bytes + n + 15) / 16 * 16;
    return at;
  };
  for (size_t b = 0; b < 2; ++b) at_[b].assign(count, kNone);
  for (int i = 0; i < count; ++i) {
    const size_t px = static_cast<size_t>(w[i]) * h[i];
    at_[0][i] = take(sizeof(float) * kStoredPlanes * px);
    if (srgb() && channels[i] == 4) at_[1][i] = take(sizeof(float) * kStoredPlanes * px);
  }
  ba_->bind();
  store_ = dev_alloc(bytes);
  try {
    if (on_device) stream_wait(ba_->region().s, caller);
    unsigned char* base = static_cast<unsigned char*>(store_);
    // mixed passes of up to `capacity` originals: every original over black, then the RGBA ones over white
    for (int bg = 0; bg < 2; ++bg) {
      std::vector<int> all;
      for (int i = 0; i < count; ++i)
        if (at_[bg][i] != kNone) all.push_back(i);
      for (size_t k = 0; k < all.size(); k += capacity) {
        const size_t m = std::min(all.size() - k, static_cast<size_t>(capacity));
        std::vector<int> cw(m), ch(m), cc(m);
        std::vector<const void*> in(m);
        std::vector<float*> to(m);
        for (size_t j = 0; j < m; ++j) {
          const int i = all[k + j];
          cw[j] = w_[i];
          ch[j] = h_[i];
          cc[j] = srgb() ? channels_[i] : 3;
          in[j] = img0[i];
          to[j] = reinterpret_cast<float*>(base + at_[bg][i]);
        }
        ba_->analyse_originals(cw.data(), ch.data(), srgb() ? cc.data() : nullptr, in.data(), static_cast<int>(m),
                               bg == 0 ? 0 : 255, to.data(), on_device);
      }
    }
  } catch (...) {
    dev_free(store_);
    throw;
  }
#endif
}

ComparatorSet::~ComparatorSet() {
  try {
    ba_->bind();
    stream_sync(ba_->region().s);
  } catch (...) {
    // as in Butteraugli::release: a failed device cannot be waited for
  }
  dev_free(store_);
}

void ComparatorSet::compare(const int* original, const void* const* img1, int n, float* const* diffmap, float* maxima,
                            bool device, Stream caller) {
  std::vector<int> w(n), h(n), ch(n, 3);
  for (int i = 0; i < n; ++i) {
    const int o = original[i];
    w[i] = w_[o];
    h[i] = h_[o];
    if (srgb()) ch[i] = channels_[o];
  }
  const int* channels = srgb() ? ch.data() : nullptr;
#if !defined(GB200_HOSTSIM)
  unsigned char* base = static_cast<unsigned char*>(store_);
  std::vector<float*> stored[2];
  for (int b = 0; b < 2; ++b)
    for (int i = 0; i < n; ++i) {
      const size_t at = at_[b][original[i]];
      stored[b].push_back(at == kNone ? nullptr : reinterpret_cast<float*>(base + at));
    }
  float* const* const st[2] = {stored[0].data(), stored[1].data()};
  ba_->compare_originals(w.data(), h.data(), channels, st, img1, n, diffmap, maxima, device, caller);
#else
  // the CPU port: the pairs (original, candidate)
  std::vector<const unsigned char*> in0(n), in1(n);
  for (int i = 0; i < n; ++i) {
    in0[i] = host_[original[i]].data();
    in1[i] = static_cast<const unsigned char*>(img1[i]);
  }
  if (srgb()) {
    ba_->compare_batch_sizes_srgb(w.data(), h.data(), channels, in0.data(), in1.data(), n, diffmap, maxima, device,
                                  caller);
  } else {
    std::vector<const float*> f0(n), f1(n);
    for (int i = 0; i < n; ++i) {
      f0[i] = reinterpret_cast<const float*>(in0[i]);
      f1[i] = reinterpret_cast<const float*>(in1[i]);
    }
    ba_->compare_batch_sizes(w.data(), h.data(), f0.data(), f1.data(), n, diffmap, maxima, device, caller);
  }
#endif
}

void Butteraugli::adaptive_quantization(const float* linear_rgb, float* quant, bool device, Stream caller) {
  bind();
  if (!device) {
    r_.upload_planes(linear_rgb, lin_, 3);
    mask_planes(lin_);
    r_.download_planes(mask_ + g_.plane, quant, 1);
    return;
  }
  lin_from_device(linear_rgb, caller);
  mask_planes(lin_);
  const size_t row = sizeof(float) * g_.w, pitch = sizeof(float) * g_.pitch;
  d2d_2d(quant, row, mask_ + g_.plane, pitch, row, g_.h, s_);
  stream_sync(s_);
}

void Butteraugli::compare_begin() {
#if !defined(GB200_HOSTSIM)
  compare_pending_ = !r_.strips();
  if (compare_pending_) return fused_compare_submit();
#endif
  compare_stash_ = compare();
}

float Butteraugli::compare_end() {
#if !defined(GB200_HOSTSIM)
  if (compare_pending_) return fused_compare_result();
#endif
  return compare_stash_;
}

void Butteraugli::debug_blur(const float* in, float* out, int id) {
  r_.upload_planes(in, xyb_, 1);
  blur(xyb_, lf_, 1, id);
  r_.download_planes(lf_, out, 1);
}

void Butteraugli::debug_opsin(const float* rgb_lin, float* xyb) {
  r_.upload_planes(rgb_lin, lin_, 3);
  opsin(lin_, xyb_);
  r_.download_planes(xyb_, xyb, 3);
}

void Butteraugli::debug_separate(const float* xyb, float* ps10) {
  r_.upload_planes(xyb, xyb_, 3);
  separate(xyb_, ps1_);
  r_.download_planes(ps1_, ps10, kPsychoPlanes);
}

void Butteraugli::debug_psycho0(float* ps10) { r_.download_planes(ps0_, ps10, kPsychoPlanes); }

}  // namespace gb200
