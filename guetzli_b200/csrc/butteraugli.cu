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

Butteraugli::Butteraugli(int w, int h, int capacity, int device) : device_(device) {
  if (capacity < 1) throw std::runtime_error("butteraugli batch: the capacity must be at least 1");
  capacity_ = capacity;
  kslot_ = kBatchSlotPlanes;
  init(w, h, nullptr);
}

// A constructor that throws never reaches the destructor: everything acquired so far (device
// buffers of owned_, the stream) is handed back here, so that an out-of-memory condition does not
// become permanent for the process.
namespace {
// GB200_COMPARE=staged keeps the round-1 kernel sequence (one kernel per stage) for A/B
// measurements and for the cross-check in tests; default is the fused chain.
bool fused_enabled() {
  const char* e = getenv("GB200_COMPARE");  // read per metric: tests switch it between images
  return !(e != nullptr && e[0] == 's');
}

}  // namespace

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
#if !defined(GB200_HOSTSIM)
    use_fused_ = fused_enabled();
#endif
    if (kslot_ != 0 && !use_fused_) return;  // compare_batch scores the pairs one by one
    t_ = build_tables(w, h, s_, &owned_, &ht_);
    malta_call_params(malta_);
    l2_asym_weights(&asym_w0_, &asym_w1_);
#if !defined(GB200_HOSTSIM)
    if (use_fused_) {
      fused_ = new Fused();
      fused_->capacity = capacity_;
    }
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

// The plane groups of both shapes.  They lie in one arena of capacity_ slots, each group at the
// same offset in every slot, so that slot n's copy of a group is the group plus n slots.  A batch
// slot holds only what the analysis of an original and the fused chain touch (DESIGN.md §4).
void Butteraugli::alloc_planes() {
  struct Group {
    float** p;
    int single, batch;  // planes in the slot of one image / of a batch
  };
  const Group groups[] = {
      {&lin_, 3, 3},    {&xyb_, 3, 3},  {&lf_, 3, 3},  {&mf_in_, 3, 3}, {&hf_raw_, 2, 2},
      {&ps0_, kPsychoPlanes, kPsychoPlanes},          {&ps1_, kPsychoPlanes, kPsychoPlanes},
      {&sup0_, 2, 2},   {&diffs6_, 6, 6}, {&noise_, 2, 1}, {&mpre_, 2, 2}, {&tmp_, 3, 3},
      {&blr_, 3, 1},    {&ac_, 2, 2},   {&dm_, 2, 2},
      // the staged chain's own planes and the mask activity
      {&mf_blr_, 3, 0}, {&hf_blr_, 2, 0}, {&diffs_, 1, 0}, {&sact_, 3, 0}};
  int slot = 0;
  for (const Group& gr : groups) slot += kslot_ ? gr.batch : gr.single;
  if (kslot_ != 0 && slot != kslot_) throw std::logic_error("butteraugli batch: slot layout");
  float* a = planes(static_cast<size_t>(slot) * capacity_);
  int at = 0;
  for (const Group& gr : groups) {
    const int n = kslot_ ? gr.batch : gr.single;
    *gr.p = n ? a + static_cast<size_t>(at) * g_.plane : nullptr;
    at += n;
  }
  block_max_ = static_cast<float*>(dev_alloc(sizeof(float) * g_.nblocks * capacity_));
  owned_.push_back(block_max_);
  d_gmax_ = static_cast<unsigned int*>(dev_alloc(sizeof(unsigned int) * capacity_));
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
#if !defined(GB200_HOSTSIM)
  delete fused_;
  fused_ = nullptr;
#endif
  if (have_stream_) destroy_stream(s_);
  have_stream_ = false;
}

void Butteraugli::analyse_original(const float* linear_rgb) {
  if (linear_rgb != nullptr) r_.upload_planes(linear_rgb, lin_, 3);
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
  const size_t row = sizeof(float) * g_.w, pitch = sizeof(float) * g_.pitch;
  stream_wait(s_, caller);
  // [3][h][w] -> [3][h][pitch]: a plane is h rows of pitch, so the three planes are 3h rows
  d2d_2d(lin_, pitch, linear_rgb, row, row, static_cast<size_t>(3) * g_.h, s_);
  const float m = compare();
  if (diffmap != nullptr) {
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
  if (use_fused_) {
    if (device) stream_wait(s_, caller);
    fused_compare_batch(rgb0, rgb1, n, diffmap, maxima);
    return;
  }
#endif
  // the staged chain and the CPU port: one single-image metric per pair
  const size_t img = static_cast<size_t>(3) * g_.w * g_.h, px = static_cast<size_t>(g_.w) * g_.h;
  std::vector<float> host0;
  for (int i = 0; i < n; ++i) {
    const float* p0 = rgb0 + i * img;
    if (device) {  // the pair's original goes through host memory, after the caller's work
      host0.resize(img);
      d2h(host0.data(), p0, img * sizeof(float), caller);
      p0 = host0.data();
    }
    Butteraugli pair(g_.w, g_.h, device_, nullptr);
    pair.analyse_original(p0);
    float* dm = diffmap != nullptr ? diffmap + i * px : nullptr;
    if (device) {
      maxima[i] = pair.compare_linear_device(rgb1 + i * img, dm, caller);
    } else {
      maxima[i] = pair.compare_linear(rgb1 + i * img);
      if (dm != nullptr) pair.download_distmap(dm);
    }
  }
}

void Butteraugli::adaptive_quantization(const float* linear_rgb, float* quant) {
  bind();
  r_.upload_planes(linear_rgb, lin_, 3);
  mask_planes(lin_);
  r_.download_planes(mask_ + g_.plane, quant, 1);
}

void Butteraugli::compare_begin() {
  compare_pending_ = use_fused_ && !r_.strips();
#if !defined(GB200_HOSTSIM)
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
