// The butteraugli metric on the device: the Compare chain (the TMA-staged fused chain, and the staged
// chain it is checked against), the float planes it works on, and the analysis of the original.
// One Butteraugli scores one image -- the encoder's candidate (ImageContext holds one) or a
// stand-alone comparator's -- or a batch of same-size pairs.  It owns the stream and the tables,
// which the encoder's kernels use as well.  See DESIGN.md §4 and §5.1.
#pragma once
#include <stddef.h>

#include <string>
#include <vector>

#include "comm.h"
#include "kernels.h"
#include "tables.h"
#if defined(__CUDACC__) && !defined(GB200_HOSTSIM)
#include <map>
#include <tuple>

#include "tma.cuh"
#endif

namespace gb200 {

struct KernelStat {
  std::string name;
  long launches;
  double ms;  // CUDA-event time accumulated when profiling is on
  double elements;  // pixels / blocks launched (for algorithmic-bytes rooflines)
};

// Devices, streams and launch accounting (backend_cuda.cu); the CPU port has one device, no
// streams and no counters.
#if defined(GB200_HOSTSIM)
inline void select_device(int) {}
inline Stream make_stream() { return 0; }
inline void destroy_stream(Stream) {}
inline long total_launches() { return 0; }
inline long long h2d_bytes_total() { return 0; }
inline long long d2h_bytes_total() { return 0; }
inline void profiling_enable(bool) {}
inline std::vector<KernelStat> profiling_snapshot() { return std::vector<KernelStat>(); }
inline void profiling_reset() {}
#else
void select_device(int device);
Stream make_stream();
void destroy_stream(Stream s);
long total_launches();
long long h2d_bytes_total();
long long d2h_bytes_total();
void profiling_enable(bool on);
std::vector<KernelStat> profiling_snapshot();
void profiling_reset();
bool profiling_on();
void add_launches(long n);
#endif

namespace {
// Runs a per-pixel functor written for "tall image" row indices (plane * h + y) on
// the rows [y0, y0 + nrows) of each plane only.
template <class F>
struct RowsOf {
  F f;
  int y0, nrows, h;
  GB_HD void operator()(int x, int yy) const {
    const int pl = yy / nrows;
    f(x, pl * h + y0 + (yy - pl * nrows));
  }
};
template <class F>
struct OffsetOf {
  F f;
  int i0;
  GB_HD void operator()(int i) const { f(i0 + i); }
};
}  // namespace

// The part of the image one context computes, and the stream it computes on; the encoder and its
// metric share one.  comm != nullptr: row-strip mode (comm.h), the context owns block rows
// strip_of(rank) and computes the pixel rows of the strip widened by the metric's receptive field.
struct Region {
  Geom g;
  Comm* comm;
  int by_lo, by_hi;  // owned block rows
  int cr_lo, cr_hi;  // pixel rows computed by the image-plane kernels (strip + 56-row halo)
  Stream s;
  bool strips() const { return comm != nullptr && comm->world() > 1; }

  template <class F>
  void px(const F& f, const char* name, int nplanes = 1) const {  // rows [cr_lo, cr_hi) of nplanes planes
    const int nrows = cr_hi - cr_lo;
    if (cr_lo == 0 && nrows == g.h) {
      launch_2d(s, f, g.w, g.h * nplanes, name);
    } else {
      launch_2d(s, RowsOf<F>{f, cr_lo, nrows, g.h}, g.w, nrows * nplanes, name);
    }
  }
  template <class F>
  void block_rows(const F& f, const char* name, int lo, int hi) const {  // blocks of block rows [lo, hi)
    const int n = (hi - lo) * g.bw;
    if (lo == 0) {
      launch_1d(s, f, n, name);
    } else {
      launch_1d(s, OffsetOf<F>{f, lo * g.bw}, n, name);
    }
  }
  // in-place all-gather of a per-block array: every rank owns the blocks of its strip
  void gather_blocks(void* dev_buf, size_t elem_bytes_per_block) const;
  // packed [n][h][w] on the host <-> n planes [h][pitch]
  void upload_planes(const float* packed, float* dst, int n) const;
  void download_planes(const float* src, float* packed, int n) const;
};

class Butteraugli {
 public:
  // One image; comm: strip mode (Region).
  Butteraugli(int w, int h, int device, Comm* comm);
  // Batched: up to `capacity` pairs of w x h images are scored per call.  Each pair has an arena
  // slot of kBatchSlotPlanes planes (DESIGN.md §4), and the analysis of the originals and the
  // Compare chain run as one launch per stage over all pairs.
  Butteraugli(int w, int h, int capacity, int device);
  static constexpr int kBatchSlotPlanes = 53;
  ~Butteraugli();
  Butteraugli(const Butteraugli&) = delete;
  Butteraugli& operator=(const Butteraugli&) = delete;

  const Region& region() const { return r_; }
  const Tables& tables() const { return t_; }
  int capacity() const { return capacity_; }
  int device() const { return device_; }
  // makes this metric's device current for the calling host thread
  void bind() { select_device(device_); }

  // PsychoImage of the original (b/butteraugli.cc:784) into ps0, resident from then on.  linear_rgb:
  // the original as linear RGB planes [3][h][w] on the host; null: the image that lin() holds.
  void analyse_original(const float* linear_rgb = nullptr);
  // Mask's activity planes (sx, sy1, sy2) of the original, from the XYB planes that
  // analyse_original() leaves behind (the encoder's block-corner mask, a13)
  const float* original_mask_activity() {
    mask_activity(xyb_);
    return sact_;
  }
  // [3] linear RGB planes of the image to score (the encoder renders its candidate here)
  float* lin() { return lin_; }
  // [nblocks] maxima of the distmap per block, left by the last compare()
  const float* block_max() const { return block_max_; }

  // S1..S13 on lin() (ButteraugliComparator::Diffmap): leaves the distmap and the per-block
  // maxima on the device and returns the distance.
  float compare();
  // the same in two halves: compare_begin() queues the kernels, compare_end() waits for the
  // distance (where the launches need a host round trip -- strip mode, the staged chain --
  // compare_begin() does it all)
  void compare_begin();
  float compare_end();
  void download_distmap(float* out) { r_.download_planes(dm_, out, 1); }  // [h][w] packed

  // Stand-alone (scope row f4): compare_linear() scores a second image, linear RGB planes [3][h][w],
  // against the original.
  float compare_linear(const float* linear_rgb);
  // The same with the second image in memory of this metric's device, packed [3][h][w].  This
  // metric's stream first waits for the work queued so far on `caller`; the image is then copied
  // into lin (the tensor maps and the captured graph are bound to lin).  diffmap: device memory,
  // packed [h][w], or null; it is written when the call returns.
  float compare_linear_device(const float* linear_rgb, float* diffmap, Stream caller);
  // ButteraugliInterface for each of n <= capacity pairs, rgb0 / rgb1 packed [n][3][h][w]:
  // diffmap [n][h][w] (or null) and maxima[n].  device: rgb0, rgb1 and diffmap are memory of this
  // metric's device; its stream first waits for the work queued so far on `caller`.
  // Either way every output is written when the call returns.
  void compare_batch(const float* rgb0, const float* rgb1, int n, float* diffmap, float* maxima, bool device,
                     Stream caller);
  // ButteraugliComparator::Mask (b/butteraugli.cc:793) of the original at every pixel, on the
  // host: mask, mask_dc [3][h][w].  Leaves the resident PsychoImage as it is.
  void mask(float* mask, float* mask_dc);
  // Mask(rgb, rgb) of linear RGB planes [3][h][w] as ButteraugliAdaptiveQuantization
  // (b/butteraugli.cc:1880) computes it: its Y plane -> quant [h][w] on the host.
  void adaptive_quantization(const float* linear_rgb, float* quant);

  // test hooks: single stages on caller-provided planes (packed [n][h][w])
  void debug_blur(const float* in, float* out, int id);
  void debug_opsin(const float* rgb_lin, float* xyb);
  void debug_separate(const float* xyb, float* ps10);
  void debug_psycho0(float* ps10);

 private:
  void init(int w, int h, Comm* comm);
  void alloc_planes();
  void release();
  float* planes(size_t n);
  // the launch sequences (these, compare() and mask()) are defined in pipeline.cu
  void blur(const float* in, float* out, int nplanes, int id);
  void opsin(const float* lin, float* xyb);
  void separate(const float* xyb, float* ps);
  // Mask's DiffPrecompute of X and Y (planes xy[0], xy[1]) and its three blurs -> sact_
  void mask_activity(const float* xy);
  // Mask(xy, xy) at every pixel -> mask_ (mask [3], then mask_dc [3], allocated on first use)
  void mask_planes(const float* xy);

  // TMA-staged fused Compare chain (fused_kernels.cuh; CUDA build only)
  struct Fused;
  Fused* fused_ = nullptr;
  bool use_fused_ = false;
  // nimg images in arena slots kslot planes apart (a single image passes 1, 0)
  void fused_opsin(const float* lin, float* xyb, int nimg, int kslot);
  void fused_separate(const float* xyb, float* ps, bool with_diffs, int nimg, int kslot);
  void fused_blur(const float* in, float* out, int nplanes, int id);
  void fused_compare_submit();
  float fused_compare_result();
  void fused_compare_launches(int nimg, int kslot);
  void fused_sup0(int nimg, int kslot);
  void fused_compare_batch(const float* rgb0, const float* rgb1, int n, float* diffmap, float* maxima);
  bool compare_pending_ = false;
  float compare_stash_ = 0.0f;

  int device_;
  Region r_;
  const Geom& g_ = r_.g;
  const Stream& s_ = r_.s;
  bool have_stream_ = false;
  // arena slots, kslot_ planes each (a single image: one slot, kslot_ = 0)
  int capacity_ = 1;
  int kslot_ = 0;
  Tables t_;
  HostTables ht_;
  MaltaParams malta_[6];
  double asym_w0_, asym_w1_;
  std::vector<void*> owned_;

  // plane groups (alloc_planes)
  float* lin_ = nullptr;     // [3]
  float* xyb_ = nullptr;     // [3]
  float* lf_ = nullptr;      // [3]
  float* mf_in_ = nullptr;   // [3]
  float* hf_raw_ = nullptr;  // [2]
  float* ps0_ = nullptr;     // [10] PsychoImage of the original
  float* ps1_ = nullptr;     // [10]
  float* sup0_ = nullptr;    // [2] DiffPrecompute neighbour sums of the original (X, Y)
  float* diffs6_ = nullptr;  // [6] Malta pre-pass planes: X uhf, hf, mf; Y uhf, hf, mf
  float* noise_ = nullptr;   // [2] pre, blurred
  float* mpre_ = nullptr;    // [2]
  float* tmp_ = nullptr;     // [3] blur x-pass output
  float* blr_ = nullptr;     // [3]
  float* ac_ = nullptr;      // [2]
  float* dm_ = nullptr;      // [2] diffmap, blurred
  float* mf_blr_ = nullptr;  // [3]
  float* hf_blr_ = nullptr;  // [2]
  float* diffs_ = nullptr;   // [1]
  float* sact_ = nullptr;    // [3] sx, sy1, sy2
  float* mask_ = nullptr;
  float* block_max_ = nullptr;      // [capacity][nblocks]
  unsigned int* d_gmax_ = nullptr;  // [capacity] global maximum of the distmap (float bits)
  float* partial_ = nullptr;        // [1024]
};

#if defined(__CUDACC__) && !defined(GB200_HOSTSIM)
// Tensor maps of the plane groups and the Compare chain captured as a CUDA graph.
struct Butteraugli::Fused {
  typedef std::tuple<const float*, int, int, int> Key;  // base, planes, box w, box h
  std::map<Key, CUtensorMap> maps;
  // the Compare chain as a CUDA graph: same kernels, same arguments every call (all buffers
  // live as long as the metric), one driver call instead of sixteen
  cudaGraphExec_t compare_graph = nullptr;
  long compare_graph_kernels = 0;
  int compare_calls = 0;
  ~Fused() {
    if (compare_graph) cudaGraphExecDestroy(compare_graph);
  }
  const CUtensorMap& map(const float* base, int nplanes, int box_w, int box_h, const Geom& g) {
    const Key key(base, nplanes, box_w, box_h);
    std::map<Key, CUtensorMap>::iterator it = maps.find(key);
    if (it == maps.end())
      it = maps.insert(std::make_pair(key, make_plane_map(base, g.w, g.h, g.pitch, g.plane, nplanes, box_w, box_h))).first;
    return it->second;
  }
  // a group of nplanes planes in each of the `capacity` arena slots of a batch, kslot planes apart
  // (kslot = 0: the group alone)
  int capacity = 1;
  const CUtensorMap& slots(const float* base, int nplanes, int box_w, int box_h, int kslot, const Geom& g) {
    return map(base, (capacity - 1) * kslot + nplanes, box_w, box_h, g);
  }
};
#endif

}  // namespace gb200
