// The butteraugli metric on the device: the Compare chain (the TMA-staged fused chain, and the staged
// chain it is checked against), the float planes it works on, and the analysis of the original.
// One Butteraugli scores one image -- the encoder's candidate (ImageContext holds one) or a
// stand-alone comparator's -- or a batch of same-size pairs, or a batch of same-size candidates
// against one original (ComparatorSet: against resident originals of sizes of their own).  It owns the
// stream and the tables,
// which the encoder's kernels use as well.  See DESIGN.md §4 and §5.1.
#pragma once
#include <stddef.h>

#include <memory>
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

struct MixPass;  // one pass of a mixed-size call over the fused chain (pipeline.cu)
struct MapReq;   // the tensor map argument of a fused launch (pipeline.cu)
struct MixSrc;   // the images of a mixed-size run, float or 8-bit (pipeline.cu)

// The stand-alone tool's choice for an RGBA image scored over black and over white: white wins only
// where it scores strictly higher; a tie keeps black (butteraugli_main.cc:414).
inline bool white_wins(float white, float black) { return white > black; }

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
  // Batched, up to `capacity` images per call, one launch per stage over all of them (DESIGN.md §4).
  //   kPairs: w x h pairs (compare_batch).  Each pair has an arena slot of kBatchSlotPlanes planes,
  //     and the originals are analysed in the call.
  //   kCandidates: w x h candidates against one original (compare_many), which analyse_original()
  //     analyses once.  Its planes lie once outside the slots, and each candidate has a slot of
  //     kCandidateSlotPlanes planes.  Capacity 1 is the single-image metric.
  enum class Slots { kPairs, kCandidates };
  Butteraugli(int w, int h, int capacity, int device, Slots slots = Slots::kPairs);
  static constexpr int kBatchSlotPlanes = 53;
  static constexpr int kCandidateSlotPlanes = 41;  // a pair's slot without ps0 and sup0
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
  // ButteraugliComparator::Diffmap against the original for each of n <= capacity candidates,
  // rgb1 packed [n][3][h][w]; outputs, device and caller as in compare_batch.  Slots kCandidates;
  // with capacity 1, the staged chain or the CPU port the candidates go one by one through slot 0.
  void compare_many(const float* rgb1, int n, float* diffmap, float* maxima, bool device, Stream caller);
  // compare_batch on n <= capacity pairs of different sizes: pair i is w[i] x h[i], each at least 8x8 and
  // at most this batch's size, rgb0[i] / rgb1[i] packed [3][h[i]][w[i]], diffmap[i] [h[i]][w[i]] (diffmap
  // itself may be null).  Outputs, device and caller as in compare_batch.  The fused chain scores all pairs
  // in one pass of launches over (image, tile) work items, with tensor maps of each distinct size; the
  // staged chain and the CPU port score each pair through a metric of its own size.
  void compare_batch_sizes(const int* w, const int* h, const float* const* rgb0, const float* const* rgb1, int n,
                           float* const* diffmap, float* maxima, bool device, Stream caller);

  // 8-bit sRGB input, as the stand-alone `butteraugli` tool reads it (b/butteraugli_main.cc:239-281,
  // :390-419): images interleaved [n][h][w][channels], channels 3 (RGB) or 4 (RGBA).  They are
  // converted to linear planes on the device (SrgbToLinear) and scored by the float entries above from
  // device memory (DESIGN.md §4).  RGBA is laid over black and scored, then over white and scored; where
  // white scores strictly higher, its score and its diffmap replace black's.
  //
  // The original of a comparator, in host memory, laid over `background` (0 or 255), into lin and
  // analysed there (analyse_original).
  void analyse_original_srgb(const uint8_t* img0, int channels, int background);
  // compare_batch on 8-bit pairs; outputs, device and caller as there.  background 0 or 255: the pairs
  // laid over that background only, with no choice between backgrounds (gb200_butteraugli_diffmap_srgb
  // makes the choice itself, on padded images after it has cropped them).
  void compare_batch_srgb(const uint8_t* img0, const uint8_t* img1, int n, int channels, float* diffmap,
                          float* maxima, bool device, Stream caller, int background = -1);
  // compare_many on 8-bit candidates against the original analyse_original_srgb() laid over black;
  // for channels 4, `white` is the metric of the same shape whose original it laid over white.
  void compare_many_srgb(const uint8_t* img1, int n, int channels, Butteraugli* white, float* diffmap,
                         float* maxima, bool device, Stream caller);
  // compare_batch_sizes on 8-bit pairs: img0[i] / img1[i] interleaved [h[i]][w[i]][channels[i]], channels 3
  // or 4 per pair; diffmap itself and its entries may be null.  The fused chain converts while it packs
  // the images into the arena (k_mix_srgb): one run over all pairs laid over black, then one over the RGBA
  // pairs alone laid over white, with passes of their own sizes.  The staged chain and the CPU port score
  // each pair through compare_batch_srgb of a pair batch of its own size.
  void compare_batch_sizes_srgb(const int* w, const int* h, const int* channels, const uint8_t* const* img0,
                                const uint8_t* const* img1, int n, float* const* diffmap, float* maxima, bool device,
                                Stream caller);
  // A comparator set's originals (ComparatorSet; fused chain only, on a pair batch).  analyse_originals: n <=
  // capacity originals of sizes w[i] x h[i] in host memory, float planes (channels null) or 8-bit pixels laid
  // over `background`, analysed in mixed passes; the kStoredPlanes planes of original i go to store[i]
  // (device memory, [kStoredPlanes][h[i]][w[i]]).  Returns when they are there.
  void analyse_originals(const int* w, const int* h, const int* channels, const void* const* img0, int n,
                         int background, float* const* store);
  // compare_batch_sizes (channels null) or compare_batch_sizes_srgb with pair i's original taken from the
  // store: stored[0][i] its analysis (over black), stored[1][i] over white (RGBA) or null.
  void compare_originals(const int* w, const int* h, const int* channels, float* const* const* stored,
                         const void* const* img1, int n, float* const* diffmap, float* maxima, bool device,
                         Stream caller);
  bool fused() const { return use_fused_; }
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
  // n 8-bit images (memory of this device) over `background` -> dst [n][3][h][pitch]
  void srgb_to_linear(const uint8_t* src, int n, int channels, int background, float* dst, int pitch);
  // the 8-bit entries' buffers, for `per_slot` images in each of the capacity slots (first use)
  void srgb_alloc(int per_slot);
  // n images laid over black by score(background, diffmap, maxima), for RGBA over white as well, and
  // the winner of each into diffmap / maxima (outputs as in compare_batch); only >= 0: that background
  // alone
  template <class Score>
  void srgb_backgrounds(int n, int channels, int only, float* diffmap, float* maxima, bool device,
                        const Score& score);

  // TMA-staged fused Compare chain (fused_kernels.cuh; CUDA build only)
  struct Fused;
  Fused* fused_ = nullptr;
  bool use_fused_ = false;
  // nimg images in arena slots kslot planes apart, the original's planes kslot0 apart (kslot0 =
  // kslot: an original per image, 0: one for all; a single image passes 1, 0, 0)
  void fused_opsin(const float* lin, float* xyb, int nimg, int kslot);
  void fused_separate(const float* xyb, float* ps, bool with_diffs, int nimg, int kslot, int kslot0);
  void fused_blur(const float* in, float* out, int nplanes, int id);
  void fused_compare_submit();
  float fused_compare_result();
  void fused_compare_launches(int nimg, int kslot, int kslot0);
  void fused_sup0(int nimg, int kslot);
  // n pairs, or with rgb0 null n candidates against the resident original
  void fused_compare_batch(const float* rgb0, const float* rgb1, int n, float* diffmap, float* maxima);
  // n and the pair sizes of compare_batch_sizes*, which the C entries have checked with their messages
  void check_sizes(const int* w, const int* h, int n) const;
  // compare_batch_sizes (channels null: float planes) and compare_batch_sizes_srgb on the fused chain; its
  // buffers and tables (allocated on the first call, kept).  stored: compare_originals (in0 null).
  void fused_compare_sizes(const int* w, const int* h, const int* channels, const void* const* in0,
                           const void* const* in1, int n, float* const* diffmap, float* maxima, bool device,
                           float* const* const* stored = nullptr);
  // the passes of a mixed run over `pairs` (indices into w, h and src's tables), with their tables uploaded:
  // the pairs sorted by size into *order, pair i's diffmap into dst[i] (dst null: none)
  std::vector<MixPass> mixed_passes(const int* w, const int* h, const std::vector<int>& pairs, const MixSrc& src,
                                    float* const* dst, std::vector<int>* order);
  void mixed_pack(const MixPass& p, void* const* ext, const MixSrc& src);
  void mixed_original(const MixPass& p, bool to_arena);
  // one run of mixed passes over `pairs`: diffmap of pair i into dst[i] (device memory, or null), its maximum
  // into maxima[i]
  void fused_mixed_run(const int* w, const int* h, const std::vector<int>& pairs, const MixSrc& src,
                       float* const* dst, float* maxima);
  struct Mixed;
  Mixed* mixed_ = nullptr;
  MixPass* mix_ = nullptr;  // set while the launches of a mixed pass are queued
  void mixed_release();
  // the tensor map argument of a launch over plane group `base` (the batch's, or a mixed pass's per size)
  MapReq maps(const float* base, int nplanes, int box_w, int box_h, int kslot);
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
  bool one_original_ = false;  // Slots::kCandidates with capacity > 1
  Tables t_ = Tables();  // null until built: the pair batch's staged chain builds none
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

  // the 8-bit entries' buffers (srgb_alloc), per_slot images in each slot, packed
  uint8_t* srgb_u8_ = nullptr;                 // [per_slot][capacity][h][w][4] host input, uploaded
  float* srgb_lin_ = nullptr;                  // [per_slot][capacity][3][h][w] converted planes
  float* srgb_dm_[2] = {nullptr, nullptr};     // [capacity][h][w] diffmaps: host output; over white
};

// A comparator set: `count` originals of sizes of their own, each analysed once when the set is made, and
// candidates scored against the original each names (DESIGN.md §4).  On the fused chain the analyses stay in
// one device buffer, the store: kStoredPlanes planes [h][w] per original, an RGBA original of an 8-bit set
// twice (over black, then over white).  A call gathers them into the slots of one pair batch of the largest
// width x largest height.  The staged chain and the CPU port keep the originals' inputs instead and score a
// call through that batch's compare_batch_sizes*.
class ComparatorSet {
 public:
  // w, h [count], each at least 8x8; channels null: img0[i] float planes [3][h][w], else 8-bit
  // [h][w][channels[i]]; all in host memory
  ComparatorSet(const int* w, const int* h, const int* channels, const void* const* img0, int count, int capacity,
                int device);
  ~ComparatorSet();
  ComparatorSet(const ComparatorSet&) = delete;
  ComparatorSet& operator=(const ComparatorSet&) = delete;
  Butteraugli& metric() { return *ba_; }
  int count() const { return static_cast<int>(w_.size()); }
  bool srgb() const { return !channels_.empty(); }
  // candidate i against original[i] (0 <= original[i] < count), img1[i] of that original's size and channels;
  // outputs, device and caller as in compare_batch_sizes
  void compare(const int* original, const void* const* img1, int n, float* const* diffmap, float* maxima,
               bool device, Stream caller);

 private:
  std::vector<int> w_, h_, channels_;
  std::unique_ptr<Butteraugli> ba_;
  void* store_ = nullptr;
  // byte offsets in store_ of each original's analysis over black and over white (kNone: none); staged chain
  // and CPU port: of its input, at_[0] only
  static constexpr size_t kNone = ~static_cast<size_t>(0);
  std::vector<size_t> at_[2];
  std::vector<std::vector<unsigned char> > host_;  // staged chain and CPU port: the inputs
};

#if defined(__CUDACC__) && !defined(GB200_HOSTSIM)
// Tensor maps of the plane groups and the Compare chain captured as a CUDA graph.
struct Butteraugli::Fused {
  typedef std::tuple<const float*, int, int, int, int, int> Key;  // base, planes, box w, box h, w, h
  std::map<Key, CUtensorMap> maps;
  // the Compare chain as a CUDA graph: same kernels, same arguments every call (all buffers
  // live as long as the metric), one driver call instead of sixteen
  cudaGraphExec_t compare_graph = nullptr;
  long compare_graph_kernels = 0;
  int compare_calls = 0;
  ~Fused() {
    if (compare_graph) cudaGraphExecDestroy(compare_graph);
  }
  // the group's planes as a w x h image (w, h 0: the metric's size)
  const CUtensorMap& map(const float* base, int nplanes, int box_w, int box_h, const Geom& g, int w = 0, int h = 0) {
    if (w == 0) {
      w = g.w;
      h = g.h;
    }
    const Key key(base, nplanes, box_w, box_h, w, h);
    std::map<Key, CUtensorMap>::iterator it = maps.find(key);
    if (it == maps.end())
      it = maps.insert(std::make_pair(key, make_plane_map(base, w, h, g.pitch, g.plane, nplanes, box_w, box_h))).first;
    return it->second;
  }
  // drops the maps of other sizes than the metric's (those of mixed-size calls)
  void drop_other_sizes(const Geom& g) {
    for (std::map<Key, CUtensorMap>::iterator it = maps.begin(); it != maps.end();) {
      if (std::get<4>(it->first) != g.w || std::get<5>(it->first) != g.h) {
        it = maps.erase(it);
      } else {
        ++it;
      }
    }
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
