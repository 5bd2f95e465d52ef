// Kernel sequences of the hot path: the encoder's (ImageContext, pipeline.h) and the metric's
// (the Butteraugli members that launch kernels; its state, plane layout and entry points are in
// butteraugli.cu).  Every kernel of the library is compiled in this one translation unit: kernels
// that share one device module keep the code and shared-memory layout they were tuned with, and
// tiled_kernels.cuh defines kernels that are not templates.  Compiled by nvcc for sm_90a in the
// product, and by g++ -DGB200_HOSTSIM for the CPU port.
#include "pipeline.h"
#include "exact_sort.h"
#include "order_exact.h"

#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <stdexcept>

#include "block_math.h"
#include "jpeg_dev.h"
#include "jpeg_in.h"
#include "walk_dev.h"
#if !defined(GB200_HOSTSIM)
#include <deque>
#include <map>
#include <mutex>
#include <set>
#include <type_traits>

#include "tiled_kernels.cuh"
#include "zeroing_warp.cuh"
#include "render_warp.cuh"
#include "fused_kernels.cuh"
#endif

namespace gb200 {

#if !defined(GB200_HOSTSIM)
// ---------------------------------------------------------------------------
// The metric: TMA-staged fused Compare chain (fused_kernels.cuh).
namespace {
template <int R>
BlurK<R> make_blurk(const HostTables& ht, int id) {
  if (static_cast<int>(ht.blur_taps[id].size()) != 2 * R + 1) throw std::runtime_error("blur radius / kernel mismatch");
  BlurK<R> k;
  for (int j = 0; j < 2 * R + 1; ++j) {
    k.n[j] = ht.blur_taps_n[id][j];
    k.raw[j] = ht.blur_taps[id][j];
  }
  return k;
}

// opt-in to more than 48 KB of dynamic shared memory: once per (device, kernel)
template <class K>
void allow_smem(K kernel, size_t bytes) {
  static std::mutex mu;
  static std::set<std::pair<int, const void*> > done;
  int dev = 0;
  GB_CUDA(cudaGetDevice(&dev));
  const std::pair<int, const void*> key(dev, reinterpret_cast<const void*>(kernel));
  std::lock_guard<std::mutex> lock(mu);
  if (done.count(key)) return;
  GB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
  done.insert(key);
}

inline int cdiv(int a, int b) { return (a + b - 1) / b; }
// rows of a rolling-blur segment for `rows` rows: whole steps, about GBR_SEG rows
inline int roll_seg(int rows) {
  const int nseg = cdiv(rows, GBR_SEG);
  return cdiv(cdiv(rows, nseg), GBR_CH) * GBR_CH;
}

}  // namespace

// One pass of a mixed-size call (Butteraugli::fused_compare_sizes, and a comparator set's analysis and
// scoring): its images, slots n0 .. n0 + m - 1,
// have at most GB_MIX_SHAPES distinct sizes.  Device tables: the images, and per tile shape of the
// chain's launches the first work item of each image.
enum MixKind { kMix2d, kMixRollLf, kMixRollMf, kMixPx, kMixX4, kMixMalta, kMixY, kMixKinds };
struct MixPass {
  int n0 = 0, m = 0;
  std::vector<std::pair<int, int> > shapes;  // (w, h) of map set index s
  const MixImage* img = nullptr;
  const int* tile0 = nullptr;  // [kMixKinds][m + 1]
  int total[kMixKinds];        // work items per tile shape
  BlurTab tab[kNumBlurs];      // border scales of the pass's sizes (MixImage::sx, sy index them)
  const int* rows_in = nullptr;   // [m + 1] rows per image packed: 3h of float planes, h of 8-bit pixels
  const int* rows_dm = nullptr;   // [m + 1] h rows per image with a diffmap, 0 per image without
  void* const* ext0 = nullptr;  // [m] first image of each pair (device memory: float or 8-bit)
  void* const* ext1 = nullptr;
  float* const* extdm = nullptr;  // [m] diffmap of each image, or null
  // a comparator set's run: kStoredPlanes * h rows per image, and its original's analysis in the store
  const int* rows_org = nullptr;  // [m + 1]
  float* const* extorg = nullptr;  // [m]
  int rows_in_total = 0, rows_dm_total = 0, rows_org_total = 0;
  std::deque<MixMaps> mapsets;  // the map sets of the launches queued so far (stable addresses)
  MixGeom geom(int kind) const { return MixGeom{img, tile0 + kind * (m + 1), m, n0}; }
};

struct MapReq {
  const CUtensorMap* one;
  const MixMaps* mix;  // a mixed pass's: one map per size
  template <int B>
  const typename MapArg<B>::type& get() const {
    if constexpr (B == 2) {
      return *mix;
    } else {
      return *one;
    }
  }
};

MapReq Butteraugli::maps(const float* base, int nplanes, int box_w, int box_h, int kslot) {
  MapReq r{&fused_->slots(base, nplanes, box_w, box_h, kslot, g_), nullptr};
  if (mix_ != nullptr) {
    mix_->mapsets.emplace_back();
    MixMaps& set = mix_->mapsets.back();
    const int planes = (fused_->capacity - 1) * kslot + nplanes;
    for (size_t i = 0; i < mix_->shapes.size(); ++i)
      set.m[i] = fused_->map(base, planes, box_w, box_h, g_, mix_->shapes[i].first, mix_->shapes[i].second);
    r.mix = &set;
  }
  return r;
}

namespace {
// f(integral_constant<int, 1>) for a launch over several images (the kernels' batched instantiation,
// which takes the image from blockIdx.z), f(<2>) for a mixed pass (images and tiles from the pass's
// work items), f(<0>) for one image.  EpiStore (stand-alone blurs) has no batched form.
template <class Epi, class F>
void with_batch(int nimg, const MixPass* mix, const F& f) {
  if constexpr (!std::is_same<Epi, EpiStore>::value) {
    if (mix != nullptr) {
      f(std::integral_constant<int, 2>());
      return;
    }
    if (nimg > 1) {
      f(std::integral_constant<int, 1>());
      return;
    }
  }
  if (nimg != 1 || mix != nullptr) throw std::runtime_error("with_batch: no batched form of this launch");
  f(std::integral_constant<int, 0>());
}

// the grid of a launch: `grid`, or a mixed pass's work items of tile shape `kind`
dim3 grid_of(dim3 grid, const MixPass* mix, int kind) { return mix == nullptr ? grid : dim3(mix->total[kind]); }
// the geometry argument of a launch of instantiation B: pg, and for a mixed pass its work items of `kind`
template <int B>
typename GeomArg<B>::type geom_arg(const PlaneGeom& pg, const MixPass* mix, int kind) {
  if constexpr (B == 2) {
    PlaneGeomMix g;
    static_cast<PlaneGeom&>(g) = pg;
    g.mix = mix->geom(kind);
    return g;
  } else {
    return pg;
  }
}
const BlurTab& tab_of(const Tables& t, const MixPass* mix, int id) { return mix ? mix->tab[id] : t.blur[id]; }

// Rolling-window blur of a plane group with epilogue (k_roll_blur); `in_map` has boxes of
// RollCfg<R, NP>::SW x GBR_CH.  The launch's rows are cut into segments of whole steps of
// about GBR_SEG rows.  nimg images: arena slots 0 .. nimg - 1 (PlaneGeom::kslot).
template <int R, int NP, class Epi>
void launch_roll(Stream s, const MapReq& in_map, int planes_z, int nimg, const BlurTab& tab, PlaneGeom pg,
                 const HostTables& ht, int id, const Epi& epi, const char* name, const MixPass* mix = nullptr,
                 int kind = 0) {
  const int rows = pg.y_end - pg.y0;
  if (rows <= 0) return;
  typedef RollCfg<R, NP> C;
  const int seg = roll_seg(rows);
  pg.zimg = planes_z;
  const dim3 grid = grid_of(dim3(cdiv(pg.w, GBR_TW), cdiv(rows, seg), planes_z * nimg), mix, kind);
  note_launch(name, s, static_cast<double>(pg.w) * rows * (NP == 1 ? planes_z : NP) * nimg);
  with_batch<Epi>(nimg, mix, [&](auto b) {
    constexpr int B = decltype(b)::value;
    allow_smem(k_roll_blur<B, R, NP, Epi>, C::kSmemBytes);
    k_roll_blur<B, R, NP, Epi><<<grid, 128, C::kSmemBytes, s>>>(in_map.get<B>(), tab.scale_x, tab.scale_y,
                                                                geom_arg<B>(pg, mix, kind), seg,
                                                                make_blurk<R>(ht, id), epi);
  });
  note_launch_end(name, s);
}

template <int R, int NP, class Epi>
void launch_tma_y(Stream s, const MapReq& in_map, int planes_z, int nimg, const BlurTab& tab, PlaneGeom pg,
                  const HostTables& ht, int id, const Epi& epi, const char* name, const MixPass* mix = nullptr,
                  int kind = 0) {
  const int rows = pg.y_end - pg.y0;
  if (rows <= 0) return;
  const size_t smem = static_cast<size_t>(NP) * (GBY_TH + 2 * R) * GBY_TW * sizeof(float) + 16;
  pg.zimg = planes_z;
  const dim3 grid = grid_of(dim3(cdiv(pg.w, GBY_TW), cdiv(rows, GBY_TH), planes_z * nimg), mix, kind);
  note_launch(name, s, static_cast<double>(pg.w) * rows * (NP == 1 ? planes_z : NP) * nimg);
  with_batch<Epi>(nimg, mix, [&](auto b) {
    constexpr int B = decltype(b)::value;
    allow_smem(k_tma_blur_y<B, R, NP, Epi>, smem);
    k_tma_blur_y<B, R, NP, Epi><<<grid, 256, smem, s>>>(in_map.get<B>(), tab.scale_y, geom_arg<B>(pg, mix, kind),
                                                        make_blurk<R>(ht, id), epi);
  });
  note_launch_end(name, s);
}

template <int R, int NP, class Epi>
void launch_tma_2d(Stream s, const MapReq& in_map, int nimg, const BlurTab& tab, PlaneGeom pg,
                   const HostTables& ht, int id, const Epi& epi, const char* name, const MixPass* mix = nullptr) {
  const int rows = pg.y_end - pg.y0;
  if (rows <= 0) return;
  typedef Blur2dCfg<R, NP> C;
  pg.zimg = 1;
  const dim3 grid = grid_of(dim3(cdiv(pg.w, GB2_TW), cdiv(rows, GB2_TH), nimg), mix, kMix2d);
  note_launch(name, s, static_cast<double>(pg.w) * rows * nimg);
  with_batch<Epi>(nimg, mix, [&](auto b) {
    constexpr int B = decltype(b)::value;
    allow_smem(k_tma_blur_2d<B, R, NP, Epi>, C::kSmemBytes);
    k_tma_blur_2d<B, R, NP, Epi><<<grid, 256, C::kSmemBytes, s>>>(in_map.get<B>(), tab.scale_x, tab.scale_y,
                                                                  geom_arg<B>(pg, mix, kMix2d),
                                                                  make_blurk<R>(ht, id), epi);
  });
  note_launch_end(name, s);
}
}  // namespace

// Radii of the nine blurs (b/butteraugli.cc:145: max(1, int(2.25 * sigma))); make_blurk checks them.
#define GB_R_OPSIN 2
#define GB_R_LF 16
#define GB_R_MF 8
#define GB_R_HF 4
#define GB_R_NOISE 23
#define GB_R_MASKX 20
#define GB_R_MASKY0 5
#define GB_R_MASKY1 20
#define GB_R_FINAL 3

// Launches over nimg images take the planes of arena slots 0 .. nimg - 1, kslot planes apart
// (kslot = 0 and nimg = 1 for a single image); their tensor maps cover every slot.  The original's
// planes are kslot0 planes apart: kslot0 = kslot when each image has its own, 0 when all share one.
namespace {
PlaneGeom fused_geom(const Geom& g, int y0, int y_end, int kslot, int kslot0) {
  return PlaneGeom{g.w, g.h, g.pitch, g.plane, y0, y_end, kslot, 1, kslot0};
}
}  // namespace

void Butteraugli::fused_opsin(const float* lin, float* xyb, int nimg, int kslot) {
  const PlaneGeom pg = fused_geom(g_, r_.cr_lo, r_.cr_hi, kslot, kslot);
  typedef Blur2dCfg<GB_R_OPSIN, 3> C;
  launch_tma_2d<GB_R_OPSIN, 3>(s_, maps(lin, 3, C::SWI, C::HI, kslot), nimg, tab_of(t_, mix_, kBlurOpsin), pg, ht_,
                               kBlurOpsin, EpiOpsin{xyb, g_.pitch, g_.plane, kslot * g_.plane}, "opsin_fused", mix_);
}

// SeparateFrequencies; with_diffs: also the Malta pre-pass and the noise difference against ps0_.
void Butteraugli::fused_separate(const float* xyb, float* ps, bool with_diffs, int nimg, int kslot, int kslot0) {
  const PlaneGeom pg = fused_geom(g_, r_.cr_lo, r_.cr_hi, kslot, kslot0);
  const size_t P = g_.plane, S = kslot * P, S0 = kslot0 * P;
  // S2: lf = Blur(xyb, 7.47); mf_in = xyb - lf
  // (launch names are those of the former y-pass kernels, which these replace)
  launch_roll<GB_R_LF, 1>(s_, maps(xyb, 3, RollCfg<GB_R_LF, 1>::SW, GBR_CH, kslot), 3, nimg, tab_of(t_, mix_, kBlurLf), pg,
                          ht_, kBlurLf, EpiLf{xyb, lf_, mf_in_, g_.pitch, P, S}, "lf_fused_y", mix_, kMixRollLf);
  // S3 + S4: mf = Blur(mf_in, 3.73); split, range tweaks, SuppressXByY (+ Malta pre-pass of the mf bands)
  EpiMf em;
  em.mf_in = mf_in_;
  em.ps = ps;
  em.hf_raw = hf_raw_;
  em.ps0 = with_diffs ? ps0_ : nullptr;
  em.diffs = diffs6_;
  em.mp_x = malta_[5];
  em.mp_y = malta_[4];
  em.pitch = g_.pitch;
  em.plane = P;
  em.slot = S;
  em.slot0 = S0;
  launch_roll<GB_R_MF, 3>(s_, maps(mf_in_, 3, RollCfg<GB_R_MF, 3>::SW, GBR_CH, kslot), 1, nimg, tab_of(t_, mix_, kBlurMf),
                          pg, ht_, kBlurMf, em, "mf_fused_y", mix_, kMixRollMf);
  // S5 + S6: hf = Blur(hf_raw, 1.87) in one kernel; uhf / hf / lf "vals" (+ Malta pre-pass, noise difference)
  EpiHf eh;
  eh.lf_raw = lf_;
  eh.ps = ps;
  eh.ps0 = with_diffs ? ps0_ : nullptr;
  eh.diffs = diffs6_;
  eh.noise = noise_;
  eh.mp_uhf_y = malta_[0];
  eh.mp_uhf_x = malta_[1];
  eh.mp_hf_y = malta_[2];
  eh.mp_hf_x = malta_[3];
  eh.pitch = g_.pitch;
  eh.plane = P;
  eh.slot = S;
  eh.slot0 = S0;
  typedef Blur2dCfg<GB_R_HF, 2> C;
  launch_tma_2d<GB_R_HF, 2>(s_, maps(hf_raw_, 2, C::SWI, C::HI, kslot), nimg, tab_of(t_, mix_, kBlurHf), pg, ht_, kBlurHf,
                            eh, "hf_fused", mix_);
}

// Neighbour sums of DiffPrecompute for the original's PsychoImage (constant during the search).
void Butteraugli::fused_sup0(int nimg, int kslot) {
  const PlaneGeom pg = fused_geom(g_, r_.cr_lo, r_.cr_hi, kslot, kslot);
  const int rows = r_.cr_hi - r_.cr_lo;
  dim3 block(32, 8), grid = grid_of(dim3(cdiv(g_.w, 32), cdiv(rows, 8), nimg), mix_, kMixPx);
  note_launch("mask_sup0", s_, static_cast<double>(g_.w) * rows * nimg);
  with_batch<void>(nimg, mix_, [&](auto b) {
    constexpr int B = decltype(b)::value;
    k_mask_sup<B><<<grid, block, 0, s_>>>(ps0_, sup0_, geom_arg<B>(pg, mix_, kMixPx));
  });
  note_launch_end("mask_sup0", s_);
}

// One separable blur of a plane group (tests, one-time mask of the original).
void Butteraugli::fused_blur(const float* in, float* out, int nplanes, int id) {
  const PlaneGeom pg = fused_geom(g_, r_.cr_lo, r_.cr_hi, 0, 0);
  const EpiStore st{out, g_.pitch, g_.plane};
#define GB_BLUR_CASE(R)                                                                                               \
  case R:                                                                                                             \
    launch_roll<R, 1>(s_, MapReq{&fused_->map(in, nplanes, RollCfg<R, 1>::SW, GBR_CH, g_), nullptr}, nplanes, 1,      \
                      t_.blur[id], pg, ht_, id, st, "tma_blur_y");                                                    \
    break;
  switch (t_.blur[id].r) {
    GB_BLUR_CASE(2)
    GB_BLUR_CASE(3)
    GB_BLUR_CASE(4)
    GB_BLUR_CASE(5)
    GB_BLUR_CASE(8)
    GB_BLUR_CASE(16)
    GB_BLUR_CASE(20)
    GB_BLUR_CASE(23)
    default: throw std::runtime_error("blur radius without a compiled kernel");
  }
#undef GB_BLUR_CASE
}

namespace {
bool graphs_enabled() {
  static const bool on = [] {
    const char* e = getenv("GB200_GRAPH");  // GB200_GRAPH=0: plain launches
    return !(e != nullptr && e[0] == '0');
  }();
  return on;
}
}  // namespace

// the launches (no host round trip) / the distance (one)
void Butteraugli::fused_compare_submit() {
  // First call: plain launches (creates the tensor maps, sets the kernel attributes).  Second
  // call: the same sequence is captured into a graph; from then on it is replayed.
  const bool use_graph = graphs_enabled() && !r_.strips() && !profiling_on();
  if (use_graph && fused_->compare_graph != nullptr) {
    GB_CUDA(cudaGraphLaunch(fused_->compare_graph, s_));
    add_launches(fused_->compare_graph_kernels);
  } else if (use_graph && fused_->compare_calls >= 1) {
    const long before = total_launches();
    GB_CUDA(cudaStreamBeginCapture(s_, cudaStreamCaptureModeThreadLocal));
    cudaGraph_t graph = nullptr;
    try {
      fused_compare_launches(1, 0, 0);
    } catch (...) {
      cudaStreamEndCapture(s_, &graph);
      if (graph) cudaGraphDestroy(graph);
      throw;
    }
    GB_CUDA(cudaStreamEndCapture(s_, &graph));
    const long recorded = total_launches() - before;
    add_launches(-recorded);  // recorded, not run
    cudaError_t e = cudaGraphInstantiate(&fused_->compare_graph, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) cuda_fail(e, "cudaGraphInstantiate", __FILE__, __LINE__);
    fused_->compare_graph_kernels = recorded;
    GB_CUDA(cudaGraphLaunch(fused_->compare_graph, s_));
    add_launches(recorded);
  } else {
    fused_compare_launches(1, 0, 0);
  }
  ++fused_->compare_calls;
}

float Butteraugli::fused_compare_result() {
  if (r_.strips()) {
    r_.gather_blocks(block_max_, sizeof(float));  // strip mode: one float per block crosses NVLink
    const int lanes = 1024;
    launch_1d(s_, PartialMax{block_max_, partial_, g_.nblocks, lanes}, lanes, "partial_max");
    float part[1024];
    d2h(part, partial_, sizeof(part), s_);
    float m = 0.0f;
    for (int i = 0; i < lanes; ++i) m = std::max(m, part[i]);
    return m;
  }
  float m = 0.0f;
  d2h(&m, d_gmax_, sizeof(float), s_);
  return m;
}

// the stream work of one Compare after the render: no host synchronisation inside
void Butteraugli::fused_compare_launches(int nimg, int kslot, int kslot0) {
  const PlaneGeom pg = fused_geom(g_, r_.cr_lo, r_.cr_hi, kslot, kslot0);
  const size_t P = g_.plane, S = kslot * P, S0 = kslot0 * P;
  const int rows = r_.cr_hi - r_.cr_lo;
  fused_opsin(lin_, xyb_, nimg, kslot);
  fused_separate(xyb_, ps1_, true, nimg, kslot, kslot0);
  // S10 mask: DiffPrecompute against the original's resident neighbour sums
  {
    dim3 block(32, 8), grid = grid_of(dim3(cdiv(g_.w, 32), cdiv(rows, 8), nimg), mix_, kMixPx);
    note_launch("mask_pre", s_, static_cast<double>(g_.w) * rows * nimg);
    with_batch<void>(nimg, mix_, [&](auto b) {
      constexpr int B = decltype(b)::value;
      k_mask_pre<B><<<grid, block, 0, s_>>>(ps1_, sup0_, mpre_, geom_arg<B>(pg, mix_, kMixPx));
    });
    note_launch_end("mask_pre", s_);
  }
  // x passes of the noise blur (S8) and of the three mask blurs in one launch:
  //   noise_ -> blr_ (r 23);  mpre[X] -> tmp_[0] (r 20);  mpre[Y] -> tmp_[1] (r 20);  mpre[Y] -> tmp_[2] (r 5)
  {
    BlurX4Args<GB_R_NOISE, GB_R_MASKX, GB_R_MASKY1, GB_R_MASKY0> xa;
    xa.out[0] = blr_;
    xa.out[1] = tmp_;
    xa.out[2] = tmp_ + P;
    xa.out[3] = tmp_ + 2 * P;
    xa.scale_x[0] = tab_of(t_, mix_, kBlurNoise).scale_x;
    xa.scale_x[1] = tab_of(t_, mix_, kBlurMaskX).scale_x;
    xa.scale_x[2] = tab_of(t_, mix_, kBlurMaskY1).scale_x;
    xa.scale_x[3] = tab_of(t_, mix_, kBlurMaskY0).scale_x;
    xa.k0 = make_blurk<GB_R_NOISE>(ht_, kBlurNoise);
    xa.k1 = make_blurk<GB_R_MASKX>(ht_, kBlurMaskX);
    xa.k2 = make_blurk<GB_R_MASKY1>(ht_, kBlurMaskY1);
    xa.k3 = make_blurk<GB_R_MASKY0>(ht_, kBlurMaskY0);
    const dim3 grid = grid_of(dim3(cdiv(g_.w, GBX_TW), cdiv(rows, GBX_TH), 4 * nimg), mix_, kMixX4);
    note_launch("tma_blur_x", s_, 4.0 * g_.w * rows * nimg);
    const MapReq m0 = maps(noise_, 1, BlurXCfg<GB_R_NOISE>::SW, GBX_TH, kslot);
    const MapReq m1 = maps(mpre_, 1, BlurXCfg<GB_R_MASKX>::SW, GBX_TH, kslot);
    const MapReq m2 = maps(mpre_ + P, 1, BlurXCfg<GB_R_MASKY1>::SW, GBX_TH, kslot);
    const MapReq m3 = maps(mpre_ + P, 1, BlurXCfg<GB_R_MASKY0>::SW, GBX_TH, kslot);
    with_batch<void>(nimg, mix_, [&](auto b) {
      constexpr int B = decltype(b)::value;
      k_tma_blur_x4<B, GB_R_NOISE, GB_R_MASKX, GB_R_MASKY1, GB_R_MASKY0>
          <<<grid, 128, 0, s_>>>(m0.get<B>(), m1.get<B>(), m2.get<B>(), m3.get<B>(), geom_arg<B>(pg, mix_, kMixX4), xa);
    });
    note_launch_end("tma_blur_x", s_);
  }
  // S7 Malta line sums of both channels: ac[ch] = ((0 + uhf) + hf) + mf
  {
    dim3 block(16, 16);
    const dim3 grid = grid_of(dim3(cdiv(g_.w, GB_MALTA_TILE_W), cdiv(rows, GB_MALTA_TILE_H), 2 * nimg), mix_, kMixMalta);
    note_launch("malta_sums", s_, 2.0 * g_.w * rows * nimg);
    const MapReq m = maps(diffs6_, 6, GB_MALTA_SW, GB_MALTA_SH, kslot);
    with_batch<void>(nimg, mix_, [&](auto b) {
      constexpr int B = decltype(b)::value;
      k_tma_malta_sums<B><<<grid, block, 0, s_>>>(m.get<B>(), ac_, geom_arg<B>(pg, mix_, kMixMalta));
    });
    note_launch_end("malta_sums", s_);
  }
  // S8 tail + S9 on block_diff_ac[Y]: blurred noise difference, asymmetric L2 of hf[Y]
  launch_tma_y<GB_R_NOISE, 1>(s_, maps(blr_, 1, GBY_TW, GBY_TH + 2 * GB_R_NOISE, kslot), 1, nimg,
                              tab_of(t_, mix_, kBlurNoise), pg, ht_, kBlurNoise,
                              EpiNoise{ps0_ + kHfY * P, ps1_ + kHfY * P, ac_ + P, asym_w0_, asym_w1_, g_.pitch, S, S0},
                              "noise_fused_y", mix_, kMixY);
  // y passes + S11 CombineChannels + first half of S12 -> dm_[1]
  {
    typedef MaskYCfg<GB_R_MASKX, GB_R_MASKY0, GB_R_MASKY1> C;
    CombineArgs ca{ps0_, ps1_, ac_, dm_ + P, t_.mask_lut, g_.pitch, P};
    const dim3 grid = grid_of(dim3(cdiv(g_.w, GBY_TW), cdiv(rows, GBY_TH), nimg), mix_, kMixY);
    note_launch("mask_y_combine", s_, static_cast<double>(g_.w) * rows * nimg);
    const MapReq ma = maps(tmp_, 1, GBY_TW, C::HA, kslot), mb = maps(tmp_ + 2 * P, 1, GBY_TW, C::HB, kslot),
                 mc = maps(tmp_ + P, 1, GBY_TW, C::HC, kslot);
    with_batch<void>(nimg, mix_, [&](auto b) {
      constexpr int B = decltype(b)::value;
      allow_smem(k_tma_mask_y<B, GB_R_MASKX, GB_R_MASKY0, GB_R_MASKY1>, C::kSmemBytes);
      k_tma_mask_y<B, GB_R_MASKX, GB_R_MASKY0, GB_R_MASKY1><<<grid, 256, C::kSmemBytes, s_>>>(
          ma.get<B>(), mb.get<B>(), mc.get<B>(), tab_of(t_, mix_, kBlurMaskX).scale_y,
          tab_of(t_, mix_, kBlurMaskY0).scale_y, tab_of(t_, mix_, kBlurMaskY1).scale_y, geom_arg<B>(pg, mix_, kMixY),
          make_blurk<GB_R_MASKX>(ht_, kBlurMaskX), make_blurk<GB_R_MASKY0>(ht_, kBlurMaskY0),
          make_blurk<GB_R_MASKY1>(ht_, kBlurMaskY1), ca);
    });
    note_launch_end("mask_y_combine", s_);
  }
  // S12 second half + S13: blur 1.73, mix, per-block maxima, global maximum (one per image)
  // (a mixed pass: the slots n0 ..; their block maxima keep the batch's block grid, and only the
  // global maxima are read)
  dev_zero(d_gmax_ + (mix_ ? mix_->n0 : 0), sizeof(unsigned int) * nimg, s_);
  {
    typedef Blur2dCfg<GB_R_FINAL, 1> C;
    EpiFinal ef{dm_, block_max_, r_.strips() ? nullptr : d_gmax_, g_.pitch, g_.bw, r_.by_lo, r_.by_hi, S, g_.nblocks};
    launch_tma_2d<GB_R_FINAL, 1>(s_, maps(dm_ + P, 1, C::SWI, C::HI, kslot), nimg, tab_of(t_, mix_, kBlurFinal), pg, ht_,
                                 kBlurFinal, ef, "final_fused", mix_);
  }
}

void Butteraugli::fused_compare_batch(const float* rgb0, const float* rgb1, int n, float* diffmap, float* maxima) {
  const size_t row = sizeof(float) * g_.w, pitch = sizeof(float) * g_.pitch;
  const size_t slot_rows = static_cast<size_t>(kslot_) * g_.h;  // a plane is h rows of pitch
  if (rgb0 != nullptr) {
    // [n][3][h][w] -> the lin planes of slots 0 .. n - 1: n slices of 3h rows
    copy_3d(lin_, pitch, slot_rows, rgb0, row, static_cast<size_t>(3) * g_.h, row, static_cast<size_t>(3) * g_.h, n, s_);
    // PsychoImage of every original (butteraugli.cc:784) and its DiffPrecompute neighbour sums
    fused_opsin(lin_, xyb_, n, kslot_);
    fused_separate(xyb_, ps0_, false, n, kslot_, kslot_);
    fused_sup0(n, kslot_);
  }
  copy_3d(lin_, pitch, slot_rows, rgb1, row, static_cast<size_t>(3) * g_.h, row, static_cast<size_t>(3) * g_.h, n, s_);
  fused_compare_launches(n, kslot_, rgb0 != nullptr ? kslot_ : 0);
  if (diffmap != nullptr) copy_3d(diffmap, row, g_.h, dm_, pitch, slot_rows, row, g_.h, n, s_);
  // one transfer of the n maxima (float bits); d2h waits for it, and so for everything queued before
  d2h(maxima, d_gmax_, sizeof(float) * n, s_);
}

// ---- pairs of different sizes (compare_batch_sizes) ----
// The buffers of the mixed calls, grown to the largest call so far and kept: the tables of a run
// (images, work items, row counts, pointers and border scales of every pass, one upload), the staging
// of host images (float or 8-bit) and of diffmaps (host output; an 8-bit call's diffmaps over white), and
// the border scales of every size seen (host libm, once per size).
struct Butteraugli::Mixed {
  std::vector<unsigned char> blob;  // host image of `tables`
  void* tables = nullptr;
  size_t tables_bytes = 0;
  std::vector<unsigned char> host_in;  // host images, packed
  unsigned char* stage_in = nullptr;
  size_t stage_in_bytes = 0;
  float* stage_dm = nullptr;
  size_t stage_dm_floats = 0;
  std::map<std::pair<int, int>, std::vector<float> > scales;  // size -> [blur][w + h] (scale_x, then scale_y)
};

void Butteraugli::mixed_release() {
  if (mixed_ == nullptr) return;
  dev_free(mixed_->tables);
  dev_free(mixed_->stage_in);
  dev_free(mixed_->stage_dm);
  delete mixed_;
  mixed_ = nullptr;
}

namespace {
// device buffer of at least `want` elements, grown (its contents are not kept)
template <class T>
T* grow(T* p, size_t* have, size_t want) {
  if (want <= *have && p != nullptr) return p;
  dev_free(p);
  *have = 0;
  p = static_cast<T*>(dev_alloc(sizeof(T) * std::max<size_t>(want, 1)));
  *have = want;
  return p;
}
size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
}  // namespace

// The images of a mixed run, per pair index, in memory of this device: float planes [3][h][w] (channels
// null), or 8-bit pixels [h][w][channels] laid over `background`.  store: a comparator set's run, the
// analysis of pair i's original in the set's store (kStoredPlanes planes [h][w]); img[0] is then unused.
struct MixSrc {
  const void* const* img[2] = {nullptr, nullptr};
  const int* channels = nullptr;
  int background = 0;
  float* const* store = nullptr;
};

void Butteraugli::fused_compare_sizes(const int* w, const int* h, const int* channels, const void* const* in0,
                                      const void* const* in1, int n, float* const* diffmap, float* maxima,
                                      bool device, float* const* const* stored) {
  if (mixed_ == nullptr) mixed_ = new Mixed();
  Mixed& mx = *mixed_;
  if (channels != nullptr && t_.srgb_lin == nullptr) t_.srgb_lin = upload_srgb_lin(s_, &owned_, nullptr);
  const auto in_bytes = [&](int i) {  // of one image of pair i
    return static_cast<size_t>(w[i]) * h[i] * (channels != nullptr ? channels[i] : 3 * sizeof(float));
  };
  const int sides = stored != nullptr ? 1 : 2;  // a comparator set's originals are in its store
  std::vector<int> all(n), rgba;
  std::vector<const void*> p0(n), p1(in1, in1 + n);
  if (in0 != nullptr) p0.assign(in0, in0 + n);
  // input staging: byte offset of pair i on one side; diffmap staging: host output, black's diffmaps of
  // every pair, then white's of the RGBA pairs with a diffmap; device output, white's alone (black's go to
  // the caller's memory)
  std::vector<size_t> in_at(n), at(n), at_white(n);
  size_t px = 0, px_white = 0, bytes = 0;
  for (int i = 0; i < n; ++i) {
    all[i] = i;
    in_at[i] = bytes;
    at[i] = px;
    px += static_cast<size_t>(w[i]) * h[i];
    bytes += in_bytes(i);
    if (channels == nullptr || channels[i] != 4) continue;
    rgba.push_back(i);
    if (diffmap != nullptr && diffmap[i] != nullptr) {
      at_white[i] = px_white;
      px_white += static_cast<size_t>(w[i]) * h[i];
    }
  }
  if (!device) {  // host images: packed once, uploaded in one copy (for both backgrounds), side 0 then side 1
    const size_t at1 = (sides - 1) * bytes;
    mx.stage_in = grow(mx.stage_in, &mx.stage_in_bytes, sides * bytes);
    mx.host_in.resize(sides * bytes);
    for (int i = 0; i < n; ++i) {
      if (sides == 2) {
        memcpy(&mx.host_in[in_at[i]], in0[i], in_bytes(i));
        p0[i] = mx.stage_in + in_at[i];
      }
      memcpy(&mx.host_in[at1 + in_at[i]], in1[i], in_bytes(i));
      p1[i] = mx.stage_in + at1 + in_at[i];
    }
    h2d(mx.stage_in, mx.host_in.data(), sides * bytes, s_);
  }
  const size_t black = diffmap != nullptr && !device ? px : 0;
  if (black + px_white > 0) mx.stage_dm = grow(mx.stage_dm, &mx.stage_dm_floats, black + px_white);
  std::vector<float*> dst(n, nullptr), dst_white(n, nullptr);
  if (diffmap != nullptr)
    for (int i = 0; i < n; ++i) {
      if (diffmap[i] == nullptr) continue;
      dst[i] = device ? diffmap[i] : mx.stage_dm + at[i];
      if (channels != nullptr && channels[i] == 4) dst_white[i] = mx.stage_dm + black + at_white[i];
    }
  MixSrc src;
  src.img[0] = p0.data();
  src.img[1] = p1.data();
  src.channels = channels;
  if (stored != nullptr) src.store = stored[0];
  fused_mixed_run(w, h, all, src, dst.data(), maxima);
  // RGBA pairs over white: a run of their own (their sizes make its passes); where white wins, its score
  // and diffmap replace black's
  std::vector<char> white_won(n, 0);
  if (!rgba.empty()) {
    std::vector<float> m_white(n);
    src.background = 255;
    if (stored != nullptr) src.store = stored[1];
    fused_mixed_run(w, h, rgba, src, dst_white.data(), m_white.data());
    bool copied = false;
    for (int i : rgba) {
      if (!white_wins(m_white[i], maxima[i])) continue;
      maxima[i] = m_white[i];
      white_won[i] = 1;
      if (device && dst_white[i] != nullptr) {
        d2d(diffmap[i], dst_white[i], sizeof(float) * w[i] * h[i], s_);
        copied = true;
      }
    }
    if (copied) stream_sync(s_);  // the white diffmaps copied into the caller's memory
  }
  if (diffmap != nullptr && !device) {
    std::vector<float> dm(black + px_white);
    d2h(dm.data(), mx.stage_dm, sizeof(float) * dm.size(), s_);
    for (int i = 0; i < n; ++i)
      if (diffmap[i] != nullptr)
        memcpy(diffmap[i], &dm[white_won[i] ? black + at_white[i] : at[i]], sizeof(float) * w[i] * h[i]);
  }
}

namespace {
// the geometry argument of a row-copy launch over a mixed pass's images
PlaneGeomMix mix_geom(const Geom& g, int kslot, const MixPass& p) {
  PlaneGeomMix pg;
  static_cast<PlaneGeom&>(pg) = fused_geom(g, 0, g.h, kslot, kslot);
  pg.mix = p.geom(0);
  return pg;
}
// mix_ is only set while a pass's launches are queued
struct MixScope {
  MixPass** p;
  ~MixScope() { *p = nullptr; }
};
}  // namespace

std::vector<MixPass> Butteraugli::mixed_passes(const int* w, const int* h, const std::vector<int>& pairs,
                                               const MixSrc& src, float* const* dst, std::vector<int>* order_out) {
  Mixed& mx = *mixed_;
  const bool u8 = src.channels != nullptr;
  // The per-size caches (border scales here, tensor maps in Fused::maps) are bounded: once they hold more
  // than kMixCachedSizes sizes, a run starts by dropping them.  No launch of an earlier run reads them
  // any more (its maps went into its launch parameters), and this run rebuilds what it uses.
  constexpr size_t kMixCachedSizes = 256;
  if (mx.scales.size() > kMixCachedSizes) {
    mx.scales.clear();
    fused_->drop_other_sizes(g_);
  }
  // Slots in the order of the sizes, so that a pass (at most GB_MIX_SHAPES sizes) is a run of slots.
  const int n = static_cast<int>(pairs.size());
  std::vector<int>& order = *order_out;
  order = pairs;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return std::make_pair(w[a], h[a]) < std::make_pair(w[b], h[b]); });
  std::vector<MixPass> passes;
  for (int k = 0; k < n; ++k) {
    const std::pair<int, int> sz(w[order[k]], h[order[k]]);
    const bool new_size = k == 0 || sz != std::make_pair(w[order[k - 1]], h[order[k - 1]]);
    if (k == 0 || (new_size && passes.back().shapes.size() == GB_MIX_SHAPES)) {
      passes.emplace_back();
      passes.back().n0 = k;
    }
    MixPass& p = passes.back();
    if (new_size) p.shapes.push_back(sz);
    ++p.m;
  }
  // The tables of every pass, laid out in one blob (offsets first, pointers filled once it has an address).
  // A comparator set's run adds the rows and pointers of its originals' analyses at the end.
  struct Layout {
    size_t img, tile0, rows_in, rows_dm, ext0, ext1, extdm, scales, blur_len, rows_org, extorg;
  };
  std::vector<Layout> lay(passes.size());
  size_t bytes = 0;
  for (size_t q = 0; q < passes.size(); ++q) {
    const MixPass& p = passes[q];
    Layout& l = lay[q];
    size_t len = 0;
    for (const std::pair<int, int>& sz : p.shapes) len += sz.first + sz.second;
    l.blur_len = len;
    l.img = bytes = align_up(bytes, 32);
    bytes += sizeof(MixImage) * p.m;
    l.tile0 = bytes = align_up(bytes, 16);
    bytes += sizeof(int) * kMixKinds * (p.m + 1);
    l.rows_in = bytes;
    bytes += sizeof(int) * (p.m + 1);
    l.rows_dm = bytes;
    bytes += sizeof(int) * (p.m + 1);
    l.ext0 = bytes = align_up(bytes, 16);
    bytes += sizeof(void*) * p.m;
    l.ext1 = bytes;
    bytes += sizeof(void*) * p.m;
    l.extdm = bytes;
    bytes += sizeof(float*) * p.m;
    l.scales = bytes = align_up(bytes, 16);
    bytes += sizeof(float) * kNumBlurs * len;
    if (src.store != nullptr) {
      l.rows_org = bytes;
      bytes += sizeof(int) * (p.m + 1);
      l.extorg = bytes = align_up(bytes, 16);
      bytes += sizeof(float*) * p.m;
    }
  }
  mx.tables = grow(static_cast<unsigned char*>(mx.tables), &mx.tables_bytes, bytes);
  mx.blob.assign(bytes, 0);
  unsigned char* dev = static_cast<unsigned char*>(mx.tables);
  // tile shapes of the chain's launches (th 0: the image's rolling-blur segment) and images per tile z
  static const int kTile[kMixKinds][3] = {{GB2_TW, GB2_TH, 1}, {GBR_TW, 0, 3},  {GBR_TW, 0, 1},
                                          {32, 8, 1},          {GBX_TW, GBX_TH, 4}, {GB_MALTA_TILE_W, GB_MALTA_TILE_H, 2},
                                          {GBY_TW, GBY_TH, 1}};
  for (size_t q = 0; q < passes.size(); ++q) {
    MixPass& p = passes[q];
    const Layout& l = lay[q];
    unsigned char* b = mx.blob.data();
    MixImage* img = reinterpret_cast<MixImage*>(b + l.img);
    int* tile0 = reinterpret_cast<int*>(b + l.tile0);
    int* rows_in = reinterpret_cast<int*>(b + l.rows_in);
    int* rows_dm = reinterpret_cast<int*>(b + l.rows_dm);
    void** ext0 = reinterpret_cast<void**>(b + l.ext0);
    void** ext1 = reinterpret_cast<void**>(b + l.ext1);
    float** extdm = reinterpret_cast<float**>(b + l.extdm);
    float* sc = reinterpret_cast<float*>(b + l.scales);
    int* rows_org = src.store != nullptr ? reinterpret_cast<int*>(b + l.rows_org) : nullptr;
    float** extorg = src.store != nullptr ? reinterpret_cast<float**>(b + l.extorg) : nullptr;
    // border scales: per blur, scale_x of every size, then scale_y of every size
    std::vector<int> sxo(p.shapes.size()), syo(p.shapes.size());
    size_t ox = 0, oy = 0, xsum = 0;
    for (const std::pair<int, int>& sz : p.shapes) xsum += sz.first;
    for (size_t s = 0; s < p.shapes.size(); ++s) {
      const int sw = p.shapes[s].first, sh = p.shapes[s].second;
      std::vector<float>& cached = mx.scales[p.shapes[s]];
      if (cached.empty()) {
        for (int id = 0; id < kNumBlurs; ++id) {
          const std::vector<float> x = blur_axis_scales(id, sw), y = blur_axis_scales(id, sh);
          cached.insert(cached.end(), x.begin(), x.end());
          cached.insert(cached.end(), y.begin(), y.end());
        }
      }
      sxo[s] = static_cast<int>(ox);
      syo[s] = static_cast<int>(xsum + oy);
      for (int id = 0; id < kNumBlurs; ++id) {
        const float* c = &cached[static_cast<size_t>(id) * (sw + sh)];
        memcpy(sc + id * l.blur_len + sxo[s], c, sizeof(float) * sw);
        memcpy(sc + id * l.blur_len + syo[s], c + sw, sizeof(float) * sh);
      }
      ox += sw;
      oy += sh;
    }
    for (int id = 0; id < kNumBlurs; ++id) {
      p.tab[id] = t_.blur[id];
      p.tab[id].scale_x = p.tab[id].scale_y = reinterpret_cast<const float*>(dev + l.scales) + id * l.blur_len;
    }
    int shape = -1;
    rows_in[0] = rows_dm[0] = 0;
    if (rows_org != nullptr) rows_org[0] = 0;
    for (int kind = 0; kind < kMixKinds; ++kind) tile0[kind * (p.m + 1)] = 0;
    for (int j = 0; j < p.m; ++j) {
      const int i = order[p.n0 + j], iw = w[i], ih = h[i];
      if (j == 0 || std::make_pair(iw, ih) != p.shapes[shape]) ++shape;
      MixImage& im = img[j];
      im.w = iw;
      im.h = ih;
      im.shape = shape;
      im.sx = sxo[shape];
      im.sy = syo[shape];
      im.seg = roll_seg(ih);
      im.channels = u8 ? src.channels[i] : 3;
      for (int kind = 0; kind < kMixKinds; ++kind) {
        const int th = kTile[kind][1] ? kTile[kind][1] : im.seg;
        const long long items = static_cast<long long>(cdiv(iw, kTile[kind][0])) * cdiv(ih, th) * kTile[kind][2];
        int* t = tile0 + kind * (p.m + 1);
        if (t[j] + items > 0x7fffffffLL) throw std::runtime_error("butteraugli batch: too many tiles in one call");
        t[j + 1] = t[j] + static_cast<int>(items);
      }
      // packing rows: 3h plane rows of float planes, h pixel rows of 8-bit images; unpacking: h rows of
      // the images with a diffmap
      const bool has_dm = dst != nullptr && dst[i] != nullptr;
      rows_in[j + 1] = rows_in[j] + (u8 ? ih : 3 * ih);
      rows_dm[j + 1] = rows_dm[j] + (has_dm ? ih : 0);
      ext0[j] = src.img[0] != nullptr ? const_cast<void*>(src.img[0][i]) : nullptr;
      ext1[j] = src.img[1] != nullptr ? const_cast<void*>(src.img[1][i]) : nullptr;
      extdm[j] = has_dm ? dst[i] : nullptr;
      if (rows_org != nullptr) {
        rows_org[j + 1] = rows_org[j] + kStoredPlanes * ih;
        extorg[j] = src.store[i];
      }
    }
    p.img = reinterpret_cast<const MixImage*>(dev + l.img);
    p.tile0 = reinterpret_cast<const int*>(dev + l.tile0);
    p.rows_in = reinterpret_cast<const int*>(dev + l.rows_in);
    p.rows_dm = reinterpret_cast<const int*>(dev + l.rows_dm);
    p.ext0 = reinterpret_cast<void* const*>(dev + l.ext0);
    p.ext1 = reinterpret_cast<void* const*>(dev + l.ext1);
    p.extdm = reinterpret_cast<float* const*>(dev + l.extdm);
    for (int kind = 0; kind < kMixKinds; ++kind) p.total[kind] = tile0[kind * (p.m + 1) + p.m];
    p.rows_in_total = rows_in[p.m];
    p.rows_dm_total = rows_dm[p.m];
    if (rows_org != nullptr) {
      p.rows_org = reinterpret_cast<const int*>(dev + l.rows_org);
      p.extorg = reinterpret_cast<float* const*>(dev + l.extorg);
      p.rows_org_total = rows_org[p.m];
    }
  }
  h2d(mx.tables, mx.blob.data(), bytes, s_);
  return passes;
}

// one side's images into the lin planes of the pass's slots
void Butteraugli::mixed_pack(const MixPass& p, void* const* ext, const MixSrc& src) {
  const PlaneGeomMix pg = mix_geom(g_, kslot_, p);
  const int total = p.rows_in_total;
  if (src.channels != nullptr) {
    note_launch("mix_pack_srgb", s_, static_cast<double>(total));
    k_mix_srgb<<<cdiv(total, 8), 256, 0, s_>>>(reinterpret_cast<const uint8_t* const*>(ext), p.rows_in,
                                               src.background, t_.srgb_lin, lin_, pg);
    note_launch_end("mix_pack_srgb", s_);
  } else {
    note_launch("mix_pack", s_, static_cast<double>(total));
    k_mix_rows<true><<<cdiv(total, 8), 256, 0, s_>>>(reinterpret_cast<float* const*>(ext), p.rows_in, lin_, pg);
    note_launch_end("mix_pack", s_);
  }
}

// the analyses of a comparator set's originals between its store and the ps0 and sup0 planes of the pass's
// slots
void Butteraugli::mixed_original(const MixPass& p, bool to_arena) {
  const PlaneGeomMix pg = mix_geom(g_, kslot_, p);
  const int rows = p.rows_org_total;
  const char* name = to_arena ? "mix_gather_original" : "mix_store_original";
  note_launch(name, s_, static_cast<double>(rows));
  if (to_arena) {
    k_mix_original<true><<<cdiv(rows, 8), 256, 0, s_>>>(p.extorg, p.rows_org, ps0_, sup0_, pg);
  } else {
    k_mix_original<false><<<cdiv(rows, 8), 256, 0, s_>>>(p.extorg, p.rows_org, ps0_, sup0_, pg);
  }
  note_launch_end(name, s_);
}

void Butteraugli::fused_mixed_run(const int* w, const int* h, const std::vector<int>& pairs, const MixSrc& src,
                                  float* const* dst, float* maxima) {
  std::vector<int> order;
  std::vector<MixPass> passes = mixed_passes(w, h, pairs, src, dst, &order);
  // one pass of the chain per run of at most GB_MIX_SHAPES sizes
  MixScope scope{&mix_};
  for (MixPass& p : passes) {
    mix_ = &p;
    if (src.store != nullptr) {  // a comparator set's originals, analysed when it was made
      mixed_original(p, true);
    } else {  // PsychoImage of every original and its DiffPrecompute neighbour sums
      mixed_pack(p, p.ext0, src);
      fused_opsin(lin_, xyb_, p.m, kslot_);
      fused_separate(xyb_, ps0_, false, p.m, kslot_, kslot_);
      fused_sup0(p.m, kslot_);
    }
    mixed_pack(p, p.ext1, src);
    fused_compare_launches(p.m, kslot_, kslot_);
    if (p.rows_dm_total > 0) {
      note_launch("mix_unpack", s_, static_cast<double>(p.rows_dm_total));
      k_mix_rows<false><<<cdiv(p.rows_dm_total, 8), 256, 0, s_>>>(p.extdm, p.rows_dm, dm_, mix_geom(g_, kslot_, p));
      note_launch_end("mix_unpack", s_);
    }
  }
  // one transfer of the n maxima (float bits), which waits for everything queued before
  const int n = static_cast<int>(pairs.size());
  std::vector<float> m(n);
  d2h(m.data(), d_gmax_, sizeof(float) * n, s_);
  for (int k = 0; k < n; ++k) maxima[order[k]] = m[k];
}

void Butteraugli::analyse_originals(const int* w, const int* h, const int* channels, const void* const* img0, int n,
                                    int background, float* const* store, bool device) {
  check_sizes(w, h, n);
  bind();
  if (mixed_ == nullptr) mixed_ = new Mixed();
  Mixed& mx = *mixed_;
  if (channels != nullptr && t_.srgb_lin == nullptr) t_.srgb_lin = upload_srgb_lin(s_, &owned_, nullptr);
  std::vector<const void*> p0(img0, img0 + n);
  std::vector<int> all(n);
  for (int i = 0; i < n; ++i) all[i] = i;
  if (!device) {  // the originals packed and uploaded in one copy
    std::vector<size_t> at(n + 1, 0);
    for (int i = 0; i < n; ++i)
      at[i + 1] = at[i] + static_cast<size_t>(w[i]) * h[i] * (channels != nullptr ? channels[i] : 3 * sizeof(float));
    mx.stage_in = grow(mx.stage_in, &mx.stage_in_bytes, at[n]);
    mx.host_in.resize(at[n]);
    for (int i = 0; i < n; ++i) {
      memcpy(&mx.host_in[at[i]], img0[i], at[i + 1] - at[i]);
      p0[i] = mx.stage_in + at[i];
    }
    h2d(mx.stage_in, mx.host_in.data(), at[n], s_);
  }
  MixSrc src;
  src.img[0] = p0.data();
  src.channels = channels;
  src.background = background;
  src.store = store;
  std::vector<int> order;
  std::vector<MixPass> passes = mixed_passes(w, h, all, src, nullptr, &order);
  MixScope scope{&mix_};
  for (MixPass& p : passes) {
    mix_ = &p;
    mixed_pack(p, p.ext0, src);
    fused_opsin(lin_, xyb_, p.m, kslot_);
    fused_separate(xyb_, ps0_, false, p.m, kslot_, kslot_);
    fused_sup0(p.m, kslot_);
    mixed_original(p, false);
  }
  stream_sync(s_);
}

void Butteraugli::compare_originals(const int* w, const int* h, const int* channels, float* const* const* stored,
                                    const void* const* img1, int n, float* const* diffmap, float* maxima, bool device,
                                    Stream caller) {
  check_sizes(w, h, n);
  bind();
  if (device) stream_wait(s_, caller);
  fused_compare_sizes(w, h, channels, nullptr, img1, n, diffmap, maxima, device, stored);
}

// The stage entries on the fused chain.
void Butteraugli::blur(const float* in, float* out, int nplanes, int id) { fused_blur(in, out, nplanes, id); }
void Butteraugli::opsin(const float* lin, float* xyb) { fused_opsin(lin, xyb, 1, 0); }
void Butteraugli::separate(const float* xyb, float* ps) { fused_separate(xyb, ps, false, 1, 0, 0); }

float Butteraugli::compare() {
  bind();
  fused_compare_submit();
  return fused_compare_result();
}

#endif  // !GB200_HOSTSIM

// The mask (Butteraugli members).
void Butteraugli::mask_activity(const float* xy) {
  r_.px(MaskDiffPreSelf{xy, mpre_, g_}, "mask_diff_pre_self");
  blur(mpre_, sact_, 1, kBlurMaskX);
  blur(mpre_ + g_.plane, sact_ + g_.plane, 1, kBlurMaskY0);
  blur(mpre_ + g_.plane, sact_ + 2 * g_.plane, 1, kBlurMaskY1);
}

void Butteraugli::mask_planes(const float* xy) {
  if (mask_ == nullptr) mask_ = planes(6);
  mask_activity(xy);
  r_.px(MaskPlanes{sact_, sact_ + g_.plane, sact_ + 2 * g_.plane, mask_, mask_ + 3 * g_.plane, g_, t_.mask_lut},
        "mask_planes");
}

void Butteraugli::mask(float* mask, float* mask_dc, bool device, Stream caller) {
  bind();
  if (device) stream_wait(s_, caller);
  // MaskPsychoImage(pi0_, pi0_) (b/butteraugli.cc:753): the mixed X and Y planes go to xyb_, which
  // every Compare rewrites before reading it
  r_.px(MaskPsychoMix{ps0_, xyb_, g_}, "mask_psycho_mix");
  mask_planes(xyb_);
  if (!device) {
    r_.download_planes(mask_, mask, 3);
    r_.download_planes(mask_ + 3 * g_.plane, mask_dc, 3);
    return;
  }
  // [3][h][pitch] -> [3][h][w], each group as 3h rows
  const size_t row = sizeof(float) * g_.w, pitch = sizeof(float) * g_.pitch, rows = static_cast<size_t>(3) * g_.h;
  d2d_2d(mask, row, mask_, pitch, row, rows, s_);
  d2d_2d(mask_dc, row, mask_ + 3 * g_.plane, pitch, row, rows, s_);
  stream_sync(s_);
}

void Butteraugli::srgb_to_linear(const uint8_t* src, int n, int channels, int background, float* dst, int pitch) {
  // a launch covers at most 65535 * 8 rows (launch_2d's grid y), so large batches go in parts
  const int per = std::max(1, 65535 * 8 / g_.h);
  const size_t in = static_cast<size_t>(g_.w) * g_.h * channels, out = static_cast<size_t>(3) * g_.h * pitch;
  for (int i = 0; i < n; i += per) {
    const int k = std::min(per, n - i);
    launch_2d(s_, SrgbToLinear{src + i * in, channels, background, dst + i * out, g_.w, g_.h, pitch, t_.srgb_lin},
              g_.w, k * g_.h, "srgb_to_linear");
  }
}

#if defined(GB200_HOSTSIM)
// The CPU port's Compare chain: one launch per stage of the functors of kernels.h.
void Butteraugli::blur(const float* in, float* out, int nplanes, int id) {
  r_.px(BlurX{in, tmp_, t_.blur[id], g_}, "blur_x", nplanes);
  r_.px(BlurY{tmp_, out, t_.blur[id], g_}, "blur_y", nplanes);
}

void Butteraugli::opsin(const float* lin, float* xyb) {
  blur(lin, blr_, 3, kBlurOpsin);
  r_.px(OpsinPx{lin, blr_, xyb, g_}, "opsin_px");
}

void Butteraugli::separate(const float* xyb, float* ps) {
  blur(xyb, lf_, 3, kBlurLf);
  r_.px(SubPlanes{xyb, lf_, mf_in_, g_}, "sub_planes", 3);
  blur(mf_in_, mf_blr_, 3, kBlurMf);
  r_.px(SplitMfHf{mf_in_, mf_blr_, ps, hf_raw_, g_}, "split_mf_hf");
  blur(hf_raw_, hf_blr_, 2, kBlurHf);
  r_.px(SplitHfUhf{hf_raw_, hf_blr_, lf_, ps, g_}, "split_hf_uhf");
}

// S1..S13 on the linear RGB planes in lin_ (butteraugli::ButteraugliComparator::Diffmap).
float Butteraugli::compare() {
  const size_t P = g_.plane;
  opsin(lin_, xyb_);
  separate(xyb_, ps1_);
  // S7 Malta: uhf[Y], uhf[X] with 9-tap lines; hf[Y], hf[X], mf[Y], mf[X] with 5-tap lines
  static const int kMaltaPlane[6] = {kUhfY, kUhfX, kHfY, kHfX, kMfY, kMfX};
  static const int kMaltaAcc[6] = {1, 0, 1, 0, 1, 0};
  for (int i = 0; i < 6; ++i) {
    const int pl = kMaltaPlane[i];
    r_.px(MaltaPre{ps0_ + pl * P, ps1_ + pl * P, diffs_, malta_[i], g_}, "malta_pre");
    MaltaAcc acc;
    acc.diffs = diffs_;
    acc.acc = ac_ + kMaltaAcc[i] * P;
    acc.pat = i < 2 ? t_.malta_hf : t_.malta_lf;
    acc.pat_len = i < 2 ? t_.malta_hf_len : nullptr;
    acc.stride = i < 2 ? 9 : 5;
    acc.first = i < 2 ? 1 : 0;
    acc.g = g_;
    r_.px(acc, i < 2 ? "malta_acc_hf" : "malta_acc_lf");
  }
  // S8 + S9 on block_diff_ac[Y]
  r_.px(NoisePre{ps0_ + kHfY * P, ps1_ + kHfY * P, noise_, g_}, "noise_pre");
  blur(noise_, noise_ + P, 1, kBlurNoise);
  r_.px(NoiseAndAsymAcc{noise_ + P, ps0_ + kHfY * P, ps1_ + kHfY * P, ac_ + P, asym_w0_, asym_w1_, g_},
        "noise_asym_acc");
  // S10 mask
  r_.px(MaskDiffPre{ps0_, ps1_, mpre_, g_}, "mask_diff_pre");
  blur(mpre_, sact_, 1, kBlurMaskX);
  blur(mpre_ + P, sact_ + P, 1, kBlurMaskY0);
  blur(mpre_ + P, sact_ + 2 * P, 1, kBlurMaskY1);
  // S11 + S12
  r_.px(CombineAndSqrt{ps0_, ps1_, ac_, sact_, sact_ + P, sact_ + 2 * P, dm_, g_, t_.mask_lut}, "combine_sqrt");
  blur(dm_, dm_ + P, 1, kBlurFinal);
  r_.px(DiffmapMix{dm_ + P, dm_, g_}, "diffmap_mix");
  // S13 + a15 first half
  r_.block_rows(BlockMax{dm_, block_max_, g_}, "block_max", r_.by_lo, r_.by_hi);
  r_.gather_blocks(block_max_, sizeof(float));  // strip mode: one float per block crosses NVLink
  const int lanes = 1024;
  launch_1d(s_, PartialMax{block_max_, partial_, g_.nblocks, lanes}, lanes, "partial_max");
  float part[1024];
  d2h(part, partial_, sizeof(part), s_);
  float m = 0.0f;
  for (int i = 0; i < lanes; ++i) m = std::max(m, part[i]);
  return m;
}

#endif  // GB200_HOSTSIM

ImageContext::ImageContext(const uint8_t* rgb, int w, int h, int device, bool prepare_now, Comm* comm)
    : ba_(w, h, device, comm) {
  guarded_init(rgb, nullptr, prepare_now);
}

ImageContext::ImageContext(const int16_t* dq_coeffs, int w, int h, int device, bool prepare_now, Comm* comm)
    : ba_(w, h, device, comm) {
  from_coeffs_ = true;
  guarded_init(nullptr, dq_coeffs, prepare_now);
}

ImageContext::ImageContext(const int16_t* dq_dev, Stream stream, int w, int h, int device, bool prepare_now)
    : ba_(w, h, device, nullptr) {
  from_coeffs_ = true;
  dq_on_device_ = true;
  dq_stream_ = stream;
  guarded_init(nullptr, dq_dev, prepare_now);
}

ImageContext::ImageContext(const ImageView& view, int w, int h, int device, bool prepare_now)
    : ba_(w, h, device, nullptr) {
  guarded_init(nullptr, nullptr, prepare_now, &view);
}

// A constructor that throws never reaches the destructor: the encoder's buffers acquired so far are
// handed back here, and the metric, a member constructed by then, hands back its own and the
// stream, so that an out-of-memory condition does not become permanent for the process.
void ImageContext::guarded_init(const uint8_t* rgb, const int16_t* dq_coeffs, bool prepare_now,
                                const ImageView* view) {
  try {
    init(rgb, dq_coeffs, prepare_now, view);
  } catch (...) {
    release();
    throw;
  }
}

void ImageContext::download_rgb(uint8_t* rgb) {
  bind();
  d2h(rgb, d_rgb_, static_cast<size_t>(3) * g_.w * g_.h, s_);
}

// The view's pixels into d_rgb_ (IngestU8), read before this returns.  A host view's span goes through
// a staging buffer, the last one owned: if anything throws, release() waits for the stream and frees it
// with the rest; otherwise it is freed here once the kernel has read it.
void ImageContext::ingest(const ImageView& view) {
  const uint8_t* src = view.data;
  if (view.device) {
    stream_wait(s_, view.stream);
  } else {
    const size_t span = view.span(g_.w, g_.h);
    void* staged = own(span);
    h2d(staged, view.data, span, s_);
    src = static_cast<const uint8_t*>(staged);
  }
  launch_2d(s_, IngestU8{src, view.stride[0], view.stride[1], view.stride[2], view.channels, d_rgb_, g_.w}, g_.w, g_.h,
            "ingest_u8");
  stream_sync(s_);
  if (!view.device) {
    dev_free(owned_.back());
    owned_.pop_back();
  }
}

void ImageContext::init(const uint8_t* rgb, const int16_t* dq_coeffs, bool prepare_now, const ImageView* view) {
  const int w = g_.w, h = g_.h;
  const size_t ncoef = static_cast<size_t>(3) * g_.nblocks * 64;
  d_rgb_ = static_cast<uint8_t*>(own(static_cast<size_t>(3) * w * h));
  d_orig_ = static_cast<int16_t*>(own(ncoef * 2));
  d_cand_ = static_cast<int16_t*>(own(ncoef * 2));
  d_q_ = static_cast<int*>(own(192 * sizeof(int)));
  corner_mask_ = static_cast<float*>(own(sizeof(float) * 3 * g_.nblocks));
  zero_block_max_ = static_cast<float*>(own(sizeof(float) * g_.nblocks));
  dev_zero(zero_block_max_, sizeof(float) * g_.nblocks, s_);
  weights_ = static_cast<float*>(own(sizeof(float) * g_.nblocks));
  const size_t slots = static_cast<size_t>(g_.nblocks) * 192;
  z_idx_ = static_cast<uint8_t*>(own(slots));
  z_err_ = static_cast<float*>(own(slots * sizeof(float)));
  z_cnt_ = static_cast<int*>(own(sizeof(int) * g_.nblocks));
  d_last_index_ = static_cast<int*>(own(sizeof(int) * g_.nblocks));
  d_max_err_ = static_cast<float*>(own(sizeof(float) * g_.nblocks));
  d_hist_ = static_cast<unsigned int*>(own(sizeof(unsigned int) * (kOrderBins + 16)));
  j_hist_ = static_cast<unsigned int*>(own(sizeof(unsigned int) * (static_cast<size_t>(kHistCopies + 1) * kHistStride + 8)));
  j_bits_ = static_cast<unsigned int*>(own(sizeof(unsigned int) * 3 * g_.nblocks));
  j_offset_ = static_cast<unsigned int*>(own(sizeof(unsigned int) * 3 * g_.nblocks));
  j_sums_ = static_cast<unsigned int*>(own(sizeof(unsigned int) * (3 * g_.nblocks / 1024 + 32)));
  j_depth_ = static_cast<uint8_t*>(own(6 * 256));
  j_code_ = static_cast<uint16_t*>(own(6 * 256 * sizeof(uint16_t)));

  metric_ = (w >= 32 && h >= 32);  // g/processor.cc:940: no Butteraugli below 32x32
  prepared_ = false;
  render_all_ = true;
  num_dirty_ = 0;
  d_dirty_ = static_cast<int*>(own(sizeof(int) * g_.nblocks));
  if (dq_on_device_) {
    stream_wait(s_, dq_stream_);
    d2d(d_orig_, dq_coeffs, ncoef * sizeof(int16_t), s_);
  } else if (from_coeffs_) {
    h2d(d_orig_, dq_coeffs, ncoef * sizeof(int16_t), s_);
  } else if (view != nullptr) {
    ingest(*view);
  } else {
    h2d(d_rgb_, rgb, static_cast<size_t>(3) * w * h, s_);
  }
  stream_sync(s_);
  if (prepare_now) prepare();
}

void ImageContext::prepare() {
  bind();
  if (prepared_) return;
  prepared_ = true;
  const size_t ncoef = static_cast<size_t>(3) * g_.nblocks * 64;
  // a2: one-time forward DCT; the host search keeps a copy of the coefficients.
  if (from_coeffs_) {
    launch_1d(s_, RenderRgb8{d_orig_, d_rgb_, g_, t_}, g_.nblocks, "render_rgb8");
  } else {
    launch_1d(s_, FdctBlocks{d_rgb_, d_orig_, g_}, g_.nblocks, "fdct_blocks");
  }
  d2d(d_cand_, d_orig_, ncoef * 2, s_);
  {
    int ones[192];
    for (int i = 0; i < 192; ++i) ones[i] = 1;
    h2d(d_q_, ones, sizeof(ones), s_);
    stream_sync(s_);
  }
  orig_host_.resize(ncoef);
  d2h(orig_host_.data(), d_orig_, ncoef * 2, s_);

  if (!metric_) {
    stream_sync(s_);
    return;
  }
  // a3: PsychoImage of the original (pi0_), resident for the whole search.
  r_.px(LinearizeRgb{d_rgb_, ba_.lin(), g_, t_.srgb_lin}, "linearize_rgb");
  ba_.analyse_original();

  // a13: mask_xyz_ = Mask(xyb0, xyb0), only its block-corner samples are ever read.
  const float* sact = ba_.original_mask_activity();
  r_.block_rows(BlockCornerMask{sact, sact + g_.plane, sact + 2 * g_.plane, corner_mask_, g_, t_.mask_lut},
                "block_corner_mask", r_.by_lo, r_.by_hi);
  stream_sync(s_);
}

ImageContext::~ImageContext() { release(); }

void ImageContext::release() {
  try {
    bind();
    stream_sync(s_);
  } catch (...) {
    // a failed device cannot be waited for; the blocks still go back to the cache
  }
  // the buffers grown on demand; the others are in owned_
  void* const grown[] = {d_sel_val2_, d_sel_block2_,
                         d_sel_pairs_, w_keys_, w_log_index_, w_log_old_, w_gblocks_, w_gcoeffs_, w_ablocks_,
                         d_sel_val_, d_sel_block_, x_items_, x_u32_, x_i32_, x_small_, j_words_, j_file_,
                         j_file_scratch_, j_best_words_, d_edit_i_, d_edit_v_, e_block_, e_slot_};
  for (void* p : grown) dev_free(p);
  for (size_t i = 0; i < owned_.size(); ++i) dev_free(owned_[i]);
  owned_.clear();
}

void ImageContext::apply_global_quant(const int q[192]) {
  render_all_ = true;
  h2d(d_q_, q, 192 * sizeof(int), s_);
  launch_1d(s_, QuantizeCoeffs{d_orig_, d_cand_, d_q_, g_.nblocks}, 3 * g_.nblocks * 64,
            "quantize_coeffs");
}

// the quant tables the candidate's coefficients are multiples of, without re-quantising it
void ImageContext::set_quant(const int q[192]) { h2d(d_q_, q, 192 * sizeof(int), s_); }

void ImageContext::scatter_coeffs(const std::vector<int>& index, const std::vector<int16_t>& value) {
  const int n = static_cast<int>(index.size());
  if (n == 0) return;
  if (static_cast<size_t>(n) > edit_cap_) {
    stream_sync(s_);
    if (d_edit_i_) { dev_free(d_edit_i_); d_edit_i_ = nullptr; }
    if (d_edit_v_) { dev_free(d_edit_v_); d_edit_v_ = nullptr; }
    edit_cap_ = static_cast<size_t>(n) * 2 + 4096;
    d_edit_i_ = static_cast<int*>(dev_alloc(edit_cap_ * sizeof(int)));
    d_edit_v_ = static_cast<int16_t*>(dev_alloc(edit_cap_ * sizeof(int16_t)));
  }
  h2d(d_edit_i_, index.data(), n * sizeof(int), s_);
  h2d(d_edit_v_, value.data(), n * sizeof(int16_t), s_);
  launch_1d(s_, ScatterCoeffs{d_edit_i_, d_edit_v_, d_cand_}, n, "scatter_coeffs");
  // blocks to re-render at the next compare()
  if (!render_all_) {
    if (dirty_flag_.empty()) dirty_flag_.assign(g_.nblocks, 0);
    for (int i = 0; i < n; ++i) {
      const int b = (index[i] / 64) % g_.nblocks;
      if (!dirty_flag_[b]) {
        dirty_flag_[b] = 1;
        dirty_list_.push_back(b);
      }
    }
  }
  stream_sync(s_);  // the host vectors may be reused by the caller
}

void ImageContext::upload_candidate(const int16_t* coeffs) {
  render_all_ = true;
  h2d(d_cand_, coeffs, static_cast<size_t>(3) * g_.nblocks * 64 * 2, s_);
  stream_sync(s_);
}

void ImageContext::download_candidate(int16_t* coeffs) {
  d2h(coeffs, d_cand_, static_cast<size_t>(3) * g_.nblocks * 64 * 2, s_);
}

void ImageContext::compare_render() {
  bind();
  // S0 render (only blocks edited since the last render), S1 opsin, S2-S6 frequency split
  const int rb_lo = r_.cr_lo / 8, rb_hi = (r_.cr_hi + 7) / 8;  // block rows that intersect the computed rows
  float* lin = ba_.lin();
  if (r_.strips() && !render_all_) {
    // strip mode: only edited blocks inside the computed rows need new pixels
    size_t keep = 0;
    for (size_t i = 0; i < dirty_list_.size(); ++i) {
      const int by = dirty_list_[i] / g_.bw;
      dirty_flag_[dirty_list_[i]] = 0;
      if (by >= rb_lo && by < rb_hi) dirty_list_[keep++] = dirty_list_[i];
    }
    dirty_list_.resize(keep);
    for (size_t i = 0; i < keep; ++i) dirty_flag_[dirty_list_[i]] = 1;
  }
  const bool all = render_all_ || dirty_list_.size() + static_cast<size_t>(pending_touched_) >
                                      static_cast<size_t>(rb_hi - rb_lo) * g_.bw / 2;
  if (all) {
#if defined(GB200_HOSTSIM)
    r_.block_rows(RenderBlocks{d_cand_, lin, g_, t_}, "render_blocks", rb_lo, rb_hi);
#else
    launch_render_blocks_warp(s_, RenderWarpArgs{d_cand_, lin, nullptr, rb_lo * g_.bw, (rb_hi - rb_lo) * g_.bw, g_, t_});
#endif
  } else {
    if (!dirty_list_.empty()) {
      const int nd = static_cast<int>(dirty_list_.size());
      h2d(d_dirty_, dirty_list_.data(), sizeof(int) * nd, s_);
#if defined(GB200_HOSTSIM)
      launch_1d(s_, RenderBlockList{RenderBlocks{d_cand_, lin, g_, t_}, d_dirty_}, nd, "render_blocks");
#else
      launch_render_blocks_warp(s_, RenderWarpArgs{d_cand_, lin, d_dirty_, 0, nd, g_, t_});
#endif
    }
    if (pending_touched_ > 0) {
      // blocks changed by the device half of the selection walk: their list is already resident
#if defined(GB200_HOSTSIM)
      launch_1d(s_, RenderBlockList{RenderBlocks{d_cand_, lin, g_, t_}, w_touched_}, pending_touched_, "render_blocks");
#else
      launch_render_blocks_warp(s_, RenderWarpArgs{d_cand_, lin, w_touched_, 0, pending_touched_, g_, t_});
#endif
    }
  }
  pending_touched_ = 0;
  render_all_ = false;
  for (size_t i = 0; i < dirty_list_.size(); ++i) dirty_flag_[dirty_list_[i]] = 0;
  dirty_list_.clear();
}

void ImageContext::block_weights(int direction, int radius, double target_distance, bool zero_distmap,
                                 float* out) {
  BlockWeights bw;
  bw.block_max = zero_distmap ? zero_block_max_ : ba_.block_max();
  bw.weight = weights_;
  bw.g = g_;
  bw.direction = direction;
  bw.radius = radius;
  bw.target_distance = target_distance;
  launch_1d(s_, bw, g_.nblocks, "block_weights");
  d2h(out, weights_, sizeof(float) * g_.nblocks, s_);
}

void ImageContext::zeroing_orders(float block_error_limit, int lookahead, bool new_model, std::vector<uint8_t>* idx,
                                  std::vector<float>* err, std::vector<int>* count) {
  const size_t slots = static_cast<size_t>(g_.nblocks) * 192;
  uint8_t* d_idx = z_idx_;
  float* d_err = z_err_;
  int* d_cnt = z_cnt_;
  ZeroingOrders z;
  z.cand = d_cand_;
  z.orig = d_orig_;
  z.rgb = d_rgb_;
  z.corner_mask = corner_mask_;
  z.out_idx = d_idx;
  z.out_err = d_err;
  z.out_count = d_cnt;
  z.g = g_;
  z.t = t_;
  z.scale8 = t_.opsin_scale8;
  z.lookahead = lookahead;
  z.block_error_limit = block_error_limit;
  z.new_model = new_model ? 1 : 0;
#if defined(GB200_HOSTSIM)
  r_.block_rows(z, "zeroing_orders", r_.by_lo, r_.by_hi);
#else
  {
    ZeroingWarpArgs zw;
    zw.cand = z.cand;
    zw.orig = z.orig;
    zw.rgb = z.rgb;
    zw.corner_mask = z.corner_mask;
    zw.out_idx = z.out_idx;
    zw.out_err = z.out_err;
    zw.out_count = z.out_count;
    zw.g = g_;
    zw.t = t_;
    zw.lookahead = lookahead;
    zw.block_error_limit = block_error_limit;
    zw.new_model = new_model ? 1 : 0;
    zw.b0 = r_.by_lo * g_.bw;
    zw.nb = (r_.by_hi - r_.by_lo) * g_.bw;
    launch_zeroing_orders_warp(s_, zw);
  }
#endif
  // strip mode: the lists of the other strips
  r_.gather_blocks(d_idx, 192);
  r_.gather_blocks(d_err, 192 * sizeof(float));
  r_.gather_blocks(d_cnt, sizeof(int));
  count->resize(g_.nblocks);
  d2h(count->data(), d_cnt, sizeof(int) * g_.nblocks, s_);
  // compact (block, slot) list of all candidates for the order-key kernels, built on the device
  // from an exclusive scan of the counts
  if (e_offset_ == nullptr) {
    e_offset_ = static_cast<unsigned int*>(own(sizeof(unsigned int) * (g_.nblocks + 1)));
  }
  unsigned long long total = 0;
  exclusive_scan(reinterpret_cast<const unsigned int*>(d_cnt), e_offset_, g_.nblocks, &total);
  num_entries_ = static_cast<size_t>(total);
  if (num_entries_ + 1 > e_cap_) {
    stream_sync(s_);
    if (e_block_) { dev_free(e_block_); e_block_ = nullptr; }
    if (e_slot_) { dev_free(e_slot_); e_slot_ = nullptr; }
    e_cap_ = num_entries_ + 1;
    e_block_ = static_cast<int*>(dev_alloc(sizeof(int) * e_cap_));
    e_slot_ = static_cast<uint8_t*>(dev_alloc(e_cap_));
  }
  launch_1d(s_, FillEntries{d_cnt, e_offset_, e_block_, e_slot_}, g_.nblocks, "fill_entries");
  if (idx != nullptr) {
    idx->resize(slots);
    d2h(idx->data(), d_idx, slots, s_);
  }
  if (err != nullptr) {
    err->resize(slots);
    d2h(err->data(), d_err, slots * sizeof(float), s_);
  }
}

// the candidate errors alone (host paths of the selection walk fetch them on first use)
void ImageContext::download_zeroing_err(std::vector<float>* err) {
  const size_t slots = static_cast<size_t>(g_.nblocks) * 192;
  err->resize(slots);
  d2h(err->data(), z_err_, slots * sizeof(float), s_);
}

// Two-level radix select of the k-th smallest key, entirely on the device, then the
// compaction of every entry whose key is <= the threshold bin into d_sel_val_ / d_sel_block_
// (unsorted).  Uses the resident candidate cursors and max errors.
void ImageContext::select_keys(int direction, size_t k, OrderSelectState* got_out) {
  OrderSelectState init;
  memset(&init, 0, sizeof(init));
  init.want = static_cast<unsigned int>(k);
  OrderSelectState* st = reinterpret_cast<OrderSelectState*>(d_hist_ + kOrderBins);
  h2d(st, &init, sizeof(init), s_);
  OrderKeyCommon c;
  c.err = z_err_;
  c.entry_block = e_block_;
  c.entry_slot = e_slot_;
  c.last_index = d_last_index_;
  c.max_err = d_max_err_;
  c.weight = weights_;
  c.direction = direction;
  for (int level = 0; level < 2; ++level) {
    dev_zero(d_hist_, sizeof(unsigned int) * kOrderBins, s_);
#if defined(GB200_HOSTSIM)
    launch_1d(s_, OrderKeyHist{c, d_hist_, st, level}, static_cast<int>(num_entries_), "order_key_hist");
    launch_1d(s_, OrderSelectBin{d_hist_, st, level}, 1, "order_select_bin");
#else
    launch_order_hist(s_, c, d_hist_, st, level, static_cast<int>(num_entries_));
    launch_order_select_bin(s_, d_hist_, st, level);
#endif
  }
  OrderSelectState got;
  d2h(&got, st, sizeof(got), s_);
  const size_t kept = got.kept;
  if (kept > sel_cap_) {
    if (d_sel_val_) { dev_free(d_sel_val_); d_sel_val_ = nullptr; }
    if (d_sel_block_) { dev_free(d_sel_block_); d_sel_block_ = nullptr; }
    sel_cap_ = kept + kept / 2 + 1024;
    d_sel_val_ = static_cast<float*>(dev_alloc(sel_cap_ * sizeof(float)));
    d_sel_block_ = static_cast<int*>(dev_alloc(sel_cap_ * sizeof(int)));
  }
  launch_1d(s_, OrderKeyCompact{c, st, d_sel_val_, d_sel_block_, static_cast<unsigned int>(sel_cap_)},
            static_cast<int>(num_entries_), "order_key_compact");
  *got_out = got;
}

size_t ImageContext::order_smallest(int direction, const std::vector<int>& last_index,
                                    const std::vector<float>& max_err, size_t k, std::vector<float>* val,
                                    std::vector<int>* block) {
  h2d(d_last_index_, last_index.data(), sizeof(int) * g_.nblocks, s_);
  h2d(d_max_err_, max_err.data(), sizeof(float) * g_.nblocks, s_);
  OrderSelectState got;
  select_keys(direction, k, &got);
  const size_t kept = got.kept;
  val->resize(kept);
  block->resize(kept);
  if (kept) {
    d2h(val->data(), d_sel_val_, kept * sizeof(float), s_);
    d2h(block->data(), d_sel_block_, kept * sizeof(int), s_);
  }
  return got.total;
}

#if !defined(GB200_HOSTSIM)
namespace {
// entries / blocks of the order implied by the weights: one thread per block, warp-shuffle and
// shared-memory reduction, two 64-bit atomics per CTA (same sums as WalkStatsPartial)
__global__ void __launch_bounds__(256) k_walk_stats(const int* last_index, const int* z_cnt, const float* weight,
                                                    int direction, int nblocks, unsigned long long* out) {
  __shared__ unsigned int sh[2][8];
  const int b = blockIdx.x * 256 + threadIdx.x;
  unsigned int m = 0u, c = 0u;
  if (b < nblocks && weight[b] != 0) {
    const int li = last_index[b], nc = z_cnt[b];
    const int v = direction > 0 ? (li < nc ? nc - li : 0) : (li > 0 ? li : 0);
    m = static_cast<unsigned int>(v);
    c = v > 0 ? 1u : 0u;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    m += __shfl_xor_sync(0xffffffffu, m, d);
    c += __shfl_xor_sync(0xffffffffu, c, d);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    sh[0][warp] = m;
    sh[1][warp] = c;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long tm = 0, tc = 0;
    for (int w = 0; w < 8; ++w) {
      tm += sh[0][w];
      tc += sh[1][w];
    }
    if (tm) atomicAdd(&out[0], tm);
    if (tc) atomicAdd(&out[1], tc);
  }
}

// The two-rank select reads every order key three times (two histogram levels, the split).
// The first pass computes the keys -- five dependent loads per entry -- and leaves their
// order-preserving integer images in a key array; the other two passes stream that array.
// 0xffffffff (the image of a NaN, never a key) marks entries that are not in the order.
__device__ __forceinline__ float sortable_to_float(unsigned int u) {
  return __uint_as_float((u & 0x80000000u) ? (u ^ 0x80000000u) : ~u);
}

__global__ void __launch_bounds__(256) k_order_hist0_keys(OrderKeyCommon c, unsigned int* hist, unsigned int* keys,
                                                          int entries) {
  __shared__ unsigned int sh[kOrderBins];
  for (int i = threadIdx.x; i < kOrderBins; i += 256) sh[i] = 0;
  __syncthreads();
  for (int e = blockIdx.x * 256 + threadIdx.x; e < entries; e += gridDim.x * 256) {
    float v;
    int b;
    unsigned int u = 0xffffffffu;
    if (c.key(e, &b, &v)) {
      u = hd_float_sortable(v);
      atomicAdd(&sh[u >> 21], 1u);
    }
    keys[e] = u;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kOrderBins; i += 256) {
    const unsigned int n = sh[i];
    if (n) atomicAdd(&hist[i], n);
  }
}

__global__ void __launch_bounds__(256) k_select2_hist1_keys(const unsigned int* keys, unsigned int* hist,
                                                            const Select2State* st, int entries) {
  __shared__ unsigned int sh[2 * kOrderBins];
  for (int i = threadIdx.x; i < 2 * kOrderBins; i += 256) sh[i] = 0;
  __syncthreads();
  const unsigned int b_lo = st->bin0_lo, b_hi = st->bin0_hi;
  for (int e = blockIdx.x * 256 + threadIdx.x; e < entries; e += gridDim.x * 256) {
    const unsigned int u = keys[e];
    if (u == 0xffffffffu) continue;
    const unsigned int top = u >> 21, mid = (u >> 10) & 0x7ffu;
    if (top == b_lo) atomicAdd(&sh[mid], 1u);
    if (top == b_hi) atomicAdd(&sh[kOrderBins + mid], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * kOrderBins; i += 256) {
    const unsigned int n = sh[i];
    if (n) atomicAdd(&hist[i], n);
  }
}

__global__ void __launch_bounds__(256) k_select2_split_keys(const unsigned int* keys, const int* entry_block,
                                                            Select2State* st, unsigned int* cnt, int* touched,
                                                            unsigned int* n_touched, float* mid_val, int* mid_block,
                                                            unsigned int mid_cap, int entries) {
  const unsigned int lo22 = st->lo22, hi22 = st->hi22;
  for (int e = blockIdx.x * 256 + threadIdx.x; e < entries; e += gridDim.x * 256) {
    const unsigned int u = keys[e];
    if (u == 0xffffffffu) continue;
    const unsigned int u22 = u >> 10;
    if (u22 < lo22) {
      const int b = entry_block[e];
      if (atomicAdd(&cnt[b], 1u) == 0u) touched[atomicAdd(n_touched, 1u)] = b;
    } else if (u22 <= hi22) {
      const unsigned int at = atomicAdd(&st->mid_count, 1u);
      if (at < mid_cap) {
        mid_val[at] = sortable_to_float(u);
        mid_block[at] = entry_block[e];
      }
    }
  }
}

// Select2Hist1 with a per-CTA shared-memory histogram pair.
__global__ void __launch_bounds__(256) k_select2_hist1(OrderKeyCommon c, unsigned int* hist, const Select2State* st,
                                                       int entries) {
  __shared__ unsigned int sh[2 * kOrderBins];
  for (int i = threadIdx.x; i < 2 * kOrderBins; i += 256) sh[i] = 0;
  __syncthreads();
  const unsigned int b_lo = st->bin0_lo, b_hi = st->bin0_hi;
  for (int e = blockIdx.x * 256 + threadIdx.x; e < entries; e += gridDim.x * 256) {
    float v;
    int b;
    if (!c.key(e, &b, &v)) continue;
    const unsigned int u = hd_float_sortable(v);
    const unsigned int top = u >> 21, mid = (u >> 10) & 0x7ffu;
    if (top == b_lo) atomicAdd(&sh[mid], 1u);
    if (top == b_hi) atomicAdd(&sh[kOrderBins + mid], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * kOrderBins; i += 256) {
    const unsigned int n = sh[i];
    if (n) atomicAdd(&hist[i], n);
  }
}

// rank_bin_serial by one CTA of 1024 threads (two bins per thread): the bin whose inclusive
// prefix first reaches `want`.
__device__ void rank_bin_block(const unsigned int* hist, unsigned int want, unsigned int* bin, unsigned int* before,
                               unsigned int* total) {
  __shared__ unsigned int warp_tot[32];
  __shared__ unsigned int res[3];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const unsigned int h0 = hist[2 * t], h1 = hist[2 * t + 1];
  const unsigned int local = h0 + h1;
  unsigned int incl = local;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  __syncthreads();  // protects warp_tot / res of a previous call
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  unsigned int base = 0, tot = 0;
  for (int k = 0; k < 32; ++k) {
    if (k < warp) base += warp_tot[k];
    tot += warp_tot[k];
  }
  const unsigned int excl = base + incl - local;
  if (t == 0) {
    res[0] = kOrderBins - 1;
    res[1] = tot - hist[kOrderBins - 1];
    res[2] = tot;
  }
  __syncthreads();
  if (excl < want && want <= excl + h0) {
    res[0] = 2 * t;
    res[1] = excl;
  } else if (excl + h0 < want && want <= excl + local) {
    res[0] = 2 * t + 1;
    res[1] = excl + h0;
  }
  __syncthreads();
  *bin = res[0];
  *before = res[1];
  *total = res[2];
}

__global__ void __launch_bounds__(1024) k_select2_level0(const unsigned int* hist, Select2State* st) {
  unsigned int bin, before, total;
  rank_bin_block(hist, st->want_lo, &bin, &before, &total);
  unsigned int bin2, before2, total2;
  rank_bin_block(hist, st->want_hi, &bin2, &before2, &total2);
  if (threadIdx.x == 0) {
    st->bin0_lo = bin;
    st->below0_lo = before;
    st->bin0_hi = bin2;
    st->below0_hi = before2;
    st->total = total;
  }
}

__global__ void __launch_bounds__(1024) k_select2_level1(const unsigned int* hist, Select2State* st) {
  const unsigned int w_lo = st->want_lo > st->below0_lo ? st->want_lo - st->below0_lo : 1u;
  const unsigned int w_hi = st->want_hi > st->below0_hi ? st->want_hi - st->below0_hi : 1u;
  unsigned int bin, before, total;
  rank_bin_block(hist, w_lo, &bin, &before, &total);
  unsigned int bin2, before2, total2;
  rank_bin_block(hist + kOrderBins, w_hi, &bin2, &before2, &total2);
  if (threadIdx.x == 0) {
    st->lo22 = (st->bin0_lo << 11) | bin;
    st->before_lo = st->below0_lo + before;
    st->hi22 = (st->bin0_hi << 11) | bin2;
    st->kept_hi = st->below0_hi + before2 + hist[kOrderBins + bin2];
    st->mid_count = 0;
  }
}

// BulkApply (walk_dev.h), one WARP per touched block.  The nonzero pattern of the block's 64
// coefficients in zig-zag order is a 64-bit mask (two ballots), so the neighbours of the edited
// coefficient are bit scans and the symbols of the affected range -- it holds at most two nonzero
// coefficients -- follow in closed form; lane 0 does that scalar part.  Same effects as the
// functor (symbol deltas, undo log, cursor, chroma count), which stays the CPU port's version;
// the symbol deltas are privatised per CTA.
__device__ __forceinline__ void warp_emit_run_symbol(unsigned int* h, int run, int value_over_q, unsigned int weight) {
  while (run > 15) {
    atomicAdd(&h[0xf0], weight);
    run -= 16;
  }
  const int nbits = 32 - __clz(static_cast<unsigned int>(value_over_q < 0 ? -value_over_q : value_over_q));
  atomicAdd(&h[(run << 4) + nbits], weight);
}

// symbols of zig-zag positions (za, zb] given the coefficient at zp (0 = none) and at zb (if zb < 64)
__device__ __forceinline__ void warp_range_symbols(unsigned int* h, int za, int zp, int zb, int at_zp_over_q,
                                                   int at_zb_over_q, unsigned int weight) {
  int last_nz = za;
  if (at_zp_over_q != 0) {
    warp_emit_run_symbol(h, zp - za - 1, at_zp_over_q, weight);
    last_nz = zp;
  }
  if (zb < 64) {
    warp_emit_run_symbol(h, zb - last_nz - 1, at_zb_over_q, weight);
  } else if (63 - last_nz > 0) {
    atomicAdd(&h[0], weight);  // end of block
  }
}

__global__ void __launch_bounds__(128) k_bulk_apply_warp(BulkApply a, const unsigned int* n_touched) {
  const int n = static_cast<int>(*n_touched);
  __shared__ unsigned int sh[3 * 256 + 1];
  for (int i = threadIdx.x; i < 3 * 256 + 1; i += 128) sh[i] = 0u;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (j < n) {
    const int b = a.touched[j];
    const int count = static_cast<int>(a.cnt[b]);
    const size_t per = static_cast<size_t>(a.s.nblocks) * 64;
    const int z0 = lane, z1 = lane + 32;                    // this lane's two zig-zag positions
    const int n0 = a.s.zz2nat[z0], n1 = a.s.zz2nat[z1];     // ... and their natural indices
    int li = a.s.last_index[b];
    for (int t = 0; t < count; ++t) {
      const int idx = a.s.z_idx[static_cast<size_t>(b) * 192 + li + (a.direction < 0 ? -1 : 0)];
      const int c = idx >> 6, k = idx & 63;
      const int* qc = a.s.q + 64 * c;
      const int16_t* ob = a.s.orig + c * per + static_cast<size_t>(b) * 64;
      int16_t* blk = a.s.cand + c * per + static_cast<size_t>(b) * 64;
      const int v0 = blk[n0], v1 = blk[n1];
      const unsigned int m_lo = __ballot_sync(0xffffffffu, v0 != 0), m_hi = __ballot_sync(0xffffffffu, v1 != 0);
      const unsigned long long mask = (static_cast<unsigned long long>(m_hi) << 32) | m_lo;
      const int zp = a.s.nat2zz[k];
      // neighbours: highest nonzero below zp (never the DC position 0), lowest above
      const unsigned long long below = mask & ((1ull << zp) - 1ull) & ~1ull;
      const int za = below ? 63 - __clzll(static_cast<long long>(below)) : 0;
      const unsigned long long above = zp < 63 ? (mask >> (zp + 1)) : 0ull;
      const int zb = above ? zp + 1 + (__ffsll(static_cast<long long>(above)) - 1) : 64;
      // precious rule (g/processor.cc:722-733): sum of |original| over the high frequencies
      bool precious = false;
      if (k == 1 || k == 8) {
        int s = 0;
        {
          const int i0 = lane, i1 = lane + 32;  // natural indices 0..63
          if (i0 >= 3 && !((i0 & 7) < 3 && i0 < 24)) {
            const int v = ob[i0];
            s += v < 0 ? -v : v;
          }
          if (!((i1 & 7) < 3 && i1 < 24)) {
            const int v = ob[i1];
            s += v < 0 ? -v : v;
          }
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
        const int limit = s < 60 ? 4 : 8;
        const int ok = ob[k];
        precious = (ok < 0 ? -ok : ok) >= limit;
      }
      if (lane == 0) {
        const int newval = a.direction > 0 ? 0 : quantize_coeff(ob[k], qc[k]);
        const bool store = !precious || newval != 0;
        const int old = blk[k];
        const int at_zb = zb < 64 ? blk[a.s.zz2nat[zb]] / qc[a.s.zz2nat[zb]] : 0;
        unsigned int* h = sh + 256 * c;
        warp_range_symbols(h, za, zp, zb, old != 0 ? old / qc[k] : 0, at_zb, 0xffffffffu);
        int now = old;
        if (store) {
          const unsigned int at = atomicAdd(a.n_log, 1u);
          a.log_index[at] = static_cast<int>(c * per + static_cast<size_t>(b) * 64 + k);
          a.log_old[at] = static_cast<int16_t>(old);
          blk[k] = static_cast<int16_t>(newval);
          now = newval;
          if (c > 0) {
            const int d = (newval != 0 ? 1 : 0) - (old != 0 ? 1 : 0);
            if (d != 0) atomicAdd(&sh[768], static_cast<unsigned int>(d));
          }
        }
        warp_range_symbols(h, za, zp, zb, now != 0 ? now / qc[k] : 0, at_zb, 1u);
      }
      li += a.direction;
      __syncwarp();  // lane 0's store is visible to the loads of the next entry
    }
    if (lane == 0) {
      a.cnt[b] = 0u;
      a.done[b] = count;
      a.stamp[b] = a.iter;
      a.s.last_index[b] = li;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * 256; i += 128)
    if (sh[i]) atomicAdd(&a.delta_hist[i], sh[i]);
  if (threadIdx.x == 0 && sh[768]) atomicAdd(a.chroma_nz, sh[768]);
}

// BulkApply (walk_dev.h) with the symbol-count deltas privatised per CTA: the symbols cluster
// in a few bins, global atomics on them would serialise the whole kernel.
__global__ void __launch_bounds__(128) k_bulk_apply(BulkApply a, const unsigned int* n_touched) {
  const int n = static_cast<int>(*n_touched);
  __shared__ unsigned int sh[3 * 256 + 1];
  for (int i = threadIdx.x; i < 3 * 256 + 1; i += 128) sh[i] = 0u;
  __syncthreads();
  unsigned int* g_hist = a.delta_hist;
  unsigned int* g_chroma = a.chroma_nz;
  a.delta_hist = sh;
  a.chroma_nz = sh + 768;
  const int j = blockIdx.x * 128 + threadIdx.x;
  if (j < n) a(j);
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * 256; i += 128)
    if (sh[i]) atomicAdd(&g_hist[i], sh[i]);
  if (threadIdx.x == 0 && sh[768]) atomicAdd(g_chroma, sh[768]);
}
}  // namespace
#endif

// ---------------------------------------------------------------------------
// Device-resident half of the selection walk (walk_dev.h).
void ImageContext::walk_begin() {
  bind();
  const size_t B = static_cast<size_t>(g_.nblocks);
  if (w_cnt_ == nullptr) {
    w_cnt_ = static_cast<unsigned int*>(own(B * sizeof(unsigned int)));
    w_done_ = static_cast<int*>(own(B * sizeof(int)));
    w_stamp_ = static_cast<int*>(own(B * sizeof(int)));
    w_touched_ = static_cast<int*>(own(B * sizeof(int)));
    w_counters_ = static_cast<unsigned int*>(own((4 + 768) * sizeof(unsigned int)));
    w_stats_ = static_cast<unsigned long long*>(own(1024 * 2 * sizeof(unsigned long long)));
  }
  dev_zero(w_cnt_, B * sizeof(unsigned int), s_);
  dev_zero(w_done_, B * sizeof(int), s_);
  dev_zero(w_stamp_, B * sizeof(int), s_);
  dev_zero(d_last_index_, B * sizeof(int), s_);
  dev_zero(d_max_err_, B * sizeof(float), s_);
  w_iter_ = 0;
  pending_touched_ = 0;
  sel_sorted_ = 0;
}

void ImageContext::walk_upload_state(const std::vector<int>& last_index, const std::vector<float>& max_err) {
  h2d(d_last_index_, last_index.data(), sizeof(int) * g_.nblocks, s_);
  h2d(d_max_err_, max_err.data(), sizeof(float) * g_.nblocks, s_);
  stream_sync(s_);
}

void ImageContext::walk_download_state(std::vector<int>* last_index, std::vector<float>* max_err) {
  last_index->resize(g_.nblocks);
  max_err->resize(g_.nblocks);
  d2h(last_index->data(), d_last_index_, sizeof(int) * g_.nblocks, s_);
  d2h(max_err->data(), d_max_err_, sizeof(float) * g_.nblocks, s_);
}

void ImageContext::walk_weights(int direction, int radius, double target_distance, bool zero_distmap,
                                unsigned long long* order_size, unsigned long long* blocks_to_change) {
  walk_weights_launch(direction, radius, target_distance, zero_distmap);
  walk_weights_fetch(order_size, blocks_to_change);
}

// the kernels / the copy back of the two sums.  A caller that knows the arguments of the next
// iteration queues the kernels behind the metric's and picks the sums up later.
void ImageContext::walk_weights_launch(int direction, int radius, double target_distance, bool zero_distmap) {
  BlockWeights bw;
  bw.block_max = zero_distmap ? zero_block_max_ : ba_.block_max();
  bw.weight = weights_;
  bw.g = g_;
  bw.direction = direction;
  bw.radius = radius;
  bw.target_distance = target_distance;
  launch_1d(s_, bw, g_.nblocks, "block_weights");
#if defined(GB200_HOSTSIM)
  const int lanes = 1024;
  launch_1d(s_, WalkStatsPartial{d_last_index_, z_cnt_, weights_, direction, g_.nblocks, lanes, w_stats_}, lanes,
            "walk_stats");
#else
  dev_zero(w_stats_, 2 * sizeof(unsigned long long), s_);
  note_launch("walk_stats", s_, g_.nblocks);
  k_walk_stats<<<(g_.nblocks + 255) / 256, 256, 0, s_>>>(d_last_index_, z_cnt_, weights_, direction, g_.nblocks, w_stats_);
  note_launch_end("walk_stats", s_);
#endif
}

void ImageContext::walk_weights_fetch(unsigned long long* order_size, unsigned long long* blocks_to_change) {
#if defined(GB200_HOSTSIM)
  const int lanes = 1024;
  unsigned long long part[2 * 1024];
  d2h(part, w_stats_, sizeof(part), s_);
  unsigned long long n = 0, c = 0;
  for (int i = 0; i < lanes; ++i) {
    n += part[2 * i];
    c += part[2 * i + 1];
  }
  *order_size = n;
  *blocks_to_change = c;
#else
  unsigned long long tot[2];
  d2h(tot, w_stats_, sizeof(tot), s_);
  *order_size = tot[0];
  *blocks_to_change = tot[1];
#endif
}

size_t ImageContext::count_nonzero_chroma() {
  const int lanes = 8192;
  void* buf = dev_alloc(sizeof(unsigned long long) * lanes);
  const size_t per = static_cast<size_t>(g_.nblocks) * 64;
  launch_1d(s_, CountNonzeroPartial{d_cand_ + per, 2 * per, lanes, static_cast<unsigned long long*>(buf)}, lanes,
            "count_nonzero");
  std::vector<unsigned long long> part(lanes);
  d2h(part.data(), buf, sizeof(unsigned long long) * lanes, s_);
  dev_free(buf);
  unsigned long long n = 0;
  for (int i = 0; i < lanes; ++i) n += part[i];
  return static_cast<size_t>(n);
}

void ImageContext::download_weights(float* out) { d2h(out, weights_, sizeof(float) * g_.nblocks, s_); }

#if defined(GB200_HOSTSIM)
void ImageContext::sort_selection(size_t n) {
  std::vector<std::pair<float, int> > v(n);
  for (size_t i = 0; i < n; ++i) v[i] = std::make_pair(d_sel_val_[i], d_sel_block_[i]);
  std::stable_sort(v.begin(), v.end(),
                   [](const std::pair<float, int>& a, const std::pair<float, int>& b) { return a.first < b.first; });
  if (n > pairs_cap_) {
    if (d_sel_pairs_) dev_free(d_sel_pairs_);
    pairs_cap_ = n + n / 2 + 4096;
    d_sel_pairs_ = dev_alloc(pairs_cap_ * 8);
  }
  std::pair<int, float>* pairs = static_cast<std::pair<int, float>*>(d_sel_pairs_);
  for (size_t i = 0; i < n; ++i) {
    d_sel_val_[i] = v[i].first;
    d_sel_block_[i] = v[i].second;
    pairs[i] = std::make_pair(v[i].second, v[i].first);
  }
}
#else
namespace {
// Ascending sort of n (float key, int payload) pairs by one CTA: least-significant-digit
// radix sort on the order-preserving integer image of the keys, 4 bits per pass, passes in
// which all keys share the digit skipped.  A thread owns a contiguous chunk of the input, so
// the scatter is stable.  The selections it sorts are 10^4 .. 10^5 entries.
__global__ void __launch_bounds__(1024) k_sort_pairs(float* k0, int* v0, float* k1, int* v1, int n) {
  extern __shared__ unsigned int cnt[];  // [16][1024]
  __shared__ unsigned int warp_tot[32];
  __shared__ unsigned int s_or, s_and;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int chunk = (n + 1023) / 1024;
  const int lo = min(n, t * chunk), hi = min(n, lo + chunk);
  if (t == 0) {
    s_or = 0u;
    s_and = 0xffffffffu;
  }
  __syncthreads();
  {
    unsigned int o = 0u, a = 0xffffffffu;
    for (int i = lo; i < hi; ++i) {
      const unsigned int u = hd_float_sortable(k0[i]);
      o |= u;
      a &= u;
    }
    atomicOr(&s_or, o);
    atomicAnd(&s_and, a);
  }
  __syncthreads();
  const unsigned int varying = s_or ^ s_and;
  float* ka = k0;
  int* va = v0;
  float* kb = k1;
  int* vb = v1;
  for (int shift = 0; shift < 32; shift += 4) {
    if (((varying >> shift) & 15u) == 0u) continue;  // uniform
#pragma unroll
    for (int d = 0; d < 16; ++d) cnt[d * 1024 + t] = 0u;
    for (int i = lo; i < hi; ++i) ++cnt[((hd_float_sortable(ka[i]) >> shift) & 15u) * 1024 + t];
    __syncthreads();
    // exclusive scan of the 16384 counters in (digit, thread) order; thread t owns [16t, 16t + 16)
    unsigned int local[16], sum = 0u;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      local[j] = cnt[16 * t + j];
      sum += local[j];
    }
    unsigned int incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned int x = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += x;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    unsigned int base = 0u;
    for (int w = 0; w < warp; ++w) base += warp_tot[w];
    unsigned int run = base + incl - sum;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      cnt[16 * t + j] = run;
      run += local[j];
    }
    __syncthreads();
    for (int i = lo; i < hi; ++i) {
      const float key = ka[i];
      const unsigned int pos = cnt[((hd_float_sortable(key) >> shift) & 15u) * 1024 + t]++;
      kb[pos] = key;
      vb[pos] = va[i];
    }
    __syncthreads();
    float* tk = ka;
    ka = kb;
    kb = tk;
    int* tv = va;
    va = vb;
    vb = tv;
  }
  if (ka != k0) {  // odd number of passes: the result sits in the second buffer
    for (int i = lo; i < hi; ++i) {
      k0[i] = ka[i];
      v0[i] = va[i];
    }
  }
}
// The same for selections that fit in shared memory (CAP entries, NT threads): the keys
// (order-preserving integer image) and 16-bit indices ping-pong between two shared-memory
// buffers; global memory is read once and written once.
constexpr int kSortSmemMax = 14336;
constexpr int kSortSmemSmall = 3072;
template <int CAP, int NT>
__global__ void __launch_bounds__(NT) k_sort_pairs_smem(float* keys, int* vals, int2* pairs, int n) {
  extern __shared__ unsigned int dyn_sort[];
  unsigned int* ka = dyn_sort;                                       // [CAP]
  unsigned int* kb = ka + CAP;                                       // [CAP]
  unsigned short* ia = reinterpret_cast<unsigned short*>(kb + CAP);  // [CAP]
  unsigned short* ib = ia + CAP;                                     // [CAP]
  unsigned short* cnt = ib + CAP;                                    // [16][NT]
  __shared__ unsigned int warp_tot[32];
  __shared__ unsigned int s_or, s_and;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t == 0) {
    s_or = 0u;
    s_and = 0xffffffffu;
  }
  __syncthreads();
  {
    unsigned int o = 0u, a = 0xffffffffu;
    for (int i = t; i < n; i += NT) {  // coalesced load
      const unsigned int u = hd_float_sortable(keys[i]);
      ka[i] = u;
      ia[i] = static_cast<unsigned short>(i);
      o |= u;
      a &= u;
    }
    atomicOr(&s_or, o);
    atomicAnd(&s_and, a);
  }
  __syncthreads();
  const unsigned int varying = s_or ^ s_and;
  const int chunk = (n + NT - 1) / NT;
  const int lo = min(n, t * chunk), hi = min(n, lo + chunk);
  for (int shift = 0; shift < 32; shift += 4) {
    if (((varying >> shift) & 15u) == 0u) continue;  // uniform
#pragma unroll
    for (int d = 0; d < 16; ++d) cnt[d * NT + t] = 0;
    for (int i = lo; i < hi; ++i) ++cnt[((ka[i] >> shift) & 15u) * NT + t];
    __syncthreads();
    unsigned int local[16], sum = 0u;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      local[j] = cnt[16 * t + j];
      sum += local[j];
    }
    unsigned int incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned int x = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += x;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    unsigned int base = 0u;
    for (int w = 0; w < warp; ++w) base += warp_tot[w];
    unsigned int run = base + incl - sum;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      cnt[16 * t + j] = static_cast<unsigned short>(run);
      run += local[j];
    }
    __syncthreads();
    for (int i = lo; i < hi; ++i) {
      const unsigned int u = ka[i];
      const unsigned int pos = cnt[((u >> shift) & 15u) * NT + t]++;
      kb[pos] = u;
      ib[pos] = ia[i];
    }
    __syncthreads();
    unsigned int* tk = ka;
    ka = kb;
    kb = tk;
    unsigned short* ti = ia;
    ia = ib;
    ib = ti;
  }
  // gather the payloads through the permutation (read all, then write: in place)
  constexpr int PER = (CAP + NT - 1) / NT;
  int pay[PER];
  float key[PER];
#pragma unroll
  for (int r = 0; r < PER; ++r) {
    const int i = t + NT * r;
    if (i < n) {
      pay[r] = vals[ia[i]];
      key[r] = keys[ia[i]];
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < PER; ++r) {
    const int i = t + NT * r;
    if (i < n) {
      vals[i] = pay[r];
      keys[i] = key[r];
      pairs[i] = make_int2(pay[r], __float_as_int(key[r]));  // std::pair<int, float> of the host's order
    }
  }
}

// (block, key) pairs in the host's layout for selections sorted by the global-memory kernel
__global__ void __launch_bounds__(256) k_make_pairs(const float* keys, const int* vals, int2* pairs, int n) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < n) pairs[i] = make_int2(vals[i], __float_as_int(keys[i]));
}
}  // namespace

int2* ImageContext::sel_pairs(size_t n) {
  if (n > pairs_cap_) {
    stream_sync(s_);
    if (d_sel_pairs_) { dev_free(d_sel_pairs_); d_sel_pairs_ = nullptr; }
    pairs_cap_ = n + n / 2 + 4096;
    d_sel_pairs_ = dev_alloc(pairs_cap_ * 8);
  }
  return static_cast<int2*>(d_sel_pairs_);
}

void ImageContext::sort_selection(size_t n) {
  if (n == 0) return;
  if (n <= kSortSmemSmall) {
    const size_t smem = kSortSmemSmall * 12 + 16 * 256 * sizeof(unsigned short);  // 44 KB
    note_launch("sort_pairs", s_, static_cast<double>(n));
    k_sort_pairs_smem<kSortSmemSmall, 256><<<1, 256, smem, s_>>>(d_sel_val_, d_sel_block_, sel_pairs(n), static_cast<int>(n));
    note_launch_end("sort_pairs", s_);
    return;
  }
  if (n <= kSortSmemMax) {
    const size_t smem = kSortSmemMax * 12 + 16 * 1024 * sizeof(unsigned short);
    GB_CUDA(cudaFuncSetAttribute(k_sort_pairs_smem<kSortSmemMax, 1024>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem)));
    note_launch("sort_pairs", s_, static_cast<double>(n));
    k_sort_pairs_smem<kSortSmemMax, 1024><<<1, 1024, smem, s_>>>(d_sel_val_, d_sel_block_, sel_pairs(n), static_cast<int>(n));
    note_launch_end("sort_pairs", s_);
    return;
  }
  if (n > sel2_cap_) {
    if (d_sel_val2_) { dev_free(d_sel_val2_); d_sel_val2_ = nullptr; }
    if (d_sel_block2_) { dev_free(d_sel_block2_); d_sel_block2_ = nullptr; }
    sel2_cap_ = n + n / 2 + 1024;
    d_sel_val2_ = static_cast<float*>(dev_alloc(sel2_cap_ * sizeof(float)));
    d_sel_block2_ = static_cast<int*>(dev_alloc(sel2_cap_ * sizeof(int)));
  }
  const size_t smem = 16 * 1024 * sizeof(unsigned int);
  GB_CUDA(cudaFuncSetAttribute(k_sort_pairs, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  note_launch("sort_pairs", s_, static_cast<double>(n));
  k_sort_pairs<<<1, 1024, smem, s_>>>(d_sel_val_, d_sel_block_, d_sel_val2_, d_sel_block2_, static_cast<int>(n));
  k_make_pairs<<<static_cast<unsigned int>((n + 255) / 256), 256, 0, s_>>>(d_sel_val_, d_sel_block_, sel_pairs(n), static_cast<int>(n));
  note_launch_end("sort_pairs", s_);
}
#endif

#if !defined(GB200_HOSTSIM)
namespace {
__global__ void __launch_bounds__(256) k_count_keys_below(OrderKeyCommon c, float limit, int entries, unsigned int* out) {
  unsigned int n = 0;
  for (int e = blockIdx.x * 256 + threadIdx.x; e < entries; e += gridDim.x * 256) {
    float v;
    int b;
    if (c.key(e, &b, &v) && v < limit) ++n;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) n += __shfl_xor_sync(0xffffffffu, n, d);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(out, n);
}
}  // namespace
#endif

size_t ImageContext::walk_count_below(int direction, float limit) {
  OrderKeyCommon c;
  c.err = z_err_;
  c.entry_block = e_block_;
  c.entry_slot = e_slot_;
  c.last_index = d_last_index_;
  c.max_err = d_max_err_;
  c.weight = weights_;
  c.direction = direction;
  unsigned int* out = reinterpret_cast<unsigned int*>(w_stats_);
  dev_zero(out, sizeof(unsigned int), s_);
  const int entries = static_cast<int>(num_entries_);
#if defined(GB200_HOSTSIM)
  launch_1d(s_, CountKeysBelow{c, limit, out}, entries, "count_keys_below");
#else
  int ctas = (entries + 256 * 8 - 1) / (256 * 8);
  if (ctas < 1) ctas = 1;
  if (ctas > 8 * kTargetSMs) ctas = 8 * kTargetSMs;
  note_launch("count_keys_below", s_, entries);
  k_count_keys_below<<<ctas, 256, 0, s_>>>(c, limit, entries, out);
  note_launch_end("count_keys_below", s_);
#endif
  unsigned int n = 0;
  d2h(&n, out, sizeof(n), s_);
  return n;
}

static const size_t kMiddleSortMax = 65536;

size_t ImageContext::walk_select_split(int direction, size_t rank_lo, size_t rank_hi, size_t* before, size_t* total) {
  // d_hist_ holds 2048 bins + the old select state; the pair of level-1 histograms and the
  // two-rank state live in w_sel2_
  if (w_sel2_ == nullptr) {
    w_sel2_ = static_cast<unsigned int*>(own(sizeof(unsigned int) * (2 * kOrderBins + 64)));
  }
  Select2State* st = reinterpret_cast<Select2State*>(w_sel2_ + 2 * kOrderBins);
  Select2State init;
  memset(&init, 0, sizeof(init));
  init.want_lo = static_cast<unsigned int>(rank_lo < 1 ? 1 : rank_lo);
  init.want_hi = static_cast<unsigned int>(rank_hi);
  h2d(st, &init, sizeof(init), s_);
  // a fresh bulk: counters for the per-block counts that the split pass starts to fill
  ++w_iter_;
  dev_zero(w_counters_, (4 + 768) * sizeof(unsigned int), s_);
  OrderKeyCommon c;
  c.err = z_err_;
  c.entry_block = e_block_;
  c.entry_slot = e_slot_;
  c.last_index = d_last_index_;
  c.max_err = d_max_err_;
  c.weight = weights_;
  c.direction = direction;
  const int entries = static_cast<int>(num_entries_);
  const size_t mid_cap_want = (rank_hi - (rank_lo < 1 ? 1 : rank_lo)) * 2 + 65536;
  if (mid_cap_want > sel_cap_) {
    stream_sync(s_);
    if (d_sel_val_) { dev_free(d_sel_val_); d_sel_val_ = nullptr; }
    if (d_sel_block_) { dev_free(d_sel_block_); d_sel_block_ = nullptr; }
    sel_cap_ = mid_cap_want;
    d_sel_val_ = static_cast<float*>(dev_alloc(sel_cap_ * sizeof(float)));
    d_sel_block_ = static_cast<int*>(dev_alloc(sel_cap_ * sizeof(int)));
  }
  dev_zero(d_hist_, sizeof(unsigned int) * kOrderBins, s_);
  dev_zero(w_sel2_, sizeof(unsigned int) * 2 * kOrderBins, s_);
#if defined(GB200_HOSTSIM)
  launch_1d(s_, OrderKeyHist{c, d_hist_, nullptr, 0}, entries, "order_key_hist");
  launch_1d(s_, Select2Level0{d_hist_, st}, 1, "select2_level");
  launch_1d(s_, Select2Hist1{c, w_sel2_, st}, entries, "select2_hist1");
  launch_1d(s_, Select2Level1{w_sel2_, st}, 1, "select2_level");
#else
  if (static_cast<size_t>(entries) > keys_cap_) {
    stream_sync(s_);
    if (w_keys_) { dev_free(w_keys_); w_keys_ = nullptr; }
    keys_cap_ = static_cast<size_t>(entries) + 1024;
    w_keys_ = static_cast<unsigned int*>(dev_alloc(keys_cap_ * sizeof(unsigned int)));
  }
  int ctas = (entries + 256 * 8 - 1) / (256 * 8);
  if (ctas < 1) ctas = 1;
  if (ctas > 8 * kTargetSMs) ctas = 8 * kTargetSMs;  // 8 resident CTAs per SM
  note_launch("order_key_hist", s_, entries);
  k_order_hist0_keys<<<ctas, 256, 0, s_>>>(c, d_hist_, w_keys_, entries);
  note_launch_end("order_key_hist", s_);
  note_launch("select2_level", s_, kOrderBins);
  k_select2_level0<<<1, 1024, 0, s_>>>(d_hist_, st);
  note_launch_end("select2_level", s_);
  note_launch("select2_hist1", s_, entries);
  k_select2_hist1_keys<<<ctas, 256, 0, s_>>>(w_keys_, w_sel2_, st, entries);
  note_launch_end("select2_hist1", s_);
  note_launch("select2_level", s_, kOrderBins);
  k_select2_level1<<<1, 1024, 0, s_>>>(w_sel2_, st);
  note_launch_end("select2_level", s_);
  note_launch("select2_split", s_, entries);
  k_select2_split_keys<<<ctas, 256, 0, s_>>>(w_keys_, e_block_, st, w_cnt_, w_touched_, w_counters_, d_sel_val_, d_sel_block_,
                                             static_cast<unsigned int>(sel_cap_), entries);
  note_launch_end("select2_split", s_);
#endif
#if defined(GB200_HOSTSIM)
  launch_1d(s_, Select2Split{c, st, w_cnt_, w_touched_, w_counters_, d_sel_val_, d_sel_block_,
                             static_cast<unsigned int>(sel_cap_)},
            entries, "select2_split");
#endif
  Select2State got;
  d2h(&got, st, sizeof(got), s_);
  *total = got.total;
  *before = got.before_lo;
  const size_t n_mid = got.kept_hi >= got.before_lo ? got.kept_hi - got.before_lo : 0;
  if (got.mid_count != n_mid) throw std::runtime_error("select2: middle count mismatch");
  if (n_mid > sel_cap_ && n_mid <= kMiddleSortMax) throw std::runtime_error("select2: middle list overflow");
  split_pending_ = true;
  pending_bulk_extra_ = got.before_lo;
  if (n_mid > kMiddleSortMax) {
    // a huge run of equal keys sits on one of the two ranks: the caller cannot use this
    // selection (it takes the reference-ordered path) and must cancel it
    sel_sorted_ = 0;
    return n_mid;
  }
  sel_sorted_ = n_mid;
  sort_selection(n_mid);
  return n_mid;
}

// drops the per-block counts of a walk_select_split that no bulk will consume
void ImageContext::walk_split_cancel() {
  if (!split_pending_) return;
  unsigned int n_touched = 0;
  d2h(&n_touched, w_counters_, sizeof(unsigned int), s_);
  if (n_touched) launch_1d(s_, ResetCounts{w_touched_, w_cnt_}, static_cast<int>(n_touched), "walk_split_cancel");
  split_pending_ = false;
  pending_bulk_extra_ = 0;
}

size_t ImageContext::walk_select_sorted(int direction, size_t want, size_t* total) {
  OrderSelectState got;
  select_keys(direction, want, &got);
  *total = got.total;
  sel_sorted_ = got.kept;
  sort_selection(sel_sorted_);
  return sel_sorted_;
}

// the sorted selection as (block, key) pairs, one copy
void ImageContext::walk_fetch_pairs(size_t n, std::pair<int, float>* out) {
  static_assert(sizeof(std::pair<int, float>) == 8, "pair<int,float> layout");
  if (n > sel_sorted_) throw std::runtime_error("walk_fetch_pairs: range outside the selection");
  if (n == 0) return;
  d2h(out, d_sel_pairs_, n * 8, s_);
}

void ImageContext::walk_fetch_sorted(size_t first, size_t n, float* val, int* block) {
  if (first + n > sel_sorted_) throw std::runtime_error("walk_fetch_sorted: range outside the selection");
  if (n == 0) return;
  d2h(val, d_sel_val_ + first, n * sizeof(float), s_);
  d2h(block, d_sel_block_ + first, n * sizeof(int), s_);
}

void ImageContext::walk_bulk_apply(int direction, size_t nbulk, BulkResult* r, const int* host_blocks, bool after_split,
                                   size_t gather_first, size_t gather_n) {
  const int* entry_blocks = d_sel_block_;
  if (host_blocks != nullptr) {
    if (nbulk > w_acap_) {
      stream_sync(s_);
      if (w_ablocks_) { dev_free(w_ablocks_); w_ablocks_ = nullptr; }
      w_acap_ = nbulk + nbulk / 2 + 4096;
      w_ablocks_ = static_cast<int*>(dev_alloc(w_acap_ * sizeof(int)));
    }
    if (nbulk) h2d(w_ablocks_, host_blocks, nbulk * sizeof(int), s_);
    entry_blocks = w_ablocks_;
  } else if (nbulk > sel_sorted_) {
    throw std::runtime_error("walk_bulk_apply: bulk larger than the selection");
  }
  const size_t log_need = nbulk + pending_bulk_extra_;
  const size_t pending_extra_for_grid = pending_bulk_extra_;
  (void)pending_extra_for_grid;
  pending_bulk_extra_ = 0;
  if (log_need > w_log_cap_) {
    stream_sync(s_);
    if (w_log_index_) { dev_free(w_log_index_); w_log_index_ = nullptr; }
    if (w_log_old_) { dev_free(w_log_old_); w_log_old_ = nullptr; }
    w_log_cap_ = log_need + log_need / 2 + 4096;
    w_log_index_ = static_cast<int*>(dev_alloc(w_log_cap_ * sizeof(int)));
    w_log_old_ = static_cast<int16_t*>(dev_alloc(w_log_cap_ * sizeof(int16_t)));
  }
  if (after_split != split_pending_) throw std::runtime_error("walk_bulk_apply: split state mismatch");
  if (!after_split) {
    ++w_iter_;
    dev_zero(w_counters_, (4 + 768) * sizeof(unsigned int), s_);
  }
  split_pending_ = false;
  unsigned int host_counters[4 + 768];
  memset(host_counters, 0, sizeof(host_counters));
  if (nbulk > 0 || after_split) {
    if (nbulk > 0)
      launch_1d(s_, BulkCount{entry_blocks, w_cnt_, w_touched_, w_counters_}, static_cast<int>(nbulk), "walk_bulk_count");
#if defined(GB200_HOSTSIM)
    unsigned int n_touched = 0;
    d2h(&n_touched, w_counters_, sizeof(unsigned int), s_);
#else
    // no round trip for the number of touched blocks: the grid covers its upper bound, the
    // kernel reads the count
    const unsigned int n_touched =
        static_cast<unsigned int>(std::min<size_t>(static_cast<size_t>(g_.nblocks), nbulk + pending_extra_for_grid));
#endif
    BulkApply a;
    a.s.orig = d_orig_;
    a.s.cand = d_cand_;
    a.s.q = d_q_;
    a.s.zz2nat = t_.zigzag;
    a.s.nat2zz = t_.nat2zz;
    a.s.z_idx = z_idx_;
    a.s.last_index = d_last_index_;
    a.s.nblocks = g_.nblocks;
    a.touched = w_touched_;
    a.cnt = w_cnt_;
    a.done = w_done_;
    a.stamp = w_stamp_;
    a.iter = w_iter_;
    a.direction = direction;
    a.delta_hist = w_counters_ + 4;
    a.chroma_nz = w_counters_ + 2;
    a.log_index = w_log_index_;
    a.log_old = w_log_old_;
    a.n_log = w_counters_ + 1;
#if defined(GB200_HOSTSIM)
    launch_1d(s_, a, static_cast<int>(n_touched), "walk_bulk_apply");
#else
    if (n_touched > 0) {
      note_launch("walk_bulk_apply", s_, n_touched);
      static const bool kThreadPerBlock = getenv("GB200_BULK_THREAD") != nullptr;  // A/B: the functor form
      if (kThreadPerBlock) {
        k_bulk_apply<<<(n_touched + 127) / 128, 128, 0, s_>>>(a, w_counters_);
      } else {
        k_bulk_apply_warp<<<(n_touched + 3) / 4, 128, 0, s_>>>(a, w_counters_);
      }
      note_launch_end("walk_bulk_apply", s_);
    }
#endif
    if (gather_n > 0) {
      if (gather_first + gather_n > sel_sorted_) throw std::runtime_error("walk_bulk_apply: gather outside the selection");
      gather_reserve(gather_n);
      const size_t n = gather_n;
      int* d_cursor = reinterpret_cast<int*>(w_gcoeffs_ + n * 192);
      launch_1d(s_, GatherBlockState{d_sel_block_ + gather_first, d_cand_, d_last_index_, w_stamp_, w_iter_, g_.nblocks,
                                     w_gcoeffs_, d_cursor, d_cursor + n},
                static_cast<int>(24 * n), "walk_gather");
    }
    d2h(host_counters, w_counters_, sizeof(host_counters), s_);
  }
  r->touched = static_cast<int>(host_counters[0]);
  r->logged = static_cast<int>(host_counters[1]);
  r->chroma_delta = static_cast<int>(host_counters[2]);
  for (int c = 0; c < 3; ++c)
    for (int i = 0; i < 256; ++i) r->delta_hist[c][i] = static_cast<int>(host_counters[4 + 256 * c + i]);
  w_last_touched_ = r->touched;
  w_last_logged_ = r->logged;
  pending_touched_ = r->touched;
}

void ImageContext::walk_bulk_undo(int direction) {
  if (w_last_logged_ > 0)
    launch_1d(s_, BulkUndoCoeffs{w_log_index_, w_log_old_, d_cand_}, w_last_logged_, "walk_bulk_undo");
  if (w_last_touched_ > 0)
    launch_1d(s_, BulkUndoCursors{w_touched_, w_done_, d_last_index_, direction}, w_last_touched_, "walk_bulk_undo");
  w_last_logged_ = 0;
  w_last_touched_ = 0;
  pending_touched_ = 0;
}

void ImageContext::gather_reserve(size_t n) {
  if (n > w_gcap_) {
    stream_sync(s_);
    if (w_gblocks_) { dev_free(w_gblocks_); w_gblocks_ = nullptr; }
    if (w_gcoeffs_) { dev_free(w_gcoeffs_); w_gcoeffs_ = nullptr; }
    w_gcap_ = n + n / 2 + 1024;
    w_gblocks_ = static_cast<int*>(dev_alloc(w_gcap_ * sizeof(int)));
    // one buffer, one copy back: [cap][192] int16 | [cap] cursors | [cap] flags
    w_gcoeffs_ = static_cast<int16_t*>(dev_alloc(w_gcap_ * (192 * sizeof(int16_t) + 2 * sizeof(int))));
  }
}

void ImageContext::gather_fetch(size_t n, std::vector<int16_t>* coeffs, std::vector<int>* cursor, std::vector<int>* in_bulk) {
  const size_t bytes = n * (192 * sizeof(int16_t) + 2 * sizeof(int));
  gather_host_.resize(bytes);
  d2h(gather_host_.data(), w_gcoeffs_, bytes, s_);
  memcpy(coeffs->data(), gather_host_.data(), n * 192 * sizeof(int16_t));
  memcpy(cursor->data(), gather_host_.data() + n * 192 * sizeof(int16_t), n * sizeof(int));
  memcpy(in_bulk->data(), gather_host_.data() + n * 192 * sizeof(int16_t) + n * sizeof(int), n * sizeof(int));
}

void ImageContext::walk_gather_selection_fetch(size_t n, std::vector<int16_t>* coeffs, std::vector<int>* cursor,
                                               std::vector<int>* in_bulk) {
  coeffs->resize(n * 192);
  cursor->resize(n);
  in_bulk->resize(n);
  if (n == 0) return;
  gather_fetch(n, coeffs, cursor, in_bulk);
}

void ImageContext::walk_gather(const std::vector<int>& blocks, std::vector<int16_t>* coeffs, std::vector<int>* cursor,
                               std::vector<int>* in_bulk) {
  const size_t n = blocks.size();
  coeffs->resize(n * 192);
  cursor->resize(n);
  in_bulk->resize(n);
  if (n == 0) return;
  gather_reserve(n);
  int* d_cursor = reinterpret_cast<int*>(w_gcoeffs_ + n * 192);
  int* d_inbulk = d_cursor + n;
  h2d(w_gblocks_, blocks.data(), n * sizeof(int), s_);
  launch_1d(s_, GatherBlockState{w_gblocks_, d_cand_, d_last_index_, w_stamp_, w_iter_, g_.nblocks, w_gcoeffs_, d_cursor,
                                 d_inbulk},
            static_cast<int>(24 * n), "walk_gather");
  gather_fetch(n, coeffs, cursor, in_bulk);
}

void ImageContext::walk_advance(const std::vector<int>& blocks, int direction) {
  const size_t n = blocks.size();
  if (n == 0) return;
  if (n > w_acap_) {
    stream_sync(s_);
    if (w_ablocks_) { dev_free(w_ablocks_); w_ablocks_ = nullptr; }
    w_acap_ = n + n / 2 + 4096;
    w_ablocks_ = static_cast<int*>(dev_alloc(w_acap_ * sizeof(int)));
  }
  // no wait here: the copy reads a buffer that lives until the next call (a pageable source is
  // staged before cudaMemcpyAsync returns in any case)
  advance_host_.assign(blocks.begin(), blocks.end());
  h2d(w_ablocks_, advance_host_.data(), n * sizeof(int), s_);
  launch_1d(s_, AdvanceCursors{w_ablocks_, d_last_index_, direction}, static_cast<int>(n), "walk_advance");
}

void ImageContext::walk_add_max_err(float val_threshold, int direction) {
  launch_1d(s_, AddMaxErr{d_max_err_, weights_, val_threshold, direction}, g_.nblocks, "walk_add_max_err");
}

// ---------------------------------------------------------------------------
// EXPERIMENTAL: reference-ordered selection order with the large partition passes on the
// device (order_exact.h).  Ranges of at most kOrderHostRange items go back to the host replay.
static const ptrdiff_t kOrderHostRange = [] {
  const char* e = getenv("GB200_ORDER_HOST_RANGE");  // tests lower it to reach the device passes on small images
  const long v = e ? atol(e) : 0;
  return static_cast<ptrdiff_t>(v >= 16 ? v : (1 << 15));
}();

void ImageContext::order_scratch(size_t n) {
  if (n <= x_cap_) return;
  stream_sync(s_);
  if (x_items_) { dev_free(x_items_); x_items_ = nullptr; }
  if (x_u32_) { dev_free(x_u32_); x_u32_ = nullptr; }
  if (x_i32_) { dev_free(x_i32_); x_i32_ = nullptr; }
  if (x_small_) { dev_free(x_small_); x_small_ = nullptr; }
  x_cap_ = n + n / 4 + 1024;
  x_items_ = static_cast<OrderItem*>(dev_alloc(x_cap_ * sizeof(OrderItem)));
  x_u32_ = static_cast<unsigned int*>(dev_alloc(4 * x_cap_ * sizeof(unsigned int)));
  x_i32_ = static_cast<int*>(dev_alloc(2 * x_cap_ * sizeof(int)));
  x_small_ = static_cast<unsigned int*>(dev_alloc((x_cap_ / 1024 + 64) * sizeof(unsigned int) + 64));
}

size_t ImageContext::device_partial_sort_resident(size_t n_, size_t want_, std::vector<std::pair<int, float> >* out) {
  typedef exact_sort::Item Item;
  static_assert(sizeof(Item) == sizeof(OrderItem), "pair<int,float> layout");
  const ptrdiff_t n = static_cast<ptrdiff_t>(n_);
  const ptrdiff_t want = static_cast<ptrdiff_t>(want_ < n_ ? want_ : n_);
  if (n < 2 || n <= kOrderHostRange) {
    out->resize(n_);
    if (n_) d2h(out->data(), x_items_, n_ * sizeof(Item), s_);
    const size_t k = exact_sort::partial_std_sort(out->data(), n_, want_);
    out->resize(k);
    return k;
  }
  // host mirror of the prefix, filled range by range as the replay hands ranges back
  Item* host = static_cast<Item*>(malloc(n_ * sizeof(Item)));
  if (host == nullptr) throw std::bad_alloc();
  unsigned int* fl = x_u32_;
  unsigned int* sl = x_u32_ + x_cap_;
  unsigned int* fr = x_u32_ + 2 * x_cap_;
  unsigned int* sr = x_u32_ + 3 * x_cap_;
  int* llist = x_i32_;
  int* rlist = x_i32_ + x_cap_;
  unsigned int* num_swaps = x_small_;
  long long* d_cut = reinterpret_cast<long long*>(x_small_ + 2);
  unsigned int* scan_scratch = x_small_ + 8;
  ptrdiff_t k_end = 0;
  ptrdiff_t st_first[160], st_last[160], st_depth[160];
  int sp = 0;
  st_first[sp] = 0;
  st_last[sp] = n;
  st_depth[sp] = exact_sort::introsort_depth_limit(n);
  ++sp;
  try {
    while (sp > 0) {
      --sp;
      ptrdiff_t first = st_first[sp], last = st_last[sp], depth = st_depth[sp];
      if (first >= want) continue;
      bool handed_back = false;
      while (last - first > 16) {
        if (depth == 0 || last - first <= kOrderHostRange) {
          // small (or depth-exhausted) range: the host replay finishes it
          d2h(host + first, x_items_ + first, static_cast<size_t>(last - first) * sizeof(Item), s_);
          exact_sort::introsort_prefix(host, first, last, depth, want, &k_end);
          handed_back = true;
          break;
        }
        --depth;
        launch_1d(s_, OrderPivot{x_items_, first, last}, 1, "order_pivot");
        const int m = static_cast<int>(last - first - 1);
        launch_1d(s_, OrderPartFlags{x_items_, first, m, fl, fr}, m, "order_part_flags");
        unsigned long long total_l = 0, total_r = 0;
        exclusive_scan_with(fl, sl, m, &total_l, scan_scratch);
        exclusive_scan_with(fr, sr, m, &total_r, scan_scratch);
        dev_zero(num_swaps, sizeof(unsigned int), s_);
        launch_1d(s_, OrderPartLists{fl, sl, fr, sr, m, llist, rlist, num_swaps}, m, "order_part_lists");
        launch_1d(s_, OrderPartCut{first, llist, rlist, num_swaps, static_cast<unsigned int>(total_l), d_cut}, 1,
                  "order_part_cut");
        unsigned int k = 0;
        d2h(&k, num_swaps, sizeof(k), s_);
        if (k) launch_1d(s_, OrderPartSwap{x_items_, first, llist, rlist}, static_cast<int>(k), "order_part_swap");
        long long cut_ll = 0;
        d2h(&cut_ll, d_cut, sizeof(cut_ll), s_);
        const ptrdiff_t cut = static_cast<ptrdiff_t>(cut_ll);
        if (cut <= first || cut > last) throw std::runtime_error("device order replay: partition out of range");
        if (cut < want) {
          st_first[sp] = cut;
          st_last[sp] = last;
          st_depth[sp] = depth;
          ++sp;
        }
        last = cut;
      }
      if (!handed_back) {
        if (last > first) d2h(host + first, x_items_ + first, static_cast<size_t>(last - first) * sizeof(Item), s_);
        if (last > k_end) k_end = last;
      }
    }
    exact_sort::final_insertion_prefix(host, n, &k_end);
    out->assign(host, host + k_end);
  } catch (...) {
    free(host);
    throw;
  }
  free(host);
  return static_cast<size_t>(k_end);
}

size_t ImageContext::debug_device_partial_sort(std::pair<int, float>* items, size_t n, size_t want) {
  bind();
  order_scratch(n);
  if (n) h2d(x_items_, items, n * sizeof(OrderItem), s_);
  std::vector<std::pair<int, float> > out;
  const size_t k = device_partial_sort_resident(n, want, &out);
  std::copy(out.begin(), out.begin() + k, items);
  return k;
}

size_t ImageContext::exact_order_prefix(int direction, const std::vector<int>& last_index,
                                        const std::vector<float>& max_err, size_t want,
                                        std::vector<std::pair<int, float> >* out, size_t* order_size) {
  h2d(d_last_index_, last_index.data(), sizeof(int) * g_.nblocks, s_);
  h2d(d_max_err_, max_err.data(), sizeof(float) * g_.nblocks, s_);
  return exact_order_prefix_resident(direction, want, out, order_size);
}

size_t ImageContext::exact_order_prefix_resident(int direction, size_t want, std::vector<std::pair<int, float> >* out,
                                                 size_t* order_size) {
  order_scratch(std::max<size_t>(num_entries_, static_cast<size_t>(g_.nblocks)) + 16);
  unsigned int* count = x_u32_;
  unsigned int* offset = x_u32_ + x_cap_;
  launch_1d(s_, OrderRefCount{d_last_index_, z_cnt_, weights_, direction, count}, g_.nblocks, "order_ref_count");
  unsigned long long total = 0;
  exclusive_scan_with(count, offset, g_.nblocks, &total, x_small_ + 8);
  *order_size = static_cast<size_t>(total);
  OrderKeyCommon c;
  c.err = z_err_;
  c.entry_block = e_block_;
  c.entry_slot = e_slot_;
  c.last_index = d_last_index_;
  c.max_err = d_max_err_;
  c.weight = weights_;
  c.direction = direction;
  launch_1d(s_, OrderRefBuild{c, offset, x_items_}, static_cast<int>(num_entries_), "order_ref_build");
  return device_partial_sort_resident(static_cast<size_t>(total), want, out);
}

// ---------------------------------------------------------------------------
// a11 on the device
#if defined(GB200_HOSTSIM)
void ImageContext::exclusive_scan(const unsigned int* in, unsigned int* out, int n, unsigned long long* total) {
  exclusive_scan_with(in, out, n, total, nullptr);
}
void ImageContext::exclusive_scan_to(const unsigned int* in, unsigned int* out, int n, unsigned long long* d_total) {
  exclusive_scan_with(in, out, n, d_total, nullptr);
}
void ImageContext::exclusive_scan_with(const unsigned int* in, unsigned int* out, int n, unsigned long long* total,
                                       unsigned int*) {
  unsigned long long acc = 0;
  for (int i = 0; i < n; ++i) {
    out[i] = static_cast<unsigned int>(acc);
    acc += in[i];
  }
  *total = acc;
}
void exclusive_scan_device(Stream, const unsigned int* in, unsigned int* out, int n, unsigned int*,
                           unsigned long long* d_total) {
  unsigned long long acc = 0;
  for (int i = 0; i < n; ++i) {
    out[i] = static_cast<unsigned int>(acc);
    acc += in[i];
  }
  *d_total = acc;
}
#else
namespace {
// 1024 elements per CTA (256 threads x 4): local exclusive scan + CTA total.
__global__ void __launch_bounds__(256) k_scan_local(const unsigned int* in, unsigned int* out, unsigned int* sums, int n) {
  __shared__ unsigned int warp_tot[8];
  const int base = blockIdx.x * 1024 + threadIdx.x * 4;
  unsigned int v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = (base + k < n) ? in[base + k] : 0u;
  const unsigned int mine = v[0] + v[1] + v[2] + v[3];
  unsigned int incl = mine;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned int t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  unsigned int warp_base = 0;
  for (int k = 0; k < warp; ++k) warp_base += warp_tot[k];
  unsigned int run = warp_base + incl - mine;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (base + k < n) out[base + k] = run;
    run += v[k];
  }
  if (threadIdx.x == 255) sums[blockIdx.x] = warp_base + incl;
}
// Single CTA: exclusive scan of the CTA totals (64-bit running sum), grand total.
__global__ void __launch_bounds__(1024) k_scan_sums(unsigned int* sums, int m, unsigned long long* total) {
  __shared__ unsigned long long carry;
  __shared__ unsigned long long warp_tot[32];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int start = 0; start < m; start += 1024) {
    const int i = start + threadIdx.x;
    const unsigned long long v = i < m ? sums[i] : 0ull;
    unsigned long long incl = v;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    unsigned long long wb = 0;
    for (int k = 0; k < warp; ++k) wb += warp_tot[k];
    const unsigned long long excl = carry + wb + incl - v;
    if (i < m) sums[i] = static_cast<unsigned int>(excl);
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}
__global__ void __launch_bounds__(256) k_scan_add(unsigned int* out, const unsigned int* sums, int n) {
  const int base = blockIdx.x * 1024 + threadIdx.x * 4;
  const unsigned int s = sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (base + k < n) out[base + k] += s;
}
}  // namespace

void ImageContext::exclusive_scan(const unsigned int* in, unsigned int* out, int n, unsigned long long* total) {
  exclusive_scan_with(in, out, n, total, j_sums_);
}
void exclusive_scan_device(Stream s, const unsigned int* in, unsigned int* out, int n, unsigned int* sums,
                           unsigned long long* d_total) {
  const int ctas = (n + 1023) / 1024;
  note_launch("scan_local", s, n);
  k_scan_local<<<ctas, 256, 0, s>>>(in, out, sums, n);
  note_launch_end("scan_local", s);
  note_launch("scan_sums", s, ctas);
  k_scan_sums<<<1, 1024, 0, s>>>(sums, ctas, d_total);
  note_launch_end("scan_sums", s);
  note_launch("scan_add", s, n);
  k_scan_add<<<ctas, 256, 0, s>>>(out, sums, n);
  note_launch_end("scan_add", s);
}
// the same without the round trip: the total goes to device memory (8-byte aligned)
void ImageContext::exclusive_scan_to(const unsigned int* in, unsigned int* out, int n, unsigned long long* d_total) {
  exclusive_scan_device(s_, in, out, n, j_sums_, d_total);
}
void ImageContext::exclusive_scan_with(const unsigned int* in, unsigned int* out, int n, unsigned long long* total,
                                       unsigned int* j_sums_) {
  const int ctas = (n + 1023) / 1024;
  unsigned long long* d_total = reinterpret_cast<unsigned long long*>(j_sums_ + ((ctas + 3) & ~1) + 2);
  // keep the 64-bit total 8-byte aligned inside the scratch buffer
  d_total = reinterpret_cast<unsigned long long*>((reinterpret_cast<uintptr_t>(d_total) + 7) & ~static_cast<uintptr_t>(7));
  exclusive_scan_device(s_, in, out, n, j_sums_, d_total);
  d2h(total, d_total, sizeof(unsigned long long), s_);
}
#endif

void ImageContext::jpeg_histograms(unsigned int* hist, bool* chroma_nonzero) {
  const size_t priv = static_cast<size_t>(kHistCopies) * kHistStride;
#if defined(GB200_HOSTSIM)
  dev_zero(j_hist_, sizeof(unsigned int) * (priv + kHistStride + 2), s_);
#else
  dev_zero(j_hist_ + priv, sizeof(unsigned int) * (kHistStride + 2), s_);
#endif
  unsigned int* flag = j_hist_ + priv + kHistStride;
#if defined(GB200_HOSTSIM)
  launch_1d(s_, JpegHistAcc{d_cand_, d_q_, t_.zigzag, j_hist_, flag, g_.nblocks}, 3 * g_.nblocks, "jpeg_hist_acc");
  launch_1d(s_, JpegHistSum{j_hist_, j_hist_ + priv}, kHistStride, "jpeg_hist_sum");
#else
  launch_jpeg_hist(s_, d_cand_, d_q_, t_.zigzag, j_hist_ + priv, flag, g_.nblocks);
#endif
  std::vector<unsigned int> buf(kHistStride + 2);
  d2h(buf.data(), j_hist_ + priv, sizeof(unsigned int) * (kHistStride + 2), s_);
  memcpy(hist, buf.data(), sizeof(unsigned int) * kHistStride);
  *chroma_nonzero = buf[kHistStride] != 0;
}

#if !defined(GB200_HOSTSIM)
namespace {
// JpegUnitBits / JpegEmit (jpeg_dev.h) with the coefficient blocks staged in shared memory: a
// CTA copies 128 consecutive blocks of one component with fully coalesced 16-byte loads (all
// in flight together) into rows padded to 33 words -- a warp that walks its 32 blocks in
// lock-step then hits 32 different banks -- and every thread visits the symbols of its block
// from there.  Same visitors, same results as the functors.
constexpr int kJpegRowWords = 33;  // 64 int16 = 32 words + 1 pad

__device__ __forceinline__ const int16_t* jpeg_stage_blocks(unsigned int* smem, const int16_t* cand, int c, int b0,
                                                            int nblocks) {
  const int16_t* base = cand + (static_cast<size_t>(c) * nblocks + b0) * 64;
  const int rows = min(128, nblocks - b0);
  for (int j = threadIdx.x; j < rows * 8; j += 128) {
    const int row = j >> 3, part = j & 7;
    const int4 v = *reinterpret_cast<const int4*>(base + static_cast<size_t>(row) * 64 + part * 8);
    unsigned int* d = smem + row * kJpegRowWords + part * 4;
    d[0] = static_cast<unsigned int>(v.x);
    d[1] = static_cast<unsigned int>(v.y);
    d[2] = static_cast<unsigned int>(v.z);
    d[3] = static_cast<unsigned int>(v.w);
  }
  __syncthreads();
  return reinterpret_cast<const int16_t*>(smem + threadIdx.x * kJpegRowWords);
}

// grid (ceil(nblocks / 128), ncomp)
__global__ void __launch_bounds__(128) k_jpeg_unit_bits(JpegUnitBits f) {
  __shared__ unsigned int smem[128 * kJpegRowWords];
  const int c = blockIdx.y, b0 = blockIdx.x * 128, b = b0 + threadIdx.x;
  const int16_t* blk = jpeg_stage_blocks(smem, f.cand, c, b0, f.nblocks);
  if (b >= f.nblocks) return;
  const int* qc = f.q + 64 * c;
  const int prev =
      b > 0 ? div_exact_multiple(f.cand[(static_cast<size_t>(c) * f.nblocks + b - 1) * 64], qc[0]) : 0;
  JpegUnitBits::Visitor v{f.codes.depth + c * 256, f.codes.depth + (3 + c) * 256, 0u};
  visit_block_symbols(blk, qc, prev, f.zigzag, v);
  f.bits[b * f.ncomp + c] = v.n;
}

__global__ void __launch_bounds__(128) k_jpeg_emit(JpegEmit f) {
  __shared__ unsigned int smem[128 * kJpegRowWords];
  const int c = blockIdx.y, b0 = blockIdx.x * 128, b = b0 + threadIdx.x;
  const int16_t* blk = jpeg_stage_blocks(smem, f.cand, c, b0, f.nblocks);
  if (b >= f.nblocks) return;
  const int* qc = f.q + 64 * c;
  const int prev =
      b > 0 ? div_exact_multiple(f.cand[(static_cast<size_t>(c) * f.nblocks + b - 1) * 64], qc[0]) : 0;
  JpegEmit::Visitor v{f.codes.depth + c * 256, f.codes.code + c * 256, f.codes.depth + (3 + c) * 256,
                      f.codes.code + (3 + c) * 256, BitCursor()};
  v.cur.start(f.words, f.offset[b * f.ncomp + c]);
  visit_block_symbols(blk, qc, prev, f.zigzag, v);
  v.cur.finish();
}
}  // namespace
#endif

// The length of the scan is known beforehand from the caller's symbol counts (expected_bits), so
// the pass runs without a host round trip in the middle: unit lengths -> exclusive scan -> emit ->
// 0xFF count, then one copy back of the device's own total (checked against the expectation) and
// the count.
void ImageContext::jpeg_encode_scan(int ncomp, const uint8_t* depth, const uint16_t* code,
                                    unsigned long long expected_bits, size_t* nbytes, size_t* num_ff) {
  if (expected_bits >= (1ull << 32)) throw std::runtime_error("jpeg scan exceeds 2^32 bits");
  h2d(j_depth_, depth, 6 * 256, s_);
  h2d(j_code_, code, 6 * 256 * sizeof(uint16_t), s_);
  JpegCodes codes{j_depth_, j_code_};
  const int units = g_.nblocks * ncomp;
  const unsigned long long total_bits = expected_bits;
  const size_t nwords = static_cast<size_t>((total_bits + 31) >> 5);
  if (nwords + 1 > j_words_cap_) {
    stream_sync(s_);
    if (j_words_) { dev_free(j_words_); j_words_ = nullptr; }
    j_words_cap_ = nwords + nwords / 4 + 1024;
    j_words_ = static_cast<unsigned int*>(dev_alloc(j_words_cap_ * sizeof(unsigned int)));
  }
  dev_zero(j_words_, (nwords + 1) * sizeof(unsigned int), s_);
  // [0] 0xFF count, [2..3] the scan's 64-bit total (copied here by the scan)
  unsigned int* result = j_hist_ + static_cast<size_t>(kHistCopies + 1) * kHistStride + 2;
  dev_zero(result, 4 * sizeof(unsigned int), s_);
#if defined(GB200_HOSTSIM)
  launch_1d(s_, JpegUnitBits{d_cand_, d_q_, t_.zigzag, codes, j_bits_, g_.nblocks, ncomp}, units, "jpeg_unit_bits");
#else
  const dim3 jgrid((g_.nblocks + 127) / 128, ncomp);
  note_launch("jpeg_unit_bits", s_, units);
  k_jpeg_unit_bits<<<jgrid, 128, 0, s_>>>(JpegUnitBits{d_cand_, d_q_, t_.zigzag, codes, j_bits_, g_.nblocks, ncomp});
  note_launch_end("jpeg_unit_bits", s_);
#endif
  exclusive_scan_to(j_bits_, j_offset_, units, reinterpret_cast<unsigned long long*>(result + 2));
#if defined(GB200_HOSTSIM)
  launch_1d(s_, JpegEmit{d_cand_, d_q_, t_.zigzag, codes, j_offset_, j_words_, g_.nblocks, ncomp}, units,
            "jpeg_emit");
#else
  note_launch("jpeg_emit", s_, units);
  k_jpeg_emit<<<jgrid, 128, 0, s_>>>(JpegEmit{d_cand_, d_q_, t_.zigzag, codes, j_offset_, j_words_, g_.nblocks, ncomp});
  note_launch_end("jpeg_emit", s_);
#endif
  if (nwords) launch_1d(s_, JpegCountFF{j_words_, total_bits, result}, static_cast<int>(nwords), "jpeg_count_ff");
  unsigned int back[4] = {0, 0, 0, 0};
  d2h(back, result, sizeof(back), s_);
  const unsigned long long device_bits = (static_cast<unsigned long long>(back[3]) << 32) | back[2];
  if (device_bits != expected_bits)
    throw std::runtime_error("jpeg scan: the device's bit count differs from the host's symbol counts");
  j_nbytes_ = static_cast<size_t>((total_bits + 7) >> 3);
  *nbytes = j_nbytes_;
  *num_ff = back[0];
}

void ImageContext::jpeg_keep_scan() {
  const size_t nwords = (j_nbytes_ + 3) / 4;
  if (nwords > j_best_cap_) {
    stream_sync(s_);
    if (j_best_words_) { dev_free(j_best_words_); j_best_words_ = nullptr; }
    j_best_cap_ = nwords + nwords / 4 + 1024;
    j_best_words_ = static_cast<unsigned int*>(dev_alloc(j_best_cap_ * sizeof(unsigned int)));
  }
  if (nwords) d2d(j_best_words_, j_words_, nwords * sizeof(unsigned int), s_);
  j_best_nbytes_ = j_nbytes_;
}

// f1: prefix | stuffed scan | trailer assembled on the device, one copy back.
void ImageContext::jpeg_fetch_file(const std::string& prefix, const std::string& trailer, std::string* file) {
  bind();
  const size_t nwords = (j_nbytes_ + 3) / 4;
  const size_t ctas = (nwords + 1023) / 1024;
  // scratch: [nwords] counts | [nwords] shifts | CTA sums + 64-bit total
  const size_t scratch_words = 2 * nwords + ctas + 16;
  if (scratch_words > j_file_scratch_cap_) {
    stream_sync(s_);
    if (j_file_scratch_) { dev_free(j_file_scratch_); j_file_scratch_ = nullptr; }
    j_file_scratch_cap_ = scratch_words + scratch_words / 4 + 1024;
    j_file_scratch_ = static_cast<unsigned int*>(dev_alloc(j_file_scratch_cap_ * sizeof(unsigned int)));
  }
  unsigned int* count = j_file_scratch_;
  unsigned int* shift = j_file_scratch_ + nwords;
  unsigned int* sums = j_file_scratch_ + 2 * nwords;
  unsigned long long num_ff = 0;
  if (nwords) {
    launch_1d(s_, JpegWordFF{j_words_, static_cast<unsigned long long>(j_nbytes_), count}, static_cast<int>(nwords),
              "jpeg_word_ff");
    exclusive_scan_with(count, shift, static_cast<int>(nwords), &num_ff, sums);
  }
  const size_t total = prefix.size() + j_nbytes_ + static_cast<size_t>(num_ff) + trailer.size();
  if (total > j_file_cap_) {
    stream_sync(s_);
    if (j_file_) { dev_free(j_file_); j_file_ = nullptr; }
    j_file_cap_ = total + total / 4 + 4096;
    j_file_ = static_cast<uint8_t*>(dev_alloc(j_file_cap_));
  }
  if (!prefix.empty()) h2d(j_file_, prefix.data(), prefix.size(), s_);
  if (nwords)
    launch_1d(s_, JpegStuffBytes{j_words_, shift, static_cast<unsigned long long>(j_nbytes_), j_file_ + prefix.size()},
              static_cast<int>(nwords), "jpeg_stuff_bytes");
  if (!trailer.empty())
    h2d(j_file_ + prefix.size() + j_nbytes_ + static_cast<size_t>(num_ff), trailer.data(), trailer.size(), s_);
  file->resize(total);
  if (total) d2h(&(*file)[0], j_file_, total, s_);
}

void ImageContext::jpeg_fetch_kept_file(const std::string& prefix, const std::string& trailer, std::string* file) {
  std::swap(j_words_, j_best_words_);
  std::swap(j_nbytes_, j_best_nbytes_);
  try {
    jpeg_fetch_file(prefix, trailer, file);
  } catch (...) {
    std::swap(j_words_, j_best_words_);
    std::swap(j_nbytes_, j_best_nbytes_);
    throw;
  }
  std::swap(j_words_, j_best_words_);
  std::swap(j_nbytes_, j_best_nbytes_);
}

void ImageContext::debug_render(float* lin3) {
  launch_1d(s_, RenderBlocks{d_cand_, ba_.lin(), g_, t_}, g_.nblocks, "render_blocks");
  r_.download_planes(ba_.lin(), lin3, 3);
}

void ImageContext::debug_corner_mask(float* out) { d2h(out, corner_mask_, sizeof(float) * 3 * g_.nblocks, s_); }

long ImageContext::launches() const { return total_launches(); }
void ImageContext::set_profiling(bool on) { profiling_enable(on); }
std::vector<KernelStat> ImageContext::kernel_stats() const { return profiling_snapshot(); }
void ImageContext::reset_stats() { profiling_reset(); }

// ---------------------------------------------------------------------------
// JPEG decode (JpegIdctIslow, JpegUpsampleYccRgb in kernels.h)
namespace {
#if !defined(GB200_HOSTSIM)
// JpegUpsampleYccRgb over the call's rows: a warp per row, 8 rows per block (as k_mix_rows)
template <class F>
__global__ void __launch_bounds__(256) k_jpeg_rows(F f, int rows) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row < rows) f(threadIdx.x & 31, row);
}
#endif

// everything a decode acquires is handed back on every path; buffers only once the stream is idle
struct JpegScope {
  Stream s = 0;
  bool have = false;
  std::vector<void*> bufs;
  void* alloc(size_t bytes) {
    bufs.push_back(dev_alloc(bytes));
    return bufs.back();
  }
  template <class T>
  T* alloc_n(size_t count) {
    return static_cast<T*>(alloc(sizeof(T) * (count ? count : 1)));
  }
  void open(int device) {
    select_device(device);
    s = make_stream();
    have = true;
  }
  ~JpegScope() {
    if (have) {
      try {
        stream_sync(s);
      } catch (...) {
      }
      destroy_stream(s);
    }
    for (void* p : bufs) dev_free(p);
  }
};

// The per-file table and block / row runs of one call (kernels.h, JpegDecFile)
struct JpegLayout {
  std::vector<JpegDecFile> tab;
  std::vector<int> blk0, row0, quant;
  long long blocks = 0, rows = 0, pixels = 0;
};

JpegLayout jpeg_layout(const JpegInput* const* files, int n) {
  JpegLayout L;
  L.tab.resize(n);
  L.blk0.resize(n + 1);
  L.row0.resize(n + 1);
  L.quant.assign(static_cast<size_t>(n) * 3 * 64, 1);
  for (int i = 0; i < n; ++i) {
    const JpegInput& j = *files[i];
    JpegDecFile& d = L.tab[i];
    d.w = j.width;
    d.h = j.height;
    d.ncomp = static_cast<int>(j.components.size());
    d.ycc = d.ncomp == 3 && libjpeg_ycbcr(j);
    d.hs = j.max_h;
    d.vs = j.max_v;
    d.cw = (d.w + d.hs - 1) / d.hs;
    d.ch = (d.h + d.vs - 1) / d.vs;
    L.blk0[i] = static_cast<int>(L.blocks);
    for (int c = 0; c < 4; ++c) {
      d.blk0[c] = static_cast<int>(L.blocks);
      if (c >= d.ncomp) continue;
      const JpegComponent& comp = j.components[c];
      d.bw[c] = comp.width_in_blocks;
      memcpy(&L.quant[(3 * i + c) * 64], j.quant[comp.quant_idx].values, 64 * sizeof(int));
      L.blocks += static_cast<long long>(comp.width_in_blocks) * comp.height_in_blocks;
    }
    d.row0 = static_cast<int>(L.rows);
    L.rows += d.h;
    d.out = nullptr;
    L.pixels += static_cast<long long>(d.w) * d.h;
    if (L.blocks > (1LL << 30) || L.rows > (1LL << 30))
      throw std::runtime_error("jpeg_decode_rgb: more than 2^30 blocks or rows in one call");
  }
  L.blk0[n] = static_cast<int>(L.blocks);
  L.row0[n] = static_cast<int>(L.rows);
  for (int i = 0; i < n; ++i) L.row0[i] = L.tab[i].row0;
  return L;
}

// The tail both entries share: the IDCT of every block of the call, then upsampling and colour conversion
// of every row into the files' outputs
void jpeg_idct_upsample(Stream s, const JpegDecFile* d_tab, const int* d_blk0, const int* d_row0, const int* d_quant,
                        const int16_t* d_coeffs, uint8_t* d_samples, int n, const JpegLayout& L) {
  launch_1d(s, JpegIdctIslow{d_coeffs, d_quant, d_tab, d_blk0, n, d_samples}, static_cast<int>(L.blocks),
            "jpeg_idct_islow");
  JpegUpsampleYccRgb up{d_tab, d_row0, n, d_samples, 1};
#if defined(GB200_HOSTSIM)
  launch_2d(s, up, 1, static_cast<int>(L.rows));
#else
  up.lanes = 32;
  note_launch("jpeg_upsample_ycc_rgb", s, static_cast<double>(L.pixels));
  k_jpeg_rows<<<cdiv(static_cast<int>(L.rows), 8), 256, 0, s>>>(up, static_cast<int>(L.rows));
  note_launch_end("jpeg_upsample_ycc_rgb", s);
#endif
}
}  // namespace

void jpeg_decode_rgb(const JpegInput* const* files, int n, int device, uint8_t* const* out, bool out_on_device,
                     Stream stream) {
  JpegLayout L = jpeg_layout(files, n);
  std::vector<JpegDecFile>& tab = L.tab;
  const long long out_bytes = 3 * L.pixels;
  std::vector<int16_t> coeffs(static_cast<size_t>(L.blocks) * 64);
  for (int i = 0; i < n; ++i)
    for (int c = 0; c < tab[i].ncomp; ++c) {
      const std::vector<int16_t>& v = files[i]->components[c].coeffs;
      memcpy(&coeffs[static_cast<size_t>(tab[i].blk0[c]) * 64], v.data(), v.size() * sizeof(int16_t));
    }

  JpegScope sc;
  sc.open(device);
  const Stream s = sc.s;
  uint8_t* staged = nullptr;
  if (out_on_device) {
    for (int i = 0; i < n; ++i) tab[i].out = out[i];
  } else {
    staged = static_cast<uint8_t*>(sc.alloc(static_cast<size_t>(out_bytes)));
    size_t o = 0;
    for (int i = 0; i < n; ++i) {
      tab[i].out = staged + o;
      o += static_cast<size_t>(3) * tab[i].w * tab[i].h;
    }
  }
  JpegDecFile* d_tab = static_cast<JpegDecFile*>(sc.alloc(sizeof(JpegDecFile) * n));
  int* d_blk0 = static_cast<int*>(sc.alloc(sizeof(int) * (n + 1)));
  int* d_row0 = static_cast<int*>(sc.alloc(sizeof(int) * (n + 1)));
  int* d_quant = static_cast<int*>(sc.alloc(sizeof(int) * L.quant.size()));
  int16_t* d_coeffs = static_cast<int16_t*>(sc.alloc(sizeof(int16_t) * coeffs.size()));
  uint8_t* d_samples = static_cast<uint8_t*>(sc.alloc(static_cast<size_t>(L.blocks) * 64));
  h2d(d_tab, tab.data(), sizeof(JpegDecFile) * n, s);
  h2d(d_blk0, L.blk0.data(), sizeof(int) * (n + 1), s);
  h2d(d_row0, L.row0.data(), sizeof(int) * (n + 1), s);
  h2d(d_quant, L.quant.data(), sizeof(int) * L.quant.size(), s);
  h2d(d_coeffs, coeffs.data(), sizeof(int16_t) * coeffs.size(), s);
  if (out_on_device) stream_wait(s, stream);
  jpeg_idct_upsample(s, d_tab, d_blk0, d_row0, d_quant, d_coeffs, d_samples, n, L);
  if (!out_on_device)
    for (int i = 0; i < n; ++i) d2h(out[i], tab[i].out, static_cast<size_t>(3) * tab[i].w * tab[i].h, s);
  stream_sync(s);
}

// ---------------------------------------------------------------------------
// Heat maps (HeatMap in kernels.h)
void butteraugli_heatmap(const int* w, const int* h, const float* const* diffmap, int n, double good, double bad,
                         uint8_t* const* rgb, bool on_device, int device, Stream stream) {
  std::vector<int> px0(n + 1, 0);
  for (int i = 0; i < n; ++i) {
    const long long end = px0[i] + static_cast<long long>(w[i]) * h[i];
    if (end > 0x7fffffffLL) throw std::runtime_error("butteraugli heatmap: more than 2^31 - 1 pixels in one call");
    px0[i + 1] = static_cast<int>(end);
  }
  const size_t total = static_cast<size_t>(px0[n]);
  JpegScope sc;  // a stream and buffers, handed back on every path
  sc.open(device);
  const Stream s = sc.s;
  std::vector<const float*> in(diffmap, diffmap + n);
  std::vector<uint8_t*> out(rgb, rgb + n);
  uint8_t* staged = nullptr;
  if (on_device) {
    stream_wait(s, stream);
  } else {  // the maps packed and uploaded in one copy, the heat maps back in one
    std::vector<float> packed(total);
    for (int i = 0; i < n; ++i) memcpy(&packed[px0[i]], diffmap[i], sizeof(float) * (px0[i + 1] - px0[i]));
    float* d_in = sc.alloc_n<float>(total);
    h2d(d_in, packed.data(), sizeof(float) * total, s);
    staged = sc.alloc_n<uint8_t>(3 * total);
    for (int i = 0; i < n; ++i) {
      in[i] = d_in + px0[i];
      out[i] = staged + 3 * static_cast<size_t>(px0[i]);
    }
  }
  // one table: the byte steps, input pointers, output pointers, first pixels
  const std::vector<double>& steps = heat_byte_steps();
  const size_t at_in = sizeof(double) * steps.size(), ptrs = sizeof(void*) * n, at_px0 = at_in + 2 * ptrs;
  std::vector<unsigned char> tab(at_px0 + sizeof(int) * (n + 1));
  memcpy(tab.data(), steps.data(), at_in);
  memcpy(tab.data() + at_in, in.data(), ptrs);
  memcpy(tab.data() + at_in + ptrs, out.data(), ptrs);
  memcpy(tab.data() + at_px0, px0.data(), sizeof(int) * (n + 1));
  unsigned char* d_tab = sc.alloc_n<unsigned char>(tab.size());
  h2d(d_tab, tab.data(), tab.size(), s);
  launch_1d(s,
            HeatMap{reinterpret_cast<const float* const*>(d_tab + at_in),
                    reinterpret_cast<uint8_t* const*>(d_tab + at_in + ptrs), reinterpret_cast<const int*>(d_tab + at_px0),
                    reinterpret_cast<const double*>(d_tab), n, good, bad},
            px0[n], "butteraugli_heatmap");
  if (!on_device) {
    std::vector<uint8_t> back(3 * total);
    d2h(back.data(), staged, back.size(), s);
    for (int i = 0; i < n; ++i)
      memcpy(rgb[i], &back[3 * static_cast<size_t>(px0[i])], 3 * static_cast<size_t>(px0[i + 1] - px0[i]));
  }
  stream_sync(s);
}

// ---------------------------------------------------------------------------
// JPEG entropy decoding on the device (JpegSegEnd .. JpegDcChunkApply in kernels.h)
namespace {

// Files the device path takes are shorter than this: bit positions in a restart interval stay below 2^31.
constexpr size_t kJpegMaxDeviceBytes = size_t(1) << 28;
// Synchronisation rounds after the first: an exact state moves on by at least one subsequence per round,
// so the bound covers 64 subsequences or 2^16 bits, whichever is more; files whose states still change
// then are decoded on the host.
int jpeg_max_sync_rounds(int S) { return std::max(64, 65536 / S); }
// What the device files of one call may add up to (scan bytes, subsequences, DC chunks); files beyond it
// are decoded on the host.  Keeps every flat index of jpeg_entropy_decode below 2^31.
constexpr long long kJpegCallBudget = 1LL << 30;

// The shape the device path takes: a file shorter than kJpegMaxDeviceBytes with a sequential 8-bit frame
// (read_jpeg_header checked the precision) of one component, or of three in a sampling libjpeg_decodable
// accepts, whose first scan carries every component with Ss = 0, Se = 63, Ah = Al = 0
bool jpeg_device_shape(const JpegScanHeader& h, size_t len) {
  if (len >= kJpegMaxDeviceBytes) return false;
  const JpegInput& j = h.jpg;
  const int n = static_cast<int>(j.components.size());
  std::string why;
  if (j.progressive || !libjpeg_decodable(j, &why)) return false;  // no coefficients: the layout checks only
  const JpegScanSpec& sp = h.scan;
  if (sp.ncomp != n || sp.ss != 0 || sp.se != 63 || sp.ah != 0 || sp.al != 0) return false;
  int slots = 0;
  for (const JpegComponent& c : j.components) slots += n > 1 ? c.h_samp * c.v_samp : 1;
  return slots <= kJpegMaxSlots;
}

// MCUs of the first scan, as scan() (jpeg_in.cc) counts them
void jpeg_scan_mcus(const JpegScanHeader& h, int* mcus_per_row, int* mcus) {
  const JpegInput& j = h.jpg;
  *mcus_per_row = j.mcu_cols;
  int mcu_rows = j.mcu_rows;
  if (h.scan.ncomp == 1) {
    const JpegComponent& c = j.components[h.scan.comp[0]];
    *mcus_per_row = (j.width * c.h_samp + 8 * j.max_h - 1) / (8 * j.max_h);
    mcu_rows = (j.height * c.v_samp + 8 * j.max_v - 1) / (8 * j.max_v);
  }
  *mcus = *mcus_per_row * mcu_rows;
}

// Upper bounds of what one file adds to jpeg_entropy_decode's flat ranges: scan bytes, subsequences, DC chunks
void jpeg_device_cost(const JpegScanHeader& h, size_t len, int S, long long cost[3]) {
  int mpr = 0, mcus = 0;
  jpeg_scan_mcus(h, &mpr, &mcus);
  const int R = h.restart_interval;
  const long long nint = R > 0 ? (mcus + R - 1) / R : 1;
  long long per_mcu = 0;
  for (int si = 0; si < h.scan.ncomp; ++si) {
    const JpegComponent& c = h.jpg.components[h.scan.comp[si]];
    per_mcu += h.scan.ncomp > 1 ? c.h_samp * c.v_samp : 1;
  }
  cost[0] = std::max(0LL, static_cast<long long>(len) - 2 - static_cast<long long>(h.scan_start));
  cost[1] = (8 * cost[0] + S - 1) / S + nint;
  cost[2] = nint * h.scan.ncomp + mcus * per_mcu / kJpegDcChunk + 1;
}

// The decoder's copy of a DHT table (JpegHuffDev, kernels.h): decode_symbol over the first 9 bits in `fast`
void jpeg_build_huff(const JpegHuffTable& t, JpegHuffDev* o) {
  memset(o, 0, sizeof(*o));
  memcpy(o->max_code, t.max_code, sizeof(o->max_code));
  memcpy(o->val_offset, t.val_offset, sizeof(o->val_offset));
  memcpy(o->symbols, t.symbols, sizeof(o->symbols));
  o->num_symbols = t.num_symbols;
  for (int w = 0; w < 512; ++w) {
    uint16_t e = 0;
    for (int l = 1; l <= 9; ++l) {
      const int code = w >> (9 - l);
      if (t.max_code[l] >= 0 && code <= t.max_code[l]) {
        const int idx = t.val_offset[l] + code;
        e = idx < t.num_symbols ? static_cast<uint16_t>(0x8000 | (l << 8) | t.symbols[idx]) : 0x4000;
        break;
      }
    }
    o->fast[w] = e;
  }
}

struct JpegDeviceFile {
  const uint8_t* data;  // device memory
  size_t len;
  const JpegScanHeader* hdr;
  const JpegDecFile* layout;  // blk0 of each component
};

// Entropy-decodes the files into d_coeffs (zeroed, laid out as `layout` says) on s; d_status[i] receives
// the kJpegBad* flags of file i, and d_end[i] (if given; else scratch) the offset of the marker that ends
// file i's scan data, EOI where no kJpegBadSegment is raised.  Returns the number of synchronisation rounds
// after the first.
int jpeg_entropy_decode(const std::vector<JpegDeviceFile>& fs, int16_t* d_coeffs, int S, Stream s, JpegScope* sc,
                        unsigned* d_status, unsigned* d_end = nullptr) {
  const int n = static_cast<int>(fs.size());
  if (n == 0) return 0;
  if (S < 8) throw std::runtime_error("jpeg entropy decode: subsequences of fewer than 8 bits");
  std::vector<JpegScanFile> tab(n);
  std::vector<int> byte0(n + 1), int0(n + 1);
  std::vector<unsigned> end(n);
  std::map<std::string, int> lut_ids;
  std::vector<JpegHuffDev> luts;
  std::vector<JpegDcTask> tasks;
  std::vector<int> chunk0;
  long long bytes = 0, intervals = 0, subs = 0, chunks = 0;
  auto lut = [&](const JpegHuffTable& t) {
    std::string key(reinterpret_cast<const char*>(t.max_code), sizeof(t.max_code));
    key.append(reinterpret_cast<const char*>(t.val_offset), sizeof(t.val_offset));
    key.append(reinterpret_cast<const char*>(t.symbols), t.num_symbols);
    key.append(1, static_cast<char>(t.num_symbols & 255)).append(1, static_cast<char>(t.num_symbols >> 8));
    auto it = lut_ids.find(key);
    if (it != lut_ids.end()) return it->second;
    const int id = static_cast<int>(lut_ids.size());
    lut_ids[key] = id;
    luts.resize(luts.size() + 1);
    jpeg_build_huff(t, &luts.back());
    return id;
  };
  for (int i = 0; i < n; ++i) {
    const JpegScanHeader& h = *fs[i].hdr;
    const JpegInput& j = h.jpg;
    JpegScanFile& d = tab[i];
    memset(&d, 0, sizeof(d));
    d.data = fs[i].data;
    d.len = static_cast<long long>(fs[i].len);
    d.s0 = static_cast<int>(h.scan_start);
    const long long nb = std::max(0LL, d.len - 2 - d.s0);
    byte0[i] = static_cast<int>(bytes);
    bytes += nb;
    end[i] = static_cast<unsigned>(d.len >= 2 ? d.len - 2 : 0);
    const bool inter = h.scan.ncomp > 1;
    jpeg_scan_mcus(h, &d.mcus_per_row, &d.mcus);
    d.R = h.restart_interval;
    d.nint = d.R > 0 ? (d.mcus + d.R - 1) / d.R : 1;
    d.int0 = static_cast<int>(intervals);
    int0[i] = d.int0;
    for (int si = 0; si < h.scan.ncomp; ++si) {
      const int c = h.scan.comp[si];
      const JpegComponent& comp = j.components[c];
      d.comp_h[c] = inter ? comp.h_samp : 1;
      d.comp_v[c] = inter ? comp.v_samp : 1;
      d.bw[c] = comp.width_in_blocks;
      d.blk0[c] = fs[i].layout->blk0[c];
      const int dc = lut(h.dc[h.scan.dc_tbl[si]]), ac = lut(h.ac[h.scan.ac_tbl[si]]);
      for (int iy = 0; iy < d.comp_v[c]; ++iy)
        for (int ix = 0; ix < d.comp_h[c]; ++ix) {
          d.slot_comp[d.nslot] = c;
          d.slot_ix[d.nslot] = ix;
          d.slot_iy[d.nslot] = iy;
          d.slot_dc[d.nslot] = dc;
          d.slot_ac[d.nslot] = ac;
          ++d.nslot;
        }
    }
    for (d.period = 1; d.period < d.nslot; ++d.period) {
      if (d.nslot % d.period) continue;
      bool same = true;
      for (int k = d.period; k < d.nslot && same; ++k)
        same = d.slot_dc[k] == d.slot_dc[k % d.period] && d.slot_ac[k] == d.slot_ac[k % d.period];
      if (same) break;
    }
    for (int k = 0; k < d.nint; ++k) {
      const int nmcu = d.R > 0 ? std::min(d.R, d.mcus - k * d.R) : d.mcus;
      for (int si = 0; si < h.scan.ncomp; ++si) {
        const int c = h.scan.comp[si];
        JpegDcTask t{i, d.int0 + k, c, nmcu * d.comp_h[c] * d.comp_v[c]};
        tasks.push_back(t);
        chunk0.push_back(static_cast<int>(chunks));
        chunks += (t.nblk + kJpegDcChunk - 1) / kJpegDcChunk;
      }
    }
    intervals += d.nint;
    subs += (8 * nb + S - 1) / S + d.nint;
  }
  byte0[n] = static_cast<int>(bytes);
  int0[n] = static_cast<int>(intervals);
  chunk0.push_back(static_cast<int>(chunks));
  if (bytes >= (1LL << 31) - 1 || subs >= (1LL << 31) - 1 || chunks >= (1LL << 31) - 1)
    throw std::runtime_error("jpeg entropy decode: more than 2^31 scan bytes or subsequences in one call");
  // (the entries keep their device files within kJpegCallBudget and kJpegMaxDeviceBytes, far below that)
  const int B = static_cast<int>(bytes), NI = static_cast<int>(intervals), U = static_cast<int>(subs);
  const int NT = static_cast<int>(tasks.size()), NC = static_cast<int>(chunks);

  const int scan_max = std::max(std::max(B, U), std::max(NI, NC)) + 1;
  unsigned* sums = sc->alloc_n<unsigned>((scan_max + 1023) / 1024 + 2);
  unsigned long long* d_total = sc->alloc_n<unsigned long long>(1);
  JpegScanFile* d_tab = sc->alloc_n<JpegScanFile>(n);
  int* d_byte0 = sc->alloc_n<int>(n + 1);
  int* d_int0 = sc->alloc_n<int>(n + 1);
  if (d_end == nullptr) d_end = sc->alloc_n<unsigned>(n);
  JpegHuffDev* d_luts = sc->alloc_n<JpegHuffDev>(luts.size());
  uint8_t* d_zz = sc->alloc_n<uint8_t>(64);
  unsigned* keep = sc->alloc_n<unsigned>(B + 1);
  unsigned* rst = sc->alloc_n<unsigned>(B + 1);
  unsigned* cpos = sc->alloc_n<unsigned>(B + 1);
  unsigned* ridx = sc->alloc_n<unsigned>(B + 1);
  uint8_t* comp = sc->alloc_n<uint8_t>(B);
  long long* istart = sc->alloc_n<long long>(NI);
  JpegInterval* ivs = sc->alloc_n<JpegInterval>(NI);
  unsigned* nsub = sc->alloc_n<unsigned>(NI + 1);
  unsigned* sub0 = sc->alloc_n<unsigned>(NI + 1);
  unsigned long long* exit_a = sc->alloc_n<unsigned long long>(U);
  unsigned long long* exit_b = sc->alloc_n<unsigned long long>(U);
  unsigned long long* entry = sc->alloc_n<unsigned long long>(U);
  unsigned* count = sc->alloc_n<unsigned>(U + 1);
  unsigned* bscan = sc->alloc_n<unsigned>(U + 1);
  unsigned* changed = sc->alloc_n<unsigned>(1);
  JpegDcTask* d_tasks = sc->alloc_n<JpegDcTask>(NT);
  int* d_chunk0 = sc->alloc_n<int>(NT + 1);
  unsigned* csum = sc->alloc_n<unsigned>(NC + 1);
  unsigned* cscan = sc->alloc_n<unsigned>(NC + 1);
  uint8_t zz[64];
  for (int k = 0; k < 64; ++k) zz[k] = static_cast<uint8_t>(zigzag_to_natural()[k]);
  h2d(d_tab, tab.data(), sizeof(JpegScanFile) * n, s);
  h2d(d_byte0, byte0.data(), sizeof(int) * (n + 1), s);
  h2d(d_int0, int0.data(), sizeof(int) * (n + 1), s);
  h2d(d_end, end.data(), sizeof(unsigned) * n, s);
  h2d(d_luts, luts.data(), sizeof(JpegHuffDev) * luts.size(), s);
  h2d(d_zz, zz, 64, s);
  h2d(d_tasks, tasks.data(), sizeof(JpegDcTask) * NT, s);
  h2d(d_chunk0, chunk0.data(), sizeof(int) * (NT + 1), s);
  dev_zero(keep + B, sizeof(unsigned), s);
  dev_zero(rst + B, sizeof(unsigned), s);
  dev_zero(istart, sizeof(long long) * std::max(NI, 1), s);
  dev_zero(nsub + NI, sizeof(unsigned), s);
  dev_zero(count, sizeof(unsigned) * (U + 1), s);
  dev_zero(csum + NC, sizeof(unsigned), s);

  // 4.1: segment pass
  launch_1d(s, JpegSegEnd{d_tab, d_byte0, n, d_end}, B, "jpeg_seg_end");
  launch_1d(s, JpegSegFlags{d_tab, d_byte0, n, d_end, keep, rst}, B, "jpeg_seg_flags");
  exclusive_scan_device(s, keep, cpos, B + 1, sums, d_total);
  exclusive_scan_device(s, rst, ridx, B + 1, sums, d_total);
  launch_1d(s, JpegSegCompact{d_tab, d_byte0, n, keep, cpos, rst, ridx, comp, istart, d_status}, B, "jpeg_seg_compact");
  launch_1d(s, JpegIntervals{d_tab, d_byte0, d_int0, n, d_end, cpos, ridx, istart, S, ivs, nsub, d_status}, NI,
            "jpeg_intervals");
  exclusive_scan_device(s, nsub, sub0, NI + 1, sums, d_total);

  // 4.2: speculative decode, synchronised until no exit state changes, or for jpeg_max_sync_rounds(S) rounds,
  // the last of which flags the files that have not converged (kJpegBadSync)
  const JpegSubs subsq{d_tab, ivs, NI, sub0, d_luts, comp, S};
  launch_1d(s, JpegHuffSync{subsq, 0, exit_b, exit_a, entry, count, changed, nullptr}, U, "jpeg_huff_sync");
  int rounds = 0;
  for (;;) {
    ++rounds;
    const bool last = rounds == jpeg_max_sync_rounds(S);
    dev_zero(changed, sizeof(unsigned), s);
    launch_1d(s, JpegHuffSync{subsq, rounds, exit_a, exit_b, entry, count, changed, last ? d_status : nullptr}, U,
              "jpeg_huff_sync");
    std::swap(exit_a, exit_b);
    unsigned h_changed = 0;
    d2h(&h_changed, changed, sizeof(unsigned), s);
    if (!h_changed || last) break;
  }
  exclusive_scan_device(s, count, bscan, U + 1, sums, d_total);
  launch_1d(s, JpegHuffWrite{subsq, entry, bscan, d_zz, d_coeffs, d_status}, U, "jpeg_huff_write");
  launch_1d(s, JpegDcChunkSum{d_tab, ivs, d_tasks, d_chunk0, NT, d_coeffs, csum}, NC, "jpeg_dc_sum");
  exclusive_scan_device(s, csum, cscan, NC + 1, sums, d_total);
  launch_1d(s, JpegDcChunkApply{d_tab, ivs, d_tasks, d_chunk0, NT, d_coeffs, cscan, d_status}, NC, "jpeg_dc_apply");
  return rounds;
}

std::string jpeg_file_reason(const std::string& who, int i, const std::string& why) {
  return who + ": file " + std::to_string(i) + ": " + why;
}

// The host path of one file: read_jpeg and the checks of gb200_jpeg_decode_rgb, then the output size;
// "" where the file is accepted
std::string jpeg_host_check(const std::vector<uint8_t>& b, int width, int height, JpegInput* jpg) {
  std::string why;
  if (!read_jpeg(b.data(), b.size(), jpg, &why)) return why;
  int w = 0, h = 0;
  if (!read_jpeg_dimensions(b.data(), b.size(), &w, &h) || w != jpg->width || h != jpg->height)
    return "the frame size differs from what gb200_jpeg_dimensions reads";
  if (width != jpg->width || height != jpg->height)
    return "the output is " + std::to_string(width) + "x" + std::to_string(height) + ", the frame " +
           std::to_string(jpg->width) + "x" + std::to_string(jpg->height);
  if (!libjpeg_decodable(*jpg, &why)) return why;
  return "";
}

constexpr size_t kJpegFirstPrefix = 4096;

// The headers of n files in device memory (read_jpeg_header), from prefixes copied to the host on s, 4 KiB
// doubling; each round covers every file still short of its first SOS.  (*head_ok)[i] where file i's was read.
void jpeg_read_headers(const uint8_t* const* jpeg, const size_t* len, int n, Stream s, std::vector<JpegScanHeader>* hdr,
                       std::vector<std::vector<uint8_t> >* pre, std::vector<char>* head_ok) {
  std::vector<char> pending(n, 1);
  for (size_t m = kJpegFirstPrefix;; m *= 2) {
    bool more = false;
    for (int i = 0; i < n; ++i) {
      if (!pending[i]) continue;
      const size_t k = std::min(m, len[i]);
      std::vector<uint8_t>& p = (*pre)[i];
      p.resize(k);
      if (k) d2h(p.data(), jpeg[i], k, s);
      if (read_jpeg_header(p.data(), k, &(*hdr)[i])) {
        (*head_ok)[i] = 1;
        pending[i] = 0;
      } else if (k == len[i]) {
        pending[i] = 0;
      } else {
        more = true;
      }
    }
    if (!more) break;
  }
}

// Whether the device route of process_jpeg_from_device takes a file whose header was read: the shape the
// entropy decode takes, within one call's budget, and a frame the encoder would encode
bool jpeg_seed_takes(const JpegScanHeader& h, size_t len, int S, bool (*encodable)(const JpegInput&)) {
  if (!jpeg_device_shape(h, len) || !encodable(h.jpg)) return false;
  long long cost[3];
  jpeg_device_cost(h, len, S, cost);
  return cost[0] < kJpegCallBudget && cost[1] < kJpegCallBudget && cost[2] < kJpegCallBudget;
}

// The device route's work on one file the route takes (d_data: its len bytes in device memory), on sc->s:
// the entropy decode, then JpegDequantSanity into *dq ([3][nblocks][64], sc's memory).  kHost where the
// decode flags the file or finds more than EOI after its scan; else kInsane or kTaken, with the offset of
// EOI in *eoi.
JpegSeed::Route jpeg_seed_decode(const uint8_t* d_data, size_t len, const JpegScanHeader& hdr, int S, JpegScope* sc,
                                 int16_t** dq, size_t* eoi) {
  const Stream s = sc->s;
  const JpegInput* one = &hdr.jpg;
  const JpegLayout L = jpeg_layout(&one, 1);
  const size_t ncoef = static_cast<size_t>(L.blocks) * 64;
  int16_t* d_coeffs = sc->alloc_n<int16_t>(ncoef);
  *dq = sc->alloc_n<int16_t>(ncoef);
  int* d_quant = sc->alloc_n<int>(3 * 64);
  unsigned* d_words = sc->alloc_n<unsigned>(2);  // the status word, the end of the scan data
  dev_zero(d_coeffs, sizeof(int16_t) * ncoef, s);
  dev_zero(d_words, sizeof(unsigned), s);
  h2d(d_quant, L.quant.data(), sizeof(int) * 3 * 64, s);
  std::vector<JpegDeviceFile> fs{JpegDeviceFile{d_data, len, &hdr, &L.tab[0]}};
  jpeg_entropy_decode(fs, d_coeffs, S, s, sc, d_words, d_words + 1);
  launch_1d(s, JpegDequantSanity{d_coeffs, d_quant, static_cast<int>(L.blocks / 3), *dq, d_words},
            static_cast<int>(ncoef), "jpeg_dequant_sanity");
  unsigned words[2];
  d2h(words, d_words, sizeof(words), s);
  if (words[0] & ~kJpegBadSanity) return JpegSeed::kHost;
  *eoi = words[1];
  return words[0] ? JpegSeed::kInsane : JpegSeed::kTaken;
}
}  // namespace

void jpeg_seed_from_device(const uint8_t* jpeg, size_t len, int device, Stream stream, int S,
                           bool (*encodable)(const JpegInput&), JpegSeed* out) {
  auto sc = std::make_shared<JpegScope>();
  sc->open(device);
  const Stream s = sc->s;
  stream_wait(s, stream);
  std::vector<JpegScanHeader> hdr(1);
  std::vector<std::vector<uint8_t> > pre(1);
  std::vector<char> head_ok(1, 0);
  jpeg_read_headers(&jpeg, &len, 1, s, &hdr, &pre, &head_ok);
  out->route = JpegSeed::kHost;
  int16_t* dq = nullptr;
  size_t eoi = 0;
  if (head_ok[0] && jpeg_seed_takes(hdr[0], len, S, encodable))
    out->route = jpeg_seed_decode(jpeg, len, hdr[0], S, sc.get(), &dq, &eoi);
  if (out->route == JpegSeed::kHost) {
    out->file.resize(len);
    d2h(out->file.data(), jpeg, len, s);
    return;
  }
  out->hdr = std::move(hdr[0]);
  out->tail.resize(len - eoi - 2);
  if (!out->tail.empty()) d2h(&out->tail[0], jpeg + eoi + 2, out->tail.size(), s);
  out->dq = dq;
  out->stream = s;
  out->keep = sc;
}

JpegSeed::Route jpeg_debug_seed(const uint8_t* data, size_t len, int S, bool (*encodable)(const JpegInput&),
                                std::vector<int16_t>* dq) {
  JpegScanHeader hdr;
  if (!read_jpeg_header(data, len, &hdr) || !jpeg_seed_takes(hdr, len, S, encodable)) return JpegSeed::kHost;
  JpegScope sc;
  sc.open(0);
  uint8_t* d_data = sc.alloc_n<uint8_t>(len);
  h2d(d_data, data, len, sc.s);
  int16_t* d_dq = nullptr;
  size_t eoi = 0;
  const JpegSeed::Route r = jpeg_seed_decode(d_data, len, hdr, S, &sc, &d_dq, &eoi);
  if (r != JpegSeed::kHost) {
    dq->resize(static_cast<size_t>(hdr.jpg.components[0].width_in_blocks) * hdr.jpg.components[0].height_in_blocks * 192);
    d2h(dq->data(), d_dq, sizeof(int16_t) * dq->size(), sc.s);
  }
  return r;
}

void jpeg_dimensions_from_device(const uint8_t* const* jpeg, const size_t* len, int n, int device, Stream stream,
                                 int* width, int* height) {
  JpegScope sc;
  sc.open(device);
  stream_wait(sc.s, stream);
  std::vector<uint8_t> b;
  for (int i = 0; i < n; ++i) {
    width[i] = height[i] = 0;
    for (size_t m = std::min(kJpegFirstPrefix, len[i]);; m = std::min(2 * m, len[i])) {
      b.resize(m);
      if (m) d2h(b.data(), jpeg[i], m, sc.s);
      int w = 0, h = 0;
      if (read_jpeg_dimensions(b.data(), m, &w, &h)) {
        width[i] = w;
        height[i] = h;
        break;
      }
      if (m == len[i]) break;
    }
  }
}

void jpeg_decode_rgb_from_device(const char* who, const uint8_t* const* jpeg, const size_t* len, int n, int device,
                                 const int* width, const int* height, uint8_t* const* out, Stream stream) {
  JpegScope sc;
  sc.open(device);
  const Stream s = sc.s;
  stream_wait(s, stream);
  std::vector<JpegScanHeader> hdr(n);
  std::vector<std::vector<uint8_t> > pre(n);
  std::vector<char> head_ok(n, 0);
  jpeg_read_headers(jpeg, len, n, s, &hdr, &pre, &head_ok);
  std::vector<char> dev(n, 0);
  std::vector<std::string> why(n);
  std::vector<JpegInput> host(n);
  std::vector<char> host_ok(n, 0);
  auto host_path = [&](int i) {
    std::vector<uint8_t> b(len[i]);
    if (len[i]) d2h(b.data(), jpeg[i], len[i], s);
    why[i] = jpeg_host_check(b, width[i], height[i], &host[i]);
    host_ok[i] = why[i].empty();
  };
  long long budget[3] = {0, 0, 0};
  for (int i = 0; i < n; ++i) {
    int w = 0, h = 0;
    dev[i] = head_ok[i] && jpeg_device_shape(hdr[i], len[i]) &&
             read_jpeg_dimensions(pre[i].data(), pre[i].size(), &w, &h) && w == hdr[i].jpg.width &&
             h == hdr[i].jpg.height;
    if (dev[i]) {
      long long cost[3];
      jpeg_device_cost(hdr[i], len[i], kJpegSubBits, cost);
      for (int k = 0; k < 3; ++k) dev[i] = dev[i] && budget[k] + cost[k] < kJpegCallBudget;
      if (dev[i])
        for (int k = 0; k < 3; ++k) budget[k] += cost[k];
    }
    if (!dev[i]) host_path(i);
  }
  static const JpegInput kEmpty;
  std::vector<const JpegInput*> lay(n);
  for (int i = 0; i < n; ++i) lay[i] = dev[i] ? &hdr[i].jpg : (host_ok[i] ? &host[i] : &kEmpty);
  JpegLayout L = jpeg_layout(lay.data(), n);
  std::vector<int> check(n);
  std::vector<JpegDeviceFile> fs;
  for (int i = 0; i < n; ++i) {
    check[i] = dev[i];
    if (check[i]) fs.push_back(JpegDeviceFile{jpeg[i], len[i], &hdr[i], &L.tab[i]});
  }
  for (int i = 0; i < n; ++i) L.tab[i].out = out[i];
  JpegDecFile* d_tab = sc.alloc_n<JpegDecFile>(n);
  int* d_blk0 = sc.alloc_n<int>(n + 1);
  int* d_row0 = sc.alloc_n<int>(n + 1);
  int* d_quant = sc.alloc_n<int>(L.quant.size());
  int* d_check = sc.alloc_n<int>(n);
  unsigned* d_status = sc.alloc_n<unsigned>(n);
  int16_t* d_coeffs = sc.alloc_n<int16_t>(static_cast<size_t>(L.blocks) * 64);
  h2d(d_tab, L.tab.data(), sizeof(JpegDecFile) * n, s);
  h2d(d_blk0, L.blk0.data(), sizeof(int) * (n + 1), s);
  h2d(d_row0, L.row0.data(), sizeof(int) * (n + 1), s);
  h2d(d_quant, L.quant.data(), sizeof(int) * L.quant.size(), s);
  h2d(d_check, check.data(), sizeof(int) * n, s);
  if (!fs.empty()) {
    dev_zero(d_coeffs, sizeof(int16_t) * 64 * static_cast<size_t>(L.blocks), s);
    // the status words of the device files, in call order
    unsigned* st = sc.alloc_n<unsigned>(fs.size());
    dev_zero(st, sizeof(unsigned) * fs.size(), s);
    jpeg_entropy_decode(fs, d_coeffs, kJpegSubBits, s, &sc, st);
    std::vector<unsigned> zeros(n, 0);
    h2d(d_status, zeros.data(), sizeof(unsigned) * n, s);
    std::vector<unsigned> hs(fs.size());
    // scatter the per-device-file words to call order through the host: one small copy each way
    d2h(hs.data(), st, sizeof(unsigned) * fs.size(), s);
    launch_1d(s, JpegRangeCheck{d_coeffs, d_quant, d_tab, d_blk0, n, d_check, d_status}, static_cast<int>(L.blocks),
              "jpeg_range_check");
    std::vector<unsigned> range(n);
    d2h(range.data(), d_status, sizeof(unsigned) * n, s);
    for (int i = 0, k = 0; i < n; ++i) {
      if (!check[i]) continue;
      const unsigned flags = hs[k++] | range[i];
      if (flags) {
        // read_jpeg decides, with its own reasons in the host entry's order (the output size among them)
        host_path(i);
        if (host_ok[i]) {
          for (size_t c = 0; c < host[i].components.size(); ++c) {
            const std::vector<int16_t>& v = host[i].components[c].coeffs;
            h2d(d_coeffs + static_cast<size_t>(L.tab[i].blk0[c]) * 64, v.data(), v.size() * sizeof(int16_t), s);
          }
        }
      } else if (width[i] != hdr[i].jpg.width || height[i] != hdr[i].jpg.height) {
        // read_jpeg accepts the file, so the size is the first reason jpeg_host_check would give
        why[i] = "the output is " + std::to_string(width[i]) + "x" + std::to_string(height[i]) + ", the frame " +
                 std::to_string(hdr[i].jpg.width) + "x" + std::to_string(hdr[i].jpg.height);
      }
    }
  }
  for (int i = 0; i < n; ++i)
    if (!why[i].empty()) throw std::runtime_error(jpeg_file_reason(who, i, why[i]));
  for (int i = 0; i < n; ++i)
    if (!dev[i])
      for (size_t c = 0; c < host[i].components.size(); ++c) {
        const std::vector<int16_t>& v = host[i].components[c].coeffs;
        h2d(d_coeffs + static_cast<size_t>(L.tab[i].blk0[c]) * 64, v.data(), v.size() * sizeof(int16_t), s);
      }
  uint8_t* d_samples = sc.alloc_n<uint8_t>(static_cast<size_t>(L.blocks) * 64);
  jpeg_idct_upsample(s, d_tab, d_blk0, d_row0, d_quant, d_coeffs, d_samples, n, L);
  stream_sync(s);
}

bool jpeg_debug_entropy_decode(const uint8_t* data, size_t len, int S, std::vector<int16_t>* coeffs) {
  JpegDebugDecode r;
  jpeg_debug_entropy_decode_flags(data, len, S, coeffs, &r);
  return r.taken && (r.flags & ~kJpegBadRange) == 0;
}

void jpeg_debug_entropy_decode_flags(const uint8_t* data, size_t len, int S, std::vector<int16_t>* coeffs,
                                     JpegDebugDecode* r) {
  *r = JpegDebugDecode();
  coeffs->clear();
  JpegScanHeader hdr;
  if (!read_jpeg_header(data, len, &hdr) || !jpeg_device_shape(hdr, len)) return;
  r->taken = true;
  const JpegInput* one = &hdr.jpg;
  JpegLayout L = jpeg_layout(&one, 1);
  JpegScope sc;
  sc.open(0);
  const Stream s = sc.s;
  uint8_t* d_data = sc.alloc_n<uint8_t>(len);
  h2d(d_data, data, len, s);
  int16_t* d_coeffs = sc.alloc_n<int16_t>(static_cast<size_t>(L.blocks) * 64);
  unsigned* d_status = sc.alloc_n<unsigned>(1);
  dev_zero(d_coeffs, sizeof(int16_t) * 64 * static_cast<size_t>(L.blocks), s);
  dev_zero(d_status, sizeof(unsigned), s);
  std::vector<JpegDeviceFile> fs{JpegDeviceFile{d_data, len, &hdr, &L.tab[0]}};
  r->rounds = jpeg_entropy_decode(fs, d_coeffs, S, s, &sc, d_status);
  // the SIMD-range test of jpeg_decode_rgb_from_device, on the same status word
  JpegDecFile* d_tab = sc.alloc_n<JpegDecFile>(1);
  int* d_blk0 = sc.alloc_n<int>(2);
  int* d_quant = sc.alloc_n<int>(L.quant.size());
  int* d_check = sc.alloc_n<int>(1);
  const int check = 1;
  h2d(d_tab, L.tab.data(), sizeof(JpegDecFile), s);
  h2d(d_blk0, L.blk0.data(), sizeof(int) * 2, s);
  h2d(d_quant, L.quant.data(), sizeof(int) * L.quant.size(), s);
  h2d(d_check, &check, sizeof(int), s);
  launch_1d(s, JpegRangeCheck{d_coeffs, d_quant, d_tab, d_blk0, 1, d_check, d_status}, static_cast<int>(L.blocks),
            "jpeg_range_check");
  d2h(&r->flags, d_status, sizeof(unsigned), s);
  if (r->flags & ~kJpegBadRange) return;
  coeffs->resize(static_cast<size_t>(L.blocks) * 64);
  d2h(coeffs->data(), d_coeffs, sizeof(int16_t) * coeffs->size(), s);
}

}  // namespace gb200
