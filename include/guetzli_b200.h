/* guetzli_b200 -- C ABI of the H100-native Guetzli hot path.
 *
 * Drop-in boundary: the reference's public entry point for this path is the
 * C++ free function
 *     bool guetzli::Process(const Params&, ProcessStats*, const std::vector<uint8_t>& rgb,
 *                           int w, int h, std::string* out)      (guetzli/processor.h:54-56,
 *                                                                 guetzli/processor.cc:926)
 * called by the CLI (guetzli/guetzli.cc:301).  gb200_process_rgb() is that call
 * with plain C types; include/guetzli_b200_compat.h re-creates the C++ signature on
 * top of it, INTEGRATION.md shows the reference-side binding.
 *
 * The gb200_image_* functions expose the device-resident stages individually
 * (the reference's internal `Comparator` seam, guetzli/comparator.h:29-96, moved
 * down to device memory) for differential tests and for hosts that own the loop.
 *
 * Conventions: plain pointers and sizes, caller-owned inputs (not retained after
 * return), library-allocated outputs freed with gb200_free(), int return 1 = ok /
 * 0 = failure with gb200_last_error() set (thread-local), no exceptions across
 * the ABI, one image context = one host thread + one CUDA stream.
 * There is NO CPU fallback: every entry point that computes fails when no CUDA
 * device (sm_90a) is present.
 */
#ifndef GUETZLI_B200_H_
#define GUETZLI_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* guetzli::Params (guetzli/processor.h:29-37), same fields, same defaults. */
typedef struct gb200_params {
  float butteraugli_target;     /* 1.0 */
  int clear_metadata;           /* 1 */
  int try_420;                  /* 0; unsupported when set (DESIGN.md, out of scope) */
  int force_420;                /* 0; unsupported when set */
  int use_silver_screen;        /* 0 */
  int zeroing_greedy_lookahead; /* 3 */
  int new_zeroing_model;        /* 1 = csf/bias score, 0 = legacy score (processor.cc:388-393) */
} gb200_params;

/* guetzli::ProcessStats counters (guetzli/stats.h:29-40) + device accounting. */
typedef struct gb200_stats {
  int iterations;      /* "number of iterations" */
  int iterations_up;   /* "number of iterations up" */
  int iterations_down; /* "number of iterations down" */
  int compares;        /* full-image Compare calls */
  long gpu_launches;   /* CUDA kernels launched by this call */
  long long h2d_bytes; /* host->device bytes copied by this call */
  long long d2h_bytes; /* device->host bytes copied by this call */
  double ms_total, ms_device_setup, ms_compare, ms_zeroing, ms_jpeg, ms_sort, ms_walk;
  int order_partial; /* selection-walk iterations served by the device top-K order */
  int order_exact;   /* ... by the complete reference-ordered std::sort */
} gb200_stats;

/* ProcessStats::debug_output / --verbose sink (guetzli/debug_print.h:28-47). */
typedef void (*gb200_log_fn)(void* user, const char* text);

void gb200_params_default(gb200_params* p);

/* guetzli::ButteraugliScoreForQuality (guetzli/quality.cc:78). */
double gb200_butteraugli_score_for_quality(double quality);

/* guetzli::Process(params, stats, rgb, w, h, &out) (guetzli/processor.cc:926).
 * rgb: interleaved 8-bit sRGB, 3*w*h bytes.  *out is allocated by the library. */
int gb200_process_rgb(const gb200_params* params, const uint8_t* rgb, int w, int h, int device,
                      gb200_log_fn log, void* log_user, uint8_t** out, size_t* out_len,
                      gb200_stats* stats);

/* ---- 8-bit images of any channel count and layout, from host or device memory ----
 * img holds w x h pixels of `channels` 8-bit samples: 1 (gray), 2 (gray + alpha), 3 (RGB) or 4 (RGBA).
 * Sample (y, x, c) is at byte y * strides[0] + x * strides[1] + c * strides[2] of img; strides (int64[3]:
 * row, pixel, channel bytes, each >= 0, 0 allowed for a broadcast view) may be NULL for contiguous
 * [h][w][channels].  The image is turned into RGB on the device as the guetzli tool turns PNG layouts into
 * RGB before guetzli::Process (guetzli/guetzli.cc:43-145): gray is replicated, gray + alpha and RGBA are
 * blended on black per sample with (v * a + 128) / 255 in integers (BlendOnBlack; not the butteraugli
 * tool's rule, which rounds with + 127), RGB is copied.  The encoder then runs as gb200_process_rgb runs on
 * that RGB, with its checks and messages; channels outside 1..4 and negative strides are refused as well.
 *
 * gb200_process_image: img in host memory; the smallest span of bytes that covers the view is uploaded. */
int gb200_process_image(const gb200_params* params, const uint8_t* img, int w, int h, int channels,
                        const int64_t* strides, int device, gb200_log_fn log, void* log_user, uint8_t** out,
                        size_t* out_len, gb200_stats* stats);
/* The same with img in device memory of `device`, read in place once the work queued on `stream` so far is
 * done (a cudaStream_t, NULL = the legacy default stream); nothing of the image crosses to the host.  The
 * image has been read when the call returns.  A host, managed or other device's pointer is refused, nothing
 * runs. */
int gb200_process_image_device(const gb200_params* params, const uint8_t* img_dev, int w, int h, int channels,
                               const int64_t* strides, int device, gb200_log_fn log, void* log_user, uint8_t** out,
                               size_t* out_len, gb200_stats* stats, void* stream);

/* guetzli::Process(params, stats, jpeg_in, &out) (guetzli/processor.h:39-41,
 * guetzli/processor.cc:890): JPEG input.  The file is parsed on the host
 * (ReadJpeg, guetzli/jpeg_data_reader.cc:931); its coefficients and quant tables
 * seed the same device search.  4:4:4 YCbCr input only: 4:2:0 input needs the
 * YUV420 path and is refused, every other rejection is the reference's. */
int gb200_process_jpeg(const gb200_params* params, const uint8_t* jpeg_in, size_t jpeg_len, int device,
                       gb200_log_fn log, void* log_user, uint8_t** out, size_t* out_len,
                       gb200_stats* stats);
/* gb200_process_jpeg on a file held in memory of `device` (jpeg_len bytes at jpeg_dev), read once the work
 * queued on `stream` (a cudaStream_t; NULL for the legacy default stream) so far is done.  For the same bytes
 * it returns what gb200_process_jpeg returns: the result, the output (best-so-far bytes on failure), the
 * --verbose trace, the iteration counters and the refusals, in the same order.  The header is read from
 * prefixes copied to the host.  A sequential 4:4:4 YCbCr file the encoder takes (its first scan carries every
 * component, under 256 MiB) is Huffman-decoded, dequantised and checked for coefficients beyond 4096 on the
 * device; only its bytes after EOI and the one coefficient plane the host search keeps (384 bytes per 8x8
 * block) come back.  Every other file (progressive, gray, subsampled, CMYK, damaged) is copied back whole
 * and read as gb200_process_jpeg reads it.  The file may be overwritten once the call returns.  Host,
 * managed and other-device pointers are refused before anything runs ("... is not device memory of device
 * N"); a NULL jpeg_dev with jpeg_len 0 is refused as an unreadable file.  The stats cover the whole call,
 * header read and decode included.  The CPU port has no device memory and refuses every call. */
int gb200_process_jpeg_from_device(const gb200_params* params, const uint8_t* jpeg_dev, size_t jpeg_len,
                                   int device, gb200_log_fn log, void* log_user, uint8_t** out,
                                   size_t* out_len, gb200_stats* stats, void* stream);

/* butteraugli::ButteraugliInterface(rgb0, rgb1, diffmap, diffvalue)
 * (third_party/butteraugli/butteraugli/butteraugli.cc:1858; the stand-alone `butteraugli`
 * tool, butteraugli_main.cc:362): both images as planar linear RGB floats [3][h][w], nominally in
 * 0..255; diffmap (may be NULL) receives w*h floats, *score their maximum.  Values outside 0..255
 * (ringing below 0, highlights above 255) are scored as the reference scores them, bit for bit; this
 * is tested from -300 to 4500.  NaN and infinities must not be passed: the reference's result is
 * undefined for them.  The same holds for every butteraugli entry below. */
int gb200_butteraugli_diffmap(const float* rgb0, const float* rgb1, int w, int h, int device, float* diffmap,
                              double* score);

/* ---- butteraugli::ButteraugliComparator (third_party/butteraugli/butteraugli/butteraugli.h:425) ----
 * One original kept resident on one GPU (its PsychoImage, the neighbour sums of its mask) and scored
 * against any number of images.  Images are planar linear RGB floats [3][h][w], nominally in 0..255
 * (values outside it as for gb200_butteraugli_diffmap), the
 * original at least 8x8 (the reference class computes nothing below that; gb200_butteraugli_diffmap
 * pads small images).  One comparator is used by one thread at a time; separate comparators may run
 * concurrently, each has its own stream.  Every call returns once its outputs are written. */
typedef struct gb200_butteraugli_comparator gb200_butteraugli_comparator;
/* ButteraugliComparator::ButteraugliComparator(rgb0) (butteraugli.cc:784); rgb0 in host memory.
 * NULL on failure (gb200_last_error). */
gb200_butteraugli_comparator* gb200_butteraugli_comparator_create(const float* rgb0, int w, int h, int device);
/* ButteraugliComparator::Diffmap (butteraugli.cc:799) and ButteraugliScoreFromDiffmap (butteraugli.cc:1623):
 * rgb1 [3][h][w] in host memory; diffmap (may be NULL) receives [h][w], *score its maximum. */
int gb200_butteraugli_comparator_diffmap(gb200_butteraugli_comparator* c, const float* rgb1, float* diffmap,
                                         double* score);
/* The same with rgb1 [3][h][w] and diffmap [h][w] (may be NULL) in device memory of the comparator's
 * device.  stream (a cudaStream_t, NULL = the legacy default stream): the comparator waits for the work
 * queued on it so far, so rgb1 may still be in the making there.  rgb1 is copied into the comparator's
 * own buffer before it is read.  A host pointer or memory of another device is refused, nothing runs. */
int gb200_butteraugli_comparator_diffmap_device(gb200_butteraugli_comparator* c, const float* rgb1_dev,
                                                float* diffmap_dev, double* score, void* stream);
/* ButteraugliComparator::Mask (butteraugli.cc:793): mask and mask_dc, [3][h][w] each, host memory. */
int gb200_butteraugli_comparator_mask(gb200_butteraugli_comparator* c, float* mask, float* mask_dc);
/* The same into mask_dev and mask_dc_dev, device memory of the comparator's device, written after the work
 * queued on `stream` so far and written when the call returns.  A host pointer or memory of another device is
 * refused, nothing runs. */
int gb200_butteraugli_comparator_mask_device(gb200_butteraugli_comparator* c, float* mask_dev, float* mask_dc_dev,
                                             void* stream);
void gb200_butteraugli_comparator_destroy(gb200_butteraugli_comparator* c);
/* A comparator that scores up to `capacity` images per call against its original, all of them in one
 * pass of the Compare chain, one launch per stage; the original is analysed once, here (DESIGN.md §4).
 * w, h as in gb200_butteraugli_comparator_create; 1 <= capacity <= 16383.  Capacity 1 is the comparator
 * gb200_butteraugli_comparator_create makes.  The other comparator calls work on it unchanged.  NULL on
 * failure (gb200_last_error), with nothing left allocated. */
gb200_butteraugli_comparator* gb200_butteraugli_comparator_create_batch(const float* rgb0, int w, int h, int capacity,
                                                                        int device);
/* The same comparator made from an original rgb0_dev [3][h][w] in device memory of `device`, read after the
 * work queued on `stream` so far (a cudaStream_t, NULL = the legacy default stream) and copied on the device:
 * no pixel crosses PCIe.  The caller may free or overwrite rgb0_dev once this returns.  A host, managed or
 * other device's pointer is refused, nothing runs.  NULL on failure, with nothing left allocated; otherwise
 * the comparator is the one gb200_butteraugli_comparator_create_batch makes, bit for bit. */
gb200_butteraugli_comparator* gb200_butteraugli_comparator_create_device(const float* rgb0_dev, int w, int h,
                                                                         int capacity, int device, void* stream);
/* ButteraugliComparator::Diffmap (butteraugli.cc:799) and ButteraugliScoreFromDiffmap (butteraugli.cc:1623)
 * for each image: rgb1 [n][3][h][w] in host memory, 1 <= n <= capacity; diffmap (may be NULL) receives
 * [n][h][w], score (may be NULL) [n], the maximum of each diffmap.  Each image gets the bits that
 * gb200_butteraugli_comparator_diffmap gives for it.  The reference class has no batched call. */
int gb200_butteraugli_comparator_diffmap_batch(gb200_butteraugli_comparator* c, const float* rgb1, int n,
                                               float* diffmap, double* score);
/* The same with rgb1 and diffmap (may be NULL) in device memory of the comparator's device; stream as in
 * gb200_butteraugli_comparator_diffmap_device.  A host pointer or memory of another device is refused,
 * nothing runs. */
int gb200_butteraugli_comparator_diffmap_batch_device(gb200_butteraugli_comparator* c, const float* rgb1_dev, int n,
                                                      float* diffmap_dev, double* score, void* stream);
/* ---- batched butteraugli: N same-size pairs per call ----
 * Each pair (rgb0[i], rgb1[i]) gets butteraugli::ButteraugliInterface (butteraugli.cc:1858), bit for bit
 * what gb200_butteraugli_diffmap gives for it alone.  Up to `capacity` pairs of w x h images run through
 * the Compare chain together, one launch per stage, each pair in its own slot of device memory
 * (DESIGN.md §4).  Images are planar linear RGB floats, nominally in 0..255 (values outside it as for
 * gb200_butteraugli_diffmap), at least 8x8.  One batch object is
 * used by one thread at a time; separate objects may run concurrently, each has its own stream.  Every
 * call returns once its outputs are written. */
typedef struct gb200_butteraugli_batch gb200_butteraugli_batch;
/* w, h at least 8 and below 65536; 1 <= capacity <= 16383; NULL on failure (gb200_last_error), with
 * nothing left allocated */
gb200_butteraugli_batch* gb200_butteraugli_batch_create(int w, int h, int capacity, int device);
/* ButteraugliInterface per pair: rgb0, rgb1 [n][3][h][w] in host memory, 1 <= n <= capacity;
 * diffmap (may be NULL) receives [n][h][w], score (may be NULL) [n], the maximum of each diffmap. */
int gb200_butteraugli_batch_diffmap(gb200_butteraugli_batch* b, const float* rgb0, const float* rgb1, int n,
                                    float* diffmap, double* score);
/* The same with rgb0, rgb1 and diffmap (may be NULL) in device memory of the batch's device; stream as in
 * gb200_butteraugli_comparator_diffmap_device.  A host pointer or memory of another device is refused,
 * nothing runs. */
int gb200_butteraugli_batch_diffmap_device(gb200_butteraugli_batch* b, const float* rgb0_dev, const float* rgb1_dev,
                                           int n, float* diffmap_dev, double* score, void* stream);
/* ButteraugliInterface per pair, pairs of different sizes: pair i is w[i] x h[i], 8 <= w[i] <= the batch's w,
 * 8 <= h[i] <= its h; 1 <= n <= capacity.  w, h: host arrays [n].  rgb0[i], rgb1[i]: [3][h[i]][w[i]] in
 * host memory; diffmap (may be NULL; entries may not be) [i]: [h[i]][w[i]]; score (may be NULL) [n].
 * All pairs go through one pass of the Compare chain (several where the call has more than 16 distinct
 * sizes), and each is bit for bit gb200_butteraugli_diffmap of that pair alone. */
int gb200_butteraugli_batch_diffmap_sizes(gb200_butteraugli_batch* b, const int* w, const int* h,
                                          const float* const* rgb0, const float* const* rgb1, int n,
                                          float* const* diffmap, double* score);
/* The same with every image and diffmap in device memory of the batch's device; stream as in
 * gb200_butteraugli_batch_diffmap_device.  A host, managed or other device's pointer is refused, nothing
 * runs. */
int gb200_butteraugli_batch_diffmap_sizes_device(gb200_butteraugli_batch* b, const int* w, const int* h,
                                                 const float* const* rgb0_dev, const float* const* rgb1_dev, int n,
                                                 float* const* diffmap_dev, double* score, void* stream);
void gb200_butteraugli_batch_destroy(gb200_butteraugli_batch* b);

/* ---- 8-bit sRGB images, scored as the stand-alone `butteraugli` tool scores them ----
 * Images are interleaved uint8 [h][w][channels] (or [n][h][w][channels]), channels 3 (RGB) or 4 (RGBA),
 * both images of a pair with the same channels.  Each is converted on the device as the tool converts
 * it (FromSrgbToLinear, butteraugli_main.cc:239-281): sRGB bytes to linear 0..255 through the tool's
 * table, and with alpha laid over a background in sRGB space first, in integers:
 * (v a + bg (255 - a) + 127) / 255, alpha 255 keeping the pixel and 0 giving the background.  RGB is
 * scored once.  RGBA is scored over black and over white (butteraugli_main.cc:390-419): the larger score
 * and its diffmap are the result, black on a tie.  The float entries above then score the converted
 * planes, so each result is bit for bit theirs on those planes.  Other channel counts are refused.
 *
 * The tool's whole comparison of one pair in host memory, any size from 1x1 (padded below 8 pixels as
 * gb200_butteraugli_diffmap pads, each background cropped back before the two are compared, as the tool
 * compares them); diffmap (may be NULL) receives [h][w], *score its maximum. */
int gb200_butteraugli_diffmap_srgb(const uint8_t* img0, const uint8_t* img1, int w, int h, int channels, int device,
                                   float* diffmap, double* score);
/* gb200_butteraugli_batch_diffmap on 8-bit pairs: img0, img1 [n][h][w][channels] in host memory, uploaded
 * once whatever the channels. */
int gb200_butteraugli_batch_diffmap_srgb(gb200_butteraugli_batch* b, const uint8_t* img0, const uint8_t* img1, int n,
                                         int channels, float* diffmap, double* score);
/* The same with img0, img1 and diffmap (may be NULL) in device memory of the batch's device, read in
 * place; stream as in gb200_butteraugli_comparator_diffmap_device. */
int gb200_butteraugli_batch_diffmap_srgb_device(gb200_butteraugli_batch* b, const uint8_t* img0_dev,
                                                const uint8_t* img1_dev, int n, int channels, float* diffmap_dev,
                                                double* score, void* stream);
/* gb200_butteraugli_batch_diffmap_sizes on 8-bit pairs: pair i is w[i] x h[i] with channels[i] (3 or 4), 8 <=
 * w[i] <= the batch's w, 8 <= h[i] <= its h (gb200_butteraugli_diffmap_srgb scores smaller pairs); RGB and
 * RGBA pairs may share a call.  w, h, channels: host arrays [n].  img0[i], img1[i]: [h[i]][w[i]][channels[i]]
 * in host memory, packed and uploaded once as bytes whatever the channels.  diffmap (may be NULL, and so may
 * its entries) [i]: [h[i]][w[i]]; score (may be NULL) [n].  Each pair is bit for bit
 * gb200_butteraugli_diffmap_srgb of that pair alone.  The bytes are converted as the Compare chain packs them;
 * RGBA pairs are scored over black with the RGB pairs, then over white in passes of their own. */
int gb200_butteraugli_batch_diffmap_sizes_srgb(gb200_butteraugli_batch* b, const int* w, const int* h,
                                               const int* channels, const uint8_t* const* img0,
                                               const uint8_t* const* img1, int n, float* const* diffmap,
                                               double* score);
/* The same with every image and diffmap in device memory of the batch's device, read in place; stream as in
 * gb200_butteraugli_batch_diffmap_device.  A host, managed or other device's pointer is refused, nothing
 * runs. */
int gb200_butteraugli_batch_diffmap_sizes_srgb_device(gb200_butteraugli_batch* b, const int* w, const int* h,
                                                      const int* channels, const uint8_t* const* img0_dev,
                                                      const uint8_t* const* img1_dev, int n,
                                                      float* const* diffmap_dev, double* score, void* stream);
/* A comparator (gb200_butteraugli_comparator_create_batch) whose original img0 [h][w][channels] is given
 * in host memory, at least 8x8; 1 <= capacity <= 16383.  With channels 4 it keeps two resident
 * originals, over black and over white.  It takes 8-bit candidates with its own channels only (the
 * entries below); the float entries refuse it, and gb200_butteraugli_comparator_mask refuses an RGBA one. */
gb200_butteraugli_comparator* gb200_butteraugli_comparator_create_srgb(const uint8_t* img0, int w, int h, int channels,
                                                                       int capacity, int device);
/* The same from img0_dev [h][w][channels] in device memory of `device`, converted where it lies after the
 * work queued on `stream` so far, as gb200_butteraugli_comparator_create_device reads its original. */
gb200_butteraugli_comparator* gb200_butteraugli_comparator_create_srgb_device(const uint8_t* img0_dev, int w, int h,
                                                                              int channels, int capacity, int device,
                                                                              void* stream);
/* img1 [n][h][w][channels] in host memory, 1 <= n <= capacity; diffmap (may be NULL) [n][h][w], score
 * (may be NULL) [n].  A comparator made from float planes refuses it. */
int gb200_butteraugli_comparator_diffmap_srgb(gb200_butteraugli_comparator* c, const uint8_t* img1, int n,
                                              float* diffmap, double* score);
/* The same with img1 and diffmap (may be NULL) in device memory of the comparator's device, read in
 * place; stream as in gb200_butteraugli_comparator_diffmap_device. */
int gb200_butteraugli_comparator_diffmap_srgb_device(gb200_butteraugli_comparator* c, const uint8_t* img1_dev, int n,
                                                     float* diffmap_dev, double* score, void* stream);

/* ---- comparator sets: many resident originals of sizes of their own ----
 * A set holds `count` >= 1 originals, each at least 8x8 and below 65536 in each dimension, of sizes that may
 * differ.  Each is analysed once, when the set is made, and its analysis stays in device memory (40 bytes
 * per pixel; an RGBA original twice, over black and over white).  A call scores 1 <= n <= capacity
 * candidates: candidate i names its original by index, original[i] in 0..count-1, and has that original's
 * size (and channels).  Each candidate's diffmap and score are bit for bit what
 * gb200_butteraugli_batch_diffmap_sizes (float set) or gb200_butteraugli_batch_diffmap_sizes_srgb (8-bit
 * set) give for the pair (original, candidate), whatever else the call holds.  All candidates go through one
 * pass of the Compare chain (several where the call has more than 16 distinct sizes).  A set is used by one
 * thread at a time; separate sets may run concurrently.  Every call returns once its outputs are written. */
typedef struct gb200_butteraugli_comparator_set gb200_butteraugli_comparator_set;
/* w, h: host arrays [count]; rgb0[i]: planar linear RGB floats [3][h[i]][w[i]] in host memory;
 * 1 <= capacity <= 16383.  NULL on failure (gb200_last_error), with nothing left allocated. */
gb200_butteraugli_comparator_set* gb200_butteraugli_comparator_set_create(const int* w, const int* h,
                                                                          const float* const* rgb0, int count,
                                                                          int capacity, int device);
/* The same for 8-bit originals: img0[i] interleaved [h[i]][w[i]][channels[i]] in host memory, channels 3 (RGB)
 * or 4 (RGBA) per original, RGB and RGBA in one set.  It takes 8-bit candidates only. */
gb200_butteraugli_comparator_set* gb200_butteraugli_comparator_set_create_srgb(const int* w, const int* h,
                                                                               const int* channels,
                                                                               const uint8_t* const* img0, int count,
                                                                               int capacity, int device);
/* The same two with the originals in device memory of `device` (w, h and channels stay host arrays), read in
 * place by the packing launch after the work queued on `stream` so far (a cudaStream_t, NULL = the legacy
 * default stream), in the same mixed passes as from host memory.  The caller may free or overwrite them once
 * this returns.  A host, managed or other device's pointer is refused, naming it (rgb0[i] / img0[i]), and
 * nothing runs.  The set is the one the host entry makes, bit for bit. */
gb200_butteraugli_comparator_set* gb200_butteraugli_comparator_set_create_device(const int* w, const int* h,
                                                                                 const float* const* rgb0_dev,
                                                                                 int count, int capacity, int device,
                                                                                 void* stream);
gb200_butteraugli_comparator_set* gb200_butteraugli_comparator_set_create_srgb_device(
    const int* w, const int* h, const int* channels, const uint8_t* const* img0_dev, int count, int capacity,
    int device, void* stream);
/* original: host array [n]; rgb1[i]: [3][h][w] of original[i]'s size, in host memory; diffmap (may be NULL,
 * and so may its entries) [i]: [h][w]; score (may be NULL) [n].  A set made from 8-bit images refuses it. */
int gb200_butteraugli_comparator_set_diffmap(gb200_butteraugli_comparator_set* s, const int* original,
                                             const float* const* rgb1, int n, float* const* diffmap, double* score);
/* The same with every candidate and diffmap in device memory of the set's device, read in place; stream as in
 * gb200_butteraugli_batch_diffmap_device.  A host, managed or other device's pointer is refused, nothing
 * runs. */
int gb200_butteraugli_comparator_set_diffmap_device(gb200_butteraugli_comparator_set* s, const int* original,
                                                    const float* const* rgb1_dev, int n, float* const* diffmap_dev,
                                                    double* score, void* stream);
/* 8-bit candidates: img1[i] [h][w][channels] of original[i]'s size and channels, in host memory, uploaded
 * once as bytes; outputs as in gb200_butteraugli_comparator_set_diffmap.  A float set refuses it. */
int gb200_butteraugli_comparator_set_diffmap_srgb(gb200_butteraugli_comparator_set* s, const int* original,
                                                  const uint8_t* const* img1, int n, float* const* diffmap,
                                                  double* score);
/* The same with every candidate and diffmap in device memory of the set's device, read in place; stream and
 * refusals as in gb200_butteraugli_comparator_set_diffmap_device. */
int gb200_butteraugli_comparator_set_diffmap_srgb_device(gb200_butteraugli_comparator_set* s, const int* original,
                                                         const uint8_t* const* img1_dev, int n,
                                                         float* const* diffmap_dev, double* score, void* stream);
void gb200_butteraugli_comparator_set_destroy(gb200_butteraugli_comparator_set* s);

/* butteraugli::ButteraugliAdaptiveQuantization (butteraugli.cc:1880): the Y plane of Mask(rgb, rgb),
 * [h][w] into quant.  rgb in host memory.  Fails below 16x16, where the reference returns false. */
int gb200_butteraugli_adaptive_quantization(const float* rgb, int w, int h, int device, float* quant);
/* The same with rgb_dev [3][h][w] and quant_dev [h][w] in device memory of `device`, read and written after the
 * work queued on `stream` so far; quant_dev is written when the call returns.  A host, managed or other device's
 * pointer is refused, nothing runs. */
int gb200_butteraugli_adaptive_quantization_device(const float* rgb_dev, int w, int h, int device, float* quant_dev,
                                                   void* stream);

/* butteraugli::CreateHeatMapImage (butteraugli.cc:1979) of n maps of sizes of their own, on `device`, with one
 * launch for all of them: diffmap[i] [h[i]][w[i]] floats -> rgb[i] [h[i]][w[i]][3] bytes, the reference's
 * ScoreToRgb bytes exactly.  The butteraugli tool's thresholds are good = ButteraugliFuzzyInverse(1.5) and
 * bad = ButteraugliFuzzyInverse(0.5) (butteraugli_main.cc:423-424); any 0 < good < bad is taken, anything
 * else refused.  Maps are at least 1x1, at most 2^31 - 1 pixels in all.  Host memory here, uploaded in one
 * copy; the heat maps come back in one.  A NaN in a map has no defined colour.  Returns 1 on success. */
int gb200_butteraugli_heatmap(const int* w, const int* h, const float* const* diffmap, int n, double good, double bad,
                              uint8_t* const* rgb, int device);
/* The same with diffmap_dev[i] and rgb_dev[i] in device memory of `device` (w, h stay host arrays), read and
 * written after the work queued on `stream` so far, written when the call returns.  A host, managed or other
 * device's pointer is refused, nothing runs. */
int gb200_butteraugli_heatmap_device(const int* w, const int* h, const float* const* diffmap_dev, int n, double good,
                                     double bad, uint8_t* const* rgb_dev, int device, void* stream);

/* ReadJpeg(JPEG_READ_HEADER) as the CLI uses it (guetzli/guetzli.cc:306): frame size only. */
int gb200_jpeg_dimensions(const uint8_t* jpeg_in, size_t jpeg_len, int* width, int* height);

/* The pixels libjpeg-turbo gives for n JPEG files (jpeg_start_decompress with the defaults the butteraugli
 * tool's ReadJPEG keeps: JDCT_ISLOW, fancy upsampling, RGB output, gray replicated into R, G and B), decoded
 * on `device` in one pass for files of any sizes: out[i] receives file i as [h][w][3] bytes in host memory,
 * w x h as gb200_jpeg_dimensions gives them.  Accepted: baseline, extended and progressive Huffman files
 * that are gray or have 3 components sampled 4:4:4, 4:2:2 or 4:2:0.  Refused, with the file's index and the
 * reason in gb200_last_error() and nothing run: what ReadJpeg rejects, 4 components (CMYK, YCCK), other
 * samplings, progressive files that libjpeg would block-smooth (some low-frequency coefficient not
 * refined to its last bit), and files with coefficients so large that libjpeg-turbo's SIMD and C IDCTs
 * give different samples.  Returns 1 on success. */
int gb200_jpeg_decode_rgb(const uint8_t* const* jpeg, const size_t* len, int n, int device, uint8_t* const* out);
/* The same with out_dev[i] in device memory of `device`, written after the work queued on `stream` so far
 * (a cudaStream_t, NULL = the legacy default stream) and written when the call returns.  A host, managed
 * or other device's pointer is refused, nothing runs. */
int gb200_jpeg_decode_rgb_device(const uint8_t* const* jpeg, const size_t* len, int n, int device,
                                 uint8_t* const* out_dev, void* stream);

/* gb200_jpeg_dimensions for n files whose bytes are in device memory of `device`, read after the work queued
 * on `stream`: a prefix of each file is copied to the host (4 KiB, doubling until the frame header is in
 * it).  A file without a readable frame size gets 0 x 0.  Returns 1 on success. */
int gb200_jpeg_dimensions_from_device(const uint8_t* const* jpeg_dev, const size_t* len, int n, int device,
                                      void* stream, int* width, int* height);
/* gb200_jpeg_decode_rgb_device for n files whose bytes are in device memory of `device`: the same pixels,
 * into out_dev[i] of width[i] x height[i] x 3 bytes, which must be the frame's size.  Everything is read
 * after the work queued on `stream` so far, and the outputs are written when the call returns.  Each
 * file's header is parsed on the host from a copied prefix.  A sequential (SOF0 / SOF1) file under 256 MiB
 * whose first scan carries every component in one pass (Ss = 0, Se = 63, Ah = Al = 0) and whose scan data
 * ends in EOI, with RSTn in order, is Huffman-decoded on the device, up to 2^30 scan bytes per call; every
 * other file, one the device finds an error in, and one whose speculative decode has not converged
 * within its rounds, is copied back and read as gb200_jpeg_decode_rgb reads it.  A file of len 0 may have
 * a null pointer.  Refusals are those of
 * gb200_jpeg_decode_rgb, with the same reasons ("jpeg_decode_rgb_from_device: file i: <reason>"), plus a
 * width or height other than the frame's; host, managed and other devices' pointers are refused too.  No
 * output is written unless every file is accepted.  Returns 1 on success. */
int gb200_jpeg_decode_rgb_from_device(const uint8_t* const* jpeg_dev, const size_t* len, int n, int device,
                                      const int* width, const int* height, uint8_t* const* out_dev, void* stream);

/* test hook: ReadJpeg(JPEG_READ_ALL) alone.  dims = {w, h, ncomp, wb0, hb0, wb1, hb1, ...} (11 ints);
 * out receives the quantised coefficients of all components, concatenated. */
int gb200_debug_read_jpeg(const uint8_t* jpeg_in, size_t jpeg_len, int* dims, int16_t* out, size_t out_cap);
/* test hook: the device path's entropy decoding (segment pass, speculative Huffman decode with subsequences
 * of S bits, DC prefix sums) of one file in host memory, uploaded first (on the CPU port: run as host loops).
 * *status = 1 where the device path takes the file and finds no error, with the coefficients in out as
 * gb200_debug_read_jpeg gives them; 0 where the file goes to the host path, out untouched.  Returns 1 on
 * success. */
int gb200_debug_entropy_decode(const uint8_t* jpeg_in, size_t jpeg_len, int S, int16_t* out, size_t out_cap,
                               int* status);
/* test hook: the same decode, then gb200_jpeg_decode_rgb_from_device's SIMD-range test, with the reason for the
 * path a file takes.  *taken = 1 where the device path's shape takes the file; *flags = the OR of its status
 * word's flags (1 scan data not ending in EOI or RSTn missing / out of order, 2 an error read_jpeg raises
 * as well, 4 the SIMD-range test, 8 no convergence within the synchronisation rounds); *rounds = the
 * synchronisation rounds after the first.  out receives the coefficients as gb200_debug_read_jpeg gives them
 * where the file is taken and flags is 0 or 4; else it is untouched.  Returns 1 on success. */
int gb200_debug_entropy_decode_flags(const uint8_t* jpeg_in, size_t jpeg_len, int S, int16_t* out, size_t out_cap,
                                     int* taken, unsigned* flags, int* rounds);
/* test hook: the seeding of gb200_process_jpeg_from_device's device route (entropy decode with subsequences
 * of S bits, then JpegDequantSanity) on one file in host memory, uploaded first (on the CPU port: run as host
 * loops).  *status = 1 where the route takes the file and it passes the sanity check, 2 where the route takes
 * it and a coefficient times its quant step exceeds 4096 in magnitude, 0 where the file goes to the host
 * route.  Where it is taken, dq receives [3][blocks][64] coefficients times their quant steps (natural order,
 * stored as int16). Returns 1 on success. */
int gb200_debug_jpeg_seed(const uint8_t* jpeg_in, size_t jpeg_len, int S, int16_t* dq, size_t dq_cap,
                          int* status);

/* ---- one image tiled over the GPUs of a node (BASELINE configs[3]) ------------
 * One process per GPU.  Rank 0 obtains an id, the host application distributes it
 * (e.g. torch.distributed broadcast), every rank calls gb200_dist_init once, then
 * gb200_process_rgb_tiled collectively with the SAME image and parameters; every
 * rank receives the same JPEG.  Rank r runs the image-plane kernels for its strip of
 * block rows (+56-row halo, the metric's receptive field); the per-block results
 * cross NVLink through NCCL (in-place all-gather).  Same bytes as gb200_process_rgb. */
int gb200_dist_unique_id(uint8_t* out128);
int gb200_dist_init(const uint8_t* id128, int rank, int world, int device);
void gb200_dist_shutdown(void);
int gb200_process_rgb_tiled(const gb200_params* params, const uint8_t* rgb, int w, int h, gb200_log_fn log,
                            void* log_user, uint8_t** out, size_t* out_len, gb200_stats* stats);
/* test entry: the same decomposition with `world` host threads sharing one device */
int gb200_process_rgb_tiled_threads(const gb200_params* params, const uint8_t* rgb, int w, int h, int device,
                                    int world, uint8_t** out, size_t* out_len, gb200_stats* stats);

void gb200_free(void* p);
const char* gb200_last_error(void);
const char* gb200_backend_name(void); /* "cuda-sm_90a" for the product library */
int gb200_device_count(void);

/* ---- device-resident stages (Comparator seam on device memory) ---------- */
typedef struct gb200_image gb200_image;

/* Upload + one-time kernels: RGB->YCbCr->FDCT (guetzli/jpeg_data_encoder.cc:66),
 * PsychoImage of the original (butteraugli.cc:784), block masks
 * (guetzli/butteraugli_comparator.cc:415). */
gb200_image* gb200_image_create(const uint8_t* rgb, int w, int h, int device);
/* prepare=0: upload only; the one-time kernels then run inside gb200_image_process */
gb200_image* gb200_image_create2(const uint8_t* rgb, int w, int h, int device, int prepare);
/* A resident image from an 8-bit view (channels, strides and conversion as in gb200_process_image), img
 * in host memory.  The image has been read and converted when the call returns, whatever `prepare`. */
gb200_image* gb200_image_create_strided(const uint8_t* img, int w, int h, int channels, const int64_t* strides,
                                        int device, int prepare);
/* The same with img in device memory of `device`, read in place after the work queued on `stream` (as in
 * gb200_process_image_device); the caller may overwrite or free it once the call returns. */
gb200_image* gb200_image_create_device(const uint8_t* img_dev, int w, int h, int channels, const int64_t* strides,
                                       int device, int prepare, void* stream);
/* test hook: the resident image's RGB as the encoder sees it, [h][w][3] into out */
int gb200_image_rgb(gb200_image* img, uint8_t* out);
void gb200_image_destroy(gb200_image* img);
/* guetzli::Process on an image that is already resident in HBM (same result as
 * gb200_process_rgb; used to time the job without the host->device upload) */
int gb200_image_process(gb200_image* img, const gb200_params* params, gb200_log_fn log, void* log_user,
                        uint8_t** out, size_t* out_len, gb200_stats* stats);
/* forgets the one-time results (FDCT, PsychoImage, masks) of a resident image: the next
 * gb200_image_process recomputes them from the resident pixels, i.e. repeats the whole job */
int gb200_image_reset(gb200_image* img);
int gb200_image_num_blocks(const gb200_image* img);
/* coefficients: int16 [3][num_blocks][64], block-major (JPEGComponent::coeffs) */
int gb200_image_orig_coeffs(gb200_image* img, int16_t* out);
/* OutputImage::ApplyGlobalQuantization (guetzli/output_image.cc:342); q: int[3][64] */
int gb200_image_apply_global_quant(gb200_image* img, const int* q);
int gb200_image_upload_candidate(gb200_image* img, const int16_t* coeffs);
int gb200_image_download_candidate(gb200_image* img, int16_t* coeffs);
/* sparse SetCoeffBlock edits: flat indices into [3][num_blocks][64] */
int gb200_image_scatter(gb200_image* img, const int* index, const int16_t* value, int n);
/* OutputImage::SaveToJpegData + WriteJpeg of the current candidate (guetzli/output_image.cc:348,
 * guetzli/jpeg_data_writer.cc:540): symbol counts, entropy coding, 0xFF stuffing and file assembly on the
 * device.  q[3][64]: the quant tables the candidate's coefficients are multiples of.  *out: gb200_free. */
int gb200_image_save_jpeg(gb200_image* img, const int* q, uint8_t** out, size_t* out_len);
/* ButteraugliComparator::Compare (guetzli/butteraugli_comparator.cc:63) */
int gb200_image_compare(gb200_image* img, float* distance);
int gb200_image_distmap(gb200_image* img, float* out /* [h][w] */);
/* ComputeBlockErrorAdjustmentWeights (guetzli/butteraugli_comparator.cc:494) */
int gb200_image_block_weights(gb200_image* img, int direction, int radius, double target_distance,
                              int zero_distmap, float* out /* [num_blocks] */);
/* ComputeBlockZeroingOrder for every block (guetzli/processor.cc:364);
 * idx/err: [num_blocks][192] slots, count[num_blocks] valid entries */
int gb200_image_zeroing_orders(gb200_image* img, float block_error_limit, int lookahead, uint8_t* idx,
                               float* err, int* count);
/* single stages on caller planes, packed float [n][h][w] (tests) */
int gb200_image_debug_blur(gb200_image* img, const float* in, float* out, int blur_id);
int gb200_image_debug_opsin(gb200_image* img, const float* rgb_linear, float* xyb);
int gb200_image_debug_separate(gb200_image* img, const float* xyb, float* psycho10);
int gb200_image_debug_render(gb200_image* img, float* linear_rgb);
int gb200_image_debug_psycho0(gb200_image* img, float* psycho10);
int gb200_image_debug_corner_mask(gb200_image* img, float* out /* [num_blocks][3] */);

/* SaveToJpegData + WriteJpeg (guetzli/output_image.cc:348, jpeg_data_writer.cc:540) of
 * dequantised coefficients that are multiples of q (host-side serialiser). */
int gb200_write_jpeg(const int16_t* coeffs, int w, int h, const int* q, uint8_t** out, size_t* out_len);

/* test hooks: prefix-exact replay of std::sort on (block, key) pairs vs std::sort itself */
size_t gb200_debug_partial_sort(int* block, float* key, size_t n, size_t want);
void gb200_debug_std_sort(int* block, float* key, size_t n);
/* test hook: length-limited Huffman code lengths of a symbol histogram (host side of the size pass and of
 * the walk; CreateHuffmanTree, guetzli/entropy_encode.cc:73).  depth[n] must be zeroed by the caller. */
void gb200_debug_huffman_depths(const uint32_t* counts, int n, int limit, uint8_t* depth);
/* experimental: the replay with the large partition passes on the device */
size_t gb200_debug_device_partial_sort(gb200_image* img, int* block, float* key, size_t n, size_t want);

/* The library keeps freed device blocks in a size-bucketed cache (cudaMalloc/cudaFree
 * would serialise concurrent image contexts); this returns the cache to the driver. */
void gb200_trim_memory(void);

/* process-wide running totals: kernels launched, bytes copied host->device and
 * device->host by this library (all threads, all contexts) */
void gb200_counters(long* launches, long long* h2d_bytes, long long* d2h_bytes);

/* per-kernel CUDA-event timing of everything launched by this library */
void gb200_profile_enable(int on);
void gb200_profile_reset(void);
/* fills up to cap entries; returns the number of distinct kernels */
int gb200_profile_get(char (*names)[48], long* launches, double* ms, double* elements, int cap);

#ifdef __cplusplus
}
#endif
#endif /* GUETZLI_B200_H_ */
