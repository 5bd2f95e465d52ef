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

/* guetzli::Process(params, stats, jpeg_in, &out) (guetzli/processor.h:39-41,
 * guetzli/processor.cc:890): JPEG input.  The file is parsed on the host
 * (ReadJpeg, guetzli/jpeg_data_reader.cc:931); its coefficients and quant tables
 * seed the same device search.  4:4:4 YCbCr input only: 4:2:0 input needs the
 * YUV420 path and is refused, every other rejection is the reference's. */
int gb200_process_jpeg(const gb200_params* params, const uint8_t* jpeg_in, size_t jpeg_len, int device,
                       gb200_log_fn log, void* log_user, uint8_t** out, size_t* out_len,
                       gb200_stats* stats);

/* butteraugli::ButteraugliInterface(rgb0, rgb1, diffmap, diffvalue)
 * (third_party/butteraugli/butteraugli/butteraugli.cc:1858; the stand-alone `butteraugli`
 * tool, butteraugli_main.cc:362): both images as planar linear RGB floats [3][h][w] in
 * 0..255; diffmap (may be NULL) receives w*h floats, *score their maximum. */
int gb200_butteraugli_diffmap(const float* rgb0, const float* rgb1, int w, int h, int device, float* diffmap,
                              double* score);

/* ReadJpeg(JPEG_READ_HEADER) as the CLI uses it (guetzli/guetzli.cc:306): frame size only. */
int gb200_jpeg_dimensions(const uint8_t* jpeg_in, size_t jpeg_len, int* width, int* height);

/* test hook: ReadJpeg(JPEG_READ_ALL) alone.  dims = {w, h, ncomp, wb0, hb0, wb1, hb1, ...} (11 ints);
 * out receives the quantised coefficients of all components, concatenated. */
int gb200_debug_read_jpeg(const uint8_t* jpeg_in, size_t jpeg_len, int* dims, int16_t* out, size_t out_cap);

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
