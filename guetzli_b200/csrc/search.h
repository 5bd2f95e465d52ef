// Host search driver: the control flow of guetzli::Process(RGB)
// (g/processor.cc:926) -- global quant-matrix bisection (a5/a6) and the
// per-block frequency masking iterations (a12, a16) -- over device-resident
// image state (pipeline.h).  g/ = /root/reference/guetzli/.
#pragma once
#include <stdint.h>

#include <string>

#include "backend.h"

namespace gb200 {

struct ImageView;

// Mirrors guetzli::Params (g/processor.h:29-37).
struct SearchParams {
  float butteraugli_target = 1.0f;
  bool clear_metadata = true;
  bool try_420 = false;
  bool force_420 = false;
  bool use_silver_screen = false;
  int zeroing_greedy_lookahead = 3;
  bool new_zeroing_model = true;
};

typedef void (*LogSink)(void* user, const char* text);

struct SearchStats {
  int iterations = 0;       // "number of iterations"
  int iterations_up = 0;    // "number of iterations up"
  int iterations_down = 0;  // "number of iterations down"
  // device-side accounting of this call
  long gpu_launches = 0;
  double ms_total = 0, ms_device_setup = 0, ms_compare = 0, ms_zeroing = 0, ms_jpeg = 0, ms_sort = 0,
         ms_walk = 0;
  int compares = 0;
  long long h2d_bytes = 0, d2h_bytes = 0;
  int order_partial = 0, order_exact = 0;
};

class ImageContext;
// Same job on an image that is already resident on the device (upload done by
// the ImageContext constructor with prepare_now=false).
bool process_resident(const SearchParams& params, ImageContext* ctx, LogSink log, void* log_user,
                      std::string* jpeg_out, SearchStats* stats, std::string* err);

class Comm;
// Row-strip mode: a collective call, every rank passes the same image and
// parameters and receives the same JPEG; rank r computes the image-plane kernels of
// block rows strip_of(r) (comm.h).  The scalar search runs redundantly on every rank.
bool process_rgb_tiled(const SearchParams& params, const uint8_t* rgb, int w, int h, int device, Comm* comm,
                       LogSink log, void* log_user, std::string* jpeg_out, SearchStats* stats, std::string* err);

// Returns true on success; *jpeg_out receives the best JPEG found (possibly
// empty on failure), error text goes to err (and stderr, like the reference).
// Process(jpeg bytes) (g/processor.cc:890): 4:4:4 YCbCr JPEG input; the search starts
// from the file's own coefficients and quant tables.
bool process_jpeg(const SearchParams& params, const uint8_t* data, size_t len, int device, LogSink log,
                  void* log_user, std::string* jpeg_out, SearchStats* stats, std::string* err);

bool process_rgb(const SearchParams& params, const uint8_t* rgb, int w, int h, int device, LogSink log,
                 void* log_user, std::string* jpeg_out, SearchStats* stats, std::string* err);

// Process(RGB) on an 8-bit image of 1 (gray), 2 (gray + alpha), 3 (RGB) or 4 (RGBA) channels, turned into
// RGB on the device as the guetzli tool turns PNG layouts into RGB (g/guetzli.cc:43-145; ImageContext's
// ImageView source).  strides: bytes per row, pixel and channel, or null for contiguous [h][w][channels].
// process_image reads img from host memory; process_image_device reads it in place from memory of `device`
// once the work queued on `stream` so far is done.  The checks and messages of process_rgb, plus refusals
// of channels outside 1..4 and of negative strides; then the RGB path.
bool process_image(const SearchParams& params, const uint8_t* img, int w, int h, int channels, const int64_t* strides,
                   int device, LogSink log, void* log_user, std::string* jpeg_out, SearchStats* stats,
                   std::string* err);
bool process_image_device(const SearchParams& params, const uint8_t* img, int w, int h, int channels,
                          const int64_t* strides, int device, Stream stream, LogSink log, void* log_user,
                          std::string* jpeg_out, SearchStats* stats, std::string* err);
// The view of such an image (on the host; the caller sets device and stream), or false + message when
// channels is outside 1..4 or a stride is negative.
bool image_view(const uint8_t* img, int w, int channels, const int64_t* strides, ImageView* view, std::string* err);

// a11 as a call of its own (SaveToJpegData + WriteJpeg, g/output_image.cc:348, g/jpeg_data_writer.cc:540):
// the JPEG file of the context's current candidate, whose coefficients are multiples of q[3][64];
// symbol counts, entropy coding, byte stuffing and file assembly on the device.  Throws on error.
void device_save_jpeg(ImageContext* ctx, const int q[192], std::string* out);

// false + message when the image needs more than the 32-bit indices of the device lists
bool image_size_supported(int w, int h, std::string* err);

// ScoreJPEG (g/score.cc:23).
double score_jpeg(double distance, int size, double target);

}  // namespace gb200
