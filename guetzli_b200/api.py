"""ctypes host mirror of the reference interface for the hot path.

Names and argument meaning follow guetzli/processor.h: ``Params``,
``ProcessStats``, ``Process(params, stats, rgb, w, h, &out)``.  All compute goes
through the C ABI of ``libguetzli_b200.so`` (include/guetzli_b200.h), which is
CUDA-only: importing works anywhere, but calling fails loudly without the built
extension or without a GPU -- there is no CPU fallback in the product.
"""
import ctypes as C
import math
import os
from dataclasses import dataclass, field

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DEFAULT_LIB = os.path.join(_HERE, "libguetzli_b200.so")


class _CParams(C.Structure):
    _fields_ = [("butteraugli_target", C.c_float), ("clear_metadata", C.c_int),
                ("try_420", C.c_int), ("force_420", C.c_int), ("use_silver_screen", C.c_int),
                ("zeroing_greedy_lookahead", C.c_int), ("new_zeroing_model", C.c_int)]


class _CStats(C.Structure):
    _fields_ = [("iterations", C.c_int), ("iterations_up", C.c_int), ("iterations_down", C.c_int),
                ("compares", C.c_int), ("gpu_launches", C.c_long),
                ("h2d_bytes", C.c_longlong), ("d2h_bytes", C.c_longlong),
                ("ms_total", C.c_double), ("ms_device_setup", C.c_double), ("ms_compare", C.c_double),
                ("ms_zeroing", C.c_double), ("ms_jpeg", C.c_double), ("ms_sort", C.c_double),
                ("ms_walk", C.c_double), ("order_partial", C.c_int), ("order_exact", C.c_int)]


_LOG_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_char_p)

_libs = {}


def library_path():
    return os.environ.get("GUETZLI_B200_LIB", _DEFAULT_LIB)


def load_library(path=None):
    """Loads the C-ABI library (default: the in-tree CUDA build)."""
    path = os.path.abspath(path or library_path())
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise RuntimeError(
            f"guetzli_b200: {path} is missing. Build it with __graft_entry__.build() "
            "(nvcc, sm_90a); there is no CPU fallback.")
    lib = C.CDLL(path)
    P = C.POINTER
    lib.gb200_butteraugli_score_for_quality.restype = C.c_double
    lib.gb200_butteraugli_score_for_quality.argtypes = [C.c_double]
    lib.gb200_last_error.restype = C.c_char_p
    lib.gb200_backend_name.restype = C.c_char_p
    lib.gb200_process_rgb.argtypes = [P(_CParams), C.c_void_p, C.c_int, C.c_int, C.c_int, _LOG_FN,
                                      C.c_void_p, P(P(C.c_uint8)), P(C.c_size_t), P(_CStats)]
    lib.gb200_process_jpeg.argtypes = [P(_CParams), C.c_void_p, C.c_size_t, C.c_int, _LOG_FN,
                                       C.c_void_p, P(P(C.c_uint8)), P(C.c_size_t), P(_CStats)]
    lib.gb200_process_jpeg_from_device.argtypes = lib.gb200_process_jpeg.argtypes + [C.c_void_p]
    process_image = [P(_CParams), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, _LOG_FN, C.c_void_p,
                     P(P(C.c_uint8)), P(C.c_size_t), P(_CStats)]
    lib.gb200_process_image.argtypes = process_image
    lib.gb200_process_image_device.argtypes = process_image + [C.c_void_p]
    lib.gb200_image_create_strided.restype = C.c_void_p
    lib.gb200_image_create_strided.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    lib.gb200_image_create_device.restype = C.c_void_p
    lib.gb200_image_create_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                              C.c_void_p]
    lib.gb200_image_rgb.argtypes = [C.c_void_p, C.c_void_p]
    lib.gb200_free.argtypes = [C.c_void_p]
    lib.gb200_process_rgb_tiled_threads.argtypes = [P(_CParams), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                                    P(P(C.c_uint8)), P(C.c_size_t), P(_CStats)]
    lib.gb200_process_rgb_tiled.argtypes = [P(_CParams), C.c_void_p, C.c_int, C.c_int, _LOG_FN, C.c_void_p,
                                            P(P(C.c_uint8)), P(C.c_size_t), P(_CStats)]
    lib.gb200_dist_unique_id.argtypes = [C.c_void_p]
    lib.gb200_dist_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.gb200_image_create.restype = C.c_void_p
    lib.gb200_image_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.gb200_image_create2.restype = C.c_void_p
    lib.gb200_image_create2.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.gb200_image_process.argtypes = [C.c_void_p, P(_CParams), _LOG_FN, C.c_void_p,
                                        P(P(C.c_uint8)), P(C.c_size_t), P(_CStats)]
    lib.gb200_image_destroy.argtypes = [C.c_void_p]
    lib.gb200_image_reset.argtypes = [C.c_void_p]
    for name in ("num_blocks", "orig_coeffs", "apply_global_quant", "upload_candidate",
                 "download_candidate", "compare", "distmap", "debug_render", "debug_psycho0",
                 "debug_corner_mask"):
        getattr(lib, "gb200_image_" + name).argtypes = [C.c_void_p] + (
            [] if name == "num_blocks" else [C.c_void_p])
    lib.gb200_image_scatter.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.gb200_image_save_jpeg.argtypes = [C.c_void_p, C.c_void_p, P(P(C.c_uint8)), P(C.c_size_t)]
    lib.gb200_image_block_weights.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_int, C.c_void_p]
    lib.gb200_image_zeroing_orders.argtypes = [C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gb200_image_debug_blur.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.gb200_image_debug_opsin.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gb200_image_debug_separate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gb200_write_jpeg.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, P(P(C.c_uint8)), P(C.c_size_t)]
    lib.gb200_counters.argtypes = [P(C.c_long), P(C.c_longlong), P(C.c_longlong)]
    lib.gb200_profile_enable.argtypes = [C.c_int]
    lib.gb200_profile_get.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.gb200_debug_read_jpeg.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t]
    lib.gb200_jpeg_dimensions.argtypes = [C.c_void_p, C.c_size_t, P(C.c_int), P(C.c_int)]
    lib.gb200_jpeg_decode_rgb.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.gb200_jpeg_decode_rgb_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.gb200_jpeg_dimensions_from_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                                      C.c_void_p, C.c_void_p]
    lib.gb200_jpeg_decode_rgb_from_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                                      C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gb200_debug_entropy_decode.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t,
                                               P(C.c_int)]
    lib.gb200_debug_jpeg_seed.argtypes = lib.gb200_debug_entropy_decode.argtypes
    lib.gb200_debug_entropy_decode_flags.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t,
                                                     P(C.c_int), P(C.c_uint), P(C.c_int)]
    lib.gb200_butteraugli_diffmap.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                              P(C.c_double)]
    lib.gb200_butteraugli_comparator_create.restype = C.c_void_p
    lib.gb200_butteraugli_comparator_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.gb200_butteraugli_comparator_diffmap.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, P(C.c_double)]
    lib.gb200_butteraugli_comparator_diffmap_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, P(C.c_double),
                                                                C.c_void_p]
    lib.gb200_butteraugli_comparator_mask.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gb200_butteraugli_comparator_destroy.argtypes = [C.c_void_p]
    lib.gb200_butteraugli_comparator_create_batch.restype = C.c_void_p
    lib.gb200_butteraugli_comparator_create_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.gb200_butteraugli_comparator_diffmap_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                               C.c_void_p]
    lib.gb200_butteraugli_comparator_diffmap_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                                      C.c_void_p, C.c_void_p]
    lib.gb200_butteraugli_adaptive_quantization.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.gb200_butteraugli_batch_create.restype = C.c_void_p
    lib.gb200_butteraugli_batch_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    lib.gb200_butteraugli_batch_diffmap.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                    C.c_void_p]
    lib.gb200_butteraugli_batch_diffmap_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                           C.c_void_p, C.c_void_p]
    lib.gb200_butteraugli_batch_diffmap_sizes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                          C.c_int, C.c_void_p, C.c_void_p]
    lib.gb200_butteraugli_batch_diffmap_sizes_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                                 C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                                                 C.c_void_p]
    lib.gb200_butteraugli_batch_destroy.argtypes = [C.c_void_p]
    lib.gb200_butteraugli_diffmap_srgb.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                                   C.c_void_p, P(C.c_double)]
    lib.gb200_butteraugli_batch_diffmap_srgb.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                         C.c_void_p, C.c_void_p]
    lib.gb200_butteraugli_batch_diffmap_srgb_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                                C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gb200_butteraugli_batch_diffmap_sizes_srgb.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                               C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                               C.c_void_p]
    lib.gb200_butteraugli_batch_diffmap_sizes_srgb_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p,
                                                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                                      C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gb200_butteraugli_comparator_create_srgb.restype = C.c_void_p
    lib.gb200_butteraugli_comparator_create_srgb.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.gb200_butteraugli_comparator_diffmap_srgb.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                              C.c_void_p]
    lib.gb200_butteraugli_comparator_diffmap_srgb_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                                     C.c_void_p, C.c_void_p]
    lib.gb200_butteraugli_comparator_set_create.restype = C.c_void_p
    lib.gb200_butteraugli_comparator_set_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                            C.c_int]
    lib.gb200_butteraugli_comparator_set_create_srgb.restype = C.c_void_p
    lib.gb200_butteraugli_comparator_set_create_srgb.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                                 C.c_int, C.c_int, C.c_int]
    for name in ("", "_srgb"):
        set_diffmap = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        entry = "gb200_butteraugli_comparator_set_diffmap" + name
        getattr(lib, entry).argtypes = set_diffmap
        getattr(lib, entry + "_device").argtypes = set_diffmap + [C.c_void_p]
    lib.gb200_butteraugli_comparator_set_destroy.argtypes = [C.c_void_p]
    lib.gb200_butteraugli_comparator_create_device.restype = C.c_void_p
    lib.gb200_butteraugli_comparator_create_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                                               C.c_void_p]
    lib.gb200_butteraugli_comparator_create_srgb_device.restype = C.c_void_p
    lib.gb200_butteraugli_comparator_create_srgb_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                                                    C.c_int, C.c_void_p]
    lib.gb200_butteraugli_comparator_set_create_device.restype = C.c_void_p
    lib.gb200_butteraugli_comparator_set_create_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                                   C.c_int, C.c_int, C.c_void_p]
    lib.gb200_butteraugli_comparator_set_create_srgb_device.restype = C.c_void_p
    lib.gb200_butteraugli_comparator_set_create_srgb_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p,
                                                                        C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                                        C.c_void_p]
    lib.gb200_butteraugli_comparator_mask_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gb200_butteraugli_adaptive_quantization_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                                   C.c_void_p, C.c_void_p]
    heatmap = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_int]
    lib.gb200_butteraugli_heatmap.argtypes = heatmap
    lib.gb200_butteraugli_heatmap_device.argtypes = heatmap + [C.c_void_p]
    _libs[path] = lib
    return lib


def _err(lib):
    return (lib.gb200_last_error() or b"").decode(errors="replace")


def _raise_device_error(lib):
    """A failed encode without output: the device's failures raise, the reference's own (bad input,
    no JPEG found) are returned as (False, b"") as guetzli::Process returns them."""
    msg = _err(lib)
    if "CUDA" in msg or "no CUDA device" in msg or "out of memory" in msg:
        raise RuntimeError(msg)


def _cparams(params):
    return _CParams(params.butteraugli_target, int(params.clear_metadata), int(params.try_420),
                    int(params.force_420), int(params.use_silver_screen),
                    int(params.zeroing_greedy_lookahead), int(params.new_zeroing_model))


def _take(lib, out, out_len):
    data = C.string_at(out, out_len.value) if out_len.value else b""
    if out:
        lib.gb200_free(out)
    return data


def _log_sink(stats):
    """The C log callback feeding stats.debug_output and stats.debug_output_file; null when neither is set."""
    if stats is None or (stats.debug_output is None and stats.debug_output_file is None):
        return C.cast(None, _LOG_FN)

    def _sink(_user, text):
        s = text.decode(errors="replace")
        if stats.debug_output is not None:
            stats.debug_output.append(s)
        if stats.debug_output_file is not None:
            stats.debug_output_file.write(s)

    return _LOG_FN(_sink)


def _fill_stats(stats, cs, directions=True):
    """The counters of an encode into stats (if not None); directions: the up and down iterations as well."""
    if stats is None:
        return
    stats.counters["number of iterations"] = cs.iterations
    if directions:
        stats.counters["number of iterations up"] = cs.iterations_up
        stats.counters["number of iterations down"] = cs.iterations_down
    stats.device = {k: getattr(cs, k) for k, _ in _CStats._fields_}


@dataclass
class Params:
    """guetzli::Params (guetzli/processor.h:29-37)."""
    butteraugli_target: float = 1.0
    clear_metadata: bool = True
    try_420: bool = False
    force_420: bool = False
    use_silver_screen: bool = False
    zeroing_greedy_lookahead: int = 3
    new_zeroing_model: bool = True


@dataclass
class ProcessStats:
    """guetzli::ProcessStats (guetzli/stats.h:33-40): counters + optional debug sink."""
    counters: dict = field(default_factory=dict)
    debug_output: list = None      # set to [] to collect the --verbose trace
    debug_output_file: object = None  # file-like; trace is also written here
    device: dict = field(default_factory=dict)  # device-side accounting of the call


def butteraugli_score_for_quality(quality, lib=None):
    """guetzli::ButteraugliScoreForQuality (quality.cc:78) narrowed to float like
    the CLI does (guetzli.cc:273-275)."""
    lib = lib or load_library()
    return float(np.float32(lib.gb200_butteraugli_score_for_quality(float(quality))))


def process(params, stats, rgb, w, h, device=0, lib=None):
    """guetzli::Process(params, stats, rgb, w, h, &out) (processor.cc:926).

    rgb: bytes / uint8 array of 3*w*h interleaved sRGB samples (host memory).
    Returns (ok, jpeg_bytes); like the reference, jpeg_bytes holds the best JPEG
    found so far even when ok is False (possibly empty)."""
    lib = lib or load_library()
    buf = np.ascontiguousarray(np.frombuffer(rgb, dtype=np.uint8) if isinstance(rgb, (bytes, bytearray))
                               else np.asarray(rgb, dtype=np.uint8)).reshape(-1)
    if buf.size != 3 * w * h:
        import sys
        sys.stderr.write("Could not create jpg data from rgb pixels\n")
        return False, b""
    cp, cs = _cparams(params), _CStats()
    cb = _log_sink(stats)
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    ok = lib.gb200_process_rgb(C.byref(cp), buf.ctypes.data, w, h, device, cb, None,
                               C.byref(out), C.byref(out_len), C.byref(cs))
    data = _take(lib, out, out_len)
    _fill_stats(stats, cs)
    if not ok and not data:
        _raise_device_error(lib)
    return bool(ok), data


def _image_view(image):
    """Checks the 8-bit image of process_image and DeviceImage.from_image: a uint8 numpy array or torch tensor
    (host or CUDA) of shape [h][w] (gray) or [h][w][C] with C = 1 (gray), 2 (gray + alpha), 3 (RGB) or 4 (RGBA),
    taken as it is laid out, strides and storage offset included -> (pointer, w, h, C, strides int64[3] in
    bytes, the torch device of a CUDA tensor or None, the object that owns the memory)."""
    if _is_torch_tensor(image):
        import torch
        if image.dtype != torch.uint8:
            raise ValueError(f"image must be uint8, got {image.dtype}")
        shape, strides, ptr = tuple(image.shape), tuple(image.stride()), image.data_ptr()
        dev = image.device if image.is_cuda else None
    else:
        image = np.asarray(image)
        if image.dtype != np.uint8:
            raise ValueError(f"image must be uint8, got {image.dtype}")
        shape, strides, ptr, dev = image.shape, image.strides, image.ctypes.data, None
    if len(shape) not in (2, 3):
        raise ValueError(f"image must have 2 or 3 axes ([h][w] or [h][w][C]), got shape {shape}")
    if len(shape) == 2:
        shape, strides = shape + (1,), strides + (0,)
    if shape[2] not in (1, 2, 3, 4):
        raise ValueError("image must have 1 (gray), 2 (gray + alpha), 3 (RGB) or 4 (RGBA) channels in its last "
                         f"axis, got shape {shape}")
    if min(strides) < 0:
        raise ValueError(f"image must have non-negative strides, got {strides}")
    h, w, ch = shape
    return ptr, w, h, ch, np.array(strides, dtype=np.int64), dev, image


def process_image(params, stats, image, device=0, lib=None):
    """guetzli::Process on an 8-bit image of any channel count, converted to RGB as the guetzli tool converts
    PNG layouts (guetzli.cc:43-145): gray replicated, gray + alpha and RGBA blended on black with
    (v * a + 128) // 255, RGB as it is.  Returns (ok, jpeg_bytes) like process().

    image: uint8 [h][w] or [h][w][C], C = 1..4, a numpy array or a torch tensor, read with its strides and
    storage offset as they are (no contiguous copy).  Host memory is uploaded (the span the view covers) and
    encoded on `device`; a CUDA tensor is read in place on its own device, after the work queued on that
    device's current torch stream, and nothing of it crosses to the host.  Malformed images raise ValueError;
    the encoder's own refusals return (False, b"") as process() does, with the message in last_error()."""
    lib = lib or load_library()
    ptr, w, h, ch, strides, dev, _owner = _image_view(image)
    cp, cs = _cparams(params), _CStats()
    cb = _log_sink(stats)
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    args = (C.byref(cp), ptr, w, h, ch, strides.ctypes.data)
    tail = (cb, None, C.byref(out), C.byref(out_len), C.byref(cs))
    if dev is not None:
        import torch
        ok = lib.gb200_process_image_device(*args, dev.index, *tail, torch.cuda.current_stream(dev).cuda_stream)
    else:
        ok = lib.gb200_process_image(*args, device, *tail)
    data = _take(lib, out, out_len)
    _fill_stats(stats, cs)
    if not ok and not data:
        if "device memory" in _err(lib):  # a pointer the device entry refused
            raise RuntimeError(_err(lib))
        _raise_device_error(lib)
    return bool(ok), data


def process_jpeg(params, stats, jpeg_in, device=0, lib=None):
    """guetzli::Process(params, stats, jpeg_in, &out) (processor.cc:890): JPEG input
    (4:4:4 YCbCr).  Returns (ok, jpeg_bytes) like process().

    jpeg_in: the file as a bytes-like object in host memory, encoded on cuda:`device`, or as a contiguous 1-D
    torch.uint8 CUDA tensor, encoded on the tensor's own device after the work queued on that device's current
    torch stream (gb200_process_jpeg_from_device: a sequential 4:4:4 file is Huffman-decoded there, and only
    its bytes after EOI and one coefficient plane come back).  Both give the same result for the same bytes.
    Other tensors raise ValueError."""
    lib = lib or load_library()
    cp, cs = _cparams(params), _CStats()
    cb = _log_sink(stats)
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    if _is_torch_tensor(jpeg_in):
        import torch
        t = jpeg_in
        if not t.is_cuda or t.dtype != torch.uint8 or t.dim() != 1 or not t.is_contiguous():
            raise ValueError(f"process_jpeg: the file must be a contiguous 1-D torch.uint8 CUDA tensor, got "
                             f"{t.dtype} {tuple(t.shape)} on {t.device}")
        ok = lib.gb200_process_jpeg_from_device(C.byref(cp), t.data_ptr() if t.numel() else None, t.numel(),
                                                t.device.index, cb, None, C.byref(out), C.byref(out_len),
                                                C.byref(cs), torch.cuda.current_stream(t.device).cuda_stream)
    else:
        buf = np.frombuffer(bytes(jpeg_in), dtype=np.uint8)
        ok = lib.gb200_process_jpeg(C.byref(cp), buf.ctypes.data if buf.size else None, buf.size, device, cb, None,
                                    C.byref(out), C.byref(out_len), C.byref(cs))
    data = _take(lib, out, out_len)
    _fill_stats(stats, cs)
    if not ok and not data:
        if "device memory" in _err(lib):  # a pointer the device entry refused
            raise RuntimeError(_err(lib))
        _raise_device_error(lib)
    return bool(ok), data


def decode_jpeg(data, device=0, cuda=True, lib=None):
    """The pixels libjpeg-turbo gives for JPEG files, as the butteraugli tool reads them (ReadJPEG,
    butteraugli_main.cc:157: JDCT_ISLOW, fancy upsampling, RGB, gray replicated), decoded on the GPU.

    data: one file or a list of files (decoded together in one pass whatever their sizes), each a bytes-like
    object in host memory or a contiguous 1-D torch.uint8 CUDA tensor holding the file's bytes.  A list is
    all host bytes or all CUDA tensors, the tensors on one device.
    Returns a uint8 [h][w][3] CUDA tensor per file, written after the work queued on the device's current
    torch stream, or a numpy array where cuda is False; a list for a list.  Host bytes are decoded on
    cuda:`device`; CUDA tensors on their own device, where the Huffman decoding of sequential files runs
    too (the headers are read from prefixes copied to the host, and other files are copied back whole).
    The outputs go as they are into the 8-bit butteraugli entries (butteraugli_srgb, diffmap_sizes_srgb,
    from_srgb).  A file the decoder does not reproduce libjpeg on raises ValueError naming its index and
    the reason: what ReadJpeg rejects, CMYK / YCCK, samplings other than 4:4:4, 4:2:2 and 4:2:0, and
    progressive files that libjpeg would block-smooth.  Mixing host bytes and tensors, tensors on several
    devices or not contiguous 1-D uint8, and cuda=False with tensors raise ValueError as well."""
    lib = lib or load_library()
    single = isinstance(data, (bytes, bytearray, memoryview)) or _is_torch_tensor(data)
    items = [data] if single else list(data)
    if not items:
        raise ValueError("decode_jpeg: no files")
    tensors = [_is_torch_tensor(d) for d in items]
    if any(tensors):
        if not all(tensors):
            raise ValueError("decode_jpeg: a list mixes host bytes and torch tensors")
        out = _decode_jpeg_tensors(items, cuda, lib)
        return out[0] if single else out
    files = [bytes(d) for d in items]
    bufs = [np.frombuffer(f, dtype=np.uint8) for f in files]
    shapes = []
    for b in bufs:
        w, h = C.c_int(), C.c_int()
        ok = b.size and lib.gb200_jpeg_dimensions(b.ctypes.data, b.size, C.byref(w), C.byref(h))
        # a file without a readable frame size gets a 1x1 output; the decoder then refuses it with its reason
        shapes.append((h.value, w.value, 3) if ok else (1, 1, 3))
    n = len(files)
    ptrs = (C.c_void_p * n)(*[b.ctypes.data if b.size else None for b in bufs])
    lens = (C.c_size_t * n)(*[b.size for b in bufs])
    if cuda:
        import torch
        dev = torch.device("cuda", device)
        out = [torch.empty(s, dtype=torch.uint8, device=dev) for s in shapes]
        outp = (C.c_void_p * n)(*[o.data_ptr() for o in out])
        ok = lib.gb200_jpeg_decode_rgb_device(ptrs, lens, n, device, outp, torch.cuda.current_stream(dev).cuda_stream)
    else:
        out = [np.empty(s, dtype=np.uint8) for s in shapes]
        outp = (C.c_void_p * n)(*[o.ctypes.data for o in out])
        ok = lib.gb200_jpeg_decode_rgb(ptrs, lens, n, device, outp)
    if not ok:
        _raise_decode_error(lib)
    return out[0] if single else out


def _raise_decode_error(lib):
    msg = _err(lib)
    if ": file " in msg:
        raise ValueError(msg)
    raise RuntimeError(msg)


def _decode_jpeg_tensors(items, cuda, lib):
    """decode_jpeg on files held in CUDA tensors (gb200_jpeg_decode_rgb_from_device)."""
    import torch
    if not cuda:
        raise ValueError("decode_jpeg: files in torch tensors are decoded into CUDA tensors; cuda=False takes "
                         "host bytes only")
    for i, t in enumerate(items):
        if not t.is_cuda or t.dtype != torch.uint8 or t.dim() != 1 or not t.is_contiguous():
            raise ValueError(f"decode_jpeg: file {i} must be a contiguous 1-D torch.uint8 CUDA tensor, got "
                             f"{t.dtype} {tuple(t.shape)} on {t.device}")
    dev = items[0].device
    if any(t.device != dev for t in items):
        raise ValueError("decode_jpeg: the tensors are on more than one device")
    n = len(items)
    ptrs = (C.c_void_p * n)(*[t.data_ptr() if t.numel() else None for t in items])
    lens = (C.c_size_t * n)(*[t.numel() for t in items])
    stream = torch.cuda.current_stream(dev).cuda_stream
    w, h = (C.c_int * n)(), (C.c_int * n)()
    if not lib.gb200_jpeg_dimensions_from_device(ptrs, lens, n, dev.index, stream, w, h):
        raise RuntimeError(_err(lib))
    # a file without a readable frame size gets a 1x1 output; the decoder then refuses it with its reason
    shapes = [(h[i], w[i], 3) if w[i] > 0 else (1, 1, 3) for i in range(n)]
    out = [torch.empty(s, dtype=torch.uint8, device=dev) for s in shapes]
    outp = (C.c_void_p * n)(*[o.data_ptr() for o in out])
    ws = (C.c_int * n)(*[s[1] for s in shapes])
    hs = (C.c_int * n)(*[s[0] for s in shapes])
    if not lib.gb200_jpeg_decode_rgb_from_device(ptrs, lens, n, dev.index, ws, hs, outp, stream):
        _raise_decode_error(lib)
    return out


def entropy_decode(jpeg_in, S, lib=None, cap=1 << 24):
    """The device path's entropy decoding of one file with subsequences of S bits (test hook) -> (taken,
    coefficients): where the device path takes the file, its quantised coefficients concatenated over the
    components as read_jpeg gives them, at the start of a buffer of cap values whose rest stays zero."""
    lib = lib or load_library()
    buf = np.frombuffer(bytes(jpeg_in), dtype=np.uint8)
    out = np.zeros(cap, dtype=np.int16)
    status = C.c_int()
    if not lib.gb200_debug_entropy_decode(buf.ctypes.data if buf.size else None, buf.size, S, out.ctypes.data, cap,
                                          C.byref(status)):
        raise RuntimeError(_err(lib))
    return bool(status.value), (out if status.value else None)


def entropy_decode_flags(jpeg_in, S, lib=None, cap=1 << 24):
    """entropy_decode with the reason for the path the file takes (test hook) -> (taken, flags, rounds,
    coefficients): taken where the device path's shape takes the file; flags the OR of its kJpegBad* flags
    (JPEG_BAD_*), the SIMD-range test of decode_jpeg included; rounds the synchronisation rounds after the
    first; the coefficients as entropy_decode gives them where taken and flags is 0 or JPEG_BAD_RANGE, else
    None."""
    lib = lib or load_library()
    buf = np.frombuffer(bytes(jpeg_in), dtype=np.uint8)
    out = np.zeros(cap, dtype=np.int16)
    taken, flags, rounds = C.c_int(), C.c_uint(), C.c_int()
    if not lib.gb200_debug_entropy_decode_flags(buf.ctypes.data if buf.size else None, buf.size, S, out.ctypes.data,
                                                cap, C.byref(taken), C.byref(flags), C.byref(rounds)):
        raise RuntimeError(_err(lib))
    coeffs = out if taken.value and not flags.value & ~JPEG_BAD_RANGE else None
    return bool(taken.value), flags.value, rounds.value, coeffs


# the kJpegBad* flags of the device path's status words (csrc/kernels.h)
JPEG_BAD_SEGMENT, JPEG_BAD_CODE, JPEG_BAD_RANGE, JPEG_BAD_SYNC = 1, 2, 4, 8


def jpeg_seed(jpeg_in, S, lib=None, cap=1 << 24):
    """The seeding of process_jpeg's device route on one file with subsequences of S bits (test hook) ->
    (route, dq): route 0 where the file goes to the host route, 1 where the device route takes it and it is
    sane, 2 where it is taken and fails the sanity check; dq the [3][blocks][64] coefficients times their
    quant steps (int16) at the start of a buffer of cap values, or None for route 0."""
    lib = lib or load_library()
    buf = np.frombuffer(bytes(jpeg_in), dtype=np.uint8)
    out = np.zeros(cap, dtype=np.int16)
    status = C.c_int()
    if not lib.gb200_debug_jpeg_seed(buf.ctypes.data if buf.size else None, buf.size, S, out.ctypes.data, cap,
                                     C.byref(status)):
        raise RuntimeError(_err(lib))
    return status.value, (out if status.value else None)


def read_jpeg(jpeg_in, lib=None, cap=1 << 24):
    """ReadJpeg alone (test hook) -> (ok, dims, quantised coefficients concatenated over components); ok is
    False as well where there are more than cap coefficients."""
    lib = lib or load_library()
    buf = np.frombuffer(bytes(jpeg_in), dtype=np.uint8)
    dims = (C.c_int * 11)()
    out = np.zeros(cap, dtype=np.int16)
    ok = lib.gb200_debug_read_jpeg(buf.ctypes.data, buf.size, dims, out.ctypes.data, cap)
    d = list(dims)
    n = sum(d[3 + 2 * c] * d[4 + 2 * c] * 64 for c in range(d[2])) if ok else 0
    return bool(ok), d, out[:n].copy()


def butteraugli_diffmap(rgb0, rgb1, device=0, lib=None):
    """butteraugli::ButteraugliInterface: rgb0, rgb1 planar linear RGB float32 [3][h][w], nominally in
    0..255 -> (diffmap [h][w] float32, score).  Values outside 0..255 (ringing below 0, highlights above 255) are scored as the reference scores
    them, bit for bit; this is tested from -300 to 4500.  NaN and infinities must not be passed: the
    reference's result is undefined for them."""
    lib = lib or load_library()
    a = np.ascontiguousarray(rgb0, dtype=np.float32)
    b = np.ascontiguousarray(rgb1, dtype=np.float32)
    assert a.shape == b.shape and a.ndim == 3 and a.shape[0] == 3
    _, h, w = a.shape
    dm = np.zeros((h, w), dtype=np.float32)
    score = C.c_double()
    if not lib.gb200_butteraugli_diffmap(a.ctypes.data, b.ctypes.data, w, h, device, dm.ctypes.data, C.byref(score)):
        raise RuntimeError(_err(lib))
    return dm, score.value


class _Handle:
    """Owns one C object of `lib`, destroyed by the C function named _destroy on close() or collection."""
    _destroy = None
    _h = None

    def close(self):
        if self._h:
            getattr(self.lib, self._destroy)(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def _ck(self, ok):
        if not ok:
            raise RuntimeError(_err(self.lib))


def _is_torch_tensor(x):
    # without importing torch: a caller that passes a tensor has imported it already
    return type(x).__module__.split(".")[0] == "torch"


def _outputs(device, shapes):
    """float32 outputs of the given shapes: CUDA tensors on the torch device `device`, or host arrays where
    it is None -> (outputs, their pointers, the device's current torch stream or None)."""
    if device is None:
        out = [np.empty(s, dtype=np.float32) for s in shapes]
        return out, [o.ctypes.data for o in out], None
    import torch
    out = [torch.empty(s, dtype=torch.float32, device=device) for s in shapes]
    return out, [o.data_ptr() for o in out], torch.cuda.current_stream(device).cuda_stream


def _srgb_images(name, x, ranks, cuda_ok=True):
    """Checks an 8-bit image argument: a uint8 numpy array, or a CUDA torch tensor where cuda_ok, whose
    rank is in `ranks` and whose last axis holds 3 (RGB) or 4 (RGBA) channels -> (x, is_cuda), contiguous."""
    cuda = _is_torch_tensor(x) and x.is_cuda
    if cuda and not cuda_ok:
        raise ValueError(f"{name} must be in host memory (a numpy array), got a CUDA tensor")
    if cuda:
        import torch
        if x.dtype != torch.uint8:
            raise ValueError(f"{name} must be uint8, got {x.dtype}")
        x = x.contiguous()
    else:
        if _is_torch_tensor(x):
            x = x.numpy()
        x = np.asarray(x)
        if x.dtype != np.uint8:
            raise ValueError(f"{name} must be uint8, got {x.dtype}")
        x = np.ascontiguousarray(x)
    if x.ndim not in ranks:
        raise ValueError(f"{name} must have {' or '.join(str(r) for r in ranks)} axes ([n][h][w][C] or [h][w][C]), "
                         f"got shape {tuple(x.shape)}")
    if x.shape[-1] not in (3, 4):
        raise ValueError(f"{name} must have 3 (RGB) or 4 (RGBA) channels in its last axis, got shape {tuple(x.shape)}")
    return x, cuda


def butteraugli_srgb(img0, img1, device=0, lib=None):
    """The stand-alone `butteraugli` tool's comparison of two 8-bit sRGB images: img0, img1 uint8
    [h][w][C] in host memory, C = 3 (RGB) or 4 (RGBA), any size from 1x1 -> (diffmap [h][w] float32,
    score).  Each image is converted to linear RGB with the tool's table; RGBA is laid over black and
    over white in sRGB space, and the larger score wins with its diffmap (black on a tie).  The result
    is butteraugli_diffmap's on the converted planes, bit for bit."""
    lib = lib or load_library()
    a, _ = _srgb_images("img0", img0, (3,), cuda_ok=False)
    b, _ = _srgb_images("img1", img1, (3,), cuda_ok=False)
    if a.shape != b.shape:
        raise ValueError(f"img0 and img1 differ in shape: {a.shape} and {b.shape}")
    h, w, ch = a.shape
    dm = np.empty((h, w), dtype=np.float32)
    score = C.c_double()
    if not lib.gb200_butteraugli_diffmap_srgb(a.ctypes.data, b.ctypes.data, w, h, ch, device, dm.ctypes.data,
                                              C.byref(score)):
        raise RuntimeError(_err(lib))
    return dm, score.value


def _planar_error(shape):
    return "must be planar [3][h][w]" if len(shape) != 3 or shape[0] != 3 else None


def _interleaved_error(shape):
    if len(shape) != 3:
        return "must be interleaved [h][w][C]"
    return "must have 3 (RGB) or 4 (RGBA) channels in its last axis" if shape[2] not in (3, 4) else None


def _sizes_items(names, seqs, n_error, dtype, shape_error, device, cuda_ok=True):
    """The images of a call on images of sizes of their own, checked in one pass (a call may hold hundreds of
    small images): equal-length sequences `seqs` named `names`, whose length passes n_error (which returns what
    is wrong with it, or None), all numpy arrays or all CUDA tensors (numpy arrays only, where not cuda_ok),
    each of `dtype` ("float32" or "uint8"), contiguous, its shape passing shape_error (which returns what is
    wrong with a shape, or None) -> (n, the torch device `device` for CUDA tensors or None, the pointers of
    every sequence in turn, their shapes)."""
    seqs = [list(x) for x in seqs]
    n = len(seqs[0])
    for name, x in zip(names[1:], seqs[1:]):
        if len(x) != n:
            raise ValueError(f"{names[0]} and {name} differ in length: {n} and {len(x)}")
    wrong = n_error(n)
    if wrong:
        raise ValueError(wrong)
    items = [x for seq in seqs for x in seq]
    cuda = cuda_ok and _is_torch_tensor(items[0]) and items[0].is_cuda
    if cuda:
        import torch
        torch_dtype = getattr(torch, dtype)
    kinds = "a numpy array or a CUDA tensor" if cuda_ok else "a numpy array (host memory)"
    ptrs, shapes = [], []
    for k, x in enumerate(items):
        name = names[k // n]
        if isinstance(x, np.ndarray):
            if cuda:
                raise ValueError("the images must all be CUDA tensors or all host arrays")
            if x.dtype != dtype:
                raise ValueError(f"{name}[{k % n}] must be {dtype}, got {x.dtype}")
            contiguous = x.flags.c_contiguous
            ptrs.append(x.ctypes.data)
        elif cuda_ok and _is_torch_tensor(x) and x.is_cuda:
            if not cuda:
                raise ValueError("the images must all be CUDA tensors or all host arrays")
            if x.dtype != torch_dtype:
                raise ValueError(f"{name}[{k % n}] must be {dtype}, got {x.dtype}")
            contiguous = x.is_contiguous()
            ptrs.append(x.data_ptr())
        else:
            raise ValueError(f"{name}[{k % n}] must be {kinds}, got {type(x).__name__}")
        shape = tuple(x.shape)
        wrong = shape_error(shape)
        if wrong:
            raise ValueError(f"{name}[{k % n}] {wrong}, got shape {shape}")
        if not contiguous:
            raise ValueError(f"{name}[{k % n}] must be contiguous")
        shapes.append(shape)
    return n, torch.device("cuda", device) if cuda else None, ptrs, shapes


class Comparator(_Handle):
    """butteraugli::ButteraugliComparator (butteraugli.h:425) on one GPU: the original rgb0, planar
    linear RGB float32 [3][h][w], nominally in 0..255 and at least 8x8, stays resident and is scored
    against any number of images, up to `capacity` (1..16383) of them per diffmap() call in one pass of
    the Compare chain.  rgb0 may be a numpy array or a float32 CUDA tensor on the comparator's device,
    read after the work queued on that device's current torch stream and copied on the device; either
    way it may be changed or freed once the comparator is made.  Used by one thread at a time.  Values outside 0..255 (ringing below 0, highlights above 255) are scored as the reference scores
    them, bit for bit; this is tested from -300 to 4500.  NaN and infinities must not be passed: the
    reference's result is undefined for them."""

    _destroy = "gb200_butteraugli_comparator_destroy"

    def __init__(self, rgb0, device=0, capacity=1, lib=None):
        self.lib = lib or load_library()
        self.channels = 0  # made from float planes
        self.device, self.capacity = device, int(capacity)
        if _is_torch_tensor(rgb0) and rgb0.is_cuda:
            import torch
            if rgb0.dtype != torch.float32 or rgb0.ndim != 3 or rgb0.shape[0] != 3:
                raise ValueError(f"rgb0 must be float32 planar [3][h][w], got {rgb0.dtype} {tuple(rgb0.shape)}")
            t = rgb0.contiguous()
            _, self.h, self.w = t.shape
            self._h = self.lib.gb200_butteraugli_comparator_create_device(
                t.data_ptr(), self.w, self.h, self.capacity, device, torch.cuda.current_stream(t.device).cuda_stream)
        else:
            a = np.ascontiguousarray(rgb0, dtype=np.float32)
            if a.ndim != 3 or a.shape[0] != 3:
                raise ValueError(f"rgb0 must be planar [3][h][w], got shape {a.shape}")
            _, self.h, self.w = a.shape
            self._h = self.lib.gb200_butteraugli_comparator_create_batch(a.ctypes.data, self.w, self.h,
                                                                         self.capacity, device)
        if not self._h:
            raise RuntimeError("gb200_butteraugli_comparator_create failed: " + _err(self.lib))

    @classmethod
    def from_srgb(cls, img0, capacity=1, device=0, lib=None):
        """A comparator whose original is an 8-bit sRGB image, uint8 [h][w][C] in host memory with C = 3
        (RGB) or 4 (RGBA), at least 8x8, scored as butteraugli_srgb scores it.  With C = 4 the original
        is kept twice, laid over black and over white.  diffmap() then takes uint8 [h][w][C] or
        [n][h][w][C] with the same C, numpy or CUDA tensors, and nothing else; mask() refuses RGBA.
        An original in CUDA memory goes to from_srgb_device."""
        a, _ = _srgb_images("img0", img0, (3,), cuda_ok=False)
        return cls._from_srgb(a, False, capacity, device, lib)

    @classmethod
    def from_srgb_device(cls, img0, capacity=1, device=0, lib=None):
        """from_srgb with the original a uint8 CUDA tensor [h][w][C] on the comparator's device, converted where it
        lies after the work queued on that device's current torch stream; no pixel goes through the host.  The
        comparator is the one from_srgb makes of the same bytes, and img0 may be changed or freed once it is made."""
        a, cuda = _srgb_images("img0", img0, (3,))
        if not cuda:
            raise ValueError(f"img0 must be a CUDA tensor, got {type(img0).__name__} (from_srgb takes host memory)")
        return cls._from_srgb(a, True, capacity, device, lib)

    @classmethod
    def _from_srgb(cls, a, cuda, capacity, device, lib):
        self = cls.__new__(cls)
        self.lib = lib or load_library()
        self.h, self.w, self.channels = a.shape
        self.device, self.capacity = device, int(capacity)
        if cuda:
            import torch
            self._h = self.lib.gb200_butteraugli_comparator_create_srgb_device(
                a.data_ptr(), self.w, self.h, self.channels, self.capacity, device,
                torch.cuda.current_stream(a.device).cuda_stream)
        else:
            self._h = self.lib.gb200_butteraugli_comparator_create_srgb(a.ctypes.data, self.w, self.h, self.channels,
                                                                        self.capacity, device)
        if not self._h:
            raise RuntimeError("gb200_butteraugli_comparator_create_srgb failed: " + _err(self.lib))
        return self

    def diffmap(self, rgb1):
        """ButteraugliComparator::Diffmap + ButteraugliScoreFromDiffmap -> (diffmap [h][w], score).

        A CUDA torch tensor (float32, [3][h][w]) is scored from device memory after the work queued
        on its device's current torch stream, and the diffmap comes back as a tensor on that device.
        Anything else is read as a numpy array in host memory.

        rgb1 float32 [n][3][h][w] with 1 <= n <= capacity scores each image the same way, all in one
        call -> (diffmaps [n][h][w], scores float64 ndarray [n]).

        On a comparator made by from_srgb, rgb1 is uint8 [h][w][C] or [n][h][w][C] instead."""
        if self.channels:
            return self._diffmap_srgb(rgb1)
        if len(getattr(rgb1, "shape", ())) == 4:
            return self._diffmap_batch(rgb1)
        if _is_torch_tensor(rgb1) and rgb1.is_cuda:
            return self._diffmap_device(rgb1)
        a = np.ascontiguousarray(rgb1, dtype=np.float32)
        if a.shape != (3, self.h, self.w):
            raise ValueError(f"rgb1 must have shape {(3, self.h, self.w)}, got {a.shape}")
        [dm], [dp], _ = _outputs(None, [(self.h, self.w)])
        score = C.c_double()
        self._ck(self.lib.gb200_butteraugli_comparator_diffmap(self._h, a.ctypes.data, dp, C.byref(score)))
        return dm, score.value

    def _diffmap_device(self, t):
        import torch
        if t.dtype != torch.float32 or tuple(t.shape) != (3, self.h, self.w):
            raise ValueError(f"rgb1 must be float32 of shape {(3, self.h, self.w)}, got {t.dtype} {tuple(t.shape)}")
        t = t.contiguous()
        [dm], [dp], stream = _outputs(t.device, [(self.h, self.w)])
        score = C.c_double()
        self._ck(self.lib.gb200_butteraugli_comparator_diffmap_device(self._h, t.data_ptr(), dp, C.byref(score),
                                                                      stream))
        return dm, score.value

    def _diffmap_batch(self, rgb1):
        shape = tuple(rgb1.shape)
        if shape[1:] != (3, self.h, self.w) or not 1 <= shape[0] <= self.capacity:
            raise ValueError(f"rgb1 must have shape [n, 3, {self.h}, {self.w}] with 1 <= n <= {self.capacity}, "
                             f"got {shape}")
        n = shape[0]
        score = np.empty(n, dtype=np.float64)
        if _is_torch_tensor(rgb1) and rgb1.is_cuda:
            import torch
            if rgb1.dtype != torch.float32:
                raise ValueError(f"rgb1 must be float32, got {rgb1.dtype}")
            t = rgb1.contiguous()
            [dm], [dp], stream = _outputs(t.device, [(n, self.h, self.w)])
            self._ck(self.lib.gb200_butteraugli_comparator_diffmap_batch_device(self._h, t.data_ptr(), n, dp,
                                                                                score.ctypes.data, stream))
            return dm, score
        a = np.asarray(rgb1)
        if a.dtype != np.float32:
            raise ValueError(f"rgb1 must be float32, got {a.dtype}")
        a = np.ascontiguousarray(a)
        [dm], [dp], _ = _outputs(None, [(n, self.h, self.w)])
        self._ck(self.lib.gb200_butteraugli_comparator_diffmap_batch(self._h, a.ctypes.data, n, dp, score.ctypes.data))
        return dm, score

    def _diffmap_srgb(self, img1):
        x, cuda = _srgb_images("img1", img1, (3, 4))
        single = x.ndim == 3
        shape = tuple(x.shape[1:] if not single else x.shape)
        n = 1 if single else x.shape[0]
        if shape != (self.h, self.w, self.channels) or not 1 <= n <= self.capacity:
            raise ValueError(f"img1 must have shape [{self.h}, {self.w}, {self.channels}] or [n, {self.h}, {self.w}, "
                             f"{self.channels}] with 1 <= n <= {self.capacity}, got {tuple(x.shape)}")
        score = np.empty(n, dtype=np.float64)
        [dm], [dp], stream = _outputs(x.device if cuda else None, [(n, self.h, self.w)])
        if cuda:
            self._ck(self.lib.gb200_butteraugli_comparator_diffmap_srgb_device(self._h, x.data_ptr(), n, dp,
                                                                               score.ctypes.data, stream))
        else:
            self._ck(self.lib.gb200_butteraugli_comparator_diffmap_srgb(self._h, x.ctypes.data, n, dp,
                                                                        score.ctypes.data))
        return (dm[0], float(score[0])) if single else (dm, score)

    def mask(self, cuda=False):
        """ButteraugliComparator::Mask -> (mask, mask_dc), float32 [3][h][w] each: numpy arrays, or with
        cuda=True tensors on the comparator's device, written in order on its current torch stream."""
        [m, mdc], [mp, mdcp], stream = _outputs(self._torch_device() if cuda else None, [(3, self.h, self.w)] * 2)
        if cuda:
            self._ck(self.lib.gb200_butteraugli_comparator_mask_device(self._h, mp, mdcp, stream))
        else:
            self._ck(self.lib.gb200_butteraugli_comparator_mask(self._h, mp, mdcp))
        return m, mdc

    def _torch_device(self):
        import torch
        return torch.device("cuda", self.device)


class ButteraugliBatch(_Handle):
    """butteraugli::ButteraugliInterface on up to `capacity` same-size pairs per call, on one GPU: each
    pair (rgb0[i], rgb1[i]) is scored as gb.butteraugli_diffmap scores it alone, bit for bit, with the
    pairs going through the Compare chain together.  Images are planar linear RGB float32, nominally in
    0..255, at least 8x8.  Used by one thread at a time.  Values outside 0..255 (ringing below 0, highlights above 255) are scored as the reference scores
    them, bit for bit; this is tested from -300 to 4500.  NaN and infinities must not be passed: the
    reference's result is undefined for them."""

    _destroy = "gb200_butteraugli_batch_destroy"

    def __init__(self, h, w, capacity, device=0, lib=None):
        self.lib = lib or load_library()
        self.h, self.w, self.capacity, self.device = int(h), int(w), int(capacity), device
        self._h = self.lib.gb200_butteraugli_batch_create(self.w, self.h, self.capacity, device)
        if not self._h:
            raise RuntimeError("gb200_butteraugli_batch_create failed: " + _err(self.lib))

    def _shape_of(self, shape):
        if len(shape) != 4 or tuple(shape[1:]) != (3, self.h, self.w) or not 1 <= shape[0] <= self.capacity:
            raise ValueError(f"rgb0 and rgb1 must have shape [n, 3, {self.h}, {self.w}] with 1 <= n <= "
                             f"{self.capacity}, got {tuple(shape)}")
        return shape[0]

    def diffmap(self, rgb0, rgb1):
        """-> (diffmaps [n][h][w], scores float64 [n]) for rgb0, rgb1 float32 [n][3][h][w].

        CUDA torch tensors are scored from device memory after the work queued on their device's
        current torch stream, and the diffmaps come back as a tensor on that device.  Anything else
        is read as numpy arrays in host memory.  The scores are a numpy array either way."""
        if _is_torch_tensor(rgb0) and _is_torch_tensor(rgb1) and rgb0.is_cuda and rgb1.is_cuda:
            return self._diffmap_device(rgb0, rgb1)
        if _is_torch_tensor(rgb0) or _is_torch_tensor(rgb1):
            if getattr(rgb0, "is_cuda", False) or getattr(rgb1, "is_cuda", False):
                raise ValueError("rgb0 and rgb1 must both be CUDA tensors or both host arrays")
        a, b = np.asarray(rgb0), np.asarray(rgb1)
        if a.dtype != np.float32 or b.dtype != np.float32:
            raise ValueError(f"rgb0 and rgb1 must be float32, got {a.dtype} and {b.dtype}")
        if a.shape != b.shape:
            raise ValueError(f"rgb0 and rgb1 differ in shape: {a.shape} and {b.shape}")
        n = self._shape_of(a.shape)
        a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
        [dm], [dp], _ = _outputs(None, [(n, self.h, self.w)])
        score = np.empty(n, dtype=np.float64)
        self._ck(self.lib.gb200_butteraugli_batch_diffmap(self._h, a.ctypes.data, b.ctypes.data, n, dp,
                                                          score.ctypes.data))
        return dm, score

    def _diffmap_device(self, t0, t1):
        import torch
        if t0.dtype != torch.float32 or t1.dtype != torch.float32:
            raise ValueError(f"rgb0 and rgb1 must be float32, got {t0.dtype} and {t1.dtype}")
        if tuple(t0.shape) != tuple(t1.shape):
            raise ValueError(f"rgb0 and rgb1 differ in shape: {tuple(t0.shape)} and {tuple(t1.shape)}")
        if t0.device != t1.device:
            raise ValueError(f"rgb0 and rgb1 are on different devices: {t0.device} and {t1.device}")
        n = self._shape_of(tuple(t0.shape))
        t0, t1 = t0.contiguous(), t1.contiguous()
        [dm], [dp], stream = _outputs(t0.device, [(n, self.h, self.w)])
        score = np.empty(n, dtype=np.float64)
        self._ck(self.lib.gb200_butteraugli_batch_diffmap_device(self._h, t0.data_ptr(), t1.data_ptr(), n, dp,
                                                                 score.ctypes.data, stream))
        return dm, score

    def _n_error(self, n):
        return None if 1 <= n <= self.capacity else f"the batch takes 1..{self.capacity} pairs, got {n}"

    def diffmap_sizes(self, rgb0s, rgb1s):
        """Pairs of different sizes in one call: rgb0s, rgb1s equal-length sequences (1 <= n <= capacity) of
        float32 [3][h_i][w_i] with 8 <= h_i <= h and 8 <= w_i <= w, pair i the same shape on both sides ->
        (list of n diffmaps [h_i][w_i], scores float64 [n]), each pair bit for bit butteraugli_diffmap's.

        The items are all numpy arrays (host memory) or all CUDA tensors, scored after the work queued on
        the batch device's current torch stream; the diffmaps come back the same kind, CUDA tensors on the
        batch's device.  As in diffmap(), a tensor on another device is refused by the C entry (RuntimeError,
        naming the argument and its device); malformed arguments raise ValueError."""
        n, dev, ptrs, shapes = _sizes_items(("rgb0s", "rgb1s"), (rgb0s, rgb1s), self._n_error, "float32",
                                            _planar_error, self.device)
        for i in range(n):
            if shapes[i] != shapes[n + i]:
                raise ValueError(f"pair {i} differs in shape: {shapes[i]} and {shapes[n + i]}")
            _, h, w = shapes[i]
            if not (8 <= h <= self.h and 8 <= w <= self.w):
                raise ValueError(f"pair {i} is {h}x{w}; the batch takes 8x8 up to {self.h}x{self.w}")
        ws = np.array([s[2] for s in shapes[:n]], dtype=np.int32)
        hs = np.array([s[1] for s in shapes[:n]], dtype=np.int32)
        P = C.c_void_p * n
        dm, dps, stream = _outputs(dev, [s[1:] for s in shapes[:n]])
        score = np.empty(n, dtype=np.float64)
        args = (self._h, ws.ctypes.data, hs.ctypes.data, P(*ptrs[:n]), P(*ptrs[n:]), n, P(*dps), score.ctypes.data)
        if dev is not None:
            self._ck(self.lib.gb200_butteraugli_batch_diffmap_sizes_device(*args, stream))
        else:
            self._ck(self.lib.gb200_butteraugli_batch_diffmap_sizes(*args))
        return dm, score

    def diffmap_srgb(self, img0, img1):
        """The same for 8-bit sRGB pairs, each scored as butteraugli_srgb scores it: img0, img1 uint8
        [n][h][w][C], C = 3 (RGB) or 4 (RGBA) -> (diffmaps [n][h][w], scores float64 [n]).  Host arrays
        are uploaded once as bytes; CUDA tensors are read in place after the work queued on their device's
        current torch stream, and the diffmaps come back as a tensor on that device."""
        a, cuda0 = _srgb_images("img0", img0, (4,))
        b, cuda1 = _srgb_images("img1", img1, (4,))
        if cuda0 != cuda1:
            raise ValueError("img0 and img1 must both be CUDA tensors or both host arrays")
        if tuple(a.shape) != tuple(b.shape):
            raise ValueError(f"img0 and img1 differ in shape: {tuple(a.shape)} and {tuple(b.shape)}")
        n, h, w, ch = a.shape
        if (h, w) != (self.h, self.w) or not 1 <= n <= self.capacity:
            raise ValueError(f"img0 and img1 must have shape [n, {self.h}, {self.w}, C] with 1 <= n <= "
                             f"{self.capacity}, got {tuple(a.shape)}")
        if cuda0 and a.device != b.device:
            raise ValueError(f"img0 and img1 are on different devices: {a.device} and {b.device}")
        [dm], [dp], stream = _outputs(a.device if cuda0 else None, [(n, h, w)])
        score = np.empty(n, dtype=np.float64)
        if cuda0:
            self._ck(self.lib.gb200_butteraugli_batch_diffmap_srgb_device(self._h, a.data_ptr(), b.data_ptr(), n, ch,
                                                                          dp, score.ctypes.data, stream))
        else:
            self._ck(self.lib.gb200_butteraugli_batch_diffmap_srgb(self._h, a.ctypes.data, b.ctypes.data, n, ch, dp,
                                                                   score.ctypes.data))
        return dm, score

    def diffmap_sizes_srgb(self, img0s, img1s):
        """diffmap_sizes for 8-bit sRGB pairs, each scored as butteraugli_srgb scores it: img0s, img1s
        equal-length sequences (1 <= n <= capacity) of uint8 [h_i][w_i][C_i] with 8 <= h_i <= h,
        8 <= w_i <= w and C_i = 3 (RGB) or 4 (RGBA), pair i the same shape on both sides; RGB and RGBA pairs
        may share a call -> (list of n diffmaps float32 [h_i][w_i], scores float64 [n]).

        The items are all numpy arrays (host memory, packed and uploaded once as bytes) or all CUDA tensors
        on the batch's device, read in place after the work queued on its current torch stream; the diffmaps
        come back the same kind.  As in diffmap_sizes(), a tensor on another device is refused by the C entry
        (RuntimeError); malformed arguments raise ValueError."""
        n, dev, ptrs, shapes = _sizes_items(("img0s", "img1s"), (img0s, img1s), self._n_error, "uint8",
                                            _interleaved_error, self.device)
        for i in range(n):
            if shapes[i][2] != shapes[n + i][2]:
                raise ValueError(f"pair {i}: different number of channels: {shapes[i][2]} and {shapes[n + i][2]}")
            if shapes[i] != shapes[n + i]:
                raise ValueError(f"pair {i} differs in shape: {shapes[i]} and {shapes[n + i]}")
            h, w, _ = shapes[i]
            if not (8 <= h <= self.h and 8 <= w <= self.w):
                raise ValueError(f"pair {i} is {h}x{w}; the batch takes 8x8 up to {self.h}x{self.w} "
                                 "(butteraugli_srgb scores smaller pairs)")
        ws = np.array([s[1] for s in shapes[:n]], dtype=np.int32)
        hs = np.array([s[0] for s in shapes[:n]], dtype=np.int32)
        chs = np.array([s[2] for s in shapes[:n]], dtype=np.int32)
        P = C.c_void_p * n
        dm, dps, stream = _outputs(dev, [s[:2] for s in shapes[:n]])
        score = np.empty(n, dtype=np.float64)
        args = (self._h, ws.ctypes.data, hs.ctypes.data, chs.ctypes.data, P(*ptrs[:n]), P(*ptrs[n:]), n, P(*dps),
                score.ctypes.data)
        if dev is not None:
            self._ck(self.lib.gb200_butteraugli_batch_diffmap_sizes_srgb_device(*args, stream))
        else:
            self._ck(self.lib.gb200_butteraugli_batch_diffmap_sizes_srgb(*args))
        return dm, score


class ComparatorSet(_Handle):
    """Many resident originals of sizes of their own, each scored against any number of candidates: the
    originals rgb0s, a sequence of planar linear RGB float32 [3][h_i][w_i], each at least 8x8, are analysed
    once on one GPU and kept there (40 bytes per pixel).  They are all numpy arrays, or all CUDA tensors on the
    set's device, read in place after the work queued on its current torch stream; either way they may be
    changed or freed once the set is made.  diffmap() scores up to `capacity`
    (1..16383) candidates per call, each against the original it names, in one pass of the Compare chain;
    each result is bit for bit ButteraugliBatch.diffmap_sizes' on the pair (original, candidate), whatever
    else the call holds.  Used by one thread at a time."""

    _destroy = "gb200_butteraugli_comparator_set_destroy"

    def __init__(self, rgb0s, capacity=1, device=0, lib=None):
        self._make(rgb0s, capacity, device, lib, srgb=False)

    @classmethod
    def from_srgb(cls, img0s, capacity=1, device=0, lib=None):
        """A set of 8-bit sRGB originals, uint8 [h_i][w_i][C_i] with C_i = 3 (RGB) or 4 (RGBA), all numpy
        arrays or all CUDA tensors on the set's device (as in the constructor), each at least 8x8, scored as butteraugli_srgb scores them (an RGBA original is kept twice,
        laid over black and over white).  diffmap() then takes uint8 [h][w][C] candidates with their
        original's shape, and nothing else."""
        self = cls.__new__(cls)
        self._make(img0s, capacity, device, lib, srgb=True)
        return self

    def _make(self, items, capacity, device, lib, srgb):
        self.lib = lib or load_library()
        self.device, self.capacity, self.srgb = device, int(capacity), srgb
        name = "img0s" if srgb else "rgb0s"
        n, dev, ptrs, self.shapes = _sizes_items(
            (name,), (items,), lambda n: None if n >= 1 else "a set holds at least 1 original, got 0",
            "uint8" if srgb else "float32", _interleaved_error if srgb else _planar_error, device)
        hw = [s[:2] if srgb else s[1:] for s in self.shapes]
        for i, (h, w) in enumerate(hw):
            if not (8 <= h < 65536 and 8 <= w < 65536):
                raise ValueError(f"{name}[{i}] is {h}x{w}; originals must be at least 8x8 (and below 65536)")
        hs = np.array([x[0] for x in hw], dtype=np.int32)
        ws = np.array([x[1] for x in hw], dtype=np.int32)
        P = C.c_void_p * n
        chs = np.array([s[2] for s in self.shapes], dtype=np.int32) if srgb else None
        args = (ws.ctypes.data, hs.ctypes.data) + ((chs.ctypes.data,) if srgb else ()) + (P(*ptrs), n,
                                                                                          self.capacity, device)
        entry = "gb200_butteraugli_comparator_set_create" + ("_srgb" if srgb else "")
        if dev is not None:
            import torch
            self._h = getattr(self.lib, entry + "_device")(*args, torch.cuda.current_stream(dev).cuda_stream)
        else:
            self._h = getattr(self.lib, entry)(*args)
        if not self._h:
            raise RuntimeError("gb200_butteraugli_comparator_set_create failed: " + _err(self.lib))

    def diffmap(self, index, candidates):
        """Candidate i against original index[i] -> (list of n diffmaps float32 [h_i][w_i], scores float64 [n]).

        index: a sequence of n ints in 0..len(originals) - 1, originals in any order, any number of times;
        candidates: n images (1 <= n <= capacity), candidate i of original index[i]'s shape.  They are all
        numpy arrays (host memory) or all CUDA tensors on the set's device, scored after the work queued on
        its current torch stream; the diffmaps come back the same kind.  A tensor on another device is refused
        by the C entry (RuntimeError); malformed arguments raise ValueError."""
        idx = np.asarray(index)
        if idx.ndim != 1 or not np.issubdtype(idx.dtype, np.integer):
            raise ValueError(f"index must be a sequence of ints, got {type(index).__name__} of {idx.dtype}")
        name = "img1s" if self.srgb else "rgb1s"
        n, dev, ptrs, shapes = _sizes_items(
            (name,), (candidates,),
            lambda n: None if 1 <= n <= self.capacity else f"the set takes 1..{self.capacity} candidates, got {n}",
            "uint8" if self.srgb else "float32", _interleaved_error if self.srgb else _planar_error, self.device)
        if len(idx) != n:
            raise ValueError(f"index and {name} differ in length: {len(idx)} and {n}")
        count = len(self.shapes)
        for i, o in enumerate(idx.tolist()):
            if not 0 <= o < count:
                raise ValueError(f"index[{i}] = {o}, the set holds originals 0..{count - 1}")
            if self.srgb and shapes[i][2] != self.shapes[o][2]:
                raise ValueError(f"{name}[{i}]: different number of channels: {shapes[i][2]}, its original {o} has "
                                 f"{self.shapes[o][2]}")
            if shapes[i] != self.shapes[o]:
                raise ValueError(f"{name}[{i}] must have original {o}'s shape {self.shapes[o]}, got {shapes[i]}")
        orig = idx.astype(np.int32)
        P = C.c_void_p * n
        dm, dps, stream = _outputs(dev, [s[:2] if self.srgb else s[1:] for s in shapes])
        score = np.empty(n, dtype=np.float64)
        args = (self._h, orig.ctypes.data, P(*ptrs), n, P(*dps), score.ctypes.data)
        entry = "gb200_butteraugli_comparator_set_diffmap" + ("_srgb" if self.srgb else "")
        if dev is not None:
            self._ck(getattr(self.lib, entry + "_device")(*args, stream))
        else:
            self._ck(getattr(self.lib, entry)(*args))
        return dm, score


def adaptive_quantization(rgb, device=0, lib=None):
    """butteraugli::ButteraugliAdaptiveQuantization: rgb planar linear RGB float32 [3][h][w], nominally
    in 0..255 -> quant [h][w] float32.  A CUDA tensor is read on its own device after the work queued on
    its current torch stream, and quant comes back as a tensor there (`device` is then not used).  Raises
    ValueError below 16x16, where the reference returns false.  Values outside 0..255 (ringing below 0, highlights above 255) are scored as the reference scores
    them, bit for bit; this is tested from -300 to 4500.  NaN and infinities must not be passed: the
    reference's result is undefined for them."""
    lib = lib or load_library()
    if _is_torch_tensor(rgb) and rgb.is_cuda:
        import torch
        if rgb.dtype != torch.float32 or rgb.ndim != 3 or rgb.shape[0] != 3:
            raise ValueError(f"rgb must be float32 planar [3][h][w], got {rgb.dtype} {tuple(rgb.shape)}")
        t = rgb.contiguous()
        _, h, w = t.shape
        if w < 16 or h < 16:
            raise ValueError(f"adaptive quantization needs at least 16x16 pixels, got {w}x{h}")
        [quant], [qp], stream = _outputs(t.device, [(h, w)])
        if not lib.gb200_butteraugli_adaptive_quantization_device(t.data_ptr(), w, h, t.device.index, qp, stream):
            raise RuntimeError(_err(lib))
        return quant
    a = np.ascontiguousarray(rgb, dtype=np.float32)
    if a.ndim != 3 or a.shape[0] != 3:
        raise ValueError(f"rgb must be planar [3][h][w], got shape {a.shape}")
    _, h, w = a.shape
    if w < 16 or h < 16:
        raise ValueError(f"adaptive quantization needs at least 16x16 pixels, got {w}x{h}")
    quant = np.empty((h, w), dtype=np.float32)
    if not lib.gb200_butteraugli_adaptive_quantization(a.ctypes.data, w, h, device, quant.ctypes.data):
        raise RuntimeError(_err(lib))
    return quant


def heatmap_thresholds():
    """The butteraugli tool's heat-map thresholds (butteraugli_main.cc:423-424): (good, bad) =
    (ButteraugliFuzzyInverse(1.5), ButteraugliFuzzyInverse(0.5))."""
    return _fuzzy_inverse(1.5), _fuzzy_inverse(0.5)


def _fuzzy_inverse(seek):
    # ButteraugliFuzzyClass / ButteraugliFuzzyInverse (butteraugli.cc:1902, :1923) in the same double arithmetic,
    # as the butteraugli CLI states them (cli/butteraugli.cc)
    def fuzzy_class(score):
        width_up, width_down, m0, scaler = 6.07887388532, 5.50793514384, 2.0, 0.840253347958
        if score < 1.0:
            v = m0 / (1.0 + math.exp((score - 1.0) * width_down))
            v -= 1.0
            v *= 2.0 - scaler
            return v + scaler
        return m0 / (1.0 + math.exp((score - 1.0) * width_up)) * scaler
    pos, r = 0.0, 1.0
    while r >= 1e-10:
        pos += -r if fuzzy_class(pos) < seek else r
        r *= 0.5
    return pos


def heatmap(diffmap, good=None, bad=None, device=0, lib=None):
    """butteraugli::CreateHeatMapImage (butteraugli.cc:1979): a diffmap float32 [h][w] -> its heat map, uint8
    [h][w][3], the reference's bytes exactly.  good, bad: the thresholds, 0 < good < bad; None for either takes
    the butteraugli tool's (heatmap_thresholds()).

    A numpy array gives a numpy array, made on GPU `device`; a CUDA tensor gives a tensor on its device, made
    after the work queued on that device's current torch stream.  A list (or tuple) of maps of sizes of their
    own, all numpy arrays or all CUDA tensors, gives a list, made in one launch."""
    lib = lib or load_library()
    tool_good, tool_bad = heatmap_thresholds()
    good = tool_good if good is None else float(good)
    bad = tool_bad if bad is None else float(bad)
    many = isinstance(diffmap, (list, tuple))
    maps = list(diffmap) if many else [diffmap]
    if not maps:
        raise ValueError("heatmap needs at least 1 map, got an empty list")
    cuda = _is_torch_tensor(maps[0]) and maps[0].is_cuda
    items = []
    for i, m in enumerate(maps):
        name = f"diffmap[{i}]" if many else "diffmap"
        if cuda != (_is_torch_tensor(m) and m.is_cuda):
            raise ValueError("the maps must all be CUDA tensors or all host arrays")
        if cuda:
            import torch
            if m.dtype != torch.float32:
                raise ValueError(f"{name} must be float32, got {m.dtype}")
            m = m.contiguous()
        else:
            m = np.asarray(m.numpy() if _is_torch_tensor(m) else m)
            if m.dtype != np.float32:
                raise ValueError(f"{name} must be float32, got {m.dtype}")
            m = np.ascontiguousarray(m)
        if m.ndim != 2 or m.shape[0] < 1 or m.shape[1] < 1:
            raise ValueError(f"{name} must be [h][w] with h, w >= 1, got shape {tuple(m.shape)}")
        items.append(m)
    n = len(items)
    hs = np.array([m.shape[0] for m in items], dtype=np.int32)
    ws = np.array([m.shape[1] for m in items], dtype=np.int32)
    P = C.c_void_p * n
    if cuda:
        import torch
        dev = items[0].device
        for i, m in enumerate(items):
            if m.device != dev:
                raise ValueError(f"the maps must be on one device: diffmap[{i}] is on {m.device}, not {dev}")
        out = [torch.empty((m.shape[0], m.shape[1], 3), dtype=torch.uint8, device=dev) for m in items]
        ok = lib.gb200_butteraugli_heatmap_device(ws.ctypes.data, hs.ctypes.data, P(*[m.data_ptr() for m in items]),
                                                  n, good, bad, P(*[o.data_ptr() for o in out]), dev.index,
                                                  torch.cuda.current_stream(dev).cuda_stream)
    else:
        out = [np.empty((m.shape[0], m.shape[1], 3), dtype=np.uint8) for m in items]
        ok = lib.gb200_butteraugli_heatmap(ws.ctypes.data, hs.ctypes.data, P(*[m.ctypes.data for m in items]), n,
                                           good, bad, P(*[o.ctypes.data for o in out]), device)
    if not ok:
        raise RuntimeError(_err(lib))
    return out if many else out[0]


def counters(lib=None):
    """-> (kernel launches, h2d bytes, d2h bytes): process-wide running totals."""
    lib = lib or load_library()
    n, a, b = C.c_long(), C.c_longlong(), C.c_longlong()
    lib.gb200_counters(C.byref(n), C.byref(a), C.byref(b))
    return n.value, a.value, b.value


def process_tiled_threads(params, rgb, w, h, world, device=0, lib=None):
    """One image decomposed into `world` row strips handled by `world` host threads
    on one device (test entry of the strip mode) -> (ok, jpeg)."""
    lib = lib or load_library()
    buf = np.ascontiguousarray(np.asarray(rgb, dtype=np.uint8)).reshape(-1)
    cp, cs = _cparams(params), _CStats()
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    ok = lib.gb200_process_rgb_tiled_threads(C.byref(cp), buf.ctypes.data, w, h, device, world,
                                             C.byref(out), C.byref(out_len), C.byref(cs))
    data = _take(lib, out, out_len)
    if not ok and not data:
        raise RuntimeError(_err(lib))
    return bool(ok), data


def dist_unique_id(lib=None):
    lib = lib or load_library()
    buf = (C.c_uint8 * 128)()
    if not lib.gb200_dist_unique_id(buf):
        raise RuntimeError(_err(lib))
    return bytes(buf)


def last_error(lib=None):
    """gb200_last_error() of the calling thread."""
    return _err(lib or load_library())


def dist_shutdown(lib=None):
    (lib or load_library()).gb200_dist_shutdown()


def dist_init(uid, rank, world, device, lib=None):
    lib = lib or load_library()
    buf = (C.c_uint8 * 128).from_buffer_copy(uid)
    if not lib.gb200_dist_init(buf, rank, world, device):
        raise RuntimeError(_err(lib))


def process_tiled(params, stats, rgb, w, h, lib=None):
    """Collective: every rank (after dist_init) passes the same image -> (ok, jpeg)."""
    lib = lib or load_library()
    buf = np.ascontiguousarray(np.asarray(rgb, dtype=np.uint8)).reshape(-1)
    cp, cs = _cparams(params), _CStats()
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    ok = lib.gb200_process_rgb_tiled(C.byref(cp), buf.ctypes.data, w, h, C.cast(None, _LOG_FN), None,
                                     C.byref(out), C.byref(out_len), C.byref(cs))
    data = _take(lib, out, out_len)
    _fill_stats(stats, cs, directions=False)
    if not ok and not data:
        raise RuntimeError(_err(lib))
    return bool(ok), data


def write_jpeg(coeffs, w, h, q, lib=None):
    lib = lib or load_library()
    coeffs = np.ascontiguousarray(coeffs, dtype=np.int16)
    q = np.ascontiguousarray(q, dtype=np.int32)
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    if not lib.gb200_write_jpeg(coeffs.ctypes.data, w, h, q.ctypes.data, C.byref(out), C.byref(out_len)):
        raise RuntimeError(_err(lib))
    return _take(lib, out, out_len)


class DeviceImage(_Handle):
    """One image resident on one GPU (gb200_image_*): the reference's Comparator /
    OutputImage pair moved onto device memory.  Used by the parity tests."""

    _destroy = "gb200_image_destroy"

    def __init__(self, rgb, device=0, lib=None, prepare=True):
        self.lib = lib or load_library()
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        self.h, self.w, _ = rgb.shape
        self._h = self.lib.gb200_image_create2(rgb.ctypes.data, self.w, self.h, device, int(prepare))
        if not self._h:
            raise RuntimeError("gb200_image_create failed: " + _err(self.lib))
        self.nblocks = self.lib.gb200_image_num_blocks(self._h)

    @classmethod
    def from_image(cls, image, device=0, prepare=True, lib=None):
        """A resident image made from an 8-bit image of any channel count and layout, converted to RGB on the
        device as process_image converts it.  A CUDA tensor is read in place on its own device after the work
        queued on that device's current torch stream; host memory goes to `device`.  The image has been read
        when this returns, so the caller may overwrite it right away."""
        self = cls.__new__(cls)
        self.lib = lib or load_library()
        ptr, self.w, self.h, ch, strides, dev, _owner = _image_view(image)
        if dev is not None:
            import torch
            self._h = self.lib.gb200_image_create_device(ptr, self.w, self.h, ch, strides.ctypes.data, dev.index,
                                                         int(prepare), torch.cuda.current_stream(dev).cuda_stream)
        else:
            self._h = self.lib.gb200_image_create_strided(ptr, self.w, self.h, ch, strides.ctypes.data, device,
                                                          int(prepare))
        if not self._h:
            raise RuntimeError("gb200_image_create failed: " + _err(self.lib))
        self.nblocks = self.lib.gb200_image_num_blocks(self._h)
        return self

    def rgb(self):
        """The resident image's RGB as the encoder sees it, uint8 [h][w][3]."""
        out = np.empty((self.h, self.w, 3), dtype=np.uint8)
        self._ck(self.lib.gb200_image_rgb(self._h, out.ctypes.data))
        return out

    def reset(self):
        """Forget the one-time results: the next process() repeats the whole job."""
        self._ck(self.lib.gb200_image_reset(self._h))

    def process(self, params, stats=None):
        """guetzli::Process on the resident image -> (ok, jpeg bytes)."""
        cp, cs = _cparams(params), _CStats()
        out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
        ok = self.lib.gb200_image_process(self._h, C.byref(cp), C.cast(None, _LOG_FN), None,
                                          C.byref(out), C.byref(out_len), C.byref(cs))
        data = _take(self.lib, out, out_len)
        _fill_stats(stats, cs)
        if not ok and not data:
            raise RuntimeError("gb200_image_process failed: " + _err(self.lib))
        return bool(ok), data

    def orig_coeffs(self):
        out = np.zeros((3, self.nblocks, 64), dtype=np.int16)
        self._ck(self.lib.gb200_image_orig_coeffs(self._h, out.ctypes.data))
        return out

    def apply_global_quant(self, q):
        q = np.ascontiguousarray(q, dtype=np.int32)
        self._ck(self.lib.gb200_image_apply_global_quant(self._h, q.ctypes.data))

    def upload_candidate(self, coeffs):
        c = np.ascontiguousarray(coeffs, dtype=np.int16)
        self._ck(self.lib.gb200_image_upload_candidate(self._h, c.ctypes.data))

    def download_candidate(self):
        out = np.zeros((3, self.nblocks, 64), dtype=np.int16)
        self._ck(self.lib.gb200_image_download_candidate(self._h, out.ctypes.data))
        return out

    def scatter(self, index, value):
        i = np.ascontiguousarray(index, dtype=np.int32)
        v = np.ascontiguousarray(value, dtype=np.int16)
        self._ck(self.lib.gb200_image_scatter(self._h, i.ctypes.data, v.ctypes.data, len(i)))

    def save_jpeg(self, q):
        """SaveToJpegData + WriteJpeg of the current candidate, entropy-coded and assembled on the device."""
        q = np.ascontiguousarray(q, dtype=np.int32)
        out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
        self._ck(self.lib.gb200_image_save_jpeg(self._h, q.ctypes.data, C.byref(out), C.byref(out_len)))
        return _take(self.lib, out, out_len)

    def compare(self):
        d = C.c_float()
        self._ck(self.lib.gb200_image_compare(self._h, C.byref(d)))
        return d.value

    def distmap(self):
        out = np.zeros((self.h, self.w), dtype=np.float32)
        self._ck(self.lib.gb200_image_distmap(self._h, out.ctypes.data))
        return out

    def block_weights(self, direction, radius, target_distance, zero_distmap=False):
        out = np.zeros(self.nblocks, dtype=np.float32)
        self._ck(self.lib.gb200_image_block_weights(self._h, direction, radius, float(target_distance),
                                                    int(zero_distmap), out.ctypes.data))
        return out

    def zeroing_orders(self, block_error_limit, lookahead=3):
        idx = np.zeros((self.nblocks, 192), dtype=np.uint8)
        err = np.zeros((self.nblocks, 192), dtype=np.float32)
        cnt = np.zeros(self.nblocks, dtype=np.int32)
        self._ck(self.lib.gb200_image_zeroing_orders(self._h, C.c_float(block_error_limit), lookahead,
                                                     idx.ctypes.data, err.ctypes.data, cnt.ctypes.data))
        return idx, err, cnt

    def debug_blur(self, plane, blur_id):
        a = np.ascontiguousarray(plane, dtype=np.float32)
        out = np.zeros_like(a)
        self._ck(self.lib.gb200_image_debug_blur(self._h, a.ctypes.data, out.ctypes.data, blur_id))
        return out

    def debug_opsin(self, rgb_lin):
        a = np.ascontiguousarray(rgb_lin, dtype=np.float32)
        out = np.zeros_like(a)
        self._ck(self.lib.gb200_image_debug_opsin(self._h, a.ctypes.data, out.ctypes.data))
        return out

    def debug_separate(self, xyb):
        a = np.ascontiguousarray(xyb, dtype=np.float32)
        out = np.zeros((10, self.h, self.w), dtype=np.float32)
        self._ck(self.lib.gb200_image_debug_separate(self._h, a.ctypes.data, out.ctypes.data))
        return out

    def debug_render(self):
        out = np.zeros((3, self.h, self.w), dtype=np.float32)
        self._ck(self.lib.gb200_image_debug_render(self._h, out.ctypes.data))
        return out

    def debug_psycho0(self):
        out = np.zeros((10, self.h, self.w), dtype=np.float32)
        self._ck(self.lib.gb200_image_debug_psycho0(self._h, out.ctypes.data))
        return out

    def debug_corner_mask(self):
        out = np.zeros((self.nblocks, 3), dtype=np.float32)
        self._ck(self.lib.gb200_image_debug_corner_mask(self._h, out.ctypes.data))
        return out
