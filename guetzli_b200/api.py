"""ctypes host mirror of the reference interface for the hot path.

Names and argument meaning follow guetzli/processor.h: ``Params``,
``ProcessStats``, ``Process(params, stats, rgb, w, h, &out)``.  All compute goes
through the C ABI of ``libguetzli_b200.so`` (include/guetzli_b200.h), which is
CUDA-only: importing works anywhere, but calling fails loudly without the built
extension or without a GPU -- there is no CPU fallback in the product.
"""
import ctypes as C
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
    _libs[path] = lib
    return lib


def _err(lib):
    return (lib.gb200_last_error() or b"").decode(errors="replace")


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
    cp = _CParams(params.butteraugli_target, int(params.clear_metadata), int(params.try_420),
                  int(params.force_420), int(params.use_silver_screen),
                  int(params.zeroing_greedy_lookahead), int(params.new_zeroing_model))
    cs = _CStats()
    want_log = stats is not None and (stats.debug_output is not None or stats.debug_output_file is not None)

    def _sink(_user, text):
        s = text.decode(errors="replace")
        if stats.debug_output is not None:
            stats.debug_output.append(s)
        if stats.debug_output_file is not None:
            stats.debug_output_file.write(s)

    cb = _LOG_FN(_sink) if want_log else C.cast(None, _LOG_FN)
    out = C.POINTER(C.c_uint8)()
    out_len = C.c_size_t()
    ok = lib.gb200_process_rgb(C.byref(cp), buf.ctypes.data, w, h, device, cb, None,
                               C.byref(out), C.byref(out_len), C.byref(cs))
    data = C.string_at(out, out_len.value) if out_len.value else b""
    if out:
        lib.gb200_free(out)
    if stats is not None:
        stats.counters["number of iterations"] = cs.iterations
        stats.counters["number of iterations up"] = cs.iterations_up
        stats.counters["number of iterations down"] = cs.iterations_down
        stats.device = {k: getattr(cs, k) for k, _ in _CStats._fields_}
    if not ok and not data:
        msg = _err(lib)
        if "CUDA" in msg or "no CUDA device" in msg or "out of memory" in msg:
            raise RuntimeError(msg)
    return bool(ok), data


def process_jpeg(params, stats, jpeg_in, device=0, lib=None):
    """guetzli::Process(params, stats, jpeg_in, &out) (processor.cc:890): JPEG input
    (4:4:4 YCbCr).  Returns (ok, jpeg_bytes) like process()."""
    lib = lib or load_library()
    buf = np.frombuffer(bytes(jpeg_in), dtype=np.uint8)
    cp, cs = _cparams(params), _CStats()
    want_log = stats is not None and (stats.debug_output is not None or stats.debug_output_file is not None)

    def _sink(_user, text):
        s = text.decode(errors="replace")
        if stats.debug_output is not None:
            stats.debug_output.append(s)
        if stats.debug_output_file is not None:
            stats.debug_output_file.write(s)

    cb = _LOG_FN(_sink) if want_log else C.cast(None, _LOG_FN)
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    ok = lib.gb200_process_jpeg(C.byref(cp), buf.ctypes.data if buf.size else None, buf.size, device, cb, None,
                                C.byref(out), C.byref(out_len), C.byref(cs))
    data = C.string_at(out, out_len.value) if out_len.value else b""
    if out:
        lib.gb200_free(out)
    if stats is not None:
        stats.counters["number of iterations"] = cs.iterations
        stats.counters["number of iterations up"] = cs.iterations_up
        stats.counters["number of iterations down"] = cs.iterations_down
        stats.device = {k: getattr(cs, k) for k, _ in _CStats._fields_}
    if not ok and not data:
        msg = _err(lib)
        if "CUDA" in msg or "no CUDA device" in msg or "out of memory" in msg:
            raise RuntimeError(msg)
    return bool(ok), data


def read_jpeg(jpeg_in, lib=None):
    """ReadJpeg alone (test hook) -> (ok, dims, quantised coefficients concatenated over components)."""
    lib = lib or load_library()
    buf = np.frombuffer(bytes(jpeg_in), dtype=np.uint8)
    dims = (C.c_int * 11)()
    cap = 1 << 24
    out = np.zeros(cap, dtype=np.int16)
    lib.gb200_debug_read_jpeg.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t]
    ok = lib.gb200_debug_read_jpeg(buf.ctypes.data, buf.size, dims, out.ctypes.data, cap)
    d = list(dims)
    n = sum(d[3 + 2 * c] * d[4 + 2 * c] * 64 for c in range(d[2])) if ok else 0
    return bool(ok), d, out[:n].copy()


def butteraugli_diffmap(rgb0, rgb1, device=0, lib=None):
    """butteraugli::ButteraugliInterface: rgb0, rgb1 planar linear RGB float32 [3][h][w] (0..255).
    -> (diffmap [h][w] float32, score)."""
    lib = lib or load_library()
    a = np.ascontiguousarray(rgb0, dtype=np.float32)
    b = np.ascontiguousarray(rgb1, dtype=np.float32)
    assert a.shape == b.shape and a.ndim == 3 and a.shape[0] == 3
    _, h, w = a.shape
    dm = np.zeros((h, w), dtype=np.float32)
    score = C.c_double()
    lib.gb200_butteraugli_diffmap.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                              C.POINTER(C.c_double)]
    if not lib.gb200_butteraugli_diffmap(a.ctypes.data, b.ctypes.data, w, h, device, dm.ctypes.data, C.byref(score)):
        raise RuntimeError(_err(lib))
    return dm, score.value


def counters(lib=None):
    """-> (kernel launches, h2d bytes, d2h bytes): process-wide running totals."""
    lib = lib or load_library()
    n, a, b = C.c_long(), C.c_longlong(), C.c_longlong()
    lib.gb200_counters(C.byref(n), C.byref(a), C.byref(b))
    return n.value, a.value, b.value


def _cparams(params):
    return _CParams(params.butteraugli_target, int(params.clear_metadata), int(params.try_420),
                    int(params.force_420), int(params.use_silver_screen),
                    int(params.zeroing_greedy_lookahead), int(params.new_zeroing_model))


def _take(lib, out, out_len):
    data = C.string_at(out, out_len.value) if out_len.value else b""
    if out:
        lib.gb200_free(out)
    return data


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
    if stats is not None:
        stats.counters["number of iterations"] = cs.iterations
        stats.device = {k: getattr(cs, k) for k, _ in _CStats._fields_}
    if not ok and not data:
        raise RuntimeError(_err(lib))
    return bool(ok), data


def write_jpeg(coeffs, w, h, q, lib=None):
    lib = lib or load_library()
    coeffs = np.ascontiguousarray(coeffs, dtype=np.int16)
    q = np.ascontiguousarray(q, dtype=np.int32)
    out = C.POINTER(C.c_uint8)()
    out_len = C.c_size_t()
    if not lib.gb200_write_jpeg(coeffs.ctypes.data, w, h, q.ctypes.data, C.byref(out), C.byref(out_len)):
        raise RuntimeError(_err(lib))
    data = C.string_at(out, out_len.value)
    lib.gb200_free(out)
    return data


class DeviceImage:
    """One image resident on one GPU (gb200_image_*): the reference's Comparator /
    OutputImage pair moved onto device memory.  Used by the parity tests."""

    def __init__(self, rgb, device=0, lib=None, prepare=True):
        self.lib = lib or load_library()
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        self.h, self.w, _ = rgb.shape
        self._h = self.lib.gb200_image_create2(rgb.ctypes.data, self.w, self.h, device, int(prepare))
        if not self._h:
            raise RuntimeError("gb200_image_create failed: " + _err(self.lib))
        self.nblocks = self.lib.gb200_image_num_blocks(self._h)

    def close(self):
        if self._h:
            self.lib.gb200_image_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def _ck(self, ok):
        if not ok:
            raise RuntimeError(_err(self.lib))

    def reset(self):
        """Forget the one-time results: the next process() repeats the whole job."""
        self._ck(self.lib.gb200_image_reset(self._h))

    def process(self, params, stats=None):
        """guetzli::Process on the resident image -> (ok, jpeg bytes)."""
        cp = _CParams(params.butteraugli_target, int(params.clear_metadata), int(params.try_420),
                      int(params.force_420), int(params.use_silver_screen),
                      int(params.zeroing_greedy_lookahead), int(params.new_zeroing_model))
        cs = _CStats()
        out = C.POINTER(C.c_uint8)()
        out_len = C.c_size_t()
        ok = self.lib.gb200_image_process(self._h, C.byref(cp), C.cast(None, _LOG_FN), None,
                                          C.byref(out), C.byref(out_len), C.byref(cs))
        data = C.string_at(out, out_len.value) if out_len.value else b""
        if out:
            self.lib.gb200_free(out)
        if stats is not None:
            stats.counters["number of iterations"] = cs.iterations
            stats.counters["number of iterations up"] = cs.iterations_up
            stats.counters["number of iterations down"] = cs.iterations_down
            stats.device = {k: getattr(cs, k) for k, _ in _CStats._fields_}
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
        out = C.POINTER(C.c_uint8)()
        out_len = C.c_size_t()
        self._ck(self.lib.gb200_image_save_jpeg(self._h, q.ctypes.data, C.byref(out), C.byref(out_len)))
        data = C.string_at(out, out_len.value)
        self.lib.gb200_free(out)
        return data

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
