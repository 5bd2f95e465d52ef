"""ctypes bindings for oracle/_ref/libguetzli_ref.so (the unmodified reference,
test infrastructure only).  See oracle/ref_hooks.cc for what each hook wraps.

Where oracle/_ref is not built (its sources are not part of this repository), replay()
switches every call below to the reference's recorded answers, golden/reference_answers.json:
per call, the sha256 of its arguments -> its scalar results as they are and the sha256 of its
arrays, bytes and text (Digest, compared with ==, parity.same or parity.bits_equal).  A call
whose arguments were never recorded fails.  GB200_REF_RECORD=<file> records the calls a live
run makes (tests/golden/make_reference_answers.sh)."""
import atexit
import ctypes as C
import functools
import hashlib
import inspect
import json
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "..", "oracle", "_ref", "libguetzli_ref.so")
ANSWERS = os.path.join(_HERE, "golden", "reference_answers.json")
_lib = None
_answers = None  # replay mode: key -> recorded result
_recorded = None  # recording: key -> result


def available():
    """True when the live reference library is built."""
    return os.path.exists(REF_SO)


def replay():
    """Answers from golden/reference_answers.json instead of the live library."""
    global _answers
    if _answers is None:
        with open(ANSWERS) as f:
            _answers = json.load(f)


def _h(data):
    return hashlib.sha256(data).hexdigest()[:32]


class Digest:
    """A recorded array, bytes or text, known by its sha256 (truncated to 128 bits)."""

    def __init__(self, d):
        self.sha256, self.kind = d["sha256"], d["kind"]
        self.dtype, self.shape = d.get("dtype"), tuple(d.get("shape", ()))

    def matches(self, x):
        if self.kind == "bytes":
            return isinstance(x, (bytes, bytearray)) and _h(bytes(x)) == self.sha256
        if self.kind == "str":
            return isinstance(x, str) and _h(x.encode()) == self.sha256
        a = np.asarray(x)
        if a.shape != self.shape:
            return False
        b = a.astype(self.dtype)
        return np.array_equal(b.astype(a.dtype), a) and _h(np.ascontiguousarray(b).tobytes()) == self.sha256

    def __eq__(self, other):
        return self.matches(other)

    __hash__ = None

    def __repr__(self):
        return f"Digest({self.kind} {self.dtype or ''}{list(self.shape) if self.kind == 'array' else ''} {self.sha256})"


def _encode(x):
    if isinstance(x, (tuple, list)):
        return [_encode(v) for v in x]
    if isinstance(x, np.ndarray):
        return {"sha256": _h(np.ascontiguousarray(x).tobytes()), "kind": "array", "dtype": x.dtype.str,
                "shape": list(x.shape)}
    if isinstance(x, (bytes, bytearray)):
        return {"sha256": _h(bytes(x)), "kind": "bytes"}
    if isinstance(x, str):
        return {"sha256": _h(x.encode()), "kind": "str"}
    if isinstance(x, (bool, np.bool_)):
        return bool(x)
    if isinstance(x, (int, np.integer)):
        return int(x)
    return float(x)


def _decode(x):
    if isinstance(x, list):
        return [_decode(v) for v in x]
    return Digest(x) if isinstance(x, dict) else x


def sha256_matches(x, hexdigest):
    """sha256(x) == hexdigest for bytes or text, live or recorded."""
    if isinstance(x, Digest):
        return hexdigest.startswith(x.sha256)
    return hashlib.sha256(x.encode() if isinstance(x, str) else x).hexdigest() == hexdigest


def _arg_bytes(v):
    if isinstance(v, np.ndarray):
        return b"A%s%s" % (v.dtype.str.encode(), str(v.shape).encode()) + np.ascontiguousarray(v).tobytes()
    if isinstance(v, (bytes, bytearray)):
        return b"B" + bytes(v)
    if isinstance(v, (list, tuple)):
        return b"L" + b"".join(_arg_bytes(u) for u in v)
    if isinstance(v, (bool, np.bool_)):
        return b"b%d" % bool(v)
    if isinstance(v, (int, np.integer)):
        return b"i%d" % int(v)
    if isinstance(v, (float, np.floating)):
        return b"f" + repr(float(v)).encode()
    raise TypeError(f"cannot key an argument of type {type(v).__name__}")


def _save_recorded():
    path = os.environ["GB200_REF_RECORD"]
    old = json.load(open(path)) if os.path.exists(path) else {}
    old.update(_recorded)
    with open(path, "w") as f:  # one call per line
        f.write("{\n" + ",\n".join(json.dumps(k) + ":" + json.dumps(old[k], separators=(",", ":"))
                                    for k in sorted(old)) + "\n}\n")


def _answered(fn):
    sig = inspect.signature(fn)

    @functools.wraps(fn)
    def call(*args, **kwargs):
        global _recorded
        b = sig.bind(*args, **kwargs)
        b.apply_defaults()
        key = fn.__name__ + ":" + _h(b"".join(k.encode() + b"=" + _arg_bytes(v) for k, v in b.arguments.items()))
        if _answers is not None:
            if key not in _answers:
                raise LookupError(f"no recorded reference answer for {fn.__name__} with these arguments "
                                  "(tests/golden/reference_answers.json); build oracle/_ref to run it live")
            return _decode(_answers[key])
        out = fn(*args, **kwargs)
        if os.environ.get("GB200_REF_RECORD"):
            if _recorded is None:
                _recorded = {}
                atexit.register(_save_recorded)
            _recorded[key] = _encode(out)
        return out
    return call


def lib():
    global _lib
    if _answers is not None:
        raise RuntimeError("reflib: replaying recorded answers; the live reference library is not loaded")
    if _lib is None:
        _lib = C.CDLL(REF_SO)
        _lib.gref_target_for_quality.restype = C.c_double
        _lib.gref_target_for_quality.argtypes = [C.c_double]
        _lib.gref_mask_lut.restype = C.c_double
        _lib.gref_mask_lut.argtypes = [C.c_int, C.c_double]
        _lib.gref_gamma.restype = C.c_double
        _lib.gref_gamma.argtypes = [C.c_double]
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


@_answered
def target_for_quality(q):
    return float(np.float32(lib().gref_target_for_quality(float(q))))


@_answered
def process_rgb(rgb, quality=95.0, trace=True, lookahead=3, new_zeroing_model=True, clear_metadata=True,
                try_420=False, force_420=False):
    """-> (ok, jpeg bytes, trace str, counters[3], seconds)"""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    h, w, _ = rgb.shape
    out = C.POINTER(C.c_uint8)()
    out_len = C.c_size_t()
    tr = C.c_char_p()
    tr_len = C.c_size_t()
    counters = (C.c_int * 3)()
    secs = C.c_double()
    lib().gref_set_clear_metadata(int(clear_metadata))
    lib().gref_set_420(int(try_420), int(force_420))
    try:
        ok = lib().gref_process_rgb_ex(
            _p(rgb, C.c_uint8), w, h, C.c_float(np.float32(lib().gref_target_for_quality(float(quality)))),
            int(lookahead), int(new_zeroing_model), C.byref(out), C.byref(out_len),
            C.byref(tr) if trace else None, C.byref(tr_len), counters, C.byref(secs))
    finally:
        lib().gref_set_clear_metadata(1)
        lib().gref_set_420(0, 0)
    data = C.string_at(out, out_len.value)
    lib().gref_free(out)
    t = ""
    if trace:
        t = C.string_at(tr, tr_len.value).decode()
        lib().gref_free(tr)
    return bool(ok), data, t, list(counters), secs.value


@_answered
def process_jpeg(jpeg_in, quality=95.0, clear_metadata=True, trace=True):
    """guetzli::Process(jpeg bytes) -> (ok, jpeg bytes, trace str, counters[3])"""
    buf = np.frombuffer(bytes(jpeg_in), dtype=np.uint8)
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    tr, tr_len = C.c_char_p(), C.c_size_t()
    counters = (C.c_int * 3)()
    ok = lib().gref_process_jpeg(_p(buf, C.c_uint8), C.c_size_t(buf.size), C.c_float(target_for_quality(quality)),
                                 int(clear_metadata), C.byref(out), C.byref(out_len),
                                 C.byref(tr) if trace else None, C.byref(tr_len), counters)
    data = C.string_at(out, out_len.value)
    lib().gref_free(out)
    t = ""
    if trace:
        t = C.string_at(tr, tr_len.value).decode()
        lib().gref_free(tr)
    return bool(ok), data, t, list(counters)


@_answered
def read_jpeg(jpeg_in):
    """ReadJpeg(JPEG_READ_ALL) -> (ok, dims, quantised coefficients of all components, concatenated)"""
    buf = np.frombuffer(bytes(jpeg_in), dtype=np.uint8)
    dims = (C.c_int * 11)()
    cap = 1 << 24
    out = np.zeros(cap, dtype=np.int16)
    ok = lib().gref_read_jpeg(_p(buf, C.c_uint8), C.c_size_t(buf.size), dims, _p(out, C.c_int16), C.c_size_t(cap))
    d = list(dims)
    n = sum(d[3 + 2 * c] * d[4 + 2 * c] * 64 for c in range(d[2])) if ok else 0
    return bool(ok), d, out[:n].copy()


@_answered
def butteraugli_interface(rgb0, rgb1):
    """butteraugli::ButteraugliInterface on planar linear float32 [3][h][w] -> (diffmap, score)"""
    a = np.ascontiguousarray(rgb0, dtype=np.float32)
    b = np.ascontiguousarray(rgb1, dtype=np.float32)
    _, h, w = a.shape
    dm = np.zeros((h, w), dtype=np.float32)
    score = C.c_double()
    assert lib().gref_butteraugli_interface(_p(a, C.c_float), _p(b, C.c_float), w, h, _p(dm, C.c_float), C.byref(score))
    return dm, score.value


def nblocks(w, h):
    return ((w + 7) // 8) * ((h + 7) // 8)


@_answered
def rgb_to_coeffs(rgb):
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    h, w, _ = rgb.shape
    out = np.zeros((3, nblocks(w, h), 64), dtype=np.int16)
    assert lib().gref_rgb_to_coeffs(_p(rgb, C.c_uint8), w, h, _p(out, C.c_int16))
    return out


@_answered
def idct_block(block):
    block = np.ascontiguousarray(block, dtype=np.int16)
    out = np.zeros(64, dtype=np.uint8)
    lib().gref_idct_block(_p(block, C.c_int16), _p(out, C.c_uint8))
    return out


@_answered
def fdct_block(block):
    block = np.array(block, dtype=np.int16).copy()
    lib().gref_fdct_block(_p(block, C.c_int16))
    return block


@_answered
def render(coeffs, w, h):
    coeffs = np.ascontiguousarray(coeffs, dtype=np.int16)
    srgb = np.zeros((h, w, 3), dtype=np.uint8)
    lin = np.zeros((3, h, w), dtype=np.float32)
    lib().gref_render(_p(coeffs, C.c_int16), w, h, _p(srgb, C.c_uint8), _p(lin, C.c_float))
    return srgb, lin


@_answered
def apply_global_quant(coeffs, w, h, q):
    coeffs = np.ascontiguousarray(coeffs, dtype=np.int16)
    q = np.ascontiguousarray(q, dtype=np.int32)
    out = np.zeros_like(coeffs)
    lib().gref_apply_global_quant(_p(coeffs, C.c_int16), w, h, _p(q, C.c_int32), _p(out, C.c_int16))
    return out


@_answered
def blur(img, sigma, border_ratio):
    img = np.ascontiguousarray(img, dtype=np.float32)
    h, w = img.shape
    out = np.zeros_like(img)
    lib().gref_blur(_p(img, C.c_float), w, h, C.c_float(sigma), C.c_float(border_ratio), _p(out, C.c_float))
    return out


@_answered
def opsin(rgb_planes):
    a = np.ascontiguousarray(rgb_planes, dtype=np.float32)
    _, h, w = a.shape
    out = np.zeros_like(a)
    lib().gref_opsin(_p(a, C.c_float), w, h, _p(out, C.c_float))
    return out


@_answered
def separate(xyb):
    a = np.ascontiguousarray(xyb, dtype=np.float32)
    _, h, w = a.shape
    out = np.zeros((10, h, w), dtype=np.float32)
    lib().gref_separate(_p(a, C.c_float), w, h, _p(out, C.c_float))
    return out


@_answered
def malta(lum0, lum1, w_0gt1, w_0lt1, norm1, lf, acc=None):
    a = np.ascontiguousarray(lum0, dtype=np.float32)
    b = np.ascontiguousarray(lum1, dtype=np.float32)
    h, w = a.shape
    out = np.zeros_like(a) if acc is None else np.array(acc, dtype=np.float32).copy()
    lib().gref_malta(_p(a, C.c_float), _p(b, C.c_float), w, h, C.c_double(w_0gt1),
                     C.c_double(w_0lt1), C.c_double(norm1), int(lf), _p(out, C.c_float))
    return out


@_answered
def mask(xyb0, xyb1):
    a = np.ascontiguousarray(xyb0, dtype=np.float32)
    b = np.ascontiguousarray(xyb1, dtype=np.float32)
    _, h, w = a.shape
    m = np.zeros_like(a)
    mdc = np.zeros_like(a)
    lib().gref_mask(_p(a, C.c_float), _p(b, C.c_float), w, h, _p(m, C.c_float), _p(mdc, C.c_float))
    return m, mdc


@_answered
def diffmap(rgb0_lin, rgb1_lin):
    a = np.ascontiguousarray(rgb0_lin, dtype=np.float32)
    b = np.ascontiguousarray(rgb1_lin, dtype=np.float32)
    _, h, w = a.shape
    out = np.zeros((h, w), dtype=np.float32)
    lib().gref_diffmap(_p(a, C.c_float), _p(b, C.c_float), w, h, _p(out, C.c_float))
    return out


@_answered
def compare_coeffs(rgb, coeffs, target):
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    h, w, _ = rgb.shape
    coeffs = np.ascontiguousarray(coeffs, dtype=np.int16)
    dm = np.zeros((h, w), dtype=np.float32)
    dist = C.c_float()
    lib().gref_compare_coeffs(_p(rgb, C.c_uint8), w, h, C.c_float(target),
                              _p(coeffs, C.c_int16), _p(dm, C.c_float), C.byref(dist))
    return dm, dist.value


@_answered
def block_mask(rgb):
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    h, w, _ = rgb.shape
    out = np.zeros((3, h, w), dtype=np.float32)
    lib().gref_block_mask(_p(rgb, C.c_uint8), w, h, _p(out, C.c_float))
    return out


@_answered
def zeroing_orders(rgb, orig_coeffs, q, target):
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    h, w, _ = rgb.shape
    nb = nblocks(w, h)
    coeffs = np.ascontiguousarray(orig_coeffs, dtype=np.int16)
    q = np.ascontiguousarray(q, dtype=np.int32)
    offs = np.zeros(nb + 1, dtype=np.int32)
    idx = np.zeros(189 * nb, dtype=np.uint8)
    err = np.zeros(189 * nb, dtype=np.float32)
    n = lib().gref_zeroing_orders(_p(rgb, C.c_uint8), w, h, C.c_float(target),
                                  _p(coeffs, C.c_int16), _p(q, C.c_int32),
                                  _p(offs, C.c_int32), _p(idx, C.c_uint8), _p(err, C.c_float))
    return offs, idx[:n].copy(), err[:n].copy()


@_answered
def block_weights(w, h, target, direction, rblock, target_mul, distmap):
    d = np.ascontiguousarray(distmap, dtype=np.float32)
    out = np.zeros(nblocks(w, h), dtype=np.float32)
    lib().gref_block_weights(w, h, C.c_float(target), direction, rblock,
                             C.c_double(target_mul), _p(d, C.c_float), _p(out, C.c_float))
    return out


@_answered
def write_jpeg(coeffs, w, h, q):
    coeffs = np.ascontiguousarray(coeffs, dtype=np.int16)
    q = np.ascontiguousarray(q, dtype=np.int32)
    out = C.POINTER(C.c_uint8)()
    out_len = C.c_size_t()
    assert lib().gref_write_jpeg(_p(coeffs, C.c_int16), w, h, _p(q, C.c_int32),
                                 C.byref(out), C.byref(out_len))
    data = C.string_at(out, out_len.value)
    lib().gref_free(out)
    return data


@_answered
def blur_kernel(sigma):
    out = np.zeros(256, dtype=np.float32)
    n = C.c_int()
    lib().gref_blur_kernel(C.c_float(sigma), _p(out, C.c_float), C.byref(n))
    return out[:n.value].copy()


@_answered
def srgb_lut():
    out = np.zeros(256, dtype=np.float64)
    lib().gref_srgb_lut(_p(out, C.c_double))
    return out


@_answered
def color_tables():
    t = [np.zeros(256, dtype=np.int32) for _ in range(4)]
    rl = np.zeros(1024, dtype=np.uint8)
    lib().gref_color_tables(*[_p(x, C.c_int32) for x in t], _p(rl, C.c_uint8))
    return t[0], t[1], t[2], t[3], rl


@_answered
def score_for_quality(q):
    """ButteraugliScoreForQuality in double precision."""
    return float(lib().gref_target_for_quality(float(q)))


@_answered
def butteraugli_heatmap(rgb0, rgb1):
    """ButteraugliInterface, then CreateHeatMapImage of its diffmap -> (heat uint8 [h][w][3], score)"""
    dm, score = butteraugli_interface.__wrapped__(rgb0, rgb1)
    h, w = dm.shape
    heat = np.zeros((h, w, 3), dtype=np.uint8)
    lib().gref_heatmap(_p(dm, C.c_float), w, h, _p(heat, C.c_uint8))
    return heat, score


@_answered
def huffman_depths(counts, limits):
    """CreateHuffmanTree on each row of counts (uint32 [n][257]) with its depth limit -> uint8 [n][257]"""
    counts = np.ascontiguousarray(counts, dtype=np.uint32)
    f = lib().gref_huffman_depths
    f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    f.restype = None
    out = np.zeros(counts.shape, dtype=np.uint8)
    for i in range(counts.shape[0]):
        f(counts[i].ctypes.data, counts.shape[1], int(limits[i]), out[i].ctypes.data)
    return out


@_answered
def block_mask_corners(rgb):
    """block_mask at the top-left pixel of every 8x8 block -> float32 [nblocks][3]"""
    m = block_mask.__wrapped__(rgb)
    return np.ascontiguousarray(np.stack([m[c][::8, ::8].reshape(-1) for c in range(3)], axis=1))
