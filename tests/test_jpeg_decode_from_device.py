"""JPEG files held in CUDA memory (gb.decode_jpeg on torch tensors, gb200_jpeg_decode_rgb_from_device): the
header read from a prefix on the host, the Huffman decoding of sequential scans on the device.

On the CPU port, the device path's entropy decoding (gb200_debug_entropy_decode: segment pass, speculative
decode with subsequences of S bits, DC prefix sums) is pinned against read_jpeg's coefficients on every
fixture, on Pillow-written files and on damaged files.  On the GPU, pixels against libjpeg-turbo's
(tests/test_jpeg_decode.py's goldens) and against the host-bytes entry, refusals, the path each file
takes, and the argument checks."""
import ctypes as C
import io
import threading

import numpy as np
import pytest

import guetzli_b200 as gb
from guetzli_b200 import synth
from test_jpeg_decode import ACCEPTED, REFUSED, check_pixels, data

S_DEFAULT = 1024  # kJpegSubBits, pipeline.h
SIZES = [S_DEFAULT, 64, 33, 8]


def progressive(b):
    """SOF2 before the first SOS"""
    sos = b.find(b"\xff\xda")
    return b.find(b"\xff\xc2", 0, sos) >= 0


def check_hook(lib, b, S, name="", cap=1 << 24):
    """The hook either gives read_jpeg's coefficients or sends the file to the host path -> taken"""
    taken, coeffs = gb.api.entropy_decode(b, S, lib=lib, cap=cap)
    if taken:
        ok, _, want = gb.api.read_jpeg(b, lib=lib, cap=cap)
        assert ok, f"{name} S={S}: the device path took a file read_jpeg refuses"
        assert np.array_equal(coeffs[:want.size], want), f"{name} S={S}: coefficients differ from read_jpeg's"
        assert not coeffs[want.size:want.size + 4096].any(), f"{name} S={S}: written beyond the coefficients"
    return taken


def pillow(h, w, sub, q, seed=1, gray=False, **kw):
    from PIL import Image
    rgb = synth.gradnoise(h, w, seed)
    img = Image.fromarray(rgb).convert("L") if gray else Image.fromarray(rgb)
    b = io.BytesIO()
    if gray:
        img.save(b, "JPEG", quality=q, **kw)
    else:
        img.save(b, "JPEG", quality=q, subsampling=sub, **kw)
    return b.getvalue()


PILLOW_CASES = [(h, w, sub, q, kw)
                for (h, w) in [(1, 1), (7, 13), (17, 9), (33, 47), (65, 40)]
                for sub in (0, 1, 2, "gray")
                for q, kw in [(50, {}), (75, {"restart_marker_blocks": 1}), (90, {"restart_marker_blocks": 3}),
                              (95, {"restart_marker_blocks": 64}), (100, {"restart_marker_rows": 1})]]


def pillow_case(h, w, sub, q, kw):
    return pillow(h, w, 0 if sub == "gray" else sub, q, seed=h * 131 + w, gray=sub == "gray", **kw)


def shared_tables_444(h, w, q=90, **kw):
    """A 4:4:4 file whose components all use DHT tables 0 / 0 (synth.jpeg_gray_as_444 of a Pillow gray file)"""
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(synth.flat_blocks_gray(h, 3 * w, w + h)).save(b, "JPEG", quality=q, **kw)
    return synth.jpeg_gray_as_444(b.getvalue(), w, h)


# ---- CPU port --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("S", SIZES)
def test_port_hook_fixtures(port_lib, S):
    for name in ACCEPTED:
        b = data(name)
        taken = check_hook(port_lib, b, S, name)
        assert taken == (not progressive(b)), name


@pytest.mark.parametrize("S", SIZES)
def test_port_hook_refused_fixtures(port_lib, S):
    for name in sorted(REFUSED):
        check_hook(port_lib, data(name), S, name)


@pytest.mark.parametrize("S", [S_DEFAULT, 33])
def test_port_hook_pillow_files(port_lib, S):
    pytest.importorskip("PIL.Image", reason="Pillow writes the files")
    for case in PILLOW_CASES:
        assert check_hook(port_lib, pillow_case(*case), S, str(case)), case


@pytest.mark.parametrize("S", [S_DEFAULT, 33])
def test_port_hook_shared_tables(port_lib, S):
    """every block of the MCU decodes with the same tables, so the bits cannot tell which slot a guess is in"""
    pytest.importorskip("PIL.Image", reason="Pillow writes the files")
    for h, w, kw in [(256, 256, {}), (512, 768, {}), (64, 48, {"restart_marker_blocks": 6})]:
        assert check_hook(port_lib, shared_tables_444(h, w, **kw), S, f"{w}x{h}"), (w, h)


def damaged(b):
    """b cut at every byte after the SOS header, and with single bytes of its scan data changed"""
    sos = b.find(b"\xff\xda")
    start = sos + 2 + ((b[sos + 2] << 8) | b[sos + 3])
    for k in range(start, len(b)):
        yield b[:k]
    for k in range(start, len(b) - 2):
        for x in (0x01, 0x80, 0xff):
            v = bytearray(b)
            v[k] ^= x
            yield bytes(v)


@pytest.mark.parametrize("name", ["jpeg/tiny444", "jpeg/sub420"])
def test_port_hook_damaged_files(port_lib, name):
    taken = 0
    for i, b in enumerate(damaged(data(name))):
        taken += check_hook(port_lib, b, 33 if i % 2 else S_DEFAULT, f"{name} variant {i}")
    assert taken > 0


def test_port_from_device_entry_refuses(port_lib):
    d = np.frombuffer(data("jpeg/tiny444"), np.uint8)
    out = np.zeros((24, 40, 3), np.uint8)
    w, h = (C.c_int * 1)(40), (C.c_int * 1)(24)
    ok = port_lib.gb200_jpeg_decode_rgb_from_device((C.c_void_p * 1)(d.ctypes.data), (C.c_size_t * 1)(d.size), 1, 0,
                                                   w, h, (C.c_void_p * 1)(out.ctypes.data), None)
    assert not ok and "no device memory" in gb.last_error(lib=port_lib)


def test_port_tensor_arguments(port_lib):
    torch = pytest.importorskip("torch")
    t = torch.frombuffer(bytearray(data("jpeg/tiny444")), dtype=torch.uint8)
    with pytest.raises(ValueError, match="mixes host bytes and torch tensors"):
        gb.decode_jpeg([data("jpeg/tiny444"), t], lib=port_lib)
    with pytest.raises(ValueError, match="cuda=False takes host bytes only"):
        gb.decode_jpeg([t], cuda=False, lib=port_lib)


# ---- on the GPU ------------------------------------------------------------------------------------------

def on_device(b, dev="cuda:0"):
    import torch
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)


@pytest.mark.gpu
def test_cuda_pixels(cuda_lib):
    for name in ACCEPTED:
        px = gb.decode_jpeg(on_device(data(name)), lib=cuda_lib)
        check_pixels(name, px.cpu().numpy())


@pytest.mark.gpu
def test_cuda_one_mixed_call(cuda_lib):
    out = gb.decode_jpeg([on_device(data(n)) for n in ACCEPTED], lib=cuda_lib)
    for n, px in zip(ACCEPTED, out):
        check_pixels(n, px.cpu().numpy())


def raw_from_device(lib, files, shapes, sentinel=None):
    """gb200_jpeg_decode_rgb_from_device on CUDA tensors -> (ok, outputs)"""
    import torch
    n = len(files)
    out = [torch.full(s, 77 if sentinel is None else sentinel, dtype=torch.uint8, device="cuda:0") for s in shapes]
    ok = lib.gb200_jpeg_decode_rgb_from_device(
        (C.c_void_p * n)(*[f.data_ptr() for f in files]), (C.c_size_t * n)(*[f.numel() for f in files]), n, 0,
        (C.c_int * n)(*[s[1] for s in shapes]), (C.c_int * n)(*[s[0] for s in shapes]),
        (C.c_void_p * n)(*[o.data_ptr() for o in out]), torch.cuda.current_stream().cuda_stream)
    return ok, out


@pytest.mark.gpu
def test_cuda_refusals(cuda_lib):
    good = data("jpeg/base444_q90")
    for name in sorted(REFUSED):
        with pytest.raises(ValueError) as host:
            gb.decode_jpeg([good, data(name)], cuda=False, lib=cuda_lib)
        reason = str(host.value).split(": file 1: ", 1)[1]
        with pytest.raises(ValueError) as dev:
            gb.decode_jpeg([on_device(good), on_device(data(name))], lib=cuda_lib)
        assert str(dev.value) == "jpeg_decode_rgb_from_device: file 1: " + reason, name
        # outputs filled beforehand stay as they were
        shapes = []
        for f in (good, data(name)):
            w, h = C.c_int(), C.c_int()
            b = np.frombuffer(f, np.uint8)
            ok = cuda_lib.gb200_jpeg_dimensions(b.ctypes.data, b.size, C.byref(w), C.byref(h))
            shapes.append((h.value, w.value, 3) if ok else (1, 1, 3))
        ok, out = raw_from_device(cuda_lib, [on_device(good), on_device(data(name))], shapes, 201)
        assert not ok and gb.last_error(lib=cuda_lib) == str(dev.value), name
        assert all(bool((o == 201).all()) for o in out), name


@pytest.mark.gpu
def test_cuda_path_taken(cuda_lib):
    for name in ACCEPTED:
        b = data(name)
        _, _, d0 = gb.counters(lib=cuda_lib)
        gb.decode_jpeg(on_device(b), lib=cuda_lib)
        _, _, d1 = gb.counters(lib=cuda_lib)
        sos = b.find(b"\xff\xda")
        prefix = 4096
        while prefix < sos + 64 and prefix < len(b):
            prefix *= 2
        prefix = min(prefix, len(b))
        if progressive(b):
            assert d1 - d0 >= len(b), name
        else:
            # the header prefix (once for the frame size, once for the header), then status words: one per
            # synchronisation round (64 at most) and two per file; the host path would add len(b), which
            # tells the two apart for every file longer than MAX_STATUS_BYTES
            assert d1 - d0 <= 2 * prefix + MAX_STATUS_BYTES, (name, d1 - d0, prefix)


MAX_STATUS_BYTES = 4 * (64 + 2)


def device_path_d2h(lib, b):
    """decode_jpeg from CUDA memory -> (pixels, bytes copied back)"""
    _, _, d0 = gb.counters(lib=lib)
    px = gb.decode_jpeg(on_device(b), lib=lib).cpu().numpy()
    _, _, d1 = gb.counters(lib=lib)
    return px, d1 - d0


def large_files():
    for h, w in [(1080, 1920), (3000, 4000)]:
        for sub in (2, 0):
            for kw in ({}, {"restart_marker_blocks": 4}):
                yield f"{w}x{h}_{sub}_{kw}", pillow(h, w, sub, 90, seed=w + sub, **kw)


@pytest.mark.gpu
def test_cuda_large_files(cuda_lib):
    pytest.importorskip("PIL.Image", reason="Pillow writes the files")
    for name, b in large_files():
        want = gb.decode_jpeg(b, cuda=False, lib=cuda_lib)
        got, d2h = device_path_d2h(cuda_lib, b)
        assert np.array_equal(got, want), name
        assert d2h <= 2 * 4096 + MAX_STATUS_BYTES, (name, d2h)  # the device path, not a copy of the file
        for S in (S_DEFAULT, 33):
            assert check_hook(cuda_lib, b, S, name, cap=1 << 26), name


@pytest.mark.gpu
def test_cuda_shared_tables(cuda_lib):
    pytest.importorskip("PIL.Image", reason="Pillow writes the files")
    for h, w in [(256, 256), (512, 768), (1080, 1920), (3000, 4000)]:
        b = shared_tables_444(h, w)
        want = gb.decode_jpeg(b, cuda=False, lib=cuda_lib)
        got, d2h = device_path_d2h(cuda_lib, b)
        assert np.array_equal(got, want), (w, h)
        assert d2h <= 2 * 4096 + MAX_STATUS_BYTES, (w, h, d2h)
        assert check_hook(cuda_lib, b, S_DEFAULT, f"{w}x{h}", cap=1 << 26), (w, h)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["jpeg/tiny444", "jpeg/sub420"])
def test_cuda_damaged_files(cuda_lib, name):
    for i, b in enumerate(damaged(data(name))):
        try:
            want = gb.decode_jpeg(b, cuda=False, lib=cuda_lib)
        except ValueError as e:
            want = str(e).split(": file 0: ", 1)[1]
        try:
            got = gb.decode_jpeg(on_device(b), lib=cuda_lib).cpu().numpy()
        except ValueError as e:
            got = str(e).split(": file 0: ", 1)[1]
        if isinstance(want, str):
            assert got == want, (name, i)
        else:
            assert isinstance(got, np.ndarray) and np.array_equal(got, want), (name, i)


@pytest.mark.gpu
def test_cuda_argument_checks(cuda_lib):
    import torch
    d = on_device(data("jpeg/tiny444"))
    host = np.frombuffer(data("jpeg/tiny444"), np.uint8)
    out = torch.empty((24, 40, 3), dtype=torch.uint8, device="cuda:0")
    ln = (C.c_size_t * 1)(d.numel())
    w, h = (C.c_int * 1)(40), (C.c_int * 1)(24)
    outp = (C.c_void_p * 1)(out.data_ptr())
    before = gb.counters(lib=cuda_lib)
    f = cuda_lib.gb200_jpeg_decode_rgb_from_device
    assert not f((C.c_void_p * 1)(host.ctypes.data), ln, 1, 0, w, h, outp, None)
    assert "jpeg[0] is not device memory of device 0" in gb.last_error(lib=cuda_lib)
    assert not f((C.c_void_p * 1)(d.data_ptr()), ln, 1, 0, w, h, (C.c_void_p * 1)(host.ctypes.data), None)
    assert "out[0] is not device memory of device 0" in gb.last_error(lib=cuda_lib)
    assert not f((C.c_void_p * 1)(d.data_ptr()), ln, 0, 0, w, h, outp, None)
    assert "n must be at least 1" in gb.last_error(lib=cuda_lib)
    assert not f(None, ln, 1, 0, w, h, outp, None)
    assert "must not be null" in gb.last_error(lib=cuda_lib)
    assert not f((C.c_void_p * 1)(d.data_ptr()), ln, 1, 0, None, h, outp, None)
    assert "must not be null" in gb.last_error(lib=cuda_lib)
    assert not f((C.c_void_p * 1)(None), ln, 1, 0, w, h, outp, None)
    assert "jpeg[0] is null" in gb.last_error(lib=cuda_lib)
    assert not f((C.c_void_p * 1)(d.data_ptr()), ln, 1, 0, w, h, (C.c_void_p * 1)(None), None)
    assert "out[0] is null" in gb.last_error(lib=cuda_lib)
    assert gb.counters(lib=cuda_lib) == before
    # a wrong size is refused before anything is written
    out.fill_(9)
    assert not f((C.c_void_p * 1)(d.data_ptr()), ln, 1, 0, (C.c_int * 1)(39), h, outp, None)
    assert "file 0: the output is 39x24, the frame 40x24" in gb.last_error(lib=cuda_lib)
    assert bool((out == 9).all())
    sizes = (C.c_int * 1)(), (C.c_int * 1)()
    assert cuda_lib.gb200_jpeg_dimensions_from_device((C.c_void_p * 1)(d.data_ptr()), ln, 1, 0, None, *sizes)
    assert (sizes[0][0], sizes[1][0]) == (40, 24)
    g = on_device(b"\x00\x01\x02")
    assert cuda_lib.gb200_jpeg_dimensions_from_device((C.c_void_p * 1)(g.data_ptr()), (C.c_size_t * 1)(3), 1, 0,
                                                      None, *sizes)
    assert (sizes[0][0], sizes[1][0]) == (0, 0)
    with pytest.raises(ValueError, match="more than one device|cuda=False"):
        gb.decode_jpeg([d], cuda=False, lib=cuda_lib)


@pytest.mark.gpu
def test_cuda_stream_order(cuda_lib):
    import torch
    names = ["jpeg/sub420", "jpeg/base444_q90", "jpeg/gray", "jpeg/prog444_q85"]
    pinned = [torch.frombuffer(bytearray(data(n)), dtype=torch.uint8).pin_memory() for n in names]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        for _ in range(3):
            dst = [torch.zeros(p.numel(), dtype=torch.uint8, device="cuda:0") for p in pinned]
            torch.cuda._sleep(2_000_000)  # the copies below wait behind this on the side stream
            for t, p in zip(dst, pinned):
                t.copy_(p, non_blocking=True)
            out = gb.decode_jpeg(dst, lib=cuda_lib)
            for n, px in zip(names, out):
                check_pixels(n, px.cpu().numpy())


@pytest.mark.gpu
def test_cuda_two_threads(cuda_lib):
    names = ACCEPTED[::3]
    errors = []

    def run(seq):
        try:
            for _ in range(3):
                for n, px in zip(seq, gb.decode_jpeg([on_device(data(n)) for n in seq], lib=cuda_lib)):
                    check_pixels(n, px.cpu().numpy())
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=run, args=(names,)), threading.Thread(target=run, args=(names[::-1],))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors[0]
