"""The encoder on 8-bit images of 1 (gray), 2 (gray + alpha), 3 (RGB) and 4 (RGBA) channels in any strided
layout, from host or CUDA memory (gb.process_image, gb.DeviceImage.from_image, gb200_process_image[_device],
gb200_image_create_strided / _device).  The image is turned into RGB on the device as the guetzli tool turns
PNG layouts into RGB (g/guetzli.cc:43-145), restated here in numpy (to_rgb), so each result is the reference's
guetzli::Process on to_rgb(image), JPEG bytes and --verbose trace.  Every reference call a GPU test makes is
also made by a CPU test with the same arguments, so that recording the CPU tests covers the GPU tests:

    GB200_REF_RECORD=$PWD/tests/golden/image_inputs_reference_answers.json \\
        python -m pytest tests/test_image_inputs.py -m "not gpu"

records them into golden/image_inputs_reference_answers.json, which replay mode reads beside
golden/reference_answers.json."""
import ctypes as C
import hashlib
import json
import os
import threading

import numpy as np
import pytest

import guetzli_b200 as gb
import parity
import reflib
from guetzli_b200 import synth
from guetzli_b200.api import _CStats, _LOG_FN, _cparams

ANSWERS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "image_inputs_reference_answers.json")
QUALITY = 90
SIZES = [(35, 41), (20, 24), (1, 1)]  # odd and large enough for Butteraugli; tiny (no Butteraugli); one pixel
YUV420 = "guetzli_b200: YUV420 is outside the GPU hot path (DESIGN.md)\n"


@pytest.fixture(scope="module")
def ref(ref):
    """The session's reference, with the recorded answers of this module's calls added in replay mode."""
    if reflib._answers is not None:
        with open(ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


def blend_on_black(v, a):
    """BlendOnBlack (g/guetzli.cc:43-45)."""
    return ((v.astype(np.int32) * a.astype(np.int32) + 128) // 255).astype(np.uint8)


def to_rgb(img):
    """ReadPNG's layouts to RGB (g/guetzli.cc:94-145): [h][w] or [h][w][C] -> [h][w][3]."""
    img = np.asarray(img)
    if img.ndim == 2:
        img = img[..., None]
    c = img.shape[2]
    if c == 1:
        return np.repeat(img, 3, axis=2)
    if c == 2:
        return np.repeat(blend_on_black(img[..., :1], img[..., 1:]), 3, axis=2)
    if c == 3:
        return np.ascontiguousarray(img)
    return blend_on_black(img[..., :3], img[..., 3:])


# (v, a) with v a = 127 (mod 255): there (v a + 128) / 255 and the butteraugli tool's (v a + 127) / 255 differ
PAIRS_127 = np.array([(v, a) for v in range(256) for a in range(256) if v * a % 255 == 127], dtype=np.uint8)


def image(h, w, c, seed):
    """uint8 [h][w][c]: gradient and noise (gray for c <= 2); the alpha of c = 2 and 4 random, with 0 and 255
    frequent, and the first pixels carrying the (v, a) pairs of PAIRS_127."""
    rgb = synth.gradnoise(max(h, 2), max(w, 2), seed)[:h, :w]  # the gradient needs two pixels a side
    color = rgb[..., 1:2] if c <= 2 else rgb
    if c in (1, 3):
        return np.ascontiguousarray(color)
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 256, (h, w), dtype=np.uint8)
    a[rng.random((h, w)) < 0.2] = 255
    a[rng.random((h, w)) < 0.1] = 0
    img = np.concatenate([color, a[..., None]], axis=2)
    flat = img.reshape(-1, c)
    k = min(len(PAIRS_127), h * w // 2)
    flat[:k, 0] = PAIRS_127[:k, 0]
    flat[:k, c - 1] = PAIRS_127[:k, 1]
    return img


def case(h, w, c):
    return image(h, w, c, 100 + 10 * c + h)


def every_pair(c):
    """256 x 256 pixels whose (value, alpha) run over every pair: value x, alpha y (c = 2 or 4)."""
    v, a = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8))
    if c == 2:
        return np.stack([v, a], axis=2)
    return np.stack([v, 255 - v, a, a], axis=2)


def params(lib, quality=QUALITY, **kw):
    return gb.Params(butteraugli_target=gb.butteraugli_score_for_quality(quality, lib=lib), **kw)


def encode(lib, img, quality=QUALITY, **kw):
    st = gb.ProcessStats(debug_output=[])
    ok, jpeg = gb.process_image(params(lib, quality, **kw), st, img, lib=lib)
    return ok, jpeg, "".join(st.debug_output), st


def check_reference(lib, ref, img, quality=QUALITY):
    """process_image(img) against the reference's Process on to_rgb(img)."""
    want = to_rgb(img.cpu().numpy() if hasattr(img, "cpu") else img)
    ok, jpeg, trace, _ = encode(lib, img, quality)
    rok, rjpeg, rtrace, _, _ = ref.process_rgb(want, quality)
    assert ok == rok
    assert jpeg == rjpeg, "JPEG bytes differ from the reference's"
    assert trace == rtrace, "verbose trace differs from the reference's"


def assert_rgb(got, want, what):
    """Equal RGB images, or the first differing pixel named."""
    assert got.shape == want.shape, f"{what}: shape {got.shape} vs {want.shape}"
    bad = np.argwhere((got != want).any(axis=2))
    if len(bad):
        y, x = bad[0]
        raise AssertionError(f"{what}: {len(bad)} pixels differ, the first at (y {y}, x {x}): "
                             f"{got[y, x].tolist()} vs {want[y, x].tolist()}")


def layouts(h, w, seed):
    """Strided host views, each with the contiguous image it shows: a crop (rows longer than w C), a CHW array
    permuted to HWC, a gray plane broadcast to three channels (channel stride 0), [h][w] against [h][w][1]."""
    base = image(h + 6, w + 10, 4, seed)
    chw = np.ascontiguousarray(image(h, w, 3, seed + 1).transpose(2, 0, 1))
    g = image(h, w, 1, seed + 2)[..., 0]
    views = {"crop": base[3:3 + h, 5:5 + w], "chw_permuted": chw.transpose(1, 2, 0),
             "gray_broadcast": np.broadcast_to(g[..., None], (h, w, 3)), "gray_2d": g}
    plain = {k: np.ascontiguousarray(v) for k, v in views.items()}
    plain["gray_2d"] = np.ascontiguousarray(g[..., None])
    return views, plain


def c_call(lib, entry, img_ptr, w, h, channels, strides, device=0, p=None, stream=None):
    """A C encode entry called directly (arguments the Python wrapper refuses) -> (return value, message)."""
    cp, cs = _cparams(p or gb.Params()), _CStats()
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    st = None if strides is None else np.asarray(strides, dtype=np.int64)
    args = [C.byref(cp), img_ptr, w, h, channels, None if st is None else st.ctypes.data, device,
            C.cast(None, _LOG_FN), None, C.byref(out), C.byref(out_len), C.byref(cs)]
    if entry.endswith("_device"):
        args.append(stream)
    r = getattr(lib, entry)(*args)
    if out:
        lib.gb200_free(out)
    return r, gb.last_error(lib=lib)


# ---- CPU port ----------------------------------------------------------------------------------------------


@pytest.mark.parametrize("c", [1, 2, 3, 4])
@pytest.mark.parametrize("h,w", SIZES)
def test_port_matches_reference(port_lib, ref, h, w, c):
    check_reference(port_lib, ref, case(h, w, c))


@pytest.mark.parametrize("c", [2, 4])
def test_port_alpha_rule(port_lib, c):
    """Every (value, alpha) pair converts by BlendOnBlack, which differs from the butteraugli tool's rule at
    v a = 127 (mod 255); the resident image's RGB equals to_rgb."""
    img = every_pair(c)
    want = to_rgb(img)
    v, a = img[..., 0].astype(int), img[..., c - 1].astype(int)
    differs = v * a % 255 == 127
    assert differs.sum() == len(PAIRS_127) and ((v * a + 127) // 255 != want[..., 0])[differs].all()
    d = gb.DeviceImage.from_image(img, prepare=False, lib=port_lib)
    try:
        assert_rgb(d.rgb(), want, f"{c} channels")
    finally:
        d.close()


@pytest.mark.parametrize("c", [1, 2, 3, 4])
def test_port_converted_rgb(port_lib, c):
    img = case(35, 41, c)
    d = gb.DeviceImage.from_image(img if c > 1 else img[..., 0], prepare=True, lib=port_lib)
    try:
        assert_rgb(d.rgb(), to_rgb(img), f"{c} channels")
        ref_img = gb.DeviceImage(to_rgb(img), lib=port_lib)
        assert np.array_equal(d.orig_coeffs(), ref_img.orig_coeffs())
        ref_img.close()
    finally:
        d.close()


def test_port_layouts(port_lib):
    """Strided views give the bytes and trace of their contiguous copies."""
    views, plain = layouts(33, 37, 7)
    for k, v in views.items():
        if k != "gray_2d":
            assert not v.flags.c_contiguous, k
        got, want = encode(port_lib, v), encode(port_lib, plain[k])
        assert got[0] and got[1] == want[1] and got[2] == want[2], k
        d = gb.DeviceImage.from_image(v, prepare=False, lib=port_lib)
        assert_rgb(d.rgb(), to_rgb(plain[k]), k)
        d.close()


def test_port_refusals(port_lib):
    lib = port_lib
    img = case(33, 35, 4)
    ptr, strides = img.ctypes.data, [35 * 4, 4, 1]
    for ch in (0, 5):
        r, msg = c_call(lib, "gb200_process_image", ptr, 35, 33, ch, strides)
        assert not r and f"an image has 1 (gray), 2 (gray + alpha), 3 (RGB) or 4 (RGBA) channels, got {ch}" in msg
        assert not lib.gb200_image_create_strided(ptr, 35, 33, ch, None, 0, 0)
        assert f"channels, got {ch}" in gb.last_error(lib=lib)
    r, msg = c_call(lib, "gb200_process_image", ptr, 35, 33, 4, [35 * 4, -4, 1])
    assert not r and "image strides must not be negative, got row 140, pixel -4, channel 1" in msg
    for args in [(None, 35, 33), (ptr, 0, 33), (ptr, 35, 0), (ptr, 65536, 1), (ptr, 1, 65536), (ptr, -1, 33)]:
        r, msg = c_call(lib, "gb200_process_image", *args, 4, None)
        want = "guetzli_b200: empty image\n" if 0 in args[1:] else "Could not create jpg data from rgb pixels\n"
        assert not r and msg == want, args
        assert not lib.gb200_image_create_strided(args[0], args[1], args[2], 4, None, 0, 0)
        assert gb.last_error(lib=lib) == "bad image size"
    # the encoder's own refusals return (False, b"") with the RGB path's message
    assert gb.process_image(params(lib), None, np.zeros((0, 5, 3), np.uint8), lib=lib) == (False, b"")
    assert gb.last_error(lib=lib) == "guetzli_b200: empty image\n"
    assert gb.process_image(params(lib, 70), None, img, lib=lib) == (False, b"")
    assert gb.last_error(lib=lib).startswith("Guetzli should be called with quality >= 84")
    for flag in ("force_420", "try_420"):
        assert gb.process_image(params(lib, **{flag: True}), None, img, lib=lib) == (False, b"")
        assert gb.last_error(lib=lib) == YUV420
        assert gb.process(params(lib, **{flag: True}), None, to_rgb(img), 35, 33, lib=lib) == (False, b"")
        assert gb.last_error(lib=lib) == YUV420
    # the device entries: the port has no device memory
    r, msg = c_call(lib, "gb200_process_image_device", ptr, 35, 33, 4, None)
    assert not r and msg == "the CPU port has no device memory"
    assert not lib.gb200_image_create_device(ptr, 35, 33, 4, None, 0, 0, None)
    assert gb.last_error(lib=lib) == "the CPU port has no device memory"
    # malformed arguments never reach the C entries
    for bad, what in [(img.astype(np.float32), "must be uint8"), (img[None], "must have 2 or 3 axes"),
                      (np.zeros((8, 8, 5), np.uint8), "channels in its last axis"),
                      (img[::-1], "non-negative strides")]:
        with pytest.raises(ValueError, match=what):
            gb.process_image(params(lib), None, bad, lib=lib)
        with pytest.raises(ValueError, match=what):
            gb.DeviceImage.from_image(bad, lib=lib)


# ---- GPU ---------------------------------------------------------------------------------------------------


def _torch():
    return pytest.importorskip("torch")


def _golden_views(torch, rgb):
    t = torch.from_numpy(rgb).cuda()
    views = {"hwc": t,
             "chw_permuted": torch.from_numpy(np.ascontiguousarray(rgb.transpose(2, 0, 1))).cuda().permute(1, 2, 0),
             "rgba_opaque": torch.cat([t, torch.full_like(t[..., :1], 255)], dim=2)}
    if (rgb == rgb[..., :1]).all():
        views["gray_2d"] = t[..., 0]
    return views


def check_golden_hashes(lib, img, g, what):
    ok, jpeg, trace, st = encode(lib, img, g["quality"])
    assert ok == g["ok"], what
    assert len(jpeg) == g["jpeg_size"] and hashlib.sha256(jpeg).hexdigest() == g["jpeg_sha256"], what
    assert hashlib.sha256(trace.encode()).hexdigest() == g["trace_sha256"], what
    assert [st.counters["number of iterations"], st.counters["number of iterations up"],
            st.counters["number of iterations down"]] == g["iterations"], what


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(parity.GOLDEN))
def test_cuda_golden_inputs(cuda_lib, name):
    """The golden inputs as CUDA tensors in several layouts reproduce the recorded answers."""
    torch = _torch()
    g = parity.GOLDEN[name]
    rgb = parity.golden_input(name)
    assert synth.sha256(rgb) == g["input_sha256"]
    for kind, t in _golden_views(torch, rgb).items():
        check_golden_hashes(cuda_lib, t, g, f"{name}, {kind}")


@pytest.mark.gpu
def test_cuda_golden_1080p(cuda_lib):
    torch = _torch()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_large.json")
    g = json.load(open(path))["noise1080p_s1234_q95"]
    rgb = synth.noise(1080, 1920, 1234)
    assert synth.sha256(rgb) == g["input_sha256"]
    check_golden_hashes(cuda_lib, torch.from_numpy(rgb).cuda(), g, "noise1080p")


@pytest.mark.gpu
@pytest.mark.parametrize("c", [2, 4])
@pytest.mark.parametrize("h,w", SIZES)
def test_cuda_blended_matches_reference(cuda_lib, ref, h, w, c):
    torch = _torch()
    check_reference(cuda_lib, ref, torch.from_numpy(case(h, w, c)).cuda())


@pytest.mark.gpu
def test_cuda_alpha_rule(cuda_lib):
    torch = _torch()
    for c in (2, 4):
        img = every_pair(c)
        d = gb.DeviceImage.from_image(torch.from_numpy(img).cuda(), prepare=False, lib=cuda_lib)
        try:
            assert_rgb(d.rgb(), to_rgb(img), f"{c} channels")
        finally:
            d.close()


def _torch_layouts(torch, h, w, seed):
    """The views of layouts() as CUDA tensor views of the same kinds."""
    base = torch.from_numpy(image(h + 6, w + 10, 4, seed)).cuda()
    chw = torch.from_numpy(np.ascontiguousarray(image(h, w, 3, seed + 1).transpose(2, 0, 1))).cuda()
    g = torch.from_numpy(image(h, w, 1, seed + 2)[..., 0]).cuda()
    return {"crop": base[3:3 + h, 5:5 + w], "chw_permuted": chw.permute(1, 2, 0),
            "gray_broadcast": g[..., None].expand(h, w, 3), "gray_2d": g}


@pytest.mark.gpu
def test_cuda_host_and_device_layouts(cuda_lib):
    """Host views, CUDA views and the contiguous copies all give the same bytes and trace."""
    torch = _torch()
    for h, w, seed in [(70, 93, 11), (33, 37, 7), (21, 9, 5)]:
        views, plain = layouts(h, w, seed)
        tviews = _torch_layouts(torch, h, w, seed)
        for k in views:
            assert not tviews[k].is_contiguous() or k == "gray_2d", k
            want = encode(cuda_lib, plain[k])
            host, dev = encode(cuda_lib, views[k]), encode(cuda_lib, tviews[k])
            assert want[0] and host[:3] == want[:3] and dev[:3] == want[:3], (h, w, k)


@pytest.mark.gpu
def test_cuda_upload_bytes(cuda_lib):
    """From CUDA memory nothing of the image is uploaded: process()'s bytes minus 3 w h.  From host memory the
    view's span is."""
    torch = _torch()
    rgb = synth.gradnoise(64, 96, 7)
    h, w, _ = rgb.shape
    p = params(cuda_lib)
    gb.process(p, None, rgb, w, h, lib=cuda_lib)
    st0, st1, st2 = gb.ProcessStats(), gb.ProcessStats(), gb.ProcessStats()
    want = gb.process(p, st0, rgb, w, h, lib=cuda_lib)
    assert gb.process_image(p, st1, torch.from_numpy(rgb).cuda(), lib=cuda_lib) == want
    assert st1.device["h2d_bytes"] == st0.device["h2d_bytes"] - 3 * w * h
    rgba = image(h + 2, w, 4, 3)[1:1 + h]
    rgba[..., :3], rgba[..., 3] = rgb, 255
    assert gb.process_image(p, st2, rgba, lib=cuda_lib) == want
    assert st2.device["h2d_bytes"] == st0.device["h2d_bytes"] - 3 * w * h + 4 * w * h


@pytest.mark.gpu
def test_cuda_stream_ordering(cuda_lib):
    """A tensor filled late on a busy side stream is read after the fill, by both entries."""
    torch = _torch()
    img = case(35, 41, 4)
    want = encode(cuda_lib, img)
    dev = torch.device("cuda", 0)
    staged = torch.from_numpy(img).to(dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        t = torch.zeros_like(staged)
        torch.cuda._sleep(20_000_000)  # keeps the side stream busy: the copy below lands late
        t.copy_(staged)
        got = encode(cuda_lib, t)
        u = torch.zeros_like(staged)
        torch.cuda._sleep(20_000_000)
        u.copy_(staged)
        d = gb.DeviceImage.from_image(u, prepare=False, lib=cuda_lib)
    torch.cuda.synchronize(dev)
    assert got[:3] == want[:3]
    try:
        assert_rgb(d.rgb(), to_rgb(img), "DeviceImage.from_image")
    finally:
        d.close()


@pytest.mark.gpu
def test_cuda_two_threads(cuda_lib):
    torch = _torch()
    imgs = [case(35, 41, 4), image(70, 93, 2, 17)]
    want = [encode(cuda_lib, x)[:3] for x in imgs]
    tensors = [torch.from_numpy(x).cuda() for x in imgs]
    torch.cuda.synchronize()
    got = [None, None]

    def run(k):
        got[k] = encode(cuda_lib, tensors[k])[:3]

    threads = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert got == want


@pytest.mark.gpu
def test_cuda_resident_context(cuda_lib):
    """A resident image made from a CUDA tensor keeps the pixels it was made from."""
    torch = _torch()
    img = case(35, 41, 4)
    want = encode(cuda_lib, img)[1]
    t = torch.from_numpy(img).cuda()
    d = gb.DeviceImage.from_image(t, prepare=False, lib=cuda_lib)
    try:
        t.fill_(0)
        torch.cuda.synchronize()
        ok, jpeg = d.process(params(cuda_lib))
        assert ok and jpeg == want
        assert_rgb(d.rgb(), to_rgb(img), "resident")
    finally:
        d.close()


def _managed(nbytes):
    """nbytes of managed memory (cuMemAllocManaged) -> (pointer, free)."""
    try:
        cuda = C.CDLL("libcuda.so.1")
    except OSError:
        pytest.skip("no libcuda")
    p = C.c_uint64()
    assert cuda.cuMemAllocManaged(C.byref(p), C.c_size_t(nbytes), 1) == 0  # CU_MEM_ATTACH_GLOBAL
    return p.value, lambda: cuda.cuMemFree_v2(p)


@pytest.mark.gpu
def test_cuda_device_refusals(cuda_lib):
    """A host pointer, managed memory and another device's memory are refused before anything runs."""
    torch = _torch()
    img = case(35, 41, 4)
    torch.cuda.synchronize()
    launches = gb.counters(lib=cuda_lib)[0]
    ptr, free = _managed(img.nbytes)
    try:
        for p, why in [(img.ctypes.data, "(host or unknown memory)"), (ptr, "(host or unknown memory)")]:
            r, msg = c_call(cuda_lib, "gb200_process_image_device", p, 41, 35, 4, None)
            assert not r and msg == f"process_image_device: img is not device memory of device 0 {why}"
            assert not cuda_lib.gb200_image_create_device(p, 41, 35, 4, None, 0, 0, None)
            assert gb.last_error(lib=cuda_lib) == f"image_create_device: img is not device memory of device 0 {why}"
    finally:
        free()
    if torch.cuda.device_count() >= 2:
        t = torch.from_numpy(img).to("cuda:1")
        torch.cuda.synchronize("cuda:1")
        r, msg = c_call(cuda_lib, "gb200_process_image_device", t.data_ptr(), 41, 35, 4, None)
        assert not r and msg == "process_image_device: img is not device memory of device 0 (device 1)"
    assert gb.counters(lib=cuda_lib)[0] == launches
