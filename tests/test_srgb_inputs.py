"""Butteraugli on 8-bit sRGB images (gb.butteraugli_srgb, ButteraugliBatch.diffmap_srgb,
Comparator.from_srgb and the gb200_*_srgb entries): the stand-alone tool's conversion and alpha rule
(butteraugli_main.cc:239-281, :390-419) on the device, bit for bit the reference's
butteraugli::ButteraugliInterface on linear(over(img, background)), with over() and linear() stated
here in numpy.  RGB is scored once; RGBA over black and over white, the larger score winning with its
diffmap (black on a tie).  Every reference call a GPU test makes is also made by a CPU test with the
same arguments, so that recording the CPU tests covers the GPU tests:

    GB200_REF_RECORD=$PWD/tests/golden/srgb_reference_answers.json \\
        python -m pytest tests/test_srgb_inputs.py -m "not gpu"

records them into golden/srgb_reference_answers.json, which replay mode reads beside
golden/reference_answers.json."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import guetzli_b200 as gb
import parity
import reflib
from guetzli_b200 import synth
from PIL import Image
from test_butteraugli import CLI, CLI_PORT, SIZES, linear
from test_comparator_batch import CASES

ANSWERS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "srgb_reference_answers.json")


@pytest.fixture(scope="module")
def ref(ref):
    """The session's reference, with the recorded answers of this module's calls added in replay mode."""
    if reflib._answers is not None:
        with open(ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


# ---- the tool's rule, stated in numpy ----------------------------------------------------------------

def over(img, bg):
    """img uint8 [..][C] -> [..][3]: RGB as it is; RGBA laid over the background `bg` in sRGB space,
    in integers (butteraugli_main.cc:264-275)."""
    if img.shape[-1] == 3:
        return img
    rgb, al = img[..., :3].astype(int), img[..., 3:].astype(int)
    v = (rgb * al + bg * (255 - al) + 127) // 255
    return np.where(al == 255, rgb, np.where(al == 0, bg, v)).astype(np.uint8)


def planes(img, bg):
    """[h][w][C] -> linear float32 [3][h][w]; [n][h][w][C] -> [n][3][h][w]."""
    if img.ndim == 4:
        return np.stack([planes(x, bg) for x in img])
    return linear(over(img, bg))


def tool(score, channels):
    """The tool's choice between the backgrounds: score(bg) -> (diffmap, score) of the pair laid over bg."""
    dm, s = score(0)
    if channels == 4:
        dmw, sw = score(255)
        if sw > s:  # strictly: a tie keeps black
            return dmw, sw
    return dm, s


def reference(ref, a, b):
    """The tool's answer for one pair [h][w][C] from the reference's ButteraugliInterface."""
    return tool(lambda bg: ref.butteraugli_interface(planes(a, bg), planes(b, bg)), a.shape[-1])


# ---- inputs --------------------------------------------------------------------------------------------

ALPHAS = np.array([0, 1, 127, 128, 254, 255], dtype=np.uint8)


def with_alpha(rgb, channels, seed):
    """RGB as it is, or with an alpha channel that takes every value of ALPHAS."""
    if channels == 3:
        return rgb
    h, w, _ = rgb.shape
    return np.dstack([rgb, ALPHAS[synth.noise(h, w, seed)[..., 0] % len(ALPHAS)]])


def perturbed(img, seed, k=3):
    """img with every channel moved by up to +-k, and a seventh of the alpha values changed."""
    h, w, ch = img.shape
    d = np.dstack([synth.noise(h, w, seed), synth.noise(h, w, seed + 1)[..., :1]])[..., :ch].astype(int)
    out = np.clip(img.astype(int) + d % (2 * k + 1) - k, 0, 255)
    if ch == 4:
        idx = np.searchsorted(ALPHAS, img[..., 3])
        out[..., 3] = ALPHAS[(idx + (d[..., 3] % 7 == 0)) % len(ALPHAS)]
    return out.astype(np.uint8)


def small_pair(h, w, channels, seed):
    """A noise pair of any size (test_butteraugli.pair with alpha)."""
    a = with_alpha((synth.noise(h, w, seed) // 2 + 64).astype(np.uint8), channels, seed + 7)
    return a, perturbed(a, seed + 1, 4)


def batch_pairs(h, w, n, channels):
    """n pairs with a distinct original each: gradient and noise, and a perturbed copy."""
    a = np.stack([with_alpha(synth.gradnoise(h, w, 4000 + 11 * i + h), channels, 4100 + i) for i in range(n)])
    b = np.stack([perturbed(a[i], 4200 + 3 * i + w, 2 + i % 4) for i in range(n)])
    return a, b


def candidates(h, w, n, channels):
    """One original and n candidates against it."""
    a = with_alpha(synth.gradnoise(h, w, 5000 + h + w), channels, 5100)
    return a, np.stack([perturbed(a, 5200 + 3 * i + h, 2 + i % 4) for i in range(n)])


# ---- checks shared by the CPU port and the GPU -----------------------------------------------------------

def float_batch(lib, a, b):
    """The float API's answer for pairs [n][h][w][C] on the converted planes, with the tool's rule."""
    n, h, w, ch = a.shape
    batch = gb.ButteraugliBatch(h, w, n, lib=lib)
    try:
        per_bg = {bg: batch.diffmap(planes(a, bg), planes(b, bg)) for bg in (0, 255)[:ch - 2]}
    finally:
        batch.close()
    return [tool(lambda bg: (per_bg[bg][0][i], per_bg[bg][1][i]), ch) for i in range(n)]


def check_pairwise(lib, ref, h, w, channels):
    a, b = small_pair(h, w, channels, 10 * h + w)
    dm, score = gb.butteraugli_srgb(a, b, lib=lib)
    dm0, score0 = reference(ref, a, b)
    assert score == score0 and parity.bits_equal(dm, dm0), f"{h}x{w}x{channels}: differs from the reference"
    dmf, scoref = tool(lambda bg: gb.api.butteraugli_diffmap(planes(a, bg), planes(b, bg), lib=lib), channels)
    assert score == scoref and parity.bits_equal(dm, dmf), f"{h}x{w}x{channels}: differs from the float call"
    dm2, score2 = gb.butteraugli_srgb(a, a, lib=lib)
    assert score2 == 0.0 and not dm2.any(), "identical images"


def check_shape(lib, ref, h, w, n, channels):
    """ButteraugliBatch.diffmap_srgb on n pairs and Comparator.from_srgb at capacity n and 1, against the
    reference and against the float API on the converted planes -> the results, for the device checks."""
    a, b = batch_pairs(h, w, n, channels)
    batch = gb.ButteraugliBatch(h, w, n, lib=lib)
    try:
        dm, score = batch.diffmap_srgb(a, b)
    finally:
        batch.close()
    assert dm.shape == (n, h, w) and dm.dtype == np.float32 and score.shape == (n,) and score.dtype == np.float64
    for i, (dmf, scoref) in enumerate(float_batch(lib, a, b)):
        dm0, score0 = reference(ref, a[i], b[i])
        assert score[i] == score0 and parity.bits_equal(dm[i], dm0), f"{h}x{w}x{channels} pair {i}: reference"
        assert score[i] == scoref and parity.bits_equal(dm[i], dmf), f"{h}x{w}x{channels} pair {i}: float batch"

    o, c = candidates(h, w, n, channels)
    o_n = np.ascontiguousarray(np.broadcast_to(o, c.shape))
    want = float_batch(lib, o_n, c)
    for i in range(n):
        dm0, score0 = reference(ref, o, c[i])
        assert want[i][1] == score0 and parity.bits_equal(want[i][0], dm0), f"{h}x{w}x{channels} candidate {i}"
    for cap in (n, 1):
        cmp = gb.Comparator.from_srgb(o, capacity=cap, lib=lib)
        try:
            got = [cmp.diffmap(c)] if cap == n else [cmp.diffmap(c[i]) for i in range(n)]
        finally:
            cmp.close()
        if cap == n:
            got = [(got[0][0][i], got[0][1][i]) for i in range(n)]
        for i, (dmc, scorec) in enumerate(got):
            assert scorec == want[i][1] and parity.bits_equal(dmc, want[i][0]), \
                f"{h}x{w}x{channels} comparator of capacity {cap}, candidate {i}"
    return a, b, dm, score, o, c, want


# SIZES of test_butteraugli for the pairwise call; shapes of test_comparator_batch.CASES for the batch and
# the comparator: pitch padding (9x17, 17x130), several strips and segments (577x70), full HD
CPU_SHAPES = [s for s in CASES if s[:2] in [(9, 17), (17, 130), (300, 411), (577, 70)]]
GPU_SHAPES = CPU_SHAPES + [s for s in CASES if s[:2] == (1080, 1920)]


def ramp():
    """16x16 images holding every byte value in every channel (the channels rotated), and a perturbed copy."""
    v = np.arange(256, dtype=np.uint8).reshape(16, 16)
    a = np.dstack([v, np.roll(v, 85), np.roll(v, 170)])
    return a, perturbed(a, 31, 3)


def check_table(lib, ref):
    """srgb_lin, the library's table, is the tool's table after rounding to float: every byte value goes
    through it, and the result is the float call's on linear() of the same images and the reference's."""
    a, b = ramp()
    for x in (b, np.ascontiguousarray(b[..., ::-1])):
        dm, score = gb.butteraugli_srgb(a, x, lib=lib)
        dmf, scoref = gb.api.butteraugli_diffmap(linear(a), linear(x), lib=lib)
        dm0, score0 = ref.butteraugli_interface(linear(a), linear(x))
        assert score == scoref == score0 and parity.bits_equal(dm, dmf) and parity.bits_equal(dm, dm0)
        assert score > 0


def alpha_cases():
    """(name, a, b, winner): dark content scores higher over white, light content over black."""
    h, w = 40, 56
    base = synth.gradnoise(h, w, 61)
    dark = with_alpha((base // 8).astype(np.uint8), 4, 62)
    light = with_alpha((255 - base // 8).astype(np.uint8), 4, 63)
    return [("dark", dark, perturbed(dark, 64, 3), 255), ("light", light, perturbed(light, 65, 3), 0)]


# (h, w, seed) of small_pair RGBA pairs below 8 px whose padded diffmaps would pick the other background
# than the tool picks on the cropped scores, in both directions
PADDED_CHOICE = [(3, 3, 1007), (2, 3, 1001), (4, 8, 1010)]


def pad8(img):
    """img [h][w][C] edge-replicated to at least 8x8, centred as ButteraugliInterface pads."""
    h, w = img.shape[:2]
    yb, xb = (8 - h) // 2 if h < 8 else 0, (8 - w) // 2 if w < 8 else 0
    return np.pad(img, ((yb, max(8, h) - h - yb), (xb, max(8, w) - w - xb), (0, 0)), mode="edge")


def check_padded_choice(lib, ref, cli, tmp_path):
    """Below 8 px each background is scored padded and then cropped, as ButteraugliInterface returns it,
    and the tool chooses on the cropped scores: through butteraugli_srgb and through the CLI."""
    for h, w, seed in PADDED_CHOICE:
        a, b = small_pair(h, w, 4, seed)
        per_bg = {bg: ref.butteraugli_interface(planes(a, bg), planes(b, bg)) for bg in (0, 255)}
        padded = {bg: gb.api.butteraugli_diffmap(planes(pad8(a), bg), planes(pad8(b), bg), lib=lib)[1]
                  for bg in (0, 255)}
        win = 255 if per_bg[255][1] > per_bg[0][1] else 0
        assert (padded[255] > padded[0]) != (win == 255), f"{h}x{w} seed {seed}: the padded maxima pick {win} too"
        dm, score = gb.butteraugli_srgb(a, b, lib=lib)
        assert score == per_bg[win][1] and parity.bits_equal(dm, per_bg[win][0]), f"{h}x{w} seed {seed}"
        pa, pb = str(tmp_path / "a.png"), str(tmp_path / "b.png")
        Image.fromarray(a).save(pa)
        Image.fromarray(b).save(pb)
        r = subprocess.run([cli, pa, pb], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        assert r.returncode == 0 and r.stdout.decode() == "%f\n" % per_bg[win][1], (h, w, seed, r.stdout, r.stderr)


def check_alpha(lib, ref):
    for name, a, b, winner in alpha_cases():
        per_bg = {bg: ref.butteraugli_interface(planes(a, bg), planes(b, bg)) for bg in (0, 255)}
        loser = 255 - winner
        assert per_bg[winner][1] > per_bg[loser][1], f"{name}: the case does not pick {winner}"
        dm, score = gb.butteraugli_srgb(a, b, lib=lib)
        assert score == per_bg[winner][1] and parity.bits_equal(dm, per_bg[winner][0]), name
        batch = gb.ButteraugliBatch(40, 56, 2, lib=lib)
        cmp = gb.Comparator.from_srgb(a, capacity=2, lib=lib)
        try:
            dmb, scoreb = batch.diffmap_srgb(np.stack([a, a]), np.stack([b, a]))
            dmc, scorec = cmp.diffmap(np.stack([b, a]))
        finally:
            batch.close()
            cmp.close()
        for d, s in ((dmb, scoreb), (dmc, scorec)):
            assert s[0] == score and parity.bits_equal(d[0], dm), name
            assert s[1] == 0.0 and not d[1].any(), f"{name}: identical images"


def refusals(lib, device_entry_message):
    """Every refusal of the 8-bit entries, each with its message, launching nothing and writing no score."""
    a, b = batch_pairs(40, 56, 3, 3)
    a4, b4 = batch_pairs(40, 56, 3, 4)
    score = np.full(4, -1.0)
    score_p = score.ctypes.data_as(C.POINTER(C.c_double))  # for the entries that take double*

    def refused(ok, msg):
        assert not ok
        assert msg in gb.last_error(lib=lib), (msg, gb.last_error(lib=lib))

    launches = gb.counters(lib=lib)[0]
    for ch in (0, 1, 2, 5):
        msg = f"channels = {ch}, 8-bit images must have 3 (RGB) or 4 (RGBA)"
        refused(lib.gb200_butteraugli_diffmap_srgb(a.ctypes.data, b.ctypes.data, 56, 40, ch, 0, None, score_p), msg)
        refused(lib.gb200_butteraugli_comparator_create_srgb(a.ctypes.data, 56, 40, ch, 2, 0), msg)
    refused(lib.gb200_butteraugli_comparator_create_srgb(a.ctypes.data, 7, 40, 3, 2, 0), "at least 8x8")
    refused(lib.gb200_butteraugli_comparator_create_srgb(a.ctypes.data, 56, 40, 3, 0, 0), "capacity must be in 1..16383")
    refused(lib.gb200_butteraugli_comparator_create_srgb(None, 56, 40, 3, 2, 0), "no image")
    refused(lib.gb200_butteraugli_diffmap_srgb(None, b.ctypes.data, 56, 40, 3, 0, None, score_p), "no image")
    assert gb.counters(lib=lib)[0] == launches

    batch = gb.ButteraugliBatch(40, 56, 3, lib=lib)
    fcmp = gb.Comparator(planes(a[0], 0), capacity=3, lib=lib)
    cmp3 = gb.Comparator.from_srgb(a[0], capacity=3, lib=lib)
    cmp4 = gb.Comparator.from_srgb(a4[0], capacity=3, lib=lib)
    try:
        launches = gb.counters(lib=lib)[0]  # after the originals' analysis
        for ch in (0, 1, 2, 5):
            msg = f"channels = {ch}, 8-bit images must have 3 (RGB) or 4 (RGBA)"
            refused(lib.gb200_butteraugli_batch_diffmap_srgb(batch._h, a.ctypes.data, b.ctypes.data, 2, ch, None,
                                                             score.ctypes.data), msg)
            refused(lib.gb200_butteraugli_batch_diffmap_srgb_device(batch._h, a.ctypes.data, b.ctypes.data, 2, ch,
                                                                    None, score.ctypes.data, None), msg)
        for n in (0, -1, 4):
            refused(lib.gb200_butteraugli_batch_diffmap_srgb(batch._h, a.ctypes.data, b.ctypes.data, n, 3, None,
                                                             score.ctypes.data), f"n = {n} pairs, the batch takes 1..3")
            refused(lib.gb200_butteraugli_batch_diffmap_srgb_device(batch._h, a.ctypes.data, b.ctypes.data, n, 3, None,
                                                                    score.ctypes.data, None),
                    f"n = {n} pairs, the batch takes 1..3")
            for c, x in ((cmp3, b), (cmp4, b4)):
                refused(lib.gb200_butteraugli_comparator_diffmap_srgb(c._h, x.ctypes.data, n, None, score.ctypes.data),
                        f"n = {n} images, the comparator takes 1..3")
                refused(lib.gb200_butteraugli_comparator_diffmap_srgb_device(c._h, x.ctypes.data, n, None,
                                                                             score.ctypes.data, None),
                        f"n = {n} images, the comparator takes 1..3")
        # host memory given to the device entries
        refused(lib.gb200_butteraugli_batch_diffmap_srgb_device(batch._h, a.ctypes.data, b.ctypes.data, 2, 3, None,
                                                                score.ctypes.data, None),
                device_entry_message.format("img0"))
        for c, x in ((cmp3, b), (cmp4, b4)):
            refused(lib.gb200_butteraugli_comparator_diffmap_srgb_device(c._h, x.ctypes.data, 2, None,
                                                                         score.ctypes.data, None),
                    device_entry_message.format("img1"))
        # kinds do not mix
        f1 = planes(b, 0)
        float_msg = "made from 8-bit images, it takes 8-bit images, not float planes"
        for c in (cmp3, cmp4):
            refused(lib.gb200_butteraugli_comparator_diffmap(c._h, f1.ctypes.data, None, score_p), float_msg)
            refused(lib.gb200_butteraugli_comparator_diffmap_device(c._h, f1.ctypes.data, None, score_p, None), float_msg)
            refused(lib.gb200_butteraugli_comparator_diffmap_batch(c._h, f1.ctypes.data, 2, None, score.ctypes.data),
                    float_msg)
            refused(lib.gb200_butteraugli_comparator_diffmap_batch_device(c._h, f1.ctypes.data, 2, None,
                                                                          score.ctypes.data, None), float_msg)
        u8_msg = "made from float planes, it takes float images, not 8-bit ones"
        refused(lib.gb200_butteraugli_comparator_diffmap_srgb(fcmp._h, b.ctypes.data, 2, None, score.ctypes.data),
                u8_msg)
        refused(lib.gb200_butteraugli_comparator_diffmap_srgb_device(fcmp._h, b.ctypes.data, 2, None,
                                                                     score.ctypes.data, None), u8_msg)
        m = np.full((3, 40, 56), -1.0, dtype=np.float32)
        refused(lib.gb200_butteraugli_comparator_mask(cmp4._h, m.ctypes.data, m.ctypes.data),
                "an RGBA comparator has two originals")
        assert (m == -1.0).all()
        assert (score == -1.0).all(), "a refused call wrote scores"
        assert gb.counters(lib=lib)[0] == launches
        # an RGB comparator made from 8-bit images has one original and its mask
        mk, mdc = cmp3.mask()
        mk0, mdc0 = fcmp.mask()
        assert parity.bits_equal(mk, mk0) and parity.bits_equal(mdc, mdc0)
    finally:
        for o in (batch, fcmp, cmp3, cmp4):
            o.close()


def python_checks(lib):
    """Shape, dtype and channel errors raise ValueError before anything reaches the library."""
    a, b = batch_pairs(40, 56, 3, 4)
    batch = gb.ButteraugliBatch(40, 56, 3, lib=lib)
    cmp = gb.Comparator.from_srgb(a[0], capacity=3, lib=lib)
    try:
        launches = gb.counters(lib=lib)[0]
        bad_pairs = [(a, b[:2]), (a[..., :2], b[..., :2]), (a[..., :3], b), (a.astype(np.float32), b),
                     (a[0], b[0]), (a[:0], b[:0]), (np.concatenate([a, a[:1]]), np.concatenate([b, b[:1]])),
                     (a[:, :39], b[:, :39]), (np.dstack([a[0], a[0, ..., :1]])[None], np.dstack([b[0], b[0, ..., :1]])[None])]
        for x, y in bad_pairs:
            with pytest.raises(ValueError):
                batch.diffmap_srgb(x, y)
        for x in [b[..., :3], b.astype(np.int16), b[:, :39], b[0, :, :, 0], np.concatenate([b, b[:1]]), b[:0],
                  planes(b[0], 0)]:
            with pytest.raises(ValueError):
                cmp.diffmap(x)
        for x, y in [(a[0], b[0, ..., :3]), (a[0, ..., :2], b[0, ..., :2]), (a[0].astype(np.float32), b[0]), (a, b)]:
            with pytest.raises(ValueError):
                gb.butteraugli_srgb(x, y, lib=lib)
        with pytest.raises(ValueError):
            gb.Comparator.from_srgb(a[0, ..., :2], lib=lib)
        assert gb.counters(lib=lib)[0] == launches
        with pytest.raises(RuntimeError, match="two originals"):
            cmp.mask()
        dm, score = cmp.diffmap(b[0])  # [h][w][C]: the single-image call
        dmn, scoren = cmp.diffmap(b[:1])
        assert dm.shape == (40, 56) and isinstance(score, float) and dmn.shape == (1, 40, 56)
        assert score == scoren[0] and parity.bits_equal(dm, dmn[0])
    finally:
        batch.close()
        cmp.close()


# ---- CPU: the port, and every reference call of the GPU tests ------------------------------------------

def test_port_table(port_lib, ref):
    check_table(port_lib, ref)


def test_port_padded_rgba_choice(port_lib, ref, tmp_path):
    check_padded_choice(port_lib, ref, CLI_PORT, tmp_path)


def test_port_alpha_rule(port_lib, ref):
    check_alpha(port_lib, ref)


@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("h,w", SIZES)
def test_port_pairwise(port_lib, ref, h, w, channels):
    check_pairwise(port_lib, ref, h, w, channels)


@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("h,w,n", CPU_SHAPES)
def test_port_batch_and_comparator(port_lib, ref, h, w, n, channels):
    check_shape(port_lib, ref, h, w, n, channels)


@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("h,w,n", [s for s in GPU_SHAPES if s not in CPU_SHAPES])
def test_reference_answers_of_gpu_shapes(ref, h, w, n, channels):
    """The reference calls of the GPU-only shape, full HD, which the port would take minutes to score."""
    a, b = batch_pairs(h, w, n, channels)
    o, c = candidates(h, w, n, channels)
    for i in range(n):
        for x, y in ((a[i], b[i]), (o, c[i])):
            assert reference(ref, x, y)[1] > 0


def test_port_refusals(port_lib):
    refusals(port_lib, "no device memory")


def test_port_python_checks(port_lib):
    python_checks(port_lib)


# ---- GPU ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_cuda_table(cuda_lib, ref):
    check_table(cuda_lib, ref)


@pytest.mark.gpu
def test_cuda_padded_rgba_choice(cuda_lib, ref, tmp_path):
    check_padded_choice(cuda_lib, ref, CLI, tmp_path)


@pytest.mark.gpu
def test_cuda_alpha_rule(cuda_lib, ref):
    check_alpha(cuda_lib, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("h,w", SIZES)
def test_cuda_pairwise(cuda_lib, ref, h, w, channels):
    check_pairwise(cuda_lib, ref, h, w, channels)


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("h,w,n", GPU_SHAPES)
def test_cuda_batch_and_comparator(cuda_lib, ref, h, w, n, channels):
    """The host entries against the reference, and the device entries against the host entries, with the
    images written late on a busy non-default stream that the library must wait for."""
    torch = pytest.importorskip("torch")
    a, b, dm, score, o, c, want = check_shape(cuda_lib, ref, h, w, n, channels)
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    batch = gb.ButteraugliBatch(h, w, n, lib=cuda_lib)
    cmp = gb.Comparator.from_srgb(o, capacity=n, lib=cuda_lib)
    try:
        staged = [torch.from_numpy(x).to(dev) for x in (a, b, c)]
        torch.cuda.synchronize(dev)
        with torch.cuda.stream(side):
            t = [torch.zeros_like(x) for x in staged]
            torch.cuda._sleep(20_000_000)  # keeps the side stream busy: the copies below land late
            for x, y in zip(t, staged):
                x.copy_(y)
            dm_t, score_t = batch.diffmap_srgb(t[0], t[1])
            dmc_t, scorec_t = cmp.diffmap(t[2])
            dm1_t, score1_t = cmp.diffmap(t[2][n - 1])
        torch.cuda.synchronize(dev)
        assert dm_t.device == dev and dm_t.dtype == torch.float32 and tuple(dm_t.shape) == (n, h, w)
        assert (score_t == score).all() and parity.bits_equal(dm_t.cpu().numpy(), dm), "batch: device != host"
        assert dmc_t.device == dev and tuple(dmc_t.shape) == (n, h, w)
        for i in range(n):
            assert scorec_t[i] == want[i][1] and parity.bits_equal(dmc_t[i].cpu().numpy(), want[i][0]), f"candidate {i}"
        assert dm1_t.device == dev and score1_t == want[n - 1][1]
        assert parity.bits_equal(dm1_t.cpu().numpy(), want[n - 1][0])
    finally:
        torch.cuda.synchronize(dev)
        batch.close()
        cmp.close()


@pytest.mark.gpu
def test_cuda_refusals_launch_nothing(cuda_lib):
    refusals(cuda_lib, "{} is not device memory of device 0")


@pytest.mark.gpu
def test_cuda_python_checks(cuda_lib):
    python_checks(cuda_lib)
    torch = pytest.importorskip("torch")
    a, b = (torch.from_numpy(x).cuda() for x in small_pair(16, 16, 4, 3))
    launches = gb.counters(lib=cuda_lib)[0]
    for x, y in ((a, b), (a, b.cpu().numpy()), (a.cpu().numpy(), b)):
        with pytest.raises(ValueError, match="host memory"):
            gb.butteraugli_srgb(x, y, lib=cuda_lib)
    with pytest.raises(ValueError, match="host memory"):
        gb.Comparator.from_srgb(a, lib=cuda_lib)
    assert gb.counters(lib=cuda_lib)[0] == launches


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [3, 4])
def test_cuda_upload_is_the_bytes(cuda_lib, channels):
    """A host batch call uploads its 8-bit images once, 2 n h w C bytes, whatever the backgrounds; no
    float planes cross the bus."""
    h, w, n = 300, 411, 4
    a, b = batch_pairs(h, w, n, channels)
    batch = gb.ButteraugliBatch(h, w, n, lib=cuda_lib)
    try:
        batch.diffmap_srgb(a, b)  # the buffers' first use
        before = gb.counters(lib=cuda_lib)[1]
        batch.diffmap_srgb(a, b)
        up = gb.counters(lib=cuda_lib)[1] - before
    finally:
        batch.close()
    assert 2 * n * h * w * channels <= up <= 2 * n * h * w * channels + 64, up
