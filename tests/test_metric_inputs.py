"""The butteraugli metric (gb.api.butteraugli_diffmap, gb.Comparator, gb.ButteraugliBatch, mask() and
gb.adaptive_quantization) on the float inputs its API accepts beyond linear(uint8): values off the
sRGB grid, black and white planes, one-ULP and full-range single-pixel changes, checkerboards,
saturated primaries, impulses, Malta's line orientations, step edges at every x mod 8 and, outside
0..255, the slightly negative values of resampling ringing, noise around -50, highlights of a few
thousand and mixed signs.  Impulses and edges are also put on the rows and columns where the
rolling blurs change segment, ring row or border rule (test_roll_layouts.layout).

These inputs take value-dependent branches of the chain that linear(uint8) never reaches: the top
clamp of the Mask LUT interpolation, the SameNoiseLevels clamp at 85.7, GammaPolynomial far outside
its fit interval and the opsin sensitivity gamma(pre) / pre with pre near 0.  Every result is
compared bit for bit with the reference (oracle/_ref, or its recorded answers).  Every reference call
a GPU test makes is also made by a CPU test with the same arguments, so that recording the CPU tests
covers the GPU tests:

    GB200_REF_RECORD=$PWD/tests/golden/metric_inputs_reference_answers.json \\
        python -m pytest tests/test_metric_inputs.py -m "not gpu"

records them into golden/metric_inputs_reference_answers.json, which replay mode reads beside
golden/reference_answers.json.  GB200_PORT_LIB=<path> runs the CPU tests on another build of the
port (tools/metric_branch_coverage.sh uses it for an instrumented one)."""
import json
import os
import zlib

import numpy as np
import pytest

import guetzli_b200 as gb
import parity
import reflib
from test_comparator import reference_adaptive_quantization, reference_comparator_mask
from test_roll_layouts import BLUR_MASKX, BLUR_NOISE, RADII, describe, impulse_planes, layout

HERE = os.path.dirname(os.path.abspath(__file__))
ANSWERS = os.path.join(HERE, "golden", "metric_inputs_reference_answers.json")


@pytest.fixture(scope="module")
def ref(ref):
    """The session's reference, with the recorded answers of this module's calls added in replay mode."""
    if reflib._answers is not None:
        with open(ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


@pytest.fixture(scope="module")
def port_lib(port_lib):
    """The session's CPU port, or the build of it that GB200_PORT_LIB names."""
    path = os.environ.get("GB200_PORT_LIB")
    return gb.load_library(path) if path else port_lib


# ---------------------------------------------------------------------------------------------
# the corpus: named generators, each (rng, h, w) -> (original [3][h][w], three candidates), float32

def _f32(x):
    """float32 [3][h][w]; a [h][w] plane is repeated in all three channels."""
    x = np.asarray(x)
    return np.ascontiguousarray(x if x.ndim == 3 else np.broadcast_to(x, (3,) + x.shape), dtype=np.float32)


def _grid(h, w):
    return np.mgrid[0:h, 0:w]


def _malta_patterns():
    """kMaltaHF (tables_data.inc): the 16 line patterns of the HF Malta filter as (dy, dx) taps."""
    text = open(os.path.join(HERE, "..", "guetzli_b200", "csrc", "tables_data.inc")).read()
    body = text[text.index("kMaltaHF[16][9]"):]
    body = body[body.index("{") + 1:body.index("};")]
    rows = [[int(v) for v in r.split(",") if v.strip()] for r in body.replace("}", "").split("{")[1:]]
    assert len(rows) == 16
    return [[(c // 9 - 4, c % 9 - 4) for c in r if c != 255] for r in rows]


MALTA = _malta_patterns()


def malta_line(h, w, p, cy, cx):
    """A 1-px line through (cy, cx) along Malta pattern p: the pattern's taps, repeated end to end."""
    taps = MALTA[p]
    sy, sx = taps[-1][0] - taps[0][0], taps[-1][1] - taps[0][1]
    out = np.zeros((h, w), dtype=bool)
    for t in range(-max(h, w), max(h, w)):
        for dy, dx in taps:
            y, x = cy + dy + t * sy, cx + dx + t * sx
            if 0 <= y < h and 0 <= x < w:
                out[y, x] = True
    return out


def offgrid_uniform(rng, h, w):
    a = rng.uniform(0, 255, (3, h, w))
    return a, [np.clip(a + rng.normal(0, s, a.shape), 0, 255) for s in (0.3, 3.0, 30.0)]


def offgrid_gradnoise(rng, h, w):
    y, x = _grid(h, w)
    g = np.stack([255 * x / max(1, w - 1), 255 * y / max(1, h - 1), 127.5 + 127.5 * np.sin(x / 5.0 + y / 7.0)])
    a = np.clip(g + rng.normal(0, 4, g.shape), 0, 255)
    return a, [np.clip(g + rng.normal(0, s, g.shape), 0, 255) for s in (4, 1, 12)]


def black_against(rng, h, w):
    a = np.zeros((3, h, w))
    return a, [np.full((3, h, w), 255.0), rng.uniform(0, 255, (3, h, w)), np.full((3, h, w), 1e-3)]


def white_against(rng, h, w):
    a = np.full((3, h, w), 255.0)
    return a, [np.zeros((3, h, w)), rng.uniform(0, 255, (3, h, w)), np.full((3, h, w), 255 - 1e-3)]


def one_pixel(rng, h, w):
    """One pixel moved by one ULP (interior, then corner) and one moved by 255."""
    a = rng.uniform(0, 255, (3, h, w)).astype(np.float32)
    a[:, h // 2, w // 3] = 0
    b0, b1, b2 = a.copy(), a.copy(), a.copy()
    b0[1, h // 3, w // 2] = np.nextafter(b0[1, h // 3, w // 2], np.float32(np.inf))
    b1[:, h // 2, w // 3] = 255
    b2[0, h - 1, w - 1] = np.nextafter(b2[0, h - 1, w - 1], np.float32(0))
    return a, [b0, b1, b2]


def checkerboards(rng, h, w):
    y, x = _grid(h, w)
    c1 = 255.0 * ((x + y) % 2)
    c2 = 255.0 * ((x // 2 + y // 2) % 2)
    return _f32(c1), [_f32(c2), _f32(255 - c1), rng.uniform(0, 255, (3, h, w))]


def primaries(rng, h, w):
    """Saturated primaries and secondaries in 5x7 tiles: hard chroma edges in both directions."""
    y, x = _grid(h, w)
    cols = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [0, 255, 255], [255, 0, 255], [255, 255, 0],
                     [0, 0, 0], [255, 255, 255]], dtype=np.float64)
    t = (y // 5 * 3 + x // 7) % 8
    a = cols[t].transpose(2, 0, 1)
    b1 = cols[(t + 1) % 8].transpose(2, 0, 1)
    return a, [np.roll(a, 1, axis=2), b1, np.clip(a + rng.normal(0, 8, a.shape), 0, 255)]


def impulses(rng, h, w):
    """Single white pixels on black at the corners, in the middle of each edge, and in the interior."""
    a = np.zeros((3, h, w))
    spots = [[(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1)],
             [(0, w // 2), (h // 2, 0), (h - 1, w // 2), (h // 2, w - 1), (1, 1), (h - 2, w - 2)],
             [(h // 2, w // 2), (h // 3, w // 4), (2 * h // 3, 3 * w // 4)]]
    out = []
    for s in spots:
        b = a.copy()
        for yy, xx in s:
            b[:, yy, xx] = 255
        out.append(b)
    return a, out


def malta_lines(rng, h, w):
    """1-px white lines on a dark flat original, along each of the 16 Malta orientations."""
    a = np.full((3, h, w), 20.0)
    out = []
    for group in (range(0, 6), range(6, 11), range(11, 16)):
        m = np.zeros((h, w), dtype=bool)
        for k, p in enumerate(group):
            m |= malta_line(h, w, p, (k + 1) * h // 7, (k + 1) * w // 7)
        out.append(np.where(m, 255.0, a))
    return a, out


def step_edges(rng, h, w):
    """Vertical black/white edges at x = 9 j + 3, j = 0..7 (every x mod 8 where the image is wide
    enough), horizontal ones likewise in y."""
    y, x = _grid(h, w)
    ex = [9 * j + 3 for j in range(8) if 9 * j + 3 < w]
    ey = [9 * j + 3 for j in range(8) if 9 * j + 3 < h]
    vx = 255.0 * (np.searchsorted(ex, x, side="right") % 2)
    vy = 255.0 * (np.searchsorted(ey, y, side="right") % 2)
    return _f32(vx), [_f32(np.roll(vx, 1, axis=1)), _f32(vy), _f32(np.abs(vx - vy))]


# ---- tier 2: outside 0..255 ------------------------------------------------------------------

def ringing(rng, h, w):
    """Noise in [-2, 0], the undershoot of a resampling filter, against itself, gray and black."""
    a = rng.uniform(-2, 0, (3, h, w))
    return a, [rng.uniform(-2, 0, (3, h, w)), np.clip(a + rng.normal(0, 0.05, a.shape), -2, 0),
               rng.uniform(-2, 40, (3, h, w))]


def around_minus50(rng, h, w):
    """Noise around -50: the absorbance far below GammaPolynomial's interval; reaches the Mask LUT's
    top clamp."""
    a = -50 + 0.2 * rng.random((3, h, w))
    return a, [-50 + 0.2 * rng.random((3, h, w)), -50 + 2 * rng.random((3, h, w)), rng.uniform(0, 255, (3, h, w))]


def highlights(rng, h, w):
    """An image in 0..255 with specular highlights up to 3000; one candidate scales it to 4500."""
    a = rng.uniform(0, 255, (3, h, w))
    spots = rng.random((h, w)) < 0.05
    a[:, spots] = rng.uniform(255, 3000, (3, int(spots.sum())))
    return a, [np.clip(a + rng.normal(0, 20, a.shape), 0, 3000), np.clip(a, 0, 255), a * 1.5]


def mixed_sign(rng, h, w):
    a = rng.uniform(-20, 300, (3, h, w))
    return a, [rng.uniform(-20, 300, (3, h, w)), a + rng.normal(0, 1, a.shape), -a]


def negative_stripes(rng, h, w):
    """Vertical stripes between -3 and +2, 8 px wide: pre = absorbance near 0, where gamma(pre) / pre
    is large; the hf Y planes exceed SameNoiseLevels' clamp of 85.7."""
    y, x = _grid(h, w)
    s = -3.0 + 5.0 * ((x // 8) % 2)
    return _f32(s), [_f32(np.roll(s, 1, axis=1)), _f32(s + rng.normal(0, 0.1, (3, h, w))), _f32(-2.0 + 0 * s)]


# ---- placement: the rolling blurs' seams and border strips -----------------------------------

def seam_impulses(rng, h, w):
    """White impulses on gray at the rows and columns where the noise and mask blurs change segment,
    ring row or border rule (test_roll_layouts.impulse_planes), and horizontal step edges on those
    rows."""
    a = np.full((3, h, w), 10.0)
    out = []
    for r in (RADII[BLUR_NOISE], RADII[BLUR_MASKX]):
        ps = impulse_planes(h, w, r)
        out.append(np.where((ps["impulse_rows"] + ps["impulse_cols"]) > 0, 255.0, a))
    starts = layout(h).starts
    y, _ = _grid(h, w)
    band = np.searchsorted([s + d for s in starts[1:] for d in (-1, 0)], y, side="right") % 2
    out.append(_f32(np.where(band, 255.0, 0.0)))
    return a, out


def seam_mixed(rng, h, w):
    """Bands of -2 and 2000 that switch on the seam rows of the mask blur, against mixed-sign noise."""
    starts = layout(h).starts
    y, x = _grid(h, w)
    r = RADII[BLUR_MASKX]
    band = np.searchsorted(sorted({s + d for s in starts[1:] for d in (-r, -1, 0, r - 1)}), y, side="right") % 2
    a = np.where(band, 2000.0, -2.0) + 0 * x
    return _f32(a), [_f32(np.where(band, -2.0, 2000.0)), rng.uniform(-2, 300, (3, h, w)), _f32(a + 1e-2)]


TIER1 = [offgrid_uniform, offgrid_gradnoise, black_against, white_against, one_pixel, checkerboards, primaries,
         impulses, malta_lines, step_edges]
TIER2 = [ringing, around_minus50, highlights, mixed_sign, negative_stripes]
GENERATORS = {g.__name__: g for g in TIER1 + TIER2 + [seam_impulses, seam_mixed]}

CASES = ([(g.__name__, 40, 56) for g in TIER1 + TIER2]
         + [(g.__name__, 64, 64) for g in TIER1 + TIER2]
         + [(g.__name__, 8, 8) for g in (black_against, checkerboards, impulses, ringing, around_minus50)]
         + [(g.__name__, 17, 130) for g in (step_edges, malta_lines, negative_stripes, highlights)]
         + [(g.__name__, 300, 411) for g in (offgrid_gradnoise, primaries, malta_lines, around_minus50, mixed_sign)]
         + [("seam_impulses", 577, 70), ("seam_mixed", 577, 70), ("seam_impulses", 1080, 100),
            ("seam_mixed", 1080, 100), ("seam_impulses", 1080, 1920)])
# shapes whose cases are also scored side by side, in neighbouring slots of one call
SLOT_SHAPES = [(40, 56), (64, 64), (300, 411), (1080, 100)]
# the tier-2 cases whose stages (opsin, frequency split, blurs) are checked on their own
STAGE_CASES = [(g.__name__, 40, 56) for g in TIER2] + [("seam_mixed", 577, 70)]


def case_id(c):
    return f"{c[0]}-{c[1]}x{c[2]}"


def corpus(name, h, w):
    """-> (original, [three candidates]), float32 [3][h][w], the same on every run."""
    rng = np.random.default_rng([zlib.crc32(name.encode()), h, w])
    a, bs = GENERATORS[name](rng, h, w)
    return _f32(np.asarray(a, np.float64)), [_f32(np.asarray(b, np.float64)) for b in bs]


def magnitude(x):
    return float(np.abs(x).max())


# ---------------------------------------------------------------------------------------------
# localisation: the first stage of the chain that differs

def _truth(other, stage, *args):
    """A stage of the live reference where it is built, else the same stage of `other`."""
    if reflib.available() and reflib._answers is None:
        return getattr(reflib, stage).__wrapped__(*args)
    return other(stage, *args)


def localise(lib, other_lib, a, b):
    """Runs the planes of a failing pair through the stage hooks of `lib` and compares each stage with
    the live reference (or, without it, with `other_lib`) -> one line naming the first stage and
    pixels that differ."""
    h, w = a.shape[1:]
    img = gb.DeviceImage(np.zeros((h, w, 3), np.uint8), lib=lib, prepare=False)
    oimg = gb.DeviceImage(np.zeros((h, w, 3), np.uint8), lib=other_lib, prepare=False) if other_lib else None

    def other(stage, *args):
        if oimg is None:
            raise LookupError("no live reference and no second library to localise against")
        if stage == "blur":
            return oimg.debug_blur(args[0], parity.BLUR_SPECS.index(tuple(args[1:])))
        return getattr(oimg, "debug_" + stage)(*args)

    def first_diff(got, want, r, what):
        got = np.asarray(got, np.float32).reshape(-1, h, w)
        want = np.asarray(want, np.float32).reshape(-1, h, w)
        for p in range(got.shape[0]):
            bad = np.argwhere(got[p].view(np.uint32) != want[p].view(np.uint32))
            if len(bad):
                return f"{what} differs first in plane {p}: {describe(bad, h, w, r)}"
        return None

    try:
        for name, x in (("original", a), ("candidate", b)):
            xyb = img.debug_opsin(x)
            msg = first_diff(xyb, _truth(other, "opsin", x), RADII[0], f"{name}: opsin")
            if msg:
                return msg
            for c in range(3):
                s, br = parity.BLUR_SPECS[0]
                msg = first_diff(img.debug_blur(x[c], 0), _truth(other, "blur", x[c], s, br), RADII[0],
                                 f"{name}: opsin blur of channel {c}")
                if msg:
                    return msg
            msg = first_diff(img.debug_separate(xyb), _truth(other, "separate", xyb), RADII[1],
                             f"{name}: frequency split")
            if msg:
                return msg
        return "opsin, its blur and the frequency split agree: the difference is after them (Malta, noise, mask or combine)"
    except LookupError as e:
        return str(e)
    finally:
        img.close()
        if oimg is not None:
            oimg.close()


def check_pair(lib, other_lib, a, b, got, want, what):
    dm, score = got
    dm0, score0 = want
    assert np.isfinite(score0), f"{what}: the reference's score is {score0}; the corpus must keep it finite"
    if isinstance(dm0, np.ndarray):
        assert np.isfinite(dm0).all(), f"{what}: the reference's diffmap is not finite"
    if score == score0 and parity.bits_equal(dm, dm0):
        return
    if isinstance(dm0, np.ndarray):
        diff = f"{int((np.asarray(dm, np.float32).view(np.uint32) != dm0.view(np.uint32)).sum())} diffmap pixels differ"
    else:
        diff = "the diffmap differs from the recorded one" if not parity.bits_equal(dm, dm0) else "the diffmaps agree"
    raise AssertionError(f"{what}: score {float(score)!r} vs the reference's {score0!r}, {diff}; "
                         + localise(lib, other_lib, a, b))


# ---------------------------------------------------------------------------------------------
# the checks, shared by the port and the device

def check_case(lib, other_lib, ref, name, h, w, device=False):
    """butteraugli_diffmap and a capacity-1 Comparator (plain launches, graph capture, graph replay on
    the device), host and, on the device, CUDA-tensor input; mask() and adaptive_quantization of the
    original."""
    a, bs = corpus(name, h, w)
    want = [ref.butteraugli_interface(a, b) for b in bs]
    for k, b in enumerate(bs):
        check_pair(lib, other_lib, a, b, gb.api.butteraugli_diffmap(a, b, lib=lib), want[k],
                   f"{name} {h}x{w} candidate {k}, butteraugli_diffmap")
    cmp = gb.Comparator(a, lib=lib)
    try:
        for k, b in enumerate(bs):
            check_pair(lib, other_lib, a, b, cmp.diffmap(b), want[k], f"{name} {h}x{w} candidate {k}, Comparator")
        if device:
            torch = pytest.importorskip("torch")
            for k, b in enumerate(bs):
                dm_t, score_t = cmp.diffmap(torch.from_numpy(b).cuda())
                check_pair(lib, other_lib, a, b, (dm_t.cpu().numpy(), score_t), want[k],
                           f"{name} {h}x{w} candidate {k}, Comparator from CUDA memory")
        dm, score = cmp.diffmap(a)
        assert score == 0.0 and not dm.any(), f"{name} {h}x{w}: the original against itself is not all zeros"
        m, mdc = cmp.mask()
        rm, rmdc = reference_comparator_mask(a)
        assert parity.bits_equal(m, rm) and parity.bits_equal(mdc, rmdc), f"{name} {h}x{w}: mask() differs"
    finally:
        cmp.close()
    if h >= 16 and w >= 16:
        q = gb.adaptive_quantization(a, lib=lib)
        assert parity.bits_equal(q, reference_adaptive_quantization(a)), f"{name} {h}x{w}: adaptive_quantization differs"


def slot_cases(h, w):
    """The cases of one shape, ordered so that neighbouring slots alternate small and large magnitudes."""
    cs = sorted((c for c in CASES if c[1:] == (h, w)), key=lambda c: magnitude(corpus(*c)[1][0]))
    return [cs[i // 2] if i % 2 == 0 else cs[-1 - i // 2] for i in range(len(cs))]


def check_slots(lib, other_lib, ref, h, w, device=False):
    """A capacity-n Comparator scoring the first candidate of every case of the shape against one
    original, and a ButteraugliBatch scoring every case's (original, first candidate) pair, neighbours
    of very different magnitudes; on the device from host and from CUDA memory."""
    cs = slot_cases(h, w)
    pairs = [corpus(*c) for c in cs]
    a = pairs[0][0]
    cands = np.stack([p[1][0] for p in pairs])
    n = len(cs)
    inputs = [cands]
    if device:
        torch = pytest.importorskip("torch")
        inputs.append(torch.from_numpy(cands).cuda())
    cmp = gb.Comparator(a, capacity=n, lib=lib)
    try:
        for x in inputs:
            dm, score = cmp.diffmap(x)
            dm = dm if isinstance(dm, np.ndarray) else dm.cpu().numpy()
            for i in range(n):
                check_pair(lib, other_lib, a, cands[i], (dm[i], score[i]), ref.butteraugli_interface(a, cands[i]),
                           f"{h}x{w} slot {i} of {n} ({case_id(cs[i])} against {case_id(cs[0])}), Comparator")
    finally:
        cmp.close()
    a0 = np.stack([p[0] for p in pairs])
    batch = gb.ButteraugliBatch(h, w, n, lib=lib)
    try:
        ins = [(a0, cands)]
        if device:
            ins.append((torch.from_numpy(a0).cuda(), torch.from_numpy(cands).cuda()))
        for x0, x1 in ins:
            dm, score = batch.diffmap(x0, x1)
            dm = dm if isinstance(dm, np.ndarray) else dm.cpu().numpy()
            for i in range(n):
                check_pair(lib, other_lib, a0[i], cands[i], (dm[i], score[i]), ref.butteraugli_interface(a0[i], cands[i]),
                           f"{h}x{w} slot {i} of {n} ({case_id(cs[i])}), ButteraugliBatch")
    finally:
        batch.close()


def check_stages(lib, ref, name, h, w):
    """OpsinDynamicsImage, SeparateFrequencies and the blurs of the opsin planes on a tier-2 case's
    original and first candidate, each stage from the library's own previous stage."""
    a, bs = corpus(name, h, w)
    img = gb.DeviceImage(np.zeros((h, w, 3), np.uint8), lib=lib, prepare=False)
    try:
        for what, x in (("original", a), ("candidate 0", bs[0])):
            xyb = img.debug_opsin(x)
            assert parity.bits_equal(xyb, ref.opsin(x)), f"{name} {h}x{w} {what}: opsin differs"
            assert np.isfinite(xyb).all(), f"{name} {h}x{w} {what}: opsin is not finite"
            assert parity.bits_equal(img.debug_separate(xyb), ref.separate(xyb)), \
                f"{name} {h}x{w} {what}: frequency split differs"
            for b, (s, br) in enumerate(parity.BLUR_SPECS):
                for c in range(3):
                    p = x[c] if b == 0 else xyb[c]
                    assert parity.bits_equal(img.debug_blur(p, b), ref.blur(p, s, br)), \
                        f"{name} {h}x{w} {what}: blur {b} of plane {c} differs"
    finally:
        img.close()


# ---------------------------------------------------------------------------------------------
# CPU: the corpus itself, the port, and every reference call of the GPU tests

def test_corpus_is_deterministic_and_in_tier():
    """Each case is the same on every call, tier-1 cases stay in 0..255 and tier-2 cases leave it."""
    for c in CASES:
        a, bs = corpus(*c)
        a2, bs2 = corpus(*c)
        assert len(bs) == 3 and all(parity.bits_equal(x, y) for x, y in zip([a] + bs, [a2] + bs2)), c
        xs = np.stack([a] + bs)
        assert xs.shape == (4, 3) + c[1:] and np.isfinite(xs).all(), c
        if GENERATORS[c[0]] in TIER1:
            assert xs.min() >= 0 and xs.max() <= 255, c
        elif GENERATORS[c[0]] in TIER2:
            assert xs.min() < 0 or xs.max() > 255, c
    # every Malta orientation is drawn, as a line longer than its pattern
    for p in range(16):
        assert malta_line(64, 64, p, 32, 32).sum() > len(MALTA[p])
    # the one-ULP candidates differ from the original in exactly one bit pattern
    a, bs = corpus("one_pixel", 40, 56)
    for b in (bs[0], bs[2]):
        assert (a.view(np.uint32) != b.view(np.uint32)).sum() == 1
        assert np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32)).max() == 1


@pytest.mark.parametrize("name,h,w", CASES, ids=[case_id(c) for c in CASES])
def test_port_case(port_lib, ref, name, h, w):
    check_case(port_lib, None, ref, name, h, w)


@pytest.mark.parametrize("h,w", SLOT_SHAPES, ids=lambda v: str(v))
def test_port_slots(port_lib, ref, h, w):
    check_slots(port_lib, None, ref, h, w)


@pytest.mark.parametrize("name,h,w", STAGE_CASES, ids=[case_id(c) for c in STAGE_CASES])
def test_port_stages(port_lib, ref, name, h, w):
    check_stages(port_lib, ref, name, h, w)


# ---------------------------------------------------------------------------------------------
# GPU

@pytest.mark.gpu
@pytest.mark.parametrize("name,h,w", CASES, ids=[case_id(c) for c in CASES])
def test_cuda_case(cuda_lib, port_lib, ref, name, h, w):
    check_case(cuda_lib, port_lib, ref, name, h, w, device=True)


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", SLOT_SHAPES, ids=lambda v: str(v))
def test_cuda_slots(cuda_lib, port_lib, ref, h, w):
    check_slots(cuda_lib, port_lib, ref, h, w, device=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name,h,w", STAGE_CASES, ids=[case_id(c) for c in STAGE_CASES])
def test_cuda_stages(cuda_lib, ref, name, h, w):
    check_stages(cuda_lib, ref, name, h, w)
