"""The rolling-window blur (k_roll_blur, fused_kernels.cuh) and the Compare chain at the shapes where
its layout changes: several segments of a launch, partial last steps and strips, the shared-memory
ring and its wrap copy, the x and y border zones, row-strip launches that start at y0 > 0, and a
Compare that is captured into a CUDA graph and replayed.

A launch of R-radius rows [y0, y_end) is cut into segments of whole GBR_CH-row steps of about
GBR_SEG rows; each CTA blurs one GBR_TW-column strip of one segment through a ring of x-pass rows.
`layout()` restates that split from the constants of the sources, so seam rows move with a retune.

Every device result is compared bit for bit with the unmodified reference and, for the blurs, with
a float64 restatement of butteraugli's Blur (`model`), which gives the size of an error and works
without recorded answers.  A mismatch names the segment, step, strip and ring row it falls on."""
import os
import re
from collections import Counter, namedtuple

import numpy as np
import pytest

import guetzli_b200 as gb
import parity
import reflib
from guetzli_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "guetzli_b200", "csrc")


def _defines(path, names):
    text = open(path).read()
    out = []
    for n in names:
        m = re.search(r"^#define\s+%s\s+(\d+)\b" % n, text, re.M)
        assert m, f"#define {n} not found in {path}"
        out.append(int(m.group(1)))
    return out


SEG, CH, TW = _defines(os.path.join(CSRC, "fused_kernels.cuh"), ["GBR_SEG", "GBR_CH", "GBR_TW"])
# radius of each blur id (tables.h BlurId order)
RADII = _defines(os.path.join(CSRC, "pipeline.cu"),
                 ["GB_R_OPSIN", "GB_R_LF", "GB_R_MF", "GB_R_HF", "GB_R_NOISE", "GB_R_MASKX", "GB_R_MASKY0",
                  "GB_R_MASKY1", "GB_R_FINAL"])
BLUR_LF, BLUR_MF, BLUR_NOISE, BLUR_MASKX, BLUR_MASKY1 = 1, 2, 4, 5, 7


def cdiv(a, b):
    return -(-a // b)


Layout = namedtuple("Layout", "seg starts last last_step")


def layout(rows, y0=0):
    """launch_roll (pipeline.cu): segment length, segment starts, length of the last segment and of
    its last step, for a launch over rows [y0, y0 + rows)."""
    nseg = cdiv(rows, SEG)
    seg = cdiv(cdiv(rows, nseg), CH) * CH
    starts = list(range(y0, y0 + rows, seg))
    last = y0 + rows - starts[-1]
    return Layout(seg, starts, last, last - (cdiv(last, CH) - 1) * CH)


def ring_rows(r, lean=False):
    """RollCfg::RING: D + 2 chunks of x rows for one plane, D + 1 for the lean multi-plane kernel."""
    d = cdiv(2 * r, CH)
    return (d + (1 if lean else 2)) * CH


def where(row, col, h, w, r, lean=False, y0=0, y_end=None):
    """Where output (row, col) of an R-radius rolling blur over rows [y0, y_end) of an h x w plane
    is made: a dict of the structural facts and a one-line description."""
    y_end = h if y_end is None else y_end
    lay = layout(y_end - y0, y0)
    i = min((row - y0) // lay.seg, len(lay.starts) - 1)
    ys = lay.starts[i]
    ye = min(ys + lay.seg, y_end)
    step, o = divmod(row - ys, CH)
    ring = ring_rows(r, lean)
    base = (step % (ring // CH)) * CH + o  # first ring row of the y window; the window is base .. base + 2R
    strip = col // TW
    x0 = strip * TW
    f = dict(segment=i, ys=ys, ye=ye, step=step, strip=strip, x0=x0, ring=(row - ys + r) % ring,
             window=(base, base + 2 * r), wrap=base + 2 * r >= ring,
             last_row=row == ye - 1 and ye < y_end, first_row=row == ys and ys > y0,
             border_strip=x0 < r or x0 + TW + r > w,
             x_border=col < r or col + r >= w, y_border=row < r or row + r >= h)
    win = "ring rows %d..%d" % f["window"]
    if f["wrap"]:
        win += " (wrap copy RING+%d..RING+%d)" % (max(0, base - ring), base + 2 * r - ring)
    f["text"] = (f"({row},{col}): segment {i} [{ys},{ye}) step {step} row {o}, strip {strip} (x0 {x0}"
                 f"{', border-rule strip' if f['border_strip'] else ''}), ring row {f['ring']} of {ring}, {win}"
                 f"{', x border' if f['x_border'] else ''}{', y border' if f['y_border'] else ''}")
    return f


def describe(bad, h, w, r, lean=False, y0=0, y_end=None):
    """The first and last of the (row, col) positions `bad`, and what all of them have in common."""
    bad = [tuple(int(v) for v in p) for p in bad]
    fs = [where(y, x, h, w, r, lean, y0, y_end) for y, x in bad]
    common = []
    for key, text in [("last_row", "last row of a non-final segment"), ("first_row", "first row of a non-first segment"),
                      ("wrap", "the y window reads the ring's wrap copy"), ("y_border", "in the y border zone"),
                      ("x_border", "in the x border zone"), ("border_strip", "in a strip that takes the x border rule")]:
        if all(f[key] for f in fs):
            common.append(text)
    if all(y < r for y, _ in bad):
        common.append("top border rows (row < R)")
    for key in ("segment", "strip", "step"):
        c = Counter(f[key] for f in fs)
        if len(c) == 1:
            common.append(f"all in {key} {next(iter(c))}")
        else:
            common.append(f"{key}s {dict(c.most_common(6))}")
    rc = Counter(f["ring"] for f in fs)
    common.append(f"ring rows {dict(rc.most_common(6))}")
    return (f"{len(bad)} differ; first {fs[0]['text']}; last {fs[-1]['text']}; R={r} RING={ring_rows(r, lean)} "
            f"segments {layout((y_end or h) - y0, y0).starts}; common: " + "; ".join(common))


# ---------------------------------------------------------------------------------------------
# float64 model of the reference Blur (butteraugli.cc:156-233)

def taps(sigma):
    """ComputeKernel (butteraugli.cc:145) in float32: exp(scaler * i * i) with the exponent formed in float."""
    s = np.float32(sigma)
    scaler = np.float32(-1.0 / float(np.float32(2) * s * s))
    diff = max(1, int(np.float32(2.25) * abs(s)))
    i = np.arange(-diff, diff + 1).astype(np.float32)
    return np.exp(((scaler * i) * i).astype(np.float64)).astype(np.float32)


def _conv_x(a, k, br):
    """One Convolution pass along x in float64: interior taps scaled by 1/sum(k); on a border
    (x < R or x + R >= w) the partial tap sum mixed with border_ratio."""
    r = len(k) // 2
    w = a.shape[1]
    out = np.zeros_like(a)
    part = np.zeros(w)
    for j in range(-r, r + 1):
        lo, hi = max(0, -j), min(w, w - j)
        if lo < hi:
            out[:, lo:hi] += a[:, lo + j:hi + j] * k[j + r]
            part[lo:hi] += k[j + r]
    x = np.arange(w)
    total = k.sum()
    border = (x < r) | (x + r >= w)
    return out / np.where(border, (1.0 - br) * part + br * total, total)


def model(img, blur_id):
    """-> (Blur(img) in float64, the same blur of |img|: the scale of the rounding error)."""
    sigma, br = parity.BLUR_SPECS[blur_id]
    k = taps(sigma).astype(np.float64)
    br = float(np.float32(br))
    a = img.astype(np.float64)
    m = _conv_x(_conv_x(a, k, br).T, k, br).T
    am = np.abs(_conv_x(_conv_x(np.abs(a), k, br).T, k, br).T)
    return m, am


# Float32 rounding of the 2(2R+1) products and sums of a pixel is at most 2(2R+1) * 2^-24 of
# |k| (*) |in| (plus 2^-149 per operation once the values are subnormal).  Measured against the
# live reference over the whole table below (test_model_matches_reference_blur), the worst ratio
# of |reference - model| to that bound is 0.537 (blur 8, R 3, uniform plane, 1153 x 64; 0.20 on the
# subnormal planes); C = 1 leaves a factor of 1.9 above it.  A wrong tap, border weight or dropped
# row is off by orders of magnitude more.
C_TOL = 1.0


def tolerance(am, r):
    return C_TOL * 2 * (2 * r + 1) * (am * 2.0 ** -24 + 2.0 ** -149)


def model_ratio(out, blur_id, img):
    m, am = model(img, blur_id)
    r = RADII[blur_id]
    return np.abs(out.astype(np.float64) - m) / (2 * (2 * r + 1) * (am * 2.0 ** -24 + 2.0 ** -149))


# ---------------------------------------------------------------------------------------------
# shapes and planes

# h x w -> what it hits under GBR_SEG = 288, GBR_CH = GBR_TW = 32 (test_shape_table_covers_layouts)
SHAPES = [
    (289, 45),    # 2 segments 160/129, last step of 1 row; R 20/23: the right-border zone spans both strips
    (577, 70),    # 3 segments of 224 (last 129); w mod 32 = 6
    (865, 33),    # 4 segments of 224 (last 193); last strip of 1 column
    (1080, 100),  # the production layout 288/288/288/216; w mod 32 = 4
    (1153, 64),   # 5 segments of 256 (last 129); whole strips
    (576, 411),   # 2 segments of exactly 288, no partial step; 13 strips; w mod 4 = 3
    (8, 40), (17, 300),  # h < R of the noise and mask blurs; R <= h < 2R for lf
    (40, 17), (46, 47),  # w < R; border zones that meet (w <= 2R + 1, h <= 2R)
]
SEP_SHAPES = [(289, 45), (577, 70), (1080, 100)]
KINDS = ["uniform", "signed", "subnormal", "negzero", "constant"]


def plane(kind, h, w):
    rng = np.random.default_rng([h, w, KINDS.index(kind)])
    if kind == "uniform":
        return (rng.random((h, w), dtype=np.float32) * 255).astype(np.float32)
    if kind == "signed":
        return ((rng.random((h, w)) * 2 - 1) * 1e3).astype(np.float32)
    if kind == "subnormal":  # ~1e-38: the products with the taps are subnormal (neither build flushes them)
        return (rng.choice([-1.0, 1.0], (h, w)) * rng.uniform(0.5e-38, 2e-38, (h, w))).astype(np.float32)
    if kind == "negzero":  # 64 x 64 blocks of -0.0 in a uniform plane
        p = (rng.random((h, w), dtype=np.float32) * 255).astype(np.float32)
        y, x = np.mgrid[0:h, 0:w]
        p[(y // 64 + x // 64) % 2 == 0] = -0.0
        return p
    if kind == "constant":
        return np.full((h, w), 77.25, dtype=np.float32)
    raise ValueError(kind)


def impulse_rows(h, r):
    """Rows where a segment's window or ring changes, for a launch over all h rows: per segment
    ys - R - 1, ys - R, ys - 1, ys, ys + R - 1, its last row, and every ring length from ys - R
    (where the one-plane and the lean ring wrap)."""
    out = set()
    lay = layout(h)
    for ys in lay.starts:
        ye = min(ys + lay.seg, h)
        out.update([ys - r - 1, ys - r, ys - 1, ys, ys + r - 1, ye - 1])
        for ring in (ring_rows(r), ring_rows(r, True)):
            out.update(range(ys - r + ring, ye + r, ring))
    return sorted(y for y in out if 0 <= y < h)


def impulse_cols(w, r):
    """x0 - R, x0 - 1, x0, x0 + 31 of every strip, and w - R - 1, w - R."""
    out = {w - r - 1, w - r}
    for x0 in range(0, w, TW):
        out.update([x0 - r, x0 - 1, x0, x0 + TW - 1])
    return sorted(x for x in out if 0 <= x < w)


def impulse_planes(h, w, r):
    """Unit impulses at the structural rows (in three columns) and at the structural columns (in
    three rows)."""
    rows = np.zeros((h, w), dtype=np.float32)
    for y in impulse_rows(h, r):
        rows[y, [0, w // 2, w - 1]] = 1.0
    cols = np.zeros((h, w), dtype=np.float32)
    for x in impulse_cols(w, r):
        cols[[0, h // 2, h - 1], x] = 1.0
    return {"impulse_rows": rows, "impulse_cols": cols}


def table_planes(h, w, blur_id):
    ps = {k: plane(k, h, w) for k in KINDS}
    ps.update(impulse_planes(h, w, RADII[blur_id]))
    return ps


# ---------------------------------------------------------------------------------------------
# CPU tests

def test_shape_table_covers_layouts():
    """Every layout class the shape table is meant to reach is still reached under the constants
    in the sources (fails when a retune makes one disappear; then extend SHAPES)."""
    r_big = min(RADII[BLUR_NOISE], RADII[BLUR_MASKX], RADII[BLUR_MASKY1])
    r_lf, r_max = RADII[BLUR_LF], max(RADII)
    lays = {h: layout(h) for h, _ in SHAPES}

    def nseg(h):
        return len(lays[h].starts)
    classes = {
        "2 segments, last step of 1 row": lambda h, w: nseg(h) == 2 and lays[h].last_step == 1,
        "3 segments": lambda h, w: nseg(h) == 3,
        "4 segments": lambda h, w: nseg(h) == 4,
        "5 segments": lambda h, w: nseg(h) == 5,
        "segments of exactly GBR_SEG rows, no partial step": lambda h, w: (
            nseg(h) >= 2 and lays[h].seg == SEG and lays[h].last == SEG),
        "the production layout of 1080 rows": lambda h, w: h == 1080 and nseg(h) >= 2,
        "partial last strip": lambda h, w: w % TW > 1,
        "last strip of 1 column": lambda h, w: w % TW == 1,
        "whole strips only, more than one": lambda h, w: w % TW == 0 and w > TW,
        "float4 slots past the right edge, many strips": lambda h, w: w % 4 == 3 and cdiv(w, TW) >= 8,
        "right-border zone spans two strips": lambda h, w: TW < w and w - r_max < (cdiv(w, TW) - 1) * TW,
        "h < R of the noise and mask blurs": lambda h, w: h < r_big,
        "R <= h < 2R for lf": lambda h, w: r_lf <= h < 2 * r_lf,
        "w < R": lambda h, w: w < r_big,
        "x border zones meet": lambda h, w: r_big <= w <= 2 * r_max + 1,
        "y border zones meet": lambda h, w: r_big <= h <= 2 * r_max,
    }
    missing = [name for name, hit in classes.items() if not any(hit(h, w) for h, w in SHAPES)]
    assert not missing, f"no shape in SHAPES reaches {missing} under GBR_SEG={SEG} GBR_CH={CH} GBR_TW={TW}"
    # the layouts the table's comments name
    assert [lays[h][:3] for h in (289, 577, 865, 1080, 1153, 576)] == [
        (160, [0, 160], 129), (224, [0, 224, 448], 129), (224, [0, 224, 448, 672], 193),
        (288, [0, 288, 576, 864], 216), (256, [0, 256, 512, 768, 1024], 129), (288, [0, 288], 288)]


def test_layout_matches_launch_grid():
    """layout() against its own definition at every row count up to 3000: whole steps, the grid
    covers the rows, no empty segment."""
    for rows in range(1, 3000):
        for y0 in (0, 37):
            lay = layout(rows, y0)
            assert lay.seg % CH == 0 and lay.seg < SEG + CH
            assert lay.starts[0] == y0 and len(lay.starts) == cdiv(rows, lay.seg)
            assert 0 < lay.last <= lay.seg and 0 < lay.last_step <= CH


@pytest.mark.parametrize("h,w", SHAPES, ids=lambda v: str(v))
def test_model_matches_reference_blur(ref, h, w):
    """The float64 model against the live reference over the whole table; C_TOL is chosen from
    the worst ratio printed here."""
    if not reflib.available():
        pytest.skip("the live reference (oracle/_ref) is not built")
    worst = (0.0, None)
    for b, (s, br) in enumerate(parity.BLUR_SPECS):
        k = ref.blur_kernel(s)
        assert len(k) == 2 * RADII[b] + 1 and parity.same(taps(s), k), f"taps of blur {b}"
        for kind, p in table_planes(h, w, b).items():
            out = ref.blur(p, s, br)
            ratio = model_ratio(out, b, p)
            i = np.unravel_index(np.argmax(ratio), ratio.shape)
            if ratio[i] > worst[0]:
                worst = (float(ratio[i]), (b, kind, i))
            assert ratio[i] <= C_TOL, f"blur {b} {kind}: model off by {ratio[i]:.3g} of the bound at {i}"
            if kind in ("negzero", "constant", "uniform"):
                assert not np.signbit(out).any(), "the reference never returns -0.0 here"
    print(f"{h}x{w}: worst |reference - model| / bound = {worst[0]:.4f} at {worst[1]}")


@pytest.mark.parametrize("h,w", SHAPES, ids=lambda v: str(v))
def test_port_blur_matches_reference(port_lib, ref, h, w):
    """The CPU port as a trusted third opinion at the same shapes: bit-equal to the reference."""
    img = gb.DeviceImage(np.zeros((h, w, 3), np.uint8), lib=port_lib, prepare=False)
    try:
        for b, (s, br) in enumerate(parity.BLUR_SPECS):
            for kind, p in table_planes(h, w, b).items():
                out = img.debug_blur(p, b)
                assert parity.bits_equal(out, ref.blur(p, s, br)), f"port blur {b} {kind} {h}x{w}"
    finally:
        img.close()


# ---------------------------------------------------------------------------------------------
# GPU tests

@pytest.fixture(scope="module")
def images():
    """One unprepared context per shape (debug_blur needs no search state)."""
    cache = {}

    def get(lib, h, w):
        key = (id(lib), h, w)
        if key not in cache:
            cache[key] = gb.DeviceImage(np.zeros((h, w, 3), np.uint8), lib=lib, prepare=False)
        return cache[key]
    yield get
    for img in cache.values():
        img.close()


def check_blur(cuda_lib, port_lib, images, ref, h, w, b, kind, p):
    s, br = parity.BLUR_SPECS[b]
    r = RADII[b]
    got = images(cuda_lib, h, w).debug_blur(p, b)
    want = ref.blur(p, s, br)
    ratio = model_ratio(got, b, p)
    if not parity.bits_equal(got, want):
        port = images(port_lib, h, w).debug_blur(p, b)
        port_ok = parity.bits_equal(port, want)
        truth = want if isinstance(want, np.ndarray) else port if port_ok else None
        if truth is not None:
            bad = np.argwhere(got.view(np.uint32) != np.asarray(truth, np.float32).view(np.uint32))
        else:
            bad = np.argwhere(ratio > C_TOL)
        msg = describe(bad, h, w, r) if len(bad) else "only in bits the model cannot see"
        raise AssertionError(f"blur {b} (R={r}) on {kind} {h}x{w} differs from the reference: {msg}; "
                             f"port equals the reference: {port_ok}, port equals CUDA: {parity.bits_equal(port, got)}; "
                             f"worst model ratio {ratio.max():.3g}")
    bad = np.argwhere(ratio > C_TOL)
    assert not len(bad), f"blur {b} on {kind} {h}x{w} is off the model: {describe(bad, h, w, r)}"


@pytest.mark.gpu
@pytest.mark.parametrize("b", range(len(parity.BLUR_SPECS)))
@pytest.mark.parametrize("h,w", SHAPES, ids=lambda v: str(v))
def test_blur_layouts(cuda_lib, port_lib, images, ref, h, w, b):
    for kind in KINDS:
        check_blur(cuda_lib, port_lib, images, ref, h, w, b, kind, plane(kind, h, w))


@pytest.mark.gpu
@pytest.mark.parametrize("b", range(len(parity.BLUR_SPECS)))
@pytest.mark.parametrize("h,w", SHAPES, ids=lambda v: str(v))
def test_blur_impulses(cuda_lib, port_lib, images, ref, h, w, b):
    for kind, p in impulse_planes(h, w, RADII[b]).items():
        check_blur(cuda_lib, port_lib, images, ref, h, w, b, kind, p)


def first_last(a, b, h, w):
    """Per-plane description of where two [planes][h][w] float arrays differ in bits, for the lf
    (one-plane) and the mf (lean) rolling kernels."""
    a = np.ascontiguousarray(a, np.float32).reshape(-1, h, w)
    b = np.ascontiguousarray(b, np.float32).reshape(-1, h, w)
    out = []
    for i in range(a.shape[0]):
        bad = np.argwhere(a[i].view(np.uint32) != b[i].view(np.uint32))
        if len(bad):
            out.append(f"plane {i}: lf view {describe(bad, h, w, RADII[BLUR_LF])} | "
                       f"mf view {describe(bad, h, w, RADII[BLUR_MF], lean=True)}")
    return "\n".join(out)


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", SEP_SHAPES, ids=lambda v: str(v))
def test_separate_layouts(cuda_lib, ref, h, w):
    """SeparateFrequencies: EpiLf on the one-plane kernel (R 16), EpiMf on the lean three-plane
    kernel (R 8), from an opsin image checked against the reference first."""
    rgb = synth.gradnoise(h, w, h + w)
    img = gb.DeviceImage(rgb, lib=cuda_lib)
    try:
        coeffs = img.orig_coeffs()
        assert parity.same(coeffs, ref.rgb_to_coeffs(rgb)), "FDCT coefficients differ"
        lin = img.debug_render()
        assert parity.bits_equal(lin, ref.render(coeffs, w, h)[1]), "rendered linear RGB differs"
        xyb = img.debug_opsin(lin)
        assert parity.bits_equal(xyb, ref.opsin(lin)), "opsin differs"
        got, want = img.debug_separate(xyb), ref.separate(xyb)
        if not parity.bits_equal(got, want):
            assert isinstance(want, np.ndarray), "frequency split differs from the recorded answer"
            raise AssertionError("frequency split differs:\n" + first_last(got, want, h, w))
    finally:
        img.close()


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,seed", [(577, 70, 9), (1080, 100, 10)])
def test_compare_graph_replay_matches_reference(cuda_lib, ref, h, w, seed, target=0.9):
    """Three Compares on one context: plain launches, then the capture into a CUDA graph, then a
    replay of the graph, each on another candidate, each bit-equal to the reference."""
    rgb = synth.noise(h, w, seed)
    img = gb.DeviceImage(rgb, lib=cuda_lib)
    try:
        coeffs = img.orig_coeffs()
        assert parity.same(coeffs, ref.rgb_to_coeffs(rgb)), "FDCT coefficients differ"
        for call, how in enumerate(["plain launches", "graph capture", "graph replay"]):
            if call < 2:
                img.apply_global_quant(parity.test_quant(2 if call == 0 else 5))
            else:
                flat = img.download_candidate().reshape(-1)
                nz = np.flatnonzero(flat)[::7][:200].astype(np.int32)
                img.scatter(nz, np.zeros(len(nz), dtype=np.int16))
            cand = img.download_candidate()
            dist = img.compare()
            dm = img.distmap()
            rdm, rdist = ref.compare_coeffs(rgb, cand, target)
            if not parity.bits_equal(dm, rdm):
                assert isinstance(rdm, np.ndarray), f"call {call + 1} ({how}): distmap differs from the recorded answer"
                raise AssertionError(f"call {call + 1} ({how}): distmap differs:\n" + first_last(dm, rdm, h, w))
            assert dist == rdist, f"call {call + 1} ({how}): distance {dist} vs {rdist}"
    finally:
        img.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_strip_mode_multi_segment(cuda_lib, port_lib, world):
    """Row-strip mode where each strip with its 56-row halo is longer than one segment, so its
    rolling blurs run as several segments that start at y0 > 0 (off the 32-row grid)."""
    h, w, q = 704, 96, 90
    rgb = synth.gradnoise(h, w, 704)
    bh = cdiv(h, 8)
    strips = []
    for rank in range(world):  # strip_of (comm.h): block rows split as evenly as possible
        lo, hi = rank * bh // world, (rank + 1) * bh // world
        y0, y1 = max(0, 8 * lo - 56), min(h, 8 * hi + 56)
        strips.append((y0, y1, layout(y1 - y0, y0).starts))
    assert any(len(s[2]) >= 2 and s[0] > 0 and s[0] % CH for s in strips), strips
    ok, tiled = gb.process_tiled_threads(
        gb.Params(butteraugli_target=gb.butteraugli_score_for_quality(q, lib=cuda_lib)), rgb, w, h, world, lib=cuda_lib)
    ok1, untiled, _, _ = parity.run_process(cuda_lib, rgb, q)
    ok2, port, _, _ = parity.run_process(port_lib, rgb, q)
    assert ok and ok1 and ok2
    assert untiled == port, f"untiled CUDA differs from the port ({len(untiled)} vs {len(port)} bytes)"
    assert tiled == untiled, (f"world {world}: strip mode differs from untiled ({len(tiled)} vs {len(untiled)} bytes); "
                              f"strips (y0, y1, segment starts) {strips}")
