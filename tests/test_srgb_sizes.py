"""Batched butteraugli on 8-bit sRGB and RGBA pairs of different sizes (gb200_butteraugli_batch_diffmap_sizes_srgb*,
gb.ButteraugliBatch.diffmap_sizes_srgb): each pair bit for bit the stand-alone tool's answer on that pair alone
(test_srgb_inputs.reference, from the reference's ButteraugliInterface) and gb.butteraugli_srgb's.  RGB and
RGBA pairs share calls; RGBA is scored over black and over white, the strictly larger score winning with its
diffmap.  Every reference call a GPU test makes is also made by a CPU test with the same arguments, so that
recording the CPU tests covers the GPU tests:

    GB200_REF_RECORD=$PWD/tests/golden/srgb_sizes_reference_answers.json \\
        python -m pytest tests/test_srgb_sizes.py -m "not gpu"

records them into golden/srgb_sizes_reference_answers.json, which replay mode reads beside
golden/reference_answers.json."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import guetzli_b200 as gb
import parity
import reflib
from guetzli_b200 import synth
from test_butteraugli_sizes import SETS
from test_srgb_inputs import alpha_cases, perturbed, planes, reference, with_alpha

ANSWERS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "srgb_sizes_reference_answers.json")


@pytest.fixture(scope="module")
def ref(ref):
    """The session's reference, with the recorded answers of this module's calls added in replay mode."""
    if reflib._answers is not None:
        with open(ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


def own_sizes(shapes):
    """RGBA on every other distinct size, RGB on the rest: no size has both, so the run over white has
    passes of other sizes than the run over black."""
    distinct = sorted(set(shapes))
    return [4 if distinct.index(s) % 2 == 0 else 3 for s in shapes]


# channel pattern -> [C of each pair] for a set's shapes
PATTERNS = {
    "rgb": lambda shapes: [3] * len(shapes),
    "rgba": lambda shapes: [4] * len(shapes),
    "alternating": lambda shapes: [3 + i % 2 for i in range(len(shapes))],
    "rgba_own_sizes": own_sizes,
}


def pair(h, w, channels, i):
    """Pair i of a set: a gradient-and-noise original, with an alpha channel that takes every value of
    test_srgb_inputs.ALPHAS for RGBA, and a copy perturbed by up to +-(2 + i % 4)."""
    a = with_alpha(synth.gradnoise(h, w, 6000 + 7 * h + w + 31 * i), channels, 6100 + i)
    return a, perturbed(a, 6200 + 3 * i + h, 2 + i % 4)


def pairs_of(shapes, channels):
    ps = [pair(h, w, c, i) for i, ((h, w), c) in enumerate(zip(shapes, channels))]
    return [p[0] for p in ps], [p[1] for p in ps]


def set_pairs(name, pattern):
    bh, bw, shapes = SETS[name]
    a, b = pairs_of(shapes, PATTERNS[pattern](shapes))
    return bh, bw, a, b


def score_set(lib, bh, bw, a, b):
    batch = gb.ButteraugliBatch(bh, bw, len(a), lib=lib)
    try:
        return batch.diffmap_sizes_srgb(a, b)
    finally:
        batch.close()


def check_against_reference(lib, ref, name, pattern):
    bh, bw, a, b = set_pairs(name, pattern)
    dm, score = score_set(lib, bh, bw, a, b)
    assert len(dm) == len(a) and score.shape == (len(a),) and score.dtype == np.float64
    for i in range(len(a)):
        assert dm[i].shape == a[i].shape[:2] and dm[i].dtype == np.float32
        dm0, score0 = reference(ref, a[i], b[i])
        assert score[i] == score0 and parity.bits_equal(dm[i], dm0), \
            f"{name}/{pattern} pair {i} {a[i].shape}: differs from the reference"
    return a, b, dm, score


def check_alone(lib, a, b, dm, score):
    """gb.butteraugli_srgb on each pair alone gives the same bits."""
    for i in range(len(a)):
        dm1, score1 = gb.butteraugli_srgb(a[i], b[i], lib=lib)
        assert score1 == score[i] and parity.bits_equal(dm1, dm[i]), f"pair {i}: differs from butteraugli_srgb"


def reference_only(ref, name, pattern):
    _, _, a, b = set_pairs(name, pattern)
    for i in range(len(a)):
        assert reference(ref, a[i], b[i])[1] >= 0


def choice_pairs():
    """RGBA pairs that white wins (dark content) and that black wins (light content), at two sizes, with RGB
    pairs of other sizes between them -> (a, b, batch h, batch w)."""
    cases = alpha_cases()
    a, b = [], []
    for k, (_, x, y, _) in enumerate(cases + cases):
        if k >= len(cases):
            x, y = np.ascontiguousarray(x[:33, :47]), np.ascontiguousarray(y[:33, :47])
        a.append(x)
        b.append(y)
        r0, r1 = pair(24 + 8 * k, 16 + 4 * k, 3, k)
        a.append(r0)
        b.append(r1)
    return a, b, 56, 56


def check_choice(lib, ref, device=False):
    """The winner of every RGBA pair is the reference's, white and black both win somewhere, and each pair
    gets the winner's bits, from host memory and (device) from CUDA memory."""
    a, b, bh, bw = choice_pairs()
    dm, score = score_set(lib, bh, bw, a, b)
    won = set()
    for i in range(len(a)):
        if a[i].shape[2] == 3:
            want = reference(ref, a[i], b[i])
        else:
            per_bg = {bg: ref.butteraugli_interface(planes(a[i], bg), planes(b[i], bg)) for bg in (0, 255)}
            winner = 255 if per_bg[255][1] > per_bg[0][1] else 0
            won.add(winner)
            want = per_bg[winner]
        assert score[i] == want[1] and parity.bits_equal(dm[i], want[0]), f"pair {i}"
    assert won == {0, 255}, won
    if device:
        import torch
        dmt, scoret = score_set(lib, bh, bw, [torch.from_numpy(x).cuda() for x in a],
                                [torch.from_numpy(x).cuda() for x in b])
        assert (scoret == score).all()
        for i in range(len(a)):
            assert parity.bits_equal(dmt[i].cpu().numpy(), dm[i]), f"pair {i} (device)"


def check_order(lib, name, pattern):
    """The pairs in another order: every pair's bits are unchanged."""
    bh, bw, a, b = set_pairs(name, pattern)
    dm, score = score_set(lib, bh, bw, a, b)
    order = np.random.default_rng(13).permutation(len(a))
    dmp, scorep = score_set(lib, bh, bw, [a[i] for i in order], [b[i] for i in order])
    for k, i in enumerate(order):
        assert scorep[k] == score[i] and parity.bits_equal(dmp[k], dm[i]), f"{name}/{pattern} pair {i} at {k}"


def c_args(x):
    """-> (w, h, channels) int32 arrays of a list of [h][w][C] images."""
    return tuple(np.array([s[k] for s in (t.shape for t in x)], dtype=np.int32) for k in (1, 0, 2))


def check_optional_outputs(lib):
    """A NULL diffmap, NULL entries in it and a NULL score: the other outputs are those of a full call.
    The RGBA pairs include one that white wins, so a NULL entry meets the replacement of diffmaps."""
    a, b, bh, bw = choice_pairs()
    n = len(a)
    dm, score = score_set(lib, bh, bw, a, b)
    ws, hs, chs = c_args(a)
    P = C.c_void_p * n
    p0, p1 = P(*[x.ctypes.data for x in a]), P(*[x.ctypes.data for x in b])
    batch = gb.ButteraugliBatch(bh, bw, n, lib=lib)
    try:
        def call(qd, qs):
            assert lib.gb200_butteraugli_batch_diffmap_sizes_srgb(batch._h, ws.ctypes.data, hs.ctypes.data,
                                                                  chs.ctypes.data, p0, p1, n, qd, qs), \
                gb.last_error(lib=lib)

        s = np.full(n, -1.0)
        call(None, s.ctypes.data)
        assert (s == score).all()
        out = [np.full(x.shape[:2], np.nan, dtype=np.float32) for x in a]
        keep = [i % 3 != 1 for i in range(n)]
        s = np.full(n, -1.0)
        call(P(*[o.ctypes.data if k else None for o, k in zip(out, keep)]), s.ctypes.data)
        assert (s == score).all()
        for i in range(n):
            if keep[i]:
                assert parity.bits_equal(out[i], dm[i]), f"pair {i}"
            else:
                assert np.isnan(out[i]).all(), f"pair {i}: a NULL entry, yet its map was written"
        out = [np.full(x.shape[:2], np.nan, dtype=np.float32) for x in a]
        call(P(*[o.ctypes.data for o in out]), None)
        assert all(parity.bits_equal(o, d) for o, d in zip(out, dm))
    finally:
        batch.close()


def refusals(lib, device_entry_message):
    """Every refusal of the C ABI, each with its message, launching nothing and writing nothing.  The batch
    is 40x56 with capacity 3."""
    a, b = pairs_of([(40, 56), (16, 24), (40, 56)], [3, 4, 4])
    batch = gb.ButteraugliBatch(40, 56, 3, lib=lib)
    try:
        P = C.c_void_p * 3
        p0, p1 = P(*[x.ctypes.data for x in a]), P(*[x.ctypes.data for x in b])
        dms = [np.zeros(x.shape[:2], dtype=np.float32) for x in a]
        pd = P(*[x.ctypes.data for x in dms])
        score = np.full(4, -1.0)
        W, H, CH = [56, 24, 56], [40, 16, 40], [3, 4, 4]

        def call(w=W, h=H, ch=CH, n=3, q0=p0, q1=p1, qd=pd, device=False, handle=batch._h):
            arrs = [None if v is None else np.array(v, dtype=np.int32) for v in (w, h, ch)]
            wp, hp, cp = [None if v is None else v.ctypes.data for v in arrs]
            if device:
                return lib.gb200_butteraugli_batch_diffmap_sizes_srgb_device(handle, wp, hp, cp, q0, q1, n, qd,
                                                                             score.ctypes.data, None)
            return lib.gb200_butteraugli_batch_diffmap_sizes_srgb(handle, wp, hp, cp, q0, q1, n, qd, score.ctypes.data)

        def refused(msg, **kw):
            assert not call(**kw), kw
            assert msg in gb.last_error(lib=lib), (msg, gb.last_error(lib=lib))

        launches = gb.counters(lib=lib)[0]
        smaller = " (gb200_butteraugli_diffmap_srgb scores smaller pairs)"
        refused("pair 1 is 7x16, the batch takes 8x8 up to 56x40" + smaller, w=[56, 7, 56])
        refused("pair 2 is 56x7, the batch takes 8x8 up to 56x40" + smaller, h=[40, 16, 7])
        refused("pair 0 is 57x40, the batch takes 8x8 up to 56x40", w=[57, 24, 56])
        assert smaller not in gb.last_error(lib=lib)
        refused("pair 1 is 24x41, the batch takes 8x8 up to 56x40", h=[40, 41, 40])
        for n in (0, -1, 4):
            refused(f"n = {n} pairs, the batch takes 1..3", n=n, w=W + [56], h=H + [40], ch=CH + [3])
        for ch in (0, 1, 2, 5):
            refused(f"pair 2: channels = {ch}, 8-bit images must have 3 (RGB) or 4 (RGBA)", ch=[3, 4, ch])
        for kw in [dict(handle=None), dict(w=None), dict(h=None), dict(ch=None), dict(q0=None), dict(q1=None)]:
            refused("no batch, no sizes, no channels or no images", **kw)
        refused("pair 1 has a null image pointer", q0=P(p0[0], None, p0[2]))
        refused("pair 2 has a null image pointer", q1=P(p1[0], p1[1], None))
        refused(device_entry_message, device=True)
        assert gb.counters(lib=lib)[0] == launches
        assert (score == -1.0).all(), "a refused call wrote scores"
        assert not any(d.any() for d in dms), "a refused call wrote diffmaps"
    finally:
        batch.close()


def python_checks(lib):
    """Malformed arguments raise ValueError before anything reaches the library."""
    a, b = pairs_of([(40, 56), (16, 24)], [3, 4])
    batch = gb.ButteraugliBatch(40, 56, 3, lib=lib)
    try:
        launches = gb.counters(lib=lib)[0]
        bad = [(a, b[:1]), ([], []), (a * 2, b * 2),  # lengths, n out of range
               ([a[0].astype(np.float32), a[1]], [b[0].astype(np.float32), b[1]]),  # dtype
               ([a[0][..., 0], a[1]], [b[0][..., 0], b[1]]), ([a[0][None], a[1]], [b[0][None], b[1]]),  # rank
               ([a[0][..., :2], a[1]], [b[0][..., :2], b[1]]),  # last axis
               ([np.dstack([a[1], a[1][..., :1]]), a[1]], [np.dstack([b[1], b[1][..., :1]]), b[1]]),
               ([a[0][:, ::2], a[1]], [b[0][:, ::2], b[1]]),  # contiguity
               ([a[0], a[1]], [b[0], b[0]]),  # a pair differing in shape
               ([a[0], a[1]], [b[0], b[1][..., :3].copy()]),  # ... and in channels
               ([a[0][:7], a[1]], [b[0][:7], b[1]]),  # below 8x8
               ([np.zeros((41, 56, 3), np.uint8)] * 2,) * 2,  # above the batch
               ([a[0].tolist(), a[1]], [b[0].tolist(), b[1]])]
        for x, y in bad:
            with pytest.raises(ValueError):
                batch.diffmap_sizes_srgb(x, y)
        with pytest.raises(ValueError, match="different number of channels: 4 and 3"):
            batch.diffmap_sizes_srgb(a, [b[0], b[1][..., :3].copy()])
        assert gb.counters(lib=lib)[0] == launches
        dm, score = batch.diffmap_sizes_srgb(a, b)  # n < capacity is fine
        assert [d.shape for d in dm] == [(40, 56), (16, 24)] and score.shape == (2,)
    finally:
        batch.close()


# set, pattern pairs of each check.  The port scores every pattern of the mixed, small and repeated sets;
# the reference calls of the capacity set (256 pairs) are made by a reference-only CPU test.
PORT_CASES = [(s, p) for s in ("mixed", "small", "repeated") for p in PATTERNS]
GPU_CASES = PORT_CASES + [("capacity", "alternating")]


# ---- CPU: the port, and every reference call of the GPU tests ------------------------------------------

@pytest.mark.parametrize("name,pattern", PORT_CASES)
def test_port_sizes_srgb_match_reference(port_lib, ref, name, pattern):
    a, b, dm, score = check_against_reference(port_lib, ref, name, pattern)
    if name == "repeated":
        check_alone(port_lib, a, b, dm, score)


@pytest.mark.parametrize("name,pattern", [c for c in GPU_CASES if c not in PORT_CASES])
def test_reference_answers_of_gpu_sets(ref, name, pattern):
    """The reference calls of the GPU-only cases, which the port would take minutes to score."""
    reference_only(ref, name, pattern)


def test_port_choice(port_lib, ref):
    check_choice(port_lib, ref)


def test_port_order(port_lib):
    check_order(port_lib, "repeated", "alternating")


def test_port_optional_outputs(port_lib):
    check_optional_outputs(port_lib)


def test_port_refusals(port_lib):
    refusals(port_lib, "no device memory")


def test_port_python_checks(port_lib):
    python_checks(port_lib)


# ---- GPU ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name,pattern", GPU_CASES)
def test_cuda_sizes_srgb_match_reference(cuda_lib, ref, name, pattern):
    a, b, dm, score = check_against_reference(cuda_lib, ref, name, pattern)
    if name in ("mixed", "repeated"):
        check_alone(cuda_lib, a, b, dm, score)


@pytest.mark.gpu
def test_cuda_choice(cuda_lib, ref):
    check_choice(cuda_lib, ref, device=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mixed", "small"])
def test_cuda_order(cuda_lib, name):
    check_order(cuda_lib, name, "alternating")


@pytest.mark.gpu
def test_cuda_optional_outputs(cuda_lib):
    """The host entry as on the port, and the device entry with NULL entries in diffmap and a NULL score."""
    torch = pytest.importorskip("torch")
    check_optional_outputs(cuda_lib)
    a, b, bh, bw = choice_pairs()
    n = len(a)
    dm, score = score_set(cuda_lib, bh, bw, a, b)
    t0, t1 = [torch.from_numpy(x).cuda() for x in a], [torch.from_numpy(x).cuda() for x in b]
    out = [torch.full(x.shape[:2], float("nan"), device="cuda") for x in a]
    torch.cuda.synchronize()
    ws, hs, chs = c_args(a)
    P = C.c_void_p * n
    batch = gb.ButteraugliBatch(bh, bw, n, lib=cuda_lib)
    try:
        keep = [i % 3 != 1 for i in range(n)]
        s = np.full(n, -1.0)
        for qd, qs in ((None, s.ctypes.data), (P(*[o.data_ptr() if k else None for o, k in zip(out, keep)]), None)):
            assert cuda_lib.gb200_butteraugli_batch_diffmap_sizes_srgb_device(
                batch._h, ws.ctypes.data, hs.ctypes.data, chs.ctypes.data, P(*[t.data_ptr() for t in t0]),
                P(*[t.data_ptr() for t in t1]), n, qd, qs, None), gb.last_error(lib=cuda_lib)
        assert (s == score).all()
        for i in range(n):
            got = out[i].cpu().numpy()
            if keep[i]:
                assert parity.bits_equal(got, dm[i]), f"pair {i}"
            else:
                assert np.isnan(got).all(), f"pair {i}: a NULL entry, yet its map was written"
    finally:
        batch.close()


@pytest.mark.gpu
def test_cuda_device_path(cuda_lib):
    """Pairs in CUDA memory give the host call's bits, also when they are written late on a busy
    non-default torch stream that the batch must wait for."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    bh, bw, a, b = set_pairs("mixed", "alternating")
    n = len(a)
    host_dm, host_score = score_set(cuda_lib, bh, bw, a, b)
    batch = gb.ButteraugliBatch(bh, bw, n, device=0, lib=cuda_lib)
    side = torch.cuda.Stream(device=dev)
    try:
        staged = [torch.from_numpy(x).to(dev) for x in a + b]
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            t = [torch.zeros_like(x) for x in staged]
            torch.cuda._sleep(20_000_000)  # keeps the side stream busy: the copies below land late
            for d, s in zip(t, staged):
                d.copy_(s)
            dm_t, score_t = batch.diffmap_sizes_srgb(t[:n], t[n:])  # torch's current stream is `side`
        torch.cuda.synchronize(dev)
        assert isinstance(score_t, np.ndarray) and (score_t == host_score).all()
        for i in range(n):
            assert dm_t[i].device == dev and dm_t[i].dtype == torch.float32
            assert parity.bits_equal(dm_t[i].cpu().numpy(), host_dm[i]), f"pair {i}: device diffmap differs"
    finally:
        torch.cuda.synchronize(dev)
        batch.close()


@pytest.mark.gpu
def test_cuda_refusals_launch_nothing(cuda_lib):
    torch = pytest.importorskip("torch")
    refusals(cuda_lib, "img0[0] is not device memory of device 0")
    python_checks(cuda_lib)
    a, b = pairs_of([(40, 56), (16, 24)], [4, 3])
    batch = gb.ButteraugliBatch(40, 56, 2, device=0, lib=cuda_lib)
    try:
        t0 = [torch.from_numpy(x).to("cuda:0") for x in a]
        t1 = [torch.from_numpy(x).to("cuda:0") for x in b]
        dm = [torch.zeros(x.shape[:2], device="cuda:0") for x in a]
        torch.cuda.synchronize()
        P = C.c_void_p * 2
        ws, hs, chs = c_args(a)
        launches = gb.counters(lib=cuda_lib)[0]

        def call(q0, q1, qd):
            return cuda_lib.gb200_butteraugli_batch_diffmap_sizes_srgb_device(
                batch._h, ws.ctypes.data, hs.ctypes.data, chs.ctypes.data, P(*q0), P(*q1), 2, qd and P(*qd), None,
                None)

        dev0, dev1, devd = [t.data_ptr() for t in t0], [t.data_ptr() for t in t1], [t.data_ptr() for t in dm]
        assert not call(dev0, [dev1[0], b[1].ctypes.data], devd)
        assert "img1[1] is not device memory of device 0 (host or unknown memory)" in gb.last_error(lib=cuda_lib)
        assert not call(dev0, dev1, [devd[0], np.zeros(1, np.float32).ctypes.data])
        assert "diffmap[1] is not device memory of device 0" in gb.last_error(lib=cuda_lib)
        with pytest.raises(ValueError, match="must all be CUDA tensors or all host arrays"):
            batch.diffmap_sizes_srgb([t0[0], a[1]], t1)
        assert gb.counters(lib=cuda_lib)[0] == launches
        if torch.cuda.device_count() < 2:
            pytest.skip("one GPU: memory of another device cannot be tried")
        other = t0[0].to("cuda:1")
        torch.cuda.synchronize("cuda:1")
        launches = gb.counters(lib=cuda_lib)[0]
        assert not call([other.data_ptr(), dev0[1]], dev1, devd)
        assert "img0[0] is not device memory of device 0 (device 1)" in gb.last_error(lib=cuda_lib)
        with pytest.raises(RuntimeError, match=r"img0\[0\] is not device memory of device 0 \(device 1\)"):
            batch.diffmap_sizes_srgb([other, t0[1]], t1)
        assert gb.counters(lib=cuda_lib)[0] == launches
    finally:
        batch.close()


def uploaded(lib, f):
    f()  # the buffers' first use
    before = gb.counters(lib=lib)[1]
    f()
    return gb.counters(lib=lib)[1] - before


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["rgb", "alternating"])
def test_cuda_upload_is_the_bytes(cuda_lib, pattern):
    """A host call uploads its 8-bit images once, as bytes, whatever the backgrounds: on an all-RGB set
    exactly sum 2 h w 3 bytes more than the float twin's call (on the converted planes) uploads besides its
    images, sum 2 h w 12 bytes.  With RGBA pairs the run over white uploads its own tables, at most the
    twin's, and no images."""
    bh, bw, a, b = set_pairs("mixed", pattern)
    batch = gb.ButteraugliBatch(bh, bw, len(a), lib=cuda_lib)
    try:
        up = uploaded(cuda_lib, lambda: batch.diffmap_sizes_srgb(a, b))
        fa, fb = [planes(x, 0) for x in a], [planes(x, 0) for x in b]
        up_float = uploaded(cuda_lib, lambda: batch.diffmap_sizes(fa, fb))
    finally:
        batch.close()
    images = sum(2 * x.size for x in a)
    tables = up_float - sum(2 * x.size * 4 for x in fa)
    assert 0 < tables < images
    if pattern == "rgb":
        assert up == images + tables, (up, images, tables)
    else:
        assert images + tables < up <= images + 2 * tables, (up, images, tables)
