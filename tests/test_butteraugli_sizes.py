"""Batched butteraugli on pairs of different sizes (gb200_butteraugli_batch_diffmap_sizes*,
gb.ButteraugliBatch.diffmap_sizes): each pair bit for bit butteraugli::ButteraugliInterface of the reference
on that pair alone (oracle/_ref, or its recorded answers).  Every reference call a GPU test makes is also
made by a CPU test with the same arguments, so that recording the CPU tests covers the GPU tests:

    GB200_REF_RECORD=$PWD/tests/golden/sizes_reference_answers.json \\
        python -m pytest tests/test_butteraugli_sizes.py -m "not gpu"

records them into golden/sizes_reference_answers.json, which replay mode reads beside
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
from guetzli_b200.api import butteraugli_diffmap
from test_butteraugli import linear

ANSWERS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sizes_reference_answers.json")


@pytest.fixture(scope="module")
def ref(ref):
    """The session's reference, with the recorded answers of this module's calls added in replay mode."""
    if reflib._answers is not None:
        with open(ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


def pair(h, w, i):
    """Pair i of a shape: a gradient-and-noise original and a candidate perturbed by up to +-(2 + i % 4)."""
    a = synth.gradnoise(h, w, 2000 + 7 * h + w + 31 * i).astype(int)
    k = i % 4
    b = np.clip(a + synth.noise(h, w, 700 + 3 * i + h) % (2 * k + 5) - (k + 2), 0, 255).astype(np.uint8)
    return linear(a.astype(np.uint8)), linear(b)


def shapes_random(n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    return [(int(h), int(w)) for h, w in rng.integers(lo, hi + 1, size=(n, 2))]


# name -> (batch h, batch w, [(h, w) of each pair]).  The batch's capacity is the number of pairs.
SETS = {
    # rolling-blur segments and strips, pitch padding, both orientations, the batch's own size
    "mixed": (1080, 1920, [(8, 8), (9, 17), (17, 9), (40, 56), (56, 40), (64, 64), (300, 411), (577, 70),
                           (70, 577), (1080, 100), (100, 1080), (1080, 1920)]),
    # every width and every height from 8 to 48 (below 2R + 1 both border rules fall in one window);
    # 41 distinct sizes: more than one pass's 16
    "small": (48, 48, [(8 + i, 8 + (17 * i) % 41) for i in range(41)]),
    # repeated sizes, not adjacent in the call
    "repeated": (64, 64, [(40, 56), (56, 40), (40, 56), (64, 64), (56, 40), (40, 56), (8, 8), (64, 64)]),
    # n = capacity: 255 small pairs of random sizes (many passes) and one large pair
    "capacity": (300, 411, shapes_random(255, 8, 64, 5) + [(300, 411)]),
}


def pairs_of(shapes):
    ps = [pair(h, w, i) for i, (h, w) in enumerate(shapes)]
    return [p[0] for p in ps], [p[1] for p in ps]


def score_sizes(lib, name, order=None):
    bh, bw, shapes = SETS[name]
    a, b = pairs_of(shapes)
    if order is not None:
        a, b = [a[i] for i in order], [b[i] for i in order]
    batch = gb.ButteraugliBatch(bh, bw, len(shapes), lib=lib)
    try:
        dm, score = batch.diffmap_sizes(a, b)
    finally:
        batch.close()
    return a, b, dm, score


def check_against_reference(lib, ref, name, alone=False):
    a, b, dm, score = score_sizes(lib, name)
    assert len(dm) == len(a) and score.shape == (len(a),) and score.dtype == np.float64
    for i in range(len(a)):
        assert dm[i].shape == a[i].shape[1:] and dm[i].dtype == np.float32
        dm0, score0 = ref.butteraugli_interface(a[i], b[i])
        assert score[i] == score0 and parity.bits_equal(dm[i], dm0), f"{name} pair {i} {a[i].shape}: differs from the reference"
        if alone:  # the single-pair entry and a same-size batch of the pair's size give the same bits
            dm1, score1 = butteraugli_diffmap(a[i], b[i], lib=lib)
            assert score1 == score[i] and parity.bits_equal(dm1, dm[i]), f"{name} pair {i}: differs from butteraugli_diffmap"
            _, h, w = a[i].shape
            one = gb.ButteraugliBatch(h, w, 1, lib=lib)
            try:
                dmb, scoreb = one.diffmap(a[i][None], b[i][None])
            finally:
                one.close()
            assert scoreb[0] == score[i] and parity.bits_equal(dmb[0], dm[i]), f"{name} pair {i}: differs from a batch"
    return a, b, dm, score


def refusals(lib, device_entry_message):
    """Every refusal of the C ABI and its message; -> None.  The batch is 40x56 with capacity 3."""
    batch = gb.ButteraugliBatch(40, 56, 3, lib=lib)
    try:
        a, b = pairs_of([(40, 56), (16, 24), (40, 56)])
        P = C.c_void_p * 3
        p0, p1 = P(*[x.ctypes.data for x in a]), P(*[x.ctypes.data for x in b])
        dms = [np.zeros(x.shape[1:], dtype=np.float32) for x in a]
        pd = P(*[x.ctypes.data for x in dms])
        score = np.full(4, -1.0)

        def call(w, h, n=3, q0=p0, q1=p1, qd=pd, device=False, handle=batch._h):
            wa = None if w is None else np.array(w, dtype=np.int32)
            ha = None if h is None else np.array(h, dtype=np.int32)
            wp = None if wa is None else wa.ctypes.data
            hp = None if ha is None else ha.ctypes.data
            if device:
                return lib.gb200_butteraugli_batch_diffmap_sizes_device(handle, wp, hp, q0, q1, n, qd,
                                                                        score.ctypes.data, None)
            return lib.gb200_butteraugli_batch_diffmap_sizes(handle, wp, hp, q0, q1, n, qd, score.ctypes.data)

        W, H = [56, 24, 56], [40, 16, 40]
        for w, h, msg in [([56, 7, 56], H, "pair 1 is 7x16, the batch takes 8x8 up to 56x40"),
                          ([56, 24, 56], [40, 16, 7], "pair 2 is 56x7, the batch takes 8x8 up to 56x40"),
                          ([57, 24, 56], H, "pair 0 is 57x40, the batch takes 8x8 up to 56x40"),
                          (W, [40, 41, 40], "pair 1 is 24x41, the batch takes 8x8 up to 56x40")]:
            assert not call(w, h), (w, h)
            assert msg in gb.last_error(lib=lib), gb.last_error(lib=lib)
        for n in (0, -1, 4):
            assert not call(W + [56], H + [40], n=n)
            assert f"n = {n} pairs, the batch takes 1..3" in gb.last_error(lib=lib)
        for kw in [dict(handle=None), dict(w=None, h=H), dict(w=W, h=None), dict(w=W, h=H, q0=None),
                   dict(w=W, h=H, q1=None)]:
            args = dict(w=W, h=H)
            args.update(kw)
            assert not call(**args), kw
            assert "no batch, no sizes or no images" in gb.last_error(lib=lib)
        for q0, q1, qd in [(P(p0[0], None, p0[2]), p1, pd), (p0, P(p1[0], p1[1], None), pd),
                           (p0, p1, P(None, pd[1], pd[2]))]:
            assert not call(W, H, q0=q0, q1=q1, qd=qd)
            assert "has a null image or diffmap pointer" in gb.last_error(lib=lib), gb.last_error(lib=lib)
        assert not call(W, H, device=True)
        assert device_entry_message in gb.last_error(lib=lib), gb.last_error(lib=lib)
        assert (score == -1.0).all(), "a refused call wrote scores"
        assert not any(d.any() for d in dms), "a refused call wrote diffmaps"
    finally:
        batch.close()


def python_checks(lib):
    batch = gb.ButteraugliBatch(40, 56, 3, lib=lib)
    try:
        a, b = pairs_of([(40, 56), (16, 24)])
        bad = [(a, b[:1]), ([], []), (a * 2, b * 2), ([a[0][0], a[1]], [b[0][0], b[1]]),
               ([a[0].astype(np.float64), a[1]], [b[0].astype(np.float64), b[1]]), ([a[0], a[1]], [b[0], b[0]]),
               ([a[0][:, :, ::2], a[1]], [b[0][:, :, ::2], b[1]]), ([a[0][:2], a[1]], [b[0][:2], b[1]]),
               ([a[0][:, :7], a[1]], [b[0][:, :7], b[1]]), ([np.zeros((3, 41, 56), np.float32)] * 2,) * 2,
               ([a[0].tolist(), a[1]], [b[0].tolist(), b[1]])]
        for x, y in bad:
            with pytest.raises(ValueError):
                batch.diffmap_sizes(x, y)
        dm, score = batch.diffmap_sizes(a, b)  # n < capacity is fine
        assert [d.shape for d in dm] == [(40, 56), (16, 24)] and score.shape == (2,)
    finally:
        batch.close()


# ---- CPU: the port (pair by pair through metrics of their own size), and every reference call of the
# GPU tests ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(SETS))
def test_port_sizes_match_reference(port_lib, ref, name):
    check_against_reference(port_lib, ref, name, alone=name == "mixed")


def test_port_refusals(port_lib):
    refusals(port_lib, "no device memory")


def test_port_python_checks(port_lib):
    python_checks(port_lib)


# ---- GPU ------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SETS))
def test_cuda_sizes_match_reference(cuda_lib, ref, name):
    check_against_reference(cuda_lib, ref, name, alone=name in ("mixed", "repeated"))


@pytest.mark.gpu
def test_cuda_sizes_one_launch_per_stage(cuda_lib):
    """A call with at most 16 sizes is one pass: the same-size batch's launches, plus packing the two
    sides and unpacking the diffmaps."""
    bh, bw, shapes = SETS["mixed"]
    a, b = pairs_of(shapes)
    batch = gb.ButteraugliBatch(bh, bw, len(shapes), lib=cuda_lib)
    try:
        batch.diffmap_sizes(a, b)
        before = gb.counters(lib=cuda_lib)[0]
        batch.diffmap_sizes(a, b)
        mixed = gb.counters(lib=cuda_lib)[0] - before
        x, y = pair(bh, bw, 0)
        before = gb.counters(lib=cuda_lib)[0]
        batch.diffmap(x[None], y[None])
        same = gb.counters(lib=cuda_lib)[0] - before
    finally:
        batch.close()
    assert mixed == same + 3, (mixed, same)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mixed", "small"])
def test_cuda_sizes_permuted(cuda_lib, name):
    """The pairs in another order: every pair's bits are unchanged."""
    a, b, dm, score = score_sizes(cuda_lib, name)
    order = np.random.default_rng(11).permutation(len(a))
    _, _, dmp, scorep = score_sizes(cuda_lib, name, order=order)
    for k, i in enumerate(order):
        assert scorep[k] == score[i] and parity.bits_equal(dmp[k], dm[i]), f"{name} pair {i} at {k}"


def flat_and_noise(shapes):
    """Pair i: for even i a high-contrast noise pair, for odd i an identical flat-gray pair (score 0)."""
    a, b = [], []
    for i, (h, w) in enumerate(shapes):
        if i % 2 == 0:
            a.append(linear(synth.noise(h, w, 70 + i)))
            b.append(linear(synth.noise(h, w, 90 + i)))
        else:
            g = linear(np.full((h, w, 3), 60 + 30 * (i % 6), dtype=np.uint8))
            a.append(g)
            b.append(g.copy())
    return a, b


@pytest.mark.gpu
def test_cuda_sizes_interleaved_with_same_size(cuda_lib):
    """Mixed calls between same-size calls on one object: no slot sees another call's planes, and every
    result equals a fresh object's."""
    h, w, cap = 64, 96, 5
    batch = gb.ButteraugliBatch(h, w, cap, lib=cuda_lib)
    try:
        rounds = [[(64, 96)] * 5, [(33, 50), (64, 96), (20, 90), (64, 17), (9, 9)], [(64, 96)] * 3,
                  [(64, 95), (63, 96), (8, 8)], [(64, 96)] * 5]
        for k, shapes in enumerate(rounds):
            a, b = flat_and_noise(shapes[::-1] if k % 2 else shapes)
            if len(set(shapes)) == 1:
                dm, score = batch.diffmap(np.stack(a), np.stack(b))
            else:
                dm, score = batch.diffmap_sizes(a, b)
            fresh = gb.ButteraugliBatch(h, w, cap, lib=cuda_lib)
            try:
                dmf, scoref = fresh.diffmap_sizes(a, b)
            finally:
                fresh.close()
            for i in range(len(a)):
                assert score[i] == scoref[i] and parity.bits_equal(dm[i], dmf[i]), f"round {k} pair {i}"
                if i % 2 == 1:
                    assert score[i] == 0.0 and not dm[i].any(), f"round {k} identical pair {i}: not all zeros"
                else:
                    assert score[i] > 1.0, f"round {k} noise pair {i}: score {score[i]}"
    finally:
        batch.close()


@pytest.mark.gpu
def test_cuda_sizes_device_path(cuda_lib):
    """Pairs in CUDA memory, written late on a non-default torch stream that the batch must wait for,
    into NaN-filled diffmaps; and scores without diffmaps."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    bh, bw, shapes = SETS["mixed"]
    a, b = pairs_of(shapes)
    n = len(shapes)
    batch = gb.ButteraugliBatch(bh, bw, n, device=0, lib=cuda_lib)
    side = torch.cuda.Stream(device=dev)
    try:
        host_dm, host_score = batch.diffmap_sizes(a, b)
        staged0 = [torch.from_numpy(x).to(dev) for x in a]
        staged1 = [torch.from_numpy(x).to(dev) for x in b]
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            t0 = [torch.full(x.shape, float("nan"), device=dev) for x in a]
            t1 = [torch.full(x.shape, float("nan"), device=dev) for x in b]
            out = [torch.full(x.shape[1:], float("nan"), device=dev) for x in a]
            torch.cuda._sleep(20_000_000)  # keeps the side stream busy: the copies below land late
            for d, s in zip(t0 + t1, staged0 + staged1):
                d.copy_(s)
            P = C.c_void_p * n
            ws = np.array([x.shape[2] for x in a], dtype=np.int32)
            hs = np.array([x.shape[1] for x in a], dtype=np.int32)
            score = np.full(n, -1.0)
            assert cuda_lib.gb200_butteraugli_batch_diffmap_sizes_device(
                batch._h, ws.ctypes.data, hs.ctypes.data, P(*[t.data_ptr() for t in t0]),
                P(*[t.data_ptr() for t in t1]), n, P(*[t.data_ptr() for t in out]), score.ctypes.data,
                side.cuda_stream), gb.last_error(lib=cuda_lib)
            dm_t, score_t = batch.diffmap_sizes(t0, t1)  # the Python path: torch's current stream is `side`
        assert (score == host_score).all() and (score_t == host_score).all()
        for i in range(n):
            assert parity.bits_equal(out[i].cpu().numpy(), host_dm[i]), f"pair {i}: device diffmap differs"
            assert dm_t[i].device == dev and dm_t[i].dtype == torch.float32
            assert parity.bits_equal(dm_t[i].cpu().numpy(), host_dm[i]), f"pair {i}: Python device diffmap differs"
        assert isinstance(score_t, np.ndarray) and score_t.dtype == np.float64
        # scores without diffmaps, from both entries
        torch.cuda.synchronize(dev)
        score = np.full(n, -1.0)
        assert cuda_lib.gb200_butteraugli_batch_diffmap_sizes_device(
            batch._h, ws.ctypes.data, hs.ctypes.data, P(*[t.data_ptr() for t in staged0]),
            P(*[t.data_ptr() for t in staged1]), n, None, score.ctypes.data, None)
        assert (score == host_score).all()
        score = np.full(n, -1.0)
        assert cuda_lib.gb200_butteraugli_batch_diffmap_sizes(
            batch._h, ws.ctypes.data, hs.ctypes.data, P(*[x.ctypes.data for x in a]), P(*[x.ctypes.data for x in b]),
            n, None, score.ctypes.data)
        assert (score == host_score).all()
    finally:
        batch.close()


@pytest.mark.gpu
def test_cuda_refusals_launch_nothing(cuda_lib):
    torch = pytest.importorskip("torch")
    launches = gb.counters(lib=cuda_lib)[0]
    refusals(cuda_lib, "rgb0[0] is not device memory of device 0")
    assert gb.counters(lib=cuda_lib)[0] == launches
    a, b = pairs_of([(40, 56), (16, 24)])
    batch = gb.ButteraugliBatch(40, 56, 2, device=0, lib=cuda_lib)
    try:
        t0 = [torch.from_numpy(x).to("cuda:0") for x in a]
        t1 = [torch.from_numpy(x).to("cuda:0") for x in b]
        dm = [torch.zeros(x.shape[1:], device="cuda:0") for x in a]
        torch.cuda.synchronize()
        P = C.c_void_p * 2
        ws, hs = np.array([56, 24], dtype=np.int32), np.array([40, 16], dtype=np.int32)
        launches = gb.counters(lib=cuda_lib)[0]

        def call(q0, q1, qd):
            return cuda_lib.gb200_butteraugli_batch_diffmap_sizes_device(batch._h, ws.ctypes.data, hs.ctypes.data,
                                                                         P(*q0), P(*q1), 2, qd and P(*qd), None, None)

        dev0, dev1, devd = [t.data_ptr() for t in t0], [t.data_ptr() for t in t1], [t.data_ptr() for t in dm]
        assert not call(dev0, [dev1[0], b[1].ctypes.data], devd)
        assert "rgb1[1] is not device memory of device 0 (host or unknown memory)" in gb.last_error(lib=cuda_lib)
        assert not call(dev0, dev1, [devd[0], np.zeros(1, np.float32).ctypes.data])
        assert "diffmap[1] is not device memory of device 0" in gb.last_error(lib=cuda_lib)
        # managed memory is refused as well (torch's CUDA runtime allocates it)
        rt = None
        for name in ("libcudart.so.12", "libcudart.so"):
            try:
                rt = C.CDLL(name)
                break
            except OSError:
                pass
        if rt is not None:
            managed = C.c_void_p()
            assert rt.cudaMallocManaged(C.byref(managed), C.c_size_t(3 * 40 * 56 * 4), 1) == 0
            try:
                assert not call([managed.value, dev0[1]], dev1, devd)
                assert "rgb0[0] is not device memory of device 0" in gb.last_error(lib=cuda_lib)
            finally:
                rt.cudaFree(managed)
        assert gb.counters(lib=cuda_lib)[0] == launches
        if torch.cuda.device_count() < 2:
            pytest.skip("one GPU: memory of another device cannot be tried")
        other = t0[0].to("cuda:1")
        dm_other = dm[1].to("cuda:1")
        torch.cuda.synchronize("cuda:1")
        launches = gb.counters(lib=cuda_lib)[0]
        assert not call([other.data_ptr(), dev0[1]], dev1, devd)
        assert "rgb0[0] is not device memory of device 0 (device 1)" in gb.last_error(lib=cuda_lib)
        assert not call(dev0, dev1, [devd[0], dm_other.data_ptr()])
        assert "diffmap[1] is not device memory of device 0 (device 1)" in gb.last_error(lib=cuda_lib)
        # the Python entry hands such a tensor to the C entry, as diffmap() does
        with pytest.raises(RuntimeError, match=r"rgb0\[0\] is not device memory of device 0 \(device 1\)"):
            batch.diffmap_sizes([other, t0[1]], t1)
        assert gb.counters(lib=cuda_lib)[0] == launches
    finally:
        batch.close()


@pytest.mark.gpu
def test_cuda_sizes_cache_bound(cuda_lib):
    """More distinct sizes over the calls than the per-size caches keep (256): the caches are dropped and
    rebuilt, and a set scored again afterwards gives the same bits."""
    batch = gb.ButteraugliBatch(64, 64, 120, lib=cuda_lib)
    try:
        everything = [(h, w) for h in range(8, 65) for w in range(8, 65)]
        rng = np.random.default_rng(3)
        order = rng.permutation(len(everything))
        sets = [[everything[i] for i in order[k * 120:(k + 1) * 120]] for k in range(4)]
        first = None
        for k, shapes in enumerate(sets + sets[:1]):
            a, b = pairs_of(shapes)
            dm, score = batch.diffmap_sizes(a, b)
            if k == 0:
                first = (dm, score)
        dm0, score0 = first
        assert (score == score0).all()
        for i in range(len(dm)):
            assert parity.bits_equal(dm[i], dm0[i]), f"pair {i}: differs after the caches were dropped"
        fresh = gb.ButteraugliBatch(64, 64, 120, lib=cuda_lib)
        try:
            dmf, scoref = fresh.diffmap_sizes(a, b)
        finally:
            fresh.close()
        assert (scoref == score).all() and all(parity.bits_equal(x, y) for x, y in zip(dmf, dm))
    finally:
        batch.close()
