"""The batched comparator (gb200_butteraugli_comparator_create_batch / _diffmap_batch[_device],
gb.Comparator(rgb0, capacity=N)): one resident original scored against N candidates per call, each
bit for bit butteraugli::ButteraugliInterface(rgb0, rgb1[i]) of the reference (oracle/_ref, or its
recorded answers).  Every reference call a GPU test makes is also made by a CPU test with the same
arguments, so that recording the CPU tests covers the GPU tests:

    GB200_REF_RECORD=$PWD/tests/golden/comparator_batch_reference_answers.json \\
        python -m pytest tests/test_comparator_batch.py -m "not gpu"

records them into golden/comparator_batch_reference_answers.json, which replay mode reads beside
golden/reference_answers.json."""
import ctypes as C
import json
import os
import threading

import numpy as np
import pytest

import guetzli_b200 as gb
import parity
import reflib
from guetzli_b200 import synth
from test_butteraugli import linear

ANSWERS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "comparator_batch_reference_answers.json")


@pytest.fixture(scope="module")
def ref(ref):
    """The session's reference, with the recorded answers of this module's calls added in replay mode."""
    if reflib._answers is not None:
        with open(ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


# (h, w, n): one comparator of capacity n per shape, scoring n distinct candidates (the shapes of the
# pair batch's tests: pitch padding, one and several strips and segments, a 1040-deep widest launch)
CASES = [(8, 8, 33), (9, 17, 7), (40, 56, 5), (17, 130, 3), (64, 64, 64), (12, 20, 260), (300, 411, 4),
         (577, 70, 3), (1080, 100, 2), (1080, 1920, 2)]
# two comparators of different shapes on two threads at once (shapes of CASES)
PAIR = [(40, 56, 5), (300, 411, 4)]


def original(h, w):
    return synth.gradnoise(h, w, 2000 + 7 * h + w).astype(int)


def candidates(h, w, n, first=0):
    """-> (rgb0 [3][h][w], rgb1 [n][3][h][w]): a gradient-and-noise original and candidates i = first ..
    first + n - 1, each perturbed by up to +-(2 + i % 4)."""
    a = original(h, w)
    out = []
    for i in range(first, first + n):
        k = i % 4
        out.append(linear(np.clip(a + synth.noise(h, w, 600 + 3 * i + h) % (2 * k + 5) - (k + 2), 0, 255)
                          .astype(np.uint8)))
    return linear(a.astype(np.uint8)), np.stack(out)


def check_against_reference(lib, ref, h, w, n, gpu=False):
    a, b = candidates(h, w, n)
    cmp = gb.Comparator(a, capacity=n, lib=lib)
    try:
        dm, score = cmp.diffmap(b)
    finally:
        cmp.close()
    assert dm.shape == (n, h, w) and dm.dtype == np.float32 and score.shape == (n,) and score.dtype == np.float64
    for i in range(n):
        dm0, score0 = ref.butteraugli_interface(a, b[i])
        assert score[i] == score0 and parity.bits_equal(dm[i], dm0), f"{h}x{w} candidate {i} of {n}: differs from the reference"
    if gpu:
        one = gb.Comparator(a, lib=lib)  # capacity 1: the single-image comparator
        try:
            for i in range(n):
                dm1, score1 = one.diffmap(b[i])
                assert score1 == score[i] and parity.bits_equal(dm1, dm[i]), f"{h}x{w} candidate {i}: differs from Comparator"
        finally:
            one.close()
        batch = gb.ButteraugliBatch(h, w, n, lib=lib)
        try:
            dmb, scoreb = batch.diffmap(np.ascontiguousarray(np.broadcast_to(a, b.shape)), b)
        finally:
            batch.close()
        assert (scoreb == score).all() and parity.bits_equal(dmb, dm), f"{h}x{w}: differs from ButteraugliBatch"
    return dm, score


def refusals(lib, device_entry_message):
    """Every refusal of the C ABI and its message, each launching nothing; -> None.  The comparator is
    40x56 with capacity 3."""
    a, b = candidates(40, 56, 3)
    launches = gb.counters(lib=lib)[0]
    for w, h, cap, msg in [(7, 20, 1, "at least 8x8"), (20, 7, 2, "at least 8x8"), (65536, 8, 2, "below 65536"),
                           (20, 20, 0, "capacity must be in 1..16383"), (20, 20, 16384, "capacity must be in 1..16383")]:
        img = np.zeros((3, min(h, 64), min(w, 64)), dtype=np.float32)  # never read: the size is refused first
        assert not lib.gb200_butteraugli_comparator_create_batch(img.ctypes.data, w, h, cap, 0), (w, h, cap)
        assert msg in gb.last_error(lib=lib), (w, h, cap, gb.last_error(lib=lib))
    assert not lib.gb200_butteraugli_comparator_create_batch(None, 56, 40, 3, 0)
    assert "no image" in gb.last_error(lib=lib)
    assert gb.counters(lib=lib)[0] == launches
    cmp = gb.Comparator(a, capacity=3, lib=lib)
    try:
        launches = gb.counters(lib=lib)[0]  # after the original's analysis
        score = np.full(4, -1.0)
        for n in (0, -1, 4):
            assert not lib.gb200_butteraugli_comparator_diffmap_batch(cmp._h, b.ctypes.data, n, None, score.ctypes.data)
            assert f"n = {n} images, the comparator takes 1..3" in gb.last_error(lib=lib)
            assert not lib.gb200_butteraugli_comparator_diffmap_batch_device(cmp._h, b.ctypes.data, n, None,
                                                                             score.ctypes.data, None)
            assert f"n = {n} images, the comparator takes 1..3" in gb.last_error(lib=lib)
        assert not lib.gb200_butteraugli_comparator_diffmap_batch(cmp._h, None, 1, None, score.ctypes.data)
        assert "no comparator or no images" in gb.last_error(lib=lib)
        assert not lib.gb200_butteraugli_comparator_diffmap_batch(None, b.ctypes.data, 1, None, score.ctypes.data)
        assert "no comparator or no images" in gb.last_error(lib=lib)
        assert not lib.gb200_butteraugli_comparator_diffmap_batch_device(cmp._h, b.ctypes.data, 2, None,
                                                                         score.ctypes.data, None)
        assert device_entry_message in gb.last_error(lib=lib), gb.last_error(lib=lib)
        assert (score == -1.0).all(), "a refused call wrote scores"
        assert gb.counters(lib=lib)[0] == launches
    finally:
        cmp.close()


def python_checks(lib):
    a, b = candidates(40, 56, 3)
    cmp = gb.Comparator(a, capacity=3, lib=lib)
    try:
        bad = [b[:0], b[None], b[:, :, :39], b[:, :2], b.astype(np.float64), b.astype(np.float16),
               np.concatenate([b, b[:1]]), b[:, :, :, :55], b[0, 0]]
        for x in bad:
            with pytest.raises(ValueError):
                cmp.diffmap(x)
        dm, score = cmp.diffmap(b[:1])  # n < capacity is fine
        assert dm.shape == (1, 40, 56) and score.shape == (1,) and score.dtype == np.float64
        dm1, score1 = cmp.diffmap(b[0])  # [3][h][w]: the single-image call, as on a capacity-1 comparator
        assert dm1.shape == (40, 56) and isinstance(score1, float)
        assert score1 == score[0] and parity.bits_equal(dm1, dm[0])
    finally:
        cmp.close()
    with pytest.raises(RuntimeError, match="capacity must be in 1..16383"):
        gb.Comparator(a, capacity=0, lib=lib)


# ---- CPU: the port (candidate by candidate through a single-image metric), and every reference call
# of the GPU tests --------------------------------------------------------------------------------

@pytest.mark.parametrize("h,w,n", CASES)
def test_port_comparator_batch_matches_reference(port_lib, ref, h, w, n):
    check_against_reference(port_lib, ref, h, w, n)


def test_port_refusals(port_lib):
    refusals(port_lib, "no device memory")


def test_port_python_checks(port_lib):
    python_checks(port_lib)


# ---- GPU ------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("h,w,n", CASES)
def test_cuda_comparator_batch_matches_reference(cuda_lib, ref, h, w, n):
    check_against_reference(cuda_lib, ref, h, w, n, gpu=True)


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,n", [(40, 56, 6), (300, 411, 5)])
def test_cuda_slots_are_isolated(cuda_lib, h, w, n):
    """Candidates alternate noise with exact copies of the original: the copies score 0 with an all-zero
    diffmap, and the reversed candidates give the reversed results."""
    a = linear(synth.noise(h, w, 77))
    b = np.stack([linear(synth.noise(h, w, 90 + i)) if i % 2 == 0 else a.copy() for i in range(n)])
    cmp = gb.Comparator(a, capacity=n, lib=cuda_lib)
    try:
        dm, score = cmp.diffmap(b)
        for i in range(n):
            if i % 2 == 1:
                assert score[i] == 0.0 and not dm[i].any(), f"copy {i}: not all zeros"
            else:
                assert score[i] > 1.0, f"noise candidate {i}: score {score[i]}"
        dmr, scorer = cmp.diffmap(b[::-1].copy())
        assert (scorer == score[::-1]).all() and parity.bits_equal(dmr, dm[::-1]), "the reversed candidates"
    finally:
        cmp.close()


@pytest.mark.gpu
def test_cuda_partial_calls(cuda_lib):
    """n = capacity, 1, capacity - 1, capacity on one object, different candidates each time, a unique one
    in the last used slot: every result equals a fresh object's."""
    h, w, cap = 64, 96, 5
    a, _ = candidates(h, w, 1)
    cmp = gb.Comparator(a, capacity=cap, lib=cuda_lib)
    try:
        first = 0
        for k, n in enumerate([cap, 1, cap - 1, cap]):
            _, b = candidates(h, w, n, first)
            first += n
            b[n - 1] = linear(synth.noise(h, w, 300 + k))  # unique: noise against a gradient
            dm, score = cmp.diffmap(b)
            fresh = gb.Comparator(a, capacity=cap, lib=cuda_lib)
            try:
                dmf, scoref = fresh.diffmap(b)
            finally:
                fresh.close()
            assert (score == scoref).all() and parity.bits_equal(dm, dmf), f"call {k} (n = {n})"
    finally:
        cmp.close()


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,cap", [(40, 56, 4), (300, 411, 3)])
def test_cuda_mixed_calls(cuda_lib, h, w, cap):
    """Single-candidate host and device calls and mask() interleaved with batched calls on one
    capacity-N comparator: every result equals a capacity-1 comparator's."""
    torch = pytest.importorskip("torch")
    a, b = candidates(h, w, cap)
    one = gb.Comparator(a, lib=cuda_lib)
    many = gb.Comparator(a, capacity=cap, lib=cuda_lib)
    try:
        want = [one.diffmap(b[i]) for i in range(cap)]
        mask_want = one.mask()
        t = torch.from_numpy(b).cuda()

        def same_batch(got, k):
            dm, score = got
            for i in range(cap):
                assert score[i] == want[i][1] and parity.bits_equal(dm[i], want[i][0]), f"step {k} candidate {i}"

        same_batch(many.diffmap(b), 0)
        for k, i in enumerate([0, cap - 1, 1]):
            dm, score = many.diffmap(b[i])  # host, single
            assert score == want[i][1] and parity.bits_equal(dm, want[i][0]), f"host single {i}"
            dm_t, score_t = many.diffmap(t[i])  # device, single
            assert score_t == want[i][1] and parity.bits_equal(dm_t.cpu().numpy(), want[i][0]), f"device single {i}"
            m, mdc = many.mask()
            assert parity.bits_equal(m, mask_want[0]) and parity.bits_equal(mdc, mask_want[1]), f"mask after step {k}"
            dm_b, score_b = many.diffmap(t)  # device, batched
            same_batch((dm_b.cpu().numpy(), score_b), k + 1)
            same_batch(many.diffmap(b), k + 1)
    finally:
        one.close()
        many.close()


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,n", [(40, 56, 5), (300, 411, 4)])
def test_cuda_device_path(cuda_lib, h, w, n):
    """Candidates in CUDA memory, written late on a non-default torch stream that the comparator must
    wait for."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    a, b = candidates(h, w, n)
    cmp = gb.Comparator(a, device=0, capacity=n, lib=cuda_lib)
    side = torch.cuda.Stream(device=dev)
    try:
        host_dm, host_score = cmp.diffmap(b)
        staged = torch.from_numpy(b).to(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            t = torch.full((n, 3, h, w), float("nan"), device=dev)
            torch.cuda._sleep(20_000_000)  # keeps the side stream busy: the copy below lands late
            t.copy_(staged)
            out = torch.full((n, h, w), float("nan"), device=dev)
            score = np.full(n, -1.0)
            assert cuda_lib.gb200_butteraugli_comparator_diffmap_batch_device(
                cmp._h, t.data_ptr(), n, out.data_ptr(), score.ctypes.data, side.cuda_stream), gb.last_error(lib=cuda_lib)
            dm_t, score_t = cmp.diffmap(t)  # the Python path: torch's current stream is `side`
        assert (score == host_score).all() and (score_t == host_score).all()
        assert parity.bits_equal(out.cpu().numpy(), host_dm), "device diffmaps differ from the host path"
        assert dm_t.device == dev and dm_t.dtype == torch.float32 and tuple(dm_t.shape) == (n, h, w)
        assert isinstance(score_t, np.ndarray) and score_t.dtype == np.float64
        assert parity.bits_equal(dm_t.cpu().numpy(), host_dm)
        # scores without diffmaps, candidates written late again
        with torch.cuda.stream(side):
            t.fill_(float("nan"))
            torch.cuda._sleep(20_000_000)
            t.copy_(staged)
            score = np.full(n, -1.0)
            assert cuda_lib.gb200_butteraugli_comparator_diffmap_batch_device(cmp._h, t.data_ptr(), n, None,
                                                                              score.ctypes.data, side.cuda_stream)
        assert (score == host_score).all()
    finally:
        torch.cuda.synchronize(dev)
        cmp.close()


def _profile(lib, f):
    """-> {kernel name: launches} of the work f() queues, timed per kernel."""
    lib.gb200_profile_reset()
    lib.gb200_profile_enable(1)
    try:
        f()
    finally:
        lib.gb200_profile_enable(0)
    cap = 64
    names = ((C.c_char * 48) * cap)()
    kl, kms, kel = (C.c_long * cap)(), (C.c_double * cap)(), (C.c_double * cap)()
    nk = lib.gb200_profile_get(names, kl, kms, kel, cap)
    out = {names[i].value.decode(): kl[i] for i in range(min(nk, cap))}
    lib.gb200_profile_reset()
    return out


@pytest.mark.gpu
def test_cuda_original_analysed_once(cuda_lib):
    """A batched call runs the Compare chain alone: no analysis launch (mask_sup0 is the analysis's
    own kernel; the chain's opsin and separation run once per call, for the candidates), the same
    launches for every n, and 5 fewer than a ButteraugliBatch call of the same n."""
    h, w, cap = 64, 96, 6
    a, b = candidates(h, w, cap)
    cmp = gb.Comparator(a, capacity=cap, lib=cuda_lib)
    batch = gb.ButteraugliBatch(h, w, cap, lib=cuda_lib)
    a_n = np.ascontiguousarray(np.broadcast_to(a, b.shape))
    try:
        cmp.diffmap(b)
        batch.diffmap(a_n, b)
        prof = _profile(cuda_lib, lambda: cmp.diffmap(b))
        assert "mask_sup0" not in prof, prof
        assert all(v == 1 for v in prof.values()) and len(prof) == 10, prof
        prof_pairs = _profile(cuda_lib, lambda: batch.diffmap(a_n, b))
        assert prof_pairs.get("mask_sup0") == 1 and sum(prof_pairs.values()) == sum(prof.values()) + 5, prof_pairs
        per_n = {}
        for n in (cap, 1, 2, cap - 1):
            before = gb.counters(lib=cuda_lib)[0]
            cmp.diffmap(b[:n])
            mid = gb.counters(lib=cuda_lib)[0]
            batch.diffmap(a_n[:n], b[:n])
            after = gb.counters(lib=cuda_lib)[0]
            per_n[n] = (mid - before, after - mid)
        assert len({v[0] for v in per_n.values()}) == 1, per_n
        assert all(v[1] - v[0] == 5 for v in per_n.values()), per_n
    finally:
        cmp.close()
        batch.close()


@pytest.mark.gpu
def test_cuda_refusals_launch_nothing(cuda_lib):
    torch = pytest.importorskip("torch")
    refusals(cuda_lib, "rgb1 is not device memory of device 0")
    a, b = candidates(40, 56, 2)
    cmp = gb.Comparator(a, device=0, capacity=2, lib=cuda_lib)
    try:
        t = torch.from_numpy(b).to("cuda:0")
        out = np.zeros((2, 40, 56), dtype=np.float32)
        torch.cuda.synchronize()
        launches = gb.counters(lib=cuda_lib)[0]
        score = np.full(3, -1.0)
        assert not cuda_lib.gb200_butteraugli_comparator_diffmap_batch_device(cmp._h, b.ctypes.data, 2, None,
                                                                              score.ctypes.data, None)
        assert "rgb1 is not device memory of device 0" in gb.last_error(lib=cuda_lib)
        assert not cuda_lib.gb200_butteraugli_comparator_diffmap_batch_device(cmp._h, t.data_ptr(), 2, out.ctypes.data,
                                                                              score.ctypes.data, None)
        assert "diffmap is not device memory of device 0" in gb.last_error(lib=cuda_lib)
        for n in (0, -1, 3):
            assert not cuda_lib.gb200_butteraugli_comparator_diffmap_batch_device(cmp._h, t.data_ptr(), n, None,
                                                                                  score.ctypes.data, None)
            assert not cuda_lib.gb200_butteraugli_comparator_diffmap_batch(cmp._h, b.ctypes.data, n, None,
                                                                           score.ctypes.data)
        assert gb.counters(lib=cuda_lib)[0] == launches
        assert (score == -1.0).all() and not out.any()
        if torch.cuda.device_count() < 2:
            pytest.skip("one GPU: memory of another device cannot be tried")
        with pytest.raises(RuntimeError, match=r"not device memory of device 0 \(device 1\)"):
            cmp.diffmap(t.to("cuda:1"))
        assert gb.counters(lib=cuda_lib)[0] == launches
    finally:
        cmp.close()


@pytest.mark.gpu
def test_cuda_comparators_concurrent(cuda_lib, ref):
    """Two batched comparators of different shapes, each on its own host thread and stream, at the same time."""
    want = {}
    for h, w, n in PAIR:
        a, b = candidates(h, w, n)
        want[(h, w, n)] = [ref.butteraugli_interface(a, b[i]) for i in range(n)]
    got, errors = {}, []

    def run(h, w, n):
        try:
            a, b = candidates(h, w, n)
            cmp = gb.Comparator(a, capacity=n, lib=cuda_lib)
            got[(h, w, n)] = [cmp.diffmap(b) for _ in range(3)]
            cmp.close()
        except Exception as e:  # noqa: BLE001 -- reported by the main thread
            errors.append(f"{h}x{w}: {e}")

    threads = [threading.Thread(target=run, args=s) for s in PAIR]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for s in PAIR:
        for k, (dm, score) in enumerate(got[s]):
            for i, (dm0, score0) in enumerate(want[s]):
                assert score[i] == score0 and parity.bits_equal(dm[i], dm0), f"{s} round {k} candidate {i}"
