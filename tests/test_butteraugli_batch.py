"""Batched butteraugli (gb200_butteraugli_batch_*, gb.ButteraugliBatch): N same-size pairs per call, each
bit for bit butteraugli::ButteraugliInterface of the reference (oracle/_ref, or its recorded answers).
Every reference call a GPU test makes is also made by a CPU test with the same arguments, so that
recording the CPU tests covers the GPU tests:

    GB200_REF_RECORD=$PWD/tests/golden/batch_reference_answers.json \\
        python -m pytest tests/test_butteraugli_batch.py -m "not gpu"

records them into golden/batch_reference_answers.json, which replay mode reads beside
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

ANSWERS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "batch_reference_answers.json")


@pytest.fixture(scope="module")
def ref(ref):
    """The session's reference, with the recorded answers of this module's calls added in replay mode."""
    if reflib._answers is not None:
        with open(ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


# (h, w, n): one batch of capacity n per shape, scoring n distinct pairs.  Pitch padding, one and
# several strips and segments; 12x20 x 260 makes the widest launch (4 z per image) 1040 deep.
CASES = [(8, 8, 33), (9, 17, 7), (40, 56, 5), (17, 130, 3), (64, 64, 64), (12, 20, 260), (300, 411, 4),
         (577, 70, 3), (1080, 100, 2), (1080, 1920, 2)]
# two batch objects of different shapes on two threads at once (shapes of CASES)
PAIR = [(40, 56, 5), (300, 411, 4)]


def pair(h, w, i):
    """Pair i of a shape: a gradient-and-noise original and a candidate perturbed by up to +-(2 + i % 4)."""
    a = synth.gradnoise(h, w, 1000 + 7 * h + w + 31 * i).astype(int)
    k = i % 4
    b = np.clip(a + synth.noise(h, w, 500 + 3 * i + h) % (2 * k + 5) - (k + 2), 0, 255).astype(np.uint8)
    return linear(a.astype(np.uint8)), linear(b)


def pairs(h, w, n, first=0):
    ps = [pair(h, w, first + i) for i in range(n)]
    return np.stack([p[0] for p in ps]), np.stack([p[1] for p in ps])


def check_against_reference(lib, ref, h, w, n, comparator=False):
    a, b = pairs(h, w, n)
    batch = gb.ButteraugliBatch(h, w, n, lib=lib)
    try:
        dm, score = batch.diffmap(a, b)
    finally:
        batch.close()
    assert dm.shape == (n, h, w) and dm.dtype == np.float32 and score.shape == (n,) and score.dtype == np.float64
    for i in range(n):
        dm0, score0 = ref.butteraugli_interface(a[i], b[i])
        assert score[i] == score0 and parity.bits_equal(dm[i], dm0), f"{h}x{w} pair {i} of {n}: differs from the reference"
        if comparator:  # the single-image device path gives the same bits
            cmp = gb.Comparator(a[i], lib=lib)
            try:
                dmc, scorec = cmp.diffmap(b[i])
            finally:
                cmp.close()
            assert scorec == score[i] and parity.bits_equal(dmc, dm[i]), f"{h}x{w} pair {i}: differs from Comparator"
    return dm, score


def refusals(lib, device_entry_message):
    """Every refusal of the C ABI and its message; -> None.  The batch is 40x56 with capacity 3."""
    for w, h, cap, msg in [(7, 20, 1, "at least 8x8"), (20, 7, 1, "at least 8x8"), (65536, 8, 1, "below 65536"),
                           (20, 20, 0, "capacity must be in 1..16383"), (20, 20, 16384, "capacity must be in 1..16383")]:
        assert not lib.gb200_butteraugli_batch_create(w, h, cap, 0), (w, h, cap)
        assert msg in gb.last_error(lib=lib), (w, h, cap, gb.last_error(lib=lib))
    a, b = pairs(40, 56, 3)
    batch = gb.ButteraugliBatch(40, 56, 3, lib=lib)
    try:
        score = np.full(4, -1.0)
        for n in (0, -1, 4):
            assert not lib.gb200_butteraugli_batch_diffmap(batch._h, a.ctypes.data, b.ctypes.data, n, None,
                                                           score.ctypes.data)
            assert f"n = {n} pairs, the batch takes 1..3" in gb.last_error(lib=lib)
        assert not lib.gb200_butteraugli_batch_diffmap(batch._h, None, b.ctypes.data, 1, None, None)
        assert "no batch or no images" in gb.last_error(lib=lib)
        assert not lib.gb200_butteraugli_batch_diffmap_device(batch._h, a.ctypes.data, b.ctypes.data, 2, None,
                                                              score.ctypes.data, None)
        assert device_entry_message in gb.last_error(lib=lib), gb.last_error(lib=lib)
        assert (score == -1.0).all(), "a refused call wrote scores"
    finally:
        batch.close()


def python_checks(lib):
    batch = gb.ButteraugliBatch(40, 56, 3, lib=lib)
    try:
        a, b = pairs(40, 56, 3)
        bad = [(a[:0], b[:0]), (a[None], b[None]), (a[0], b[0]), (a[:, :, :39], b[:, :, :39]),
               (a[:, :2], b[:, :2]), (a[:2], b), (a.astype(np.float64), b.astype(np.float64)),
               (a, b.astype(np.float16)), (np.concatenate([a, a[:1]]), np.concatenate([b, b[:1]]))]
        for x, y in bad:
            with pytest.raises(ValueError):
                batch.diffmap(x, y)
        dm, score = batch.diffmap(a[:1], b[:1])  # n < capacity is fine
        assert dm.shape == (1, 40, 56) and score.shape == (1,)
    finally:
        batch.close()


# ---- CPU: the port (pair by pair through the metric-only context), and every reference call of the
# GPU tests ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("h,w,n", CASES)
def test_port_batch_matches_reference(port_lib, ref, h, w, n):
    check_against_reference(port_lib, ref, h, w, n)


def test_port_refusals(port_lib):
    refusals(port_lib, "no device memory")


def test_port_python_checks(port_lib):
    python_checks(port_lib)


# ---- GPU ------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("h,w,n", CASES)
def test_cuda_batch_matches_reference(cuda_lib, ref, h, w, n):
    check_against_reference(cuda_lib, ref, h, w, n, comparator=True)


@pytest.mark.gpu
def test_cuda_batch_matches_reference_staged(cuda_lib, ref, monkeypatch):
    """GB200_COMPARE=staged: the batch scores pair by pair through the staged chain, host and device entry."""
    torch = pytest.importorskip("torch")
    monkeypatch.setenv("GB200_COMPARE", "staged")
    h, w, n = PAIR[0]
    a, b = pairs(h, w, n)
    batch = gb.ButteraugliBatch(h, w, n, lib=cuda_lib)
    try:
        dm, score = batch.diffmap(a, b)
        dm_t, score_t = batch.diffmap(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda())
    finally:
        batch.close()
    for i in range(n):
        dm0, score0 = ref.butteraugli_interface(a[i], b[i])
        assert score[i] == score0 and parity.bits_equal(dm[i], dm0), f"pair {i}"
    assert (score_t == score).all() and parity.bits_equal(dm_t.cpu().numpy(), dm)


def isolation_pairs(h, w, n):
    """Slots alternate a high-contrast noise pair with an identical flat-gray pair."""
    a, b = [], []
    for i in range(n):
        if i % 2 == 0:
            a.append(linear(synth.noise(h, w, 70 + i)))
            b.append(linear(synth.noise(h, w, 90 + i)))
        else:
            g = linear(np.full((h, w, 3), 60 + 30 * (i % 6), dtype=np.uint8))
            a.append(g)
            b.append(g.copy())
    return np.stack(a), np.stack(b)


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,n", [(40, 56, 6), (300, 411, 5)])
def test_cuda_slots_are_isolated(cuda_lib, h, w, n):
    a, b = isolation_pairs(h, w, n)
    batch = gb.ButteraugliBatch(h, w, n, lib=cuda_lib)
    one = gb.ButteraugliBatch(h, w, 1, lib=cuda_lib)
    try:
        dm, score = batch.diffmap(a, b)
        for i in range(n):
            if i % 2 == 1:
                assert score[i] == 0.0 and not dm[i].any(), f"identical pair {i}: not all zeros"
            else:
                assert score[i] > 1.0, f"noise pair {i}: score {score[i]}"
            dm1, score1 = one.diffmap(a[i:i + 1], b[i:i + 1])
            assert score1[0] == score[i] and parity.bits_equal(dm1[0], dm[i]), f"pair {i}: differs from a batch of 1"
        dmr, scorer = batch.diffmap(a[::-1].copy(), b[::-1].copy())
        assert (scorer == score[::-1]).all() and parity.bits_equal(dmr, dm[::-1]), "the reversed batch"
    finally:
        batch.close()
        one.close()


@pytest.mark.gpu
def test_cuda_partial_batches(cuda_lib):
    """n = capacity, 1, capacity - 1, capacity on one object, different pairs each time, a unique pair in
    the last used slot: every result equals a fresh object's."""
    h, w, cap = 64, 96, 5
    batch = gb.ButteraugliBatch(h, w, cap, lib=cuda_lib)
    try:
        first = 0
        for k, n in enumerate([cap, 1, cap - 1, cap]):
            a, b = pairs(h, w, n, first)
            first += n
            a[n - 1] = linear(synth.noise(h, w, 300 + k))  # unique: noise against a gradient
            dm, score = batch.diffmap(a, b)
            fresh = gb.ButteraugliBatch(h, w, cap, lib=cuda_lib)
            try:
                dmf, scoref = fresh.diffmap(a, b)
            finally:
                fresh.close()
            assert (score == scoref).all() and parity.bits_equal(dm, dmf), f"call {k} (n = {n})"
    finally:
        batch.close()


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,n", [(40, 56, 5), (300, 411, 4)])
def test_cuda_device_path(cuda_lib, h, w, n):
    """Pairs in CUDA memory, written late on a non-default torch stream that the batch must wait for."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    a, b = pairs(h, w, n)
    batch = gb.ButteraugliBatch(h, w, n, device=0, lib=cuda_lib)
    side = torch.cuda.Stream(device=dev)
    try:
        host_dm, host_score = batch.diffmap(a, b)
        staged0, staged1 = torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            t0 = torch.full((n, 3, h, w), float("nan"), device=dev)
            t1 = torch.full((n, 3, h, w), float("nan"), device=dev)
            torch.cuda._sleep(20_000_000)  # keeps the side stream busy: the copies below land late
            t0.copy_(staged0)
            t1.copy_(staged1)
            out = torch.full((n, h, w), float("nan"), device=dev)
            score = np.full(n, -1.0)
            assert cuda_lib.gb200_butteraugli_batch_diffmap_device(batch._h, t0.data_ptr(), t1.data_ptr(), n,
                                                                   out.data_ptr(), score.ctypes.data,
                                                                   side.cuda_stream), gb.last_error(lib=cuda_lib)
            dm_t, score_t = batch.diffmap(t0, t1)  # the Python path: torch's current stream is `side`
        assert (score == host_score).all() and (score_t == host_score).all()
        assert parity.bits_equal(out.cpu().numpy(), host_dm), "device diffmaps differ from the host path"
        assert dm_t.device == dev and dm_t.dtype == torch.float32 and tuple(dm_t.shape) == (n, h, w)
        assert isinstance(score_t, np.ndarray) and score_t.dtype == np.float64
        assert parity.bits_equal(dm_t.cpu().numpy(), host_dm)
        # scores without diffmaps
        score = np.full(n, -1.0)
        torch.cuda.synchronize(dev)
        assert cuda_lib.gb200_butteraugli_batch_diffmap_device(batch._h, staged0.data_ptr(), staged1.data_ptr(), n,
                                                               None, score.ctypes.data, None)
        assert (score == host_score).all()
    finally:
        batch.close()


@pytest.mark.gpu
def test_cuda_refusals_launch_nothing(cuda_lib):
    torch = pytest.importorskip("torch")
    launches = gb.counters(lib=cuda_lib)[0]
    refusals(cuda_lib, "rgb0 is not device memory of device 0")
    assert gb.counters(lib=cuda_lib)[0] == launches
    a, b = pairs(40, 56, 2)
    batch = gb.ButteraugliBatch(40, 56, 2, device=0, lib=cuda_lib)
    try:
        t0, t1 = torch.from_numpy(a).to("cuda:0"), torch.from_numpy(b).to("cuda:0")
        out = np.zeros((2, 40, 56), dtype=np.float32)
        torch.cuda.synchronize()
        launches = gb.counters(lib=cuda_lib)[0]
        assert not cuda_lib.gb200_butteraugli_batch_diffmap_device(batch._h, t0.data_ptr(), b.ctypes.data, 2, None,
                                                                   None, None)
        assert "rgb1 is not device memory of device 0" in gb.last_error(lib=cuda_lib)
        assert not cuda_lib.gb200_butteraugli_batch_diffmap_device(batch._h, t0.data_ptr(), t1.data_ptr(), 2,
                                                                   out.ctypes.data, None, None)
        assert "diffmap is not device memory of device 0" in gb.last_error(lib=cuda_lib)
        assert not cuda_lib.gb200_butteraugli_batch_diffmap_device(batch._h, t0.data_ptr(), t1.data_ptr(), 3, None,
                                                                   None, None)
        assert gb.counters(lib=cuda_lib)[0] == launches
        if torch.cuda.device_count() < 2:
            pytest.skip("one GPU: memory of another device cannot be tried")
        with pytest.raises(RuntimeError, match=r"not device memory of device 0 \(device 1\)"):
            batch.diffmap(t0.to("cuda:1"), t1.to("cuda:1"))
        assert gb.counters(lib=cuda_lib)[0] == launches
    finally:
        batch.close()


@pytest.mark.gpu
def test_cuda_batches_concurrent(cuda_lib, ref):
    """Two batch objects of different shapes, each on its own host thread and stream, at the same time."""
    want = {}
    for h, w, n in PAIR:
        a, b = pairs(h, w, n)
        want[(h, w, n)] = [ref.butteraugli_interface(a[i], b[i]) for i in range(n)]
    got, errors = {}, []

    def run(h, w, n):
        try:
            batch = gb.ButteraugliBatch(h, w, n, lib=cuda_lib)
            got[(h, w, n)] = [batch.diffmap(*pairs(h, w, n)) for _ in range(3)]
            batch.close()
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
                assert score[i] == score0 and parity.bits_equal(dm[i], dm0), f"{s} round {k} pair {i}"
