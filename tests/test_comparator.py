"""butteraugli::ButteraugliComparator on the device (gb200_butteraugli_comparator_*, gb.Comparator)
and butteraugli::ButteraugliAdaptiveQuantization, bit for bit against the reference (oracle/_ref, or
its recorded answers).  Every reference call a GPU test makes is also made by a CPU test with the
same arguments, so that recording the CPU tests covers the GPU tests:

    GB200_REF_RECORD=$PWD/tests/golden/comparator_reference_answers.json \\
        python -m pytest tests/test_comparator.py -m "not gpu"

records them into golden/comparator_reference_answers.json, which replay mode reads beside
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

ANSWERS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "comparator_reference_answers.json")


@pytest.fixture(scope="module")
def ref(ref):
    """The session's reference, with the recorded answers of this module's calls added in replay mode."""
    if reflib._answers is not None:
        with open(ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


# The reference's two entry points, composed from its hooks for OpsinDynamicsImage, SeparateFrequencies and
# Mask (oracle/ref_hooks.cc).  Only the live reference computes them; replay mode answers from the record.
@reflib._answered
def reference_comparator_mask(rgb0):
    """ButteraugliComparator(rgb0).Mask (b/butteraugli.cc:784-795): Mask of MaskPsychoImage(pi0, pi0)
    -> (mask, mask_dc), float32 [3][h][w] each."""
    ps = reflib.separate.__wrapped__(reflib.opsin.__wrapped__(rgb0))  # uhf0 uhf1 hf0 hf1 mf0..2 lf0..2
    # MaskPsychoImage (:753-781): row = a * uhf + b * hf in double, stored as float; the B plane is not read
    muls = (0.0, 1.64178305129, 0.831081703362, 3.23680933546)
    mixed = np.zeros_like(ps[:3])
    for i in range(2):
        a, b = muls[2 * i], muls[2 * i + 1]
        mixed[i] = (a * ps[i].astype(np.float64) + b * ps[2 + i].astype(np.float64)).astype(np.float32)
    return reflib.mask.__wrapped__(mixed, mixed)


@reflib._answered
def reference_adaptive_quantization(rgb):
    """ButteraugliAdaptiveQuantization (b/butteraugli.cc:1880-1902) for images of at least 16x16:
    the Y plane of Mask(rgb, rgb) -> float32 [h][w]."""
    return reflib.mask.__wrapped__(rgb, rgb)[0][1].copy()


# (h, w): one comparator per shape, each scoring NCAND candidates in a row (plain launches, graph
# capture, graph replay)
DIFF_SHAPES = [(8, 8), (40, 56), (17, 130), (64, 64), (300, 411), (577, 70), (1080, 100), (1080, 1920)]
NCAND = 3
MASK_SHAPES = [(8, 8), (40, 56), (17, 130), (300, 411)]
AQ_SHAPES = [(16, 16), (17, 130), (40, 56), (300, 411)]
AQ_REFUSED = [(15, 40), (40, 15)]
# comparators of two sizes used in turn by one thread, and from two threads at once
PAIR = [(40, 56), (300, 411)]


def original(h, w):
    return linear(synth.gradnoise(h, w, 7 * h + w))


def candidates(h, w):
    a = synth.gradnoise(h, w, 7 * h + w).astype(int)
    return [linear(np.clip(a + synth.noise(h, w, 100 + k) % (2 * k + 5) - (k + 2), 0, 255).astype(np.uint8))
            for k in range(NCAND)]


def check_diffmaps(lib, ref, h, w):
    a = original(h, w)
    cmp = gb.Comparator(a, lib=lib)
    try:
        for k, b in enumerate(candidates(h, w)):
            dm, score = cmp.diffmap(b)
            dm0, score0 = ref.butteraugli_interface(a, b)
            assert score == score0 and parity.bits_equal(dm, dm0), f"{h}x{w} candidate {k}: differs from the reference"
        dm, score = cmp.diffmap(a)
        assert score == 0.0 and not dm.any(), "the original against itself is not all zeros"
    finally:
        cmp.close()


def check_interleaved(lib, ref):
    cmps = [gb.Comparator(original(h, w), lib=lib) for h, w in PAIR]
    try:
        cands = [candidates(h, w) for h, w in PAIR]
        for k in range(NCAND):
            for i, (h, w) in enumerate(PAIR):
                dm, score = cmps[i].diffmap(cands[i][k])
                dm0, score0 = ref.butteraugli_interface(original(h, w), cands[i][k])
                assert score == score0 and parity.bits_equal(dm, dm0), f"{h}x{w} candidate {k}"
    finally:
        for c in cmps:
            c.close()


def check_mask(lib, ref, h, w):
    a = original(h, w)
    cands = candidates(h, w)
    cmp = gb.Comparator(a, lib=lib)
    try:
        before = [cmp.diffmap(b) for b in cands[:2]]
        m, mdc = cmp.mask()
        rm, rmdc = reference_comparator_mask(a)
        assert parity.bits_equal(m, rm), f"{h}x{w}: mask differs from the reference"
        assert parity.bits_equal(mdc, rmdc), f"{h}x{w}: mask_dc differs from the reference"
        # Mask leaves the resident original alone: the same candidates score the same afterwards
        for b, (dm0, s0) in zip(cands[:2], before):
            dm, s = cmp.diffmap(b)
            assert s == s0 and parity.bits_equal(dm, dm0), f"{h}x{w}: diffmap changed after mask()"
        m2, mdc2 = cmp.mask()
        assert parity.bits_equal(m2, m) and parity.bits_equal(mdc2, mdc)
    finally:
        cmp.close()


def check_aq(lib, ref, h, w):
    a = original(h, w)
    q = gb.adaptive_quantization(a, lib=lib)
    assert parity.bits_equal(q, reference_adaptive_quantization(a)), f"{h}x{w}: differs from the reference"


def check_aq_refused(lib, h, w):
    # the reference returns false when either side is below 16 (b/butteraugli.cc:1882-1884)
    a = original(h, w)
    with pytest.raises(ValueError, match="16x16"):
        gb.adaptive_quantization(a, lib=lib)
    q = np.zeros((h, w), dtype=np.float32)
    assert not lib.gb200_butteraugli_adaptive_quantization(a.ctypes.data, w, h, 0, q.ctypes.data)
    assert "16x16" in gb.last_error(lib=lib)


def check_small_refused(lib):
    for h, w in [(7, 20), (20, 7)]:
        with pytest.raises(RuntimeError, match="at least 8x8"):
            gb.Comparator(np.zeros((3, h, w), dtype=np.float32), lib=lib)


# ---- CPU: the port, and every reference call of the GPU tests -------------------------------

@pytest.mark.parametrize("h,w", DIFF_SHAPES)
def test_port_comparator_diffmaps(port_lib, ref, h, w):
    check_diffmaps(port_lib, ref, h, w)


def test_port_comparators_interleaved(port_lib, ref):
    check_interleaved(port_lib, ref)


@pytest.mark.parametrize("h,w", MASK_SHAPES)
def test_port_comparator_mask(port_lib, ref, h, w):
    check_mask(port_lib, ref, h, w)


@pytest.mark.parametrize("h,w", AQ_SHAPES)
def test_port_adaptive_quantization(port_lib, ref, h, w):
    check_aq(port_lib, ref, h, w)


@pytest.mark.parametrize("h,w", AQ_REFUSED)
def test_port_adaptive_quantization_refuses_small(port_lib, h, w):
    check_aq_refused(port_lib, h, w)


def test_port_refusals(port_lib):
    check_small_refused(port_lib)
    a = original(40, 56)
    cmp = gb.Comparator(a, lib=port_lib)
    try:
        score = C.c_double(-1.0)
        assert not port_lib.gb200_butteraugli_comparator_diffmap_device(cmp._h, a.ctypes.data, None, C.byref(score), None)
        assert "no device memory" in gb.last_error(lib=port_lib) and score.value == -1.0
        assert not port_lib.gb200_butteraugli_comparator_mask(cmp._h, None, None)
    finally:
        cmp.close()


# ---- GPU ------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("h,w", DIFF_SHAPES)
def test_cuda_comparator_diffmaps(cuda_lib, ref, h, w):
    check_diffmaps(cuda_lib, ref, h, w)


@pytest.mark.gpu
def test_cuda_comparators_interleaved(cuda_lib, ref):
    check_interleaved(cuda_lib, ref)


@pytest.mark.gpu
def test_cuda_comparators_concurrent(cuda_lib, ref):
    """Two comparators, each on its own host thread and stream, at the same time."""
    want = {(h, w): [ref.butteraugli_interface(original(h, w), b) for b in candidates(h, w)] for h, w in PAIR}
    got, errors = {}, []

    def run(h, w):
        try:
            cmp = gb.Comparator(original(h, w), lib=cuda_lib)
            got[(h, w)] = [cmp.diffmap(b) for b in candidates(h, w)]
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
        for k, ((dm, score), (dm0, score0)) in enumerate(zip(got[s], want[s])):
            assert score == score0 and parity.bits_equal(dm, dm0), f"{s} candidate {k}"


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(40, 56), (300, 411)])
def test_cuda_device_path(cuda_lib, ref, h, w):
    """Candidates in CUDA memory, written on a non-default torch stream that the comparator must wait for."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    a = original(h, w)
    cmp = gb.Comparator(a, device=0, lib=cuda_lib)
    side = torch.cuda.Stream(device=dev)
    try:
        for k, b in enumerate(candidates(h, w)):
            host_dm, host_score = cmp.diffmap(b)
            dm0, score0 = ref.butteraugli_interface(a, b)
            assert host_score == score0 and parity.bits_equal(host_dm, dm0)
            staged = torch.from_numpy(b).to(dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                cand = torch.full((3, h, w), float("nan"), device=dev)
                torch.cuda._sleep(20_000_000)  # keeps the side stream busy: the copy below lands late
                cand.copy_(staged)
                out = torch.full((h, w), float("nan"), device=dev)
                score = C.c_double(-1.0)
                assert cuda_lib.gb200_butteraugli_comparator_diffmap_device(
                    cmp._h, cand.data_ptr(), out.data_ptr(), C.byref(score), side.cuda_stream), gb.last_error(lib=cuda_lib)
                dm_t, score_t = cmp.diffmap(cand)  # the Python path: torch's current stream is `side`
            assert score.value == host_score and score_t == host_score, k
            assert parity.bits_equal(out.cpu().numpy(), host_dm), f"candidate {k}: device diffmap differs"
            assert dm_t.device == dev and dm_t.dtype == torch.float32
            assert parity.bits_equal(dm_t.cpu().numpy(), host_dm)
        # a score without a diffmap
        score = C.c_double(-1.0)
        cand = torch.from_numpy(a).to(dev)
        torch.cuda.synchronize(dev)
        assert cuda_lib.gb200_butteraugli_comparator_diffmap_device(cmp._h, cand.data_ptr(), None, C.byref(score), None)
        assert score.value == 0.0
    finally:
        cmp.close()


@pytest.mark.gpu
def test_cuda_device_path_refuses_other_memory(cuda_lib):
    a = original(40, 56)
    cmp = gb.Comparator(a, device=0, lib=cuda_lib)
    try:
        out = np.zeros((40, 56), dtype=np.float32)
        score = C.c_double(-1.0)
        launches = gb.counters(lib=cuda_lib)[0]
        assert not cuda_lib.gb200_butteraugli_comparator_diffmap_device(cmp._h, a.ctypes.data, None, C.byref(score), None)
        assert "rgb1 is not device memory of device 0" in gb.last_error(lib=cuda_lib)
        torch = pytest.importorskip("torch")
        cand = torch.from_numpy(a).to("cuda:0")
        assert not cuda_lib.gb200_butteraugli_comparator_diffmap_device(cmp._h, cand.data_ptr(), out.ctypes.data,
                                                                        C.byref(score), None)
        assert "diffmap is not device memory of device 0" in gb.last_error(lib=cuda_lib)
        assert gb.counters(lib=cuda_lib)[0] == launches and score.value == -1.0
        if torch.cuda.device_count() < 2:
            pytest.skip("one GPU: memory of another device cannot be tried")
        with pytest.raises(RuntimeError, match=r"not device memory of device 0 \(device 1\)"):
            cmp.diffmap(torch.from_numpy(a).to("cuda:1"))
        assert gb.counters(lib=cuda_lib)[0] == launches
    finally:
        cmp.close()


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", MASK_SHAPES)
def test_cuda_comparator_mask(cuda_lib, ref, h, w):
    check_mask(cuda_lib, ref, h, w)


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", AQ_SHAPES)
def test_cuda_adaptive_quantization(cuda_lib, ref, h, w):
    check_aq(cuda_lib, ref, h, w)


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", AQ_REFUSED)
def test_cuda_adaptive_quantization_refuses_small(cuda_lib, h, w):
    check_aq_refused(cuda_lib, h, w)


@pytest.mark.gpu
def test_cuda_comparator_refuses_small(cuda_lib):
    check_small_refused(cuda_lib)
