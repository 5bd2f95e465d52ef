"""Butteraugli comparator sets (gb200_butteraugli_comparator_set_*, gb.ComparatorSet): originals of sizes of
their own, analysed once and kept on the device, and candidates that name their original by index.  Each
candidate is bit for bit what ButteraugliBatch.diffmap_sizes (diffmap_sizes_srgb for 8-bit sets) gives for the
pair (original, candidate), and so butteraugli::ButteraugliInterface of the reference on that pair (oracle/_ref,
or its recorded answers).  Every reference call a GPU test makes is also made by a CPU test with the same
arguments, so that recording the CPU tests covers the GPU tests:

    GB200_REF_RECORD=$PWD/tests/golden/comparator_set_reference_answers.json \\
        python -m pytest tests/test_comparator_set.py -m "not gpu"

records them into golden/comparator_set_reference_answers.json, which replay mode reads beside
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
from test_butteraugli_sizes import SETS
from test_srgb_inputs import alpha_cases, perturbed, planes, reference, with_alpha

ANSWERS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "comparator_set_reference_answers.json")


@pytest.fixture(scope="module")
def ref(ref):
    """The session's reference, with the recorded answers of this module's calls added in replay mode."""
    if reflib._answers is not None:
        with open(ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


def original(h, w, k):
    """Original k of a set: a gradient with noise, uint8 [h][w][3]."""
    return synth.gradnoise(h, w, 9000 + 7 * h + w + 31 * k).astype(np.uint8)


def candidate(a, v):
    """Candidate v of an 8-bit RGB original: every channel moved by up to +-(2 + v % 4)."""
    h, w, _ = a.shape
    k = v % 4
    return np.clip(a.astype(int) + synth.noise(h, w, 9500 + 3 * v + h) % (2 * k + 5) - (k + 2), 0, 255).astype(np.uint8)


def float_set(shapes, index):
    """Float originals of `shapes` and candidate i of original index[i] (linear RGB planes)."""
    u8 = [original(h, w, k) for k, (h, w) in enumerate(shapes)]
    return [linear(a) for a in u8], [linear(candidate(u8[o], v)) for v, o in enumerate(index)]


def srgb_set(shapes, channels, index):
    """8-bit originals of `shapes` with channels[k] channels, and candidate i of original index[i]."""
    imgs = [with_alpha(original(h, w, k), c, 9700 + k) for k, ((h, w), c) in enumerate(zip(shapes, channels))]
    return imgs, [perturbed(imgs[o], 9800 + 5 * v, 2 + v % 3) for v, o in enumerate(index)]


def make_set(lib, originals, capacity, srgb=False, device=0):
    if srgb:
        return gb.ComparatorSet.from_srgb(originals, capacity=capacity, device=device, lib=lib)
    return gb.ComparatorSet(originals, capacity=capacity, device=device, lib=lib)


def scored(lib, originals, index, cands, capacity=None, srgb=False):
    s = make_set(lib, originals, capacity or len(index), srgb)
    try:
        return s.diffmap(index, cands)
    finally:
        s.close()


def pairs_scored(lib, originals, index, cands, srgb=False):
    """The same pairs through ButteraugliBatch.diffmap_sizes*, in a batch of the largest width x height."""
    shapes = [x.shape[:2] if srgb else x.shape[1:] for x in originals]
    bh, bw = max(s[0] for s in shapes), max(s[1] for s in shapes)
    batch = gb.ButteraugliBatch(bh, bw, len(index), lib=lib)
    try:
        a = [originals[o] for o in index]
        return (batch.diffmap_sizes_srgb if srgb else batch.diffmap_sizes)(a, cands)
    finally:
        batch.close()


def assert_same(got, want, what):
    dm, score = got
    dm0, score0 = want
    assert len(dm) == len(dm0)
    for i in range(len(dm0)):
        assert score[i] == score0[i], f"{what}: candidate {i}: {score[i]} != {score0[i]}"
        assert parity.bits_equal(np.asarray(dm[i]), np.asarray(dm0[i])), f"{what}: candidate {i}: diffmap differs"


# A small float set: out of order, originals 1 and 4 twice, original 3 not at all.
SMALL = [(8, 8), (17, 9), (40, 48), (24, 16), (9, 33), (33, 40)]
SMALL_INDEX = [4, 0, 2, 4, 1, 5, 1]

# An 8-bit set mixing RGB and RGBA; original 3 is alpha_cases' "dark" (white wins), and candidate 5 is its
# original unchanged (both backgrounds score 0: black keeps it on the tie).
SRGB_SHAPES = [(8, 8), (20, 13), (32, 24)]
SRGB_CHANNELS = [4, 3, 4]
SRGB_INDEX = [2, 1, 0, 3, 2, 0, 3]


def srgb_small():
    imgs, cands = srgb_set(SRGB_SHAPES, SRGB_CHANNELS, [i for i in SRGB_INDEX if i < 3])
    _, dark, dark_b, winner = alpha_cases()[0]
    assert winner == 255
    imgs = imgs + [dark]
    cands = cands[:3] + [dark_b] + cands[3:] + [dark_b]
    cands[5] = imgs[0].copy()
    return imgs, cands


def mixed_case():
    """The shapes of SETS["mixed"] plus 20 small sizes (32 in all, more than one pass's 16), each original
    scored once and four of them twice, in a shuffled order."""
    shapes = SETS["mixed"][2] + [(8 + i, 10 + 2 * i) for i in range(20)]
    index = list(range(len(shapes))) + [0, 13, 31, 5]
    index = [index[i] for i in np.random.default_rng(21).permutation(len(index))]
    return shapes, index


def mixed_reference_subset(shapes, index):
    """The candidates of mixed_case checked against the reference as well: those of at most 64x64."""
    return [i for i, o in enumerate(index) if shapes[o][0] * shapes[o][1] <= 64 * 64]


def mixed_reference_pairs():
    shapes, index = mixed_case()
    subset = mixed_reference_subset(shapes, index)
    used = sorted({index[i] for i in subset})
    u8 = {o: original(*shapes[o], o) for o in used}
    return [(linear(u8[index[i]]), linear(candidate(u8[index[i]], i))) for i in subset]


def check_reference(ref, originals, index, got, srgb=False, cands=None):
    dm, score = got
    for i, o in enumerate(index):
        if srgb:
            dm0, score0 = reference(ref, originals[o], cands[i])
        else:
            dm0, score0 = ref.butteraugli_interface(originals[o], cands[i])
        assert score[i] == score0 and parity.bits_equal(np.asarray(dm[i]), dm0), f"candidate {i} (original {o})"


def refusals(lib, device_message, launches=lambda: 0):
    """Every refusal of the C ABI and its message; nothing written and nothing launched (launches() counts
    the launches so far) by a refused call."""
    before = launches()
    err = lambda: gb.last_error(lib=lib)
    origs, cands = float_set(SMALL[:3], [0, 1, 2])
    P3 = C.c_void_p * 3
    po = P3(*[x.ctypes.data for x in origs])
    W = np.array([s[1] for s in SMALL[:3]], dtype=np.int32)
    H = np.array([s[0] for s in SMALL[:3]], dtype=np.int32)

    def create(w=W, h=H, imgs=po, count=3, capacity=3):
        return lib.gb200_butteraugli_comparator_set_create(None if w is None else w.ctypes.data,
                                                           None if h is None else h.ctypes.data, imgs, count,
                                                           capacity, 0)

    for kw, msg in [(dict(w=np.array([8, 7, 48], np.int32)), "original 1 is 7x17, the originals must be at least 8x8"),
                    (dict(h=np.array([8, 17, 65536], np.int32)), "original 2 is 48x65536, the originals must be at least"),
                    (dict(capacity=0), "butteraugli comparator set: the capacity must be in 1..16383"),
                    (dict(capacity=16384), "butteraugli comparator set: the capacity must be in 1..16383"),
                    (dict(count=0), "count = 0, a set holds at least 1 original"),
                    (dict(w=None), "butteraugli comparator set: no sizes or no images"),
                    (dict(h=None), "butteraugli comparator set: no sizes or no images"),
                    (dict(imgs=None), "butteraugli comparator set: no sizes or no images"),
                    (dict(imgs=P3(po[0], None, po[2])), "original 1 has a null image pointer")]:
        assert not create(**kw), kw
        assert msg in err(), (kw, err())
    u8, _ = srgb_set(SMALL[:3], [3, 4, 3], [])
    pu = P3(*[x.ctypes.data for x in u8])
    for chs, msg in [(None, "no sizes, no channels or no images"),
                     (np.array([3, 5, 4], np.int32), "original 1: channels = 5, 8-bit images must have 3 (RGB) or 4")]:
        assert not lib.gb200_butteraugli_comparator_set_create_srgb(W.ctypes.data, H.ctypes.data,
                                                                    None if chs is None else chs.ctypes.data, pu, 3, 3, 0)
        assert msg in err(), err()

    assert launches() == before
    fset = make_set(lib, origs, 3)
    sset = gb.ComparatorSet.from_srgb(u8, capacity=3, lib=lib)
    before = launches()
    try:
        pc = P3(*[x.ctypes.data for x in cands])
        dms = [np.zeros(x.shape[1:], dtype=np.float32) for x in cands]
        pd = P3(*[x.ctypes.data for x in dms])
        score = np.full(4, -1.0)
        index = np.array([0, 1, 2, 0], dtype=np.int32)

        def call(s=fset._h, idx=index, imgs=pc, n=3, entry="", device=False):
            name = "gb200_butteraugli_comparator_set_diffmap" + entry + ("_device" if device else "")
            args = (s, None if idx is None else idx.ctypes.data, imgs, n, pd, score.ctypes.data)
            return getattr(lib, name)(*(args + ((None,) if device else ())))

        for n in (0, -1, 4):
            assert not call(n=n)
            assert f"butteraugli comparator set: n = {n} images, the comparator set takes 1..3" in err(), err()
        for idx, msg in [([0, 3, 1], "original[1] = 3, the set holds originals 0..2"),
                         ([0, 1, -1], "original[2] = -1, the set holds originals 0..2")]:
            assert not call(idx=np.array(idx, dtype=np.int32))
            assert msg in err(), err()
        for kw in [dict(s=None), dict(idx=None), dict(imgs=None)]:
            assert not call(**kw), kw
            assert "butteraugli comparator set: no set, no indices or no images" in err(), err()
        assert not call(imgs=P3(pc[0], None, pc[2]))
        assert "butteraugli comparator set: image 1 has a null pointer" in err(), err()
        for device in (False, True):
            assert not call(entry="_srgb", device=device)
            assert "made from float planes, it takes float images, not 8-bit ones" in err(), err()
            assert not call(s=sset._h, device=device)
            assert "made from 8-bit images, it takes 8-bit images, not float planes" in err(), err()
        assert not call(device=True)
        assert device_message in err(), err()
        assert (score == -1.0).all(), "a refused call wrote scores"
        assert not any(d.any() for d in dms), "a refused call wrote diffmaps"
        assert launches() == before
    finally:
        fset.close()
        sset.close()


def python_checks(lib):
    origs, cands = float_set(SMALL[:3], [0, 1, 2])
    for bad in ([], [origs[0][0]], [origs[0].astype(np.float64)], [origs[0][:, :, ::2]], [origs[0][:, :7]],
                [origs[0].tolist()]):
        with pytest.raises(ValueError):
            gb.ComparatorSet(bad, capacity=2, lib=lib)
    s = gb.ComparatorSet(origs, capacity=3, lib=lib)
    try:
        for index, c in [([0, 1], cands), ([0, 1, 2, 0], cands + cands[:1]), ([0, 1, 3], cands),
                         ([0, 1, -1], cands), ([0.0, 1.0, 2.0], cands), ([[0, 1, 2]], cands), ([1, 0, 2], cands),
                         ([0, 1, 2], [cands[0], cands[1], cands[2].astype(np.float64)]), ([], []),
                         ([0, 1, 2], [cands[0], cands[1], np.ascontiguousarray(cands[2][:, :, ::-1])[:, :, :5]])]:
            with pytest.raises(ValueError):
                s.diffmap(index, c)
        u8, u8c = srgb_set(SMALL[:3], [3, 4, 3], [0, 1, 2])
        with pytest.raises(ValueError):
            s.diffmap([0, 1, 2], u8c)
        dm, score = s.diffmap(range(2), cands[:2])  # n < capacity, any int sequence
        assert [d.shape for d in dm] == [(8, 8), (17, 9)] and score.shape == (2,) and score.dtype == np.float64
    finally:
        s.close()
    t = gb.ComparatorSet.from_srgb(u8, capacity=3, lib=lib)
    try:
        rgba_as_rgb = u8c[1][..., :3].copy()
        for c in ([u8c[0], rgba_as_rgb, u8c[2]], [u8c[0], u8c[1], u8c[2][..., :2].copy()], cands):
            with pytest.raises(ValueError):
                t.diffmap([0, 1, 2], c)
        with pytest.raises(ValueError):
            gb.ComparatorSet.from_srgb([u8[0][..., :2].copy()], lib=lib)
    finally:
        t.close()


# ---- CPU: the port (pair by pair through the owning batch's compare_batch_sizes*), and every reference
# call of the GPU tests ----------------------------------------------------------------------------------

def test_port_set_matches_reference(port_lib, ref):
    origs, cands = float_set(SMALL, SMALL_INDEX)
    got = scored(port_lib, origs, SMALL_INDEX, cands)
    check_reference(ref, origs, SMALL_INDEX, got, cands=cands)
    assert_same(got, pairs_scored(port_lib, origs, SMALL_INDEX, cands), "diffmap_sizes")


def test_port_srgb_set_matches_reference(port_lib, ref):
    imgs, cands = srgb_small()
    got = scored(port_lib, imgs, SRGB_INDEX, cands, srgb=True)
    check_reference(ref, imgs, SRGB_INDEX, got, srgb=True, cands=cands)
    assert_same(got, pairs_scored(port_lib, imgs, SRGB_INDEX, cands, srgb=True), "diffmap_sizes_srgb")
    assert got[1][5] == 0.0, "an unchanged RGBA candidate scores 0 over both backgrounds"
    # the dark RGBA original: white scores strictly higher, and its diffmap is the result
    black, white = [ref.butteraugli_interface(planes(imgs[3], bg), planes(cands[3], bg)) for bg in (0, 255)]
    assert white[1] > black[1] and got[1][3] == white[1] and parity.bits_equal(got[0][3], white[0])


def test_port_mixed_reference_subset(ref):
    """The reference calls of test_cuda_set_mixed."""
    for a, b in mixed_reference_pairs():
        ref.butteraugli_interface(a, b)


def test_port_refusals(port_lib):
    refusals(port_lib, "no device memory")


def test_port_python_checks(port_lib):
    python_checks(port_lib)


# ---- GPU --------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_cuda_set_mixed(cuda_lib, ref):
    """Originals from 8x8 to 1920x1080 and more than 16 distinct sizes in one call (several passes): every
    candidate equals diffmap_sizes on the same pairs, and those up to 64x64 the reference."""
    shapes, index = mixed_case()
    origs, cands = float_set(shapes, index)
    got = scored(cuda_lib, origs, index, cands)
    assert_same(got, pairs_scored(cuda_lib, origs, index, cands), "diffmap_sizes")
    for k, (i, (a, b)) in enumerate(zip(mixed_reference_subset(shapes, index), mixed_reference_pairs())):
        assert parity.bits_equal(a, origs[index[i]]) and parity.bits_equal(b, cands[i])
        dm0, score0 = ref.butteraugli_interface(a, b)
        assert got[1][i] == score0 and parity.bits_equal(got[0][i], dm0), f"candidate {i}: differs from the reference"


@pytest.mark.gpu
def test_cuda_set_capacity_one_original(cuda_lib):
    """n = capacity, with one original scored against most of the call's candidates."""
    shapes = [(40, 56), (300, 411), (17, 9)]
    index = [1] * 20 + [0, 2, 0, 2]
    origs, cands = float_set(shapes, index)
    got = scored(cuda_lib, origs, index, cands, capacity=len(index))
    assert_same(got, pairs_scored(cuda_lib, origs, index, cands), "diffmap_sizes")


@pytest.mark.gpu
def test_cuda_set_independence(cuda_lib):
    """The same candidates in another order and in other company, after calls on other originals, and from
    two threads on two sets: the same bits."""
    shapes, index = mixed_case()
    shapes, index = shapes[:8] + shapes[12:], [o if o < 8 else o - 4 for o in index if not 8 <= o < 12]
    origs, cands = float_set(shapes, index)
    cap = len(index)
    s = make_set(cuda_lib, origs, cap)
    try:
        dm, score = s.diffmap(index, cands)
        order = np.random.default_rng(5).permutation(cap)
        dmp, scorep = s.diffmap([index[k] for k in order], [cands[k] for k in order])
        for j, k in enumerate(order):
            assert scorep[j] == score[k] and parity.bits_equal(dmp[j], dm[k]), f"permuted: candidate {k}"
        # candidates 0..3 alone, then in the company of other candidates of other originals
        others = [o for o in range(len(origs)) if o not in index[:4]][:6]
        _, extra = float_set(shapes, others + others)
        for idx, c in [(index[:4], cands[:4]), (others + index[:4], extra[:len(others)] + cands[:4])]:
            d, sc = s.diffmap(idx, c)
            assert (sc[-4:] == score[:4]).all() and all(parity.bits_equal(d[-4 + k], dm[k]) for k in range(4))
        # after a call on other originals only
        s.diffmap(others, extra[:len(others)])
        d, sc = s.diffmap(index, cands)
        assert (sc == score).all() and all(parity.bits_equal(x, y) for x, y in zip(d, dm))
    finally:
        s.close()
    # two sets on one device from two threads
    shapes2 = [(64, 64), (9, 40), (128, 30)]
    index2 = [0, 1, 2, 1, 0]
    origs2, cands2 = float_set(shapes2, index2)
    alone2 = scored(cuda_lib, origs2, index2, cands2)
    sets = [make_set(cuda_lib, origs, cap), make_set(cuda_lib, origs2, len(index2))]
    results, errors = [None, None], []

    def run(k, idx, c):
        try:
            for _ in range(3):
                results[k] = sets[k].diffmap(idx, c)
        except Exception as e:  # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(0, index, cands)), threading.Thread(target=run, args=(1, index2, cands2))]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        for x in sets:
            x.close()
    assert not errors, errors
    assert_same(results[0], (dm, score), "thread 0")
    assert_same(results[1], alone2, "thread 1")


@pytest.mark.gpu
def test_cuda_set_device_memory(cuda_lib):
    """Candidates in CUDA memory, written late on a side torch stream that the set must wait for: the bits of
    host memory; and 8-bit sets the same."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    shapes, index = SMALL, SMALL_INDEX
    origs, cands = float_set(shapes, index)
    imgs, ucands = srgb_set(shapes, [4, 3, 4, 3, 3, 4], index)
    side = torch.cuda.Stream(device=dev)
    for srgb, o, c in [(False, origs, cands), (True, imgs, ucands)]:
        s = make_set(cuda_lib, o, len(index), srgb=srgb)
        try:
            host = s.diffmap(index, c)
            staged = [torch.from_numpy(x).to(dev) for x in c]
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                t = [torch.zeros(x.shape, dtype=x.dtype, device=dev) for x in staged]
                torch.cuda._sleep(20_000_000)  # keeps the side stream busy: the copies below land late
                for d, x in zip(t, staged):
                    d.copy_(x)
                got = s.diffmap(index, t)
            torch.cuda.synchronize(dev)
            assert all(d.device == dev and d.dtype == torch.float32 for d in got[0])
            assert_same(([d.cpu().numpy() for d in got[0]], got[1]), host, f"device memory, srgb={srgb}")
        finally:
            s.close()


@pytest.mark.gpu
def test_cuda_srgb_set_matches_pairs(cuda_lib, ref):
    """8-bit sets, RGB and RGBA mixed, against diffmap_sizes_srgb of the same pairs, from host and CUDA memory,
    and the small set against the reference."""
    torch = pytest.importorskip("torch")
    imgs, cands = srgb_small()
    got = scored(cuda_lib, imgs, SRGB_INDEX, cands, srgb=True)
    check_reference(ref, imgs, SRGB_INDEX, got, srgb=True, cands=cands)
    shapes, index = mixed_case()
    channels = [3 + k % 2 for k in range(len(shapes))]
    imgs, cands = srgb_set(shapes, channels, index)
    want = pairs_scored(cuda_lib, imgs, index, cands, srgb=True)
    s = make_set(cuda_lib, imgs, len(index), srgb=True)
    try:
        assert_same(s.diffmap(index, cands), want, "host")
        dm, score = s.diffmap(index, [torch.from_numpy(x).cuda() for x in cands])
        assert_same(([d.cpu().numpy() for d in dm], score), want, "device")
    finally:
        s.close()


@pytest.mark.gpu
def test_cuda_set_refusals(cuda_lib):
    """Every refusal launches nothing; the device entries refuse a host pointer and a CPU tensor."""
    torch = pytest.importorskip("torch")
    refusals(cuda_lib, "rgb1[0] is not device memory of device 0 (host or unknown memory)",
             lambda: gb.counters(lib=cuda_lib)[0])
    origs, cands = float_set(SMALL[:2], [0, 1])
    s = make_set(cuda_lib, origs, 2)
    try:
        t = [torch.from_numpy(x).cuda() for x in cands]
        out = [torch.zeros(x.shape[1:], device="cuda") for x in cands]
        torch.cuda.synchronize()
        P = C.c_void_p * 2
        idx = np.array([0, 1], dtype=np.int32)
        launches = gb.counters(lib=cuda_lib)[0]

        def call(imgs, dms):
            return cuda_lib.gb200_butteraugli_comparator_set_diffmap_device(s._h, idx.ctypes.data, P(*imgs), 2,
                                                                           P(*dms), None, None)

        cpu = torch.from_numpy(cands[1].copy())
        assert not call([t[0].data_ptr(), cpu.data_ptr()], [o.data_ptr() for o in out])
        assert "rgb1[1] is not device memory of device 0 (host or unknown memory)" in gb.last_error(lib=cuda_lib)
        assert not call([x.data_ptr() for x in t], [out[0].data_ptr(), np.zeros(1, np.float32).ctypes.data])
        assert "diffmap[1] is not device memory of device 0" in gb.last_error(lib=cuda_lib)
        with pytest.raises(ValueError):  # a CPU tensor among CUDA tensors never reaches the C entry
            s.diffmap([0, 1], [t[0], cpu])
        assert gb.counters(lib=cuda_lib)[0] == launches
    finally:
        s.close()
