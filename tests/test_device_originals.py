"""Comparators and comparator sets made from originals in CUDA memory, and the mask and adaptive quantization
into CUDA memory: each is the object, or gives the bits, that its host twin does (gb200_*_create[_srgb]_device,
gb200_butteraugli_comparator_set_create[_srgb]_device, gb200_butteraugli_comparator_mask_device,
gb200_butteraugli_adaptive_quantization_device and gb.Comparator / gb.ComparatorSet / gb.adaptive_quantization on
tensors).  Stream order, no pixel copies, refusals that run nothing, and JPEG files decoded in CUDA memory scored
end to end."""
import ctypes as C
import io

import numpy as np
import pytest
from PIL import Image

import guetzli_b200 as gb
from guetzli_b200 import synth
from test_srgb_inputs import small_pair


def floats(h, w, seed):
    return np.ascontiguousarray(synth.gradnoise(h, w, seed).transpose(2, 0, 1).astype(np.float32))


def srgb(h, w, channels, seed):
    img = synth.gradnoise(h, w, seed)
    if channels == 4:
        alpha = (synth.noise(h, w, seed + 7)[..., :1] // 64 * 85).astype(np.uint8)
        img = np.concatenate([img, alpha], axis=2)
    return np.ascontiguousarray(img)


def near(x, seed):
    """x with small changes, same dtype"""
    d = synth.noise(*(x.shape[:2] if x.dtype == np.uint8 else x.shape[-2:]), seed)[..., 0].astype(np.int16) % 7 - 3
    if x.dtype == np.uint8:
        return np.clip(x.astype(np.int16) + (d[..., None] if x.ndim == 3 else d), 0, 255).astype(np.uint8)
    return (x + d.astype(np.float32)).astype(np.float32)


def same(a, b):
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    b = b.cpu().numpy() if hasattr(b, "cpu") else np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _managed(nbytes):
    """nbytes of managed memory (cuMemAllocManaged) -> (pointer, free)."""
    try:
        cuda = C.CDLL("libcuda.so.1")
    except OSError:
        pytest.skip("no libcuda")
    p = C.c_uint64()
    assert cuda.cuMemAllocManaged(C.byref(p), C.c_size_t(nbytes), 1) == 0  # CU_MEM_ATTACH_GLOBAL
    return p.value, lambda: cuda.cuMemFree_v2(p)


# ---- CPU port: the device entries refuse, as every other device entry of the port does ----

def test_port_device_entries_refuse(port_lib):
    a = floats(16, 16, 1)
    u = srgb(16, 16, 3, 1)
    P = C.c_void_p * 1
    w, h, ch = np.array([16], np.int32), np.array([16], np.int32), np.array([3], np.int32)
    msg = "the CPU port has no device memory"
    assert not port_lib.gb200_butteraugli_comparator_create_device(a.ctypes.data, 16, 16, 1, 0, None)
    assert gb.last_error(port_lib) == msg
    assert not port_lib.gb200_butteraugli_comparator_create_srgb_device(u.ctypes.data, 16, 16, 3, 1, 0, None)
    assert gb.last_error(port_lib) == msg
    assert not port_lib.gb200_butteraugli_comparator_set_create_device(w.ctypes.data, h.ctypes.data,
                                                                       P(a.ctypes.data), 1, 1, 0, None)
    assert gb.last_error(port_lib) == msg
    assert not port_lib.gb200_butteraugli_comparator_set_create_srgb_device(w.ctypes.data, h.ctypes.data,
                                                                            ch.ctypes.data, P(u.ctypes.data), 1, 1,
                                                                            0, None)
    assert gb.last_error(port_lib) == msg
    q = np.empty((16, 16), np.float32)
    assert not port_lib.gb200_butteraugli_adaptive_quantization_device(a.ctypes.data, 16, 16, 0, q.ctypes.data, None)
    assert gb.last_error(port_lib) == msg
    c = gb.Comparator(a, lib=port_lib)
    m = np.empty((3, 16, 16), np.float32)
    assert not port_lib.gb200_butteraugli_comparator_mask_device(c._h, m.ctypes.data, m.ctypes.data, None)
    assert gb.last_error(port_lib) == msg
    # the host twins' checks come first, with their messages
    assert not port_lib.gb200_butteraugli_comparator_create_device(a.ctypes.data, 7, 16, 1, 0, None)
    assert gb.last_error(port_lib) == "butteraugli comparator: the image must be at least 8x8 (and below 65536)"
    assert not port_lib.gb200_butteraugli_adaptive_quantization_device(a.ctypes.data, 15, 16, 0, q.ctypes.data, None)
    assert gb.last_error(port_lib) == ("butteraugli adaptive quantization: the image must be at least 16x16 "
                                       "(and below 65536)")


# ---- GPU ----

def _torch():
    import torch
    return torch


@pytest.mark.gpu
@pytest.mark.parametrize("capacity", [1, 3])
def test_cuda_float_comparator(cuda_lib, capacity):
    torch = _torch()
    h, w = 37, 53
    rgb0 = floats(h, w, 3)
    cands = np.stack([near(rgb0, 10 + i) for i in range(capacity)])
    host = gb.Comparator(rgb0, capacity=capacity, lib=cuda_lib)
    dev = gb.Comparator(torch.from_numpy(rgb0).cuda(), capacity=capacity, lib=cuda_lib)
    for c1 in (cands[0], torch.from_numpy(cands[0]).cuda(), cands, torch.from_numpy(cands).cuda()):
        d0, s0 = host.diffmap(c1)
        d1, s1 = dev.diffmap(c1)
        assert same(d0, d1) and np.array_equal(np.asarray(s0), np.asarray(s1))
    m0, mdc0 = host.mask()
    m1, mdc1 = dev.mask(cuda=True)
    assert m1.is_cuda and same(m0, m1) and same(mdc0, mdc1)
    assert same(m0, dev.mask()[0])


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [3, 4])
def test_cuda_srgb_comparator(cuda_lib, channels):
    torch = _torch()
    h, w = 41, 30
    img0 = srgb(h, w, channels, 5)
    cands = np.stack([near(img0, 20 + i) for i in range(3)])
    host = gb.Comparator.from_srgb(img0, capacity=3, lib=cuda_lib)
    dev = gb.Comparator.from_srgb_device(torch.from_numpy(img0).cuda(), capacity=3, lib=cuda_lib)
    for c1 in (cands[1], torch.from_numpy(cands[1]).cuda(), cands, torch.from_numpy(cands).cuda()):
        d0, s0 = host.diffmap(c1)
        d1, s1 = dev.diffmap(c1)
        assert same(d0, d1) and np.array_equal(np.asarray(s0), np.asarray(s1))
    if channels == 3:
        assert same(host.mask()[1], dev.mask(cuda=True)[1])


SET_SIZES = [(24, 40), (8, 8), (57, 33), (24, 40), (16, 65)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["float", "srgb"])
def test_cuda_sets(cuda_lib, kind):
    torch = _torch()
    if kind == "float":
        origs = [floats(h, w, 30 + i) for i, (h, w) in enumerate(SET_SIZES)]
        make = gb.ComparatorSet
    else:
        origs = [srgb(h, w, 4 if i % 2 else 3, 30 + i) for i, (h, w) in enumerate(SET_SIZES)]
        make = gb.ComparatorSet.from_srgb
    cands = [near(o, 60 + i) for i, o in enumerate(origs)]
    host = make(origs, capacity=4, lib=cuda_lib)
    dev = make([torch.from_numpy(o).cuda() for o in origs], capacity=4, lib=cuda_lib)
    index = [4, 0, 2, 1]
    for c1 in ([cands[i] for i in index], [torch.from_numpy(cands[i]).cuda() for i in index]):
        d0, s0 = host.diffmap(index, c1)
        d1, s1 = dev.diffmap(index, c1)
        assert all(same(a, b) for a, b in zip(d0, d1)) and np.array_equal(s0, s1)
    # and each pair as a batch of pairs of different sizes scores it
    batch = gb.ButteraugliBatch(65, 65, 4, lib=cuda_lib)
    sizes = batch.diffmap_sizes if kind == "float" else batch.diffmap_sizes_srgb
    d2, s2 = sizes([origs[i] for i in index], [cands[i] for i in index])
    d1, s1 = dev.diffmap(index, [cands[i] for i in index])
    assert all(same(a, b) for a, b in zip(d1, d2)) and np.array_equal(s1, s2)


@pytest.mark.gpu
def test_cuda_adaptive_quantization(cuda_lib):
    torch = _torch()
    for h, w in [(16, 16), (45, 70)]:
        rgb = floats(h, w, h + w)
        q1 = gb.adaptive_quantization(torch.from_numpy(rgb).cuda(), lib=cuda_lib)
        assert q1.is_cuda and same(gb.adaptive_quantization(rgb, lib=cuda_lib), q1)
    with pytest.raises(ValueError, match="at least 16x16"):
        gb.adaptive_quantization(torch.zeros((3, 15, 20), device="cuda"), lib=cuda_lib)


@pytest.mark.gpu
def test_cuda_stream_order_and_analysed_once(cuda_lib):
    """Originals still being written on a side stream are read after that work; overwriting them after creation
    changes no later score."""
    torch = _torch()
    rgb0, img0 = floats(40, 48, 8), srgb(40, 48, 4, 8)
    cand, cand8 = near(rgb0, 9), near(img0, 9)
    want = gb.Comparator(rgb0, lib=cuda_lib).diffmap(cand)
    want8 = gb.Comparator.from_srgb(img0, lib=cuda_lib).diffmap(cand8)
    want_set = gb.ComparatorSet.from_srgb([img0], lib=cuda_lib).diffmap([0], [cand8])
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t = torch.zeros(rgb0.shape, dtype=torch.float32, device="cuda")
        t8 = torch.zeros(img0.shape, dtype=torch.uint8, device="cuda")
        src, src8 = torch.from_numpy(rgb0).cuda(), torch.from_numpy(img0).cuda()
        torch.cuda._sleep(100_000_000)
        t.copy_(src)
        t8.copy_(src8)
        c = gb.Comparator(t, lib=cuda_lib)
        c8 = gb.Comparator.from_srgb_device(t8, lib=cuda_lib)
        s = gb.ComparatorSet.from_srgb([t8], lib=cuda_lib)
        t.zero_()
        t8.zero_()
    torch.cuda.synchronize()
    got = c.diffmap(cand)
    assert same(got[0], want[0]) and got[1] == want[1]
    got8 = c8.diffmap(cand8)
    assert same(got8[0], want8[0]) and got8[1] == want8[1]
    got_set = s.diffmap([0], [cand8])
    assert same(got_set[0][0], want_set[0][0]) and np.array_equal(got_set[1], want_set[1])


@pytest.mark.gpu
def test_cuda_no_pixel_copies(cuda_lib):
    torch = _torch()
    h, w = 96, 128
    rgb0, img0 = floats(h, w, 2), srgb(h, w, 4, 2)
    t, t8 = torch.from_numpy(rgb0).cuda(), torch.from_numpy(img0).cuda()
    origs = [srgb(hh, ww, 3 + i % 2, i) for i, (hh, ww) in enumerate(SET_SIZES)]
    touts = [torch.from_numpy(o).cuda() for o in origs]
    torch.cuda.synchronize()

    def moved(make):
        make()  # first: whatever is made once per process
        c0 = gb.counters(cuda_lib)
        make()
        c1 = gb.counters(cuda_lib)
        return c1[1] - c0[1], c1[2] - c0[2]

    for host, dev, pixel_bytes in [
            (lambda: gb.Comparator(rgb0, lib=cuda_lib), lambda: gb.Comparator(t, lib=cuda_lib), 3 * h * 128 * 4),
            (lambda: gb.Comparator.from_srgb(img0, lib=cuda_lib),
             lambda: gb.Comparator.from_srgb_device(t8, lib=cuda_lib), 2 * h * w * 4),
            (lambda: gb.ComparatorSet.from_srgb(origs, capacity=2, lib=cuda_lib),
             lambda: gb.ComparatorSet.from_srgb(touts, capacity=2, lib=cuda_lib), sum(o.nbytes for o in origs))]:
        h2d_host, _ = moved(host)
        h2d_dev, d2h_dev = moved(dev)
        assert d2h_dev == 0
        assert h2d_dev <= h2d_host - pixel_bytes, (h2d_dev, h2d_host, pixel_bytes)


@pytest.mark.gpu
def test_cuda_refusals(cuda_lib):
    torch = _torch()
    rgb0, img0 = floats(16, 16, 1), srgb(16, 16, 3, 1)
    t = torch.from_numpy(rgb0).cuda()
    w, h, ch = np.array([16], np.int32), np.array([16], np.int32), np.array([3], np.int32)
    P = C.c_void_p * 1
    torch.cuda.synchronize()
    before = gb.counters(cuda_lib)
    ptr, free = _managed(rgb0.nbytes)
    try:
        for p in (rgb0.ctypes.data, ptr):
            why = "is not device memory of device 0 (host or unknown memory)"
            assert not cuda_lib.gb200_butteraugli_comparator_create_device(p, 16, 16, 1, 0, None)
            assert gb.last_error(cuda_lib) == f"butteraugli comparator: rgb0 {why}"
            assert not cuda_lib.gb200_butteraugli_comparator_create_srgb_device(p, 16, 16, 3, 1, 0, None)
            assert gb.last_error(cuda_lib) == f"butteraugli comparator: img0 {why}"
            assert not cuda_lib.gb200_butteraugli_comparator_set_create_device(w.ctypes.data, h.ctypes.data, P(p), 1,
                                                                               1, 0, None)
            assert gb.last_error(cuda_lib) == f"butteraugli comparator set: rgb0[0] {why}"
            assert not cuda_lib.gb200_butteraugli_comparator_set_create_srgb_device(w.ctypes.data, h.ctypes.data,
                                                                                    ch.ctypes.data, P(p), 1, 1, 0,
                                                                                    None)
            assert gb.last_error(cuda_lib) == f"butteraugli comparator set: img0[0] {why}"
            assert not cuda_lib.gb200_butteraugli_adaptive_quantization_device(p, 16, 16, 0, t.data_ptr(), None)
            assert gb.last_error(cuda_lib) == f"butteraugli adaptive quantization: rgb {why}"
    finally:
        free()
    # null pointers, small sizes and capacities: the host twins' messages
    assert not cuda_lib.gb200_butteraugli_comparator_create_device(None, 16, 16, 1, 0, None)
    assert gb.last_error(cuda_lib) == "butteraugli comparator: no image"
    assert not cuda_lib.gb200_butteraugli_comparator_create_device(t.data_ptr(), 16, 7, 1, 0, None)
    assert gb.last_error(cuda_lib) == "butteraugli comparator: the image must be at least 8x8 (and below 65536)"
    for cap in (0, 16384):
        assert not cuda_lib.gb200_butteraugli_comparator_create_device(t.data_ptr(), 16, 16, cap, 0, None)
        assert gb.last_error(cuda_lib) == "butteraugli comparator: the capacity must be in 1..16383"
        assert not cuda_lib.gb200_butteraugli_comparator_set_create_device(w.ctypes.data, h.ctypes.data,
                                                                           P(t.data_ptr()), 1, cap, 0, None)
        assert gb.last_error(cuda_lib) == "butteraugli comparator set: the capacity must be in 1..16383"
    h[0] = 7
    assert not cuda_lib.gb200_butteraugli_comparator_set_create_device(w.ctypes.data, h.ctypes.data,
                                                                       P(t.data_ptr()), 1, 1, 0, None)
    assert gb.last_error(cuda_lib) == ("butteraugli comparator set: original 0 is 16x7, the originals must be at "
                                       "least 8x8 (and below 65536)")
    assert not cuda_lib.gb200_butteraugli_comparator_set_create_device(w.ctypes.data, h.ctypes.data, P(None), 1, 1,
                                                                       0, None)
    c = gb.Comparator.from_srgb(srgb(16, 16, 4, 3), lib=cuda_lib)
    torch.cuda.synchronize()
    before = gb.counters(cuda_lib)
    assert not cuda_lib.gb200_butteraugli_comparator_mask_device(c._h, t.data_ptr(), t.data_ptr(), None)
    assert gb.last_error(cuda_lib).startswith("butteraugli comparator: an RGBA comparator has two originals")
    c = gb.Comparator(rgb0, lib=cuda_lib)
    torch.cuda.synchronize()
    before = gb.counters(cuda_lib)
    m = np.empty_like(rgb0)
    assert not cuda_lib.gb200_butteraugli_comparator_mask_device(c._h, m.ctypes.data, t.data_ptr(), None)
    assert gb.last_error(cuda_lib) == ("butteraugli comparator: mask is not device memory of device 0 "
                                       "(host or unknown memory)")
    assert gb.counters(cuda_lib) == before
    # mixed lists are refused in Python
    with pytest.raises(ValueError, match="must all be CUDA tensors or all host arrays"):
        gb.ComparatorSet([rgb0, t], lib=cuda_lib)


@pytest.mark.gpu
def test_cuda_refusals_run_nothing(cuda_lib):
    torch = _torch()
    rgb0 = floats(16, 16, 1)
    w, h = np.array([16], np.int32), np.array([16], np.int32)
    P = C.c_void_p * 1
    torch.cuda.synchronize()
    before = gb.counters(cuda_lib)
    assert not cuda_lib.gb200_butteraugli_comparator_create_device(rgb0.ctypes.data, 16, 16, 4, 0, None)
    assert not cuda_lib.gb200_butteraugli_comparator_set_create_device(w.ctypes.data, h.ctypes.data,
                                                                       P(rgb0.ctypes.data), 1, 4, 0, None)
    assert not cuda_lib.gb200_butteraugli_adaptive_quantization_device(rgb0.ctypes.data, 16, 16, 0,
                                                                       rgb0.ctypes.data, None)
    assert gb.counters(cuda_lib) == before


def test_port_from_srgb_device_checks(port_lib):
    """from_srgb keeps taking host memory only; from_srgb_device takes CUDA tensors only.  Both refuse before the
    library is called."""
    launches = gb.counters(lib=port_lib)[0]
    with pytest.raises(ValueError, match="must be a CUDA tensor"):
        gb.Comparator.from_srgb_device(srgb(16, 16, 3, 1), lib=port_lib)
    with pytest.raises(ValueError, match="must have 3 axes"):
        gb.Comparator.from_srgb_device(srgb(16, 16, 3, 1)[None], lib=port_lib)
    assert gb.counters(lib=port_lib)[0] == launches


@pytest.mark.gpu
def test_cuda_from_srgb_device_checks(cuda_lib):
    """A tensor goes to from_srgb_device, which makes the comparator from_srgb makes of the same bytes; from_srgb
    itself still refuses a tensor (as butteraugli_srgb does) and runs nothing."""
    torch = _torch()
    a, b = (torch.from_numpy(x).cuda() for x in small_pair(16, 16, 4, 3))
    launches = gb.counters(lib=cuda_lib)[0]
    with pytest.raises(ValueError, match="host memory"):
        gb.Comparator.from_srgb(a, lib=cuda_lib)
    with pytest.raises(ValueError, match="must be uint8"):
        gb.Comparator.from_srgb_device(a.float(), lib=cuda_lib)
    assert gb.counters(lib=cuda_lib)[0] == launches
    d0, s0 = gb.Comparator.from_srgb(a.cpu().numpy(), lib=cuda_lib).diffmap(b)
    d1, s1 = gb.Comparator.from_srgb_device(a, lib=cuda_lib).diffmap(b)
    assert same(d0, d1) and s0 == s1


def _pillow_jpeg(img, q):
    b = io.BytesIO()
    Image.fromarray(img).save(b, format="JPEG", quality=q)
    return b.getvalue()


@pytest.mark.gpu
def test_cuda_decoded_originals_end_to_end(cuda_lib):
    """Pillow-written files decoded from CUDA memory, a set made from the decoded originals and decoded candidates
    scored against it: the all-host pipeline's scores, with nothing copied back but header prefixes and status
    words."""
    torch = _torch()
    sizes = [(480, 640), (389, 517), (256, 256)]
    imgs = [synth.gradnoise(h, w, 40 + i) for i, (h, w) in enumerate(sizes)]
    files0 = [_pillow_jpeg(im, 95) for im in imgs]
    files1 = [_pillow_jpeg(im, 60) for im in imgs]
    # all host: decode to numpy, set from numpy, candidates numpy
    orig_h = gb.decode_jpeg(files0, cuda=False, lib=cuda_lib)
    cand_h = gb.decode_jpeg(files1, cuda=False, lib=cuda_lib)
    index = [2, 0, 1]
    want = gb.ComparatorSet.from_srgb(orig_h, capacity=3, lib=cuda_lib).diffmap(index, [cand_h[i] for i in index])
    # CUDA memory end to end
    t0 = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in files0]
    t1 = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in files1]
    torch.cuda.synchronize()
    c0 = gb.counters(cuda_lib)
    orig_d = gb.decode_jpeg(t0, lib=cuda_lib)
    cand_d = gb.decode_jpeg(t1, lib=cuda_lib)
    c1 = gb.counters(cuda_lib)
    s = gb.ComparatorSet.from_srgb(orig_d, capacity=3, lib=cuda_lib)
    c2 = gb.counters(cuda_lib)
    got = s.diffmap(index, [cand_d[i] for i in index])
    torch.cuda.synchronize()
    c3 = gb.counters(cuda_lib)
    assert np.array_equal(got[1], want[1])
    assert all(same(a, b) for a, b in zip(got[0], want[0]))
    # decode_jpeg reads each header twice (the frame sizes, then the decode) from prefixes of at most 4 KiB, and
    # copies back its status words; the set's creation copies back nothing, its call the n scores
    prefixes = sum(min(len(f), 4096) for f in files0 + files1)
    assert c1[2] - c0[2] <= 2 * prefixes + 4096, (c1[2] - c0[2], prefixes)
    assert c1[2] - c0[2] < sum(len(f) for f in files0 + files1) and c1[2] - c0[2] < sum(3 * h * w for h, w in sizes)
    assert c2[2] == c1[2]
    assert c3[2] - c2[2] == 4 * len(index)
