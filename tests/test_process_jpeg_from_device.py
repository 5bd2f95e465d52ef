"""The encoder's JPEG input from CUDA memory (gb.process_jpeg on a torch tensor, gb200_process_jpeg_from_device).

A sequential 4:4:4 YCbCr file the encoder takes is Huffman-decoded, dequantised and sanity-checked on the device
(the device route); every other file is copied back and read as gb200_process_jpeg reads it (the host route).
On the CPU port, the device route's seeding (gb200_debug_jpeg_seed: entropy decode, then JpegDequantSanity) is
pinned against read_jpeg's coefficients times their quant steps and against check_jpeg_sanity's verdict.  On the
GPU, the tensor entry gives the goldens of tests/golden/golden_jpeg.json and the host entry's result, bytes, trace,
counters and refusals, takes the route the counters show, and keeps to the calling rules of the device entries."""
import ctypes as C
import hashlib
import threading

import numpy as np
import pytest

import guetzli_b200 as gb
from test_jpeg_decode_from_device import damaged, pillow
from test_jpeg_input import GOLDEN, fixture

S_DEFAULT = 1024  # kJpegSubBits, pipeline.h
SANE, INSANE, HOST = 1, 2, 0  # the hook's routes

# natural index of each zig-zag position
ZIGZAG = sorted(range(64), key=lambda i: (i // 8 + i % 8, (i % 8) if (i // 8 + i % 8) % 2 == 0 else i // 8))


def quant_of(b):
    """[components][64] quant steps (natural order) of a file, as read_jpeg assigns them: a component takes the
    first DQT table with its Tq"""
    pos, tables, comps = 2, [], []
    while pos + 4 <= len(b) and b[pos] == 0xff:
        m, n = b[pos + 1], (b[pos + 2] << 8) | b[pos + 3]
        seg = b[pos + 4:pos + 2 + n]
        if m == 0xdb:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                i += 1
                vals = [(seg[i + 2 * k] << 8) | seg[i + 2 * k + 1] if pq else seg[i + k] for k in range(64)]
                i += 128 if pq else 64
                nat = [0] * 64
                for k in range(64):
                    nat[ZIGZAG[k]] = vals[k]
                tables.append((tq, nat))
        elif m in (0xc0, 0xc1, 0xc2):
            comps = [seg[6 + 3 * c + 2] for c in range(seg[5])]
        elif m == 0xda:
            break
        pos += 2 + n
    return np.array([next(t for q, t in tables if q == tq) for tq in comps], dtype=np.int64)


def check_seed(lib, b, S, name="", cap=1 << 24):
    """The hook's plane is read_jpeg's coefficients times their quant steps (stored as int16) and its verdict
    check_jpeg_sanity's, where it takes the file -> route"""
    route, dq = gb.api.jpeg_seed(b, S, lib=lib, cap=cap)
    if route == HOST:
        return route
    ok, dims, coeffs = gb.api.read_jpeg(b, lib=lib, cap=cap)
    assert ok and dims[2] == 3, f"{name} S={S}: the device route took a file the encoder does not take"
    v = coeffs.astype(np.int64).reshape(3, -1, 64) * quant_of(b)[:, None, :]
    assert np.array_equal(dq[:v.size], v.reshape(-1).astype(np.int16)), f"{name} S={S}: dq differs"
    assert not dq[v.size:v.size + 4096].any(), f"{name} S={S}: written beyond the plane"
    assert route == (SANE if np.abs(v).max() <= 4096 else INSANE), f"{name} S={S}: sanity verdict"
    return route


def progressive(b):
    return b.find(b"\xff\xc2", 0, b.find(b"\xff\xda")) >= 0


def params_for(quality, clear_metadata=True, lib=None):
    return gb.Params(butteraugli_target=gb.butteraugli_score_for_quality(quality, lib=lib),
                     clear_metadata=clear_metadata)


# the sequential 4:4:4 fixtures the encoder takes, and the ones it refuses or reads on the host
DEVICE_ROUTE = ["base444_q90", "noise444_q92", "opt444_q97", "q100_tables1", "restart444", "tiny444", "tiny444_meta",
                "meta_kept", "meta_stripped", "corrupt_scan", "lowq"]


# ---- CPU port ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("S", [S_DEFAULT, 64, 8])
def test_port_seed_fixtures(port_lib, S):
    for name in sorted(GOLDEN):
        route = check_seed(port_lib, fixture(name), S, name)
        assert (route != HOST) == (name in DEVICE_ROUTE), name


def test_port_corrupt_scan_is_insane(port_lib):
    """read_jpeg accepts corrupt_scan and the sanity check refuses it: the device route decides that alone, with the
    host entry's message"""
    route, _ = gb.api.jpeg_seed(fixture("corrupt_scan"), S_DEFAULT, lib=port_lib)
    assert route == INSANE
    ok, out = gb.process_jpeg(params_for(92, lib=port_lib), None, fixture("corrupt_scan"), lib=port_lib)
    assert not ok and out == b""
    assert gb.last_error(lib=port_lib) == "Unsupported input JPEG (unexpectedly large coefficient values).\n"


def boundary_file(lib, k, step, coef, w=16, h=16):
    """A 4:4:4 file (written by the encoder's own writer) whose block 0 has coefficient `coef` at natural index k
    under quant step `step` there, every other step 1"""
    nb = ((w + 7) // 8) * ((h + 7) // 8)
    dq = np.zeros((3, nb, 64), dtype=np.int16)
    dq[:, :, 0] = [[40], [-24], [16]]
    dq[0, 1, 5] = -3
    dq[0, 0, k] = coef * step
    q = np.ones((3, 64), dtype=np.int32)
    q[0, k] = step
    b = gb.write_jpeg(dq.reshape(-1), w, h, q, lib=lib)
    ok, _, coeffs = gb.api.read_jpeg(b, lib=lib)
    assert ok and coeffs[k] == coef and not progressive(b)
    return b


@pytest.mark.parametrize("k", [0, 9])
@pytest.mark.parametrize("sign", [1, -1])
def test_port_sanity_boundary(port_lib, k, sign):
    """|coef * q| = 4096 passes, 4097 is refused, in DC and in AC"""
    for step, coef, want in [(16, 256, SANE), (17, 241, INSANE), (4, 1024, SANE), (241, 17, INSANE)]:
        b = boundary_file(port_lib, k, step, sign * coef)
        for S in (S_DEFAULT, 8):
            assert check_seed(port_lib, b, S, f"k={k} {sign * coef}x{step}") == want


PILLOW_444 = [(h, w, q, kw)
              for (h, w) in [(1, 1), (3, 7), (8, 8), (13, 24), (24, 17), (33, 33), (65, 40), (19, 65)]
              for q, kw in [(50, {}), (75, {"restart_marker_blocks": 1}), (90, {"restart_marker_blocks": 3}),
                            (95, {"restart_marker_rows": 1}), (100, {"restart_marker_blocks": 64})]]


def pillow_444(h, w, q, kw):
    return pillow(h, w, 0, q, seed=h * 131 + w, **kw)


@pytest.mark.parametrize("S", [S_DEFAULT, 64])
def test_port_seed_pillow_files(port_lib, S):
    pytest.importorskip("PIL.Image", reason="Pillow writes the files")
    for case in PILLOW_444:
        assert check_seed(port_lib, pillow_444(*case), S, str(case)) == SANE, case


def test_port_seed_damaged_files(port_lib):
    """files cut at every byte and with scan bytes flipped: taken only as read_jpeg reads them"""
    taken = 0
    for i, b in enumerate(damaged(fixture("tiny444"))):
        taken += check_seed(port_lib, b, 33 if i % 2 else S_DEFAULT, f"tiny444 variant {i}") != HOST
    assert taken > 0


def test_port_entry_refuses(port_lib):
    d = np.frombuffer(fixture("tiny444"), np.uint8)
    out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
    cp = gb.api._cparams(params_for(95, lib=port_lib))
    ok = port_lib.gb200_process_jpeg_from_device(C.byref(cp), d.ctypes.data, d.size, 0, C.cast(None, gb.api._LOG_FN),
                                                 None, C.byref(out), C.byref(out_len), None, None)
    assert not ok and not out_len.value and "no device memory" in gb.last_error(lib=port_lib)


def test_port_tensor_arguments(port_lib):
    torch = pytest.importorskip("torch")
    t = torch.frombuffer(bytearray(fixture("tiny444")), dtype=torch.uint8)
    with pytest.raises(ValueError, match="must be a contiguous 1-D torch.uint8 CUDA tensor"):
        gb.process_jpeg(params_for(95, lib=port_lib), None, t, lib=port_lib)


# ---- on the GPU ----------------------------------------------------------------------------------------------

def on_device(b, dev="cuda:0"):
    import torch
    if not b:
        return torch.empty(0, dtype=torch.uint8, device=dev)
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)


def encode(lib, b, quality, clear_metadata=True, tensor=True):
    """-> (ok, bytes, trace, counters, device stats, last_error)"""
    st = gb.ProcessStats(debug_output=[])
    ok, out = gb.process_jpeg(params_for(quality, clear_metadata, lib=lib), st, on_device(b) if tensor else b,
                              lib=lib)
    counters = [st.counters.get(k) for k in ("number of iterations", "number of iterations up",
                                              "number of iterations down")]
    return ok, out, "".join(st.debug_output), counters, st.device, "" if ok else gb.last_error(lib=lib)


def same_as_host(lib, b, quality, clear_metadata=True, name=""):
    """the tensor entry against the host entry on the same bytes -> both device stats"""
    dev = encode(lib, b, quality, clear_metadata)
    host = encode(lib, b, quality, clear_metadata, tensor=False)
    assert dev[:4] == host[:4] and dev[5] == host[5], name
    return dev[4], host[4]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_cuda_goldens(cuda_lib, name):
    g = GOLDEN[name]
    ok, out, trace, counters, _, err = encode(cuda_lib, fixture(name), g["quality"], g["clear_metadata"])
    if name == "sub420":  # the YUV420 search is not built: refused, as by the host entry
        assert not ok and out == b"" and "YUV420" in err
        return
    assert ok == g["ok"], name
    assert len(out) == g["jpeg_size"] and hashlib.sha256(out).hexdigest() == g["jpeg_sha256"], name
    assert hashlib.sha256(trace.encode()).hexdigest() == g["trace_sha256"], name
    assert counters == g["iterations"], name


REFUSING = ["cmyk", "gray", "sub420", "sub422", "corrupt_header", "corrupt_scan", "corrupt_scan_prog", "garbage",
            "truncated", "lowq"]


@pytest.mark.gpu
def test_cuda_refusals(cuda_lib):
    for name in REFUSING:
        g = GOLDEN[name]
        same_as_host(cuda_lib, fixture(name), g["quality"], name=name)
    # the read or sanity message comes before the params one, as on the host
    for name, want in [("truncated", "Can't read jpg data"), ("corrupt_scan", "unexpectedly large coefficient")]:
        ok, _, _, _, _, err = encode(cuda_lib, fixture(name), 80)
        assert not ok and want in err, name
        same_as_host(cuda_lib, fixture(name), 80, name=name)
    ok, _, _, _, _, err = encode(cuda_lib, b"", 90)
    assert not ok and err == "Can't read jpg data from input file\n"


def with_tail(b, tail=b"\x00trailing bytes\xff\xd9after"):
    return b + tail


@pytest.mark.gpu
def test_cuda_same_as_host_entry(cuda_lib):
    pytest.importorskip("PIL.Image", reason="Pillow writes the files")
    for h, w, q, kw in [(33, 33, 90, {}), (65, 40, 95, {"restart_marker_blocks": 3}), (48, 72, 100, {}),
                        (40, 64, 85, {"restart_marker_rows": 1})]:
        same_as_host(cuda_lib, pillow(h, w, 0, q, seed=w, **kw), 92, name=(h, w, q, kw))
    for clear in (True, False):
        b = with_tail(fixture("base444_q90"))
        dev, host = same_as_host(cuda_lib, b, 92, clear, name=f"tail, clear_metadata={clear}")
        assert dev["d2h_bytes"] < host["d2h_bytes"] + 16384  # the device route: the tail, not the file


@pytest.mark.gpu
def test_cuda_1080p(cuda_lib):
    pytest.importorskip("PIL.Image", reason="Pillow writes the files")
    b = pillow(1080, 1920, 0, 90, seed=5)
    dev, host = same_as_host(cuda_lib, b, 90, name="1080p")
    plane = 384 * 240 * 135
    assert dev["h2d_bytes"] + plane // 2 < host["h2d_bytes"], (dev, host)
    assert dev["d2h_bytes"] < host["d2h_bytes"] + 16384, (dev, host)


def intervals(b):
    """restart intervals of a file's scan (MCUs of a 4:4:4 frame)"""
    pos, r, w, h = 2, 0, 0, 0
    while b[pos] == 0xff and b[pos + 1] != 0xda:
        n = (b[pos + 2] << 8) | b[pos + 3]
        if b[pos + 1] == 0xdd:
            r = (b[pos + 4] << 8) | b[pos + 5]
        if b[pos + 1] in (0xc0, 0xc1, 0xc2):
            h, w = (b[pos + 5] << 8) | b[pos + 6], (b[pos + 7] << 8) | b[pos + 8]
        pos += 2 + n
    mcus = ((w + 7) // 8) * ((h + 7) // 8)
    return mcus, (mcus + r - 1) // r if r else 1


MAX_STATUS_BYTES = 4 * (64 + 2) + 8


@pytest.mark.gpu
def test_cuda_route_from_counters(cuda_lib):
    """device route: no coefficient plane goes up, and what comes back beyond the host entry's own copies is the
    header prefix, the status words and the tail; host route: the whole file comes back"""
    for name in sorted(GOLDEN):
        g = GOLDEN[name]
        if not g["ok"]:
            continue
        b = fixture(name)
        dev, host = same_as_host(cuda_lib, b, g["quality"], g["clear_metadata"], name=name)
        extra = dev["d2h_bytes"] - host["d2h_bytes"]
        if name in DEVICE_ROUTE:
            mcus, nint = intervals(b)
            tables = 16384 + 64 * 3 * nint
            assert dev["h2d_bytes"] <= host["h2d_bytes"] - 3 * 128 * mcus + tables, (name, dev, host)
            assert 0 < extra <= 2 * 4096 + MAX_STATUS_BYTES, (name, extra)
        else:
            assert extra >= len(b), (name, extra)


@pytest.mark.gpu
def test_cuda_damaged_files(cuda_lib):
    """each cut or flipped variant gives the host entry's outcome"""
    pytest.importorskip("PIL.Image", reason="Pillow writes the files")
    for name, b in [("tiny444", fixture("tiny444")), ("pillow 24x16 rst1", pillow(16, 24, 0, 90, restart_marker_blocks=1))]:
        for i, v in enumerate(damaged(b)):
            same_as_host(cuda_lib, v, 95, name=f"{name} variant {i}")


@pytest.mark.gpu
def test_cuda_stream_order(cuda_lib):
    import torch
    b = fixture("base444_q90")
    want = encode(cuda_lib, b, 92, tensor=False)
    pinned = torch.frombuffer(bytearray(b), dtype=torch.uint8).pin_memory()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        for _ in range(2):
            t = torch.zeros(pinned.numel(), dtype=torch.uint8, device="cuda:0")
            torch.cuda._sleep(2_000_000)  # the copy below waits behind this on the side stream
            t.copy_(pinned, non_blocking=True)
            st = gb.ProcessStats(debug_output=[])
            ok, out = gb.process_jpeg(params_for(92, lib=cuda_lib), st, t, lib=cuda_lib)
            assert ok and out == want[1] and "".join(st.debug_output) == want[2]


@pytest.mark.gpu
def test_cuda_overwritten_after_return(cuda_lib):
    t = on_device(fixture("base444_q90"))
    p = params_for(92, lib=cuda_lib)
    ok, out = gb.process_jpeg(p, None, t, lib=cuda_lib)
    t.fill_(0)
    ok2, out2 = gb.process_jpeg(p, None, fixture("base444_q90"), lib=cuda_lib)
    assert ok and ok2 and out == out2


@pytest.mark.gpu
def test_cuda_pointer_refusals(cuda_lib):
    import torch
    from test_image_inputs import _managed
    b = fixture("tiny444")
    host = np.frombuffer(b, np.uint8)
    cp = gb.api._cparams(params_for(95, lib=cuda_lib))
    torch.cuda.synchronize()
    before = gb.counters(lib=cuda_lib)

    def call(ptr, n):
        out, out_len = C.POINTER(C.c_uint8)(), C.c_size_t()
        ok = cuda_lib.gb200_process_jpeg_from_device(C.byref(cp), ptr, n, 0, C.cast(None, gb.api._LOG_FN), None,
                                                     C.byref(out), C.byref(out_len), None, None)
        assert not out_len.value
        return ok, gb.last_error(lib=cuda_lib)

    ptr, free = _managed(len(b))
    try:
        for p in (host.ctypes.data, ptr):
            assert call(p, len(b)) == (0, "process_jpeg_from_device: jpeg is not device memory of device 0 "
                                          "(host or unknown memory)")
    finally:
        free()
    if torch.cuda.device_count() >= 2:
        t = on_device(b, "cuda:1")
        torch.cuda.synchronize("cuda:1")
        assert call(t.data_ptr(), len(b)) == (0, "process_jpeg_from_device: jpeg is not device memory of device 0 "
                                                 "(device 1)")
    assert gb.counters(lib=cuda_lib) == before
    with pytest.raises(ValueError, match="must be a contiguous 1-D torch.uint8 CUDA tensor"):
        gb.process_jpeg(params_for(95, lib=cuda_lib), None, on_device(b).view(2, -1) if len(b) % 2 == 0
                        else on_device(b)[::2], lib=cuda_lib)
    with pytest.raises(ValueError, match="must be a contiguous 1-D torch.uint8 CUDA tensor"):
        gb.process_jpeg(params_for(95, lib=cuda_lib), None, torch.frombuffer(bytearray(b), dtype=torch.uint8),
                        lib=cuda_lib)


@pytest.mark.gpu
def test_cuda_two_threads(cuda_lib):
    names = ["base444_q90", "restart444", "prog444_q85", "tiny444"]
    want = {n: encode(cuda_lib, fixture(n), GOLDEN[n]["quality"], tensor=False)[:4] for n in names}
    errors = []

    def run(seq):
        try:
            for n in seq:
                got = encode(cuda_lib, fixture(n), GOLDEN[n]["quality"])[:4]
                assert got == want[n], n
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=run, args=(names,)), threading.Thread(target=run, args=(names[::-1],))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors[0]
