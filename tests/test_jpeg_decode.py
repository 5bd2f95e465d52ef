"""JPEG decode on the device (gb.decode_jpeg, gb200_jpeg_decode_rgb[_device]) against libjpeg-turbo's pixels
as Pillow gave them (tests/golden/make_jpeg_decode_answers.py -> jpeg_decode_reference_answers.json, with
the generated files and small decodes in jpeg_decode_files.npz), and the `butteraugli` tool on a JPEG
argument against butteraugli::ButteraugliInterface on those pixels.  The reference calls the GPU tests make
are made by the CPU tests with the same arguments, so that

    GB200_REF_RECORD=$PWD/tests/golden/jpeg_decode_butteraugli_answers.json \\
        python -m pytest tests/test_jpeg_decode.py -m "not gpu"

records them; replay mode reads them beside golden/reference_answers.json."""
import hashlib
import json
import os
import subprocess
import threading

import numpy as np
import pytest

import guetzli_b200 as gb
import reflib
from guetzli_b200 import synth
from test_butteraugli import CLI, CLI_PORT, linear

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
ANSWERS = json.load(open(os.path.join(GOLDEN, "jpeg_decode_reference_answers.json")))["files"]
with np.load(os.path.join(GOLDEN, "jpeg_decode_files.npz")) as _z:
    NPZ = {k: _z[k] for k in _z.files}  # read once: threads of a test share it
REF_ANSWERS = os.path.join(GOLDEN, "jpeg_decode_butteraugli_answers.json")

# file -> what the refusal says (the decoder does not reproduce libjpeg-turbo on it)
REFUSED = {
    "jpeg/cmyk": "4 components (CMYK or YCCK)",
    "jpeg/truncated": "Unexpected end of scan.",
    "jpeg/garbage": "Unexpected end of input",
    "jpeg/corrupt_header": "SOS marker: Could not find AC Huffman table",
    "jpeg/corrupt_scan_prog": "Extra zero run before end-of-block.",
    # read_jpeg accepts it; its Huffman desync leaves coefficients far out of range, where Pillow's
    # (SIMD) libjpeg-turbo gives other pixels than libjpeg's C IDCT (the two differ in 4026 samples)
    "jpeg/corrupt_scan": "beyond the range in which libjpeg-turbo's SIMD IDCT computes its C IDCT's samples",
    "q255_ac": "beyond the range in which libjpeg-turbo's SIMD IDCT computes its C IDCT's samples",
    "sub440": "sampling factors 1x2, 1x1, 1x1: only 4:4:4, 4:2:2 and 4:2:0 are decoded",
    "sub411": "sampling factors 4x1, 1x1, 1x1: only 4:4:4, 4:2:2 and 4:2:0 are decoded",
    "prog_cut": "not refined to their last bit: libjpeg block-smooths it",
}


def data(name):
    if name.startswith("jpeg/"):
        return open(os.path.join(GOLDEN, name + ".jpg"), "rb").read()
    return NPZ["file_" + name].tobytes()


ACCEPTED = sorted(n for n in ANSWERS if n not in REFUSED)
SWEEP = [n for n in ACCEPTED if n.startswith("sweep_")]


def check_pixels(name, px):
    px = np.asarray(px)
    want = ANSWERS[name]
    assert list(px.shape) == want["shape"], name
    if hashlib.sha256(np.ascontiguousarray(px).tobytes()).hexdigest() == want["pillow"]:
        return
    key = "px_" + name.replace("/", "_")
    if key in NPZ:
        bad = np.argwhere(px != NPZ[key])[0]
        raise AssertionError(f"{name}: first differing sample (y, x, c) = {tuple(bad)}: "
                             f"{px[tuple(bad)]} against libjpeg-turbo's {NPZ[key][tuple(bad)]}")
    raise AssertionError(f"{name}: pixels differ from libjpeg-turbo's")


def test_answers_cover_the_fixtures():
    fixtures = {"jpeg/" + f[:-4] for f in os.listdir(os.path.join(GOLDEN, "jpeg"))}
    assert fixtures <= set(ANSWERS)
    assert {"sweep_444_1x9", "sweep_422_2x9", "sweep_420_11x1", "sweep_gray_65x65", "rgb_ids", "q255_dc",
            "guetzli_q90"} <= set(ACCEPTED)


# ---- CPU port: the same kernel bodies through the host entry -------------------------------------------

def test_port_bit_equal(port_lib):
    for name in ACCEPTED:
        check_pixels(name, gb.decode_jpeg(data(name), cuda=False, lib=port_lib))


def test_port_one_mixed_call(port_lib):
    names = [n for n in ACCEPTED if not n.startswith("sweep_")] + SWEEP[::7]
    out = gb.decode_jpeg([data(n) for n in names], cuda=False, lib=port_lib)
    for n, px in zip(names, out):
        check_pixels(n, px)


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_port_refusals(port_lib, name):
    before = gb.counters(lib=port_lib)
    ok_file = data("jpeg/base444_q90")
    with pytest.raises(ValueError) as e:
        gb.decode_jpeg([ok_file, data(name)], cuda=False, lib=port_lib)
    assert str(e.value).startswith("jpeg_decode_rgb: file 1: ") and REFUSED[name] in str(e.value)
    assert gb.counters(lib=port_lib) == before


def test_port_device_entry_refuses(port_lib):
    import ctypes as C
    d = np.frombuffer(data("jpeg/tiny444"), np.uint8)
    out = np.zeros((24, 40, 3), np.uint8)
    ok = port_lib.gb200_jpeg_decode_rgb_device((C.c_void_p * 1)(d.ctypes.data), (C.c_size_t * 1)(d.size), 1, 0,
                                              (C.c_void_p * 1)(out.ctypes.data), None)
    assert not ok and "no device memory" in gb.last_error(lib=port_lib)


def cli_case(name):
    """(original [h][w][3], the JPEG's libjpeg-turbo pixels) of a CLI case"""
    if name == "guetzli_q90":
        return synth.gradnoise(64, 96, 7), NPZ["px_guetzli_q90"]
    return synth.gradnoise(72, 100, 3), NPZ["px_jpeg_sub420"]  # make_golden_jpeg.py's image of sub420


@pytest.fixture(scope="module")
def ref(ref):
    if reflib._answers is not None:
        with open(REF_ANSWERS) as f:
            reflib._answers.update(json.load(f))
    return ref


def check_cli(cli, ref, tmp_path, name):
    from PIL import Image
    orig, px = cli_case(name)
    po, pj = str(tmp_path / "orig.png"), str(tmp_path / "out.jpg")
    Image.fromarray(orig).save(po)
    open(pj, "wb").write(data(name if name == "guetzli_q90" else "jpeg/sub420"))
    _, score = ref.butteraugli_interface(linear(orig), linear(px))
    r = subprocess.run([cli, po, pj], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 0, r.stderr
    assert r.stdout.decode() == "%f\n" % score
    # a refused JPEG, and a JPEG against an RGBA PNG
    open(pj, "wb").write(data("jpeg/cmyk"))
    r = subprocess.run([cli, po, pj], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 1 and f"File {pj} is a malformed JPEG.\n" in r.stderr.decode()
    open(pj, "wb").write(data(name if name == "guetzli_q90" else "jpeg/sub420"))
    Image.fromarray(np.dstack([orig, orig[..., :1]])).save(po)
    r = subprocess.run([cli, po, pj], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 1 and r.stderr.decode() == "Different number of channels: 4 vs 3\n"


@pytest.mark.parametrize("name", ["guetzli_q90", "sub420"])
def test_port_cli(port_lib, ref, tmp_path, name):
    check_cli(CLI_PORT, ref, tmp_path, name)


def test_port_decode_then_comparator_set(port_lib, ref):
    for name in ["guetzli_q90", "sub420"]:
        orig, px = cli_case(name)
        img = gb.decode_jpeg(data(name if name == "guetzli_q90" else "jpeg/sub420"), cuda=False, lib=port_lib)
        s = gb.ComparatorSet.from_srgb([orig], capacity=1, lib=port_lib)
        _, score = s.diffmap([0], [img])
        _, want = ref.butteraugli_interface(linear(orig), linear(px))
        assert float(score[0]) == want


# ---- on the GPU ---------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_cuda_bit_equal_host_and_device(cuda_lib):
    import torch
    for name in ACCEPTED:
        host = gb.decode_jpeg(data(name), cuda=False, lib=cuda_lib)
        check_pixels(name, host)
        dev = gb.decode_jpeg(data(name), lib=cuda_lib)
        assert dev.is_cuda and dev.dtype == torch.uint8
        assert np.array_equal(dev.cpu().numpy(), host), name


@pytest.mark.gpu
def test_cuda_one_mixed_call(cuda_lib):
    out = gb.decode_jpeg([data(n) for n in ACCEPTED], lib=cuda_lib)
    for n, px in zip(ACCEPTED, out):
        check_pixels(n, px.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("sub", [0, 2])
def test_cuda_1080p_against_pillow(cuda_lib, sub):
    Image = pytest.importorskip("PIL.Image", reason="Pillow writes and decodes the 1080p files")
    import io
    rgb = synth.gradnoise(1080, 1920, 11)
    b = io.BytesIO()
    Image.fromarray(rgb).save(b, "JPEG", quality=90, subsampling=sub)
    want = np.asarray(Image.open(io.BytesIO(b.getvalue())).convert("RGB"))
    got = gb.decode_jpeg(b.getvalue(), lib=cuda_lib).cpu().numpy()
    assert np.array_equal(got, want)


@pytest.mark.gpu
def test_cuda_decode_then_comparator_set_on_one_stream(cuda_lib):
    import torch
    names = ["guetzli_q90", "sub420"]
    origs = [cli_case(n)[0] for n in names]
    s = gb.ComparatorSet.from_srgb(origs, capacity=2, lib=cuda_lib)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        imgs = gb.decode_jpeg([data("guetzli_q90"), data("jpeg/sub420")], lib=cuda_lib)
        _, dev_scores = s.diffmap([0, 1], imgs)
    _, host_scores = s.diffmap([0, 1], [cli_case(n)[1] for n in names])
    assert np.array_equal(np.asarray(dev_scores), np.asarray(host_scores))


@pytest.mark.gpu
def test_cuda_refusals_launch_nothing(cuda_lib):
    for name in sorted(REFUSED):
        before = gb.counters(lib=cuda_lib)
        with pytest.raises(ValueError, match="file 0: "):
            gb.decode_jpeg(data(name), cuda=False, lib=cuda_lib)
        with pytest.raises(ValueError, match="file 0: "):
            gb.decode_jpeg(data(name), lib=cuda_lib)
        assert gb.counters(lib=cuda_lib) == before, name


@pytest.mark.gpu
def test_cuda_device_pointer_refusals(cuda_lib):
    import ctypes as C
    import torch
    d = np.frombuffer(data("jpeg/tiny444"), np.uint8)
    jp, ln = (C.c_void_p * 1)(d.ctypes.data), (C.c_size_t * 1)(d.size)
    host = np.zeros((24, 40, 3), np.uint8)
    before = gb.counters(lib=cuda_lib)
    assert not cuda_lib.gb200_jpeg_decode_rgb_device(jp, ln, 1, 0, (C.c_void_p * 1)(host.ctypes.data), None)
    assert "out[0] is not device memory of device 0 (host or unknown memory)" in gb.last_error(lib=cuda_lib)
    pinned = torch.empty((24, 40, 3), dtype=torch.uint8).pin_memory()
    assert not cuda_lib.gb200_jpeg_decode_rgb_device(jp, ln, 1, 0, (C.c_void_p * 1)(pinned.data_ptr()), None)
    assert "out[0] is not device memory" in gb.last_error(lib=cuda_lib)
    if torch.cuda.device_count() > 1:
        other = torch.empty((24, 40, 3), dtype=torch.uint8, device="cuda:1")
        assert not cuda_lib.gb200_jpeg_decode_rgb_device(jp, ln, 1, 0, (C.c_void_p * 1)(other.data_ptr()), None)
        assert "(device 1)" in gb.last_error(lib=cuda_lib)
    assert not cuda_lib.gb200_jpeg_decode_rgb_device(jp, ln, 1, 0, (C.c_void_p * 1)(None), None)
    assert "out[0] is null" in gb.last_error(lib=cuda_lib)
    assert gb.counters(lib=cuda_lib) == before


@pytest.mark.gpu
def test_cuda_two_threads(cuda_lib):
    names = ACCEPTED[::3]
    errors = []

    def run(seq):
        try:
            for _ in range(3):
                for n, px in zip(seq, gb.decode_jpeg([data(n) for n in seq], lib=cuda_lib)):
                    check_pixels(n, px.cpu().numpy())
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=run, args=(names,)), threading.Thread(target=run, args=(names[::-1],))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["guetzli_q90", "sub420"])
def test_cuda_cli(cuda_lib, ref, tmp_path, name):
    check_cli(CLI, ref, tmp_path, name)


@pytest.mark.gpu
def test_cuda_decode_then_comparator_set_scores(cuda_lib, ref):
    for name in ["guetzli_q90", "sub420"]:
        orig, px = cli_case(name)
        img = gb.decode_jpeg(data(name if name == "guetzli_q90" else "jpeg/sub420"), lib=cuda_lib)
        s = gb.ComparatorSet.from_srgb([orig], capacity=1, lib=cuda_lib)
        _, score = s.diffmap([0], [img])
        _, want = ref.butteraugli_interface(linear(orig), linear(px))
        assert float(score[0]) == want
