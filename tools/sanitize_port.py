"""Workload of tools/sanitize_port.sh: known-answer images, every JPEG fixture, damaged JPEG
files, a small butteraugli comparison, an image of twin tiles (reference-ordered path and the
experimental device order replay in check mode) and strip mode, all on the sanitised CPU port."""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import guetzli_b200 as gb  # noqa: E402
import parity  # noqa: E402
from guetzli_b200 import synth  # noqa: E402

lib = gb.load_library(os.environ["GB200_SAN_LIB"])
for name in ("gradnoise_64x96_s7_q90", "tiny_20x40_s5_q95", "gray_64x64_s9_q90", "odd_70x51_s3_q88",
             "gradnoise_128x128_s11_q84"):
    parity.check_golden(lib, name)
print("golden images ok", flush=True)
G = json.load(open(os.path.join(ROOT, "tests", "golden", "golden_jpeg.json")))
for name in sorted(G):
    data = open(os.path.join(ROOT, "tests", "golden", "jpeg", name + ".jpg"), "rb").read()
    g = G[name]
    p = gb.Params(butteraugli_target=gb.butteraugli_score_for_quality(g["quality"], lib=lib),
                  clear_metadata=g["clear_metadata"])
    ok, j = gb.process_jpeg(p, None, data, lib=lib)
    if name != "sub420":
        assert ok == g["ok"] and hashlib.sha256(j).hexdigest() == g["jpeg_sha256"], name
print("jpeg fixtures ok", flush=True)
rng = np.random.default_rng(5)
for fx in ("prog444_q85", "restart444", "meta_kept", "sub420"):
    base = open(os.path.join(ROOT, "tests", "golden", "jpeg", fx + ".jpg"), "rb").read()
    for t in range(200):
        b = bytearray(base)
        for _ in range(rng.integers(1, 5)):
            b[rng.integers(2, len(b))] = rng.integers(0, 256)
        if t % 4 == 0:
            b = b[:rng.integers(4, len(b))]
        gb.api.read_jpeg(bytes(b), lib=lib)
print("damaged jpeg files ok", flush=True)
# the device path's entropy decoding (segment pass, speculative decode, DC sums) as host loops, on baseline
# files cut after their SOS header and with single scan bytes changed: read_jpeg's coefficients or the host path
for fx in ("tiny444", "sub420"):
    base = open(os.path.join(ROOT, "tests", "golden", "jpeg", fx + ".jpg"), "rb").read()
    sos = base.find(b"\xff\xda")
    start = sos + 2 + ((base[sos + 2] << 8) | base[sos + 3])
    variants = [base[:k] for k in range(start, len(base))]
    for k in range(start, len(base) - 2):
        for x in (0x01, 0x80, 0xff):
            v = bytearray(base)
            v[k] ^= x
            variants.append(bytes(v))
    for i, b in enumerate(variants):
        taken, coeffs = gb.api.entropy_decode(b, 33 if i % 2 else 1024, lib=lib)
        if taken:
            ok, _, want = gb.api.read_jpeg(b, lib=lib)
            assert ok and np.array_equal(coeffs[:want.size], want), (fx, i)
print("device entropy decoding of damaged files ok", flush=True)
a = synth.gradnoise(20, 33, 2).astype(np.float32).transpose(2, 0, 1)
gb.api.butteraugli_diffmap(a, a[:, ::-1].copy(), lib=lib)
rgb = np.ascontiguousarray(np.tile(synth.noise(64, 64, 3), (1, 2, 1)))
parity.run_process(lib, rgb, 93)
print("twin tiles ok", flush=True)
p = gb.Params(butteraugli_target=gb.butteraugli_score_for_quality(90, lib=lib))
img = synth.gradnoise(96, 80, 5)
ok1, j1 = gb.process(p, None, img, 80, 96, lib=lib)
for world in (2, 3):
    ok, j = gb.process_tiled_threads(p, img, 80, 96, world, lib=lib)
    assert ok and j == j1, world
print("strip mode ok", flush=True)
# the size pass / file assembly as a call of its own on adversarial coefficient patterns, the
# Huffman builder on skewed histograms, force_420 on a grayscale image
import reflib  # noqa: E402

if reflib.available():
    parity.check_device_save_jpeg(lib, reflib, synth.gradnoise(40, 33, 2), 2)
    print("device save_jpeg ok", flush=True)
import ctypes as C  # noqa: E402

lib.gb200_debug_huffman_depths.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
lib.gb200_debug_huffman_depths.restype = None
for t in range(300):
    counts = (1 + 4_000_000 * rng.random(257) ** 8).astype(np.uint32)
    counts[rng.random(257) < 0.3] = 0
    counts[256] = 1
    depth = np.zeros(257, dtype=np.uint8)
    lib.gb200_debug_huffman_depths(counts.ctypes.data, 257, 16, depth.ctypes.data)
    assert depth.max() <= 16
print("huffman ok", flush=True)
ok, _ = gb.process(gb.Params(butteraugli_target=gb.butteraugli_score_for_quality(90, lib=lib), force_420=True), None,
                   parity.gray(48, 40, 3), 40, 48, lib=lib)
assert ok
print("force_420 on a grayscale image ok", flush=True)
