#!/usr/bin/env python3
"""The reference's heat maps, recorded for tests/test_heatmap.py: butteraugli::CreateHeatMapImage
(butteraugli.cc:1979) of oracle/_ref/libguetzli_ref.so, called with thresholds of the caller's choice through a
small shim compiled here against that library -> tests/golden/heatmap_reference_answers.json.  Runs where
build() could make oracle/_ref; the tests read only what it writes.

Maps (float32, each recorded with its values):
  real_pair: the reference's diffmap of test_butteraugli's 48x40 CLI pair;
  real_bees: the reference's diffmap of a 64x96 crop of bees_rgb.npz against the crop with every value raised
      by 3 on one channel per pixel row;
  edges_<pair>: 0, -0, negatives, denormals, the smallest normal, each threshold and its float32 neighbours
      (3 either side of the float nearest it), the scores at which score * 11 crosses 1..10 with their
      neighbours, and values far above `bad` up to FLT_MAX and +inf;
  sweep: 16384 floats evenly spread over 0..4, and 4096 more geometric from 1e-6 to 1e6.
Threshold pairs: the butteraugli tool's (ButteraugliFuzzyInverse(1.5), (0.5)), (1.0, 2.0) and (0.25, 3.0).
Each map is recorded under every pair: sha256 of the [h][w][3] bytes."""
import base64
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..", "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import reflib  # noqa: E402
from guetzli_b200 import synth  # noqa: E402

SHIM = r"""
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include <vector>
namespace butteraugli {
double ButteraugliFuzzyInverse(double seek);
void CreateHeatMapImage(const std::vector<float>& distmap, double good_threshold, double bad_threshold,
                        size_t xsize, size_t ysize, std::vector<uint8_t>* heatmap);
}
extern "C" double shim_fuzzy_inverse(double seek) { return butteraugli::ButteraugliFuzzyInverse(seek); }
extern "C" void shim_heatmap(const float* dm, int w, int h, double good, double bad, uint8_t* rgb) {
  std::vector<float> in(dm, dm + (size_t)w * h);
  std::vector<uint8_t> out;
  butteraugli::CreateHeatMapImage(in, good, bad, w, h, &out);
  memcpy(rgb, out.data(), out.size());
}
"""

# test_butteraugli's sRGB -> linear table (butteraugli_main.cc:137)
_TABLE = np.array([255.0 * ((i / 255.0) / 12.92 if i / 255.0 <= 0.04045 else ((i / 255.0 + 0.055) / 1.055) ** 2.4)
                   for i in range(256)])


def linear(rgb):
    return np.ascontiguousarray(_TABLE[rgb].transpose(2, 0, 1)).astype(np.float32)


def shim():
    ref_dir = os.path.abspath(os.path.join(ROOT, "oracle", "_ref"))
    tmp = tempfile.mkdtemp()
    src, so = os.path.join(tmp, "shim.cc"), os.path.join(tmp, "libheatshim.so")
    open(src, "w").write(SHIM)
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, src, "-L" + ref_dir, "-lguetzli_ref",
                           "-Wl,-rpath," + ref_dir])
    lib = C.CDLL(so)
    lib.shim_fuzzy_inverse.restype = C.c_double
    lib.shim_fuzzy_inverse.argtypes = [C.c_double]
    lib.shim_heatmap.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p]
    return lib


def neighbours(x, k=3):
    f = np.float32(x)
    out = [f]
    lo = hi = f
    for _ in range(k):
        lo = np.nextafter(lo, np.float32(-np.inf))
        hi = np.nextafter(hi, np.float32(np.inf))
        out += [lo, hi]
    return out


def edges(good, bad):
    tiny = np.finfo(np.float32).tiny
    v = [0.0, -0.0, -1.0, -1e-30, 1e-45, 3e-45, 1e-40, tiny, np.nextafter(tiny, np.float32(0))]
    for t in (good, bad):
        v += neighbours(t)
    # the mapped score s (before * 11) as ScoreToRgb maps it, inverted per segment: j / 11 for j = 1..10
    for j in range(1, 11):
        s = j / 11.0
        if s < 0.3:
            x = s / 0.3 * good
        elif s < 0.45:
            x = good + (s - 0.3) / 0.15 * (bad - good)
        else:
            x = bad + (s - 0.45) / 0.5 * (bad * 12)
        v += neighbours(x)
    v += [bad * 13, bad * 100, 1e3, 1e10, 1e30, np.finfo(np.float32).max, np.inf]
    return np.array(v, dtype=np.float32)


def main():
    sh = shim()
    if not reflib.available():
        sys.exit("oracle/_ref is missing: run __graft_entry__.build() where the reference sources are")
    good, bad = sh.shim_fuzzy_inverse(1.5), sh.shim_fuzzy_inverse(0.5)
    pairs = {"tool": (good, bad), "1_2": (1.0, 2.0), "q_3": (0.25, 3.0)}

    maps = {}
    a = synth.noise(48, 40, 77) // 2 + 64
    b = np.clip(a.astype(int) + synth.noise(48, 40, 78) % 9 - 4, 0, 255).astype(np.uint8)
    maps["real_pair"] = reflib.butteraugli_interface(linear(a.astype(np.uint8)), linear(b))[0]
    bees = np.load(os.path.join(HERE, "bees_rgb.npz"))["rgb"][100:164, 200:296]
    other = bees.astype(int)
    for y in range(other.shape[0]):
        other[y, :, y % 3] += 3
    maps["real_bees"] = reflib.butteraugli_interface(linear(bees), linear(np.clip(other, 0, 255).astype(np.uint8)))[0]
    for name, (g, bd) in pairs.items():
        e = edges(g, bd)
        maps["edges_" + name] = e.reshape(1, -1)
    sweep = np.concatenate([np.linspace(0, 4, 16384, dtype=np.float32),
                            np.geomspace(1e-6, 1e6, 4096).astype(np.float32)])
    maps["sweep"] = sweep.reshape(160, 128)

    out = {"thresholds": {k: [v[0].hex(), v[1].hex()] for k, v in pairs.items()}, "maps": {}, "heatmaps": {}}
    for name, m in maps.items():
        m = np.ascontiguousarray(m, dtype=np.float32)
        h, w = m.shape
        out["maps"][name] = {"h": h, "w": w, "f32": base64.b64encode(m.tobytes()).decode()}
        for pname, (g, bd) in pairs.items():
            rgb = np.zeros((h, w, 3), np.uint8)
            sh.shim_heatmap(m.ctypes.data, w, h, g, bd, rgb.ctypes.data)
            out["heatmaps"][name + ":" + pname] = hashlib.sha256(rgb.tobytes()).hexdigest()
    path = os.path.join(HERE, "heatmap_reference_answers.json")
    json.dump(out, open(path, "w"), indent=0, sort_keys=True)
    print(f"{path}: {len(maps)} maps x {len(pairs)} threshold pairs")


if __name__ == "__main__":
    main()
