"""Heat maps: gb200_butteraugli_heatmap[_device] / gb.heatmap against butteraugli::CreateHeatMapImage of the
reference, byte for byte (tests/golden/heatmap_reference_answers.json, tests/golden/make_heatmap_answers.py):
real diffmaps, edge values around every threshold and segment boundary, a dense sweep, under the butteraugli
tool's thresholds and two other pairs; on the CPU port and on the GPU, one map per call and all maps in one."""
import base64
import hashlib
import json
import os

import numpy as np
import pytest

import guetzli_b200 as gb

HERE = os.path.dirname(os.path.abspath(__file__))
ANSWERS = json.load(open(os.path.join(HERE, "golden", "heatmap_reference_answers.json")))
PAIRS = {k: (float.fromhex(v[0]), float.fromhex(v[1])) for k, v in ANSWERS["thresholds"].items()}
MAPS = {k: np.frombuffer(base64.b64decode(v["f32"]), np.float32).reshape(v["h"], v["w"]).copy()
        for k, v in ANSWERS["maps"].items()}


def digest(rgb):
    return hashlib.sha256(np.ascontiguousarray(rgb).tobytes()).hexdigest()


def check_answers(lib, to_input, to_host):
    names = sorted(MAPS)
    for pname, (good, bad) in PAIRS.items():
        for name in names:
            rgb = to_host(gb.heatmap(to_input(MAPS[name]), good, bad, lib=lib))
            assert rgb.shape == MAPS[name].shape + (3,) and rgb.dtype == np.uint8
            assert digest(rgb) == ANSWERS["heatmaps"][name + ":" + pname], (name, pname)
        # every map of the pair in one call
        out = gb.heatmap([to_input(MAPS[k]) for k in names], good, bad, lib=lib)
        assert [digest(to_host(o)) for o in out] == [ANSWERS["heatmaps"][k + ":" + pname] for k in names], pname


def test_tool_thresholds():
    # the Python restatement of ButteraugliFuzzyInverse gives the reference's doubles
    assert gb.heatmap_thresholds() == PAIRS["tool"]


def test_port_matches_reference(port_lib):
    check_answers(port_lib, lambda m: m, lambda x: x)
    # None thresholds are the tool's
    m = MAPS["real_pair"]
    assert digest(gb.heatmap(m, lib=port_lib)) == ANSWERS["heatmaps"]["real_pair:tool"]


def test_port_refusals(port_lib):
    m = MAPS["real_pair"]
    for good, bad in [(0.0, 1.0), (-1.0, 1.0), (1.0, 1.0), (2.0, 1.0), (float("nan"), 1.0), (1.0, float("nan"))]:
        with pytest.raises(RuntimeError, match="butteraugli heatmap: the thresholds must satisfy 0 < good < bad"):
            gb.heatmap(m, good, bad, lib=port_lib)
    with pytest.raises(ValueError, match="at least 1 map"):
        gb.heatmap([], lib=port_lib)
    with pytest.raises(ValueError, match="must be float32"):
        gb.heatmap(m.astype(np.float64), lib=port_lib)
    with pytest.raises(ValueError, match=r"must be \[h\]\[w\]"):
        gb.heatmap(m.reshape(-1), lib=port_lib)
    # the C entry's own checks
    import ctypes as C
    P = C.c_void_p * 1
    w, h = np.array([4], np.int32), np.array([0], np.int32)
    out = np.zeros(12, np.uint8)
    assert not port_lib.gb200_butteraugli_heatmap(w.ctypes.data, h.ctypes.data, P(m.ctypes.data), 1, 1.0, 2.0,
                                                  P(out.ctypes.data), 0)
    assert gb.last_error(port_lib) == "butteraugli heatmap: map 0 is 4x0, a map has at least 1x1 pixels"
    assert not port_lib.gb200_butteraugli_heatmap(w.ctypes.data, h.ctypes.data, P(m.ctypes.data), 0, 1.0, 2.0,
                                                  P(out.ctypes.data), 0)
    assert gb.last_error(port_lib) == "butteraugli heatmap: n = 0, a call takes at least 1 map"
    # the port has no device memory: its device entry refuses
    h[0] = 3
    assert not port_lib.gb200_butteraugli_heatmap_device(w.ctypes.data, h.ctypes.data, P(m.ctypes.data), 1, 1.0, 2.0,
                                                         P(out.ctypes.data), 0, None)
    assert gb.last_error(port_lib) == "the CPU port has no device memory"


@pytest.mark.gpu
def test_cuda_matches_reference(cuda_lib):
    import torch
    check_answers(cuda_lib, lambda m: m, lambda x: x)
    check_answers(cuda_lib, lambda m: torch.from_numpy(m).cuda(), lambda x: x.cpu().numpy())


@pytest.mark.gpu
def test_cuda_one_launch_no_copies(cuda_lib):
    import torch
    names = sorted(MAPS)
    maps = [torch.from_numpy(MAPS[k]).cuda() for k in names]
    torch.cuda.synchronize()
    l0, h2d0, d2h0 = gb.counters(cuda_lib)
    out = gb.heatmap(maps, lib=cuda_lib)
    l1, h2d1, d2h1 = gb.counters(cuda_lib)
    assert l1 - l0 == 1
    assert d2h1 == d2h0
    # the table alone goes up: 256 byte steps, two pointers and a first pixel per map, and the total
    assert h2d1 - h2d0 == 8 * 256 + 16 * len(names) + 4 * (len(names) + 1)
    assert [digest(o.cpu().numpy()) for o in out] == [ANSWERS["heatmaps"][k + ":tool"] for k in names]
    # host maps: one copy up, one back, one launch
    l0, h2d0, d2h0 = gb.counters(cuda_lib)
    gb.heatmap([MAPS[k] for k in names], lib=cuda_lib)
    l1, h2d1, d2h1 = gb.counters(cuda_lib)
    px = sum(MAPS[k].size for k in names)
    assert l1 - l0 == 1 and d2h1 - d2h0 == 3 * px and h2d1 - h2d0 == 4 * px + 8 * 256 + 16 * len(names) + 4 * (
        len(names) + 1)


@pytest.mark.gpu
def test_cuda_stream_order_and_refusals(cuda_lib):
    import torch
    m = MAPS["sweep"]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t = torch.zeros(m.shape, dtype=torch.float32, device="cuda")
        torch.cuda._sleep(50_000_000)
        t.copy_(torch.from_numpy(m).cuda(non_blocking=False))
        heat = gb.heatmap(t, lib=cuda_lib)
    torch.cuda.synchronize()
    assert digest(heat.cpu().numpy()) == ANSWERS["heatmaps"]["sweep:tool"]
    # host, managed and null pointers through the C entry: refused, nothing runs
    import ctypes as C
    P = C.c_void_p * 1
    w, h = np.array([m.shape[1]], np.int32), np.array([m.shape[0]], np.int32)
    out = torch.empty(m.shape + (3,), dtype=torch.uint8, device="cuda")
    l0 = gb.counters(cuda_lib)[0]
    assert not cuda_lib.gb200_butteraugli_heatmap_device(w.ctypes.data, h.ctypes.data, P(m.ctypes.data), 1, 1.0, 2.0,
                                                         P(out.data_ptr()), 0, None)
    assert gb.last_error(cuda_lib) == ("butteraugli heatmap: diffmap[0] is not device memory of device 0 "
                                       "(host or unknown memory)")
    assert not cuda_lib.gb200_butteraugli_heatmap_device(w.ctypes.data, h.ctypes.data, P(t.data_ptr()), 1, 1.0, 2.0,
                                                         P(None), 0, None)
    assert gb.last_error(cuda_lib) == "butteraugli heatmap: map 0 has a null pointer"
    assert gb.counters(cuda_lib)[0] == l0


COMPAT_MAIN = r"""
#include <stdio.h>
#include <stdlib.h>
#include "guetzli_b200_compat.h"
int main(int argc, char** argv) {
  const int w = atoi(argv[1]), h = atoi(argv[2]);
  const double good = strtod(argv[3], nullptr), bad = strtod(argv[4], nullptr);
  std::vector<float> d(static_cast<size_t>(w) * h);
  if (fread(d.data(), sizeof(float), d.size(), stdin) != d.size()) return 2;
  std::vector<uint8_t> heat;
  if (!guetzli_b200::CreateHeatMapImage(d, good, bad, w, h, &heat)) return 1;
  fwrite(heat.data(), 1, heat.size(), stdout);
  return 0;
}
"""


def test_port_compat_create_heat_map_image(port_lib, tmp_path):
    """guetzli_b200::CreateHeatMapImage (the compat header) on the CPU port: the reference's bytes."""
    import subprocess
    root = os.path.dirname(HERE)
    src, exe = tmp_path / "heat.cc", tmp_path / "heat"
    src.write_text(COMPAT_MAIN)
    build = os.path.join(root, "oracle", "_build")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(root, "include"), "-o", str(exe), str(src),
                           "-L" + build, "-lguetzli_port", "-Wl,-rpath," + build])
    for name, pname in [("real_bees", "tool"), ("edges_q_3", "q_3")]:
        m = MAPS[name]
        good, bad = PAIRS[pname]
        r = subprocess.run([str(exe), str(m.shape[1]), str(m.shape[0]), good.hex(), bad.hex()], input=m.tobytes(),
                           stdout=subprocess.PIPE, check=True)
        assert hashlib.sha256(r.stdout).hexdigest() == ANSWERS["heatmaps"][name + ":" + pname], name
    r = subprocess.run([str(exe), "4", "3", "1.0", "1.0"], input=bytes(48), stdout=subprocess.PIPE)
    assert r.returncode == 1
