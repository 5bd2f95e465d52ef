"""The C-ABI shared library loads without a GPU and exports every symbol that
include/guetzli_b200.h declares (no compute calls here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "guetzli_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(gb200_[a-z0-9_]+)\s*\(", text)) - {"gb200_log_fn"})


def test_product_library_exports_declared_abi():
    import guetzli_b200 as gb
    path = gb.library_path()
    if not os.path.exists(path):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(path)
    names = declared_symbols()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/guetzli_b200.h but not exported"
    lib.gb200_backend_name.restype = ctypes.c_char_p
    assert lib.gb200_backend_name() == b"cuda-sm_90a"


def test_product_has_no_cpu_fallback():
    """Without a GPU the product must fail loudly, not compute on the host."""
    import numpy as np
    import pytest
    import guetzli_b200 as gb
    lib = gb.load_library()
    if lib.gb200_device_count() > 0:
        pytest.skip("a GPU is present")
    rgb = np.zeros((40, 40, 3), dtype=np.uint8)
    with pytest.raises(RuntimeError, match="CUDA|no CUDA device"):
        gb.process(gb.Params(), None, rgb, 40, 40)
    with pytest.raises(RuntimeError):
        gb.DeviceImage(rgb)


def test_product_sources_do_not_reference_oracle():
    """oracle/ is test infrastructure: nothing under guetzli_b200/ may touch it."""
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "guetzli_b200")):
        for f in files:
            if f.endswith((".py", ".cc", ".cu", ".h", ".inc")) or f == "Makefile":
                t = open(os.path.join(d, f), errors="replace").read()
                if re.search(r"oracle/_ref|libguetzli_ref|libguetzli_port|import reflib", t):
                    bad.append(f)
    assert not bad, bad
