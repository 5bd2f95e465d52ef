import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
# every frequency-masking iteration also runs the device histogram pass and checks the
# host-maintained symbol histograms against it (search.cc, encoded_size)
os.environ.setdefault("GB200_CHECK_HOST_HIST", "1")
# The CPU port runs its emulated kernels as OpenMP loops, thousands of tiny parallel regions per
# image: with spinning waits they crawl whenever the box is busy (another job on one core is
# enough), so the workers sleep instead and the team stays small.
os.environ.setdefault("OMP_WAIT_POLICY", "passive")
os.environ.setdefault("OMP_NUM_THREADS", str(max(1, min(4, len(os.sched_getaffinity(0))))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def port_lib():
    """CPU restatement of the hot path (oracle/_build/libguetzli_port.so)."""
    import guetzli_b200 as gb
    path = os.path.join(ROOT, "oracle", "_build", "libguetzli_port.so")
    if not os.path.exists(path):
        import __graft_entry__
        __graft_entry__.build()
    return gb.load_library(path)


@pytest.fixture(scope="session")
def cuda_lib():
    """The product library; requires a GPU."""
    import guetzli_b200 as gb
    lib = gb.load_library()
    assert lib.gb200_backend_name() == b"cuda-sm_90a"
    assert lib.gb200_device_count() >= 1, "no CUDA device visible"
    return lib


@pytest.fixture(scope="session")
def ref():
    """The unmodified reference: oracle/_ref where build() could make it, else its recorded
    answers (tests/golden/reference_answers.json, see reflib.py)."""
    import reflib
    if not reflib.available():
        reflib.replay()
    return reflib
