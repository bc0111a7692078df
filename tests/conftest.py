import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    if os.environ.get("CLARABEL_EMU") == "1":
        # test_emu_cpu.py re-runs GPU test modules in a subprocess against the CUDA-on-CPU emulated build of the cone /
        # KKT / IPM layer (tests/emu/cuda_emu.h).  Test-side switch only: the product loader is not involved.
        import clarabel_rs_b200 as cb
        cb.pkg._LIBPATH = os.path.join(ROOT, "tests", "emu", "libclarabel_emu_full.so" if os.environ.get("CLARABEL_EMU_FULL") == "1" else "libclarabel_emu.so")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure both shared libraries exist (build is idempotent and quick)."""
    import subprocess
    need = [os.path.join(ROOT, "clarabel.rs_b200", "libclarabel_b200.so"),
            os.path.join(ROOT, "oracle", "liboracle.so"),
            os.path.join(ROOT, "tests", "host_harness", "libns3_host.so"),
            os.path.join(ROOT, "tests", "host_harness", "libfake_cudart.so"),
            os.path.join(ROOT, "tests", "emu", "libclarabel_emu.so"),
            os.path.join(ROOT, "tests", "emu", "libclarabel_emu_full.so")]
    if not all(os.path.exists(p) for p in need):
        subprocess.check_call(["make", "-s", "-C", ROOT, "-j8"], stdout=subprocess.DEVNULL,
                              stderr=subprocess.DEVNULL)
    yield
