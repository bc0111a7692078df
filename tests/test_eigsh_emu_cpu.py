"""Eigenvalues nearest a shift executed on the CPU: tests/test_eigsh_gpu.py re-run against the emulated full build
(tests/emu/libclarabel_emu_full.so: ldl.cu with the sweeps and ldl_eig.cuh compiled for the host, CUDA threads as
fibers, see tests/emu/cuda_emu.h), with the threads of every block run in ascending order, in descending order, and in
a fresh random order in every scheduling pass -- the reductions' block partials are written in any order and must be
folded in one, so the results (bitwise repeatability included) must not change.  The C2-sized test is deselected: it
takes minutes under emulation.  Not a statement about the GPU: the -m gpu run is."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODULE = "tests/test_eigsh_gpu.py"


@pytest.mark.parametrize("order", ["ascending", "reverse", "random:11"])
def test_eigsh_module_on_the_emulated_build(order):
    lib = os.path.join(ROOT, "tests", "emu", "libclarabel_emu_full.so")
    assert os.path.exists(lib), f"{lib} missing: run `make`"
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", MODULE,
           "--deselect", MODULE + "::test_c2_sized_kkt_against_scipy_eigsh"]
    env = dict(os.environ, CLARABEL_EMU="1", CLARABEL_EMU_FULL="1", EMU_ORDER=order)
    r = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3000)
    tail = r.stdout[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail
