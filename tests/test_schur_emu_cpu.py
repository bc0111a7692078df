"""Schur complement handles executed on the CPU: tests/test_schur_gpu.py re-run against the emulated full build
(tests/emu/libclarabel_emu_full.so: ldl.cu with k_schur_assemble and the sweeps compiled for the host, CUDA threads as
fibers, see tests/emu/cuda_emu.h), with the threads of every block run in ascending order, in descending order, and
in a fresh random order in every scheduling pass -- the B-only backward queue's tasks interleave arbitrarily between
their synchronisation points, and the results (including the bitwise repeatability test) must not change.  The C4
test is deselected: it takes minutes under emulation.  Not a statement about the GPU: the -m gpu run is."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODULE = "tests/test_schur_gpu.py"


@pytest.mark.parametrize("order", ["ascending", "reverse", "random:11"])
def test_schur_module_on_the_emulated_build(order):
    lib = os.path.join(ROOT, "tests", "emu", "libclarabel_emu_full.so")
    assert os.path.exists(lib), f"{lib} missing: run `make`"
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", MODULE,
           "--deselect", MODULE + "::test_reduced_c4_linking_rows"]
    env = dict(os.environ, CLARABEL_EMU="1", CLARABEL_EMU_FULL="1", EMU_ORDER=order)
    r = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3000)
    tail = r.stdout[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail
