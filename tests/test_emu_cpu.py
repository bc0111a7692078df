"""The product's kernels, KKT layer and IPM driver executed on the CPU.

tests/emu builds clarabel.rs_b200/csrc/{cones,cones_psd,cones_nonsym,solver}.cu for the host (CUDA threads = fibers,
see tests/emu/cuda_emu.h; the multifrontal LDL is replaced by a dense host factorisation with the same pivot rule,
tests/emu/ldl_emu.cpp) and this test re-runs the GPU test modules of those layers against that build in a subprocess.
It is how the code written while no GPU was available (exponential / power / generalised power cones, the
nonsymmetric branches of the IPM loop, the inf-bound presolve) was exercised end to end before its first device run,
and it acts as a race detector for warp-synchronous code: the emulator runs the lanes of a warp one after the other
between synchronisation points, so a kernel that silently relies on lockstep execution computes something else (this
is how a missing __syncwarp in the PSD Cholesky was found).  Not a statement about the GPU: the -m gpu run is."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODULES = ["tests/test_cones_gpu.py", "tests/test_psd_gpu.py", "tests/test_ipm_gpu.py", "tests/test_zz_nonsym_gpu.py",
           "tests/test_zz_golden.py", "tests/test_zz_psd_large_gpu.py", "tests/test_zz_equilibration_gpu.py",
           "tests/test_zz_data_updating_gpu.py", "tests/test_zz_algebra_gpu.py", "tests/test_cone_shapes_gpu.py",
           "tests/test_nonsym_shapes_gpu.py"]
# lists of tests/cone_shapes.py whose KKT matrix exceeds the dense stand-in's cap (PSD 64 and up, the 1e5 SOC, the
# nonnegative pass boundaries); the full build runs PSD(64, 65)
CONE_SHAPES_BIG = ["psd-n96-97", "psd-n128", "soc-long", "nonneg-75775", "nonneg-75776", "nonneg-75777", "nonneg-300000"]
# the dense stand-in for the LDL caps the KKT dimension at 3000
TOO_BIG = ["tests/test_ipm_gpu.py::test_random_sparse_qp_same_iterations[2000-4000-60-2]",
           "tests/test_ipm_gpu.py::test_random_sparse_qp_same_iterations[1500-2000-None-3]",
           "tests/test_ipm_gpu.py::test_paired_solves_are_bitwise_the_unpaired_ones",
           "tests/test_zz_psd_large_gpu.py::test_large_psd_cone_ops_match_oracle[global-scratch]"]     # runs in the full build below
_SHAPE_TESTS = ["test_scaling_lambda_and_H", "test_combined_shift_and_ds_offset", "test_step_length"]
_SHAPE_BIG = [f"tests/test_cone_shapes_gpu.py::{t}[{n}-{r}]" for n in CONE_SHAPES_BIG for t in _SHAPE_TESTS
              for r in ("opening", "late")] + \
             [f"tests/test_cone_shapes_gpu.py::test_margins[{n}-{r}]" for n in CONE_SHAPES_BIG for r in ("opening", "late", "indefinite")] + \
             [f"tests/test_cone_shapes_gpu.py::test_nonnegative_pass_boundaries[{n}]" for n in CONE_SHAPES_BIG]
TOO_BIG += _SHAPE_BIG + [t.replace("[psd-n96-97", "[psd-n64-65") for t in _SHAPE_BIG if "psd-n96-97" in t]
# the list of tests/nonsym_shapes.py with more exp / pow cones than one grid-stride pass of the barrier sum
_NS_BIG = [f"tests/test_nonsym_shapes_gpu.py::test_update_scaling_Hs_and_secant[ns-big-{r}-{s}]"
           for r in ("opening", "late", "late-off", "edge") for s in ("primal-dual", "dual")] + \
          [f"tests/test_nonsym_shapes_gpu.py::test_barrier[ns-big-{r}]" for r in ("opening", "late", "late-off", "edge")] + \
          [f"tests/test_nonsym_shapes_gpu.py::test_step_length[ns-big-{r}]" for r in ("opening", "late")]
TOO_BIG += _NS_BIG


# ---- the whole product, multifrontal kernels included (tests/emu/libclarabel_emu_full.so) ----
FULL_MODULES = ["tests/test_ldl_gpu.py", "tests/test_ldl_shapes_gpu.py", "tests/test_zz_shard_gpu.py"] + MODULES
FULL_SKIP = [
    # minutes each under emulation (they pass: 68 of 68 in the complete run recorded in DESIGN.md)
    "tests/test_ipm_gpu.py::test_paired_solves_are_bitwise_the_unpaired_ones",
    "tests/test_ldl_gpu.py::test_full_size_roundtrip_property",
    "tests/test_ipm_gpu.py::test_random_sparse_qp_same_iterations[2000-4000-60-2]",
    "tests/test_ipm_gpu.py::test_random_sparse_qp_same_iterations[1500-2000-None-3]",
    "tests/test_ipm_gpu.py::test_update_data_then_solve_matches_fresh_solver",
    # 28 pivots replaced by +-2e-7: condition ~1e14, the host build's rounding (other FMA contraction than nvcc's) is
    # amplified past the test's 1e-7; both thread orders agree bitwise with each other and the regularisation counts
    # equal the oracle's
    "tests/test_ldl_gpu.py::test_dynamic_regularisation_counts",
] + _SHAPE_BIG + _NS_BIG



import pytest

# The four runs are independent subprocesses; all of them are started when the first test asks for its result, so the
# module costs about as long as its slowest run instead of the sum.
_JOBS = {}


def _reap():
    for job in _JOBS.values():      # -x stopped the session early: do not leave the other runs behind
        if job.poll() is None:
            job.kill()


import atexit
atexit.register(_reap)


def _spec(kind, order):
    full = kind == "full" or kind == "full-ldl"
    lib = os.path.join(ROOT, "tests", "emu", "libclarabel_emu_full.so" if full else "libclarabel_emu.so")
    modules = {"dense": MODULES, "full": FULL_MODULES, "full-ldl": ["tests/test_ldl_gpu.py", "tests/test_ldl_shapes_gpu.py",
                                                                   "tests/test_zz_shard_gpu.py"]}[kind]
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider"] + modules
    for t in (FULL_SKIP if full else TOO_BIG):
        cmd += ["--deselect", t]
    env = dict(os.environ, CLARABEL_EMU="1", EMU_ORDER=order)
    if full:
        env["CLARABEL_EMU_FULL"] = "1"
    return lib, cmd, env


ALL_RUNS = [("dense", "ascending"), ("dense", "reverse"), ("full", "ascending"), ("full-ldl", "random:7")]


def _result(kind, order):
    if not _JOBS:
        for k, o in ALL_RUNS:
            lib, cmd, env = _spec(k, o)
            assert os.path.exists(lib), f"{lib} missing: run `make`"
            _JOBS[(k, o)] = subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    job = _JOBS[(kind, order)]
    try:
        out, _ = job.communicate(timeout=3000)
    except subprocess.TimeoutExpired:
        job.kill()
        raise
    tail = out[-3000:]
    assert job.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail


@pytest.mark.parametrize("order", ["ascending", "reverse"])
def test_gpu_test_modules_pass_on_the_emulated_build(order):
    """`reverse` runs the threads of every block in descending order between synchronisation points: a kernel that is
    correct under the CUDA execution model cannot tell the difference, one that relies on lockstep lanes can."""
    _result("dense", order)


def test_every_layer_including_the_multifrontal_kernels_on_the_emulated_build():
    """ldl.cu itself -- the level-0 kernel, the persistent dataflow factorisation with its spin-waits on dependency
    counters, the pipelined dataflow solves -- runs here: the blocks of those launches are resident together as
    fibers and __nanosleep is their yield point."""
    _result("full", "ascending")


def test_multifrontal_kernels_with_a_random_schedule():
    """a fresh random permutation of all resident fibers in every scheduling pass: lanes of a warp and blocks of a
    persistent kernel interleave arbitrarily between their synchronisation points -- results (including the bitwise
    reproducibility and sharded bit-identity tests) must not change"""
    _result("full-ldl", "random:7")
