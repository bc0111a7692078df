"""Solution derivatives on the CPU, against the CUDA-on-CPU emulated build of the whole product
(tests/emu/libclarabel_emu_full.so): the cases of tests/test_zz_derivative_gpu.py without the full-size one, and a
sharded handle over torch.distributed (gloo) whose derivatives are bitwise those of an unsharded handle."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_FULL = os.path.join(ROOT, "tests", "emu", "libclarabel_emu_full.so")


def test_derivative_module_on_the_emulated_build():
    assert os.path.exists(EMU_FULL), "tests/emu/libclarabel_emu_full.so missing: run `make`"
    env = dict(os.environ, CLARABEL_EMU="1", CLARABEL_EMU_FULL="1")
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_zz_derivative_gpu.py",
           "--deselect", "tests/test_zz_derivative_gpu.py::test_full_size_c2_adjoint_and_reproducibility"]
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (out.stdout + out.stderr)[-3000:]
    assert out.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail


WORKER = r'''
import os, sys
import numpy as np
import torch.distributed as dist
sys.path.insert(0, ROOT); sys.path.insert(0, ROOT + "/tests")
os.environ["CLARABEL_EMU"] = "1"
import clarabel_rs_b200 as cb
cb.pkg._LIBPATH = ROOT + "/tests/emu/libclarabel_emu_full.so"
from helpers import workloads
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
pr = workloads.random_sparse_qp(n=400, m=800, nnz_per_row=4, seed=2, window=30)
args = (pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"])
kw = dict(ordering=cb.ORDER_ND, nd_leaf=60)
one = cb.CudaSolver(*args, **kw)
dev = cb.CudaSolver(*args, shard=(world, rank), **kw)
r1, r2 = one.solve(), dev.solve()
assert r1["status"] == r2["status"] == "Solved"
rng = np.random.default_rng(11)                      # the same inputs on every rank
nP, nA = len(one._cur["P"]), len(one._cur["A"])
d = rng.standard_normal(nP), rng.standard_normal(one.n), rng.standard_normal(nA), rng.standard_normal(one.m)
g = rng.standard_normal(one.n), rng.standard_normal(one.m), rng.standard_normal(one.m)
c0 = dev._transport.calls
f1, f2 = one.derivative(*d), dev.derivative(*d)
a1, a2 = one.adjoint_derivative(*g), dev.adjoint_derivative(*g)
assert dev._transport.calls > c0                     # the sharded refactor and solves exchanged
assert all(np.array_equal(u, v) for u, v in zip(f1, f2))
assert all(np.array_equal(a1[k].data if k in "PA" else a1[k], a2[k].data if k in "PA" else a2[k]) for k in "PqAb")
print("DERIV_OK %d/%d" % (rank, world), flush=True)
dist.destroy_process_group()
'''


def test_sharded_derivatives_are_bitwise_the_unsharded_ones_over_gloo(tmp_path):
    assert os.path.exists(EMU_FULL), "tests/emu/libclarabel_emu_full.so missing: run `make`"
    world = 2
    script = tmp_path / "worker.py"
    script.write_text("ROOT = %r\n" % ROOT + WORKER)
    port = 29800 + (os.getpid() % 90)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.count("DERIV_OK") == world, out.stdout[-2000:]
