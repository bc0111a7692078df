"""Termination callbacks and verbose output on the CPU, against the CUDA-on-CPU emulated build of the whole product
(tests/emu/libclarabel_emu_full.so): the cases of tests/test_zz_callbacks_print_gpu.py, and a sharded solve over
torch.distributed (gloo) where one rank's callback stops every rank."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_FULL = os.path.join(ROOT, "tests", "emu", "libclarabel_emu_full.so")


def test_callback_and_print_cases_on_the_emulated_build():
    assert os.path.exists(EMU_FULL), "tests/emu/libclarabel_emu_full.so missing: run `make`"
    env = dict(os.environ, CLARABEL_EMU="1", CLARABEL_EMU_FULL="1")
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
           "tests/test_zz_callbacks_print_gpu.py"]
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (out.stdout + out.stderr)[-3000:]
    assert out.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail


WORKER = r'''
import os, sys
import torch.distributed as dist
sys.path.insert(0, ROOT); sys.path.insert(0, ROOT + "/tests")
os.environ["CLARABEL_EMU"] = "1"
import clarabel_rs_b200 as cb
cb.pkg._LIBPATH = ROOT + "/tests/emu/libclarabel_emu_full.so"
from helpers import workloads
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
pr = workloads.random_sparse_qp(n=400, m=800, nnz_per_row=4, seed=2, window=30)
dev = cb.CudaSolver(pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"], cb.default_settings(verbose=1), ordering=cb.ORDER_ND,
                    nd_leaf=60, shard=(world, rank))
dev.print_to_buffer()
L = cb.pkg._lib2()
def solve_counted():
    c0, n0 = dev._transport.calls, L.cipm_collective_count(dev._h)
    r = dev.solve()
    return r, dev._transport.calls - c0, L.cipm_collective_count(dev._h) - n0
plain, calls_plain, coll_plain = solve_counted()
assert plain["status"] == "Solved", plain["status"]
# verbose on rank 0 only: the binding turns it off on the other ranks
text = dev.get_print_buffer()
assert ("Terminated with status = Solved" in text) == (rank == 0), text[-300:]
# rank 1 stops at iteration 2, rank 0 never does: every rank ends there
dev.set_termination_callback(lambda info: rank == 1 and info.iterations >= 2)
r, calls_cb, coll_cb = solve_counted()
assert r["status"] == "CallbackTerminated" and r["iterations"] == 2, (r["status"], r["iterations"])
assert calls_cb > 0
# no callback: not one exchange more than a plain sharded solve
dev.unset_termination_callback()
again, calls_again, coll_again = solve_counted()
assert again["status"] == "Solved" and again["iterations"] == plain["iterations"]
assert (calls_again, coll_again) == (calls_plain, coll_plain), (calls_again, coll_again, calls_plain, coll_plain)
print("CB_OK %d/%d it=%d exchanges=%d/%d" % (rank, world, plain["iterations"], calls_plain, calls_cb), flush=True)
dist.destroy_process_group()
'''


def test_sharded_callback_stops_every_rank_over_gloo(tmp_path):
    assert os.path.exists(EMU_FULL), "tests/emu/libclarabel_emu_full.so missing: run `make`"
    world = 2
    script = tmp_path / "worker.py"
    script.write_text("ROOT = %r\n" % ROOT + WORKER)
    port = 29900 + (os.getpid() % 90)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.count("CB_OK") == world, out.stdout[-2000:]
