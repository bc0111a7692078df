"""Device time of the differentiable sparse solve and log-determinant (autograd.SparseLDL) on the KKT matrices of the
benchmark's C2 and C4 workloads, with CUDA events on torch's stream (the layer makes torch's stream wait for the
handle's, so the events bracket the library's work), 10 calls after 2 of warm-up:
  solve forward      refactor + one LDL solve (the values alternate between two sets, so every call refactors)
  solve backward     one adjoint solve: one LDL solve + the pattern-gradient kernel (the factor is reused)
  slogdet forward    refactor + the log|d| reduction
  slogdet backward   one selected inversion (the factor is reused)
The card's name and power limit are read in the same run.  Usage: python scripts/ldl_autograd_time.py [reps] [out_dir]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import clarabel_rs_b200 as cb  # noqa: E402
from clarabel_rs_b200_pkg.autograd import SparseLDL  # noqa: E402
from helpers import workloads  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
out_dir = sys.argv[2] if len(sys.argv) > 2 else None
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
print("device:", card)
res = {"device": card, "reps": reps, "workloads": {}}


def timed(fn, warmup=2):
    for i in range(warmup):
        fn(i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        fn(i)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


for which in ("c2", "c4"):
    if which == "c2":
        pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
        ordering = cb.ORDER_ND
    else:
        pr = workloads.block_angular_qp(seed=3)
        ordering = cb.ORDER_BEST
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    # P + 1e-3 I: the KKT matrix is then quasidefinite and no pivot is regularised, which the layer requires (P alone
    # may be singular); the work of a refactor does not depend on the values
    col = np.repeat(np.arange(N), np.diff(cp))
    nz[(rv == col) & (col < pr["P"].shape[0])] += 1e-3
    probe = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=ordering)
    perm = probe.perm()
    probe.close()
    K = SparseLDL(N, cp, rv, ds, perm=perm)
    v = [torch.tensor(nz, device="cuda"), torch.tensor(nz * (1 + 1e-6), device="cuda")]
    vg = v[0].clone().requires_grad_(True)
    b = torch.tensor(np.random.default_rng(1).standard_normal(N), device="cuda", requires_grad=True)
    gx = torch.tensor(np.random.default_rng(2).standard_normal(N), device="cuda")
    r = {"n": N, "nnzA": len(rv)}
    n0 = K.refactors
    r["solve_forward_ms"] = timed(lambda i: K.solve(v[i % 2], b))
    r["refactors_in_solve_forward"] = K.refactors - n0
    x = K.solve(vg, b)
    n0 = K.refactors
    r["solve_backward_ms"] = timed(lambda i: torch.autograd.grad(x, (vg, b), gx, retain_graph=True))
    r["refactors_in_solve_backward"] = K.refactors - n0
    n0 = K.refactors
    r["slogdet_forward_ms"] = timed(lambda i: K.slogdet(v[i % 2]))
    r["refactors_in_slogdet_forward"] = K.refactors - n0
    lad = K.slogdet(vg)[1]
    n0 = K.refactors
    r["slogdet_backward_ms"] = timed(lambda i: torch.autograd.grad(lad, vg, retain_graph=True))
    r["refactors_in_slogdet_backward"] = K.refactors - n0
    r["logabsdet"] = lad.item()
    res["workloads"][which] = r
    print("%s: n %d, solve forward %.2f ms, backward %.2f ms; slogdet forward %.2f ms, backward %.2f ms "
          "(refactors per window: %d %d %d %d)"
          % (which, N, r["solve_forward_ms"], r["solve_backward_ms"], r["slogdet_forward_ms"], r["slogdet_backward_ms"],
             r["refactors_in_solve_forward"], r["refactors_in_solve_backward"], r["refactors_in_slogdet_forward"],
             r["refactors_in_slogdet_backward"]))
    K.close()
    del K, v, vg, b, gx, x, lad
    torch.cuda.empty_cache()
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "ldl_autograd_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
