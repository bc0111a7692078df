"""Time of solves preconditioned by the factor (CudaLDLSolver.solve_gmres_dev, restarted FGMRES with the defaults) on the
KKT matrices of the benchmark's C2 and C4 workloads, built as scripts/refine_time.py builds them (P + 1e-3 I, so that no
pivot is regularised).  The factor is always that of the original values; the cases change the handle's values after it:
  fresh          no change
  all 1e-6       every value times (1 + U(-1e-6, 1e-6))
  all 1e-2       every value times (1 + U(-1e-2, 1e-2))
  H block        the -H diagonal times (1 + U(-0.1, 0.1)), the interior-point iteration-to-iteration change
For each case: FGMRES (steps, cycles, omega, converged), refined solves on the same stale factor
(cldl_solve_refined_dev, steps, omega, converged), and refactor + solve on the changed values, each the average of a
window of `reps` calls bracketed by CUDA events on the handle's stream after 2 of warm-up.  An Arnoldi step is split
into the timed plain solve and the inferred remainder (product with K, orthogonalisation, synchronisation, the cycles'
analyses, host work): (FGMRES time - (1 + steps) solves) / steps.  The card's name and power limit are read in the same
run.  Usage: python scripts/gmres_time.py [reps] [out_dir]"""
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
from helpers import workloads  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
out_dir = sys.argv[2] if len(sys.argv) > 2 else None
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
print("device:", card)
res = {"device": card, "reps": reps, "workloads": {}}


def timed(stream, fn, warmup=2):
    """average ms per call of fn(), CUDA events on `stream` (the handle's), and the last call's result"""
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    out = [fn() for _ in range(reps)]
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / reps, out[-1]


for which in ("c2", "c4"):
    if which == "c2":
        pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
        ordering = cb.ORDER_ND
    else:
        pr = workloads.block_angular_qp(seed=3)
        ordering = cb.ORDER_BEST
    n = pr["P"].shape[0]
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    col = np.repeat(np.arange(N), np.diff(cp))
    nz[(rv == col) & (col < n)] += 1e-3
    idx = np.arange(nz.size)
    hd = (rv == col) & (col >= n)
    rng = np.random.default_rng(2)
    cases = {"fresh": nz,
             "all 1e-6": nz * (1.0 + 1e-6 * rng.uniform(-1, 1, nz.size)),
             "all 1e-2": nz * (1.0 + 1e-2 * rng.uniform(-1, 1, nz.size)),
             "H block": np.where(hd, nz * (1.0 + 0.1 * rng.uniform(-1, 1, nz.size)), nz)}
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=ordering)
    assert s.refactor()
    st = torch.cuda.ExternalStream(s.stream_ptr())
    b = torch.tensor(np.random.default_rng(1).standard_normal(N), device="cuda")
    x = torch.empty_like(b)
    torch.cuda.synchronize()
    s.solve_gmres_dev(x.data_ptr(), b.data_ptr())          # the mirrored pattern is set up outside the windows
    solve_ms, _ = timed(st, lambda: s.solve_dev(x.data_ptr(), b.data_ptr()))
    r = {"n": N, "nnzA": len(rv), "plain_solve_ms": solve_ms, "cases": {}}
    print("%s: n %d, plain solve %.3f ms" % (which, N, solve_ms))
    for name, vals in cases.items():
        s.update_values(idx, vals)
        g_ms, gi = timed(st, lambda: s.solve_gmres_dev(x.data_ptr(), b.data_ptr()))
        f_ms, fi = timed(st, lambda: s.solve_refined_dev(x.data_ptr(), b.data_ptr()))

        def refactor_solve():
            assert s.refactor()
            s.solve_dev(x.data_ptr(), b.data_ptr())
        rs_ms, _ = timed(st, refactor_solve)
        s.update_values(idx, nz)                  # back to the original values and their factor
        assert s.refactor()
        rest = (g_ms - (1 + gi.iterations) * solve_ms) / gi.iterations if gi.iterations else float("nan")
        c = {"gmres_ms": g_ms, "steps": gi.iterations, "cycles": gi.cycles, "omega": gi.omega1 + gi.omega2,
             "converged": gi.converged, "step_solve_ms": solve_ms, "step_rest_ms": rest,
             "refined_ms": f_ms, "refined_steps": fi.steps, "refined_omega": fi.omega1 + fi.omega2,
             "refined_converged": fi.converged, "refactor_plus_solve_ms": rs_ms}
        r["cases"][name] = c
        print("  %-9s FGMRES %.2f ms (%d steps, %d cycles, omega %.1e, converged %s; a step = %.3f ms solve + %.3f ms "
              "rest); refined %.2f ms (%d steps, omega %.1e, converged %s); refactor + solve %.2f ms"
              % (name, g_ms, gi.iterations, gi.cycles, c["omega"], gi.converged, solve_ms, rest, f_ms, fi.steps,
                 c["refined_omega"], fi.converged, rs_ms))
    res["workloads"][which] = r
    s.close()
    del b, x
    torch.cuda.empty_cache()
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "gmres_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
