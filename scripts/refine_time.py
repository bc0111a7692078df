"""Time of refined solves and their error analysis (CudaLDLSolver.solve_refined_dev) on the KKT matrices of the
benchmark's C2 and C4 workloads, built as scripts/ldl_autograd_time.py builds them (P + 1e-3 I, so that no pivot is
regularised).  CUDA events on the handle's stream bracket each window of 10 calls after 2 of warm-up:
  plain solve            cldl_solve_dev
  refined                cldl_solve_refined_dev with the default options (tol = eps, at most 10 steps)
  error analysis         the same with error_analysis = 1 (cond1, cond2, ferr: the estimator's extra solves)
  stale refined          after cldl_update_values with a relative change of 1e-6 to every value, refined solves on the
                         factor of the old values
  refactor + solve       cldl_refactor (which collects its verdict) and one solve, on the changed values
The first refined call (mirrored pattern built and uploaded, work vectors allocated) is timed on the host clock.  The
card's name and power limit are read in the same run.  Usage: python scripts/refine_time.py [reps] [out_dir]"""
import json
import os
import subprocess
import sys
import time

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
    """average ms per call of fn(), CUDA events on `stream` (the handle's)"""
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    out = [fn() for _ in range(reps)]
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / reps, out


for which in ("c2", "c4"):
    if which == "c2":
        pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
        ordering = cb.ORDER_ND
    else:
        pr = workloads.block_angular_qp(seed=3)
        ordering = cb.ORDER_BEST
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    col = np.repeat(np.arange(N), np.diff(cp))
    nz[(rv == col) & (col < pr["P"].shape[0])] += 1e-3
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=ordering)
    assert s.refactor()
    st = torch.cuda.ExternalStream(s.stream_ptr())
    b = torch.tensor(np.random.default_rng(1).standard_normal(N), device="cuda")
    x = torch.empty_like(b)
    torch.cuda.synchronize()
    r = {"n": N, "nnzA": len(rv), "regularize_count": s.linear_solver_info().regularize_count}
    t0 = time.perf_counter()
    s.solve_refined_dev(x.data_ptr(), b.data_ptr())
    r["first_refined_call_ms"] = (time.perf_counter() - t0) * 1e3
    r["plain_solve_ms"], _ = timed(st, lambda: s.solve_dev(x.data_ptr(), b.data_ptr()))
    r["refined_ms"], infos = timed(st, lambda: s.solve_refined_dev(x.data_ptr(), b.data_ptr()))
    r["refined_steps"], r["refined_omega"] = infos[-1].steps, infos[-1].omega1 + infos[-1].omega2
    r["refined_converged"] = infos[-1].converged
    r["error_analysis_ms"], infos = timed(st, lambda: s.solve_refined_dev(x.data_ptr(), b.data_ptr(),
                                                                           error_analysis=True))
    i = infos[-1]
    r["error_analysis_solves"], r["cond1"], r["cond2"], r["ferr"] = i.solves, i.cond1, i.cond2, i.ferr
    # a relative change of 1e-6 to every value: refined solves on the old factor, then refactor + solve
    nz2 = nz * (1.0 + 1e-6 * np.random.default_rng(2).uniform(-1, 1, nz.size))
    s.update_values(np.arange(nz.size), nz2)
    i0 = s.solve_refined_dev(x.data_ptr(), b.data_ptr(), max_iter=0)
    r["stale_plain_omega"] = i0.omega1 + i0.omega2
    r["stale_refined_ms"], infos = timed(st, lambda: s.solve_refined_dev(x.data_ptr(), b.data_ptr()))
    i = infos[-1]
    r["stale_refined_steps"], r["stale_refined_omega"], r["stale_refined_converged"] = i.steps, i.omega1 + i.omega2, i.converged

    def refactor_solve():
        assert s.refactor()
        s.solve_dev(x.data_ptr(), b.data_ptr())
    r["refactor_plus_solve_ms"], _ = timed(st, refactor_solve)
    res["workloads"][which] = r
    print("%s: n %d; plain solve %.2f ms; refined %.2f ms (%d steps, omega %.1e); error analysis %.2f ms (%d solves, "
          "cond1 %.2e cond2 %.2e ferr %.1e); stale factor (1e-6): plain omega %.1e, refined %.2f ms (%d steps, omega "
          "%.1e, converged %s) against refactor + solve %.2f ms; first refined call %.0f ms (host clock)"
          % (which, N, r["plain_solve_ms"], r["refined_ms"], r["refined_steps"], r["refined_omega"],
             r["error_analysis_ms"], r["error_analysis_solves"], r["cond1"], r["cond2"], r["ferr"],
             r["stale_plain_omega"], r["stale_refined_ms"], r["stale_refined_steps"], r["stale_refined_omega"],
             r["stale_refined_converged"], r["refactor_plus_solve_ms"], r["first_refined_call_ms"]))
    s.close()
    del b, x
    torch.cuda.empty_cache()
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "refine_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
