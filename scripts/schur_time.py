"""Device time of one Schur refactor (B's fronts: level-0 kernels + k_factor_df over B's tasks, then k_schur_assemble)
next to one ordinary refactor of the same matrix, with CUDA events on the handle's stream (cldl_time_refactor_ms), on
the KKT matrices of the benchmark's C2 (a random Schur set of 500) and C4 (the Schur set = its 2000 linking rows).
Handle creation -- ordering, analysis, plans and allocations, all on the host -- is timed for both handles with the
host clock.  The card's name and power limit are read in the same run.
Usage: python scripts/schur_time.py [reps] [out_dir]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

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
for which in ("c2", "c4"):
    if which == "c2":
        pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
        ordering = cb.ORDER_ND
    else:
        pr = workloads.block_angular_qp(seed=3)
        ordering = cb.ORDER_BEST
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    S = np.random.default_rng(1).choice(N, size=500, replace=False) if which == "c2" else np.arange(N - 2000, N)
    r = {"n": N, "nschur": int(S.size)}
    for kind, kw in (("ordinary", {}), ("schur", {"schur": S})):
        t0 = time.perf_counter()
        s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=ordering, **kw)
        r[kind + "_create_ms_host"] = (time.perf_counter() - t0) * 1e3
        for _ in range(2):
            assert s.refactor()
        r[kind + "_refactor_ms"] = s.time_refactor_ms(reps)
        assert s.refactor()
        if kind == "schur":
            Sc = s.schur_complement()
            r["schur_finite"] = bool(np.isfinite(Sc).all())
            b = np.random.default_rng(2).standard_normal(N)
            t0 = time.perf_counter()
            w = s.schur_reduce(b)
            x = s.schur_expand(np.linalg.solve(Sc, w))
            r["reduce_solve_expand_ms_host"] = (time.perf_counter() - t0) * 1e3
            r["x_finite"] = bool(np.isfinite(x).all())
        r[kind + "_nnzL_stored"] = s.linear_solver_info().nnzL_stored
        s.close()
    res["workloads"][which] = r
    print("%s: n %d, |S| %d: refactor %.2f ms, Schur refactor %.2f ms; create %.0f ms, Schur create %.0f ms (host clock)"
          % (which, N, S.size, r["ordinary_refactor_ms"], r["schur_refactor_ms"], r["ordinary_create_ms_host"],
             r["schur_create_ms_host"]))
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "schur_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
