"""Time of cldl_eigsh_dev (the nev eigenvalues nearest sigma = 0, thick-restart Lanczos with one solve per step) next
to one solve (cldl_solve_dev), on the KKT matrices of the benchmark's C2 and C4 workloads built as
scripts/factor_parts_time.py builds them, with 1e-3 added to P's diagonal and regularisation off (the KKT matrix is then
quasidefinite and factors without it).  nev = 1, 6 and 32 with the default basis size.  Each case: one warm-up call,
then 3 calls between CUDA events on the handle's stream (the call synchronises once per Lanczos step, so the events
bracket whole calls).  Reported per case: ms per call, solves, restarts, and the split of a call's time per Lanczos
step into the solve (the separately timed one-solve time) and an inferred remainder (call time / solves - solve time):
the Gram-Schmidt kernels and norms, the per-step synchronisation, the host Jacobi solves, the restarts and the
residuals together.  The remainder is not timed by events of its own.
The card's name and power limit are read in the same run.
Usage: python scripts/eigsh_time.py [out_dir]"""
import json
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import clarabel_rs_b200 as cb  # noqa: E402
from helpers import workloads  # noqa: E402

WARM, REPS = 1, 3
out_dir = sys.argv[1] if len(sys.argv) > 1 else None
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
print("device:", card)
res = {"device": card, "warmup": WARM, "reps": REPS, "workloads": {}}


def timed(stream, fn, reps):
    for _ in range(WARM):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        out = fn()
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
    P = pr["P"] + 1e-3 * sp.identity(pr["P"].shape[0])
    N, cp, rv, nz, ds = workloads.kkt_triu(P, pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=ordering, regularize_enable=False)
    nb = s.factor_shifted(nz, 0.0)
    stream = torch.cuda.ExternalStream(s.stream_ptr())
    b = torch.from_numpy(np.random.default_rng(0).standard_normal(N)).cuda()
    x = torch.empty_like(b)
    torch.cuda.synchronize()
    solve_ms, _ = timed(stream, lambda: s.solve_dev(x.data_ptr(), b.data_ptr()), 10)
    w = {"n": N, "n_below": nb, "solve_ms": solve_ms, "cases": {}}
    print("%s: n %d, n_below %d, one solve %.3f ms" % (which, N, nb, solve_ms))
    for nev in (1, 6, 32):
        X = torch.empty((nev, N), dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        ms, (lam, info) = timed(stream, lambda: s.eigsh_dev(nev, 0.0, None, X.data_ptr()), REPS)
        step = ms / max(info.solves, 1)
        c = {"ms": ms, "status": info.status, "solves": info.solves, "restarts": info.restarts,
             "max_resid": info.max_resid, "step_ms": step, "step_solve_ms": solve_ms,
             "step_remainder_ms_inferred": step - solve_ms, "lam_min_abs": float(np.min(np.abs(lam)))}
        w["cases"]["nev %d" % nev] = c
        print("  nev %2d: %9.2f ms  status %d  solves %4d  restarts %3d  max_resid %.1e  per step %.3f ms = solve "
              "%.3f + inferred remainder %.3f" % (nev, ms, info.status, info.solves, info.restarts, info.max_resid, step, solve_ms,
                                     step - solve_ms))
        del X
    res["workloads"][which] = w
    s.close()
    torch.cuda.empty_cache()
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "eigsh_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
