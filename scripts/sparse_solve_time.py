"""Device time of pruned solves (cldl_solve_sparse_dev, cldl_inverse_entries) next to one full solve
(cldl_solve_dev), on the KKT matrices of the benchmark's C2 and C4 workloads built as scripts/selinv_time.py builds
them.  Each case: 2 warm-up calls, then 10 calls between CUDA events on the handle's stream.  Printed per case: the
time, its ratio to a full solve, the fronts and panel entries the pruned sweeps reach (share of all fronts / of the
stored factor) and the host time spent building the plans.  The card's name and power limit are read in the same
run.  Usage: python scripts/sparse_solve_time.py [out_dir]"""
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

WARM, REPS = 2, 10
out_dir = sys.argv[1] if len(sys.argv) > 1 else None
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
print("device:", card)
res = {"device": card, "warmup": WARM, "reps": REPS, "workloads": {}}


def timed(stream, fn):
    for _ in range(WARM):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(REPS):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / REPS


for which in ("c2", "c4"):
    if which == "c2":
        pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
        ordering = cb.ORDER_ND
    else:
        pr = workloads.block_angular_qp(seed=3)
        ordering = cb.ORDER_BEST
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=ordering)
    assert s.refactor()
    info = s.linear_solver_info()
    stream = torch.cuda.ExternalStream(s.stream_ptr())
    rng = np.random.default_rng(1)
    db = torch.tensor(rng.standard_normal(N), dtype=torch.float64, device="cuda")
    dx = torch.empty(N, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    full_ms = timed(stream, lambda: s._L.cldl_solve_dev(s._h, dx.data_ptr(), db.data_ptr()))
    w = {"n": N, "fronts": info.n_supernodes, "nnzL_stored": info.nnzL_stored, "full_solve_ms": full_ms, "cases": {}}
    print("%s: n %d, %d fronts, full solve %.3f ms" % (which, N, info.n_supernodes, full_ms))

    def record(label, ms, st):
        c = {"ms": ms, "vs_full": ms / full_ms, **st,
             "share_fronts_fwd": st["fronts_fwd"] / info.n_supernodes,
             "share_fronts_bwd": st["fronts_bwd"] / info.n_supernodes,
             "share_entries_fwd": st["entries_fwd"] / info.nnzL_stored,
             "share_entries_bwd": st["entries_bwd"] / info.nnzL_stored}
        w["cases"][label] = c
        print("  %-26s %8.3f ms (%.2fx full)  fronts fwd %d / bwd %d, entries %.1f%% / %.1f%%, plan %.3f ms (host)"
              % (label, ms, ms / full_ms, st["fronts_fwd"], st["fronts_bwd"], 100 * c["share_entries_fwd"],
                 100 * c["share_entries_bwd"], st["plan_ms"]))

    # one column of K^-1: b = e_j, x wanted everywhere and at the one entry
    j = int(rng.integers(N))
    dv = torch.ones(1, dtype=torch.float64, device="cuda")
    dxs = torch.empty(1000, dtype=torch.float64, device="cuda")
    ms = timed(stream, lambda: s.solve_sparse_dev([j], dv.data_ptr(), 1, None, dx.data_ptr()))
    record("column of K^-1", ms, s.sparse_stats())
    ms = timed(stream, lambda: s.solve_sparse_dev([j], dv.data_ptr(), 1, [j], dxs.data_ptr()))
    record("diagonal entry of K^-1", ms, s.sparse_stats())
    for nb in (10, 100):
        bi = rng.choice(N, nb, replace=False)
        bv = torch.tensor(rng.standard_normal(nb), dtype=torch.float64, device="cuda")
        wi = rng.choice(N, 10, replace=False)
        ms = timed(stream, lambda: s.solve_sparse_dev(bi, bv.data_ptr(), nb, None, dx.data_ptr()))
        record("b nnz %d, x full" % nb, ms, s.sparse_stats())
        ms = timed(stream, lambda: s.solve_sparse_dev(bi, bv.data_ptr(), nb, wi, dxs.data_ptr()))
        record("b nnz %d, x at 10" % nb, ms, s.sparse_stats())
    for k in (100, 1000):
        ri, ci = rng.integers(0, N, k), rng.integers(0, N, k)
        for _ in range(WARM):
            s.inverse_entries(ri, ci)
        t0 = time.perf_counter()
        for _ in range(REPS):
            s.inverse_entries(ri, ci)      # host call, synchronises: timed with the host clock
        ms = (time.perf_counter() - t0) * 1e3 / REPS
        st = s.sparse_stats()
        record("%d entries of K^-1" % k, ms, st)
        w["cases"]["%d entries of K^-1" % k]["full_solves_equivalent_ms"] = k * full_ms
    res["workloads"][which] = w
    s.close()
    torch.cuda.empty_cache()
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "sparse_solve_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
