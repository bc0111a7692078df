"""Device time of rank-k updates of the factor (cldl_updown_dev + cldl_sync_status) next to one refactor
(cldl_refactor_dev), on the KKT matrices of the benchmark's C2 and C4 workloads built as scripts/sparse_solve_time.py
builds them.  The columns are diagonals e_v (always inside the pattern) with sigma = 0.01 * dsign_v, so each update
moves a pivot away from zero; consecutive calls alternate the update and its downdate so that the matrix does not
drift.  Cases: rank 1 at a leaf (the first pivot eliminated), mid-tree and in the root separator (the last pivot),
and ranks 8, 64 and 256 at random pivots.  Each case: 2 warm-up calls, then 10 calls between CUDA events on the
handle's stream (each call waits for its verdict, as a caller who checks it does).  Printed per case: the time, its
ratio to one refactor, the fronts and panel entries reached (share of all fronts / of the stored factor), the passes
and the host time of the checks and plans; then the rank at which the update would cost a refactor, from the rank-64
and rank-256 cost per column.  The card's name and power limit are read in the same run.
Usage: python scripts/updown_time.py [out_dir]"""
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

WARM, REPS = 2, 10
out_dir = sys.argv[1] if len(sys.argv) > 1 else None
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
print("device:", card)
res = {"device": card, "warmup": WARM, "reps": REPS, "workloads": {}}


def timed(stream, fn):
    for i in range(WARM):
        fn(i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(REPS):
        fn(WARM + i)
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
    perm = s.perm()
    torch.cuda.synchronize()

    def refactor(_):
        s.refactor_dev()

    refactor_ms = timed(stream, refactor)
    assert s.sync_status() == 1
    w = {"n": N, "fronts": info.n_supernodes, "nnzL_stored": info.nnzL_stored, "refactor_ms": refactor_ms, "cases": {}}
    print("%s: n %d, %d fronts, refactor %.3f ms" % (which, N, info.n_supernodes, refactor_ms))
    rng = np.random.default_rng(1)

    def case(label, verts):
        k = len(verts)
        sigma = 0.01 * ds[verts].astype(np.float64)
        colptr = np.arange(k + 1)
        dw = torch.ones(k, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()

        def call(i):
            s.updown_dev(colptr, verts, dw.data_ptr(), sigma if i % 2 == 0 else -sigma)
            assert s.sync_status() == 1

        ms = timed(stream, call)
        st = s.updown_stats()
        c = {"rank": k, "ms": ms, "vs_refactor": ms / refactor_ms, **st,
             "share_fronts": st["fronts"] / info.n_supernodes, "share_entries": st["entries"] / info.nnzL_stored}
        w["cases"][label] = c
        print("  %-22s %8.3f ms (%.3fx refactor)  %d passes, fronts %d (%.2f%%), entries %.2f%%, plan %.3f ms (host)"
              % (label, ms, ms / refactor_ms, st["passes"], st["fronts"], 100 * c["share_fronts"],
                 100 * c["share_entries"], st["plan_ms"]))
        return ms

    case("rank 1 at a leaf", np.array([perm[0]]))
    case("rank 1 mid-tree", np.array([perm[N // 2]]))
    case("rank 1 in the root", np.array([perm[N - 1]]))
    per_col = {}
    for k in (8, 64, 256):
        ms = case("rank %d spread" % k, rng.choice(N, k, replace=False))
        per_col[k] = ms / k
    # the update's cost grows about linearly in the rank once the passes dominate: the rank at which it would cost one
    # refactor, from the marginal cost per column between ranks 64 and 256
    slope = (w["cases"]["rank 256 spread"]["ms"] - w["cases"]["rank 64 spread"]["ms"]) / (256 - 64)
    cross = 64 + (refactor_ms - w["cases"]["rank 64 spread"]["ms"]) / slope if slope > 0 else float("inf")
    w["crossover_rank"] = cross
    print("  crossover: about rank %.0f (marginal %.3f ms per column)" % (cross, slope))
    res["workloads"][which] = w
    s.close()
    torch.cuda.empty_cache()
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "updown_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
