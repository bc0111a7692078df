"""Cost of null-pivot detection and of the null-space basis.  On the KKT matrices of the benchmark's C2 and C4 workloads
(built as scripts/sparse_solve_time.py builds them): device time of a refactor with the test off and with it on at a
tolerance below every pivot (nothing found), alternated, REPS of each between CUDA events on the handle's stream after 2
of warm-up.  On the Laplacian of a 600 x 600 grid cut into 8 strips (8 null pivots): host-clock time of
cldl_null_space_dev per column, with and without the residuals, next to one full solve.  The card's name and power
limit are read in the same run.  Usage: python scripts/null_space_time.py [reps] [out_dir]"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import clarabel_rs_b200 as cb  # noqa: E402
from helpers import workloads  # noqa: E402

WARM = 2
REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
out_dir = sys.argv[2] if len(sys.argv) > 2 else None
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
print("device:", card)
res = {"device": card, "warmup": WARM, "reps": REPS, "workloads": {}}


def refactor_ms(s, stream):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    s.refactor_dev()
    e1.record(stream)
    assert s.sync_status() == 1
    return e0.elapsed_time(e1)


for which in ("c2", "c4"):
    if which == "c2":
        pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
        ordering = cb.ORDER_ND
    else:
        pr = workloads.block_angular_qp(seed=3)
        ordering = cb.ORDER_BEST
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=ordering)
    stream = torch.cuda.ExternalStream(s.stream_ptr())
    assert s.refactor()
    tol = 1e-30                       # below every pivot of these matrices: the test runs, nothing is null
    for _ in range(WARM):
        s.set_null_pivot_tol(0.0); refactor_ms(s, stream)
        s.set_null_pivot_tol(tol); refactor_ms(s, stream)
    off, on = [], []
    for _ in range(REPS):
        s.set_null_pivot_tol(0.0); off.append(refactor_ms(s, stream))
        s.set_null_pivot_tol(tol); on.append(refactor_ms(s, stream))
    assert s.inertia()[2] == 0
    w = {"n": N, "refactor_off_ms": float(np.mean(off)), "refactor_on_ms": float(np.mean(on)),
         "refactor_off_median_ms": float(np.median(off)), "refactor_on_median_ms": float(np.median(on))}
    print("%s: n %d  refactor, test off %.3f ms (median %.3f), on with nothing found %.3f ms (median %.3f)"
          % (which, N, w["refactor_off_ms"], w["refactor_off_median_ms"], w["refactor_on_ms"], w["refactor_on_median_ms"]))
    res["workloads"][which] = w
    s.close()
    torch.cuda.empty_cache()

# the Laplacian of a grid cut into strips: one null pivot per strip
nx, ny, strips = 600, 600, 8
idx = np.arange(nx * ny).reshape(ny, nx)
keep = (np.arange(nx - 1) + 1) % (nx // strips) != 0
i = np.concatenate([idx[:, :-1][:, keep].ravel(), idx[:-1, :].ravel()])
j = np.concatenate([idx[:, 1:][:, keep].ravel(), idx[1:, :].ravel()])
n = nx * ny
A = sp.coo_matrix((np.ones(i.size), (i, j)), shape=(n, n))
A = ((A + A.T) > 0).astype(np.float64)
U = sp.triu(sp.diags(np.asarray(A.sum(axis=1)).ravel()) - A).tocsc()
U.sort_indices()
s = cb.CudaLDLSolver(n, U.indptr.astype(np.int64), U.indices.astype(np.int64), U.data, np.ones(n, np.int8),
                     null_pivot_tol=1e-8)
assert s.refactor()
r = s.inertia()[2]
assert r == strips, r
dV = torch.empty((r, n), dtype=torch.float64, device="cuda")
f = s._L.cldl_null_space_dev
f.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(C.c_double)]
f.restype = C.c_int
torch.cuda.synchronize()
lap = {"n": n, "null_pivots": r}
for label, with_resid in (("null_space_per_column_ms", True), ("null_space_per_column_no_resid_ms", False)):
    resid = np.empty(r)
    rp = resid.ctypes.data_as(C.POINTER(C.c_double)) if with_resid else None
    for _ in range(WARM):
        assert f(s._h, r, C.c_void_p(dV.data_ptr()), rp) == 0
    t0 = time.perf_counter()
    for _ in range(REPS):
        assert f(s._h, r, C.c_void_p(dV.data_ptr()), rp) == 0     # synchronises: timed with the host clock
    lap[label] = (time.perf_counter() - t0) * 1e3 / REPS / r
    if with_resid:
        lap["max_resid"] = float(resid.max())
lap["full_solve_ms"] = s.time_solve_ms(REPS)
print("laplacian %dx%d in %d strips: n %d, null_space %.3f ms per column (%.3f without residuals), full solve %.3f ms,"
      " max resid %.1e" % (nx, ny, strips, n, lap["null_space_per_column_ms"], lap["null_space_per_column_no_resid_ms"],
                           lap["full_solve_ms"], lap["max_resid"]))
res["laplacian"] = lap
s.close()
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "null_space_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
