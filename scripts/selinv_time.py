"""Device time of one selected inversion (cldl_selected_inverse_dev: k_selinv + the caller-order gather) next to one
numeric refactor, on the KKT matrices of the benchmark's C2 and C4 workloads, with CUDA events on the handle's stream.
The first call, which builds the plan and allocates, is timed separately (host clock, synchronised).  The card's name
and power limit are read in the same run.  Usage: python scripts/selinv_time.py [reps] [out_dir]"""
import ctypes as C
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
for which in ("c2", "c4"):
    if which == "c2":
        pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
        ordering = cb.ORDER_ND
    else:
        pr = workloads.block_angular_qp(seed=3)
        ordering = cb.ORDER_BEST
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=ordering)
    for _ in range(2):
        assert s.refactor()
    refactor_ms = s.time_refactor_ms(reps)
    assert s.refactor()
    L = cb.lib()
    f = L.cldl_selected_inverse_dev
    f.argtypes = [C.c_void_p, C.c_void_p]
    f.restype = C.c_int
    out = torch.empty(len(rv), dtype=torch.float64, device="cuda")
    stream = torch.cuda.ExternalStream(s.stream_ptr())
    t0 = time.perf_counter()
    assert f(s._h, C.c_void_p(out.data_ptr())) == 0
    stream.synchronize()
    first_ms = (time.perf_counter() - t0) * 1e3
    for _ in range(2):
        assert f(s._h, C.c_void_p(out.data_ptr())) == 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        assert f(s._h, C.c_void_p(out.data_ptr())) == 0
    e1.record(stream)
    e1.synchronize()
    selinv_ms = e0.elapsed_time(e1) / reps
    info = s.linear_solver_info()
    diag_ok = bool(torch.isfinite(out).all().item())
    r = {"n": N, "nnzA": len(rv), "nnzL_stored": info.nnzL_stored, "refactor_ms": refactor_ms,
         "selected_inverse_ms": selinv_ms, "first_call_ms_host": first_ms, "finite": diag_ok}
    res["workloads"][which] = r
    print("%s: n %d, nnzL_stored %d, refactor %.2f ms, selected inversion %.2f ms (%.2fx), first call %.0f ms (host clock)"
          % (which, N, info.nnzL_stored, refactor_ms, selinv_ms, selinv_ms / refactor_ms, first_ms))
    s.close()
    del out
    torch.cuda.empty_cache()
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "selinv_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
