"""Device time of the factor's parts (cldl_solve_part_dev, cldl_mul_part_dev, cldl_get_factor_csc_dev,
cldl_sample_dev) next to one full solve (cldl_solve_dev), on the KKT matrices of the benchmark's C2 and C4 workloads
built as scripts/updown_time.py builds them.  Every partial solve, the products with L and L^T, one export of L in
compressed-column form (with D and 1/D) and one two-column sample of each form.  The KKT matrices are quasidefinite,
so the sampler (which refuses negative pivots) runs on a positive definite matrix with the same pattern: the KKT
values with every diagonal replaced by |K_ii| + the magnitudes of row i's off-diagonals.  Each case: 2 warm-up calls,
then 10 calls between CUDA events on the handle's stream.  The card's name and power limit are read in the same run.
Usage: python scripts/factor_parts_time.py [out_dir]"""
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


def dominant(N, cp, rv, nz):
    """the same pattern, positive definite: every diagonal |K_ii| + sum of |off-diagonals| of row i"""
    cols = np.repeat(np.arange(N), np.diff(cp))
    off = rv != cols
    rs = np.zeros(N)
    np.add.at(rs, rv[off], np.abs(nz[off]))
    np.add.at(rs, cols[off], np.abs(nz[off]))
    return np.where(off, nz, np.abs(nz) + rs[rv])


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
    b = torch.from_numpy(np.random.default_rng(0).standard_normal(N)).cuda()
    x = torch.empty_like(b)
    torch.cuda.synchronize()
    full = timed(stream, lambda: s.solve_dev(x.data_ptr(), b.data_ptr()))
    w = {"n": N, "fronts": info.n_supernodes, "nnzL_stored": info.nnzL_stored, "solve_ms": full, "cases": {}}
    print("%s: n %d, %d fronts, one full solve %.3f ms" % (which, N, info.n_supernodes, full))

    def case(label, fn):
        ms = timed(stream, fn)
        w["cases"][label] = {"ms": ms, "vs_solve": ms / full}
        print("  %-28s %8.3f ms (%.2fx solve)" % (label, ms, ms / full))

    for sys_ in ("LDLt", "LD", "DLt", "L", "Lt", "D", "P", "Pt", "Dhalf"):
        case("solve_part " + sys_, lambda: s.solve_part_dev(sys_, x.data_ptr(), b.data_ptr()))
    for sys_ in ("L", "Lt", "LDLt", "A"):
        case("mul_part " + sys_, lambda: s.mul_part_dev(sys_, x.data_ptr(), b.data_ptr()))
    nnz = s.factor_csc_nnz()
    dcp = torch.empty(N + 1, dtype=torch.int64, device="cuda")
    dri = torch.empty(nnz, dtype=torch.int64, device="cuda")
    dlx = torch.empty(nnz, dtype=torch.float64, device="cuda")
    dD, dDi = torch.empty_like(b), torch.empty_like(b)
    torch.cuda.synchronize()
    case("factor_csc (%d entries)" % nnz,
         lambda: s.factor_csc_dev(dcp.data_ptr(), dri.data_ptr(), dlx.data_ptr(), dD.data_ptr(), dDi.data_ptr()))
    del dri, dlx
    s.close()
    torch.cuda.empty_cache()
    t = cb.CudaLDLSolver(N, cp, rv, dominant(N, cp, rv, nz), np.ones(N, np.int8), ordering=ordering)
    assert t.refactor()
    stream = torch.cuda.ExternalStream(t.stream_ptr())
    X = torch.empty((2, N), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    w["spd_solve_ms"] = timed(stream, lambda: t.solve_dev(x.data_ptr(), b.data_ptr()))
    print("  %-28s %8.3f ms" % ("full solve (SPD values)", w["spd_solve_ms"]))
    for form in ("precision", "covariance"):
        case("sample 2 columns, " + form, lambda: t.sample_dev(2, 1, 0, None, X.data_ptr(), None, form=form))
    res["workloads"][which] = w
    t.close()
    torch.cuda.empty_cache()
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "factor_parts_time.json"), "w") as fp:
        json.dump(res, fp, indent=1)
