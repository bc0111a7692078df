"""Task timeline of the dataflow triangular solves (k_solve2, ldl_solve.cuh) on the KKT matrix of a workload.
Usage (on the GPU): python scripts/df_trace_solve.py c2|c4"""
import os, sys, struct
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("CB_DF_TRACE_SOLVE", "/tmp/df_trace_solve.bin")
import clarabel_rs_b200 as cb
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from helpers import workloads

which = sys.argv[1] if len(sys.argv) > 1 else "c2"
if which == "c2":
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
else:
    pr = workloads.block_angular_qp(seed=3)
N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=cb.ORDER_ND)
assert s.refactor()
b = np.random.default_rng(1).standard_normal(N)
for _ in range(3):
    x = s.solve(b)
print("solve_ms", s.time_solve_ms(10), "refactor_ms", s.time_refactor_ms(5))
x = s.solve(b)
raw = open(os.environ["CB_DF_TRACE_SOLVE"], "rb").read()
nt = struct.unpack("q", raw[:8])[0]
rec = np.frombuffer(raw, dtype=np.int32, count=24 * nt, offset=8).reshape(nt, 24)
kind, front, ns, nr, r0, r1, nrt = rec[:, 0], rec[:, 1], rec[:, 4], rec[:, 5], rec[:, 6], rec[:, 7], rec[:, 15]
tr = np.frombuffer(raw, dtype=np.uint64, count=8 * nt, offset=8 + 96 * nt).reshape(2, nt, 4).astype(np.int64)
names = {0: "narrow x8", 1: "head", 2: "rows"}
for di, name in ((0, "forward"), (1, "backward")):
    t = tr[di]
    t0 = t[:, 0].min()
    grab, ready, end = [(t[:, i] - t0) / 1e3 for i in (0, 1, 2)]
    landed = (t[:, 3] - t0) / 1e3
    rd = np.where(t[:, 1] > 0, ready, grab)
    print(f"== {name}: span {end.max():.1f} us, tasks {nt}")
    for k in (0, 1, 2):
        q = kind == k
        if not q.any():
            continue
        ent = (np.where(k == 1, ns[q], 0) + (r1[q] - r0[q])) * ns[q] if k else np.zeros(q.sum())
        print(f"  {names[k]:9s} n={q.sum():6d} busy sum {np.sum(end[q]-rd[q])/1e3:8.2f} ms mean {np.mean(end[q]-rd[q]):6.2f} us | wait mean {np.mean(rd[q]-grab[q]):6.2f} us | slab mean {ent.mean():7.0f} doubles")
    if (kind == 1).any():
        q = kind == 1
        for lo, hi in ((0, 2048), (2048, 4096), (4096, 6144), (6144, 1 << 30)):
            ent = (ns + r1 - r0) * ns
            qq = q & (ent >= lo) & (ent < hi)
            if qq.any():
                extra = f" | slab landed {np.mean(landed[qq]-rd[qq]):6.2f} us after ready" if di == 0 else ""
                print(f"     head slabs {lo:5d}-{hi if hi < 1 << 29 else 99999:5d}: n={qq.sum():6d} busy mean {np.mean(end[qq]-rd[qq]):6.2f} us wait mean {np.mean(rd[qq]-grab[qq]):6.2f} us{extra}")
    nb = 20
    edges = np.linspace(0, end.max(), nb + 1)
    print("  slice(us) busyCTAs waitingCTAs")
    for i in range(nb):
        lo, hi = edges[i], edges[i + 1]
        bz = np.clip(np.minimum(end, hi) - np.maximum(rd, lo), 0, None).sum() / (hi - lo)
        wt = np.clip(np.minimum(rd, hi) - np.maximum(grab, lo), 0, None).sum() / (hi - lo)
        print(f"  {lo:8.0f} {bz:8.1f} {wt:8.1f}")
    order = np.argsort(end)[-30:]
    print("  last tasks to finish: front kind ns nr rows | grab ready end busy")
    for i in order:
        print(f"  {front[i]:7d} {names[kind[i]]:9s} ns={ns[i]:3d} nr={nr[i]:5d} rows={r0[i]:4d}-{r1[i]:4d} | {grab[i]:8.1f} {rd[i]:8.1f} {end[i]:8.1f} {end[i]-rd[i]:6.1f}")
