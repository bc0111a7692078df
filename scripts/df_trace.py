"""Task timeline of the dataflow factorisation (k_factor_df) on a C2-like KKT.

Usage (on the GPU): CB_DF_TRACE=/tmp/t.bin python scripts/df_trace.py 100000 200000 200 [out.txt]
Prints per-task-kind busy/wait totals, SM utilisation over time and the D/R/T stages along the path that
finishes last (the critical chain to the root)."""
import os, sys, struct
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("CB_DF_TRACE", "/tmp/df_trace.bin")
import clarabel_rs_b200 as cb
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from helpers import workloads

n, m = int(sys.argv[1]), int(sys.argv[2])
window = None if sys.argv[3] == "None" else int(sys.argv[3])
pr = workloads.random_sparse_qp(n=n, m=m, nnz_per_row=5, seed=1, window=window)
N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, m))
s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=cb.ORDER_ND)
for _ in range(4):
    assert s.refactor()
print("refactor_ms", s.time_refactor_ms(5))
assert s.refactor()
raw = open(os.environ["CB_DF_TRACE"], "rb").read()
nt = struct.unpack("q", raw[:8])[0]
tasks = np.frombuffer(raw, dtype=np.int32, count=16 * nt, offset=8).reshape(nt, 16)
tr = np.frombuffer(raw, dtype=np.uint64, count=10 * nt, offset=8 + 64 * nt).reshape(nt, 10).astype(np.int64)
t0 = tr[:, 0].min()
grab, ready, end, sm = (tr[:, 0] - t0) / 1e3, (tr[:, 1] - t0) / 1e3, (tr[:, 2] - t0) / 1e3, tr[:, 3]
m1, m2 = (tr[:, 4] - t0) / 1e3, (tr[:, 5] - t0) / 1e3
span = end.max()
print(f"tasks {nt}  span {span:.1f} us")
names = "FDRT"
for k in range(4):
    sel = tasks[:, 0] == k
    if not sel.any():
        continue
    busy, wait = (end - ready)[sel], (ready - grab)[sel]
    print(f"{names[k]}: n={sel.sum():7d} busy sum {busy.sum()/1e3:9.2f} ms mean {busy.mean():7.2f} us p50 {np.median(busy):7.2f} max {busy.max():7.2f} | "
          f"wait sum {wait.sum()/1e3:9.2f} ms mean {wait.mean():7.2f} us")
    if k == 1:
        print(f"   D phases: assemble {np.mean((m1-ready)[sel]):6.2f} us, pivots+store {np.mean((end-m1)[sel]):6.2f} us")
    if k == 2:
        print(f"   R phases: assemble {np.mean((m1-ready)[sel]):6.2f} us, wait-diag {np.mean((m2-m1)[sel]):6.2f} us, trsm {np.mean((end-m2)[sel]):6.2f} us")
    if k == 3:
        print(f"   T phases: extend-add {np.mean((m1-ready)[sel]):6.2f} us, gemm {np.mean((m2-m1)[sel]):6.2f} us, store {np.mean((end-m2)[sel]):6.2f} us")
# busy CTAs over time
nb = 40
edges = np.linspace(0, span, nb + 1)
busy_t = np.zeros(nb); wait_t = np.zeros(nb)
for a, b, acc in ((ready, end, busy_t), (grab, ready, wait_t)):
    for i in range(nb):
        lo, hi = edges[i], edges[i + 1]
        acc[i] = np.clip(np.minimum(b, hi) - np.maximum(a, lo), 0, None).sum() / (hi - lo)
print("time-slice(us)  busyCTAs  waitingCTAs")
for i in range(nb):
    print(f"{edges[i]:9.0f} {busy_t[i]:9.1f} {wait_t[i]:9.1f}")
# the chain that ends last: per front D/R/T windows
S = cb.SymbolicAnalysis(N, cp, rv, perm=s.perm())
par = S.sn_parent
front_end = {}
for i in range(nt):
    f = tasks[i, 1]
    front_end[f] = max(front_end.get(f, 0.0), end[i])
kids = {}
for c, p in enumerate(par):
    if p >= 0:
        kids.setdefault(int(p), []).append(c)
root = max(front_end, key=front_end.get)
chain = [root]
while True:
    ks = [c for c in kids.get(chain[-1], []) if c in front_end]
    if not ks:
        break
    chain.append(max(ks, key=lambda c: front_end[c]))
print("critical chain (root first): front ns nr | D ready..end | R first-ready..last-end | T first-ready..last-end")
nsv, nrv = np.diff(S.sn_first), np.diff(S.sn_rowptr)
for f in chain[:60]:
    sel = tasks[:, 1] == f
    out = f"{f:7d} ns={nsv[f]:3d} nr={nrv[f]:4d}"
    for k in (0, 1, 2, 3):
        q = sel & (tasks[:, 0] == k)
        if q.any():
            out += f" | {names[k]} n={q.sum():3d} {ready[q].min():8.1f}..{end[q].max():8.1f} (busy mean {(end-ready)[q].mean():6.1f})"
    print(out)
# T prologue time against the number of child records / sorted entries of the tile
selT = tasks[:, 0] == 3
nch = (tasks[:, 8] - tasks[:, 7])[selT]
nen = (tasks[:, 10] - tasks[:, 9])[selT]
pro = (m1 - ready)[selT]
gem = (m2 - m1)[selT]
print("T prologue by #child records:")
for c in range(0, 8):
    q = nch == c
    if q.any():
        print(f"  children={c}: n={q.sum():6d} prologue {pro[q].mean():6.2f} us  gemm {gem[q].mean():5.2f}  entries mean {nen[q].mean():7.1f}")
q = nch >= 8
if q.any():
    print(f"  children>=8: n={q.sum():6d} prologue {pro[q].mean():6.2f} us entries mean {nen[q].mean():7.1f}")
print("T prologue by #entries (children==1):")
for lo, hi in ((0, 1), (1, 16), (16, 64), (64, 256), (256, 512), (512, 10**9)):
    q = (nch == 1) & (nen >= lo) & (nen < hi)
    if q.any():
        print(f"  entries [{lo},{hi}): n={q.sum():6d} prologue {pro[q].mean():6.2f} us")

x6, x7, x8 = (tr[:, 6] - t0) / 1e3, (tr[:, 7] - t0) / 1e3, (tr[:, 8] - t0) / 1e3
for c in (0, 1, 2):
    q = np.where(selT)[0][nch == c]
    print(f"T children={c}: issue+panel stores {np.mean(x6[q]-ready[q]):5.2f}  zero+sync {np.mean(x7[q]-x6[q]):5.2f}  children {np.mean(x8[q]-x7[q]):5.2f}  entries {np.mean(m1[q]-x8[q]):5.2f}")
