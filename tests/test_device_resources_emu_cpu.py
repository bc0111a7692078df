"""Device resources of the host objects, counted on the emulated full build (tests/emu/libclarabel_emu_full.so, whose
CUDA runtime counts live device allocations, pinned allocations, streams and events and can make any creation fail):

* balance: creating, using and destroying an LDL handle, a Schur handle, a sharded group and an interior-point solver
  leaves every count where it was;
* constructors: whichever allocation of a constructor fails, it raises and leaves nothing behind;
* lazy set-up (selected inverse, log-determinant, adjoint solve, growing staging buffers, solution derivatives):
  whichever allocation of a first call fails, the call raises, and a retry works and returns bitwise what a handle
  that never failed returns.
Not a statement about the GPU: the -m gpu run is."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r'''
import ctypes as C, os, sys
import numpy as np
import scipy.sparse as sp
sys.path.insert(0, ROOT); sys.path.insert(0, ROOT + "/tests")
os.environ["CLARABEL_EMU"] = "1"
import clarabel_rs_b200 as cb
cb.pkg._LIBPATH = ROOT + "/tests/emu/libclarabel_emu_full.so"
from helpers import small_kkt
L = cb.lib()
L.emu_live_resources.argtypes = [C.POINTER(C.c_int64)]
L.emu_fail_alloc_at.argtypes = [C.c_int]

def live():
    a = (C.c_int64 * 4)()
    L.emu_live_resources(a)
    return tuple(a)

def arm(k):
    L.emu_fail_alloc_at(k)

def same(a, b):
    if isinstance(a, tuple):
        return len(a) == len(b) and all(same(u, v) for u, v in zip(a, b))
    if sp.issparse(a):
        return np.array_equal(a.toarray(), b.toarray())
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    return np.array_equal(np.asarray(a), np.asarray(b))

N, cp, rv, nz, ds = small_kkt(60, 90, seed=3, window=12, k=3)
rng = np.random.default_rng(5)
b = rng.standard_normal(N)
g = rng.standard_normal(N)

def ldl(**kw):
    return cb.CudaLDLSolver(N, cp, rv, nz, ds, **kw)

# a problem with every cone type: min 1/2 |x|^2 + q'x  s.t.  x_0 = 1/2, b + x in the other cones
CONES = [("zero", 1), ("nonneg", 3), ("soc", 3), ("psd", 3), ("exp", 3), ("pow", 0.3), ("genpow", ([0.3, 0.7], 2))]
n = 3 + 3 + 6 + 3 + 3 + 4
A = sp.vstack([sp.csc_matrix(([1.0], ([0], [0])), shape=(1, n)), -sp.identity(n)], format="csc")
bq = np.concatenate([[0.5], rng.uniform(0.5, 1.5, n)])
bq[1 + 3:1 + 6] = [2.0, 0.3, 0.2]
P = sp.identity(n, format="csc")
q = rng.standard_normal(n)

def ipm():
    return cb.CudaSolver(P, q, A, bq, CONES)

def ipm_use(s):
    r = s.solve()
    assert r["status"] == "Solved", r["status"]
    s.update_data(q=q * 1.01)
    r = s.solve()
    assert r["status"] == "Solved", r["status"]
    s.derivative(dq=np.ones(n))
    s.adjoint_derivative(dx=np.ones(n))
    s.test_spmv(1, np.zeros(A.shape[0]), np.ones(n), 1.0, 0.0)
    s.test_vec(0, np.ones(7))

start = live()

# ---- balance
s = ldl()
assert s.refactor()
s.solve(b); s.selected_inverse(); s.slogdet(); s.adjoint_solve(g, s.solve(b))
for k in (5, 50, 400):
    idx = np.arange(k) % len(nz)
    s.update_values(idx, np.asarray(nz)[idx])
s.close()
assert live() == start, ("plain", live(), start)
sch = ldl(schur=list(range(N - 6, N)))
assert sch.refactor()
w = sch.schur_reduce(b); sch.schur_expand(np.linalg.solve(sch.schur_complement(), w))
sch.close()
assert live() == start, ("schur", live(), start)
grp = cb.ShardedLDLGroup(N, cp, rv, nz, ds, 3, ordering=cb.ORDER_ND, nd_leaf=10)
assert grp.refactor()
grp.solve(b)
grp.close()
assert live() == start, ("sharded", live(), start)
s = ipm(); ipm_use(s); s.close()
assert live() == start, ("ipm", live(), start)

# ---- constructors: every allocation they make, made to fail in turn
for name, make in [("plain", ldl), ("schur", lambda: ldl(schur=list(range(N - 6, N)))), ("ipm", ipm)]:
    k = 1
    while True:
        arm(k)
        try:
            h = make()
        except cb.BackendError:
            arm(0)
            assert live() == start, (name, k, live(), start)
            k += 1
            continue
        arm(0)
        h.close()
        break
    assert k > 5, (name, k)
    assert live() == start, (name, live(), start)
    print("CTOR %s %d" % (name, k - 1), flush=True)

# ---- lazy set-up: every allocation of a first call made to fail in turn, then a retry
def growing(s):
    idx = np.arange(300) % len(nz)
    s.update_values(idx, np.asarray(nz)[idx] * 1.5)
    assert s.refactor()
    return s.solve(b)

def with_ldl(call):
    def run():
        s = ldl()
        assert s.refactor()
        s.update_values([0], [nz[0]])         # the staging buffers exist, at their first size
        return s, (lambda: call(s))
    return run

def with_ipm(call):
    def run():
        s = ipm()
        assert s.solve()["status"] == "Solved"
        return s, (lambda: call(s))
    return run

CASES = [
    ("selected_inverse", with_ldl(lambda s: s.selected_inverse())),
    ("slogdet", with_ldl(lambda s: s.slogdet())),
    ("adjoint_solve", with_ldl(lambda s: s.adjoint_solve(g, s.solve(b)))),
    ("update_values", with_ldl(growing)),
    ("derivative", with_ipm(lambda s: s.derivative(dq=np.ones(n), db=np.ones(A.shape[0])))),
    ("adjoint_derivative", with_ipm(lambda s: s.adjoint_derivative(dx=np.ones(n), dz=np.ones(A.shape[0])))),
]
for name, setup in CASES:
    h, call = setup()
    want = call()
    h.close()
    k = 1
    while True:                               # until the call makes fewer than k allocations
        h, call = setup()
        arm(k)
        try:
            call()
            failed = False
        except cb.BackendError:
            failed = True
        arm(0)
        if failed:
            got = call()
            assert same(got, want), (name, k)
        h.close()
        assert live() == start, (name, k, live(), start)
        if not failed:
            break
        k += 1
    assert k > 1, name
    print("LAZY %s %d" % (name, k - 1), flush=True)
print("RESOURCES_OK", flush=True)
'''


def test_device_resources_balance_and_failed_allocations(tmp_path):
    lib = os.path.join(ROOT, "tests", "emu", "libclarabel_emu_full.so")
    assert os.path.exists(lib), f"{lib} missing: run `make`"
    script = tmp_path / "resources.py"
    script.write_text("ROOT = %r\n" % ROOT + SCRIPT)
    env = dict(os.environ, CLARABEL_EMU="1", CLARABEL_EMU_FULL="1")
    r = subprocess.run([sys.executable, str(script)], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=1800)
    tail = r.stdout[-4000:]
    assert r.returncode == 0, tail
    assert "RESOURCES_OK" in r.stdout, tail
