"""The factor's parts (CudaLDLSolver.solve_part / mul_part / factor_csc / sample and their _dev forms; cldl_solve_part,
cldl_mul_part, cldl_get_factor_csc, cldl_sample).

Matrices: the shape matrices of tests/ldl_shapes.py (every front shape the kernels dispatch on: wide and narrow pivot
blocks, level-0 leaf kinds, the separator chain), a regularised one, a helpers.small_kkt, a Laplacian with null pivots
and one C2-sized KKT matrix.
- Export: L and D against the CPU oracle's QDLDL on the same permutation (simplicial pattern, FACTOR_TOL), L21 and
  narrow pivot blocks bitwise against the decoded cldl_get_factor panels, P (K + E) P^T = L D L^T.
- Partial solves and products against dense numpy on the exported (L, D, P); the compositions that are the solve's own
  launches bitwise; op (op^-1 v) = v; P, P^T, D and |D|^-1/2 bitwise; after an update like a fresh refactor.
- Sampling: the Philox restatement against numpy.random.Philox, Z against its Box-Muller restatement, X against the
  dense formula on the returned Z, the offset and pairing identities bitwise, the sample covariance of 2e4 draws, and a
  quasidefinite matrix refused.
- Refusals, repeatability, the _dev forms, and cldl_solve and the factor unchanged by every call."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import scipy.linalg as sla
import scipy.sparse as sp

import clarabel_rs_b200 as cb
import ldl_shapes
import oracle
from helpers import small_kkt

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
FACTOR_TOL = 1e-10      # exported L and D against the oracle's, relative to max(1, |entry|)
SOLVE_TOL = 1e-9        # partial solves and products against dense numpy, relative to max(1, ||reference||_inf)
SYS = ["A", "LDLt", "LD", "DLt", "L", "Lt", "D", "Dhalf", "P", "Pt"]
EMU = os.environ.get("CLARABEL_EMU") == "1"


# ---- matrices ----
class Case:
    def __init__(self, name, N, cp, rv, nz, ds, perm=None, null_tol=0.0):
        self.name, self.N, self.cp, self.rv, self.nz, self.ds, self.perm, self.null_tol = name, N, cp, rv, nz, ds, perm, null_tol

    def solver(self, nz=None):
        return cb.CudaLDLSolver(self.N, self.cp, self.rv, self.nz if nz is None else nz, self.ds, perm=self.perm,
                                null_pivot_tol=self.null_tol)

    def dense(self, nz=None):
        K = sp.csc_matrix((self.nz if nz is None else nz, self.rv, self.cp), shape=(self.N, self.N)).toarray()
        return K + np.triu(K, 1).T


def _laplacian_with_nulls():
    """a path graph's Laplacian in three components, plus 1e-1 on every other diagonal of the first: 2 null pivots"""
    n, comps = 90, [(0, 30), (30, 60), (60, 90)]
    K = np.zeros((n, n))
    for a, b in comps:
        for i in range(a, b - 1):
            K[i, i] += 1.0; K[i + 1, i + 1] += 1.0; K[i, i + 1] -= 1.0; K[i + 1, i] -= 1.0
    K[np.arange(0, 30, 2), np.arange(0, 30, 2)] += 0.1
    U = sp.csc_matrix(np.triu(K))
    U.sort_indices()
    return Case("laplacian_nulls", n, U.indptr, U.indices, U.data, np.ones(n, np.int8), null_tol=1e-9)


def _spd(sh):
    """the shape with every diagonal positive: still strictly diagonally dominant, so positive definite"""
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    nz = np.where(sh.rv == cols, np.abs(sh.nz), sh.nz)
    return Case(sh.name + "_spd", sh.N, sh.cp, sh.rv, nz, np.ones(sh.N, np.int8), sh.perm)


def _cases():
    out = [Case(sh.name, sh.N, sh.cp, sh.rv, sh.nz, sh.ds, sh.perm) for sh in ldl_shapes.all_shapes()]
    out += [_spd(sh) for sh in ldl_shapes.all_shapes()]
    sh = ldl_shapes.regularised("D", 1)
    out.append(Case(sh.name, sh.N, sh.cp, sh.rv, sh.nz, sh.ds, sh.perm))
    out.append(Case("small_kkt", *small_kkt(300, 500, seed=4, window=30, k=4)))
    out.append(_laplacian_with_nulls())
    return out


CASES = {c.name: c for c in _cases()}


def c2_case():
    from helpers import workloads
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    return Case("c2", N, cp, rv, nz, ds)


# ---- helpers ----
def _raw_factor(s):
    info = s.linear_solver_info()
    L, D, Dinv = np.empty(info.nnzL_stored), np.empty(s.n), np.empty(s.n)
    f = cb.lib().cldl_get_factor
    f.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * 3
    f.restype = C.c_int
    assert f(s._h, *(a.ctypes.data_as(C.POINTER(C.c_double)) for a in (L, D, Dinv))) == 0
    return L, D, Dinv


def _digest(s):
    return [hashlib.sha256(a.tobytes()).hexdigest() for a in _raw_factor(s)]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _dense_parts(s):
    L, D, Dinv, perm = s.factor_csc()
    Lf = L.toarray() + np.eye(s.n)
    return Lf, D, Dinv, perm


def _refs(Lf, D, Dinv, perm):
    """dense op^-1 and op for every sys, on the exported factor"""
    n = Lf.shape[0]
    lo = lambda v: sla.solve_triangular(Lf, v, lower=True, unit_diagonal=True)
    up = lambda v: sla.solve_triangular(Lf.T, v, lower=False, unit_diagonal=True)
    def pin(v): return v[perm]
    def pout(v):
        x = np.empty(n); x[perm] = v; return x
    inv = {"LDLt": lambda b: up(Dinv * lo(b)), "LD": lambda b: Dinv * lo(b), "DLt": lambda b: up(Dinv * b),
           "L": lo, "Lt": up, "D": lambda b: Dinv * b, "Dhalf": lambda b: np.sqrt(np.abs(Dinv)) * b,
           "P": pin, "Pt": pout, "A": lambda b: pout(up(Dinv * lo(pin(b))))}
    mul = {"LDLt": lambda x: Lf @ (D * (Lf.T @ x)), "LD": lambda x: Lf @ (D * x), "DLt": lambda x: D * (Lf.T @ x),
           "L": lambda x: Lf @ x, "Lt": lambda x: Lf.T @ x, "D": lambda x: D * x,
           "Dhalf": lambda x: np.sqrt(np.abs(D)) * x, "P": pin, "Pt": pout,
           "A": lambda x: pout(Lf @ (D * (Lf.T @ pin(x))))}
    return inv, mul


def _close(x, ref, tol=SOLVE_TOL):
    return np.max(np.abs(x - ref)) <= tol * max(1.0, np.max(np.abs(ref)))


# ---- export ----
@pytest.mark.parametrize("name", list(CASES))
def test_export_against_the_oracle_and_the_panels(name):
    c = CASES[name]
    s = c.solver()
    assert s.refactor()
    L, D, Dinv, perm = s.factor_csc()
    n = c.N
    # layout: strictly lower, rows ascending, nnz = sum ns (ns - 1) / 2 + ns nr
    sym = cb.SymbolicAnalysis(n, c.cp, c.rv, perm=c.perm) if c.perm is not None else cb.SymbolicAnalysis(n, c.cp, c.rv)
    assert np.array_equal(sym.perm, perm)
    ns = np.diff(sym.sn_first)
    nr = np.diff(sym.sn_rowptr)
    assert L.nnz == s.factor_csc_nnz() == int(np.sum(ns * (ns - 1) // 2 + ns * nr))
    for j in range(n):
        r = L.indices[L.indptr[j]:L.indptr[j + 1]]
        assert np.all(r > j) and np.all(np.diff(r) > 0)
    # D and 1/D as stored; L21 and narrow pivot blocks bitwise from the panels, wide blocks within rounding
    P, D0, Dinv0 = _raw_factor(s)
    assert np.array_equal(_bits(D), _bits(D0)) and np.array_equal(_bits(Dinv), _bits(Dinv0))
    pos = 0
    for k in range(sym.nsup):
        f, a, b = int(sym.sn_first[k]), int(ns[k]), int(nr[k])
        panel = P[pos:pos + (a + b) * a].reshape(a, a + b).T      # column-major (ns + nr) x ns
        pos += (a + b) * a
        for j in range(a):
            col = L.data[L.indptr[f + j]:L.indptr[f + j + 1]]
            assert np.array_equal(_bits(col[a - 1 - j:]), _bits(panel[a:, j]))
            if a <= 8:
                assert np.array_equal(_bits(col[:a - 1 - j]), _bits(panel[j + 1:a, j]))
    # the oracle on the same permutation: simplicial pattern at FACTOR_TOL, the rest of the stored pattern ~ 0
    if c.null_tol == 0.0:
        f = oracle.QDLDL((n, n), c.cp, c.rv, c.nz, perm, dsigns=c.ds, regularize_eps=1e-13, regularize_delta=2e-7)
        Lo = sp.csc_matrix((f.Lx, f.Li, f.Lp), shape=(n, n)).toarray()
        Ld = L.toarray()
        assert np.max(np.abs(Ld - Lo) / np.maximum(1.0, np.abs(Lo))) <= FACTOR_TOL
        assert np.max(np.abs(D - f.D) / np.maximum(1.0, np.abs(f.D))) <= FACTOR_TOL
    # P (K + E) P^T = L D L^T, E the regularisation (at most a few pivots, nonzero only on the diagonal)
    Lf = L.toarray() + np.eye(n)
    K = c.dense()[np.ix_(perm, perm)]
    R = Lf @ np.diag(D) @ Lf.T - K
    np.fill_diagonal(R, np.where(np.abs(np.diag(R)) > 1e-3, 0.0, np.diag(R)))     # the regularised pivots
    assert np.max(np.abs(R)) <= 1e-12 * max(1.0, np.max(np.abs(K)))
    s.close()


# ---- partial solves and products ----
@pytest.mark.parametrize("name", list(CASES))
def test_partial_solves_and_products(name):
    c = CASES[name]
    s = c.solver()
    assert s.refactor()
    want = _digest(s)
    rng = np.random.default_rng(7)
    b = rng.standard_normal(c.N)
    B = rng.standard_normal((c.N, 3))
    x_full = s.solve(b)
    inv, mul = _refs(*_dense_parts(s))
    nulls = c.null_tol > 0.0
    for sys in SYS:
        if nulls and sys in ("A", "LDLt", "LD", "DLt"):
            continue      # a singular system: the generalised inverse, checked through the compositions below
        x = s.solve_part(sys, b)
        assert _close(x, inv[sys](b)), sys
        y = s.mul_part(sys, b)
        assert _close(y, mul[sys](b)), sys
        X = s.solve_part(sys, B)
        for j in range(3):
            assert np.array_equal(_bits(X[:, j]), _bits(s.solve_part(sys, B[:, j]))), sys
        if sys not in ("P", "Pt") and (sys not in ("D", "Dhalf") or not nulls):
            assert _close(s.mul_part(sys, s.solve_part(sys, b)), b, 1e-8), sys
    # the exact ones
    perm = s.perm()
    Lf, D, Dinv, _ = _dense_parts(s)
    assert np.array_equal(_bits(s.solve_part("P", b)), _bits(b[perm]))
    xt = np.empty(c.N); xt[perm] = b
    assert np.array_equal(_bits(s.solve_part("Pt", b)), _bits(xt))
    assert np.array_equal(_bits(s.mul_part("P", b)), _bits(b[perm]))
    assert np.array_equal(_bits(s.mul_part("Pt", b)), _bits(xt))
    assert np.array_equal(_bits(s.mul_part("Pt", s.solve_part("P", b))), _bits(b))     # P and P^T as in CHOLMOD: x = P b
    assert np.array_equal(_bits(s.solve_part("D", b)), _bits(Dinv * b))
    assert np.array_equal(_bits(s.mul_part("D", b)), _bits(D * b))
    assert np.array_equal(_bits(s.solve_part("Dhalf", b)), _bits(np.sqrt(np.abs(Dinv)) * b))
    assert np.array_equal(_bits(s.mul_part("Dhalf", b)), _bits(np.sqrt(np.abs(D)) * b))
    # the solve's own launches, bit for bit
    pb = b[perm]
    assert np.array_equal(_bits(s.solve_part("A", b)), _bits(x_full))
    assert np.array_equal(_bits(s.solve_part("LDLt", pb)), _bits(x_full[perm]))
    assert np.array_equal(_bits(s.solve_part("DLt", s.solve_part("L", pb))), _bits(x_full[perm]))
    # L D then L^T: 1/D applied apart from the backward sweep's subtraction, so equal at rounding level
    assert _close(s.solve_part("Lt", s.solve_part("LD", pb)), x_full[perm])
    # nothing changed
    assert _digest(s) == want
    assert np.array_equal(_bits(s.solve(b)), _bits(x_full))
    s.close()


def test_after_an_update_like_a_fresh_refactor():
    sh = ldl_shapes.big_fronts()
    c = CASES["big_fronts_spd"]
    s = c.solver()
    assert s.refactor()
    cols = np.repeat(np.arange(c.N), np.diff(c.cp))
    v = int(sh.groups["sep"][5])
    w = np.zeros(c.N); w[v] = 1.5
    assert s.updown(w, 2.0)
    nz = c.nz.copy()
    nz[np.flatnonzero((c.rv == v) & (cols == v))] += 2.0 * 1.5 * 1.5
    t = c.solver(nz)
    assert t.refactor()
    b = np.random.default_rng(3).standard_normal(c.N)
    for sys in SYS:
        assert _close(s.solve_part(sys, b), t.solve_part(sys, b), 1e-10), sys
        assert _close(s.mul_part(sys, b), t.mul_part(sys, b), 1e-10), sys
    Ls, Ds, _, _ = s.factor_csc()
    Lt, Dt, _, _ = t.factor_csc()
    assert np.max(np.abs((Ls - Lt).toarray())) <= 1e-10 and np.max(np.abs(Ds - Dt)) <= 1e-10 * np.max(np.abs(Dt))
    assert _close(s.sample(2, seed=1), t.sample(2, seed=1), 1e-10)
    s.close()
    t.close()


# ---- sampling ----
M0, M1 = 0xD2E7470EE14C6C93, 0xCA5A826395121157
W0, W1 = 0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B
MASK = (1 << 64) - 1


def philox4x64(ctr, key):
    """Philox4x64-10 (Salmon et al., SC 2011), restated"""
    c, k0, k1 = list(ctr), key[0], key[1]
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> 64) ^ c[1] ^ k0, p1 & MASK, (p0 >> 64) ^ c[3] ^ k1, p0 & MASK]
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return c


def normals(n, seed, col):
    """the sampler's standard normals of stream position col, restated (Box-Muller on (1 - u0, u1), (1 - u2, u3))"""
    z = np.empty(4 * ((n + 3) // 4))
    for j in range(len(z) // 4):
        r = philox4x64([j, col, 0, 0], [seed, 0])
        u = [(w >> 11) * 2.0 ** -53 for w in r]
        for p in range(2):
            rad = np.sqrt(-2.0 * np.log(1.0 - u[2 * p]))
            z[4 * j + 2 * p] = rad * np.cos(2.0 * np.pi * u[2 * p + 1])
            z[4 * j + 2 * p + 1] = rad * np.sin(2.0 * np.pi * u[2 * p + 1])
    return z[:n]


def test_philox_restatement_matches_numpy():
    for seed, ctr in [(0, [1, 0, 0, 0]), (12345, [7, 3, 0, 0]), (2 ** 63 + 5, [2 ** 40, 2 ** 33 + 1, 0, 0])]:
        bg = np.random.Philox(counter=np.array([ctr[0] - 1, ctr[1], 0, 0], np.uint64),      # numpy counts up first
                               key=np.array([seed, 0], np.uint64))
        assert list(int(v) for v in bg.random_raw(4)) == philox4x64(ctr, [seed, 0])


def _spd50():
    n = 50
    rng = np.random.default_rng(5)
    K = np.diag(np.full(n, 3.0))
    for i in range(n - 1):
        K[i, i + 1] = K[i + 1, i] = -1.0
    for _ in range(30):
        i, j = sorted(rng.choice(n, 2, replace=False))
        K[i, j] = K[j, i] = 0.3 * rng.uniform(-1, 1)
    U = sp.csc_matrix(np.triu(K))
    U.sort_indices()
    return Case("spd50", n, U.indptr, U.indices, U.data, np.ones(n, np.int8)), K


@pytest.mark.parametrize("name", ["big_fronts_spd", "child_records_spd", "laplacian_nulls"])
def test_draws_against_the_formula_and_their_normals(name):
    c = CASES[name]
    s = c.solver()
    assert s.refactor()
    Lf, D, Dinv, perm = _dense_parts(s)
    mu = np.random.default_rng(1).standard_normal(c.N)
    for form in ("precision", "covariance"):
        X, Z = s.sample(3, seed=99, offset=4, mean=mu, form=form, return_z=True)
        for j in range(3):
            zr = normals(c.N, 99, 4 + j)
            assert np.max(np.abs(Z[:, j] - zr) / np.maximum(1.0, np.abs(zr))) <= 16 * EPS
            if form == "precision":
                t = sla.solve_triangular(Lf.T, np.sqrt(np.abs(Dinv)) * Z[:, j], lower=False, unit_diagonal=True)
            else:
                t = Lf @ (np.sqrt(np.abs(D)) * Z[:, j])
            ref = np.empty(c.N); ref[perm] = t
            assert _close(X[:, j], mu + ref), (form, j)
        # offsets and pairing: draw c of a call is draw 0 of a call at offset + c, bit for bit
        X5 = s.sample(5, seed=99, offset=4, mean=mu, form=form)
        assert np.array_equal(_bits(X5[:, :3]), _bits(X))
        for j in range(5):
            assert np.array_equal(_bits(s.sample(1, seed=99, offset=4 + j, mean=mu, form=form)[:, 0]), _bits(X5[:, j]))
        assert np.array_equal(_bits(s.sample(5, seed=99, offset=4, mean=mu, form=form)), _bits(X5))
    s.close()


def test_sample_covariance_of_many_draws():
    c, K = _spd50()
    s = c.solver()
    assert s.refactor()
    N = 20_000
    for form, Sigma in (("precision", np.linalg.inv(K)), ("covariance", K)):
        X = s.sample(N, seed=2024, form=form)
        Sc = X @ X.T / N                          # mean 0 known
        # each entry of the sample covariance has standard deviation sqrt((S_ii S_jj + S_ij^2) / N)
        sd = np.sqrt((np.outer(np.diag(Sigma), np.diag(Sigma)) + Sigma ** 2) / N)
        assert np.max(np.abs(Sc - Sigma) / sd) <= 5.0, form
    s.close()


def test_quasidefinite_matrix_is_refused():
    c = CASES["small_kkt"]
    s = c.solver()
    assert s.refactor()
    for form in ("precision", "covariance"):
        with pytest.raises(cb.BackendError, match="BadArgument"):
            s.sample(1, form=form)
    s.close()


# ---- refusals, repeatability, device pointers ----
def test_refusals():
    c = CASES["big_fronts"]
    s = c.solver()
    b = np.ones(c.N)
    for call in (lambda: s.solve_part("L", b), lambda: s.mul_part("Lt", b), lambda: s.factor_csc(),
                 lambda: s.sample(1)):
        with pytest.raises(cb.BackendError, match="NotFactored"):
            call()
    assert s.refactor()
    lib = cb.lib()
    bb, xx = np.ones(c.N), np.empty(c.N)
    pd = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    for fn in (lib.cldl_solve_part, lib.cldl_mul_part):
        fn.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        fn.restype = C.c_int
        for bad in (-1, 10):
            assert fn(s._h, bad, pd(xx), pd(bb)) == -21
    fs = lib.cldl_sample
    fs.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64] + [C.POINTER(C.c_double)] * 3
    fs.restype = C.c_int
    X = np.empty(c.N)
    assert fs(s._h, 2, 1, 0, 0, None, pd(X), None) == -21
    assert fs(s._h, 0, 1, 0, 0, None, None, None) == -21
    with pytest.raises(cb.BackendError):
        s.solve_part("X", b)
    # an update whose verdict is 0 leaves the factor invalid
    v = int(ldl_shapes.big_fronts().groups["sep"][0])
    w = np.zeros(c.N); w[v] = 1.0
    assert not s.updown(w, -1e6 * float(c.ds[v]))      # the pivot's sign flips: verdict 0
    for call in (lambda: s.solve_part("L", b), lambda: s.mul_part("L", b), lambda: s.factor_csc(),
                 lambda: s.sample(1)):
        with pytest.raises(cb.BackendError, match="NotFactored"):
            call()
    s.close()
    sh = ldl_shapes.big_fronts()
    sc = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, schur=[int(sh.groups["sep"][-1])])
    assert sc.refactor()
    for call in (lambda: sc.solve_part("L", b), lambda: sc.mul_part("L", b), lambda: sc.factor_csc(),
                 lambda: sc.sample(1)):
        with pytest.raises(cb.BackendError, match="BadArgument"):
            call()
    sc.close()


def test_repeatable_and_leaves_the_factor_and_solves_unchanged():
    c = CASES["child_records_spd"]
    s = c.solver()
    assert s.refactor()
    want = _digest(s)
    b = np.random.default_rng(11).standard_normal(c.N)
    x0 = s.solve(b)
    first = [s.solve_part(sys, b) for sys in SYS] + [s.mul_part(sys, b) for sys in SYS] + \
            [s.factor_csc()[0].data, s.sample(3, seed=5), s.sample(3, seed=5, form="covariance")]
    again = [s.solve_part(sys, b) for sys in SYS] + [s.mul_part(sys, b) for sys in SYS] + \
            [s.factor_csc()[0].data, s.sample(3, seed=5), s.sample(3, seed=5, form="covariance")]
    for a, b2 in zip(first, again):
        assert np.array_equal(_bits(a), _bits(b2))
    assert _digest(s) == want
    assert np.array_equal(_bits(s.solve(b)), _bits(x0))
    s.close()


def test_device_pointer_forms():
    import torch
    dev = torch.device("cpu") if EMU else torch.device("cuda", 0)
    c = CASES["big_fronts_spd"]
    s = c.solver()
    assert s.refactor()
    n = c.N
    b = np.random.default_rng(2).standard_normal(n)
    db = torch.from_numpy(b).to(dev)
    dx = torch.empty(n, dtype=torch.float64, device=dev)
    sync = (lambda: torch.cuda.synchronize()) if dev.type == "cuda" else (lambda: None)
    sync()
    for sys in SYS:
        s.solve_part_dev(sys, dx.data_ptr(), db.data_ptr())
        s.sync_status()
        assert np.array_equal(_bits(dx.cpu().numpy()), _bits(s.solve_part(sys, b))), sys
        s.mul_part_dev(sys, dx.data_ptr(), db.data_ptr())
        s.sync_status()
        assert np.array_equal(_bits(dx.cpu().numpy()), _bits(s.mul_part(sys, b))), sys
    L, D, Dinv, _ = s.factor_csc()
    nnz = s.factor_csc_nnz()
    dcp = torch.empty(n + 1, dtype=torch.int64, device=dev)
    dri = torch.empty(nnz, dtype=torch.int64, device=dev)
    dlx = torch.empty(nnz, dtype=torch.float64, device=dev)
    dD, dDi = torch.empty(n, dtype=torch.float64, device=dev), torch.empty(n, dtype=torch.float64, device=dev)
    s.factor_csc_dev(dcp.data_ptr(), dri.data_ptr(), dlx.data_ptr(), dD.data_ptr(), dDi.data_ptr())
    s.sync_status()
    assert np.array_equal(dcp.cpu().numpy(), L.indptr) and np.array_equal(dri.cpu().numpy(), L.indices)
    assert np.array_equal(_bits(dlx.cpu().numpy()), _bits(L.data))
    assert np.array_equal(_bits(dD.cpu().numpy()), _bits(D)) and np.array_equal(_bits(dDi.cpu().numpy()), _bits(Dinv))
    mu = np.random.default_rng(4).standard_normal(n)
    dmu = torch.from_numpy(mu).to(dev)
    for form in ("precision", "covariance"):
        dX = torch.empty((3, n), dtype=torch.float64, device=dev)
        dZ = torch.empty((3, n), dtype=torch.float64, device=dev)
        s.sample_dev(3, 8, 1, dmu.data_ptr(), dX.data_ptr(), dZ.data_ptr(), form=form)
        s.sync_status()
        X, Z = s.sample(3, seed=8, offset=1, mean=mu, form=form, return_z=True)
        assert np.array_equal(_bits(dX.cpu().numpy().T), _bits(X)) and np.array_equal(_bits(dZ.cpu().numpy().T), _bits(Z))
    s.close()


def test_autograd_sample_passes_gradient_to_the_mean_only():
    import torch
    from clarabel_rs_b200_pkg.autograd import SparseLDL
    c, K = _spd50()
    layer = SparseLDL(c.N, c.cp, c.rv, c.ds)
    v = torch.from_numpy(np.asarray(c.nz, dtype=np.float64)).to(layer.device)
    mu = torch.zeros(c.N, dtype=torch.float64, device=layer.device, requires_grad=True)
    X = layer.sample(v, 4, seed=3, mean=mu)
    ref = layer.solver.sample(4, seed=3)
    assert np.array_equal(_bits(X.detach().cpu().numpy()), _bits(ref + 0.0))
    X.sum().backward()
    assert np.array_equal(mu.grad.cpu().numpy(), np.full(c.N, 4.0))
    with pytest.raises(RuntimeError):
        layer.sample(v.clone().requires_grad_(True), 1, seed=0)
    layer.close()


def test_c2_sized_kkt():
    c = c2_case()
    s = c.solver()
    assert s.refactor()
    want = _digest(s)
    n = c.N
    b = np.random.default_rng(0).standard_normal(n)
    x = s.solve(b)
    perm = s.perm()
    assert np.array_equal(_bits(s.solve_part("LDLt", b[perm])), _bits(x[perm]))
    assert np.array_equal(_bits(s.solve_part("DLt", s.solve_part("L", b[perm]))), _bits(x[perm]))
    for sys in ("L", "Lt", "LD", "DLt", "LDLt"):
        assert _close(s.mul_part(sys, s.solve_part(sys, b)), b, 1e-7), sys
    # K x = b through the product with the factor
    Kx = s.mul_part("A", x)
    assert np.max(np.abs(Kx - b)) <= 1e-8 * max(1.0, np.max(np.abs(b)))
    L, D, Dinv, _ = s.factor_csc()
    assert L.nnz == s.factor_csc_nnz()
    # L D L^T x through the exported factor equals the product with the factor
    xp = np.random.default_rng(1).standard_normal(n)
    Lf = L + sp.identity(n, format="csc")
    assert _close(Lf @ (D * (Lf.T @ xp)), s.mul_part("LDLt", xp), 1e-10)
    assert _digest(s) == want
    s.close()
