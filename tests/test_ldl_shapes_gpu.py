"""The device LDL^T on the matrices of tests/ldl_shapes.py, whose fronts sit at the shapes where the factor and solve
kernels switch code paths (tests/test_ldl_shapes_cpu.py checks that every such path is in their plans), against an
extended-precision reference.

(a) Solves: the reference x* is a sparse LU solve refined with residuals in np.longdouble.  Asserted: the normwise
backward error |b - K x|_inf / (|K|_inf |x|_inf + |b|_inf) (in longdouble), the forward error |x - x*|_inf / |x*|_inf
over eps cond_1(K), exact inertia and no regularisation; after two value updates as well; two solves bitwise equal.
(b) Regularisation: one wrong-signed diagonal whose pivot lands in a k_factor_leaf1 column, a level-0 k_factor_level
front, an F task, or a D task at pivots 0..3 and ns - 1.  The reference is a dense LDL^T in longdouble in the device's
elimination order with the same rule (D_k s_k < eps: D_k = delta s_k); the regularisation count and inertia must be
the reference's, and the device's x must have a small backward error against K + E, E the diagonal correction the
regularisation applied.  That bound does not depend on the ~1e7 conditioning the delta pivot causes.

Worst values measured on an H100 (SXM, 80 GB, at its default power limit; the host-emulated build gives the same
figures to two digits):
  (a) big_fronts     backward error 1.1e-16, forward error / (eps cond_1) 3.4e-2 (cond_1 1.6e2)
      child_records  backward error 7.0e-17, forward error / (eps cond_1) 2.1e-2 (cond_1 6.3e1)
  (b) backward error against K + E: leaf1 1.7e-22, level 4.1e-20, F 7.0e-19, D 3.7e-22 .. 1.3e-17 (pivot 3)
The thresholds below keep a margin of at least 100x to these."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import clarabel_rs_b200 as cb
import ldl_shapes

pytestmark = pytest.mark.gpu

BWD_TOL = 2e-14       # normwise backward error
FWD_TOL = 5.0         # forward error / (eps cond_1(K))
REG_BWD_TOL = 2e-15   # backward error against K + E
EPS = np.finfo(np.float64).eps
LD = np.longdouble


def _csc(sh):
    K = sp.csc_matrix((sh.nz, sh.rv, sh.cp), shape=(sh.N, sh.N))
    return (K + sp.triu(K, 1).T).tocsc()


def _bwd(Kl, x, b):
    """normwise backward error in longdouble (Kl: the dense matrix in longdouble)"""
    xl, bl = x.astype(LD), b.astype(LD)
    r = bl - Kl @ xl
    return float(np.max(np.abs(r)) / (np.max(np.abs(Kl).sum(axis=1)) * np.max(np.abs(xl)) + np.max(np.abs(bl))))


def _reference(lu, Kl, b):
    x = lu.solve(b)
    for _ in range(3):
        x = x + lu.solve(np.asarray(b.astype(LD) - Kl @ x.astype(LD), dtype=np.float64))
    return x


@pytest.fixture(scope="module", params=[f.__name__ for f in (ldl_shapes.big_fronts, ldl_shapes.child_records)])
def shape(request):
    sh = getattr(ldl_shapes, request.param)()
    K = _csc(sh)
    Kd = K.toarray()
    return sh, K, Kd.astype(LD), np.linalg.cond(Kd, 1)


def _rhs(sh, rng):
    N = sh.N
    yield "normal", rng.standard_normal(N)
    yield "1e-6..1e6", rng.choice([-1.0, 1.0], N) * 10.0 ** rng.uniform(-6, 6, N)
    one = np.zeros(N)
    name = max(sh.groups, key=lambda k: len(sh.groups[k]) if k != "sep" else 0)
    one[sh.groups[name]] = rng.standard_normal(len(sh.groups[name]))
    yield "on group " + name, one


def _check(s, sh, K, Kl, cond, rng, worst):
    info = s.linear_solver_info()
    assert info.regularize_count == 0
    assert info.positive_inertia == int((sh.ds > 0).sum())
    lu = spla.splu(K)
    for what, b in _rhs(sh, rng):
        x = s.solve(b)
        xs = _reference(lu, Kl, b)
        be = _bwd(Kl, x, b)
        fe = float(np.max(np.abs(x - xs)) / np.max(np.abs(xs))) / (EPS * cond)
        worst["bwd"], worst["fwd"] = max(worst["bwd"], be), max(worst["fwd"], fe)
        assert be <= BWD_TOL, (sh.name, what, be)
        assert fe <= FWD_TOL, (sh.name, what, fe)
    assert not s.solve(np.zeros(sh.N)).any()


def test_solves_match_the_extended_precision_reference(shape):
    sh, K, Kl, cond = shape
    rng = np.random.default_rng(5)
    worst = {"bwd": 0.0, "fwd": 0.0}
    s = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm)
    assert s.refactor()
    _check(s, sh, K, Kl, cond, rng, worst)
    # new values on off-diagonal entries, no larger in magnitude (the matrix stays diagonally dominant): the
    # refactorisation reuses the arenas at these shapes
    nz = sh.nz.copy()
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    off = np.nonzero(sh.rv != cols)[0]
    for _ in range(2):
        idx = rng.choice(off, size=len(off) // 3, replace=False)
        vals = nz[idx] * rng.uniform(-1.0, 1.0, idx.size)
        s.update_values(idx, vals)
        nz[idx] = vals
        sh2 = ldl_shapes.Shape(sh.name, sh.N, sh.cp, sh.rv, nz, sh.ds, sh.perm, sh.groups)
        K2 = _csc(sh2)
        Kd2 = K2.toarray()
        assert s.refactor()
        _check(s, sh2, K2, Kd2.astype(LD), np.linalg.cond(Kd2, 1), rng, worst)
    b = rng.standard_normal(sh.N)
    assert np.array_equal(s.solve(b), s.solve(b))
    print("%s: worst backward error %.2e, forward error / (eps cond) %.2e (cond_1 %.1e)"
          % (sh.name, worst["bwd"], worst["fwd"], cond))


def _ldl_reference(Kp, sp_, eps=1e-13, delta=2e-7):
    """dense LDL^T in longdouble with the device's pivot rule; returns D before and after regularisation"""
    A = Kp.astype(LD).copy()
    n = A.shape[0]
    d0, d = np.zeros(n, LD), np.zeros(n, LD)
    for k in range(n):
        d0[k] = d[k] = A[k, k]
        if d[k] * sp_[k] < eps:
            d[k] = delta * sp_[k]
        l = A[k + 1:, k] / d[k]
        A[k + 1:, k + 1:] -= np.outer(l, A[k, k + 1:])
    return d0, d


def _site(sh, s, v):
    """(kind, pivot index in its front) of the pivot of vertex v on the device"""
    S = cb.SymbolicAnalysis(sh.N, sh.cp, sh.rv, perm=sh.perm)
    assert np.array_equal(S.perm, s.perm())
    k = int(np.nonzero(S.perm == v)[0][0])
    f = int(np.searchsorted(S.sn_first, k, side="right") - 1)
    ns, nr = int(S.sn_first[f + 1] - S.sn_first[f]), int(S.sn_rowptr[f + 1] - S.sn_rowptr[f])
    lvl = int(S.sn_level[f])
    big = nr >= 96 and ns <= 64
    kind = "D" if big else ("leaf1" if ns == 1 else "level") if lvl == 0 else "F"
    return kind, k - int(S.sn_first[f]), ns


@pytest.mark.parametrize("group,j", ldl_shapes.REG_SITES)
def test_regularised_pivot_at_a_chosen_position(group, j):
    sh = ldl_shapes.regularised(group, j)
    v = int(sh.groups["flip0"][0])
    s = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm)
    assert s.refactor()
    kind, jj, ns = _site(sh, s, v)
    assert kind == group and jj == j, (kind, jj)
    if group == "D":
        assert j < 4 or j == ns - 1
    p = s.perm()
    Kd = sh.dense()
    d0, d = _ldl_reference(Kd[np.ix_(p, p)], sh.ds[p].astype(LD))
    info = s.linear_solver_info()
    assert info.regularize_count == int((d != d0).sum()) >= 1
    assert info.positive_inertia == int((d > 0).sum())
    E = np.zeros(sh.N, LD)
    E[p] = d - d0
    KE = Kd.astype(LD) + np.diag(E)
    rng = np.random.default_rng(9)
    worst = 0.0
    for b in (rng.standard_normal(sh.N), rng.choice([-1.0, 1.0], sh.N) * 10.0 ** rng.uniform(-6, 6, sh.N)):
        be = _bwd(KE, s.solve(b), b)
        worst = max(worst, be)
        assert be <= REG_BWD_TOL, be
    print("reg %s %d: regularised %d, backward error against K + E %.2e" % (group, j, info.regularize_count, worst))
