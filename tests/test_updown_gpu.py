"""Rank-k updates and downdates of the factor (CudaLDLSolver.updown / updown_dev, cldl_updown(_dev)).

Every front shape: on the matrices of tests/ldl_shapes.py and on the matrices of every site of ldl_shapes.REG_SITES
(factored with regularisation off, so that E = 0 and a fresh refactor is the reference), rank 1, 3, 8, 9 and 17 with
sigma of one sign or mixed, the columns drawn as cliques inside dense groups, single edges and diagonals.  Checked:
the stored values bitwise against the numpy restatement v += (sigma_r * w_i) * w_j; D, 1/D, L and a solve against a
handle refactored on the updated values, at FACTOR_TOL / SOLVE_TOL; a refined solve converging within 2 steps.
With regularisation on (E kept): solves against Sherman-Morrison-Woodbury on the factor before the update.
Also: an update and its downdate returning the factor; effective resistances of a Laplacian after edge-weight
changes; pivots changing sign with regularisation off (inertia, slogdet); a downdate through zero (verdict 0, then a
refactor); the other solve-type calls on the updated factor; the refusals; repeatability and the device-pointer form;
a C2-sized KKT matrix."""
import ctypes as C
import hashlib
import os
import zlib

import numpy as np
import pytest
import scipy.sparse as sp

import clarabel_rs_b200 as cb
import ldl_shapes

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
# measured on the shape matrices (pivots >= 1, condition numbers below 1e3): the updated factor differs from a fresh
# one by a few 1e-15 relative to the largest entry; the bounds leave two orders of magnitude
FACTOR_TOL = 1e-12
SOLVE_TOL = 1e-11
ARG = -21             # CLDL_E_ARG
RANKS = [1, 3, 8, 9, 17]
SIGNS = ["+", "-", "mixed"]
MATRICES = [f.__name__ for f in (ldl_shapes.big_fronts, ldl_shapes.child_records)] + \
    ["reg_%s_%d" % site for site in ldl_shapes.REG_SITES]


def _shape(name):
    if name.startswith("reg_"):
        _, g, j = name.split("_")
        return ldl_shapes.regularised(g, int(j))
    return getattr(ldl_shapes, name)()


def _solver(sh, nz=None, **kw):
    return cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz if nz is None else nz, sh.ds, perm=sh.perm, **kw)


def _device():
    import torch
    return torch.device("cpu") if os.environ.get("CLARABEL_EMU") == "1" else torch.device("cuda", 0)


def _values(s, nnz):
    """the handle's current values (cldl_values_dev), copied out"""
    import torch
    t = torch.empty(nnz, dtype=torch.float64, device=_device())
    L = cb.lib()
    assert L.cldl_copy_dev(C.c_void_p(t.data_ptr()), C.c_void_p(L.cldl_values_dev(s._h)), 8 * nnz) == 0
    return t.cpu().numpy()


def _factor(s):
    info = s.linear_solver_info()
    L, D, Dinv = np.empty(info.nnzL_stored), np.empty(s.n), np.empty(s.n)
    f = cb.lib().cldl_get_factor
    f.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * 3
    f.restype = C.c_int
    rc = f(s._h, *(a.ctypes.data_as(C.POINTER(C.c_double)) for a in (L, D, Dinv)))
    return rc, L, D, Dinv


def _digest(s):
    rc, L, D, Dinv = _factor(s)
    assert rc == 0
    return [hashlib.sha256(a.tobytes()).hexdigest() for a in (L, D, Dinv)]


def _pattern(sh):
    """the stored upper-triangle pairs: (i, j) -> CSC position"""
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    return {(int(i), int(j)): p for p, (i, j) in enumerate(zip(sh.rv, cols))}


def _columns(sh, rank, rng):
    """rank columns of W (lists of caller rows), cycling through a clique inside a dense group, a single edge and a
    diagonal"""
    groups = [np.asarray(g) for g in sh.groups.values() if len(g) >= 2]
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    off = np.flatnonzero(sh.rv != cols)
    out = []
    for r in range(rank):
        kind = r % 3
        if kind == 0:
            g = groups[rng.integers(len(groups))]
            out.append(sorted(rng.choice(g, size=min(len(g), int(rng.integers(2, 7))), replace=False).tolist()))
        elif kind == 1:
            p = off[rng.integers(off.size)]
            out.append([int(sh.rv[p]), int(cols[p])])
        else:
            out.append([int(rng.integers(sh.N))])
    return out


def _sigma(rank, sign, rng):
    mag = rng.uniform(0.05, 0.25, rank)
    if sign == "+":
        return mag
    if sign == "-":
        return -mag
    return mag * np.where(np.arange(rank) % 2 == 0, 1.0, -1.0)


def _W(sh, cols, rng):
    rows = [np.asarray(c, np.int64) for c in cols]
    vals = [rng.uniform(-1.0, 1.0, len(c)) for c in cols]
    cp = np.concatenate([[0], np.cumsum([len(c) for c in cols])])
    return sp.csc_matrix((np.concatenate(vals), np.concatenate(rows), cp), shape=(sh.N, len(cols)))


def _restated(sh, nz, W, sigma):
    """the values after the update, as the header states them: per stored (i, j), i <= j, ascending r,
    v += (sigma_r * w_i) * w_j"""
    pat = _pattern(sh)
    v = nz.copy()
    for r in range(W.shape[1]):
        if sigma[r] == 0.0:
            continue
        rows = W.indices[W.indptr[r]:W.indptr[r + 1]]
        vals = W.data[W.indptr[r]:W.indptr[r + 1]]
        for a in range(len(rows)):
            for b in range(a, len(rows)):
                (i, wi), (j, wj) = sorted([(int(rows[a]), float(vals[a])), (int(rows[b]), float(vals[b]))])
                p = pat[(i, j)]
                v[p] = v[p] + (float(sigma[r]) * wi) * wj
    return v


def _woodbury(s0, W, sigma, b):
    """((K + E) + W diag(sigma) W^T)^-1 b from the handle s0 that factors K + E"""
    Wd = W.toarray()
    y = s0.solve(b)
    Y = np.column_stack([s0.solve(Wd[:, r]) for r in range(Wd.shape[1])])
    M = np.diag(1.0 / sigma) + Wd.T @ Y
    return y - Y @ np.linalg.solve(M, Wd.T @ y)


def _close(a, b, tol):
    return np.max(np.abs(a - b)) <= tol * max(1.0, np.max(np.abs(b)))


def _check_against_fresh(sh, s, nz_new, **kw):
    ref = _solver(sh, nz_new, **kw)
    assert ref.refactor()
    _, L1, D1, I1 = _factor(s)
    _, L2, D2, I2 = _factor(ref)
    assert _close(D1, D2, FACTOR_TOL) and _close(I1, I2, FACTOR_TOL) and _close(L1, L2, FACTOR_TOL)
    b = np.random.default_rng(5).standard_normal(sh.N)
    assert _close(s.solve(b), ref.solve(b), SOLVE_TOL)
    assert s.inertia() == ref.inertia()
    ref.close()


# ---- every front shape ----
@pytest.mark.parametrize("sign", SIGNS)
@pytest.mark.parametrize("rank", RANKS)
@pytest.mark.parametrize("name", MATRICES)
def test_every_shape(name, rank, sign):
    sh = _shape(name)
    rng = np.random.default_rng(zlib.crc32(f"{name}-{rank}-{sign}".encode()))
    s = _solver(sh, regularize_enable=False)
    assert s.refactor()
    W = _W(sh, _columns(sh, rank, rng), rng)
    sigma = _sigma(rank, sign, rng)
    assert s.updown(W, sigma)
    st = s.updown_stats()
    assert st["passes"] == (rank + 7) // 8 and st["fronts"] >= 1 and st["tasks"] >= st["fronts"]
    nz_new = _restated(sh, sh.nz, W, sigma)
    assert np.array_equal(_values(s, sh.nz.size).view(np.uint64), nz_new.view(np.uint64))
    _check_against_fresh(sh, s, nz_new, regularize_enable=False)
    b = rng.standard_normal(sh.N)
    x, info = s.solve_refined(b, max_iter=2, tol=1e-14)
    assert info.converged and info.steps <= 2
    s.close()


@pytest.mark.parametrize("group,j", ldl_shapes.REG_SITES)
def test_regularisation_is_kept(group, j):
    sh = ldl_shapes.regularised(group, j)
    s0, s = _solver(sh), _solver(sh)
    assert s0.refactor() and s.refactor()
    nreg = s.linear_solver_info().regularize_count
    assert nreg > 0
    rng = np.random.default_rng(zlib.crc32(f"kept-{group}-{j}".encode()))
    W = _W(sh, _columns(sh, 9, rng), rng)
    sigma = _sigma(9, "mixed", rng)
    assert s.updown(W, sigma)
    assert s.linear_solver_info().regularize_count == nreg
    b = rng.standard_normal(sh.N)
    assert _close(s.solve(b), _woodbury(s0, W, sigma, b), SOLVE_TOL)
    s.close()
    s0.close()


def test_update_then_downdate_returns_the_factor():
    sh = ldl_shapes.big_fronts()
    s = _solver(sh)
    assert s.refactor()
    _, L0, D0, I0 = _factor(s)
    rng = np.random.default_rng(7)
    W = _W(sh, _columns(sh, 17, rng), rng)
    sigma = _sigma(17, "+", rng)
    assert s.updown(W, sigma)
    assert s.updown(W, -sigma)
    _, L1, D1, I1 = _factor(s)
    assert _close(D1, D0, FACTOR_TOL) and _close(I1, I0, FACTOR_TOL) and _close(L1, L0, FACTOR_TOL)
    s.close()


def _grid_laplacian(nx, ny, rng):
    n = nx * ny
    idx = np.arange(n).reshape(nx, ny)
    e = np.concatenate([np.stack([idx[:-1, :].ravel(), idx[1:, :].ravel()], 1),
                        np.stack([idx[:, :-1].ravel(), idx[:, 1:].ravel()], 1)])
    w = rng.uniform(0.5, 2.0, len(e))
    return e, w


def _laplacian_triu(n, e, w, shift):
    Lp = sp.coo_matrix((np.concatenate([-w, -w]), (np.concatenate([e[:, 0], e[:, 1]]), np.concatenate([e[:, 1], e[:, 0]]))),
                       shape=(n, n)).tocsc()
    Lp = Lp + sp.diags(-np.asarray(Lp.sum(axis=1)).ravel() + shift)
    T = sp.triu(Lp).tocsc()
    T.sort_indices()
    return T


def test_graph_laplacian_effective_resistances():
    rng = np.random.default_rng(11)
    e, w = _grid_laplacian(30, 40, rng)
    n = 1200
    T = _laplacian_triu(n, e, w, 1e-3)
    s = cb.CudaLDLSolver(n, T.indptr, T.indices, T.data, np.ones(n, np.int8))
    assert s.refactor()
    pick = rng.choice(len(e), 5, replace=False)
    dw = rng.uniform(-0.4, 1.0, 5)
    cols = []
    for k in pick:
        cols.append(np.zeros(n))
        cols[-1][e[k, 0]], cols[-1][e[k, 1]] = 1.0, -1.0
    W = sp.csc_matrix(np.column_stack(cols))
    assert s.updown(W, dw)
    w2 = w.copy()
    w2[pick] += dw
    T2 = _laplacian_triu(n, e, w2, 1e-3)
    ref = cb.CudaLDLSolver(n, T2.indptr, T2.indices, T2.data, np.ones(n, np.int8))
    assert ref.refactor()
    q = rng.choice(len(e), 20, replace=False)
    i, j = e[q, 0], e[q, 1]

    def resistances(h):
        rows = np.concatenate([i, j, i])
        cls = np.concatenate([i, j, j])
        v = h.inverse_entries(rows, cls)
        return v[:20] + v[20:40] - 2 * v[40:]

    r1, r2 = resistances(s), resistances(ref)
    assert np.max(np.abs(r1 - r2) / np.abs(r2)) <= 1e-8
    s.close()
    ref.close()


def test_sign_flips_with_regularisation_off():
    sh = ldl_shapes.big_fronts()
    s = _solver(sh, regularize_enable=False)
    assert s.refactor()
    pos0 = s.inertia()[0]
    _, _, D, _ = _factor(s)
    perm = s.perm()
    # downdates on three diagonals of positive pivots, each past the pivot: the pivots become negative
    ks = [k for k in np.argsort(D) if D[k] > 0][:3]
    v = [int(perm[k]) for k in ks]
    W = sp.csc_matrix((np.ones(3), (np.array(v), np.arange(3))), shape=(sh.N, 3))
    sigma = -(np.array([D[k] for k in ks]) + 2.0)
    assert s.updown(W, sigma)
    nz_new = _restated(sh, sh.nz, W, sigma)
    ref = _solver(sh, nz_new, regularize_enable=False)
    assert ref.refactor()
    assert s.inertia() == ref.inertia() and s.inertia()[0] < pos0
    sg1, ld1 = s.slogdet()
    sg2, ld2 = ref.slogdet()
    assert sg1 == sg2 and abs(ld1 - ld2) <= 1e-10 * abs(ld2)
    s.close()
    ref.close()


def test_downdate_through_zero_gives_verdict_0_and_a_refactor_recovers():
    sh = ldl_shapes.big_fronts()
    nz = sh.nz.copy()
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    diag = sh.rv == cols
    nz[diag] = np.abs(nz[diag])          # every pivot positive: a positive definite matrix
    ds = np.ones(sh.N, np.int8)
    s = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, nz, ds, perm=sh.perm)
    assert s.refactor() and s.linear_solver_info().regularize_count == 0
    v = int(sh.groups["sep"][5])
    W = sp.csc_matrix((np.ones(1), (np.array([v]), np.array([0]))), shape=(sh.N, 1))
    assert not s.updown(W, -2.0 * abs(nz[sh.cp[v + 1] - 1]))
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.solve(np.ones(sh.N))
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.updown(W, 1.0)
    assert s.refactor()
    assert s.linear_solver_info().regularize_count > 0
    s.close()


def test_other_calls_on_the_updated_factor():
    sh = ldl_shapes.child_records()
    s = _solver(sh)
    assert s.refactor()
    rng = np.random.default_rng(13)
    W = _W(sh, _columns(sh, 8, rng), rng)
    sigma = _sigma(8, "mixed", rng)
    assert s.updown(W, sigma)
    ref = _solver(sh, _restated(sh, sh.nz, W, sigma))
    assert ref.refactor()
    Z1, Z2 = s.selected_inverse(), ref.selected_inverse()
    assert _close(Z1.data, Z2.data, SOLVE_TOL)
    r, c = rng.integers(0, sh.N, 50), rng.integers(0, sh.N, 50)
    assert _close(s.inverse_entries(r, c), ref.inverse_entries(r, c), SOLVE_TOL)
    bi = rng.choice(sh.N, 5, replace=False)
    bv = rng.standard_normal(5)
    assert _close(s.solve_sparse((bi, bv), bi), ref.solve_sparse((bi, bv), bi), SOLVE_TOL)
    (g1, l1), (g2, l2) = s.slogdet(), ref.slogdet()
    assert g1 == g2 and abs(l1 - l2) <= 1e-12 * abs(l2)
    s.close()
    ref.close()


def test_refusals_and_no_ops():
    sh = ldl_shapes.child_records()
    s = _solver(sh)
    W = sp.csc_matrix((np.ones(1), (np.array([0]), np.array([0]))), shape=(sh.N, 1))
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.updown(W, 1.0)
    assert s.refactor()
    before = _digest(s)
    nz0 = _values(s, sh.nz.size)
    pat = _pattern(sh)
    a = int(sh.groups["sep"][0])
    far = next(b for b in range(sh.N) if (min(a, b), max(a, b)) not in pat)
    f = cb.lib().cldl_updown
    f.argtypes = [C.c_void_p, C.c_uint64] + [C.POINTER(C.c_uint64)] * 2 + [C.POINTER(C.c_double)] * 2
    f.restype = C.c_int
    u64 = lambda x: np.ascontiguousarray(x, np.uint64)
    f64 = lambda x: np.ascontiguousarray(x, np.float64)
    P = lambda x, t: x.ctypes.data_as(C.POINTER(t))

    def call(cp, ri, wv, sg):
        cp, ri, wv, sg = u64(cp), u64(ri), f64(wv), f64(sg)
        return f(s._h, cp.size - 1, P(cp, C.c_uint64), P(ri, C.c_uint64), P(wv, C.c_double), P(sg, C.c_double))

    assert call([0, 1], [sh.N], [1.0], [1.0]) == ARG                    # index >= n
    assert call([0, 2], [a, a], [1.0, 1.0], [1.0]) == ARG               # duplicate row
    assert call([0, 1], [a], [1.0], [np.nan]) == ARG                    # sigma not finite
    assert call([0, 1], [a], [1.0], [np.inf]) == ARG
    assert call([0, 2], [a, far], [1.0, 1.0], [1.0]) == ARG             # a pair outside the pattern
    assert call([0, 1, 3], [a, a, far], [1.0, 1.0, 1.0], [1.0, 1.0]) == ARG   # the second column refused: nothing changes
    one = u64([0, 1])
    assert f(s._h, 1, P(one, C.c_uint64), None, None, P(f64([1.0]), C.c_double)) == ARG   # NULL arrays
    assert f(s._h, 1, None, None, None, None) == ARG
    assert _digest(s) == before and np.array_equal(_values(s, sh.nz.size), nz0)
    # no-ops: k = 0, an empty column, sigma = 0
    assert f(s._h, 0, None, None, None, None) == 1
    assert call([0, 0], [], [], [1.0]) == 1
    assert call([0, 1], [a], [1.0], [0.0]) == 1
    assert _digest(s) == before and np.array_equal(_values(s, sh.nz.size), nz0)
    assert s.refactor()
    s.close()
    t = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, shard_nranks=2, shard_rank=0)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        t.updown(W, 1.0)
    t.close()
    u = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, schur=[0, 1])
    assert u.refactor()
    with pytest.raises(cb.BackendError, match="BadArgument"):
        u.updown(W, 1.0)
    u.close()
    # a refactor that found null pivots
    nz = sh.nz.copy()
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    z = (sh.rv == a) | (cols == a)
    nz[z] = 0.0
    v = _solver(sh, nz, null_pivot_tol=1e-12)
    assert v.refactor() and v.inertia()[2] == 1
    with pytest.raises(cb.BackendError, match="BadArgument"):
        v.updown(W, 1.0)
    v.close()


def test_repeatable_device_form_and_untouched_handles():
    import torch
    sh = ldl_shapes.big_fronts()
    rng = np.random.default_rng(17)
    W = _W(sh, _columns(sh, 9, rng), rng)
    sigma = _sigma(9, "mixed", rng)
    a, b, c = _solver(sh), _solver(sh), _solver(sh)
    for h in (a, b, c):
        assert h.refactor()
    untouched = _digest(c)
    assert a.updown(W, sigma) and b.updown(W, sigma)
    assert _digest(a) == _digest(b)
    assert _digest(c) == untouched
    d = _solver(sh)
    assert d.refactor()
    dw = torch.tensor(W.data, dtype=torch.float64, device=_device())
    if dw.is_cuda:
        torch.cuda.synchronize()
    d.updown_dev(W.indptr, W.indices, dw.data_ptr(), sigma)
    assert d.sync_status() == 1
    assert _digest(d) == _digest(a)
    assert np.array_equal(_values(d, sh.nz.size), _values(a, sh.nz.size))
    x = np.random.default_rng(1).standard_normal(sh.N)
    assert np.array_equal(d.solve(x), a.solve(x))
    for h in (a, b, c, d):
        h.close()


@pytest.mark.parametrize("rank", [1, 8])
def test_c2_sized_kkt(rank):
    from helpers import workloads
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    s0 = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=cb.ORDER_ND)
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=cb.ORDER_ND)
    assert s0.refactor() and s.refactor()
    rng = np.random.default_rng(rank)
    cols = np.repeat(np.arange(N), np.diff(cp))
    n = pr["P"].shape[0]
    off = np.flatnonzero((rv != cols) & (cols >= n) & (rv < n))     # entries of A: (variable, constraint) edges
    rows, wv = [], []
    for k in rng.choice(off, rank, replace=False):
        rows.append([int(rv[k]), int(cols[k])])
        wv.append(rng.uniform(-1, 1, 2))
    W = sp.csc_matrix((np.concatenate(wv), np.concatenate(rows), np.arange(0, 2 * rank + 1, 2)), shape=(N, rank))
    sigma = rng.uniform(0.05, 0.2, rank)          # a positive term: the (1,1) block stays positive definite
    assert s.updown(W, sigma)
    b = rng.standard_normal(N)
    assert _close(s.solve(b), _woodbury(s0, W, sigma, b), SOLVE_TOL)
    s.close()
    s0.close()
