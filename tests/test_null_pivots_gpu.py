"""Null pivots (CudaLDLSolver(null_pivot_tol=...), cldl_set_null_pivot_tol / cldl_null_pivots / cldl_inertia /
cldl_null_space(_dev)).

Off is off: with the test off, or with a tolerance below every |d_k|, the factor is bitwise the one of a handle that
never set a tolerance (the shape matrices of tests/ldl_shapes.py and a C2-sized KKT matrix).
Every pivot site: one null pivot at each of ldl_shapes.REG_SITES (k_factor_leaf1, k_factor_level, an F task and a D
task at pivots 0, 1, 2, 3, 8), in a positive semidefinite matrix with the layout of ldl_shapes.regularised: (a) a
vertex whose row and column are zero (structure kept), an exact 0.0 pivot with null vector e_v; (b) a vertex that
duplicates the one before it in its front, a pivot at rounding level with null vector e_u - e_v.
Laplacians of graphs with c components (a few thousand nodes under ORDER_BEST, and a grid of more than 1e5 nodes cut
into strips): c null pivots, whose null space is spanned by the components' indicators.
Solves with the generalised inverse, selected inversion, slogdet, an indefinite block (the residual tells), the
refusals, repeatability, an unchanged factor and the device-pointer form."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import scipy.linalg as sla
import scipy.sparse as sp
from scipy.spatial import cKDTree

import clarabel_rs_b200 as cb
import ldl_shapes

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
TOL = 1e-8          # every pivot of the matrices below that is not null is >= 0.1


def _layout(seed=3):
    """the groups and couplings of ldl_shapes.regularised (pivot sites leaf1, level, F, D), every diagonal positive"""
    b = ldl_shapes.Builder(seed)
    sep = b.group(100, "sep")
    order = []
    g = {}
    for name, ns, rows, lift in [("leaf1", 1, np.arange(1, 6), False), ("level", 6, np.arange(2, 12), False),
                                 ("F", 9, np.arange(5, 30), True), ("D", 9, np.arange(1, 97), False)]:
        g[name] = b.group(ns, name)
        b.couple(g[name], sep, None, rows)
        if lift:
            order.append(b.lift(g[name]))
        order.append(g[name])
    return b.build("null_layout", ldl_shapes._blocked(b, sep, order), minus=0.0)


def _with_values(sh, K):
    """the shape with its stored upper-triangle entries taken from the dense symmetric K (pattern unchanged)"""
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    return ldl_shapes.Shape(sh.name, sh.N, sh.cp, sh.rv, K[sh.rv, cols].copy(), sh.ds, sh.perm, sh.groups)


def _site_matrix(group, j, kind):
    """(shape, null vector) with the null pivot at pivot j of `group`.  'zero': vertex v's row and column are 0.  'dup':
    K = T^T K0' T, K0' the matrix without v and T x = x with x_u + x_v at u, so v's row and column repeat u's (u the
    vertex before v in the group) and K (e_u - e_v) = 0; K stays positive semidefinite."""
    sh = _layout()
    K = sh.dense()
    v = int(sh.groups[group][j])
    w = np.zeros(sh.N)
    if kind == "zero":
        K[v, :] = 0.0
        K[:, v] = 0.0
        w[v] = 1.0
    else:
        u = int(sh.groups[group][j - 1])
        K[v, :] = K[u, :]
        K[:, v] = K[:, u]
        K[v, v] = K[u, v] = K[v, u] = K[u, u]
        w[u], w[v] = -1.0, 1.0
    return _with_values(sh, K), w


def _solver(sh, tol=TOL, **kw):
    return cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, null_pivot_tol=tol, **kw)


def _sym(n, cp, rv, nz):
    K = sp.csc_matrix((nz, rv, cp), shape=(n, n))
    return (K + sp.triu(K, 1).T).tocsr()


def _factor_bytes(s):
    info = s.linear_solver_info()
    L, D, Dinv = np.empty(info.nnzL_stored), np.empty(s.n), np.empty(s.n)
    f = cb.lib().cldl_get_factor
    f.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * 3
    f.restype = C.c_int
    assert f(s._h, *(a.ctypes.data_as(C.POINTER(C.c_double)) for a in (L, D, Dinv))) == 0
    return [hashlib.sha256(a.tobytes()).hexdigest() for a in (L, D, Dinv)], D


def _parallel(v, w):
    """1 - |cos| of the angle between v and w"""
    return 1.0 - abs(float(v @ w)) / (np.linalg.norm(v) * np.linalg.norm(w))


SITE_CASES = [(g, j, "zero") for g, j in ldl_shapes.REG_SITES] + \
             [(g, j, "dup") for g, j in ldl_shapes.REG_SITES if j >= 1]


# ---- off is off ----
def _off_is_off(N, cp, rv, nz, ds, perm=None, **kw):
    ref = cb.CudaLDLSolver(N, cp, rv, nz, ds, perm=perm, **kw)
    assert ref.refactor()
    want, D = _factor_bytes(ref)
    below = 0.5 * float(np.min(np.abs(D)))
    assert below > 0.0
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, perm=perm, null_pivot_tol=0.0, **kw)
    s.set_null_pivot_tol(0.0)
    assert s.refactor() and _factor_bytes(s)[0] == want
    assert s.inertia() == (ref.linear_solver_info().positive_inertia, N - ref.linear_solver_info().positive_inertia, 0)
    s.set_null_pivot_tol(below)
    assert s.refactor() and _factor_bytes(s)[0] == want
    assert s.null_pivots().size == 0 and s.inertia()[2] == 0
    assert s.linear_solver_info().regularize_count == ref.linear_solver_info().regularize_count
    s.set_null_pivot_tol(0.0)
    assert s.refactor() and _factor_bytes(s)[0] == want
    s.close()
    ref.close()


@pytest.mark.parametrize("name", ["big_fronts", "child_records"])
def test_off_is_off_on_the_shapes(name):
    sh = getattr(ldl_shapes, name)()
    _off_is_off(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, sh.perm)


def test_off_is_off_on_a_c2_sized_kkt():
    from helpers import workloads
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    _off_is_off(N, cp, rv, nz, ds, ordering=cb.ORDER_ND)


# ---- every pivot site ----
@pytest.mark.parametrize("group,j,kind", SITE_CASES)
def test_one_null_pivot_at_every_site(group, j, kind):
    sh, w = _site_matrix(group, j, kind)
    s = _solver(sh)
    assert s.refactor() == 1
    info = s.linear_solver_info()
    assert info.regularize_count == 0
    N = sh.N
    assert s.inertia() == (N - 1, 0, 1)
    idx = s.null_pivots()
    assert idx.size == 1
    pos = np.empty(N, np.int64)
    pos[s.perm()] = np.arange(N)
    cand = np.flatnonzero(w)
    assert idx[0] == cand[np.argmax(pos[cand])]          # the later of the pair in elimination order
    _, D = _factor_bytes(s)
    assert D[pos[idx[0]]] == 0.0
    if kind == "zero":
        ref = _solver(sh, tol=0.0, regularize_enable=False)
        with pytest.raises(cb.BackendError, match="ZeroPivot"):
            ref.refactor()          # the pivot is exactly 0.0
        ref.close()
    V, resid = s.null_space()
    assert V.shape == (N, 1) and V[idx[0], 0] == 1.0
    assert _parallel(V[:, 0], w) <= 1e-12
    assert resid[0] <= 100 * N * EPS, resid
    assert s.slogdet() == (0, -np.inf)
    s.close()


def _generalised_inverse_by_solves(s):
    n = s.n
    X = np.empty((n, n))
    for j in range(n):
        e = np.zeros(n)
        e[j] = 1.0
        X[:, j] = s.solve(e)
    return X


@pytest.mark.parametrize("group,j,kind", [("leaf1", 0, "zero"), ("D", 8, "dup"), ("F", 4, "dup")])
def test_solves_and_selected_inverse_with_the_generalised_inverse(group, j, kind):
    sh, w = _site_matrix(group, j, kind)
    s = _solver(sh)
    assert s.refactor()
    K = _sym(sh.N, sh.cp, sh.rv, sh.nz)
    rng = np.random.default_rng(11)
    b = K @ rng.standard_normal(sh.N)            # compatible: in the range of K
    x = s.solve(b)
    assert np.max(np.abs(K @ x - b)) <= 1e-10 * np.max(np.abs(b))
    xr, info = s.solve_refined(b, tol=1e-13)
    assert info.converged
    assert np.max(np.abs(K @ xr - b)) <= 1e-10 * np.max(np.abs(b))
    X = _generalised_inverse_by_solves(s)
    Z = s.selected_inverse().tocoo()
    scale = float(np.max(np.abs(X)))
    assert float(np.max(np.abs(Z.data - X[Z.row, Z.col]))) <= 1e-12 * scale
    # the pruned solves and entries of the inverse compare equal to the full solve, as without null pivots
    wi = rng.choice(sh.N, 17, replace=False)
    bi = rng.choice(sh.N, 5, replace=False)
    bv = rng.standard_normal(5)
    bd = np.zeros(sh.N)
    bd[bi] = bv
    full = s.solve(bd)
    assert np.array_equal(s.solve_sparse((bi, bv), wi), full[wi])
    assert np.array_equal(s.solve_sparse(bd), full)
    assert np.array_equal(s.inverse_entries(wi, np.full(wi.size, bi[0])), X[wi, bi[0]])
    s.close()


# ---- Laplacians ----
def _laplacian(edges, n):
    """upper-triangular CSC of the graph Laplacian (every diagonal stored), all expected signs +"""
    i, j = edges
    A = sp.coo_matrix((np.ones(i.size), (i, j)), shape=(n, n))
    A = ((A + A.T) > 0).astype(np.float64)
    L = (sp.diags(np.asarray(A.sum(axis=1)).ravel()) - A).tocsc()
    U = sp.triu(L).tocsc()
    U.sort_indices()
    return U.indptr.astype(np.int64), U.indices.astype(np.int64), U.data, np.ones(n, np.int8)


def _grid_edges(nx, ny, cut_every):
    """an nx x ny grid; the edges between column blocks of width cut_every are left out"""
    idx = np.arange(nx * ny).reshape(ny, nx)
    h = (idx[:, :-1], idx[:, 1:])
    keep = (np.arange(nx - 1) + 1) % cut_every != 0
    hi, hj = h[0][:, keep].ravel(), h[1][:, keep].ravel()
    vi, vj = idx[:-1, :].ravel(), idx[1:, :].ravel()
    return np.concatenate([hi, vi]), np.concatenate([hj, vj])


def _components(edges, n):
    i, j = edges
    A = sp.coo_matrix((np.ones(i.size), (i, j)), shape=(n, n))
    c, lab = sp.csgraph.connected_components(A, directed=False)
    return c, lab


def _check_laplacian(edges, n, **kw):
    c, lab = _components(edges, n)
    cp, rv, nz, ds = _laplacian(edges, n)
    s = cb.CudaLDLSolver(n, cp, rv, nz, ds, null_pivot_tol=TOL, **kw)
    assert s.refactor()
    assert s.inertia() == (n - c, 0, c)
    idx = s.null_pivots()
    assert idx.size == c
    assert sorted(lab[idx]) == list(range(c))                  # one null pivot per component
    V, resid = s.null_space()
    assert np.all(resid <= 100 * n * EPS), resid.max()
    ind = np.zeros((n, c))
    ind[np.arange(n), lab] = 1.0
    ang = sla.subspace_angles(V, ind)
    assert float(np.max(ang)) <= 1e-10, ang
    Q, _ = s.null_space(orthonormalize=True)
    assert np.allclose(Q.T @ Q, np.eye(c), atol=1e-12)
    return s, c


def test_laplacian_with_components_under_the_default_ordering():
    rng = np.random.default_rng(5)
    # three random geometric-style graphs of 700 - 1500 nodes side by side, and two isolated pairs
    edges, off = ([], []), 0
    for m in (700, 1100, 1500):
        pts = rng.random((m, 2))
        ij = cKDTree(pts).query_pairs(0.07, output_type="ndarray")
        i, j = ij[:, 0], ij[:, 1]
        # a path through all nodes keeps each graph connected
        i, j = np.concatenate([i, np.arange(m - 1)]), np.concatenate([j, np.arange(1, m)])
        edges[0].append(i + off); edges[1].append(j + off)
        off += m
    edges[0].append(np.array([off, off + 2])); edges[1].append(np.array([off + 1, off + 3]))
    n = off + 4
    e = (np.concatenate(edges[0]), np.concatenate(edges[1]))
    s, c = _check_laplacian(e, n)
    assert c == 5
    cp, rv, nz, _ = _laplacian(e, n)
    K = _sym(n, cp, rv, nz)
    b = K @ rng.standard_normal(n)
    x = s.solve(b)
    assert np.max(np.abs(K @ x - b)) <= 1e-10 * np.max(np.abs(b))
    _, info = s.solve_refined(b, tol=1e-13)
    assert info.converged
    assert s.slogdet() == (0, -np.inf)
    s.close()


def test_grid_laplacian_cut_into_strips():
    nx, ny, w = 400, 260, 100                  # 104 000 nodes, four strips of 100 x 260
    s, c = _check_laplacian(_grid_edges(nx, ny, w), nx * ny, ordering=cb.ORDER_ND)
    assert c == nx // w
    s.close()


# ---- an indefinite block: the residual shows it ----
def test_indefinite_zero_block_is_exposed_by_the_residual():
    """a tridiagonal definite matrix with the block [[0, 1], [1, 0]] at two decoupled vertices: both pivots of the block
    are 0.0 and are declared null, but K e_p != 0 there, and resid says so"""
    n, a, b = 60, 20, 21
    K = np.diag(np.full(n, 4.0)) - np.diag(np.ones(n - 1), 1) - np.diag(np.ones(n - 1), -1)
    K[[a, b], :] = 0.0
    K[:, [a, b]] = 0.0
    K[a, b] = K[b, a] = 1.0
    U = sp.csc_matrix(np.triu(K) + np.diag(np.where(np.diag(K) == 0.0, 1.0, 0.0)))   # every diagonal stored ...
    U.sort_indices()
    nz = np.triu(K)[U.indices, np.repeat(np.arange(n), np.diff(U.indptr))]          # ... with its value
    s = cb.CudaLDLSolver(n, U.indptr.astype(np.int64), U.indices.astype(np.int64), nz, np.ones(n, np.int8),
                         perm=np.arange(n), null_pivot_tol=TOL)
    assert s.refactor()
    assert list(s.null_pivots()) == [a, b]
    assert s.inertia() == (n - 2, 0, 2)
    _, resid = s.null_space()
    assert np.all(resid >= 1e-3), resid
    s.close()


# ---- refusals and repeatability ----
def test_refusals():
    sh, _ = _site_matrix("D", 3, "zero")
    s = _solver(sh)
    for bad in (-1.0, float("nan")):
        with pytest.raises(cb.BackendError, match="BadArgument"):
            s.set_null_pivot_tol(bad)
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.null_pivots()
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.null_space()
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.inertia()
    assert s.refactor()
    f = cb.lib().cldl_null_space
    f.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    f.restype = C.c_int
    V = np.empty((sh.N, 2))
    res = np.empty(2)
    for r in (0, 2):
        assert f(s._h, r, V.ctypes.data_as(C.POINTER(C.c_double)), res.ctypes.data_as(C.POINTER(C.c_double))) == -21
    # a refactor that returns 0 leaves nothing to report
    nz = sh.nz.copy()
    nz[0] = np.nan
    s.update_values(np.arange(1), nz[:1])
    assert not s.refactor()
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.null_space()
    s.close()
    t = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, shard_nranks=2, shard_rank=0)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        t.set_null_pivot_tol(TOL)
    t.close()
    u = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, schur=[0, 1])
    with pytest.raises(cb.BackendError, match="BadArgument"):
        u.set_null_pivot_tol(TOL)
    u.close()


def test_repeatable_and_leaves_the_factor_and_solves_unchanged():
    sh, _ = _site_matrix("D", 2, "dup")
    s = _solver(sh)
    assert s.refactor()
    b = np.random.default_rng(3).standard_normal(sh.N)
    before, x0 = _factor_bytes(s)[0], s.solve(b)
    V1, r1 = s.null_space()
    V2, r2 = s.null_space()
    assert np.array_equal(V1.view(np.uint64), V2.view(np.uint64))
    assert np.array_equal(r1.view(np.uint64), r2.view(np.uint64))
    assert _factor_bytes(s)[0] == before
    assert np.array_equal(s.solve(b).view(np.uint64), x0.view(np.uint64))
    # a second refactor with the same values and tolerance gives the same factor and null space
    assert s.refactor()
    assert _factor_bytes(s)[0] == before
    V3, _ = s.null_space()
    assert np.array_equal(V1.view(np.uint64), V3.view(np.uint64))
    s.close()


def test_device_pointer_form():
    import torch
    dev = torch.device("cpu") if os.environ.get("CLARABEL_EMU") == "1" else torch.device("cuda", 0)
    # three null pivots: two zeroed vertices and a duplicate, so that the columns go as a pair and a single
    sh = _layout()
    K = sh.dense()
    for v in (int(sh.groups["level"][2]), int(sh.groups["D"][0])):
        K[v, :] = 0.0
        K[:, v] = 0.0
    u, v = int(sh.groups["F"][3]), int(sh.groups["F"][4])
    K[v, :] = K[u, :]
    K[:, v] = K[:, u]
    K[v, v] = K[u, v] = K[v, u] = K[u, u]
    sh = _with_values(sh, K)
    s = _solver(sh)
    assert s.refactor()
    assert s.inertia() == (sh.N - 3, 0, 3)
    V, resid = s.null_space()
    dV = torch.empty((3, sh.N), dtype=torch.float64, device=dev)     # column-major n x 3
    if dev.type == "cuda":
        torch.cuda.synchronize()
    rd = s.null_space_dev(3, dV.data_ptr())
    assert np.array_equal(dV.cpu().numpy().T, V)
    assert np.array_equal(rd, resid)
    assert np.all(resid <= 100 * sh.N * EPS)
    s.close()
