"""Eigenvalues nearest a shift (CudaLDLSolver.eigsh / eigsh_dev / factor_shifted; cldl_eigsh, cldl_eigsh_dev).

- Analytic: the Dirichlet Laplacian of a 13 x 9 grid, whose eigenvalues are 4 - 2 cos(i pi / 14) - 2 cos(j pi / 10),
  at sigma = 0 (a definite factor) and at a sigma inside a gap mid-spectrum (an indefinite factor): eigenvalues,
  reported residuals, X^T X = I, signs, order and n_below against the exact spectrum.
- Generalised: P1 finite-element stiffness and mass matrices of a triangulated rectangle against scipy.linalg.eigh.
- A quasidefinite KKT matrix at sigma = 0 against numpy.linalg.eigvalsh, with n_below its negative count.
- The shape matrices of tests/ldl_shapes.py (every front shape the kernels dispatch on) with SPD values.
- Edges: n = 2 .. 5 with nev = n - 1 (the basis is the whole space), and a block-diagonal matrix with double
  eigenvalues whose Krylov space from one start vector is invariant (beta = 0, fresh vectors find the second copies).
- Repeatability, the factor and the values unchanged, the device-pointer form, every refusal, M not positive definite,
  factor_shifted's counts against the analytic spectrum, the ABI sizes, and one C2-sized problem against
  scipy.sparse.linalg.eigsh."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.linalg as sla
import scipy.sparse as sp

import clarabel_rs_b200 as cb
import ldl_shapes
from helpers import small_kkt, workloads

pytestmark = pytest.mark.gpu

EMU = os.environ.get("CLARABEL_EMU") == "1"
EIG_TOL = 1e-10          # eigenvalues, relative to max(1, |lambda|)
RESID_TOL = 1e-12        # reported residuals
ORTH_TOL = 1e-12         # ||X^T M X - I||_max


def _triu(K):
    U = sp.csc_matrix(sp.triu(sp.csc_matrix(K)))
    U.sort_indices()
    return U


def _on_pattern(U, K):
    """the values of the dense or sparse symmetric K at U's stored entries (explicit zeros kept)"""
    cols = np.repeat(np.arange(U.shape[0]), np.diff(U.indptr))
    Kd = K.toarray() if sp.issparse(K) else K
    return np.ascontiguousarray(Kd[U.indices, cols], dtype=np.float64)


def _solver(U, perm=None):
    return cb.CudaLDLSolver(U.shape[0], U.indptr, U.indices, np.zeros(U.nnz), np.ones(U.shape[0], np.int8),
                            perm=perm, regularize_enable=False)


def _grid_laplacian(nx, ny):
    T = lambda k: sp.diags([-np.ones(k - 1), 2 * np.ones(k), -np.ones(k - 1)], [-1, 0, 1])
    K = sp.kron(sp.identity(ny), T(nx)) + sp.kron(T(ny), sp.identity(nx))
    ex = np.sort([4 - 2 * np.cos(i * np.pi / (nx + 1)) - 2 * np.cos(j * np.pi / (ny + 1))
                  for i in range(1, nx + 1) for j in range(1, ny + 1)])
    return sp.csc_matrix(K), ex


def _nearest(ex, sigma, k):
    """the k exact eigenvalues nearest sigma, after checking that they are simple and set apart from the next one"""
    d = np.abs(ex - sigma)
    o = np.argsort(d, kind="stable")
    assert d[o[k]] > d[o[k - 1]] * 1.001 + 1e-9, "no gap after the k-th nearest eigenvalue"
    near = np.sort(ex[o[:k]])
    assert np.all(np.diff(np.sort(ex[o[:k + 1]])) > 1e-6), "a repeated eigenvalue among the wanted"
    return near


def _check_pairs(A, M, lam, X, info, ref, n_below):
    """lam against ref, X M-orthonormal with the sign rule, the reported residuals and a recomputed one, n_below"""
    k = lam.size
    assert info.status == 1 and info.nconv == k, info
    assert np.all(np.diff(lam) >= 0)
    assert np.max(np.abs(lam - ref) / np.maximum(1.0, np.abs(ref))) <= EIG_TOL, (lam, ref)
    Md = np.eye(A.shape[0]) if M is None else M
    assert np.max(np.abs(X.T @ Md @ X - np.eye(k))) <= ORTH_TOL
    for c in range(k):
        j = int(np.argmax(np.abs(X[:, c])))
        assert X[j, c] > 0
    assert np.all(info.resid <= RESID_TOL) and info.max_resid == np.max(info.resid), info.resid
    R = A @ X - (Md @ X) * lam
    assert np.max(np.abs(R)) <= 1e-9 * max(1.0, np.max(np.abs(lam))) * np.max(np.abs(X))
    assert info.n_below == n_below
    assert info.solves >= k and (info.m_products == 0) == (M is None)


# ---- 1. analytic ----
@pytest.mark.parametrize("where", ["zero", "mid"])
def test_grid_laplacian_against_the_exact_spectrum(where):
    K, ex = _grid_laplacian(13, 9)
    U = _triu(K)
    A = _on_pattern(U, K)
    if where == "zero":
        sigma = 0.0
    else:                  # the middle of the widest gap between simple eigenvalues near the middle of the spectrum
        mid = [i for i in range(40, 76) if ex[i + 1] - ex[i] > 1e-6 and ex[i] - ex[i - 1] > 1e-6]
        i = max(mid, key=lambda i: ex[i + 1] - ex[i])
        sigma = 0.5 * (ex[i] + ex[i + 1])
    s = _solver(U)
    nb = s.factor_shifted(A, sigma)
    assert nb == int(np.count_nonzero(ex < sigma))
    lam, X, info = s.eigsh(6, sigma)
    _check_pairs(K.toarray(), None, lam, X, info, _nearest(ex, sigma, 6), nb)
    s.close()


# ---- 2. generalised: P1 finite elements ----
def _p1_fem(nx, ny, lx=1.0, ly=0.7):
    """stiffness and mass matrices of P1 elements on a rectangle cut into nx x ny cells of two triangles each,
    Dirichlet boundary (interior nodes only), on one pattern"""
    hx, hy = lx / nx, ly / ny
    node = lambda i, j: (j - 1) * (nx - 1) + (i - 1) if 0 < i < nx and 0 < j < ny else -1
    n = (nx - 1) * (ny - 1)
    Kd, Md = np.zeros((n, n)), np.zeros((n, n))
    for i in range(nx):
        for j in range(ny):
            for tri in (((i, j), (i + 1, j), (i + 1, j + 1)), ((i, j), (i + 1, j + 1), (i, j + 1))):
                P = np.array([[a * hx, b * hy] for a, b in tri])
                B = np.array([P[1] - P[0], P[2] - P[0]]).T
                area = 0.5 * abs(np.linalg.det(B))
                G = np.linalg.solve(B.T, np.array([[-1.0, 1.0, 0.0], [-1.0, 0.0, 1.0]]))
                Ke = area * G.T @ G
                Me = area / 12.0 * (np.ones((3, 3)) + np.eye(3))
                ids = [node(a, b) for a, b in tri]
                for p in range(3):
                    for q in range(3):
                        if ids[p] >= 0 and ids[q] >= 0:
                            Kd[ids[p], ids[q]] += Ke[p, q]
                            Md[ids[p], ids[q]] += Me[p, q]
    return Kd, Md


@pytest.mark.parametrize("sigma", [0.0, 150.0])
def test_p1_stiffness_and_mass_against_dense_generalised_eigh(sigma):
    Kd, Md = _p1_fem(12, 9)
    U = _triu(sp.csc_matrix((np.abs(Kd) + np.abs(Md)) > 0))
    A, M = _on_pattern(U, Kd), _on_pattern(U, Md)
    ex = sla.eigh(Kd, Md, eigvals_only=True)
    s = _solver(U)
    nb = s.factor_shifted(A, sigma, M)
    assert nb == int(np.count_nonzero(ex < sigma))
    lam, X, info = s.eigsh(5, sigma, M)
    _check_pairs(Kd, Md, lam, X, info, _nearest(ex, sigma, 5), nb)
    s.close()


# ---- 3. quasidefinite KKT ----
def test_quasidefinite_kkt_smallest_magnitude():
    N, cp, rv, nz, ds = small_kkt(60, 90, seed=5, window=12)
    U = sp.csc_matrix((nz, rv, cp), shape=(N, N))
    K = (U + sp.triu(U, 1).T).toarray()
    ex = np.linalg.eigvalsh(K)
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, regularize_enable=False)
    assert s.factor_shifted(nz, 0.0) == int(np.count_nonzero(ex < 0))
    lam, X, info = s.eigsh(6, 0.0)
    _check_pairs(K, None, lam, X, info, _nearest(ex, 0.0, 6), int(np.count_nonzero(ex < 0)))
    s.close()


# ---- 4. every front shape ----
@pytest.mark.parametrize("name", ["big_fronts", "child_records"])
def test_shape_matrices_with_spd_values(name):
    sh = getattr(ldl_shapes, name)()
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    nz = np.where(sh.rv == cols, np.abs(sh.nz), sh.nz)
    U = sp.csc_matrix((nz, sh.rv, sh.cp), shape=(sh.N, sh.N))
    K = (U + sp.triu(U, 1).T).toarray()
    ex = np.linalg.eigvalsh(K)
    s = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, nz, np.ones(sh.N, np.int8), perm=sh.perm, regularize_enable=False)
    assert s.factor_shifted(nz, 0.0) == 0
    lam, X, info = s.eigsh(4, 0.0)
    _check_pairs(K, None, lam, X, info, _nearest(ex, 0.0, 4), 0)
    s.close()


# ---- 5. edges ----
@pytest.mark.parametrize("n", [2, 3, 4, 5])
def test_basis_is_the_whole_space(n):
    rng = np.random.default_rng(n)
    Q = rng.standard_normal((n, n))
    K = Q @ Q.T + n * np.eye(n)
    U = _triu(sp.csc_matrix(np.ones((n, n))))
    s = _solver(U)
    ex = np.linalg.eigvalsh(K)
    sigma = 0.5 * (ex[0] + ex[1]) if n > 2 else 0.0
    nb = s.factor_shifted(_on_pattern(U, K), sigma)
    lam, X, info = s.eigsh(n - 1, sigma)
    _check_pairs(K, None, lam, X, info, _nearest(ex, sigma, n - 1), nb)
    assert info.restarts == 0 and info.solves == n


def test_invariant_krylov_space_deflation_finds_both_copies():
    """K = diag(B, B): every eigenvalue is double and the Krylov space of one start vector has dimension 5 < ncv, so
    step 4 meets beta = 0; the fresh vector's Krylov space holds the second copies"""
    B = np.diag(np.arange(1.0, 6.0) * 1.5) + np.diag(-0.4 * np.ones(4), 1) + np.diag(-0.4 * np.ones(4), -1)
    K = np.kron(np.eye(2), B)
    U = _triu(sp.csc_matrix(np.abs(K) > 0))
    s = _solver(U)
    s.factor_shifted(_on_pattern(U, K), 0.0)
    lam, X, info = s.eigsh(2, 0.0, ncv=8)
    mu = np.linalg.eigvalsh(B)[0]
    assert info.status == 1 and np.max(np.abs(lam - mu)) <= EIG_TOL * max(1.0, mu)
    assert np.max(np.abs(X.T @ X - np.eye(2))) <= ORTH_TOL
    assert np.max(info.resid) <= RESID_TOL


# ---- 6. repeatability and side effects ----
def _values(s, nnz):
    """the handle's current values, through cldl_values_dev"""
    import torch
    L = s._L
    ptr = L.cldl_values_dev(s._h)
    if EMU:
        out = np.empty(nnz)
        C.memmove(out.ctypes.data, ptr, nnz * 8)
        return out
    t = torch.empty(nnz, dtype=torch.float64, device="cuda")
    assert L.cldl_copy_dev(C.c_void_p(t.data_ptr()), C.c_void_p(ptr), nnz * 8) == 0
    return t.cpu().numpy()


def test_repeatable_and_without_side_effects():
    Kd, Md = _p1_fem(10, 7)
    U = _triu(sp.csc_matrix((np.abs(Kd) + np.abs(Md)) > 0))
    A, M = _on_pattern(U, Kd), _on_pattern(U, Md)
    s = _solver(U)
    s.factor_shifted(A, 30.0, M)
    b = np.random.default_rng(0).standard_normal(U.shape[0])
    x0, v0 = s.solve(b), _values(s, U.nnz)
    r1 = s.eigsh(4, 30.0, M, seed=3)
    r2 = s.eigsh(4, 30.0, M, seed=3)
    for a, c in ((r1[0], r2[0]), (r1[1], r2[1]), (r1[2].resid, r2[2].resid)):
        assert a.tobytes() == c.tobytes()
    assert s.solve(b).tobytes() == x0.tobytes()
    assert _values(s, U.nnz).tobytes() == v0.tobytes()
    r3 = s.eigsh(4, 30.0, M, seed=4, vectors=False)             # another start vector: the same pairs
    assert r3[1] is None and np.max(np.abs(r3[0] - r1[0])) <= EIG_TOL * np.max(np.abs(r1[0]))
    # the device-pointer form: the same bits
    import torch
    dev = torch.device("cpu") if EMU else torch.device("cuda", 0)
    dM = torch.from_numpy(M).to(dev)
    dX = torch.empty((4, U.shape[0]), dtype=torch.float64, device=dev)
    if not EMU:
        torch.cuda.synchronize()
    lam, info = s.eigsh_dev(4, 30.0, dM.data_ptr(), dX.data_ptr(), seed=3)
    assert lam.tobytes() == r1[0].tobytes() and info.resid.tobytes() == r1[2].resid.tobytes()
    assert dX.cpu().numpy().tobytes() == r1[1].tobytes(order="F")
    s.close()


# ---- 7. refusals ----
def _raw_eigsh(s, nev, sigma=0.0, M=None, ncv=0, max_restarts=300, tol=0.0, evals=True):
    f = s._L.cldl_eigsh
    f.argtypes = [C.c_void_p, C.c_double, C.POINTER(C.c_double), C.c_uint64, C.POINTER(cb.pkg.cldl_eig_opts)] + \
        [C.POINTER(C.c_double)] * 3 + [C.POINTER(cb.pkg.cldl_eig_info)]
    f.restype = C.c_int
    o = cb.pkg.cldl_eig_opts()
    s._L.cldl_default_eig_opts(C.byref(o))
    o.ncv, o.max_restarts, o.tol = ncv, max_restarts, tol
    lam = np.empty(max(nev, 1))
    pd = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    return f(s._h, sigma, None if M is None else pd(M), nev, C.byref(o), pd(lam) if evals else None, None, None, None)


def test_refusals():
    K, ex = _grid_laplacian(7, 5)
    U = _triu(K)
    A, n = _on_pattern(U, K), U.shape[0]
    s = _solver(U)
    assert _raw_eigsh(s, 3) == cb.CLDL_E_NOT_FACTORED
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.eigsh(3, 0.0)
    s.factor_shifted(A, 0.0)
    assert _raw_eigsh(s, 3) == cb.CLDL_OK
    for kw in (dict(nev=0), dict(nev=n), dict(nev=3, ncv=3), dict(nev=3, ncv=n + 1), dict(nev=3, max_restarts=-1),
               dict(nev=3, tol=-1.0), dict(nev=3, tol=float("nan")), dict(nev=3, evals=False)):
        assert _raw_eigsh(s, **kw) == cb.CLDL_E_ARG, kw
    big = _grid_laplacian(30, 20)[0]
    Ub = _triu(big)
    sb = _solver(Ub)
    sb.factor_shifted(_on_pattern(Ub, big), 0.0)
    assert _raw_eigsh(sb, 3, ncv=513) == cb.CLDL_E_ARG          # above 512
    assert _raw_eigsh(sb, 512) == cb.CLDL_E_ARG                  # default ncv: min(n, 512) is not above nev
    sb.close()
    # (the refusal of a mirrored pattern beyond int32, 2 nnzA - n > 2^31 - 1, is not exercised: it needs a matrix of
    # more than 10^9 stored entries)
    # null pivots: sigma at an eigenvalue of a singular matrix (the path Laplacian, null vector of ones)
    P = sp.diags([-np.ones(9), np.r_[1.0, 2 * np.ones(8), 1.0], -np.ones(9)], [-1, 0, 1])
    Up = _triu(P)
    sn = cb.CudaLDLSolver(10, Up.indptr, Up.indices, Up.data, np.ones(10, np.int8), regularize_enable=False,
                          null_pivot_tol=1e-9)
    assert sn.refactor() and sn.inertia()[2] == 1
    assert _raw_eigsh(sn, 2) == cb.CLDL_E_ARG
    sn.close()
    # a regularised factor (one pivot of the wrong sign, regularisation on)
    rg = ldl_shapes.regularised("D", 1)
    sr = cb.CudaLDLSolver(rg.N, rg.cp, rg.rv, rg.nz, rg.ds, perm=rg.perm)
    assert sr.refactor() and sr.linear_solver_info().regularize_count > 0
    assert _raw_eigsh(sr, 2) == cb.CLDL_E_ARG
    sr.close()
    # Schur and sharded handles
    sh = ldl_shapes.big_fronts()
    sc = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, schur=[int(sh.groups["sep"][-1])])
    assert sc.refactor()
    assert _raw_eigsh(sc, 2) == cb.CLDL_E_ARG
    sc.close()
    ss = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, shard_nranks=2, shard_rank=0)
    assert _raw_eigsh(ss, 2) == cb.CLDL_E_ARG
    ss.close()
    # M not positive definite: status -1, NaN results, CLDL_OK
    lam, X, info = s.eigsh(3, 0.0, -np.abs(A))
    assert info.status == -1 and info.nconv == 0 and np.all(np.isnan(lam)) and np.all(np.isnan(X))
    # the handle stays usable
    lam, X, info = s.eigsh(3, 0.0)
    assert info.status == 1
    s.close()


# ---- 8. spectrum slicing ----
def test_factor_shifted_counts_intervals():
    K, ex = _grid_laplacian(13, 9)
    U = _triu(K)
    A = _on_pattern(U, K)
    s = _solver(U)
    cuts = [0.3, 1.0, 2.5, 3.9, 4.1, 6.2, 7.95]
    counts = [s.factor_shifted(A, c) for c in cuts]
    for a, b, ca, cb_ in zip(cuts, cuts[1:], counts, counts[1:]):
        assert cb_ - ca == int(np.count_nonzero((ex >= a) & (ex < b))), (a, b)
    s.close()
    # with regularisation on, the wrong-signed pivots of A - sigma I are regularised: the count would be that of
    # A - sigma I + E, so factor_shifted raises; at sigma = 0 nothing is regularised and the count stands
    r = cb.CudaLDLSolver(U.shape[0], U.indptr, U.indices, A, np.ones(U.shape[0], np.int8))
    with pytest.raises(cb.BackendError, match="regularised"):
        r.factor_shifted(A, 0.3)
    assert r.factor_shifted(A, 0.0) == 0
    r.close()


# ---- 9. ABI ----
def test_abi_sizes_match_the_ctypes_mirrors():
    L = cb.lib()
    out = np.zeros(2, np.uint64)
    L.cldl_eig_abi_sizes.argtypes = [C.POINTER(C.c_uint64)]
    L.cldl_eig_abi_sizes.restype = None
    L.cldl_eig_abi_sizes(out.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert [int(v) for v in out] == [C.sizeof(cb.pkg.cldl_eig_opts), C.sizeof(cb.pkg.cldl_eig_info)]
    o = cb.pkg.cldl_eig_opts()
    L.cldl_default_eig_opts(C.byref(o))
    assert (o.ncv, o.max_restarts, o.tol, o.seed) == (0, 300, 0.0, 0)


# ---- 10. larger size ----
def test_c2_sized_kkt_against_scipy_eigsh():
    import scipy.sparse.linalg as spla
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    P = pr["P"] + 1e-3 * sp.identity(pr["P"].shape[0])
    N, cp, rv, nz, ds = workloads.kkt_triu(P, pr["A"], np.full(pr["A"].shape[0], 1e-3))
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, regularize_enable=False)
    nb = s.factor_shifted(nz, 0.0)
    lam, X, info = s.eigsh(6, 0.0)
    assert info.status == 1 and info.max_resid <= RESID_TOL
    U = sp.csc_matrix((nz, rv, cp), shape=(N, N))
    K = sp.csc_matrix(U + sp.triu(U, 1).T)
    # ARPACK's shift-invert with the handle's solve as OPinv (SuperLU takes minutes at this size); the residuals
    # below are checked against K itself
    op = spla.LinearOperator((N, N), matvec=lambda v: s.solve(np.ravel(v)), dtype=np.float64)
    ref = np.sort(spla.eigsh(K, k=6, sigma=0.0, which="LM", OPinv=op, tol=1e-14, return_eigenvectors=False))
    assert np.max(np.abs(K @ X - X * lam)) <= 1e-9 * max(1.0, np.max(np.abs(lam)))
    assert np.max(np.abs(lam - ref) / np.maximum(1.0, np.abs(ref))) <= EIG_TOL
    assert nb == N - s.inertia()[0]
    s.close()
