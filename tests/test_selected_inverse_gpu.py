"""Selected inversion (CudaLDLSolver.selected_inverse, cldl_selected_inverse): the entries of (K + E)^-1 on the
caller's pattern, against extended-precision references.

(a) The matrices of tests/ldl_shapes.py, whose fronts sit at every shape the factor and solve kernels dispatch on (and
so at every shape of the selected-inversion tasks: whole fronts, row tasks with partial last blocks, pivot blocks of 1
to 64 columns, L11^-1 stored or substituted).  Reference: the dense inverse, refined once with the residual I - K X
in np.longdouble.  Error: max |Z - Z*| / max |Z*| over the pattern, divided by eps cond_1(K).
(b) The regularised-pivot matrices of tests/test_ldl_shapes_gpu.py: against (K + E)^-1, E the diagonal correction
of a dense longdouble LDL^T with the device's pivot rule, the same error over eps cond_1(K + E).
(c) C4 at 1/25 of its size: sampled columns j against K^-1 e_j from a device solve refined with longdouble residuals;
error max |z_j - x_j| / max |x_j| / eps on the pattern of column j.
Also: two calls give identical bits; the stored factor and a following solve are bitwise unchanged; NotFactored
before a refactor, BadArgument on a sharded handle.

Worst values measured on an H100 (SXM, 80 GB HBM3, 700 W power limit; the host-emulated build gives the same (a) and
(b) figures to three digits):
  (a) big_fronts 5.9e-3, child_records 1.2e-2 (cond_1 1.6e2, 6.3e1)
  (b) 2.8e-3 (leaf1 and D pivot 0; cond_1 8.6e8)
  (c) 4.0
The thresholds below keep a margin of at least 100x to these."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import clarabel_rs_b200 as cb
import ldl_shapes

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
LD = np.longdouble
SHAPE_TOL = 5.0      # (a), (b): error / (eps cond_1)
C4_TOL = 1e4         # (c): error / eps


def _sym(sh_or_csc, N=None):
    K = sh_or_csc if N is not None else sp.csc_matrix((sh_or_csc.nz, sh_or_csc.rv, sh_or_csc.cp),
                                                      shape=(sh_or_csc.N, sh_or_csc.N))
    return (K + sp.triu(K, 1).T).tocsr()


def _ld_matmul(Kcsr, X, chunk=128):
    """K X with the products and sums in longdouble (K sparse CSR with no empty row)"""
    out = np.empty((Kcsr.shape[0], X.shape[1]), LD)
    data = Kcsr.data.astype(LD)[:, None]
    for c0 in range(0, X.shape[1], chunk):
        prod = data * X[Kcsr.indices, c0:c0 + chunk].astype(LD)
        out[:, c0:c0 + chunk] = np.add.reduceat(prod, Kcsr.indptr[:-1], axis=0)
    return out


def _inverse_reference(Kcsr):
    Kd = Kcsr.toarray()
    X = np.linalg.inv(Kd)
    R = np.eye(Kd.shape[0], dtype=LD) - _ld_matmul(Kcsr, X)
    return X.astype(LD) + (X @ np.asarray(R, np.float64)).astype(LD), np.linalg.cond(Kd, 1)


def _on_pattern(Z, ref):
    """Z: csc_matrix of the device's result; ref: dense longdouble reference.  Normwise error over the pattern."""
    Zc = Z.tocoo()
    r = ref[Zc.row, Zc.col]
    return float(np.max(np.abs(Zc.data.astype(LD) - r)) / np.max(np.abs(r)))


def _solver(sh):
    return cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm)


@pytest.mark.parametrize("name", [f.__name__ for f in (ldl_shapes.big_fronts, ldl_shapes.child_records)])
def test_shape_matrices_against_the_extended_precision_inverse(name):
    sh = getattr(ldl_shapes, name)()
    s = _solver(sh)
    assert s.refactor()
    assert s.linear_solver_info().regularize_count == 0
    Z = s.selected_inverse()
    assert Z.shape == (sh.N, sh.N) and Z.nnz == len(sh.rv)
    assert np.array_equal(Z.indptr, sh.cp) and np.array_equal(Z.indices, sh.rv)
    ref, cond = _inverse_reference(_sym(sh))
    err = _on_pattern(Z, ref) / (EPS * cond)
    print("%s: error / (eps cond_1) %.2e (cond_1 %.1e)" % (name, err, cond))
    assert err <= SHAPE_TOL, (name, err)


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


@pytest.mark.parametrize("group,j", ldl_shapes.REG_SITES)
def test_regularised_matrices_against_the_inverse_of_k_plus_e(group, j):
    sh = ldl_shapes.regularised(group, j)
    s = _solver(sh)
    assert s.refactor()
    p = s.perm()
    Kd = sh.dense()
    d0, d = _ldl_reference(Kd[np.ix_(p, p)], sh.ds[p].astype(LD))
    assert s.linear_solver_info().regularize_count == int((d != d0).sum()) >= 1
    # E rounded to double: a perturbation of K + E at the level of eps |K|, inside the eps cond_1 scale of the error
    E = np.zeros(sh.N)
    E[p] = np.asarray(d - d0, np.float64)
    KE = (_sym(sh) + sp.diags(E)).tocsr()
    KE.sort_indices()
    ref, cond = _inverse_reference(KE)
    err = _on_pattern(s.selected_inverse(), ref) / (EPS * cond)
    print("reg %s %d: error / (eps cond_1) %.2e (cond_1 %.1e)" % (group, j, err, cond))
    assert err <= SHAPE_TOL, (group, j, err)


def _ld_matvec(Kcsr, x):
    return _ld_matmul(Kcsr, x[:, None], chunk=1)[:, 0]


def test_reduced_c4_sampled_columns_against_refined_solves():
    import factor_digest
    c = factor_digest.reduced_c4()
    s = factor_digest.solver(c)
    assert s.refactor()
    assert s.linear_solver_info().regularize_count == 0
    Z = s.selected_inverse()
    Zs = (Z + sp.triu(Z, 1).T).tocsc()
    K = _sym(sp.csc_matrix((c.nz, c.rv, c.cp), shape=(c.N, c.N)), c.N)
    rng = np.random.default_rng(11)
    worst = 0.0
    for j in rng.choice(c.N, size=24, replace=False):
        e = np.zeros(c.N)
        e[j] = 1.0
        x = s.solve(e)
        for _ in range(3):
            r = e.astype(LD) - _ld_matvec(K, x)
            x = x + s.solve(np.asarray(r, np.float64))
        rows = Zs.indices[Zs.indptr[j]:Zs.indptr[j + 1]]
        z = Zs.data[Zs.indptr[j]:Zs.indptr[j + 1]]
        err = float(np.max(np.abs(z - x[rows])) / np.max(np.abs(x[rows]))) / EPS
        worst = max(worst, err)
        assert err <= C4_TOL, (int(j), err)
    print("c4_reduced: worst sampled-column error / eps %.2e" % worst)


def _factor_bytes(s):
    info = s.linear_solver_info()
    L, D, Dinv = np.empty(info.nnzL_stored), np.empty(s.n), np.empty(s.n)
    f = cb.lib().cldl_get_factor
    f.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * 3
    f.restype = C.c_int
    assert f(s._h, *(a.ctypes.data_as(C.POINTER(C.c_double)) for a in (L, D, Dinv))) == 0
    return [hashlib.sha256(a.tobytes()).hexdigest() for a in (L, D, Dinv)]


def test_repeatable_and_leaves_the_factor_and_solves_unchanged():
    sh = ldl_shapes.big_fronts()
    s = _solver(sh)
    assert s.refactor()
    b = np.random.default_rng(3).standard_normal(sh.N)
    before, x0 = _factor_bytes(s), s.solve(b)
    Z1 = s.selected_inverse()
    Z2 = s.selected_inverse()
    assert np.array_equal(Z1.data.view(np.uint64), Z2.data.view(np.uint64))
    assert _factor_bytes(s) == before
    assert np.array_equal(s.solve(b).view(np.uint64), x0.view(np.uint64))
    # after a value update and a refactor, the next call inverts the new matrix
    nz = sh.nz.copy()
    diag = np.nonzero(sh.rv == np.repeat(np.arange(sh.N), np.diff(sh.cp)))[0]
    nz[diag] *= 2.0
    s.update_values(diag, nz[diag])
    assert s.refactor()
    sh2 = ldl_shapes.Shape(sh.name, sh.N, sh.cp, sh.rv, nz, sh.ds, sh.perm, sh.groups)
    ref, cond = _inverse_reference(_sym(sh2))
    assert _on_pattern(s.selected_inverse(), ref) / (EPS * cond) <= SHAPE_TOL


def test_refusals():
    sh = ldl_shapes.child_records()
    s = _solver(sh)
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.selected_inverse()
    t = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, shard_nranks=2, shard_rank=0)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        t.selected_inverse()
    t.close()
    s.close()
