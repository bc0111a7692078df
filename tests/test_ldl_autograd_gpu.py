"""Log-determinants and adjoint solves from the multifrontal LDL^T (CudaLDLSolver.slogdet / adjoint_solve, cldl_logdet /
cldl_adjoint_solve) and the differentiable layer on top (autograd.SparseLDL), against extended-precision references.

(a) slogdet on the matrices of tests/ldl_shapes.py: against sum log|d*_k| of an LDL^T in np.longdouble in the device's
permutation.  The sign must be exact.  Error: |logabsdet - logabsdet*| in units of eps cond_1(K) (1 + sum |log|d*_k||):
to first order a backward error dK of the factorisation changes log|det K| by tr(K^-1 dK), a multiple of eps cond_1,
and the sum of n logarithms adds its own rounding, a multiple of eps sum |log|d_k||.  (The rounding of the result alone
is eps |logabsdet|: on big_fronts, 7599 eps, 24 eps cond_1.)
(b) slogdet on the regularised-pivot matrices: against log|det(K + E)| with E the diagonal correction of a longdouble
LDL^T with the device's pivot rule; the same error unit with cond_1(K + E).
(c) slogdet on a Schur handle: against log|det K_BB|, B's pivots of the same longdouble LDL^T.
(d) adjoint_solve: gb against the longdouble-refined K^-1 g, and gvals against -(gb*_i x_j + x_i gb*_j) on the
pattern; error max |y - y*| / max |y*| / (eps cond_1).
(e) SparseLDL: gradcheck in float64 of solve (in values and b, b of shape (n,) and (n, 2)) and of slogdet (in values)
on small SPD and quasidefinite matrices with mixed dsigns; the gradients equal those of torch.linalg.solve / slogdet on
the dense symmetric matrix to GRAD_TOL relative.
Also: the refactor counts of factorisation reuse; two calls give identical bits; the stored factor and a later solve
are bitwise unchanged; NotFactored before a refactor, BadArgument on sharded and (adjoint) Schur handles; the layer
raises on a matrix whose refactor regularises.

Worst values measured on an H100 (SXM, 80 GB HBM3, 700 W power limit; the host-emulated build gives the same figures
to two digits, except gvals on big_fronts, 1.2e-2):
  (a) big_fronts 3.2e-3, child_records 6.7e-3 (cond_1 1.6e2, 6.3e1)
  (b) 5.7e-10 (F 4; cond_1 8.6e8)
  (c) 2.7e-3
  (d) gb 1.5e-2 (big_fronts), gvals 7.9e-3 (child_records)
The thresholds of (a) to (d) keep a margin of at least 100x to these."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import clarabel_rs_b200 as cb
import ldl_shapes
from test_selected_inverse_gpu import _factor_bytes, _inverse_reference, _ldl_reference, _on_pattern, _sym

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
LD = np.longdouble
LOGDET_TOL = 1.0     # (a), (b), (c): error / (eps cond_1 (1 + sum |log|d_k||))
ADJ_TOL = 5.0        # (d): error / (eps cond_1)
GRAD_TOL = 1e-10     # (e): relative difference to the dense torch gradients


def _solver(sh, **kw):
    return cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, **kw)


def _ld_pivots(Kp):
    """the pivots of the LDL^T of the dense (permuted) Kp in longdouble, without pivoting; each elimination step updates
    only the rows its column reaches, so the cost is that of the sparse factorisation"""
    A = Kp.astype(LD)
    n = A.shape[0]
    d = np.zeros(n, LD)
    for k in range(n):
        d[k] = A[k, k]
        nz = k + 1 + np.flatnonzero(A[k + 1:, k])
        if nz.size:
            A[np.ix_(nz, nz)] -= np.outer(A[nz, k] / d[k], A[k, nz])
    return d


def _slogdet_ref(d):
    """(sign, logabsdet, sum |log|d_k||) from longdouble pivots"""
    lg = np.log(np.abs(d))
    return (-1 if int((d < 0).sum()) % 2 else 1), np.sum(lg), float(np.sum(np.abs(lg)))


def _logdet_err(lad, ref, cond):
    """|logabsdet - logabsdet*| / (eps cond_1 (1 + sum |log|d*_k||))"""
    return float(abs(LD(lad) - ref[1])) / (EPS * cond * (1.0 + ref[2]))


SHAPES = [f.__name__ for f in (ldl_shapes.big_fronts, ldl_shapes.child_records)]


@pytest.mark.parametrize("name", SHAPES)
def test_slogdet_of_the_shape_matrices_against_the_extended_precision_ldl(name):
    sh = getattr(ldl_shapes, name)()
    s = _solver(sh)
    assert s.refactor()
    assert s.linear_solver_info().regularize_count == 0
    p = s.perm()
    Kd = sh.dense()
    ref = _slogdet_ref(_ld_pivots(Kd[np.ix_(p, p)]))
    sign, lad = s.slogdet()
    cond = np.linalg.cond(Kd, 1)
    err = _logdet_err(lad, ref, cond)
    print("%s: slogdet error / (eps cond_1 (1 + sum|log|d||)) %.2e (cond_1 %.1e, logabsdet %.6e)" % (name, err, cond, lad))
    assert sign == ref[0]
    assert err <= LOGDET_TOL, (name, err)


@pytest.mark.parametrize("group,j", ldl_shapes.REG_SITES)
def test_slogdet_of_the_regularised_matrices_is_that_of_k_plus_e(group, j):
    sh = ldl_shapes.regularised(group, j)
    s = _solver(sh)
    assert s.refactor()
    p = s.perm()
    Kd = sh.dense()
    d0, d = _ldl_reference(Kd[np.ix_(p, p)], sh.ds[p].astype(LD))
    assert s.linear_solver_info().regularize_count == int((d != d0).sum()) >= 1
    E = np.zeros(sh.N)
    E[p] = np.asarray(d - d0, np.float64)
    ref = _slogdet_ref(d)
    sign, lad = s.slogdet()
    cond = np.linalg.cond(Kd + np.diag(E), 1)
    err = _logdet_err(lad, ref, cond)
    print("reg %s %d: slogdet error / (eps cond_1 (1 + sum|log|d||)) %.2e (cond_1 %.1e)" % (group, j, err, cond))
    assert sign == ref[0]
    assert err <= LOGDET_TOL, (group, j, err)


def test_slogdet_on_a_schur_handle_is_that_of_k_bb():
    sh = ldl_shapes.child_records()
    S = np.random.default_rng(7).choice(sh.N, size=40, replace=False)
    s = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, schur=S)
    assert s.refactor()
    p = s.perm()
    B = p[:sh.N - len(S)]
    assert not np.isin(B, S).any()
    Kd = sh.dense()
    ref = _slogdet_ref(_ld_pivots(Kd[np.ix_(B, B)]))
    sign, lad = s.slogdet()
    assert s.linear_solver_info().positive_inertia == int((sh.ds[B] > 0).sum())
    cond = np.linalg.cond(Kd[np.ix_(B, B)], 1)
    err = _logdet_err(lad, ref, cond)
    print("schur: slogdet error / (eps cond_1 (1 + sum|log|d||)) %.2e (cond_1 %.1e)" % (err, cond))
    assert sign == ref[0]
    assert err <= LOGDET_TOL, err
    s.close()


@pytest.mark.parametrize("name", SHAPES)
def test_adjoint_solve_against_the_extended_precision_inverse(name):
    sh = getattr(ldl_shapes, name)()
    s = _solver(sh)
    assert s.refactor()
    rng = np.random.default_rng(5)
    b, g = rng.standard_normal(sh.N), rng.standard_normal(sh.N)
    x = s.solve(b)
    gb, gv = s.adjoint_solve(g, x)
    assert gv.shape == (sh.N, sh.N) and np.array_equal(gv.indptr, sh.cp) and np.array_equal(gv.indices, sh.rv)
    Z, cond = _inverse_reference(_sym(sh))
    gb_ref = Z @ g.astype(LD)
    err_gb = float(np.max(np.abs(gb.astype(LD) - gb_ref)) / np.max(np.abs(gb_ref))) / (EPS * cond)
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    xl = x.astype(LD)
    ref = -(gb_ref[sh.rv] * xl[cols] + xl[sh.rv] * gb_ref[cols])
    diag = sh.rv == cols
    ref[diag] = -(gb_ref[sh.rv] * xl[cols])[diag]
    err_gv = float(np.max(np.abs(gv.data.astype(LD) - ref)) / np.max(np.abs(ref))) / (EPS * cond)
    print("%s: adjoint error / (eps cond_1) gb %.2e gvals %.2e (cond_1 %.1e)" % (name, err_gb, err_gv, cond))
    assert err_gb <= ADJ_TOL and err_gv <= ADJ_TOL, (name, err_gb, err_gv)
    # gb alone: the same bits as the solve of g
    assert np.array_equal(gb.view(np.uint64), s.solve(g).view(np.uint64))


def test_repeatable_and_leaves_the_factor_and_solves_unchanged():
    sh = ldl_shapes.big_fronts()
    s = _solver(sh)
    assert s.refactor()
    rng = np.random.default_rng(3)
    b, g = rng.standard_normal(sh.N), rng.standard_normal(sh.N)
    before, x0 = _factor_bytes(s), s.solve(b)
    l1, l2 = s.slogdet(), s.slogdet()
    assert l1[0] == l2[0] and np.float64(l1[1]).view(np.uint64) == np.float64(l2[1]).view(np.uint64)
    a1, a2 = s.adjoint_solve(g, x0), s.adjoint_solve(g, x0)
    assert np.array_equal(a1[0].view(np.uint64), a2[0].view(np.uint64))
    assert np.array_equal(a1[1].data.view(np.uint64), a2[1].data.view(np.uint64))
    assert _factor_bytes(s) == before
    assert np.array_equal(s.solve(b).view(np.uint64), x0.view(np.uint64))


def test_refusals():
    sh = ldl_shapes.child_records()
    s = _solver(sh)
    z = np.zeros(sh.N)
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.slogdet()
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.adjoint_solve(z, z)
    t = _solver(sh, shard_nranks=2, shard_rank=0)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        t.slogdet()
    with pytest.raises(cb.BackendError, match="BadArgument"):
        t.adjoint_solve(z, z)
    t.close()
    u = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, schur=[0, 1, 2])
    assert u.refactor()
    with pytest.raises(cb.BackendError, match="BadArgument"):
        u.adjoint_solve(z, z)
    u.close()
    s.close()


# ---------------------------------------------------------------- the differentiable layer
def _ag():
    import clarabel_rs_b200_pkg.autograd as ag
    return ag


def _dev():
    """where the layer's tensors live: host memory on the emulated build"""
    return torch.device("cpu") if os.environ.get("CLARABEL_EMU") == "1" else torch.device("cuda", 0)


def _small(kind, seed=0):
    """(n, colptr, rowval, values, dsigns) of a small sparse SPD (kind "spd") or quasidefinite ("qd": [P + I, A'; A, -I]
    with the -1 signs interleaved) matrix, upper triangle"""
    rng = np.random.default_rng(seed)
    n = 14
    M = sp.random(n, n, density=0.25, random_state=rng).toarray()
    M = np.triu(M + M.T, 1)
    if kind == "spd":
        ds = np.ones(n, np.int8)
    else:
        ds = np.where(np.arange(n) % 3 == 2, -1, 1).astype(np.int8)
        M[np.ix_(ds < 0, ds < 0)] = 0.0
    M += np.diag(ds * (1.0 + np.abs(M).sum(0) + np.abs(M).sum(1)))
    U = sp.csc_matrix(np.triu(M))
    U.sort_indices()
    return n, U.indptr.astype(np.int64), U.indices.astype(np.int64), U.data.copy(), ds


def _dense(n, cp, rv, v):
    col = torch.as_tensor(np.repeat(np.arange(n), np.diff(cp)), device=v.device)
    rows = torch.as_tensor(rv, device=v.device)
    U = torch.zeros(n, n, dtype=v.dtype, device=v.device).index_put((rows, col), v)
    return U + U.T - torch.diag(torch.diagonal(U))


@pytest.mark.parametrize("kind", ["spd", "qd"])
def test_gradcheck_and_the_dense_gradients(kind):
    ag, dev = _ag(), _dev()
    n, cp, rv, nz, ds = _small(kind)
    K = ag.SparseLDL(n, cp, rv, ds, device=0)
    rng = np.random.default_rng(1)
    v = torch.tensor(nz, device=dev, requires_grad=True)
    for shape in [(n,), (n, 2)]:
        b = torch.tensor(rng.standard_normal(shape), device=dev, requires_grad=True)
        assert torch.autograd.gradcheck(lambda vv, bb: K.solve(vv, bb), (v, b))
        w = torch.tensor(rng.standard_normal(shape), device=dev)
        gv, gb = torch.autograd.grad((K.solve(v, b) * w).sum(), (v, b))
        rv_, rb_ = torch.autograd.grad((torch.linalg.solve(_dense(n, cp, rv, v), b) * w).sum(), (v, b))
        assert torch.allclose(gv, rv_, rtol=GRAD_TOL, atol=GRAD_TOL * rv_.abs().max().item())
        assert torch.allclose(gb, rb_, rtol=GRAD_TOL, atol=GRAD_TOL * rb_.abs().max().item())
    assert torch.autograd.gradcheck(lambda vv: K.slogdet(vv)[1], (v,))
    sign, lad = K.slogdet(v)
    sref, lref = torch.linalg.slogdet(_dense(n, cp, rv, v))
    assert sign.item() == sref.item() and abs(lad.item() - lref.item()) <= GRAD_TOL * abs(lref.item())
    (g,) = torch.autograd.grad(lad, v)
    (gref,) = torch.autograd.grad(lref, v)
    assert torch.allclose(g, gref, rtol=GRAD_TOL, atol=GRAD_TOL * gref.abs().max().item())
    K.close()


def test_factorisation_reuse():
    ag, dev = _ag(), _dev()
    n, cp, rv, nz, ds = _small("qd", seed=2)
    K = ag.SparseLDL(n, cp, rv, ds, device=0)
    b = torch.tensor(np.random.default_rng(4).standard_normal(n), device=dev)
    a = torch.tensor(nz, device=dev, requires_grad=True)
    K.solve(a, b).sum().backward()                        # forward + backward: one refactor
    assert K.refactors == 1
    K.slogdet(a.detach().clone())                          # the same values: no refactor
    assert K.refactors == 1
    K2 = ag.SparseLDL(n, cp, rv, ds, device=0)
    K2.solve(a, b)
    K2.slogdet(a)
    assert K2.refactors == 1                               # solve + slogdet on the same values: one refactor
    # forward(A), forward(B), backward(A): three refactors, and A's gradient is A's
    K3 = ag.SparseLDL(n, cp, rv, ds, device=0)
    A = torch.tensor(nz, device=dev, requires_grad=True)
    Bv = torch.tensor(nz * 1.5, device=dev, requires_grad=True)
    la = K3.slogdet(A)[1]
    xb = K3.solve(Bv, b)
    (ga,) = torch.autograd.grad(la, A)
    assert K3.refactors == 3
    (gref,) = torch.autograd.grad(torch.linalg.slogdet(_dense(n, cp, rv, A))[1], A)
    assert torch.allclose(ga, gref, rtol=GRAD_TOL, atol=GRAD_TOL * gref.abs().max().item())
    xb.sum().backward()                                    # B's backward refactors B again
    assert K3.refactors == 4
    for k in (K, K2, K3):
        k.close()


def test_layer_refuses_a_regularising_matrix():
    ag, dev = _ag(), _dev()
    sh = ldl_shapes.regularised("D", 0)
    K = ag.SparseLDL(sh.N, sh.cp, sh.rv, sh.ds, perm=sh.perm, device=0)
    with pytest.raises(RuntimeError, match="regularised"):
        K.solve(torch.tensor(sh.nz, device=dev), torch.ones(sh.N, dtype=torch.float64, device=dev))
    K.close()
