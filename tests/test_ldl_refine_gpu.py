"""Iterative refinement and error analysis of the multifrontal LDL^T (CudaLDLSolver.solve_refined / solve_refined_dev,
cldl_solve_refined(_dev)), against a restatement of the definitions of include/clarabel_b200.h in numpy, with the
residual and |K||x| summed in np.longdouble from the returned x:
    den1_i = (|K||x|)_i + |b_i|,  den2_i = (|K||x|)_i + ||K_i||_inf ||x||_inf,  tau_i = 1000 n eps (||K_i||_inf ||x||_inf + |b_i|),
    I1 = {den1 > tau}, I2 the rest, omega1 = max_I1 |r|/den1, omega2 = max_I2 |r|/den2 (0/0 counts 0).
(a) On the shape matrices of tests/ldl_shapes.py and on a badly scaled variant D K D (D from 1e-6 to 1e6): omega1,
omega2 (absolute difference in units of eps), resid_inf (in units of eps max(|K||x| + |b|)), ||K||_inf and ||x||_inf
match the restatement; the refined solve reaches omega1 + omega2 <= tol, and on the scaled variant the plain solve's
omega is larger (on every one of these, the plain solve's omega1 + omega2 is above the default tol = eps).
(b) Forward error: ||x - x*||_inf / ||x*||_inf, x* the longdouble-refined solution, is at most FERR_FAC ferr.
(c) cond1 / cond2 against || |K^-1| g ||_inf / ||x||_inf with K^-1 from the refined dense inverse: the estimate is not
above the exact value (to 1e-6 relative) and not below a tenth of it; a right-hand side with a zero block puts rows in
I2.
(d) max_iter = 0 returns the plain solve's bits, with its analysis.
(e) A stale factor: after a 1e-6 relative value change the refined solve converges while the plain solve's omega stays
near 1e-6; after a 50 % change it reports converged = 0 and returns an iterate no worse than x0.
(f) Regularised factors: the call terminates and its info is the restatement's.
(g) Long rows: an arrow matrix with a dense row of 1e5 entries, and the KKT matrix of the benchmark's C2.
Also: two calls give the same bits, the _dev form the host form's, and the factor and a plain solve are unchanged;
the refusals; the ABI sizes.

Worst values measured on an H100 (SXM, 80 GB HBM3, 700 W power limit; the host-emulated build gives the same figures to
two digits):
  (a), (e), (f), (g) |omega - omega*| 1.5 eps (regularised, F 4 / D 0 / D 8), 0.55 eps elsewhere; resid_inf 1.3 eps
  (b) forward error / ferr 0.72 (child_records, zero-block right-hand side)
  (c) estimate / exact: cond1 1.000 on every matrix, cond2 0.944 (big_fronts) and 0.973 (child_records)
  refined omega1 + omega2 0.36 to 0.97 eps after 1 to 3 steps; the plain solve's 1.5 to 3.1 eps
The thresholds keep a margin of at least 10x to these."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import clarabel_rs_b200 as cb
import ldl_shapes
from test_selected_inverse_gpu import _factor_bytes, _inverse_reference, _ld_matmul, _sym

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
LD = np.longdouble
OMEGA_TOL = 16.0     # (a), (f), (g): |omega - omega*| / eps
RESID_TOL = 64.0     # |resid_inf - resid_inf*| / (eps max(|K||x| + |b|))
FERR_FAC = 10.0      # (b)


def _solver(sh, **kw):
    return cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, **kw)


def _scaled(sh, seed=9):
    """(D K D, D) with D a random permutation of logspace(-6, 6)"""
    d = np.random.default_rng(seed).permutation(np.logspace(-6, 6, sh.N))
    cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
    return ldl_shapes.Shape(sh.name + "_scaled", sh.N, sh.cp, sh.rv, sh.nz * d[sh.rv] * d[cols], sh.ds, sh.perm,
                            sh.groups), d


def _restate(K, x, b):
    """the analysis of x for K (symmetric CSR, float64 values) and b, the header's definitions; sums in longdouble"""
    n = K.shape[0]
    absK = abs(K)
    r = b.astype(LD) - _ld_matmul(K, x[:, None])[:, 0]
    kx = _ld_matmul(absK, np.abs(x)[:, None])[:, 0]
    rmax = np.asarray(absK.max(axis=1).todense()).ravel()
    xn = float(np.max(np.abs(x)))
    ab = np.abs(b).astype(LD)
    den1 = kx + ab
    den2 = kx + LD(xn) * rmax
    tau = LD(1000.0 * n * EPS) * (rmax * LD(xn) + ab)
    in1 = den1 > tau
    ar = np.abs(r)
    o1 = float(np.max(ar[in1] / den1[in1])) if in1.any() else 0.0
    q = ~in1 & ((den2 != 0) | (ar != 0))
    o2 = float(np.max(ar[q] / den2[q])) if q.any() else 0.0
    return dict(omega1=o1, omega2=o2, resid_inf=float(np.max(ar)), norm_x_inf=xn, den1=den1, den2=den2, in1=in1,
                norm_K_inf=float(np.max(_ld_matmul(absK, np.ones((n, 1)))[:, 0])), scale=float(np.max(den1)))


def _check_info(info, ref, what):
    e1, e2 = abs(info.omega1 - ref["omega1"]) / EPS, abs(info.omega2 - ref["omega2"]) / EPS
    er = abs(info.resid_inf - ref["resid_inf"]) / (EPS * ref["scale"])
    print("%s: |omega1 - ref| %.2f eps, |omega2 - ref| %.2f eps, resid %.2f eps (omega1 %.2e omega2 %.2e, %d steps, "
          "%d solves)" % (what, e1, e2, er, info.omega1, info.omega2, info.steps, info.solves))
    assert e1 <= OMEGA_TOL and e2 <= OMEGA_TOL, (what, e1, e2)
    assert er <= RESID_TOL, (what, er)
    assert info.norm_x_inf == ref["norm_x_inf"]
    assert abs(info.norm_K_inf - ref["norm_K_inf"]) <= 1e-14 * ref["norm_K_inf"]
    den = info.norm_K_inf * info.norm_x_inf
    assert info.scaled_resid == (0.0 if info.resid_inf == 0.0 else info.resid_inf / den)
    return max(e1, e2)


SHAPES = [f.__name__ for f in (ldl_shapes.big_fronts, ldl_shapes.child_records)]


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("name", SHAPES)
def test_omega_is_what_it_claims(name, scaled):
    sh, d = getattr(ldl_shapes, name)(), 1.0
    if scaled:
        sh, d = _scaled(sh)
    s = _solver(sh)
    assert s.refactor()
    K = _sym(sh)
    b = np.random.default_rng(5).standard_normal(sh.N) * d      # scaled: the right-hand side D b of D K D
    x0, i0 = s.solve_refined(b, max_iter=0)
    _check_info(i0, _restate(K, x0, b), "%s plain" % sh.name)
    x, info = s.solve_refined(b)
    _check_info(info, _restate(K, x, b), "%s refined" % sh.name)
    assert info.converged and info.omega1 + info.omega2 <= EPS
    assert info.solves == 1 + info.steps
    assert i0.omega1 + i0.omega2 > EPS and info.steps >= 1     # the plain solve does not reach tol = eps
    s.close()


def _rhs_with_zero_block(sh, K, seed=6):
    """b = K x_t with x_t zero outside the first group: rows away from it get b_i = 0 and x_i ~ 0, so they fall in I2"""
    xt = np.zeros(sh.N)
    g = np.asarray(sh.groups[0] if isinstance(sh.groups, list) else next(iter(sh.groups.values())))
    xt[g] = np.random.default_rng(seed).standard_normal(g.size)
    return K @ xt


@pytest.mark.parametrize("rhs", ["random", "zero_block"])
@pytest.mark.parametrize("name", SHAPES)
def test_forward_error_and_condition_estimates(name, rhs):
    sh = getattr(ldl_shapes, name)()
    s = _solver(sh)
    assert s.refactor()
    K = _sym(sh)
    b = np.random.default_rng(7).standard_normal(sh.N) if rhs == "random" else _rhs_with_zero_block(sh, K)
    x, info = s.solve_refined(b, error_analysis=True)
    ref = _restate(K, x, b)
    _check_info(info, ref, "%s %s" % (name, rhs))
    Z, _ = _inverse_reference(K)
    xs = Z @ b.astype(LD)
    fe = float(np.max(np.abs(x.astype(LD) - xs)) / np.max(np.abs(xs)))
    absZ = np.abs(Z)
    xn = LD(ref["norm_x_inf"])
    exact = [float(np.max(absZ @ np.where(ref["in1"], ref["den1"], 0)) / xn),
             float(np.max(absZ @ np.where(ref["in1"], 0, ref["den2"])) / xn)]
    est = [info.cond1, info.cond2]
    print("%s %s: forward error %.2e, ferr %.2e; cond1 %.3e (exact %.3e), cond2 %.3e (exact %.3e), |I2| %d, %d solves"
          % (name, rhs, fe, info.ferr, est[0], exact[0], est[1], exact[1], int((~ref["in1"]).sum()), info.solves))
    assert fe <= FERR_FAC * info.ferr, (fe, info.ferr)
    assert info.ferr == info.omega1 * info.cond1 + info.omega2 * info.cond2
    for e, x_ in zip(est, exact):
        assert e <= x_ * (1 + 1e-6) and e >= x_ / 10, (e, x_)
    if rhs == "zero_block":
        assert (~ref["in1"]).any() and info.cond2 > 0
    else:
        assert info.cond2 == 0.0 and ref["in1"].all()
    assert info.solves <= 1 + info.steps + 2 * 11
    s.close()


def test_max_iter_zero_is_the_plain_solve():
    sh = ldl_shapes.child_records()
    s = _solver(sh)
    assert s.refactor()
    b = np.random.default_rng(1).standard_normal(sh.N)
    x, info = s.solve_refined(b, max_iter=0)
    assert np.array_equal(x.view(np.uint64), s.solve(b).view(np.uint64))
    assert info.steps == 0 and info.solves == 1 and info.cond1 == info.cond2 == info.ferr == 0.0
    _check_info(info, _restate(_sym(sh), x, b), "max_iter 0")
    assert info.converged == (info.omega1 + info.omega2 <= EPS)
    s.close()


def _perturbed(sh, rel, seed):
    return sh.nz * (1.0 + rel * np.random.default_rng(seed).uniform(-1, 1, sh.nz.size))


def test_stale_factor():
    sh = ldl_shapes.big_fronts()
    s = _solver(sh)
    assert s.refactor()
    b = np.random.default_rng(2).standard_normal(sh.N)
    idx = np.arange(sh.nz.size)
    nz = _perturbed(sh, 1e-6, 3)
    s.update_values(idx, nz)
    K = _sym(ldl_shapes.Shape(sh.name, sh.N, sh.cp, sh.rv, nz, sh.ds, sh.perm, sh.groups))
    x0, i0 = s.solve_refined(b, max_iter=0)
    _check_info(i0, _restate(K, x0, b), "stale 1e-6 plain")
    x, info = s.solve_refined(b)
    _check_info(info, _restate(K, x, b), "stale 1e-6 refined")
    assert 1e-9 <= i0.omega1 + i0.omega2 <= 1e-5
    assert info.converged and info.steps <= 10
    nz = _perturbed(sh, 0.5, 4)
    s.update_values(idx, nz)
    K = _sym(ldl_shapes.Shape(sh.name, sh.N, sh.cp, sh.rv, nz, sh.ds, sh.perm, sh.groups))
    x0, i0 = s.solve_refined(b, max_iter=0)
    x, info = s.solve_refined(b)
    _check_info(info, _restate(K, x, b), "stale 50% refined")
    assert not info.converged
    assert info.omega1 + info.omega2 <= i0.omega1 + i0.omega2
    s.close()


@pytest.mark.parametrize("group,j", ldl_shapes.REG_SITES)
def test_regularised_factors(group, j):
    sh = ldl_shapes.regularised(group, j)
    s = _solver(sh)
    assert s.refactor()
    assert s.linear_solver_info().regularize_count >= 1
    b = np.random.default_rng(8).standard_normal(sh.N)
    x, info = s.solve_refined(b, error_analysis=True)
    _check_info(info, _restate(_sym(sh), x, b), "reg %s %d" % (group, j))
    assert info.steps <= 10 and info.solves <= 1 + info.steps + 2 * 11
    assert np.isfinite(info.cond1) and info.cond1 >= 0 and info.converged == (info.omega1 + info.omega2 <= EPS)


def test_arrow_matrix_with_a_dense_row():
    n = 100_001
    rng = np.random.default_rng(4)
    a = rng.uniform(-1, 1, n - 1) / np.sqrt(n)
    cp = np.concatenate([np.arange(n), [2 * n - 1]]).astype(np.int64)
    rv = np.concatenate([np.arange(n - 1), np.arange(n)]).astype(np.int64)
    nz = np.concatenate([rng.uniform(1, 2, n - 1), a, [2.0 + np.sum(a * a)]])
    s = cb.CudaLDLSolver(n, cp, rv, nz, np.ones(n, np.int8))
    assert s.refactor()
    K = _sym(sp.csc_matrix((nz, rv, cp), shape=(n, n)), n)
    assert K.indptr[-1] - K.indptr[-2] == n
    b = rng.standard_normal(n)
    x, info = s.solve_refined(b)
    _check_info(info, _restate(K, x, b), "arrow")
    assert info.converged
    s.close()


def test_c2_kkt_matrix():
    from helpers import workloads
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=cb.ORDER_ND)
    assert s.refactor()
    K = _sym(sp.csc_matrix((nz, rv, cp), shape=(N, N)), N)
    b = np.random.default_rng(1).standard_normal(N)
    x, info = s.solve_refined(b)
    _check_info(info, _restate(K, x, b), "C2 (regularised %d)" % s.linear_solver_info().regularize_count)
    s.close()


def _dev():
    return torch.device("cpu") if os.environ.get("CLARABEL_EMU") == "1" else torch.device("cuda", 0)


def test_repeatable_dev_form_and_factor_unchanged():
    sh = ldl_shapes.big_fronts()
    s = _solver(sh)
    assert s.refactor()
    b = np.random.default_rng(3).standard_normal(sh.N)
    before, xp = _factor_bytes(s), s.solve(b)
    x1, i1 = s.solve_refined(b, error_analysis=True)
    x2, i2 = s.solve_refined(b, error_analysis=True)
    assert np.array_equal(x1.view(np.uint64), x2.view(np.uint64)) and i1 == i2
    db = torch.tensor(b, device=_dev())
    dx = torch.empty_like(db)
    if db.is_cuda:
        torch.cuda.synchronize()
    i3 = s.solve_refined_dev(dx.data_ptr(), db.data_ptr(), error_analysis=True)
    assert np.array_equal(dx.cpu().numpy().view(np.uint64), x1.view(np.uint64)) and i3 == i1
    assert _factor_bytes(s) == before
    assert np.array_equal(s.solve(b).view(np.uint64), xp.view(np.uint64))
    s.close()


def test_refusals():
    sh = ldl_shapes.child_records()
    z = np.zeros(sh.N)
    s = _solver(sh)
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.solve_refined(z)
    assert s.refactor()
    for kw in (dict(max_iter=-1), dict(tol=-1.0), dict(stop_ratio=0.5), dict(stop_ratio=float("nan"))):
        with pytest.raises(cb.BackendError, match="BadArgument"):
            s.solve_refined(z, **kw)
    x, info = s.solve_refined(z, error_analysis=True)       # b = 0: x = 0, nothing to refine or estimate
    assert not x.any() and info.omega1 == info.omega2 == info.cond1 == info.cond2 == 0.0 and info.converged
    s.close()
    t = _solver(sh, shard_nranks=2, shard_rank=0)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        t.solve_refined(z)
    t.close()
    u = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, schur=[0, 1, 2])
    assert u.refactor()
    with pytest.raises(cb.BackendError, match="BadArgument"):
        u.solve_refined(z)
    u.close()


def test_abi_sizes():
    out = np.zeros(2, np.uint64)
    cb.lib().cldl_refine_abi_sizes(out.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert [int(v) for v in out] == [C.sizeof(cb.cldl_refine_opts), C.sizeof(cb.cldl_refine_info)]
