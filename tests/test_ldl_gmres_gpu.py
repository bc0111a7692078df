"""Solves preconditioned by the factor (CudaLDLSolver.solve_gmres / solve_gmres_dev, cldl_solve_gmres(_dev)): restarted
flexible GMRES against the handle's current values, with omega1 / omega2 restated in np.longdouble from the returned x
by the refined solves' tests (_restate).
(a) The shape matrices of tests/ldl_shapes.py, plain and D K D-scaled: converged, the analysis matches the restatement.
(b) Regularised factors: every REG_SITES matrix (one wrong-signed pivot replaced by +-delta) reaches the rounding
    floor in a few steps (K~^-1 K is the identity plus rank 1).
(c) Low-rank changes: values of r <= 4 columns scaled after the refactor, so far that the refined solve reports
    converged = 0; 2 r steps of FGMRES reach the rounding floor.
(d) The stale factors of the refined solves' tests: a 1e-6 relative change converges; after a 50 % change only what
    was measured is asserted.
(e) Forward error: ||x - x*||_inf / ||x*||_inf <= FERR_FAC ferr under error analysis.
(f) The C2 KKT matrix with its -H block scaled by (1 +- U(0, 0.1)) after the refactor.
Also: two calls give the same bits, the _dev form the host form's, the factor and a plain solve are unchanged; the
refusals; the ABI sizes and defaults.

Worst values measured on an H100 (SXM, 80 GB HBM3, 700 W power limit; the host-emulated build gives the same figures
to about one digit).  The thresholds keep a margin of at least 10x to the accuracy figures:
  |omega - omega*| 0.60 eps, resid_inf 0.56 eps
  At the rounding floor the call may end slightly above tol = eps: a short cycle there need not lower omega1 + omega2,
  and the call then stops (the stagnation rule).  So (b), (c), the 50 % case of (d) and (f) assert omega1 + omega2 <= FLOOR_TOL eps:
  (a) 1 step, converged
  (b) 3 or 4 steps in 2 or 3 cycles, omega1 + omega2 0.73 to 1.26 eps
  (c) after 2 r steps omega1 + omega2 <= 3.0 eps; the whole call 3 to 11 steps in 2 cycles, 0.70 to 2.2 eps; the
      refined solve reports converged = 0 on each
  (d) 1e-6: 3 steps; 50 %: 32 steps in 3 cycles to 0.76 eps, where refinement ends at 0.18
  (e) forward error / ferr 0.70
  (f) 14 steps in 4 cycles to 1.13 eps, where 10 refinement steps end at 5.1e-12"""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import clarabel_rs_b200 as cb
import ldl_shapes
from test_ldl_refine_gpu import _restate, _scaled, _solver
from test_selected_inverse_gpu import _factor_bytes, _inverse_reference, _sym

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
LD = np.longdouble
OMEGA_TOL = 16.0     # |omega - omega*| / eps
RESID_TOL = 64.0     # |resid_inf - resid_inf*| / (eps max(|K||x| + |b|))
FERR_FAC = 10.0
FLOOR_TOL = 32.0         # omega1 + omega2 in units of eps where the default tol = eps may not be reached


def _check(info, ref, what):
    e1, e2 = abs(info.omega1 - ref["omega1"]) / EPS, abs(info.omega2 - ref["omega2"]) / EPS
    er = abs(info.resid_inf - ref["resid_inf"]) / (EPS * ref["scale"])
    print("%s: |omega1 - ref| %.2f eps, |omega2 - ref| %.2f eps, resid %.2f eps (omega1 %.2e omega2 %.2e, %d steps, "
          "%d cycles, %d solves)" % (what, e1, e2, er, info.omega1, info.omega2, info.iterations, info.cycles,
                                     info.solves))
    assert e1 <= OMEGA_TOL and e2 <= OMEGA_TOL, (what, e1, e2)
    assert er <= RESID_TOL, (what, er)
    assert info.norm_x_inf == ref["norm_x_inf"]
    assert abs(info.norm_K_inf - ref["norm_K_inf"]) <= 1e-14 * ref["norm_K_inf"]
    den = info.norm_K_inf * info.norm_x_inf
    assert info.scaled_resid == (0.0 if info.resid_inf == 0.0 else info.resid_inf / den)
    assert info.converged == (info.omega1 + info.omega2 <= EPS)


def _with(sh, nz):
    return ldl_shapes.Shape(sh.name, sh.N, sh.cp, sh.rv, nz, sh.ds, sh.perm, sh.groups)


SHAPES = [f.__name__ for f in (ldl_shapes.big_fronts, ldl_shapes.child_records)]


# ---- (a) shapes ----
@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("name", SHAPES)
def test_shapes(name, scaled):
    sh, d = getattr(ldl_shapes, name)(), 1.0
    if scaled:
        sh, d = _scaled(sh)
    s = _solver(sh)
    assert s.refactor()
    K = _sym(sh)
    b = np.random.default_rng(5).standard_normal(sh.N) * d
    x0, i0 = s.solve_gmres(b, max_iter=0)
    _check(i0, _restate(K, x0, b), "%s x0" % sh.name)
    assert np.array_equal(x0.view(np.uint64), s.solve(b).view(np.uint64))
    assert i0.iterations == i0.cycles == 0 and i0.solves == 1 and i0.products == 1
    x, info = s.solve_gmres(b)
    _check(info, _restate(K, x, b), "%s gmres" % sh.name)
    assert info.converged and info.iterations <= 4 and info.solves == 1 + info.iterations
    assert info.products == info.iterations + info.cycles + 1
    s.close()


# ---- (b) regularised factors ----
@pytest.mark.parametrize("group,j", ldl_shapes.REG_SITES)
def test_regularised_factors(group, j):
    sh = ldl_shapes.regularised(group, j)
    s = _solver(sh)
    assert s.refactor()
    rc = s.linear_solver_info().regularize_count
    assert rc >= 1
    b = np.random.default_rng(8).standard_normal(sh.N)
    x, info = s.solve_gmres(b)
    _check(info, _restate(_sym(sh), x, b), "reg %s %d (regularised %d)" % (group, j, rc))
    assert info.omega1 + info.omega2 <= FLOOR_TOL * EPS
    assert info.iterations <= 4 * (rc + 1) and info.cycles <= 4
    s.close()


# ---- (c) low-rank value changes ----
def _change_columns(sh, r, seed):
    """sh's values with every stored entry of r random columns (of the upper triangle) scaled by a factor in +-[3, 6]:
    a symmetric change of rank <= 2 r"""
    rng = np.random.default_rng(seed)
    cols = rng.choice(sh.N, r, replace=False)
    nz = sh.nz.copy()
    for c in cols:
        nz[sh.cp[c]:sh.cp[c + 1]] *= rng.uniform(3, 6) * rng.choice([-1.0, 1.0])
    return nz


@pytest.mark.parametrize("r", [1, 2, 4])
@pytest.mark.parametrize("name", SHAPES)
def test_low_rank_changes(name, r):
    sh = getattr(ldl_shapes, name)()
    s = _solver(sh)
    assert s.refactor()
    nz = _change_columns(sh, r, seed=30 + r)
    s.update_values(np.arange(nz.size), nz)
    K = _sym(_with(sh, nz))
    b = np.random.default_rng(6).standard_normal(sh.N)
    _, ri = s.solve_refined(b)
    assert not ri.converged
    x1, i1 = s.solve_gmres(b, max_iter=2 * r)      # 2 r steps: a residual at rounding level
    _check(i1, _restate(K, x1, b), "%s, %d columns changed, %d steps" % (name, r, 2 * r))
    assert i1.omega1 + i1.omega2 <= FLOOR_TOL * EPS
    x, info = s.solve_gmres(b)
    _check(info, _restate(K, x, b), "%s, %d columns changed" % (name, r))
    assert info.omega1 + info.omega2 <= FLOOR_TOL * EPS and info.iterations <= 3 * r + 4 and info.cycles <= 4
    s.close()


# ---- (d) stale factors ----
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
    x, info = s.solve_gmres(b)
    _check(info, _restate(_sym(_with(sh, nz)), x, b), "stale 1e-6")
    assert info.converged and info.iterations <= 10
    nz = _perturbed(sh, 0.5, 4)
    s.update_values(idx, nz)
    _, i0 = s.solve_gmres(b, max_iter=0)
    _, ri = s.solve_refined(b)
    x, info = s.solve_gmres(b)
    _check(info, _restate(_sym(_with(sh, nz)), x, b), "stale 50%% (x0 omega %.1e, refined %.1e)"
           % (i0.omega1 + i0.omega2, ri.omega1 + ri.omega2))
    assert not ri.converged and ri.omega1 + ri.omega2 > 1e-3
    assert info.omega1 + info.omega2 <= FLOOR_TOL * EPS and info.iterations <= 100
    s.close()


# ---- (e) forward error ----
@pytest.mark.parametrize("which", ["big_fronts", "child_records", "reg_D_1", "changed"])
def test_forward_error(which):
    if which.startswith("reg"):
        sh = ldl_shapes.regularised("D", 1)
    else:
        sh = getattr(ldl_shapes, "child_records" if which == "changed" else which)()
    s = _solver(sh)
    assert s.refactor()
    if which == "changed":
        nz = _change_columns(sh, 2, seed=40)
        s.update_values(np.arange(nz.size), nz)
        sh = _with(sh, nz)
    K = _sym(sh)
    b = np.random.default_rng(7).standard_normal(sh.N)
    x, info = s.solve_gmres(b, error_analysis=True)
    ref = _restate(K, x, b)
    _check(info, ref, "ferr %s" % which)
    Z, _ = _inverse_reference(K)
    xs = Z @ b.astype(LD)
    fe = float(np.max(np.abs(x.astype(LD) - xs)) / np.max(np.abs(xs)))
    print("%s: forward error %.2e, ferr %.2e (%.3f), cond1 %.2e cond2 %.2e, %d solves"
          % (which, fe, info.ferr, fe / info.ferr, info.cond1, info.cond2, info.solves))
    assert fe <= FERR_FAC * info.ferr, (fe, info.ferr)
    assert info.ferr == info.omega1 * info.cond1 + info.omega2 * info.cond2 and info.cond1 > 0
    assert info.solves <= 1 + info.iterations + 2 * 11
    s.close()


# ---- (f) C2 ----
def test_c2_kkt_matrix_with_a_changed_h_block():
    from helpers import workloads
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    n = pr["P"].shape[0]
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    col = np.repeat(np.arange(N), np.diff(cp))
    nz[(rv == col) & (col < n)] += 1e-3
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=cb.ORDER_ND)
    assert s.refactor()
    hd = np.flatnonzero((rv == col) & (col >= n))            # the -H diagonal
    nz2 = nz.copy()
    nz2[hd] *= 1.0 + np.random.default_rng(3).uniform(-0.1, 0.1, hd.size)
    s.update_values(hd, nz2[hd])
    K = _sym(sp.csc_matrix((nz2, rv, cp), shape=(N, N)), N)
    b = np.random.default_rng(1).standard_normal(N)
    _, ri = s.solve_refined(b)
    x, info = s.solve_gmres(b)
    _check(info, _restate(K, x, b), "C2, -H scaled by 1 +- U(0, 0.1) (refined: %d steps, omega %.1e)"
           % (ri.steps, ri.omega1 + ri.omega2))
    assert info.omega1 + info.omega2 <= FLOOR_TOL * EPS
    assert ri.omega1 + ri.omega2 >= 1e3 * (info.omega1 + info.omega2)      # where refinement stalls
    s.close()


# ---- repeatability and side effects ----
def _dev():
    return torch.device("cpu") if os.environ.get("CLARABEL_EMU") == "1" else torch.device("cuda", 0)


def test_repeatable_dev_form_and_factor_unchanged():
    sh = ldl_shapes.child_records()
    s = _solver(sh)
    assert s.refactor()
    nz = _change_columns(sh, 2, seed=50)
    b = np.random.default_rng(3).standard_normal(sh.N)
    before = _factor_bytes(s)
    s.update_values(np.arange(nz.size), nz)
    xp = s.solve(b)
    x1, i1 = s.solve_gmres(b, error_analysis=True)
    x2, i2 = s.solve_gmres(b, error_analysis=True)
    assert np.array_equal(x1.view(np.uint64), x2.view(np.uint64)) and i1 == i2 and i1.iterations >= 2
    db = torch.tensor(b, device=_dev())
    dx = torch.empty_like(db)
    if db.is_cuda:
        torch.cuda.synchronize()
    i3 = s.solve_gmres_dev(dx.data_ptr(), db.data_ptr(), error_analysis=True)
    if db.is_cuda:
        torch.cuda.synchronize()
    assert np.array_equal(dx.cpu().numpy().view(np.uint64), x1.view(np.uint64)) and i3 == i1
    assert _factor_bytes(s) == before
    assert np.array_equal(s.solve(b).view(np.uint64), xp.view(np.uint64))
    vals = np.empty(nz.size)
    assert np.array_equal(_values(s, vals), nz)
    # refinement after the call: unchanged by it
    _, r1 = s.solve_refined(b)
    s.solve_gmres(b, restart=3)
    _, r2 = s.solve_refined(b)
    assert r1 == r2
    s.close()


def _values(s, out):
    """the handle's current values, read back from cldl_values_dev"""
    f = cb.lib().cldl_values_dev
    f.argtypes = [C.c_void_p]
    f.restype = C.c_void_p
    p = f(s._h)
    if os.environ.get("CLARABEL_EMU") == "1":
        C.memmove(out.ctypes.data, p, out.nbytes)
    else:
        torch.cuda.synchronize()
        t = torch.empty(out.size, dtype=torch.float64, device="cuda")
        cb.lib().cldl_copy_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        cb.lib().cldl_copy_dev(C.c_void_p(t.data_ptr()), C.c_void_p(p), out.nbytes)
        torch.cuda.synchronize()
        out[:] = t.cpu().numpy()
    return out


# ---- refusals and ABI ----
def _raw(s, restart=20, max_iter=100, tol=EPS):
    f = s._L.cldl_solve_gmres
    f.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(cb.pkg.cldl_gmres_opts),
                  C.POINTER(cb.pkg.cldl_gmres_info)]
    f.restype = C.c_int
    o = cb.pkg.cldl_gmres_opts()
    s._L.cldl_default_gmres_opts(C.byref(o))
    o.restart, o.max_iter, o.tol = restart, max_iter, tol
    x, b = np.zeros(s.n), np.ones(s.n)
    pd = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    return f(s._h, pd(x), pd(b), C.byref(o), None)


def test_refusals():
    sh = ldl_shapes.child_records()
    s = _solver(sh)
    assert _raw(s) == cb.CLDL_E_NOT_FACTORED
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.solve_gmres(np.zeros(sh.N))
    assert s.refactor()
    assert _raw(s) == cb.CLDL_OK and _raw(s, restart=512) == cb.CLDL_OK
    for kw in (dict(restart=0), dict(restart=-1), dict(restart=513), dict(max_iter=-1), dict(tol=-1.0),
               dict(tol=float("nan"))):
        assert _raw(s, **kw) == cb.CLDL_E_ARG, kw
    x, info = s.solve_gmres(np.zeros(sh.N), error_analysis=True)     # b = 0: x = 0, nothing to do
    assert not x.any() and info.omega1 == info.omega2 == info.cond1 == info.cond2 == 0.0 and info.converged
    assert info.iterations == 0
    s.close()
    # restart above n
    P = sp.diags([-np.ones(9), 2 * np.ones(10), -np.ones(9)], [-1, 0, 1])
    Up = sp.csc_matrix(sp.triu(P))
    sp_ = cb.CudaLDLSolver(10, Up.indptr, Up.indices, Up.data, np.ones(10, np.int8))
    assert sp_.refactor()
    assert _raw(sp_, restart=10) == cb.CLDL_OK and _raw(sp_, restart=11) == cb.CLDL_E_ARG
    sp_.close()
    # null pivots: the path Laplacian, singular
    L = sp.diags([-np.ones(9), np.r_[1.0, 2 * np.ones(8), 1.0], -np.ones(9)], [-1, 0, 1])
    Ul = sp.csc_matrix(sp.triu(L))
    sn = cb.CudaLDLSolver(10, Ul.indptr, Ul.indices, Ul.data, np.ones(10, np.int8), regularize_enable=False,
                          null_pivot_tol=1e-9)
    assert sn.refactor() and sn.inertia()[2] == 1
    assert _raw(sn) == cb.CLDL_E_ARG
    sn.close()
    # Schur and sharded handles
    big = ldl_shapes.big_fronts()
    sc = cb.CudaLDLSolver(big.N, big.cp, big.rv, big.nz, big.ds, perm=big.perm, schur=[int(big.groups["sep"][-1])])
    assert sc.refactor()
    assert _raw(sc) == cb.CLDL_E_ARG
    sc.close()
    ss = _solver(big, shard_nranks=2, shard_rank=0)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        ss.solve_gmres(np.zeros(big.N))
    ss.close()


def test_abi_sizes_and_defaults():
    L = cb.lib()
    out = np.zeros(2, np.uint64)
    L.cldl_gmres_abi_sizes.argtypes = [C.POINTER(C.c_uint64)]
    L.cldl_gmres_abi_sizes.restype = None
    L.cldl_gmres_abi_sizes(out.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert [int(v) for v in out] == [C.sizeof(cb.pkg.cldl_gmres_opts), C.sizeof(cb.pkg.cldl_gmres_info)]
    o = cb.pkg.cldl_gmres_opts()
    L.cldl_default_gmres_opts(C.byref(o))
    assert (o.restart, o.max_iter, o.tol, o.error_analysis) == (20, 100, EPS, 0)
