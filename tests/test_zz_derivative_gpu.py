"""Derivatives of the solution at the last solve (cipm_derivative / cipm_adjoint_derivative, CudaSolver.derivative /
adjoint_derivative, clarabel.rs_b200/autograd.py) against an independent dense reference, the exact active-set
derivative, central finite differences of the solver itself, and each other.  tests/test_derivative_cpu.py runs this
module against the CUDA-on-CPU emulated build."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import clarabel_rs_b200 as cb
import oracle
import ref_problems as rp
import test_oracle_nonsym as nonsym
from helpers import workloads
from test_oracle_psd import sdp_data

pytestmark = pytest.mark.gpu


def powcone_data():  # basic_powcone.rs:5-52
    n = 6
    A = sp.vstack([-sp.identity(n, format="csc"),
                   sp.csc_matrix(np.array([[1., 2., 0., 3., 0., 0.], [0., 0., 0., 0., 1., 0.]]))]).tocsc()
    return sp.csc_matrix((n, n)), np.array([0., 0., -1., 0., 0., -1.]), A, np.concatenate([np.zeros(n), [3., 1.]]), \
        [("pow", 0.6), ("pow", 0.1), ("zero", 2)]


def small_qp():
    pr = workloads.random_sparse_qp(n=40, m=80, nnz_per_row=3, seed=5, window=10)
    return pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"]


def socp_sparse():
    P, q, A, b, _ = rp.basic_socp()
    return P, q, A, b, [("nonneg", 3), ("soc", 6)]


PROBLEMS = {
    "basic_qp": rp.basic_qp, "basic_lp": rp.basic_lp, "basic_socp": rp.basic_socp, "basic_socp_sparse": socp_sparse,
    "hs35": rp.hs35,
    "basic_eq_constrained": lambda: (sp.identity(3, format="csc"), [0., 0., 0.], rp.eq_A1(), [2., 0.], [("zero", 2)]),
    "basic_sdp": sdp_data, "basic_expcone": nonsym.expcone_data, "basic_powcone": powcone_data,
    "basic_genpowcone": nonsym.genpow_data, "random_sparse_qp": small_qp,
}
NONSYM = ("basic_expcone", "basic_powcone", "basic_genpowcone")


def degree(cones):
    """nu of the product cone (the cones' degree())"""
    nu = 0
    for k, d in cones:
        nu += len(d[0]) + 1 if k == "genpow" else {"zero": 0, "nonneg": d, "soc": 1, "psd": d, "exp": 3, "pow": 3}[k]
    return nu


def solved(name, **st):
    P, q, A, b, cones = PROBLEMS[name]()
    dev = cb.CudaSolver(P, q, A, b, cones, cb.default_settings(**st))
    r = dev.solve()
    assert r["status"] in ("Solved", "AlmostSolved"), (name, r["status"])
    return (sp.csc_matrix(P), np.asarray(q, float), sp.csc_matrix(A), np.asarray(b, float), cones), dev, r


def patterns(P, A):
    Pt = sp.triu(P, format="csc"); Pt.sort_indices()
    A = sp.csc_matrix(A); A.sort_indices()
    return Pt, A


def random_direction(P, A, rng):
    Pt, A = patterns(P, A)
    return rng.standard_normal(Pt.nnz), rng.standard_normal(Pt.shape[0]), rng.standard_normal(A.nnz), \
        rng.standard_normal(A.shape[0])


def on_pattern(M, v):
    return sp.csc_matrix((v, M.indices, M.indptr), shape=M.shape)


def dense_K(data, r):
    """K = [P A'; A -H] in the caller's coordinates, H from the oracle's cones at the returned (s, z)"""
    P, q, A, b, cones = data
    x, z, s = r["x"], r["z"], r["s"]
    n, m = len(x), len(z)
    ora = oracle.IPM(P, q, A, b, cones)
    if any(k in ("exp", "pow", "genpow") for k, _ in cones):
        assert ora.update_scaling_ex(s, z, float(s @ z) / degree(cones), 1)
    else:
        assert ora.update_scaling(s, z)
    H = np.column_stack([ora.mul_Hs(np.eye(m)[k]) for k in range(m)]) if m else np.zeros((0, 0))
    Pt = sp.triu(P).toarray()
    Pf = Pt + np.triu(Pt, 1).T
    Ad = A.toarray()
    return np.block([[Pf, Ad.T], [Ad, -H]])


def dense_rhs(data, r, d):
    """[r1; r2] of the forward system in the caller's coordinates"""
    P, q, A, b, cones = data
    Pt, Ac = patterns(P, A)
    dP, dq, dA, db = d
    x, z = r["x"], r["z"]
    dPs = on_pattern(Pt, dP).toarray(); dPs = dPs + np.triu(dPs, 1).T
    dAm = on_pattern(Ac, dA).toarray()
    return np.concatenate([-dq - dPs @ x - dAm.T @ z, db - dAm @ x])


def refined_solve(K, rhs):
    """K y = rhs by LU with iterative refinement on extended-precision residuals: the reference is as accurate as K
    allows, so what remains of a difference is the device's"""
    Kl, rl = K.astype(np.longdouble), rhs.astype(np.longdouble)
    y = np.linalg.solve(K, rhs).astype(np.longdouble)
    for _ in range(6):
        y = y + np.linalg.solve(K, (rl - Kl @ y).astype(np.float64)).astype(np.longdouble)
    return y.astype(np.float64)


def backward_error(K, y, rhs):
    """componentwise (Oettli-Prager) backward error of y as a solution of K y = rhs: max_i |K y - rhs|_i / (|K||y| +
    |rhs|)_i.  Invariant to row and column scaling, so the cone scalings of 1e-9 and 1e9 at a solution do not loosen it;
    a wrong H on a row shows up in that row's own residual"""
    den = np.abs(K) @ np.abs(y) + np.abs(rhs)
    res = np.abs(K @ y - rhs)
    return float(np.max(np.where(den > 0, res / np.where(den > 0, den, 1.0), res), initial=0.0))


def last_bit_spread(data, r, make_rhs):
    """how far the dense reference moves when x, s and z change in their last bits: the part of a difference that no
    solver can remove, since the derivative is a function of a solution known to double precision only (about 1e-5 on
    basic_socp, where s and z sit on the cone's boundary; 1e-16 on the polyhedral problems)"""
    K, rhs = dense_K(data, r), make_rhs(r)
    ref = refined_solve(K, rhs)
    spread = 0.0
    for k in range(3):
        rng = np.random.default_rng(100 + k)
        rr = {key: r[key] * (1.0 + 4e-16 * rng.standard_normal(len(r[key]))) for key in ("x", "s", "z")}
        spread = max(spread, float(np.max(np.abs(refined_solve(dense_K(data, rr), make_rhs(rr)) - ref), initial=0.0)))
    return K, rhs, ref, spread


def near(got, ref, tol, spread):
    return float(np.max(np.abs(got - ref), initial=0.0)) <= tol * max(1.0, float(np.max(np.abs(ref), initial=0.0))) + \
        4.0 * spread


def close(a, b, tol):
    a, b = np.asarray(a), np.asarray(b)
    scale = max(1.0, float(np.max(np.abs(b), initial=0.0)))
    return float(np.max(np.abs(a - b), initial=0.0)) <= tol * scale


# basic_qp states x1 + x2 = 1 twice (x1 + x2 >= 1 and x1 + x2 <= 1, both active): its dual solution is not unique and
# the solution map has no derivative there (K is singular to working precision), so it is left out of the value
# checks; the adjoint identity, reproducibility and the refused states cover it
WELL_POSED = [k for k in PROBLEMS if k != "basic_qp"]


@pytest.mark.parametrize("name", WELL_POSED)
def test_matches_the_dense_reference(name):
    """the device derivative against K = [P A'; A -H] assembled with numpy in the caller's coordinates, with H from the
    oracle's cones at the returned (s, z): (i) the componentwise backward error of the device's solution in the dense
    system and (ii) the values dx, dz, ds and the adjoint's u = -dq, w = db against the dense solution, up to `tol` plus
    what last-bit changes of the solution move the reference by.  Against K with H scaled by 1.01 one of the two is
    checked to fail"""
    data, dev, r = solved(name)
    P, q, A, b, cones = data
    n, m = len(r["x"]), len(r["z"])
    tol = 1e-5 if name in NONSYM else 1e-6
    rng = np.random.default_rng(1)
    d = random_direction(P, A, rng)
    dx, dz, ds = dev.derivative(*d)
    y = np.concatenate([dx, dz])
    K, rhs, ref, spread = last_bit_spread(data, r, lambda rr: dense_rhs(data, rr, d))
    assert backward_error(K, y, rhs) <= tol, (name, backward_error(K, y, rhs))
    assert near(y, ref, tol, spread), (name, np.max(np.abs(y - ref)), spread)
    if m and np.any(K[n:, n:]):
        # (i) and (ii) together tell H from 1.01 H: (i) on diagonal scalings, where a row's residual is its own H entry
        # times dz; (ii) on dense cone blocks, where H dz cancels in the residual but moves the solution
        Kw = K.copy(); Kw[n:, n:] *= 1.01
        assert backward_error(Kw, y, rhs) > tol or not near(y, refined_solve(Kw, rhs), tol, spread), name
    assert near(ds, rhs[n:] - A @ ref[:n], tol, np.max(np.abs(A.toarray()), initial=0.0) * spread), name
    assert np.allclose(ds, rhs[n:] - A @ dx, rtol=0, atol=1e-12 * max(1.0, np.max(np.abs(rhs)), np.max(np.abs(dx))))
    # adjoint: K [u; v] = [gx - A' gs; gz], w = v + gs
    gx, gz, gs = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
    Ad = A.toarray()
    _, rhs_a, ref_a, spread_a = last_bit_spread(data, r, lambda rr: np.concatenate([gx - Ad.T @ gs, gz]))
    g = dev.adjoint_derivative(gx, gz, gs)
    u, w = -g["q"], g["b"]
    assert near(u, ref_a[:n], tol, spread_a), (name, np.max(np.abs(u - ref_a[:n])), spread_a)
    assert near(w, ref_a[n:] + gs, tol, spread_a), (name, np.max(np.abs(w - ref_a[n:] - gs)), spread_a)
    # the first block row, P u + A' w = gx, holds without the cancellation of v = w - gs
    top = np.concatenate([u, w])
    assert backward_error(K[:n], top, gx) <= tol, name
    # the pattern gradients from u, w and the solution
    Pt, Ac = patterns(P, A)
    ia = np.repeat(np.arange(Ac.shape[1]), np.diff(Ac.indptr))
    assert close(g["A"].data, -(r["z"][Ac.indices] * u[ia] + w[Ac.indices] * r["x"][ia]), 1e-14), name
    ip = np.repeat(np.arange(Pt.shape[1]), np.diff(Pt.indptr)) if Pt.nnz else np.zeros(0, int)
    i, j = Pt.indices, ip
    x = r["x"]
    refP = np.where(i == j, -u[i] * x[i], -(u[i] * x[j] + x[i] * u[j]))
    assert close(g["P"].data, refP, 1e-14), name


@pytest.mark.parametrize("name", ["hs35", "basic_lp"])
def test_matches_the_active_set_derivative(name):
    """strictly complementary LP / QP: the derivative of the solution map is that of the equality-constrained problem
    on the active rows"""
    data, dev, r = solved(name)
    P, q, A, b, cones = data
    x, z = r["x"], r["z"]
    n = len(x)
    act = z > r["s"]
    Pt, Ac = patterns(P, A)
    Pd = Pt.toarray(); Pd = Pd + np.triu(Pd, 1).T
    Aa = A.toarray()[act]
    ka = int(act.sum())
    K = np.block([[Pd, Aa.T], [Aa, np.zeros((ka, ka))]])
    rng = np.random.default_rng(2)
    for _ in range(3):
        d = random_direction(P, A, rng)
        dP, dq, dA, db = d
        dPs = on_pattern(Pt, dP).toarray(); dPs = dPs + np.triu(dPs, 1).T
        dAm = on_pattern(Ac, dA).toarray()
        r1 = -dq - dPs @ x - dAm.T @ z
        r2 = db - dAm @ x
        y = np.linalg.solve(K, np.concatenate([r1, r2[act]]))
        dx_ref = y[:n]
        dz_ref = np.zeros(len(z)); dz_ref[act] = y[n:]
        ds_ref = r2 - A.toarray() @ dx_ref
        dx, dz, ds = dev.derivative(*d)
        assert close(dx, dx_ref, 1e-6) and close(dz, dz_ref, 1e-6) and close(ds, ds_ref, 1e-6), name


TIGHT = dict(tol_gap_abs=1e-10, tol_gap_rel=1e-10, tol_feas=1e-10, tol_ktratio=1e-10)


@pytest.mark.parametrize("name", ["hs35", "basic_lp", "random_sparse_qp"])
def test_matches_central_finite_differences(name):
    """on polyhedral cones H = s/z row by row, whose limit does not depend on how centred the final iterate is, so the
    derivative is the solution map's (on second-order and PSD cones with s, z both on the boundary it is the derivative
    of the linearisation at the returned point, see include/clarabel_b200.h)"""
    data, dev, r = solved(name, **TIGHT)
    P, q, A, b, cones = data
    Pt, Ac = patterns(P, A)
    rng = np.random.default_rng(3)
    d = random_direction(P, A, rng)
    dx, dz, ds = dev.derivative(*d)
    eps = 1e-6
    other = cb.CudaSolver(P, q, A, b, cones, cb.default_settings(**TIGHT))
    sols = []
    for sg in (1.0, -1.0):
        other.update_data(P=Pt.data + sg * eps * d[0], q=q + sg * eps * d[1], A=Ac.data + sg * eps * d[2],
                          b=b + sg * eps * d[3])
        rr = other.solve()
        assert rr["status"] == "Solved"
        sols.append(rr)
    for key, got in (("x", dx), ("z", dz), ("s", ds)):
        fd = (sols[0][key] - sols[1][key]) / (2 * eps)
        assert close(got, fd, 1e-4), (name, key, np.max(np.abs(got - fd)))


def pair_products(dev, data, rng):
    P, q, A, b, cones = data
    Pt, Ac = patterns(P, A)
    d = random_direction(P, A, rng)
    n, m = P.shape[0], A.shape[0]
    g = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
    Jd = dev.derivative(*d)
    Jt = dev.adjoint_derivative(*g)
    terms_l = np.concatenate([g[k] * Jd[k] for k in range(3)])
    terms_r = np.concatenate([Jt["P"].data * d[0], Jt["q"] * d[1], Jt["A"].data * d[2], Jt["b"] * d[3]])
    return terms_l, terms_r


IDENTITY_TOL = {                 # measured on the H100 / on the emulated build (cond(K))
    "basic_socp": 3e-7,          # 8.4e-8 / 5.1e-8 (3.0e11)
    "basic_expcone": 5e-8,       # 9.1e-9 / 1.0e-8 (6.8e12)
    "basic_sdp": 3e-8,           # 7.1e-9 / 1.3e-10 (1.2e10)
    "basic_powcone": 5e-9,       # 3.3e-9 / 5.6e-9 (9.5e17; 1.3e-9 / 5.7e-10 at cond 6.2e8, where the solve ended
                                 # while the power cone's primal gradient stopped at its Newton start)
}
# the emulated build (another FMA contraction and libm than nvcc's) where it exceeds the device's bound
EMU_IDENTITY_TOL = {"basic_powcone": 2e-8}


@pytest.mark.parametrize("name", list(PROBLEMS))
def test_adjoint_is_the_transpose_of_the_forward_derivative(name):
    """<g, J d> = <J' g, d> to 1e-10 relative.  Each side is one refined solve with K, and on four problems K's
    condition number limits how far two solves can agree: fixed bounds 3 to 6 times the larger of the discrepancies
    measured on the H100 and on the emulated build.  The other seven problems, cond(K) up to 5e19 among them, hold
    1e-10 (measured <= 3.2e-16)"""
    data, dev, r = solved(name)
    rng = np.random.default_rng(4)
    tol = IDENTITY_TOL.get(name, 1e-10)
    if os.environ.get("CLARABEL_EMU") == "1":
        tol = EMU_IDENTITY_TOL.get(name, tol)
    for _ in range(2):
        tl, tr = pair_products(dev, data, rng)
        scale = max(np.abs(tl).sum(), np.abs(tr).sum())
        assert abs(tl.sum() - tr.sum()) <= tol * scale, (name, tl.sum(), tr.sum(), tol)


def snapshot(dev, r):
    i = r["info"]
    fields = [f for f, _ in cb.cipm_info._fields_ if f not in ("solve_time", "device_ms", "t_kkt_update", "t_kkt_solve",
                                                                  "t_scale_cones")]
    return r["x"].copy(), r["z"].copy(), r["s"].copy(), dev.trace.copy(), {f: getattr(i, f) for f in fields}


def counted_solve(dev):
    l0 = cb.launch_count()
    r = dev.solve()
    return r, cb.launch_count() - l0


@pytest.mark.parametrize("name", ["basic_socp", "basic_sdp", "basic_expcone", "random_sparse_qp"])
def test_solve_is_unchanged_by_a_derivative_in_between(name):
    data = PROBLEMS[name]()
    a, b_ = cb.CudaSolver(*data), cb.CudaSolver(*data)
    ra, la = counted_solve(a)
    rb, lb = counted_solve(b_)
    info_before = snapshot(a, ra)[4]
    n, m = a.n, a.m
    a.derivative(dq=np.ones(n), db=np.ones(m))
    a.adjoint_derivative(np.ones(n), np.ones(m), np.ones(m))
    info = cb.cipm_info()
    a._L.cipm_get_info(a._h, cb.pkg.C.byref(info))
    assert {f: getattr(info, f) for f in info_before} == info_before      # the calls leave the info alone
    ra2, la2 = counted_solve(a)
    rb2, lb2 = counted_solve(b_)
    sa, sb = snapshot(a, ra2), snapshot(b_, rb2)
    for u, v in zip(sa[:4], sb[:4]):
        assert np.array_equal(u, v), name
    assert sa[4] == sb[4]
    assert la == lb == la2 == lb2


@pytest.mark.parametrize("name", ["basic_qp", "basic_sdp", "basic_genpowcone", "random_sparse_qp"])
def test_identical_calls_give_identical_bits(name):
    data, dev, r = solved(name)
    rng = np.random.default_rng(5)
    d = random_direction(data[0], data[2], rng)
    g = rng.standard_normal(dev.n), rng.standard_normal(dev.m), rng.standard_normal(dev.m)
    f1, f2 = dev.derivative(*d), dev.derivative(*d)
    assert all(np.array_equal(u, v) for u, v in zip(f1, f2))
    a1, a2 = dev.adjoint_derivative(*g), dev.adjoint_derivative(*g)
    for k in ("P", "q", "A", "b"):
        u, v = (a1[k].data, a2[k].data) if k in "PA" else (a1[k], a2[k])
        assert np.array_equal(u, v), k


def refused(dev):
    with pytest.raises(cb.BackendError):
        dev.derivative(dq=np.ones(dev.n))
    with pytest.raises(cb.BackendError):
        dev.adjoint_derivative(np.ones(dev.n))


def test_refused_states_and_the_handle_stays_usable():
    P, q, A, b, cones = rp.basic_qp()
    dev = cb.CudaSolver(P, q, A, b, cones)
    refused(dev)                                          # before any solve
    assert dev.solve()["status"] == "Solved"
    d1 = dev.derivative(dq=np.ones(2))
    dev.update_data(q=[1., 1.])                           # same values, but new data
    refused(dev)
    assert dev.solve()["status"] == "Solved"
    assert all(np.array_equal(u, v) for u, v in zip(d1, dev.derivative(dq=np.ones(2))))
    # the KKT solver's own value updates: the handle's values through ckkt_update_P / ckkt_update_A, scaled like the
    # solver's copy (c D P D, E A D), so that the next solve is the same problem
    dd, ee, cc = dev.equilibration()
    Pt, Ac = patterns(sp.csc_matrix(P), sp.csc_matrix(A))
    ip = np.repeat(np.arange(Pt.shape[1]), np.diff(Pt.indptr))
    ia = np.repeat(np.arange(Ac.shape[1]), np.diff(Ac.indptr))
    Ps = np.ascontiguousarray(cc * dd[Pt.indices] * Pt.data * dd[ip])
    As = np.ascontiguousarray(ee[Ac.indices] * Ac.data * dd[ia])
    f64p = cb.pkg.C.POINTER(cb.pkg.C.c_double)
    for fn, v in ((dev._L.ckkt_update_P, Ps), (dev._L.ckkt_update_A, As)):
        assert fn(dev._h, v.ctypes.data_as(f64p)) == 0
        refused(dev)
        assert dev.solve()["status"] == "Solved"
        dev.derivative(dq=np.ones(2))
    bad = list(b); bad[0] = -10.0                         # x1 + x2 >= 10 and x1 + x2 <= 1
    inf = cb.CudaSolver(P, q, A, bad, cones)
    assert inf.solve()["status"] == "PrimalInfeasible"
    refused(inf)
    inf.update_data(b=b)
    assert inf.solve()["status"] == "Solved"
    inf.derivative(dq=np.ones(2))
    # a presolved problem: the row with an infinite bound was removed
    Pb, qb, Ab, bb, cb_ = rp.box_qp3()
    bb = list(bb); bb[3] = 1e30
    pre = cb.CudaSolver(Pb, qb, Ab, bb, cb_)
    assert pre.m_reduced == 5 and pre.solve()["status"] == "Solved"
    with pytest.raises(cb.BackendError, match="presolve"):
        pre.derivative(dq=np.ones(3))
    with pytest.raises(cb.BackendError, match="presolve"):
        pre.adjoint_derivative(np.ones(3))
    assert pre.solve()["status"] == "Solved"


def test_autograd_gradients_are_the_adjoint_derivative():
    torch = pytest.importorskip("torch")
    import clarabel_rs_b200_pkg.autograd as ag
    P, q, A, b, cones = rp.hs35()
    Pt, Ac = patterns(P, A)
    dev = cb.CudaSolver(P, q, A, b, cones, cb.default_settings(**TIGHT))
    t = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (Pt.data, q, Ac.data, b)]
    rng = np.random.default_rng(6)
    wx, wz, ws = (torch.tensor(rng.standard_normal(k), dtype=torch.float64) for k in (3, 4, 4))

    def loss(*args):
        x, z, s = ag.solve(dev, *args)
        return (x * wx).sum() + (z * wz).sum() + (s * ws).sum()
    L = loss(*t)
    L.backward()
    g = dev.adjoint_derivative(wx.numpy(), wz.numpy(), ws.numpy())
    for tt, ref in zip(t, (g["P"].data, g["q"], g["A"].data, g["b"])):
        assert np.array_equal(tt.grad.numpy(), ref)
    # one scalar loss against central differences along a random direction
    d = [rng.standard_normal(v.numel()) for v in t]
    eps = 1e-6
    with torch.no_grad():
        lp = loss(*[v + eps * torch.tensor(dd) for v, dd in zip(t, d)]).item()
        lm = loss(*[v - eps * torch.tensor(dd) for v, dd in zip(t, d)]).item()
    fd = (lp - lm) / (2 * eps)
    an = sum(float(tt.grad.numpy() @ dd) for tt, dd in zip(t, d))
    assert abs(fd - an) <= 1e-4 * max(1.0, abs(an)), (fd, an)
    # a later solve on the same handle makes the old graph's backward pass refuse
    L2 = loss(*t)
    dev.solve()
    with pytest.raises(RuntimeError):
        L2.backward()


def test_full_size_c2_adjoint_and_reproducibility():
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    data = (pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"])
    dev = cb.CudaSolver(*data)
    assert dev.solve()["status"] == "Solved"
    rng = np.random.default_rng(7)
    tl, tr = pair_products(dev, (sp.csc_matrix(pr["P"]), pr["q"], sp.csc_matrix(pr["A"]), pr["b"], pr["cones"]), rng)
    assert abs(tl.sum() - tr.sum()) <= 1e-10 * max(np.abs(tl).sum(), np.abs(tr).sum())
    g = rng.standard_normal(dev.n), rng.standard_normal(dev.m), rng.standard_normal(dev.m)
    a1, a2 = dev.adjoint_derivative(*g), dev.adjoint_derivative(*g)
    assert all(np.array_equal(a1[k].data if k in "PA" else a1[k], a2[k].data if k in "PA" else a2[k]) for k in "PqAb")
