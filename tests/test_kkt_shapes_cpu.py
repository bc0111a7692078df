"""The cases and references of tests/kkt_shapes.py, without a device: the lists reach the shapes they are there for, the
longdouble solve agrees with mpmath, and the refinement restatement follows the reference's rules on the oracle's
factor."""
import mpmath as mp
import numpy as np
import pytest

import kkt_shapes as ks
import oracle


def test_every_case_is_well_formed():
    names = set()
    for c in ks.CASES:
        assert c.name not in names
        names.add(c.name)
        P, q, A, b = ks.problem(c.name)
        assert A.shape == (c.m, c.n) and P.shape == (c.n, c.n) and q.size == c.n and b.size == c.m
        assert np.all(np.diff(A.tocsr().indptr) > 0), f"{c.name}: a constraint row without entries"
        ora = oracle.IPM(P, q, A, b, c.cones, settings=oracle.default_settings(equilibrate_enable=0))
        assert ora.N == c.N, c.name
        nsp = sum(1 for k, d in c.cones if k == "soc" and d > ks.SOC_NO_EXPANSION_MAX_SIZE)
        ngp = sum(1 for k, _ in c.cones if k == "genpow")
        for k in range(nsp):
            assert ora.sparse_map(k, "u").size == ora.sparse_map(k, "v").size and ora.sparse_map(k, "D").size == 2
        for k in range(ngp):
            assert ora.genpow_map(k, "D").size == 3
        assert ora.map("diag_full").size == c.N
    # the shapes the lists are there for
    soc = {d for c in ks.CASES for k, d in c.cones if k == "soc"}
    assert {2, 3, 4, 5, 127, 128, 129, 257, 5000} <= soc
    psd = {d for c in ks.CASES for k, d in c.cones if k == "psd"}
    assert {1, 2, 4, 32, 33, 56, 57, 96} <= psd and max(psd) > ks.PSD_SMEM_MAX
    for cnt in (1, 127, 128, 129):
        assert f"ns-{cnt}" in ks.BY_NAME and f"gp-{cnt}-7x40" in ks.BY_NAME
    assert [c.N for c in ks.CASES if c.peak_last] == [ks.RED_PASS - 1, ks.RED_PASS, ks.RED_PASS + 1]
    alt = ks.BY_NAME["soc-alternating"].cones
    assert any(d <= 4 for _, d in alt[1:]) and alt[0][1] <= 4 < alt[1][1]
    gs = ks.BY_NAME["gp+soc"]
    assert gs.p > 3 * sum(1 for k, _ in gs.cones if k == "genpow")


@pytest.mark.parametrize("regime", ks.REGIMES)
@pytest.mark.parametrize("name", ["soc-alternating", "zero+nonneg", "all", "psd-1-2-4", "gp-1-2x1", "lp", "diag-75775"])
def test_points_are_interior(name, regime):
    case = ks.BY_NAME[name]
    s, z, mu = ks.point(name, regime)
    assert s.size == z.size == case.m and mu > 0
    o = 0
    for kind, d in case.cones:
        r = ks.rows(kind, d)
        sb, zb = s[o:o + r], z[o:o + r]
        if kind == "nonneg":
            assert np.all(sb > 0) and np.all(zb > 0)
        elif kind == "soc":
            assert sb[0] > np.linalg.norm(sb[1:]) and zb[0] > np.linalg.norm(zb[1:])
        elif kind == "psd":
            for v in (sb, zb):
                assert np.linalg.eigvalsh(ks.cs.Ext(0, use_mp=False).f64(ks.cs.Ext(0, use_mp=False).smat(v, d)))[0] > 0
        elif kind != "zero":
            dd = (tuple(d[0]), d[1]) if kind == "genpow" else d
            assert ks.ns.in_primal(kind, dd, sb) and ks.ns.in_dual(kind, dd, zb)
        o += r
    if case.peak_last:
        d = s / z
        assert np.argmax(d) == case.m - 1


def _small_kkt(name, regime):
    case = ks.BY_NAME[name]
    P, q, A, b = ks.problem(name)
    ora = oracle.IPM(P, q, A, b, case.cones, settings=oracle.default_settings(equilibrate_enable=0))
    ora.set_perm(np.arange(ora.N))
    if case.m:
        s, z, mu = ks.point(name, regime)
        assert ora.update_scaling_ex(s, z, mu, 0)
    assert ora.kkt_update()
    return case, ora


@pytest.mark.parametrize("name,regime", [("soc-dense", "opening"), ("soc-dense", "late"), ("psd-1-2-4", "opening"),
                                         ("zero+nonneg", "opening"), ("zero+nonneg", "late"), ("lp", "late")])
def test_ext_solve_against_mpmath(name, regime):
    case, ora = _small_kkt(name, regime)
    N, cp, rv, nz, ds = ora.kkt()
    K = ks.full(N, cp, rv, nz)
    b = np.concatenate([np.random.default_rng(1).standard_normal(case.n + case.m), np.zeros(case.p)])
    x, conv = ks.ext_solve(K, b)
    assert conv
    xh = x.astype(np.float64)
    xl = (x - xh.astype(ks.LD)).astype(np.float64)       # x = xh + xl exactly: a longdouble as two doubles
    with mp.workdps(60):
        xm = mp.lu_solve(mp.matrix(K.toarray().tolist()), mp.matrix(b.tolist()))
        err = max(abs(mp.mpf(float(xh[i])) + mp.mpf(float(xl[i])) - xm[i]) for i in range(N))
        big = max(abs(v) for v in xm)
    assert float(err / big) <= 2.0 ** -58


@pytest.mark.parametrize("name", ["soc-dense", "soc-alternating", "zero+nonneg", "all"])
def test_refinement_restatement_follows_the_reference(name):
    case, ora = _small_kkt(name, "opening")
    N, cp, rv, nz, ds = ora.kkt()
    diag = ora.map("diag_full")
    b = np.concatenate([np.random.default_rng(2).standard_normal(case.n + case.m), np.zeros(case.p)])
    perm = np.arange(N)
    st = oracle.default_settings(equilibrate_enable=0)
    r = ks.refine(N, cp, rv, nz, ds, diag, perm, st, b)
    assert r.ok and r.eps == st.static_regularization_constant + st.static_regularization_proportional * np.max(np.abs(nz[diag]))
    # the stopping rule: within tolerance, or a step that did not improve by stop_ratio
    K = ks.full(N, cp, rv, nz)
    e = np.max(np.abs(b - K @ r.x))
    tol = st.iterative_refinement_abstol + st.iterative_refinement_reltol * np.max(np.abs(b))
    assert e <= tol or r.n_solve - 1 == st.iterative_refinement_max_iter or \
        (len(r.steps) >= 1 and (len(r.steps) < 2 or r.steps[-2] / r.steps[-1] < st.iterative_refinement_stop_ratio))
    # no refinement: one solve with the regularised factor
    off = oracle.default_settings(equilibrate_enable=0, iterative_refinement_enable=0)
    r0 = ks.refine(N, cp, rv, nz, ds, diag, perm, off, b)
    assert r0.n_solve == 1
    f = oracle.QDLDL((N, N), cp, rv, ks.shifted(nz, diag, ds, r0.eps), perm, dsigns=ds,
                     regularize_eps=off.dynamic_regularization_eps, regularize_delta=off.dynamic_regularization_delta)
    assert np.array_equal(r0.x, f.solve(b))
    # refinement repairs the regularisation: its residual is below the plain solve's against the unregularised K
    big = oracle.default_settings(equilibrate_enable=0, static_regularization_constant=1e-4)
    rb = ks.refine(N, cp, rv, nz, ds, diag, perm, big, b)
    rb0 = ks.refine(N, cp, rv, nz, ds, diag, perm, oracle.default_settings(
        equilibrate_enable=0, static_regularization_constant=1e-4, iterative_refinement_enable=0), b)
    assert rb.n_solve > 1
    assert np.max(np.abs(b - K @ rb.x)) < 1e-3 * np.max(np.abs(b - K @ rb0.x))
