"""The KKT layer (solver.cu, KKTDevice) on the cone lists of tests/kkt_shapes.py, against the oracle run on the device's
permutation and against the extended-precision solve of the same module.

  values     after ckkt_update, class by class through the oracle's maps: P, A and the constant genpow diagonal bit for
             bit, the Hs blocks bit for bit equal to the negated ccone_get_Hs of the same handle, and every class within
             TOL of its largest entry of the oracle's values (LATE at the late points, where the cone kernels' own errors
             grow with the conditioning: test_cone_shapes_gpu.py, test_nonsym_shapes_gpu.py)
  restore    the static regularisation is undone: entries outside the Hs / expansion maps keep their bits, repeated
             updates give the same bits, and an update after another one gives the bits of a fresh handle's
  eps        with refinement off and eps ~ 1e-3 of the typical diagonal, ckkt_solve is (K + eps diag(dsigns))^-1 b with
             eps computed here from the oracle's diagonal (the diag-* lists put the largest |diagonal| in the last row,
             on either side of k_max_nonneg's grid-stride pass)
  refined    ckkt_solve's true residual against the handle's unregularised K and its forward error from the
             extended-precision solution, bounded by those of the reference's own refinement (kkt_shapes.refine) on the
             oracle's factor and values, before and after a second update at a new scaling (a stale refinement matrix
             shows there)
  settings   whole solves under the static regularisation and refinement settings, against the oracle: status,
             iterations and refactorisations equal, LDL solve counts within an eighth (see the test)
  paired     solve2 (the two systems of an iteration solved together) is bit for bit the unpaired path with extension
             rows present, at tolerances of 1e-15 where the refinements end on the ratio test
  non-finite an inf in the right-hand side makes ckkt_solve report failure, as the reference does"""
import functools

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import clarabel_rs_b200 as cb
import kkt_shapes as ks
import oracle

pytestmark = pytest.mark.gpu

TOL = 1e-12
LATE = 1e-9
EPS = float(np.finfo(np.float64).eps)
SOLVE = [(c.name, "opening") for c in ks.CASES if c.solve]
REFINE = SOLVE + [(name, "late") for name in ("soc-dense", "soc-sparse", "soc-5000")]


def make(name, perm=None, **kw):
    P, q, A, b = ks.problem(name)
    case = ks.BY_NAME[name]
    kw = dict(dict(equilibrate_enable=0), **kw)
    dev = cb.CudaSolver(P, q, A, b, case.cones, settings=cb.default_settings(**kw), kkt_perm=perm)
    ora = oracle.IPM(P, q, A, b, case.cones, settings=oracle.default_settings(**kw))
    ora.set_perm(dev.kkt_perm())
    return dev, ora


def scale(obj, name, regime, seed=0):
    if ks.BY_NAME[name].m == 0:
        return True
    s, z, mu = ks.point(name, regime, seed)
    if isinstance(obj, cb.CudaSolver):
        return obj.cone_update_scaling_ex(s, z, mu, cb.SCALING_PRIMAL_DUAL)
    return obj.update_scaling_ex(s, z, mu, 0)


def classes(ora, case):
    """{class: index array into the KKT values} from the oracle's maps"""
    out = {"P": ora.map("P"), "A": ora.map("A"), "Hs": ora.map("Hsblocks"), "diag": ora.map("diag_full")}
    nsp = sum(1 for k, d in case.cones if k == "soc" and d > ks.SOC_NO_EXPANSION_MAX_SIZE)
    ngp = sum(1 for k, _ in case.cones if k == "genpow")
    for w in ("u", "v", "D"):
        out["soc-" + w] = np.concatenate([ora.sparse_map(k, w) for k in range(nsp)] or [np.zeros(0, np.int64)])
    for w in ("q", "r", "p", "D"):
        out["gp-" + w] = np.concatenate([ora.genpow_map(k, w) for k in range(ngp)] or [np.zeros(0, np.int64)])
    return out


UPDATED = ["Hs", "soc-u", "soc-v", "soc-D", "gp-q", "gp-r", "gp-p", "gp-D"]


def rel(a, b):
    return float(np.max(np.abs(a - b), initial=0.0) / max(np.max(np.abs(b), initial=0.0), 1e-300))


@pytest.mark.parametrize("regime", ks.REGIMES)
@pytest.mark.parametrize("name", ks.NAMES)
def test_values_after_update(name, regime):
    case = ks.BY_NAME[name]
    dev, ora = make(name)
    assert scale(dev, name, regime) == scale(ora, name, regime)
    assert dev.kkt_update() == ora.kkt_update()
    got, want = dev.kkt_values(), ora.kkt()[3]
    cl = classes(ora, case)
    for c in ("P", "A"):
        assert np.array_equal(got[cl[c]], want[cl[c]]), c
    if case.m:
        assert np.array_equal(got[cl["Hs"]], -dev.cone_get_Hs()), "Hs scatter"
    const = np.abs(want[cl["gp-D"]]) == 1.0
    assert np.array_equal(got[cl["gp-D"]][const], want[cl["gp-D"]][const]), "genpow constant diagonal"
    tol = LATE if regime == "late" else TOL
    # a late SOC's residual z0^2 - |z1|^2 is 2e-6 z0^2: the rounding of |z1|^2 (summed in another order than the
    # oracle's) reaches w, eta, u and v amplified by 1e6
    dmax = max([d for k, d in case.cones if k == "soc"], default=0)
    soc_tol = max(tol, 4 * EPS * dmax / 1e-6) if regime == "late" else tol
    for c in ("Hs", "soc-u", "soc-v", "soc-D", "gp-q", "gp-r", "gp-p", "gp-D", "diag"):
        e = rel(got[cl[c]], want[cl[c]])
        assert e <= (soc_tol if c.startswith("soc") or c in ("Hs", "diag") else tol), f"{c}: {e:.3e} [{name}, {regime}]"
    rest = np.ones(got.size, bool)
    for c in cl.values():
        rest[c] = False
    assert np.array_equal(got[rest], want[rest])


@pytest.mark.parametrize("name", ks.NAMES)
def test_regularisation_is_undone(name):
    case = ks.BY_NAME[name]
    dev, ora = make(name)
    v0 = dev.kkt_values()
    cl = classes(ora, case)
    keep = np.ones(v0.size, bool)
    for c in UPDATED:
        keep[cl[c]] = False
    assert scale(dev, name, "opening")
    assert dev.kkt_update()
    v1 = dev.kkt_values()
    assert np.array_equal(v1[keep], v0[keep])
    assert dev.kkt_update() and dev.kkt_update()
    assert np.array_equal(dev.kkt_values(), v1)
    assert scale(dev, name, "late", seed=1)
    assert dev.kkt_update()
    fresh, _ = make(name, perm=dev.kkt_perm())
    assert scale(fresh, name, "late", seed=1)
    assert fresh.kkt_update()
    assert np.array_equal(dev.kkt_values(), fresh.kkt_values())


def rhs(case, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(case.n), rng.standard_normal(case.m)


def reference(ora, case, eps, b):
    N, cp, rv, nz, ds = ora.kkt()
    vals = ks.shifted(nz, ora.map("diag_full"), ds, eps) if eps else nz
    x, conv = ks.ext_solve(ks.full(N, cp, rv, vals), b)
    assert conv, "extended-precision reference did not converge"
    return x.astype(np.float64)


def ferr(x, xs, k):
    return float(np.max(np.abs(x[:k] - xs[:k]), initial=0.0))


@pytest.mark.parametrize("name,regime", SOLVE)
def test_eps_is_the_references(name, regime):
    case = ks.BY_NAME[name]
    base, ora = make(name)
    assert scale(ora, name, regime) and ora.kkt_update()
    N, cp, rv, nz, ds = ora.kkt()
    diag = np.abs(nz[ora.map("diag_full")])
    typical = float(np.median(diag[diag > 0])) if np.any(diag > 0) else 1.0
    prop = 1e-3 * typical / float(diag.max())
    st = dict(static_regularization_constant=0.0, static_regularization_proportional=prop,
              iterative_refinement_enable=0)
    dev, ora = make(name, perm=base.kkt_perm(), **st)
    assert scale(dev, name, regime) and scale(ora, name, regime)
    assert dev.kkt_update() and ora.kkt_update()
    rx, rz = rhs(case, 3)
    b = np.concatenate([rx, rz, np.zeros(case.p)])
    dev.kkt_setrhs(rx, rz)
    ok, x, z = dev.kkt_solve()
    assert ok
    eps = ks.regulariser(nz[ora.map("diag_full")], ora.settings)
    assert eps == prop * float(diag.max())
    xs = reference(ora, case, eps, b)
    r = ks.refine(N, cp, rv, nz, ds, ora.map("diag_full"), dev.kkt_perm(), ora.settings, b)
    k = case.n + case.m
    e_dev, e_ref = ferr(np.concatenate([x, z]), xs, k), ferr(r.x, xs, k)
    assert e_dev <= 10 * e_ref + 1e-13 * np.max(np.abs(xs[:k])), (e_dev, e_ref)


def true_residual(K, case, xm, b):
    """|b - K x|_inf in longdouble, the extension rows' unknowns solved from their own rows"""
    k = case.n + case.m
    x = np.zeros(K.shape[0])
    x[:k] = xm
    if case.p:
        Kee, Kem = K[k:, k:], K[k:, :k]
        x[k:] = spla.splu(sp.csc_matrix(Kee)).solve(-(Kem @ xm))
    return float(np.max(np.abs(ks.residual_ld(K, x, b))[:k], initial=0.0))


SETTINGS = {"defaults": {}, "constant-1e-4": dict(static_regularization_constant=1e-4)}


@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("name,regime", REFINE)
def test_refined_solve(name, regime, setting):
    case = ks.BY_NAME[name]
    dev, ora = make(name, **SETTINGS[setting])
    st = ora.settings
    for step, (reg, seed) in enumerate([(regime, 0), (regime, 1)]):
        assert scale(dev, name, reg, seed) and scale(ora, name, reg, seed)
        assert dev.kkt_update() and ora.kkt_update()
        N, cp, rv, nz, ds = ora.kkt()
        # the device's own unregularised K: at late SOC points its values differ from the oracle's (see above)
        K = ks.full(N, cp, rv, dev.kkt_values())
        rx, rz = rhs(case, 5 + step)
        b = np.concatenate([rx, rz, np.zeros(case.p)])
        dev.kkt_setrhs(rx, rz)
        ok, x, z = dev.kkt_solve()
        r = ks.refine(N, cp, rv, nz, ds, ora.map("diag_full"), dev.kkt_perm(), st, b)
        assert ok and r.ok
        k = case.n + case.m
        xd = np.concatenate([x, z])
        res_dev, res_ref = true_residual(K, case, xd, b), true_residual(ks.full(N, cp, rv, nz), case, r.x[:k], b)
        bound = max(st.iterative_refinement_abstol + st.iterative_refinement_reltol * np.max(np.abs(b)), 4 * res_ref)
        assert res_dev <= bound, f"update {step}: residual {res_dev:.3e} > {bound:.3e}"
        xs, conv = ks.ext_solve(K, b)
        xo, convo = ks.ext_solve(ks.full(N, cp, rv, nz), b)
        assert conv and convo
        e_dev, e_ref = ferr(xd, xs.astype(np.float64), k), ferr(r.x, xo.astype(np.float64), k)
        # where refinement stops on the ratio test the forward error is that of the last accepted step: 1e-12 |x*|
        assert e_dev <= 4 * e_ref + 1e-12 * np.max(np.abs(xo[:k])), f"update {step}: {e_dev:.3e} vs {e_ref:.3e}"


# ------------------------------------------------------------------------------------------------- whole solves
MIXES = ["soc-alternating", "psd-1-2-4", "zero+nonneg", "lp", "soc-sparse", "gp+soc", "all", "ns-1"]
SOLVE_SETTINGS = {
    "defaults": {},
    "static-off": dict(static_regularization_enable=0),
    "constant-1e-5": dict(static_regularization_constant=1e-5),
    "proportional-1e-7": dict(static_regularization_proportional=1e-7),
    "refinement-off": dict(iterative_refinement_enable=0),
    "max-iter-0": dict(iterative_refinement_max_iter=0),
    "max-iter-1": dict(iterative_refinement_max_iter=1),
    "stop-ratio-1.5": dict(iterative_refinement_stop_ratio=1.5, iterative_refinement_reltol=1e-15,
                           iterative_refinement_abstol=1e-15),
}


@functools.lru_cache(maxsize=None)
def solve_problem(name):
    """the case's P, q, A with b = an interior point of the cones: x = 0 is strictly feasible"""
    P, q, A, _ = ks.problem(name)
    s, _, _ = ks.point(name, "opening", seed=2)
    return P, q, A, s


# without refinement (or with one step) the libm noise of the nonsymmetric cones decides their final status
WEAK = ("refinement-off", "max-iter-0", "max-iter-1")
SOLVE_CASES = [(name, st) for name in MIXES for st in SOLVE_SETTINGS if ks.BY_NAME[name].symmetric or st not in WEAK]


@pytest.mark.parametrize("name,setting", SOLVE_CASES)
def test_solve_under_settings(name, setting):
    case = ks.BY_NAME[name]
    P, q, A, b = solve_problem(name)
    kw = SOLVE_SETTINGS[setting]
    dev = cb.CudaSolver(P, q, A, b, case.cones, settings=cb.default_settings(**kw) if kw else None)
    rd = dev.solve()
    ora = oracle.IPM(P, q, A, b, case.cones, settings=oracle.default_settings(**kw) if kw else None)
    ora.set_perm(dev.kkt_perm())
    ro = ora.solve()
    assert rd["status"] == ro["status"]
    if case.symmetric:
        assert rd["iterations"] == ro["iterations"]
        assert dev.info.n_refactor == ro["info"].n_refactor
        # a refinement that ends at the tolerance or on the ratio test decides on residual norms whose roundings differ
        # between the device's CSR gather and the oracle's symv: a step more or less in some of the solves (up to 7 in
        # 90 on the emulated build, whose contractions differ again)
        assert abs(int(dev.info.n_ldl_solve) - ro["info"].n_ldl_solve) <= max(3, ro["info"].n_ldl_solve // 8)
    else:       # libm noise may move the last iterations (test_zz_nonsym_gpu.py): the opening ones and the optimum
        k = min(4, len(dev.trace), len(ora.trace))
        assert np.allclose(dev.trace[:k, 0], ora.trace[:k, 0], rtol=1e-6, atol=0)
    if rd["status"] == "Solved":
        assert abs(rd["obj_val"] - ro["obj_val"]) <= 1e-6 * max(1.0, abs(ro["obj_val"]))


@pytest.mark.parametrize("name", ["soc-alternating", "gp+soc", "all", "soc5-x2000"])
def test_paired_solves_with_extension_rows(name, monkeypatch):
    case = ks.BY_NAME[name]
    assert case.p > 0
    P, q, A, b = solve_problem(name)
    st = dict(iterative_refinement_reltol=1e-15, iterative_refinement_abstol=1e-15, iterative_refinement_stop_ratio=1.5)
    monkeypatch.delenv("CB_NO_PAIRED_SOLVES", raising=False)
    a = cb.CudaSolver(P, q, A, b, case.cones, settings=cb.default_settings(**st))
    ra = a.solve()
    monkeypatch.setenv("CB_NO_PAIRED_SOLVES", "1")
    c = cb.CudaSolver(P, q, A, b, case.cones, settings=cb.default_settings(**st), kkt_perm=a.kkt_perm())
    rc = c.solve()
    assert ra["status"] == rc["status"] and ra["iterations"] == rc["iterations"]
    for key in ("x", "z", "s"):
        assert np.array_equal(ra[key], rc[key]), key
    assert a.info.n_ldl_solve == c.info.n_ldl_solve and a.info.n_refactor == c.info.n_refactor


@pytest.mark.parametrize("setting", ["defaults", "refinement-off"])
@pytest.mark.parametrize("name", ["soc-alternating", "gp+soc", "zero+nonneg"])
def test_nonfinite_rhs_is_reported(name, setting):
    case = ks.BY_NAME[name]
    dev, ora = make(name, **SOLVE_SETTINGS[setting])
    assert scale(dev, name, "opening") and scale(ora, name, "opening")
    assert dev.kkt_update() and ora.kkt_update()
    rx, rz = rhs(case, 7)
    rx[1] = np.inf
    dev.kkt_setrhs(rx, rz)
    ok, _, _ = dev.kkt_solve()
    N, cp, rv, nz, ds = ora.kkt()
    r = ks.refine(N, cp, rv, nz, ds, ora.map("diag_full"), dev.kkt_perm(), ora.settings,
                  np.concatenate([rx, rz, np.zeros(case.p)]))
    assert not ok and not r.ok
    rx[1] = 0.0                        # and the handle still solves a finite right-hand side afterwards
    dev.kkt_setrhs(rx, rz)
    assert dev.kkt_solve()[0]
