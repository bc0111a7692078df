"""The symmetric cone kernels (cones.cu: nonnegative, SOC; cones_psd.cu: PSD triangle) on the cone lists of
tests/cone_shapes.py, whose shapes sit where the kernels change launch geometry or code path, at the conditioning of
the first and of the last interior-point iterations, against the extended-precision reference of the same module.

Each error is printed as relative error / (eps * kappa), kappa a condition measure of the cone's point:
  PSD  kappa = |S| |Z| / lam_min^2, the first-order bound on the relative change of lambda^2 under a normwise
       perturbation of S or Z (about 60 for the opening points, 1e10 for the late ones)
  SOC  kappa = (|s0 z0| + sum |s1_i z1_i|) / |s'z|, the componentwise condition number of s'z = lam'lam, which NT
       scaling reproduces (about 1 for the opening points; late, about 1 .. 20 where s1 is not parallel to -z1, and
       1 / r for the SOC(2) cones, whose s1 = -z1 / 1024 makes s'z a difference of two nearly equal products).  The
       late points have |z1|, |s1| exact in double, so the margins r z0 of the given data are exact and kappa does
       not scale with 1 / r: a kernel that forms z0^2 - |z1|^2 by cancellation loses digits the measure shows.
  lambda   max_k |lam_k^2 - ref| / ref (PSD), |lam o lam - ref| / |ref| (SOC)
  H        max |Hs - H| / max |H| (PSD: every packed entry of skron(W_nt); SOC dense: 2ww' - J, sparse: the diagonal)
           and |mul_Hs(x) - H x| / (|H| |x|), over eps kappa_lam
  NT       |mul_Hs(z) - s| / |s| over eps kappa_lam
  shift    |(W^-T ds) o (W dz) - sigma mu e - shift| / |shift| over eps kappa_lam (PSD: in the device's eigenvector
           signs, read off the first row of its result)
  offset   |lambda o (W^-T out) - ds| with the reference lambda and W, in extended precision: over |ds| eps kappa (PSD),
           over (|lambda| |W^-T out| + |ds|) eps kappa (SOC: the normwise backward error; kappa for W's own error)
  step     |alpha - alpha*| / alpha* over eps kappa_lam, alpha* the exact bound; amax bit for bit when nothing binds
  margins  |min - ref| / max|eig| and |sum - ref| / sum of max|eig| over eps, where an SOC counts max(|z0|, |z1|)
           (its margin z0 - |z1| is one subtraction after an overflow-safe norm, rounded at that size)

  The near-amax directions sit 1e-9 (opening) and 1e-4 (late) below amax, above eps kappa.  For SOC `opposite`
  (y = -x / 2, a double root) the error is measured against sqrt(eps cond(b)), b = 2 (x0 y0 - x1'y1) the linear
  coefficient of the step quadratic.

Worst err / (eps kappa), PSD / SOC, opening and late together (margins over eps).  Host-emulated dense build
(tests/emu; every list up to PSD(57), the SOC dimensions 2..257; the full emulated build also runs PSD(64, 65), its
values were not recorded):
  lambda 1.2 / 1.6   H 1.0 / 1.6   NT 1.0 / 5.5   shift 12 / 5.0   offset 12 / 1.4   step 0.9 / 5.5   margins 50 / 0.1
On an H100 (SXM 80 GB, default power limit), every list (the SOC lambda and NT maxima are the 1e5-long cone):
  lambda 2.5 / 49    H 2.0 / 1.8   NT 2.0 / 23    shift 40 / 5.4   offset 40 / 1.4   step 2.3 / 6.2   margins 121 / 0.8
LIMIT keeps a margin of at least 100x to both."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp

import clarabel_rs_b200 as cb
import cone_shapes as cs
import mpmath as mp

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
REGIMES = ["opening", "late"]
SIGMAMU = 0.37e-3
LIMIT = dict(lam=5000.0, H=300.0, NT=5000.0, shift=5000.0, offset=5000.0, step=1000.0, margins=15000.0)
NEAR = dict(opening=1e-9, late=1e-4)     # gap below amax of the near-amax directions: above eps kappa_lam


@functools.lru_cache(maxsize=2)
def solver(name):
    case = cs.BY_NAME[name]
    m, n = case.m, 2
    A = sp.csc_matrix((np.ones(m), (np.arange(m), np.arange(m) % n)), shape=(m, n))
    return cb.CudaSolver(sp.identity(n, format="csc"), np.zeros(n), A, np.zeros(m), case.cones,
                         settings=cb.default_settings(equilibrate_enable=0))


@functools.lru_cache(maxsize=2)
def reference(name, regime):
    case = cs.BY_NAME[name]
    s, z = cs.interior(case, regime, seed=10 * cs.CASES.index(case) + REGIMES.index(regime))
    refs = []
    for (kind, d), sb, zb in zip(case.cones, cs.blocks(case, s), cs.blocks(case, z)):
        refs.append(cs.psd_reference(sb, zb, d) if kind == "psd" else cs.soc_reference(sb, zb) if kind == "soc" else None)
    return s, z, refs


def kappa(kind, ref, sb, zb):
    if kind == "psd":
        S, Z = cs.Ext(0).smat(sb, ref.n), cs.Ext(0).smat(zb, ref.n)
        return float(np.linalg.norm(S.astype(float), 2) * np.linalg.norm(Z.astype(float), 2) / ref.lam[-1] ** 2)
    return cs.soc_dot_cond(sb, zb)


def label(case, regime, k=None):
    kind, d = case.cones[k] if k is not None else (None, None)
    return f"[{case.name}: {case.reaches}; {case.row or ''}; regime {regime}" + (f"; cone {k} {kind}({d})]" if k is not None else "]")


def report(what, case, regime, k, val, kap):
    print(f"{what:8s} {case.name:14s} {regime:8s} cone {k:2d} err/(eps kappa) {val:9.2e}  kappa {kap:8.1e}")
    assert val <= LIMIT[what], f"{what} {val:.3e} > {LIMIT[what]} {label(case, regime, k)}"


SYM = [c.name for c in cs.PSD_CASES + cs.SOC_CASES]


def hs_offsets(case):
    out, o = [], 0
    for kind, d in case.cones:
        ln = d * (d + 1) // 2 * (d * (d + 1) // 2 + 1) // 2 if kind == "psd" else d * (d + 1) // 2 if (kind == "soc" and d <= 4) else d
        out.append((o, ln)); o += ln
    return out


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("name", SYM)
def test_scaling_lambda_and_H(name, regime):
    case = cs.BY_NAME[name]
    dev = solver(name)
    s, z, refs = reference(name, regime)
    assert dev.cone_update_scaling(s, z), label(case, regime)
    ds = dev.cone_affine_ds()
    Hs = dev.cone_get_Hs()
    x = np.random.default_rng(1).standard_normal(case.m)
    Hx, Hz = dev.cone_mul_Hs(x), dev.cone_mul_Hs(z)
    for k, ((kind, d), ref, (ho, hl)) in enumerate(zip(case.cones, refs, hs_offsets(case))):
        if kind == "nonneg":
            continue
        sb, zb = cs.blocks(case, s)[k], cs.blocks(case, z)[k]
        dsb, xb, Hxb, Hzb = (cs.blocks(case, v)[k] for v in (ds, x, Hx, Hz))
        kap = kappa(kind, ref, sb, zb)
        if kind == "psd":
            lam2 = dsb[[j * (j + 3) // 2 for j in range(d)]]
            err = np.max(np.abs(lam2 - ref.lam ** 2) / ref.lam ** 2)
            report("lam", case, regime, k, err / (EPS * kap), kap)
            report("H", case, regime, k, cs.skron_error(Hs[ho:ho + hl], ref.W) / (EPS * kap), kap)
            e = ref.ext
            Wx = e.f64(e.svec(e.arr(ref.W) @ e.smat(xb, d) @ e.arr(ref.W)))
            nW = np.linalg.norm(ref.W, 2)
            report("H", case, regime, k, np.max(np.abs(Hxb - Wx)) / (nW ** 2 * np.max(np.abs(xb))) / (EPS * kap), kap)
        else:
            l2 = [float(v) for v in cs.circ(ref.lam, ref.lam)]
            err = np.max(np.abs(dsb - l2)) / np.max(np.abs(l2))
            report("lam", case, regime, k, err / (EPS * kap), kap)
            e2, w = float(ref.eta ** 2), [float(v) for v in ref.w]
            if d <= 4:
                Href = np.array([e2 * (2 * w[r] * w[c] - (1 if r == c == 0 else -1 if r == c else 0))
                                 for c in range(d) for r in range(c + 1)])
            else:
                Href = np.array([e2 * 0.5 / float(cs._dot(ref.w, ref.w))] + [e2] * (d - 1))
            report("H", case, regime, k, np.max(np.abs(Hs[ho:ho + hl] - Href)) / np.max(np.abs(Href)) / (EPS * kap), kap)
            y = [float(v) for v in cs.soc_H(ref, xb)]
            nH = e2 * (w[0] + np.linalg.norm(w[1:])) ** 2
            report("H", case, regime, k, np.max(np.abs(Hxb - y)) / (nH * np.max(np.abs(xb))) / (EPS * kap), kap)
        report("NT", case, regime, k, np.max(np.abs(Hzb - sb)) / np.max(np.abs(sb)) / (EPS * kap), kap)
    # repeatability: the same call twice gives the same bits
    assert dev.cone_update_scaling(s, z)
    assert np.array_equal(dev.cone_affine_ds(), ds) and np.array_equal(dev.cone_get_Hs(), Hs), label(case, regime)
    assert np.array_equal(dev.cone_mul_Hs(x), Hx), label(case, regime)


def _align(shd, shr):
    """column signs D with shd = D shr D (D_0 = 1), from the largest-magnitude entry of each column"""
    n = shd.shape[0]
    D = np.ones(n)
    for j in range(1, n):
        i = int(np.argmax(np.abs(shr[:j, j])))
        D[j] = D[i] * np.sign(shd[i, j] * shr[i, j]) if shr[i, j] != 0 else 1.0
    return D


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("name", SYM)
def test_combined_shift_and_ds_offset(name, regime):
    case = cs.BY_NAME[name]
    dev = solver(name)
    s, z, refs = reference(name, regime)
    assert dev.cone_update_scaling(s, z), label(case, regime)
    rng = np.random.default_rng(2)
    dz, dsv = rng.standard_normal(case.m), rng.standard_normal(case.m)
    sh = dev.cone_combined_ds_shift(dz, dsv, SIGMAMU)
    assert np.array_equal(dev.cone_combined_ds_shift(dz, dsv, SIGMAMU), sh), label(case, regime)
    ds_in = sh.copy()
    out = dev.cone_ds_from_dz_offset(ds_in, z)
    assert np.array_equal(dev.cone_ds_from_dz_offset(ds_in, z), out), label(case, regime)
    for k, ((kind, d), ref) in enumerate(zip(case.cones, refs)):
        if kind == "nonneg":
            continue
        sb, zb = cs.blocks(case, s)[k], cs.blocks(case, z)[k]
        dzb, dsb, shb, ob, dib = (cs.blocks(case, v)[k] for v in (dz, dsv, sh, out, ds_in))
        kap = kappa(kind, ref, sb, zb)
        if kind == "psd":
            shr = cs.psd_shift(ref, dzb, dsb, SIGMAMU)
            e0 = cs.Ext(0)
            D = _align(e0.smat(shb, d).astype(float), e0.smat(shr, d).astype(float))
            shr_d = cs.svec(np.outer(D, D) * e0.smat(shr, d).astype(float))
            report("shift", case, regime, k, np.max(np.abs(shb - shr_d)) / np.max(np.abs(shr_d)) / (EPS * kap), kap)
            res = cs.psd_ds_residual(ref, ob, dib, D)
        else:
            a = cs.soc_W(ref, cs._m(dsb), inverse=True)
            b = cs.soc_W(ref, cs._m(dzb))
            shr = [float(v) for v in cs.circ(a, b)]
            shr[0] -= SIGMAMU
            report("shift", case, regime, k, np.max(np.abs(shb - shr)) / np.max(np.abs(shr)) / (EPS * kap), kap)
            # normwise backward error of lam o X = ds at X = W^-1 out: lam o . has the condition lam0^2 / det(lam),
            # about 1 / r at the late points, which a forward measure would have to carry
            X = cs.soc_W(ref, cs._m(ob), inverse=True)
            res = [float(v) for v in (np.array(cs.circ(ref.lam, X)) - np.array(cs._m(dib)))]
            den = float(max(abs(v) for v in ref.lam) * max(abs(v) for v in X)) + np.max(np.abs(dib))
            report("offset", case, regime, k, np.max(np.abs(res)) / den / (EPS * kap), kap)   # kap: W's own error
            continue
        report("offset", case, regime, k, np.max(np.abs(res)) / np.max(np.abs(dib)) / (EPS * kap), kap)


def _psd_dirs(rng, sb, d, gap):
    """(label, direction) for a PSD cone: inside (no bound), one negative generalised eigenvalue (bound 0.5), a random
    symmetric direction, and the one-negative direction scaled so that the bound is amax (1 - 1e-9), amax = 1"""
    X = cs.Ext(0).smat(sb, d).astype(float)
    G = rng.standard_normal((d, d))
    v = rng.standard_normal(d)
    t = 2.1 / (v @ np.linalg.solve(X, v))
    one = 0.1 * X - t * np.outer(v, v)
    out = [("inside", cs.svec(G @ G.T)), ("one-negative", cs.svec(one)), ("random", cs.svec((G + G.T) / 2))]
    out.append(("near-amax", cs.svec(one * (0.5 / (1 - gap)))))
    return out


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("name", SYM)
def test_step_length(name, regime):
    case = cs.BY_NAME[name]
    dev = solver(name)
    s, z, refs = reference(name, regime)
    assert dev.cone_update_scaling(s, z), label(case, regime)     # the PSD step works in the scaled frame
    rng = np.random.default_rng(3)
    o = 0
    for k, ((kind, d), ref) in enumerate(zip(case.cones, refs)):
        ne = cs.numel(kind, d)
        if kind == "nonneg":
            o += ne
            continue
        sb, zb = s[o:o + ne], z[o:o + ne]
        for side, xb in (("z", zb), ("s", sb)):
            dirs = _psd_dirs(rng, xb, d, NEAR[regime]) if kind == "psd" else cs.soc_directions(rng, xb, 1.0, NEAR[regime])
            for lab, y in dirs:
                for amax in (1.0, 1e6) if lab != "near-amax" else (1.0,):
                    dzv, dsv = np.zeros(case.m), np.zeros(case.m)
                    (dzv if side == "z" else dsv)[o:o + ne] = y
                    got = dev.cone_step_length(dzv, dsv, z, s, amax)
                    want = cs.psd_maxstep(ref, side, y, amax) if kind == "psd" else cs.soc_maxstep(xb, y, amax)
                    tag = f"{label(case, regime, k)} side {side} direction {lab} amax {amax}"
                    if lab == "inside":
                        assert want == amax and got == amax, f"{got!r} != amax {tag}"
                        continue
                    kap = kappa(kind, ref, sb, zb)
                    if lab == "opposite":     # a double root: the error is sqrt(eps cond(b)), b = 2 <x, J y>
                        kap = np.sqrt(cs.soc_dot_cond(xb, np.concatenate([y[:1], -y[1:]])) / EPS)
                    print(f"step     {case.name:14s} {regime:8s} cone {k:2d} {side} {lab:12s} {abs(got - want) / want / (EPS * kap):9.2e}")
                    assert abs(got - want) / want / (EPS * kap) <= LIMIT["step"], f"{got!r} vs {want!r} {tag}"
                    assert dev.cone_step_length(dzv, dsv, z, s, amax) == got, tag
        o += ne


def _margins_ref(case, z):
    mn, ps, scale, sscale = np.inf, 0.0, 0.0, 0.0
    for (kind, d), zb in zip(case.cones, cs.blocks(case, z)):
        if kind == "psd":
            ev = cs.psd_eig(zb, d)
        elif kind == "soc":
            ev = np.array([cs.soc_margin(zb)])
        else:
            ev = zb
        # an SOC margin z0 - |z1| is rounded at the size of z (scaled: |z1| of 1e200 entries overflows in numpy)
        sc = abs(zb[0]) * max(1.0, np.linalg.norm(zb[1:] / abs(zb[0]))) if kind == "soc" else np.max(np.abs(ev))
        mn, ps, scale, sscale = min(mn, ev.min()), ps + ev[ev > 0].sum(), max(scale, sc), sscale + sc
    return mn, ps, scale, sscale


@pytest.mark.parametrize("regime", REGIMES + ["indefinite"])
@pytest.mark.parametrize("name", SYM)
def test_margins(name, regime):
    case = cs.BY_NAME[name]
    dev = solver(name)
    if regime == "indefinite":
        z = np.random.default_rng(4).standard_normal(case.m)
    else:
        z = reference(name, regime)[1]
    mn, ps = dev.cone_margins(z)
    assert dev.cone_margins(z) == (mn, ps), label(case, regime)
    rmn, rps, scale, sscale = _margins_ref(case, z)
    e1, e2 = abs(mn - rmn) / scale / EPS, abs(ps - rps) / max(rps, sscale) / EPS
    print(f"margins  {case.name:14s} {regime:10s} min {e1:9.2e} sum {e2:9.2e}")
    assert e1 <= LIMIT["margins"] and e2 <= LIMIT["margins"], f"({mn!r}, {ps!r}) vs ({rmn!r}, {rps!r}) {label(case, regime)}"


@pytest.mark.parametrize("scale", [1e200, 1e-200])
def test_soc_margins_at_extreme_magnitudes(scale):
    """entries of 1e+-200: a plain sum of squares overflows to inf or underflows to 0, the Blue accumulators do not"""
    case = cs.SOC_CASES[0]
    dev = solver(case.name)
    z = np.concatenate([cs.soc_pair(np.random.default_rng(5), d, "late", k)[1] for k, (_, d) in enumerate(case.cones)])
    z = z * scale
    z[0] = -z[0]     # one cone outside: the minimum is negative
    mn, ps = dev.cone_margins(z)
    rmn, rps, sc, ssc = _margins_ref(case, z)
    assert np.isfinite(mn) and np.isfinite(ps), f"({mn!r}, {ps!r}) scale {scale:g} {label(case, 'late')}"
    e1, e2 = abs(mn - rmn) / sc / EPS, abs(ps - rps) / ssc / EPS
    print(f"margins  {case.name:14s} 1e{int(np.log10(scale)):+d}  min {e1:9.2e} sum {e2:9.2e}")
    assert e1 <= LIMIT["margins"] and e2 <= LIMIT["margins"], f"({mn!r}, {ps!r}) vs ({rmn!r}, {rps!r}) scale {scale:g}"


def test_soc_step_from_the_boundary():
    """x exactly on the boundary (c == 0 in socone.rs): a direction in the cone allows amax, one with a < 0 and b < 0
    (leaving at once) gives 0, both exact"""
    case = cs.SOC_CASES[0]
    dev = solver(case.name)
    z = np.concatenate([cs.on_boundary(d, 2.0) for _, d in case.cones])
    s = np.concatenate([cs.on_boundary(d, 2.0) + np.eye(d)[0] for _, d in case.cones])
    for k, (o, (_, d)) in enumerate(zip(np.cumsum([0] + [d for _, d in case.cones[:-1]]), case.cones)):
        for lab, y, want in (("in", np.eye(d)[0], 1e6), ("out", np.concatenate([[0.0], cs.on_boundary(d)[1:]]) if d > 2 else np.array([0.0, 1.0]), 0.0)):
            dzv = np.zeros(case.m)
            dzv[o:o + d] = y
            got = dev.cone_step_length(dzv, np.zeros(case.m), z, s, 1e6)
            assert got == want, f"{got!r} != {want!r} direction {lab} {label(case, 'boundary', k)}"


@pytest.mark.parametrize("name", [c.name for c in cs.NN_CASES])
def test_nonnegative_pass_boundaries(name):
    """one binding row at the end (past the first grid-stride pass for m > 75 776) and the margins; the ratio
    -z_i / dz_i is one correctly rounded division, so the step is exact to the bit"""
    case = cs.BY_NAME[name]
    dev = solver(name)
    m = case.m
    rng = np.random.default_rng(6)
    s, z = rng.uniform(0.5, 2.0, m), rng.uniform(0.5, 2.0, m)
    for i in sorted({m - 1, min(m - 1, cs.RED_BLOCKS * cs.RED_THREADS), 0}):
        dz = np.full(m, 0.1)
        dz[i] = -z[i] * 3.0 + 0.1
        want = -z[i] / dz[i]
        got = dev.cone_step_length(dz, np.zeros(m), z, s, 1e6)
        assert got == want, f"{got!r} != {want!r} row {i} {label(case, 'opening')}"
        assert dev.cone_step_length(np.full(m, 0.1), np.zeros(m), z, s, 1e6) == 1e6
    zz = rng.standard_normal(m)
    zz[-1] = -5.0
    mn, ps = dev.cone_margins(zz)
    assert mn == -5.0, f"{mn!r} {label(case, 'indefinite')}"
    ref = mp.fsum(float(v) for v in zz[zz > 0])
    assert abs(ps - float(ref)) / float(ref) <= 1e3 * EPS, f"{ps!r} vs {float(ref)!r} {label(case, 'indefinite')}"
