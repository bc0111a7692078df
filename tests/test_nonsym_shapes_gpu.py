"""The nonsymmetric cone kernels (cones_nonsym.cu: exponential, 3-D power, generalised power) on the cone lists of
tests/nonsym_shapes.py, at the opening, late (on the central path at mu = 1e-8, and off it by 1e-3) and edge points
of the same module, against its extended-precision reference.

Each error is err / (eps kappa), kappa = max(|s| |g(s)|, |z| |grad f*(z)|) / nu the condition measure of the cone's
point (1 at the unit initialisation, growing like 1 / margin near the boundary, as the primal gradient does):
  Hs       max |Hs - Hs*| / max |Hs*| (get_Hs, 3x3 packed; both strategies).  Where the primal-dual formula applies,
           kappa is multiplied by (|zt' H zt| + 3 mut^2) / |de2|, the cancellation in the denominator de2 of its
           rank-one correction (about 1e6 off the central path by 1e-3)
  secant   |mul_Hs(zt*) - st*| / |st*| with the exact g(s) = zt* and grad f*(z) = st*, and |mul_Hs(z) - s| / |s|
           (the primal-dual scaling satisfies both; mu H does on the central path): the primal gradient seen through Hs
  shift    |shift - (sigma mu grad f*(z) - eta)| / max(|sigma mu grad f*|, |eta|), eta the third-order correction;
           with kappa = cond(Hess f*(z)), which eta is solved with
  barrier  |sum - sum*| / sum over cones of (|f* + f| + kappa)
  step     the count J: the smallest j with a0 step^j exactly inside, or a neighbour when a0 step^j is within
           1000 eps kappa of the exact crossing alpha*; a0 bit for bit when nothing binds, 0 on a collapse

Worst err / (eps kappa) on an H100 (SXM 80 GB, default power limit), every list and regime:
  Hs 920   secant 1200   shift 3.7   barrier 9.4
The step counts were exact or within the stated band everywhere.
LIMIT keeps a margin of at least 100x."""
import functools

import mpmath as mp
import numpy as np
import pytest
import scipy.sparse as sp

import clarabel_rs_b200 as cb
import nonsym_shapes as ns

pytestmark = pytest.mark.gpu

EPS = ns.EPS
LIMIT = dict(Hs=1e5, secant=2e5, shift=5e3, barrier=1e3)
SIGMAMU = 0.37
NAMES = [c.name for c in ns.CASES]
SMALL = [c.name for c in ns.CASES if c.name != "ns-big"]


@functools.lru_cache(maxsize=2)
def solver(name):
    case = ns.BY_NAME[name]
    m, n = case.m, 2
    A = sp.csc_matrix((np.ones(m), (np.arange(m), np.arange(m) % n)), shape=(m, n))
    return cb.CudaSolver(sp.identity(n, format="csc"), np.zeros(n), A, np.zeros(m), case.cones,
                         settings=cb.default_settings(equilibrate_enable=0))


def _sym_point(kind, d, rng):
    if kind == "nonneg":
        return rng.uniform(0.5, 2, d), rng.uniform(0.5, 2, d)
    if kind == "soc":
        s, z = 0.3 * rng.standard_normal(d), 0.3 * rng.standard_normal(d)
        s[0], z[0] = 2.0, 2.0
        return s, z
    e = np.eye(d) * 2
    return ns_svec(e), ns_svec(e)


def ns_svec(M):
    n = M.shape[0]
    return np.array([M[r, c] if r == c else M[r, c] * np.sqrt(2.0) for c in range(n) for r in range(c + 1)])


@functools.lru_cache(maxsize=4)
def points(name, regime):
    """s, z (m-vectors), and per nonsymmetric / generalised power cone (kind, d, offset, s_k, z_k, mu_k)"""
    case = ns.BY_NAME[name]
    s, z = np.zeros(case.m), np.zeros(case.m)
    cones = []
    rng = np.random.default_rng(0)
    cnt = {}
    for (kind, d), o in zip(case.cones, case.offsets):
        r = ns.rows(kind, d)
        if kind in ("exp", "pow", "genpow"):
            k = cnt.get(kind, 0)
            cnt[kind] = k + 1
            sk, zk, mu = ns.point(case, k, kind, d, regime)
            cones.append((kind, d, o, sk, zk, mu))
        else:
            sk, zk = _sym_point(kind, d, rng)
        s[o:o + r], z[o:o + r] = sk, zk
    return s, z, cones


def report(what, name, regime, k, val, kap):
    assert val <= LIMIT[what], f"{what} {val:.3e} > {LIMIT[what]} [{name}, regime {regime}, cone {k}, kappa {kap:.2g}]"


def _mu(cones):
    return cones[0][5]


def _err(a, b):
    b = [mp.mpf(x) if not isinstance(x, mp.mpf) else x for x in b]
    return float(max(abs(mp.mpf(float(x)) - y) for x, y in zip(a, b)) / max(abs(y) for y in b))


def _hs_offsets(case):
    out, o = {}, 0
    for i, (kind, d) in enumerate(case.cones):
        r = ns.rows(kind, d)
        out[i] = o
        o += r * (r + 1) // 2 if (kind in ("exp", "pow", "psd") or (kind == "soc" and r <= 4)) else r
    return out


def _check_every(name, cones):
    """the long list repeats its points with period 37: the reference of one period stands for all"""
    if ns.BY_NAME[name].period:
        return [c for i, c in enumerate(cones) if i < 2 * ns.BY_NAME[name].period or i >= len(cones) - 40]
    return cones


@pytest.mark.parametrize("strategy", [cb.SCALING_PRIMAL_DUAL, cb.SCALING_DUAL], ids=["primal-dual", "dual"])
@pytest.mark.parametrize("regime", ns.REGIMES)
@pytest.mark.parametrize("name", NAMES)
def test_update_scaling_Hs_and_secant(name, regime, strategy):
    case = ns.BY_NAME[name]
    dev = solver(name)
    s, z, cones = points(name, regime)
    mu = _mu(cones)
    if regime == "edge" and any(c[5] != mu for c in cones):
        pytest.skip("one mu per call")
    assert dev.cone_update_scaling_ex(s, z, mu, strategy), name
    Hs = dev.cone_get_Hs()
    hoff = _hs_offsets(case)
    zt_all, st_all = np.zeros(case.m), np.zeros(case.m)
    refs = []
    idx = {o: i for i, o in enumerate(case.offsets)}
    worst = dict(Hs=0.0, secant=0.0)
    for kind, d, o, sk, zk, _ in cones:
        r = ns.ref(kind, d, sk, zk)
        refs.append((kind, d, o, r))
        n = ns.rows(kind, d)
        zt_all[o:o + n] = [float(v) for v in r.zt]
        st_all[o:o + n] = [float(v) for v in r.st]
    y1, y2 = dev.cone_mul_Hs(zt_all), dev.cone_mul_Hs(z)
    for k, (kind, d, o, r) in enumerate(_check_every(name, refs)):
        n = ns.rows(kind, d)
        if kind != "genpow":
            kap = r.kappa
            if strategy == cb.SCALING_DUAL:
                Href = ns.packed(mu * r.H)
            else:
                H, c2 = ns.pd_Hs(r.s, r.z, r.st, r.zt, r.H, mp.mpf(mu))
                Href, kap = ns.packed(H), r.kappa * float(c2 or 1)
            b = hoff[idx[o]]
            e = _err(Hs[b:b + 6], Href) / (EPS * kap)
            if strategy == cb.SCALING_PRIMAL_DUAL and e > LIMIT["Hs"] / 100:
                # mu mut - 1 within eps kappa of its threshold sqrt(eps): either formula is a correct outcome
                de1 = mp.fsum(a * b for a, b in zip(r.s, r.z)) * mp.fsum(a * b for a, b in zip(r.st, r.zt)) / 9 - 1
                if abs(abs(de1) - ns.SQRT_EPS) <= 1e4 * EPS * r.kappa or abs(de1) <= 1e3 * ns.SQRT_EPS:
                    alt, c2a = (mu * r.H, None) if c2 is not None else ns.pd_Hs(r.s, r.z, r.st, r.zt, r.H, mp.mpf(mu), force=True)
                    ka = r.kappa * float(c2a or 1)
                    ea = _err(Hs[b:b + 6], ns.packed(alt)) / (EPS * ka)
                    if ea < e:
                        e, kap = ea, ka
            worst["Hs"] = max(worst["Hs"], e)
            report("Hs", name, regime, k, e, kap)
            if strategy == cb.SCALING_PRIMAL_DUAL:
                e1 = _err(y1[o:o + 3], r.st) / (EPS * kap)
                e2 = _err(y2[o:o + 3], r.s) / (EPS * kap)
                worst["secant"] = max(worst["secant"], e1, e2)
                report("secant", name, regime, k, max(e1, e2), kap)
        else:
            # dual scaling only: mul_Hs = mu Hess f*(z) x, Hess from differences of grad f*
            want = [mu * v for v in ns.hess_vec(kind, d, r.z, ns.M(zt_all[o:o + n]))]
            e = _err(y1[o:o + n], want) / (EPS * r.kappa)
            worst["Hs"] = max(worst["Hs"], e)
            report("Hs", name, regime, k, e, r.kappa)
    print(f"scaling  {name:8s} {regime:9s} strategy {strategy}: " + ", ".join(f"{a} {v:.2g}" for a, v in worst.items()))


@pytest.mark.parametrize("regime", ns.REGIMES)
@pytest.mark.parametrize("name", SMALL)
def test_combined_shift(name, regime):
    case = ns.BY_NAME[name]
    dev = solver(name)
    s, z, cones = points(name, regime)
    mu = _mu(cones)
    assert dev.cone_update_scaling_ex(s, z, mu, cb.SCALING_DUAL), name
    rng = np.random.default_rng(2)
    zero = np.zeros(case.m)
    sh0 = dev.cone_combined_ds_shift(zero, zero, SIGMAMU)
    dz = np.zeros(case.m)
    dsv = np.zeros(case.m)
    for kind, d, o, sk, zk, _ in cones:
        n = ns.rows(kind, d)
        dz[o:o + n] = 0.3 * rng.standard_normal(n) * np.abs(zk)
        dsv[o:o + n] = 0.3 * rng.standard_normal(n) * np.abs(sk)
    sh = dev.cone_combined_ds_shift(dz, dsv, SIGMAMU)
    worst = 0.0
    for k, (kind, d, o, sk, zk, _) in enumerate(cones):
        n = ns.rows(kind, d)
        r = ns.ref(kind, d, sk, zk)
        g = [SIGMAMU * v for v in r.st]
        e = _err(sh0[o:o + n], g) / (EPS * r.kappa)
        worst = max(worst, e)
        report("shift", name, regime, k, e, r.kappa)
        if kind != "genpow":
            eta = ns.eta(r, dsv[o:o + 3], dz[o:o + 3])
            want = [a - b for a, b in zip(g, eta)]
            scale = max(max(abs(v) for v in g), max(abs(v) for v in eta))
            # eta goes through a solve with Hess f*(z): its condition number is the measure here
            ch = float(np.linalg.cond(np.array([[float(r.H[i, j]) for j in range(3)] for i in range(3)])))
            e = float(max(abs(mp.mpf(float(x)) - y) for x, y in zip(sh[o:o + 3], want)) / scale) / (EPS * ch)
            worst = max(worst, e)
            report("shift", name, regime, k, e, ch)
    print(f"shift    {name:8s} {regime:9s} {worst:.2g}")


@pytest.mark.parametrize("regime", ns.REGIMES)
@pytest.mark.parametrize("name", NAMES)
def test_barrier(name, regime):
    case = ns.BY_NAME[name]
    dev = solver(name)
    s, z, cones = points(name, regime)
    dz, dsv = np.zeros(case.m), np.zeros(case.m)
    for k, (kind, d, o, sk, zk, _) in enumerate(cones):
        n = ns.rows(kind, d)
        u = (k % 37) / 37          # repeats with the points of the long list, whose reference is one period
        dz[o:o + n] = 1e-3 * (zk if kind == "exp" else np.abs(zk)) * u
        dsv[o:o + n] = 1e-3 * (sk if kind == "exp" else np.abs(sk)) * (1 - u)
    sym = [(kind, d, o) for (kind, d), o in zip(case.cones, case.offsets) if kind not in ("exp", "pow", "genpow")]
    for al in (0.0, 0.5):
        got = dev.cone_compute_barrier(z, s, dz, dsv, al)
        total, scale = mp.mpf(0), mp.mpf(0)
        memo = {}
        for kind, d, o, sk, zk, _ in cones:
            n = ns.rows(kind, d)
            key = (kind, str(d), sk.tobytes(), zk.tobytes(), dsv[o:o + n].tobytes(), dz[o:o + n].tobytes())
            if key not in memo:
                sa = [mp.mpf(float(a)) + al * mp.mpf(float(b)) for a, b in zip(sk, dsv[o:o + n])]
                za = [mp.mpf(float(a)) + al * mp.mpf(float(b)) for a, b in zip(zk, dz[o:o + n])]
                v = ns.fstar(kind, d, za) + ns.f_primal(kind, d, sa)
                memo[key] = (v, abs(v) + ns.ref(kind, d, sk, zk).kappa)
            total += memo[key][0]
            scale += memo[key][1]
        for kind, d, o in sym:
            n = ns.rows(kind, d)
            sa = [mp.mpf(float(a)) + al * mp.mpf(float(b)) for a, b in zip(s[o:o + n], dsv[o:o + n])]
            za = [mp.mpf(float(a)) + al * mp.mpf(float(b)) for a, b in zip(z[o:o + n], dz[o:o + n])]
            if kind == "nonneg":
                v = -mp.fsum(mp.log(a * b) for a, b in zip(sa, za))
            elif kind == "soc":
                q = lambda x: x[0] ** 2 - mp.fsum(t * t for t in x[1:])
                v = -mp.log(q(sa) * q(za)) / 2
            else:
                v = -mp.log(mp.det(_smat(sa, d))) - mp.log(mp.det(_smat(za, d)))
            total += v
            scale += abs(v) + 1
        e = float(abs(mp.mpf(got) - total) / scale) / EPS
        print(f"barrier  {name:8s} {regime:9s} alpha {al}: {e:.2g}")
        report("barrier", name, regime, -1, e, 1.0)


def _smat(x, n):
    A = mp.matrix(n, n)
    t = 0
    for c in range(n):
        for r in range(c + 1):
            A[r, c] = A[c, r] = x[t] if r == c else x[t] / mp.sqrt(2)
            t += 1
    return A


def _step_cones(name, cones):
    if ns.BY_NAME[name].period:
        return [0, len(cones) - 1] + [k for k in (ns.RED_BLOCKS * ns.RED_THREADS - 1, ns.RED_BLOCKS * ns.RED_THREADS) if k < len(cones)]
    if len(cones) <= 40:
        return list(range(len(cones)))
    return sorted({0, 1, 31, 32, 33, 63, 64, 127, 128, 129, len(cones) - 2, len(cones) - 1} & set(range(len(cones))))


@pytest.mark.parametrize("regime", ["opening", "late"])
@pytest.mark.parametrize("name", NAMES)
def test_step_length(name, regime):
    case = ns.BY_NAME[name]
    dev = solver(name)
    s, z, cones = points(name, regime)
    rng = np.random.default_rng(3)
    gap = dict(opening=1e-9, late=1e-4)[regime]
    amax = 0.61
    a0 = min(amax, 1 - ns.SQRT_EPS)
    for k in _step_cones(name, cones):
        kind, d, o, sk, zk, _ = cones[k]
        if kind == "genpow" and ns.rows(kind, d) > 60:
            continue        # the crossing search costs seconds per direction at 300 rows; dims 1..53 cover the loop
        n = ns.rows(kind, d)
        kap = ns.ref(kind, d, sk, zk).kappa
        for side, q in (("z", zk), ("s", sk)):
            for lab, y in ns.directions(kind, d, q, side == "z", rng, a0, gap):
                dzv, dsv = np.zeros(case.m), np.zeros(case.m)
                (dzv if side == "z" else dsv)[o:o + n] = y
                got = dev.cone_step_length(dzv, dsv, z, s, amax)
                tag = f"[{name}, regime {regime}, cone {k} {kind}({d}), side {side}, direction {lab}]"
                if lab == "inside":
                    assert got == a0, f"{got!r} != {a0!r} {tag}"
                    continue
                j = ns.exact_count(kind, d, q, y, side == "z", a0)
                want = 0.0 if j == ns.J_ZERO else ns.backtrack(a0, j)
                if got != want:
                    astar = ns.crossing(kind, d, q, y, side == "z")
                    near = min(abs(mp.mpf(ns.backtrack(a0, i)) - astar) / astar for i in (j - 1, j) if 0 <= i < ns.J_ZERO)
                    ok = (ns.backtrack(a0, j - 1), ns.backtrack(a0, j + 1)) if j < ns.J_ZERO else ()
                    assert got in ok and float(near) <= 1e3 * EPS * kap, \
                        f"{got!r} vs {want!r} (J = {j}, alpha* {mp.nstr(astar, 17)}) {tag}"
    # every cone moving at once: the composite count is the largest
    dzv = np.zeros(case.m)
    counts = []
    for kind, d, o, sk, zk, _ in cones[:40]:
        n = ns.rows(kind, d)
        y = -(1.5 + 0.5 * (len(counts) % 7)) * zk        # crossings at 1 / (1.5 .. 4.5)
        dzv[o:o + n] = y
        counts.append(ns.exact_count(kind, d, zk, y, True, a0))
    assert dev.cone_step_length(dzv, np.zeros(case.m), z, s, amax) == ns.backtrack(a0, max(counts)), name
