"""The cone lists of tests/cone_shapes.py reach every launch shape of the symmetric cone kernels, the extended-precision
reference there is right, and the CPU oracle (oracle/ipm_oracle.c, the parity target of the device cone tests) is as
accurate against it as the device is asked to be.  CPU only."""
import os
import re

import numpy as np
import pytest
import scipy.sparse as sp

import cone_shapes as cs
import oracle

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "clarabel.rs_b200", "csrc")
EPS = np.finfo(np.float64).eps


def _define(fname, name):
    src = open(os.path.join(CSRC, fname)).read()
    m = re.search(rf"(?:#define\s+{name}\s+|constexpr int {name} = )\(?([0-9 *]+)\)?", src)
    assert m, f"{name} not found in {fname}"
    return eval(m.group(1))


def test_shape_constants_are_the_kernels():
    """a change to the budget, the matrix count or the block sizes shows up here, and the lists must follow it"""
    assert _define("cones_psd.cu", "PSD_SMEM_BUDGET") == cs.PSD_SMEM_BUDGET
    assert _define("cones_psd.cu", "PSD_NMAT") == cs.PSD_NMAT
    assert _define("cones_psd.cu", "PSD_WARPS") == cs.PSD_WARPS
    assert _define("cones.cu", "SOC_NT") == cs.SOC_NT
    assert _define("vec.cuh", "RED_BLOCKS") == cs.RED_BLOCKS and _define("vec.cuh", "RED_THREADS") == cs.RED_THREADS
    assert _define("problem_setup.h", "CB_PSD_MAX_N") == cs.CB_PSD_MAX_N


def test_psd_warps_table():
    want = {28: 4, 29: 3, 32: 3, 33: 2, 40: 2, 41: 1, 56: 1, 57: 0, 128: 0}
    assert {n: cs.psd_warps(n) for n in want} == want


def test_every_shape_is_reached():
    rows = {}
    for c in cs.PSD_CASES:
        assert c.reaches.split(",")[0] == c.row or c.name in ("psd-mixed", "psd-partial"), c.name
        rows.setdefault(c.row, []).append(c.name)
    print("\n".join(f"{r:16s} {', '.join(v)}" for r, v in rows.items()))
    assert set(rows) == set(cs.PSD_ROWS)
    # rows per lane 1..4, up to the supported maximum
    assert {(n + 31) // 32 for c in cs.PSD_CASES for n in c.psd} == {1, 2, 3, 4}
    assert cs.CB_PSD_MAX_N in cs.BY_NAME["psd-n128"].psd
    assert {32, 64, 65, 96, 97} <= {n for c in cs.PSD_CASES for n in c.psd}
    # a CTA of cones of different sizes (shared-memory stride nmax), and a partly filled last CTA
    mixed = cs.BY_NAME["psd-mixed"].ctas()
    assert len(mixed) == 1 and len(set(mixed[0])) == len(mixed[0]) == 4 and cs.psd_warps(max(mixed[0])) == 4
    part = cs.BY_NAME["psd-partial"].ctas()
    assert len(part) == 2 and len(part[0]) == cs.PSD_WARPS and 0 < len(part[1]) < cs.PSD_WARPS
    # SOC: dense 2..4, sparse 5+, thread 0 alone on the second pass (129), three passes (257), a long reduction
    dims = {d for c in cs.SOC_CASES for k, d in c.cones if k == "soc"}
    assert {2, 3, 4, 5, cs.SOC_NT - 1, cs.SOC_NT, cs.SOC_NT + 1, cs.SOC_NT + 2, 2 * cs.SOC_NT + 1} <= dims
    assert max(dims) >= 100000
    # nonnegative: both sides of the second grid-stride pass
    ms = {c.m for c in cs.NN_CASES}
    P = cs.RED_BLOCKS * cs.RED_THREADS
    assert {P - 1, P, P + 1} <= ms and max(ms) > 3 * P


@pytest.mark.parametrize("n", [5, 20, 33])
@pytest.mark.parametrize("regime", ["opening", "late"])
def test_mpmath_and_longdouble_references_agree(n, regime):
    S, Z = cs.psd_pair(np.random.default_rng(n), n, regime)
    s, z = cs.svec(S), cs.svec(Z)
    a, b = cs.psd_reference(s, z, n, use_mp=True), cs.psd_reference(s, z, n, use_mp=False)
    # longdouble carries about 1e-19 * cond (measured: at most 0.2 of that late, for lambda, W and min eig(Z)), the
    # results are rounded to double: the device limits of test_cone_shapes_gpu.py sit many orders above this
    tol = 2 * EPS + 1e-19 * max(a.condS, a.condZ)
    assert np.max(np.abs(a.lam - b.lam) / a.lam) <= tol
    assert np.max(np.abs(a.W - b.W)) <= tol * np.max(np.abs(a.W))
    assert abs(a.zmin - b.zmin) <= tol * abs(a.zmin)


def test_commuting_points_and_the_identity():
    """S, Z diagonal in one basis: lambda_i = sqrt(sigma_i tau_i); S = Z = I: W = I and H = I"""
    n = 6
    sig, tau = np.array([1e-8, 1e-4, 0.5, 1.0, 3.0, 1e2]), np.array([2.0, 1e-3, 5.0, 7.0, 1e-6, 0.25])
    for use_mp in (True, False):
        r = cs.psd_reference(cs.svec(np.diag(sig)), cs.svec(np.diag(tau)), n, use_mp)
        want = np.sort(np.sqrt(sig * tau))[::-1]
        assert np.max(np.abs(r.lam - want) / want) <= 1e-15
        r = cs.psd_reference(cs.svec(np.eye(n)), cs.svec(np.eye(n)), n, use_mp)
        assert np.array_equal(r.W, np.eye(n)) and np.array_equal(r.lam, np.ones(n))
        N = n * (n + 1) // 2
        Hs = np.concatenate([np.eye(N)[:q + 1, q] for q in range(N)])
        assert cs.skron_error(Hs, r.W) <= 2 * EPS     # sqrt2 * sqrt2 / 2 rounds off the diagonal


@pytest.mark.parametrize("regime", ["opening", "late"])
def test_soc_reference_nt_identities(regime):
    """H z = s and W z = lambda = W^-1 s (the NT identities) hold to the reference's 50 digits"""
    rng = np.random.default_rng(7)
    for k, d in enumerate([2, 3, 5, 130]):
        s, z = cs.soc_pair(rng, d, regime, k)
        r = cs.soc_reference(s, z)
        assert max(abs(float(a) - b) for a, b in zip(cs.soc_H(r, z), s)) <= 1e-30 * max(abs(s))
        for a, b in zip(cs.soc_W(r, z), r.lam):
            assert abs(a - b) <= 1e-40 * abs(r.lam[0])
        for a, b in zip(cs.soc_W(r, cs._m(s), inverse=True), r.lam):
            assert abs(a - b) <= 1e-40 * abs(r.lam[0])
        if regime == "late":     # the margin is exact in double
            assert cs.soc_margin(z) == z[0] - np.sqrt(z[1:] @ z[1:])


ORACLE_CASES = ["psd-n28", "psd-n33x2", "psd-mixed", "soc-dims"]


@pytest.mark.parametrize("regime", ["opening", "late"])
@pytest.mark.parametrize("name", ORACLE_CASES)
def test_oracle_against_the_reference(name, regime):
    """the oracle's lambda, Hs and step length, measured like the device's in test_cone_shapes_gpu.py and held to the
    same limits"""
    import test_cone_shapes_gpu as g
    case = cs.BY_NAME[name]
    m, n = case.m, 2
    A = sp.csc_matrix((np.ones(m), (np.arange(m), np.arange(m) % n)), shape=(m, n))
    ora = oracle.IPM(sp.identity(n, format="csc"), np.zeros(n), A, np.zeros(m), case.cones,
                     settings=oracle.default_settings(equilibrate_enable=0))
    s, z, refs = g.reference(name, regime)
    assert ora.update_scaling(s, z)
    ds, Hs = ora.affine_ds(), ora.get_Hs()
    for k, ((kind, d), ref, (ho, hl)) in enumerate(zip(case.cones, refs, g.hs_offsets(case))):
        if kind == "nonneg":
            continue
        sb, zb = cs.blocks(case, s)[k], cs.blocks(case, z)[k]
        kap = g.kappa(kind, ref, sb, zb)
        if kind == "soc":
            # the oracle restates the reference's overflow-safe norm (vecmath.rs stable_norm), which rounds |x1| by a
            # few eps even where |x1| is exact; (x0 - |x1|)(x0 + |x1|) amplifies that by x0 / (x0 - |x1|).  The device
            # sums squares, exact on these points, and is held to kappa alone.
            kap *= max(x[0] / cs.soc_margin(x) for x in (sb, zb))
        dsb = cs.blocks(case, ds)[k]
        if kind == "psd":
            lam2 = dsb[[j * (j + 3) // 2 for j in range(d)]]
            g.report("lam", case, regime, k, np.max(np.abs(lam2 - ref.lam ** 2) / ref.lam ** 2) / (EPS * kap), kap)
            g.report("H", case, regime, k, cs.skron_error(Hs[ho:ho + hl], ref.W) / (EPS * kap), kap)
            y = cs.svec(np.random.default_rng(k).standard_normal((d, d)))
            y = cs.svec(0.1 * cs.Ext(0).smat(zb, d).astype(float)) - 2.0 * y / np.linalg.norm(y)
        else:
            l2 = [float(v) for v in cs.circ(ref.lam, ref.lam)]
            g.report("lam", case, regime, k, np.max(np.abs(dsb - l2)) / np.max(np.abs(l2)) / (EPS * kap), kap)
            y = cs.soc_directions(np.random.default_rng(k), zb, 1.0)[3][1]
        dz = np.zeros(m)
        dz[sum(cs.numel(*c) for c in case.cones[:k]):][:len(y)] = y
        got = ora.step_length(dz, np.zeros(m), z, s, 1e6)
        want = cs.psd_maxstep(ref, "z", y, 1e6) if kind == "psd" else cs.soc_maxstep(zb, y, 1e6)
        g.report("step", case, regime, k, abs(got - want) / want / (EPS * kap), kap)
