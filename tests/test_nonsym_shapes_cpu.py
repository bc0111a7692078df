"""The cone lists of tests/nonsym_shapes.py reach the launch shapes of the nonsymmetric cone kernels, the
extended-precision reference there is right, and the kernels' per-cone arithmetic -- compiled for the host by
tests/host_harness/ns3_host.cpp, the same __host__ __device__ bodies -- meets it.  CPU only.

Errors are in units of eps * kappa, kappa = max(|s| |g(s)|, |z| |grad f*(z)|) / nu: 1 at the unit initialisation,
growing like 1 / margin near the boundary.  Worst values of the host build (g++ -O2, x86-64): primal gradient 110
(exp, the Wright omega series near 1 + pi), 53 (pow), 16 (genpow); primal barrier 58.  LIMIT keeps a margin of at
least 100x."""
import os
import re

import mpmath as mp
import numpy as np
import pytest

import ctypes as C

import nonsym_shapes as ns
from test_nonsym_host import P, Pair, _glib, _lib, GPair

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "clarabel.rs_b200", "csrc")
EPS = ns.EPS
LIMIT = dict(grad=2e4, barrier=1e4)


def _src(f):
    return open(os.path.join(CSRC, f)).read()


def test_shape_constants_are_the_kernels():
    cu = _src("cones_nonsym.cu")
    for grid in ("NS_GRID", "GP_GRID"):
        m = re.search(rf"#define {grid} \(\(dev\.n(?:ns|gp) \+ (\d+)\) / (\d+)\)", cu)
        assert m and int(m.group(1)) + 1 == int(m.group(2)) == ns.NS_BLOCK, grid
    blocks = re.findall(r"<<<(?:NS|GP)_GRID, (\d+),", cu)
    assert len(blocks) >= 15 and set(blocks) == {str(ns.NS_BLOCK)}
    vec = _src("vec.cuh")
    for name, val in (("RED_BLOCKS", ns.RED_BLOCKS), ("RED_THREADS", ns.RED_THREADS)):
        assert re.search(rf"constexpr int {name} = {val};", vec), name
    cuh = _src("cones_nonsym.cuh")
    assert f"J_ZERO = 1 << {ns.J_ZERO.bit_length() - 1}" in cuh and "SQRT_EPS = 1.4901161193847656e-08" in cuh


def test_every_shape_is_reached():
    counts = {len(c.ns()) for c in ns.CASES}
    B = ns.NS_BLOCK
    assert {1, 31, 32, 33, B - 1, B, B + 1, 2 * B + 1} <= counts
    assert max(counts) > ns.RED_BLOCKS * ns.RED_THREADS
    for c in ns.CASES:      # exp and pow inside one warp wherever a warp holds more than one cone
        kinds = [k for _, k, _, _ in c.ns()]
        for w in range(0, len(kinds), 32):
            assert len(kinds[w:w + 32]) == 1 or {"exp", "pow"} <= set(kinds[w:w + 32]), c.name
    gp = [(len(d[0]), d[1]) for _, _, d, _ in ns.BY_NAME["gp-dims"].gp()]
    assert set(gp) == {(a, b) for a in (1, 2, 3, 8) for b in (1, 2, 50, 300)} and len(gp) <= ns.NS_BLOCK
    mixed = ns.BY_NAME["mixed"]
    offs = [o for _, _, _, o in mixed.ns() + mixed.gp()]
    assert any(b - a != 3 for a, b in zip(sorted(offs), sorted(offs)[1:]))
    assert {"nonneg", "soc", "psd"} <= {k for k, _ in mixed.cones}
    assert {d for c in ns.CASES for _, k, d, _ in c.ns() if k == "pow"} == set(ns.ALPHAS)


PTS = [("exp", 3), ("pow", 0.01), ("pow", 0.3), ("pow", 0.6), ("pow", 0.99), ("genpow", ([0.2, 0.3, 0.5], 3)),
       ("genpow", ([1.0], 2))]


def _points(kind, d, n=12):
    case = ns.BY_NAME["ns-33"]
    return [(reg, j) + ns.point(case, j, kind, d, reg)[:2] for reg in ns.REGIMES for j in range(n)]


@pytest.mark.parametrize("kind,d", PTS, ids=[f"{k}-{d}" for k, d in PTS])
def test_reference_gradient_and_conjugacy(kind, d):
    """grad f* against central differences of f*; -grad f*(-g(s)) = s to 40 digits"""
    for reg, j, s, z in _points(kind, d, 6):
        zm = ns.M(z)
        g = ns.grad_fstar(kind, d, zm)
        for i in range(len(z)):
            e = [mp.mpf(int(i == k)) * (abs(zm[i]) or max(abs(v) for v in zm)) for k in range(len(z))]
            fd = ns._jvp(lambda q: [ns.fstar(kind, d, q)], zm, e)[0] / e[i]
            assert abs(fd - g[i]) <= mp.mpf(10) ** -35 * max(abs(g[i]), abs(fstar_scale(kind, d, zm)) / abs(e[i])), (reg, j, i)
        sm = ns.M(s)
        back = [-v for v in ns.grad_fstar(kind, d, [-v for v in ns.grad_primal(kind, d, sm)])]
        assert max(abs(a - b) for a, b in zip(back, sm)) <= mp.mpf(10) ** -40 * max(abs(v) for v in sm), (reg, j)


def fstar_scale(kind, d, z):
    return max(abs(ns.fstar(kind, d, z)), 1)


def test_wright_omega_against_lambertw():
    """the harness's Wright omega (the device function) on both sides of 1 + pi, up to 1e9: 98 eps is the known
    worst near 4.135, where the series branch ends"""
    L = _lib()
    zs = sorted(set(ns.OMEGA_ARGS) | set(np.linspace(1.0, 4.2, 33)) | {1 + np.pi, np.nextafter(1 + np.pi, 0)})
    worst = 0.0
    for z in zs:
        w, r = L.ns3h_wright_omega(float(z)), ns.wright_omega(mp.mpf(float(z)))
        worst = max(worst, float(abs(w - r) / r) / EPS)
    print(f"wright omega worst {worst:.1f} eps")
    assert worst <= 300


def _harness_grad(kind, d, s):
    if kind == "genpow":
        pr = GPair([(kind, d)])
        g = np.zeros(pr.m)
        pr.L.gph_grad_primal(pr.h, P(np.array(s, float)), P(g))
        return g
    pr = Pair([(kind, d)])
    g = np.zeros(3)
    pr.L.ns3h_grad_primal(pr.h, P(np.array(s, float)), P(g))
    return g


@pytest.fixture(autouse=True, scope="module")
def _argtypes():
    L = _glib()
    for nm in ("ns3h_grad_primal", "gph_grad_primal"):
        getattr(L, nm).argtypes = [C.c_void_p, f64p, f64p]


f64p = C.POINTER(C.c_double)


@pytest.mark.parametrize("kind,d", PTS, ids=[f"{k}-{d}" for k, d in PTS])
def test_primal_gradient_and_barrier_of_the_kernel_bodies(kind, d):
    """the kernels' primal gradient (Wright omega / one-sided Newton) and the primal barrier built from it, at the
    opening, late and edge points: every alpha, tiny and near-boundary third components, phi over 1e+-8"""
    worst = dict(grad=0.0, barrier=0.0)
    for reg, j, s, z in _points(kind, d):
        r = ns.ref(kind, d, s, z)
        g = _harness_grad(kind, d, s)
        err = max(abs(mp.mpf(float(a)) - b) for a, b in zip(g, r.zt)) / max(abs(b) for b in r.zt)
        e = float(err) / (EPS * r.kappa)
        worst["grad"] = max(worst["grad"], e)
        assert e <= LIMIT["grad"], f"{kind}({d}) {reg} #{j}: g {list(g)} vs {[mp.nstr(v, 17) for v in r.zt]}, {e:.3g} eps kappa"
        fb = ns.f_primal(kind, d, ns.M(s))
        if kind == "genpow":
            pr = GPair([(kind, d)])
            b = pr.L.gph_barrier(pr.h, P(np.array(z, float)), P(np.array(s, float)), P(np.zeros(pr.m)), P(np.zeros(pr.m)), 0.0)
            b -= float(ns.fstar(kind, d, ns.M(z)))
        else:
            pr = Pair([(kind, d)])
            b = pr.L.ns3h_barrier(pr.h, P(np.array(z, float)), P(np.array(s, float)), P(np.zeros(3)), P(np.zeros(3)), 0.0)
            b -= float(ns.fstar(kind, d, ns.M(z)))
        e = float(abs(b - fb)) / (EPS * (abs(float(fb)) + r.kappa))
        worst["barrier"] = max(worst["barrier"], e)
        assert e <= LIMIT["barrier"], f"{kind}({d}) {reg} #{j}: f {b!r} vs {mp.nstr(fb, 17)}, {e:.3g}"
    print(f"{kind}({d}) worst err/(eps kappa): " + ", ".join(f"{k} {v:.2g}" for k, v in worst.items()))


def test_eta_sign_against_the_oracle():
    """the sign convention of the reference's third-order correction, fixed once at a well-conditioned point"""
    pr = Pair([("exp", 3), ("pow", 0.3)])
    rng = np.random.default_rng(5)
    z, s = pr.interior_point(rng, 0.05)
    mu = float(s @ z) / 6
    assert pr.ora.update_scaling_ex(s, z, mu, 1)
    dz, ds = 0.3 * rng.standard_normal(6), 0.3 * rng.standard_normal(6)
    sh = pr.ora.combined_ds_shift(dz, ds, 0.0)
    for k, (kind, d) in enumerate(pr.cones):
        o = 3 * k
        r = ns.ref(kind, d, s[o:o + 3], z[o:o + 3])
        eta = ns.eta(r, ds[o:o + 3], dz[o:o + 3])
        assert np.allclose(-sh[o:o + 3], [float(v) for v in eta], rtol=1e-10, atol=1e-12 * np.abs(sh).max())
