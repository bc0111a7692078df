"""Cone lists at the launch shapes of the nonsymmetric cone kernels (cones_nonsym.cu: exponential, 3-D power and
generalised power cones), points in the regimes an interior-point solve passes through and at the edges of the
per-cone arithmetic, and an extended-precision reference for all of it.  No GPU: tests/test_nonsym_shapes_cpu.py
checks the shapes and the reference, tests/test_nonsym_shapes_gpu.py holds the device to it.

Shapes (the constants below restate cones_nonsym.cu / vec.cuh; the CPU test reads them back from the sources): every
kernel runs one thread per cone in NS_BLOCK-thread blocks; the step counts add a warp max and an atomicMax;
compute_barrier is a grid-stride sum over RED_BLOCKS x RED_THREADS threads, so cone 75 776 starts a second pass.

Reference, from the double inputs as given, in mpmath at 50 digits:
  f*, grad f*   closed form (exp: expcone.rs's dual barrier; pow = genpow with alpha = (a, 1 - a))
  Hess f*, D3   central differences of grad f* at 80 digits (not the hand-coded formulas of expcone.rs / powcone.rs)
  g(s)          the exact solution of -grad f*(-g) = s: Lambert W for the exponential cone, a bracketed root of the
                scalar equation  r (phi(x) - x^2) = 2x  (r = |w|) for the power cones
  f(s)          -f*(-g(s)) - nu
  Hs            nonsymmetric_common.rs:72-143 evaluated on the exact s, z, grad f*(z), g(s), Hess f*(z)
  eta           ETA_SIGN * 1/2 D3 f*(z)[Hess^-1 ds, dz]; the sign is fixed against the oracle by the CPU test
  alpha*        the exact crossing of q + alpha dq with the cone's boundary (bisection on the exact membership test)"""
import functools
from dataclasses import dataclass

import mpmath as mp
import numpy as np

mp.mp.dps = 50

NS_BLOCK = 128                        # cones_nonsym.cu: <<<(n + 127) / 128, 128>>>
RED_BLOCKS, RED_THREADS = 296, 256    # vec.cuh
EPS = float(np.finfo(np.float64).eps)
SQRT_EPS = 1.4901161193847656e-08
J_ZERO = 1 << 20
A_MIN, STEP = 1e-4, 0.8               # default min_terminate_step_length, linesearch_backtrack_step
ETA_SIGN = 1
ALPHAS = [0.01, 0.1, 0.3, 0.5, 0.6, 0.9, 0.99]
W_RATIOS = [0.0, 0.5 * EPS, 2 * EPS, 1e-12, 1e-9, 1e-6, 0.5, 1 - 1e-6]     # |s3| / sqrt(phi), |w| / sqrt(phi)
OMEGA_ARGS = [1.5, 4.0, 4.1, 4.14159, 4.2, 5.0, 30.0, 1e3, 1e6, 1e9]       # Wright omega arguments (series ends at 1 + pi)
MU_LATE = 1e-8
REGIMES = ["opening", "late", "late-off", "edge"]


# ------------------------------------------------------------------------------------------------------- cone lists
def rows(kind, d):
    return 3 if kind in ("exp", "pow") else len(d[0]) + d[1] if kind == "genpow" else d * (d + 1) // 2 if kind == "psd" else d


@dataclass
class Case:
    name: str
    cones: list
    reaches: str
    period: int = 0        # > 0: the points repeat with this period in the cone index (long lists)

    @property
    def m(self):
        return sum(rows(k, d) for k, d in self.cones)

    @property
    def offsets(self):
        return list(np.cumsum([0] + [rows(k, d) for k, d in self.cones])[:-1])

    def ns(self):
        """(index in case.cones, kind, param, row offset) of the exp / pow cones, in kernel order"""
        return [(i, k, d, o) for i, ((k, d), o) in enumerate(zip(self.cones, self.offsets)) if k in ("exp", "pow")]

    def gp(self):
        return [(i, k, d, o) for i, ((k, d), o) in enumerate(zip(self.cones, self.offsets)) if k == "genpow"]


def _interleaved(n):
    """exp and pow cones alternating, so every warp takes both branches; pow exponents cycle through ALPHAS"""
    return [("exp", 3) if k % 2 == 0 else ("pow", ALPHAS[(k // 2) % len(ALPHAS)]) for k in range(n)]


def _gp_alphas(d1, j):
    if d1 == 1:
        return [1.0]
    w = np.array([1.0 + ((j + 3 * i) % 5) for i in range(d1)])
    a = w / w.sum()
    a[-1] = 1.0 - a[:-1].sum()
    return [float(v) for v in a]


GP_DIMS = [(d1, d2) for d1 in (1, 2, 3, 8) for d2 in (1, 2, 50, 300)]
NS_COUNTS = [1, 31, 32, 33, 127, 128, 129, 257]
BIG = RED_BLOCKS * RED_THREADS + 24           # exp / pow cones: the barrier sum takes a second grid-stride pass
CASES = [Case(f"ns-{n}", _interleaved(n), f"{(n + NS_BLOCK - 1) // NS_BLOCK} block(s), {n % 32 or 32} lanes in the last warp")
         for n in NS_COUNTS]
CASES += [
    Case("gp-dims", [("genpow", (_gp_alphas(d1, j), d2)) for j, (d1, d2) in enumerate(GP_DIMS)],
         "dim1 1..8 x dim2 1..300 in one block"),
    Case("mixed", [("nonneg", 3), ("exp", 3), ("soc", 4), ("pow", 0.3), ("genpow", ([0.3, 0.7], 2)), ("psd", 3),
                   ("exp", 3), ("soc", 7), ("pow", 0.9), ("nonneg", 1), ("genpow", ([0.2, 0.3, 0.5], 3)), ("exp", 3)],
         "offsets interleaved with nonnegative, SOC and PSD rows"),
    Case("ns-big", _interleaved(BIG), "barrier sum past the first grid-stride pass", period=37),
]
BY_NAME = {c.name: c for c in CASES}


# ------------------------------------------------------------------------------------------------ dual barrier, grad
def M(x):
    return [mp.mpf(float(v)) for v in x]


def split(kind, d):
    """(alphas, d1) of the power-type cones"""
    if kind == "pow":
        a = mp.mpf(float(d))
        return [a, 1 - a], 2
    return [mp.mpf(float(v)) for v in d[0]], len(d[0])


def _phi_dual(al, u):
    return mp.fprod((u[i] / al[i]) ** (2 * al[i]) for i in range(len(al)))


def fstar(kind, d, z):
    if kind == "exp":
        return -mp.log(-z[0] * z[2]) - mp.log(z[1] - z[0] - z[0] * mp.log(-z[2] / z[0]))
    al, d1 = split(kind, d)
    u, w = z[:d1], z[d1:]
    return -mp.log(_phi_dual(al, u) - mp.fsum(v * v for v in w)) - mp.fsum((1 - al[i]) * mp.log(u[i]) for i in range(d1))


def grad_fstar(kind, d, z):
    if kind == "exp":
        l = mp.log(-z[2] / z[0])
        psi = z[1] - z[0] - z[0] * l
        return [-1 / z[0] + l / psi, -1 / psi, -1 / z[2] + z[0] / (z[2] * psi)]
    al, d1 = split(kind, d)
    u, w = z[:d1], z[d1:]
    phi = _phi_dual(al, u)
    zeta = phi - mp.fsum(v * v for v in w)
    return [-2 * al[i] * phi / (u[i] * zeta) - (1 - al[i]) / u[i] for i in range(d1)] + [2 * v / zeta for v in w]


def in_dual(kind, d, z):
    z = M(z) if not isinstance(z[0], mp.mpf) else z
    if kind == "exp":
        return z[2] > 0 and z[0] < 0 and z[1] - z[0] - z[0] * mp.log(-z[2] / z[0]) > 0
    al, d1 = split(kind, d)
    return all(v > 0 for v in z[:d1]) and _phi_dual(al, z[:d1]) - mp.fsum(v * v for v in z[d1:]) > 0


def in_primal(kind, d, s):
    s = M(s) if not isinstance(s[0], mp.mpf) else s
    if kind == "exp":
        return s[2] > 0 and s[1] > 0 and s[1] * mp.log(s[2] / s[1]) - s[0] > 0
    al, d1 = split(kind, d)
    return all(v > 0 for v in s[:d1]) and mp.fprod(s[i] ** (2 * al[i]) for i in range(d1)) - mp.fsum(v * v for v in s[d1:]) > 0


def _jvp(F, z, v):
    """d/dt F(z + t v) at 0, central differences at 80 digits"""
    with mp.workdps(80):
        h = mp.mpf(10) ** -30
        a = F([zi + h * vi for zi, vi in zip(z, v)])
        b = F([zi - h * vi for zi, vi in zip(z, v)])
        out = [(x - y) / (2 * h) for x, y in zip(a, b)]
    return [+x for x in out]


def hess_vec(kind, d, z, v):
    return _jvp(lambda q: grad_fstar(kind, d, q), z, v)


def hess(kind, d, z):
    n = len(z)
    cols = [hess_vec(kind, d, z, [mp.mpf(int(i == j)) for i in range(n)]) for j in range(n)]
    return mp.matrix([[cols[j][i] for j in range(n)] for i in range(n)])


def third(kind, d, z, u, v):
    """D3 f*(z)[u, v] = d/dt Hess f*(z + t u) v"""
    with mp.workdps(80):
        h = mp.mpf(10) ** -20
        a = hess_vec(kind, d, [zi + h * ui for zi, ui in zip(z, u)], v)
        b = hess_vec(kind, d, [zi - h * ui for zi, ui in zip(z, u)], v)
        out = [(x - y) / (2 * h) for x, y in zip(a, b)]
    return [+x for x in out]


# ---------------------------------------------------------------------------------------------------- primal side
def grad_primal(kind, d, s):
    """g with -grad f*(-g) = s"""
    if kind == "exp":
        zarg = 1 - s[0] / s[1] - mp.log(s[1] / s[2])
        w = wright_omega(zarg)
        g0 = 1 / ((w - 1) * s[1])
        return [g0, g0 + g0 * mp.log(w * s[1] / s[2]) - 1 / s[1], w / ((1 - w) * s[2])]
    al, d1 = split(kind, d)
    u, w = s[:d1], s[d1:]
    r = mp.sqrt(mp.fsum(v * v for v in w))
    if r == 0:
        return [-(1 + al[i]) / u[i] for i in range(d1)] + [mp.mpf(0)] * len(w)

    def gu(x):
        return [-(1 + al[i] + al[i] * x * r) / u[i] for i in range(d1)]

    def h(x):   # r (phi(-g_u(x)) - x^2) - 2x: positive at 0, negative past the root
        return r * (_phi_dual(al, [-v for v in gu(x)]) - x * x) - 2 * x

    hi = mp.mpf(1) / r
    while h(hi) > 0:
        hi *= 4
    lo = hi / 4
    while h(lo) <= 0:
        lo /= 4
    for _ in range(400):          # bisection, geometric while the bracket spans orders of magnitude
        mid = (lo + hi) / 2 if hi / lo < 4 else mp.sqrt(lo * hi)
        (lo, hi) = (mid, hi) if h(mid) > 0 else (lo, mid)
        if hi - lo <= hi * mp.mpf(10) ** -48:
            break
    x = (lo + hi) / 2
    return gu(x) + [(x / r) * v for v in w]


def wright_omega(zarg):
    return mp.lambertw(mp.exp(zarg)).real


def nu(kind, d):
    return 3 if kind in ("exp", "pow") else len(d[0]) + 1


def f_primal(kind, d, s):
    return -fstar(kind, d, [-v for v in grad_primal(kind, d, s)]) - nu(kind, d)


def pd_Hs(s, z, st, zt, H, mu_dual, force=False):
    """nonsymmetric_common.rs:72-143 on exact inputs; also the cancellation factor of de2 when the primal-dual formula
    applies, None where it falls back to mu H.  force: the primal-dual formula whatever the test says"""
    dot = lambda a, b: mp.fsum(x * y for x, y in zip(a, b))
    dsz = dot(s, z)
    mu, mut = dsz / 3, dot(st, zt) / 3
    ds = [s[i] + mu * st[i] for i in range(3)]
    dz = [z[i] + mu * zt[i] for i in range(3)]
    ddsz = dot(ds, dz)
    Hzt = H * mp.matrix(zt)
    de1 = mu * mut - 1
    de2 = dot(zt, Hzt) - 3 * mut * mut
    if force or (abs(de1) > SQRT_EPS and abs(de2) > EPS and dsz > 0 and ddsz > 0):
        tmp = [mut * st[i] - Hzt[i] for i in range(3)]
        W = mp.matrix(3, 3)
        for i in range(3):
            for j in range(3):
                W[i, j] = H[i, j] - st[i] * st[j] / 3 - tmp[i] * tmp[j] / de2
        t = mu * mp.sqrt(mp.fsum(W[i, j] ** 2 for i in range(3) for j in range(3)))
        ax = [z[1] * zt[2] - z[2] * zt[1], z[2] * zt[0] - z[0] * zt[2], z[0] * zt[1] - z[1] * zt[0]]
        na = mp.sqrt(dot(ax, ax))
        ax = [v / na for v in ax] if na > 0 else ax
        Hs = mp.matrix(3, 3)
        for i in range(3):
            for j in range(3):
                Hs[i, j] = s[i] * s[j] / dsz + ds[i] * ds[j] / ddsz + t * ax[i] * ax[j]
        # the formula divides by de2, a difference of two terms of size |zt' H zt|: its relative rounding error is
        # eps times this cancellation factor, and Hs inherits it
        return Hs, (abs(dot(zt, Hzt)) + 3 * mut * mut) / abs(de2)
    return mu_dual * H, None


def packed(H):
    return [H[i, j] for j in range(3) for i in range(j + 1)]


# -------------------------------------------------------------------------------------------------------- points
def dual_boundary_point(kind, d, rng, margin):
    """z in the interior of K*, relative distance about `margin` from its boundary"""
    if kind == "exp":
        z0, z2 = -float(rng.uniform(0.5, 2.0)), float(rng.uniform(0.5, 2.0))
        z1b = z0 + z0 * np.log(-z2 / z0)
        return np.array([z0, z1b + margin * (abs(z0) + abs(z2) + abs(z1b)), z2])
    al, d1 = split(kind, d)
    u = rng.uniform(0.5, 2.0, d1)
    phi = float(_phi_dual(al, M(u)))
    n2 = len(d[0]) + d[1] - d1 if kind == "genpow" else 1
    w = rng.standard_normal(n2)
    w *= np.sqrt(phi) * (1 - margin) / np.linalg.norm(w)
    return np.concatenate([u, w])


def central(kind, d, z, mu):
    """s = -mu grad f*(z), rounded"""
    return np.array([float(-mu * v) for v in grad_fstar(kind, d, M(z))])


def unit(kind, d):
    if kind == "exp":
        return np.array([-1.051383945322714, 0.556409619469370, 1.258967884768947])
    al, d1 = split(kind, d)
    n2 = len(d[0]) + d[1] - d1 if kind == "genpow" else 1
    return np.concatenate([[np.sqrt(1.0 + float(a)) for a in al], np.zeros(n2)])


def edge_point(kind, d, j):
    """the j-th edge point of the cone: Wright-omega arguments for exp; for the power cones s0/s1 and phi over 1e+-8
    with |w| / sqrt(phi) from W_RATIOS.  z = -g(s), the central-path partner at mu = 1, perturbed by 1e-3 relative."""
    if kind == "exp":
        za = OMEGA_ARGS[j % len(OMEGA_ARGS)]
        sc = [1.0, 1e-8, 1e8][(j // len(OMEGA_ARGS)) % 3]
        s = np.array([1.0 - za, 1.0, 1.0]) * sc               # 1 - s0/s1 - log(s1/s2) = za
    else:
        al, d1 = split(kind, d)
        ratio = W_RATIOS[j % len(W_RATIOS)]
        u = np.array([[1.0, 1e8, 1e-8][(j // len(W_RATIOS) + i) % 3] for i in range(d1)]) * [1.0, 1e8, 1e-8][(j // 3) % 3]
        phi = float(mp.fprod(mp.mpf(u[i]) ** (2 * al[i]) for i in range(d1)))
        n2 = len(d[0]) + d[1] - d1 if kind == "genpow" else 1
        w = np.cos(np.arange(n2) + 0.3 * j) + 0.1
        w = w / np.linalg.norm(w) * ratio * np.sqrt(phi)
        s = np.concatenate([u, w])
    z0 = s_to_z_partner(kind, d, s)
    for rel in (1e-3, 1e-5, 1e-7, 1e-9):       # less where s sits that close to the boundary
        z = z0 * (1 + rel * np.cos(np.arange(z0.size) + j))
        if in_dual(kind, d, z):
            return s, z
    raise RuntimeError("no edge point")


def s_to_z_partner(kind, d, s):
    """the dual point whose central-path partner at mu = 1 is s: z = -g(s)"""
    return np.array([float(-v) for v in grad_primal(kind, d, M(s))])


def point(case, k, kind, d, regime):
    """(s, z, mu) of the k-th cone of its kind in `case`"""
    key = k % case.period if case.period else k
    return _point(kind, (tuple(d[0]), d[1]) if kind == "genpow" else d, regime, key)


@functools.lru_cache(maxsize=None)
def _point(kind, d, regime, key):
    rng = np.random.default_rng(1000 * REGIMES.index(regime) + key)
    if regime == "opening":
        e = unit(kind, d)
        for _ in range(1000):
            sp = 0.05 * (1 + key % 6) / np.sqrt(e.size / 3)
            s, z = e + sp * rng.standard_normal(e.size), e + sp * rng.standard_normal(e.size)
            if in_primal(kind, d, s) and in_dual(kind, d, z):
                return s, z, float(s @ z) / nu(kind, d)
        raise RuntimeError("no opening point")
    if regime == "edge":
        s, z = edge_point(kind, d, key)
        return s, z, 1.0
    # on the path down to a relative margin of 1e-6; off it by 1e-3 only where the margin leaves room for that
    z = dual_boundary_point(kind, d, rng, ([1e-2, 1e-4, 1e-6] if regime == "late" else [1e-1, 3e-2, 1e-2])[key % 3])
    s = central(kind, d, z, MU_LATE)
    if regime == "late-off":
        s = s * (1 + 1e-3 * rng.uniform(-1, 1, s.size))
        assert in_primal(kind, d, s)
    return s, z, MU_LATE


# ---------------------------------------------------------------------------------------------------- reference
@dataclass
class Ref:
    kind: str
    d: object
    s: list
    z: list
    st: list          # grad f*(z)
    zt: list          # g(s)
    H: object         # Hess f*(z)
    kappa: float      # condition measure of the point


@functools.lru_cache(maxsize=None)
def _ref(kind, d, sb, zb):
    s, z = M(np.frombuffer(sb)), M(np.frombuffer(zb))
    st, zt = grad_fstar(kind, d, z), grad_primal(kind, d, s)
    n = lambda v: mp.sqrt(mp.fsum(x * x for x in v))
    kap = float(max(n(s) * n(zt), n(z) * n(st)) / nu(kind, d))
    return Ref(kind, d, s, z, st, zt, hess(kind, d, z) if kind != "genpow" else None, kap)


def ref(kind, d, s, z):
    d = tuple((tuple(d[0]), d[1])) if kind == "genpow" else d
    return _ref(kind, d, np.ascontiguousarray(s, float).tobytes(), np.ascontiguousarray(z, float).tobytes())


def eta(r, ds, dz):
    u = mp.lu_solve(r.H, mp.matrix(M(ds)))
    T = third(r.kind, r.d, r.z, [u[i] for i in range(3)], M(dz))
    return [ETA_SIGN * v / 2 for v in T]


# ------------------------------------------------------------------------------------------------- step lengths
def crossing(kind, d, q, dq, dual, amax=10.0):
    """largest alpha <= amax with q + t dq inside for all t in [0, alpha] (the cone is convex: one crossing)"""
    inside = (lambda x: in_dual(kind, d, x)) if dual else (lambda x: in_primal(kind, d, x))
    q, dq = M(q), M(dq)
    at = lambda a: [x + a * y for x, y in zip(q, dq)]
    hi = mp.mpf(amax)
    if inside(at(hi)):
        return hi
    lo = mp.mpf(0)
    for _ in range(170):
        mid = (lo + hi) / 2
        (lo, hi) = (mid, hi) if inside(at(mid)) else (lo, mid)
    return (lo + hi) / 2


def backtrack(a0, j):
    a = a0
    for _ in range(j):
        a *= STEP
    return a


def exact_count(kind, d, q, dq, dual, a0):
    """smallest j with a0 step^j (the doubles the kernel walks) exactly inside, J_ZERO below A_MIN"""
    inside = (lambda x: in_dual(kind, d, x)) if dual else (lambda x: in_primal(kind, d, x))
    a = a0
    for j in range(4096):
        if inside([mp.mpf(float(x)) + mp.mpf(a) * mp.mpf(float(y)) for x, y in zip(q, dq)]):
            return j
        a *= STEP
        if a < A_MIN:
            return J_ZERO
    return J_ZERO


def directions(kind, d, q, dual, rng, a0, gap):
    """(label, dq) for each step-length case: nothing binds, an interior crossing, a crossing `gap` below a0 and a
    collapse below A_MIN"""
    out = [("inside", np.array(q, float) * 0.5)]
    for _ in range(200):
        y = rng.standard_normal(len(q)) * np.abs(q).max()
        a = float(crossing(kind, d, q, y, dual, amax=1e6))
        if 1e-6 < a < 1e5:
            break
    out.append(("interior", y * a / (a0 * STEP ** 3.5)))
    out.append(("near-amax", y * a / (a0 * (1 - gap))))
    out.append(("collapse", y * a / (A_MIN * 0.01)))
    return out
