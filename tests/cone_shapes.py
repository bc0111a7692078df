"""Cone lists at the launch shapes where the symmetric cone kernels (cones.cu, cones_psd.cu) change behaviour, points
in the conditioning regimes an interior-point solve passes through, search directions for each step-length case, and
an extended-precision reference for all of it.  No GPU: tests/test_cone_shapes_cpu.py checks the shapes and the
reference, tests/test_cone_shapes_gpu.py holds the device to it.

Shapes (the constants below restate cones_psd.cu / cones.cu / vec.cuh; the CPU test reads them back from the sources):
  PSD: one warp per cone; warps per CTA = min(4, 200 KiB / (8 matrices * nmax^2 * 8 B)) with nmax the largest PSD cone
       of the problem, and none fitting (nmax >= 57) means the global scratch arena.  Lane k owns rows k, k+32, ...
  SOC: one CTA of 128 threads per cone, strided loops from index 1; dimensions 2..4 are dense Hs blocks, 5 and up the
       sparse expansion.
  nonnegative: grid-stride reductions over 296 x 256 threads; row 75 776 starts a second pass.

Reference: every quantity is computed from the double inputs as given (svec entries are unscaled by an exact 1/sqrt2).
PSD cones up to MP_MAX_N use mpmath at 50 digits; larger ones a LAPACK eigendecomposition refined in np.longdouble
(Ogita-Aishima), with Cholesky and products in longdouble.  Both go through the same code, on object arrays of mpf or
on longdouble arrays.  The longdouble path carries relative errors of about 1e-19 * cond, four orders below what the
double-precision kernels reach in the same regime.  SOC quantities use mpmath throughout."""
import math
from dataclasses import dataclass

import mpmath as mp
import numpy as np

mp.mp.dps = 50

PSD_WARPS, PSD_NMAT, PSD_SMEM_BUDGET = 4, 8, 200 * 1024      # cones_psd.cu
CB_PSD_MAX_N = 128                                          # problem_setup.h
SOC_NT = 128                                                # cones.cu
RED_BLOCKS, RED_THREADS = 296, 256                          # vec.cuh
MP_MAX_N = 20            # larger PSD cones: refined longdouble (mpmath costs ~1 s per decomposition at n = 33)
LD = np.longdouble


def psd_warps(nmax):
    """warps (cones) per CTA of the PSD kernels, 0 for the global scratch arena (ConeSet::psd_prepare)"""
    w = PSD_SMEM_BUDGET // (PSD_NMAT * nmax * nmax * 8)
    return min(w, PSD_WARPS) if w >= 1 else 0


def psd_row(nmax):
    w = psd_warps(nmax)
    return f"{w} warps/CTA" if w else "global scratch"


PSD_ROWS = ["4 warps/CTA", "3 warps/CTA", "2 warps/CTA", "1 warps/CTA", "global scratch"]


def numel(kind, d):
    return d * (d + 1) // 2 if kind == "psd" else d


@dataclass
class Case:
    name: str
    cones: list
    reaches: str         # the shape this list is there for

    @property
    def m(self):
        return sum(numel(k, d) for k, d in self.cones)

    @property
    def psd(self):
        return [d for k, d in self.cones if k == "psd"]

    @property
    def row(self):
        return psd_row(max(self.psd)) if self.psd else None

    def ctas(self):
        """the PSD cones of each CTA, in launch order"""
        w = psd_warps(max(self.psd)) or PSD_WARPS
        return [self.psd[i:i + w] for i in range(0, len(self.psd), w)]


PSD_CASES = [
    Case("psd-n28", [("psd", 28), ("nonneg", 3)], "4 warps/CTA, one row per lane"),
    Case("psd-n29x3", [("psd", 29)] * 3, "3 warps/CTA, one full CTA of equal cones"),
    Case("psd-n32", [("psd", 32)], "3 warps/CTA, n = 32: every lane owns one row"),
    Case("psd-n33x2", [("psd", 33)] * 2, "2 warps/CTA, two rows per lane"),
    Case("psd-n41", [("psd", 41)], "1 warps/CTA"),
    Case("psd-n56", [("psd", 56)], "1 warps/CTA, largest shared-memory cone"),
    Case("psd-n57", [("psd", 57), ("soc", 4)], "global scratch, smallest"),
    Case("psd-n64-65", [("psd", 64), ("psd", 65)], "global scratch, two and three rows per lane"),
    Case("psd-n96-97", [("psd", 96), ("psd", 97)], "global scratch, three and four rows per lane"),
    Case("psd-n128", [("psd", 128)], "global scratch, CB_PSD_MAX_N, four rows per lane"),
    Case("psd-mixed", [("psd", 20), ("psd", 3), ("psd", 12), ("psd", 28)], "one CTA of four cones of different sizes"),
    Case("psd-partial", [("psd", 28)] + [("psd", 3)] * 4, "two CTAs of 4 warps, the last one partly filled"),
]
SOC_DIMS = [2, 3, 4, 5, 127, 128, 129, 130, 257]
SOC_CASES = [
    Case("soc-dims", [("soc", d) for d in SOC_DIMS], "dense 2-4, sparse 5+, 1-3 strided passes"),
    Case("soc-long", [("soc", 100000), ("nonneg", 2)], "a 1e5-long block reduction"),
]
NN_CASES = [Case(f"nonneg-{m}", [("nonneg", m)], "grid-stride pass boundary") for m in (75775, 75776, 75777, 300000)]
CASES = PSD_CASES + SOC_CASES + NN_CASES
BY_NAME = {c.name: c for c in CASES}


# ------------------------------------------------------------------------------------------------------------- points
def svec(M):
    n = M.shape[0]
    return np.array([M[r, c] if r == c else M[r, c] * math.sqrt(2.0) for c in range(n) for r in range(c + 1)])


def _orth(rng, n):
    Q, R = np.linalg.qr(rng.standard_normal((n, n)))
    return Q * np.sign(np.diag(R))


def psd_pair(rng, n, regime, mu=1e-6):
    """(S, Z) as double matrices (symmetrised) for one PSD cone"""
    if regime == "opening":     # cond 10 each, unrelated eigenvectors
        Q1, Q2 = _orth(rng, n), _orth(rng, n)
        S = Q1 @ np.diag(np.logspace(0, 1, n)) @ Q1.T
        Z = Q2 @ np.diag(rng.permutation(np.logspace(0, 1, n))) @ Q2.T
    else:   # late: S = Q diag(sig) Q', Z = Qt diag(mu / sig (1 + 0.1 u)) Qt', Qt = Q after a small rotation
        Q = _orth(rng, n)
        sig = rng.permutation(np.logspace(-8, 2, n))
        K = rng.standard_normal((n, n)) * 1e-6       # small enough to keep lambda^2 near mu (S Z leaks 1e4 K^2)
        Qt = Q @ _expm_skew(K - K.T)
        S = Q @ np.diag(sig) @ Q.T
        Z = Qt @ np.diag(mu / sig * (1 + 0.1 * rng.random(n))) @ Qt.T
    return (S + S.T) / 2, (Z + Z.T) / 2


def _expm_skew(A):
    w, V = np.linalg.eig(A)
    return np.real(V @ np.diag(np.exp(w)) @ np.linalg.inv(V))


SOC_LATE = (1e-6, 1e-10, 1e-13)


def soc_pair(rng, d, regime, k=0):
    """(s, z) for one SOC of dimension d.  late: z0 - |z1| = r z0 with r = SOC_LATE[k % 3], s pointing the other way
    along the boundary (nearly complementary)"""
    if regime == "opening":
        z1, s1 = rng.standard_normal(d - 1), rng.standard_normal(d - 1)
        return (np.concatenate([[1.5 * np.linalg.norm(s1) + 0.2], s1]),
                np.concatenate([[1.5 * np.linalg.norm(z1) + 0.2], z1]))
    r = SOC_LATE[k % 3]
    z1 = exact_norm_vector(rng, d - 1)
    s1 = -z1.copy()
    s1[: (d - 1) // 2] += rng.integers(-1, 2, (d - 1) // 2)
    s1 = exact_norm_fix(s1, 1.0) * 2.0 ** -10        # along -z1: nearly complementary
    return tuple(np.concatenate([[np.sqrt(v @ v) * (1 + r)], v]) for v in (s1, z1))


def exact_norm_vector(rng, k):
    """small integers whose sum of squares is a perfect square below 2^53: |v| and v'v are exact in double, so a
    margin z0 - |z1| = r z0 is exactly the given data's and only the kernel's own arithmetic can lose it"""
    return exact_norm_fix(rng.integers(-3, 4, k).astype(float), 1.0)


def exact_norm_fix(v, unit):
    """change the last entry (a multiple of unit) so that |v|^2 / unit^2 is a perfect square"""
    u = np.rint(v / unit).astype(np.int64)
    if len(u) == 1:
        return np.where(u == 0, 1, u).astype(float) * unit
    Q = int((u[:-1] ** 2).sum())
    if Q % 4 == 2:
        u[0] += 1
        Q = int((u[:-1] ** 2).sum())
    if Q == 0:
        u[-1] = 1
    elif Q % 2:
        u[-1] = (Q - 1) // 2
    else:
        u[-1] = (Q // 2 - 2) // 2       # Q = 4 q: (t - e)(t + e) = Q with t - e = 2
    t2 = int((u ** 2).sum())
    assert int(np.sqrt(t2)) ** 2 == t2 and t2 < 2 ** 53
    return u.astype(float) * unit


def interior(case, regime, seed):
    """(s, z) in the interior of every cone of the list"""
    rng = np.random.default_rng(seed)
    ss, zz = [], []
    for k, (kind, d) in enumerate(case.cones):
        if kind == "nonneg":
            if regime == "opening":
                s, z = rng.uniform(0.5, 2.0, d), rng.uniform(0.5, 2.0, d)
            else:
                s = np.logspace(-8, 2, d)[rng.permutation(d)]
                z = 1e-6 / s * (1 + 0.1 * rng.random(d))
        elif kind == "soc":
            s, z = soc_pair(rng, d, regime, k)
        else:
            S, Z = psd_pair(rng, d, regime)
            s, z = svec(S), svec(Z)
        ss.append(s); zz.append(z)
    return np.concatenate(ss), np.concatenate(zz)


def blocks(case, v):
    """split a length-m vector into per-cone pieces"""
    out, o = [], 0
    for kind, d in case.cones:
        ne = numel(kind, d)
        out.append(v[o:o + ne]); o += ne
    return out


# -------------------------------------------------------------------------------- extended-precision arithmetic (PSD)
class Ext:
    """mpmath (object arrays of mpf) or longdouble arrays, with one set of operations"""
    def __init__(self, n, use_mp=None):
        self.mp = n <= MP_MAX_N if use_mp is None else use_mp
        self.iters = 4 if self.mp else 3

    def arr(self, x):
        x = np.asarray(x, dtype=np.float64)
        if self.mp:
            return np.vectorize(mp.mpf, otypes=[object])(x) if x.size else x.astype(object)
        return x.astype(LD)

    def sqrt(self, x):
        return np.vectorize(mp.sqrt, otypes=[object])(x) if self.mp else np.sqrt(x)

    def rsqrt2(self):
        return 1 / mp.sqrt(2) if self.mp else 1 / np.sqrt(LD(2))

    def f64(self, x):
        return np.asarray(np.vectorize(float)(x) if self.mp else x, dtype=np.float64)

    def eye(self, n):
        return self.arr(np.eye(n))

    def smat(self, x, n):
        """svec (sqrt2-scaled packed upper triangle) -> symmetric matrix, exactly"""
        x = self.arr(x)
        M = self.arr(np.zeros((n, n)))
        r2 = self.rsqrt2()
        k = 0
        for c in range(n):
            for r in range(c + 1):
                M[r, c] = M[c, r] = x[k] if r == c else x[k] * r2
                k += 1
        return M

    def svec(self, M):
        n = M.shape[0]
        r2 = 1 / self.rsqrt2()
        return np.array([M[r, c] if r == c else (M[r, c] + M[c, r]) / 2 * r2 for c in range(n) for r in range(c + 1)],
                        dtype=M.dtype)

    def chol(self, A):
        n = A.shape[0]
        L = self.arr(np.zeros((n, n)))
        A = A.copy()
        for j in range(n):
            d = A[j, j]
            assert d > 0, "not positive definite"
            L[j, j] = self.sqrt(np.array([d], dtype=A.dtype))[0]
            L[j + 1:, j] = A[j + 1:, j] / L[j, j]
            A[j + 1:, j + 1:] -= np.outer(L[j + 1:, j], L[j + 1:, j])
        return L

    def tri_inv(self, L):
        """inverse of a lower triangular matrix, by forward substitution"""
        n = L.shape[0]
        X = self.arr(np.zeros((n, n)))
        for i in range(n):
            X[i, :] = (-(L[i, :i] @ X[:i, :]) if i else X[i, :] * 0)
            X[i, i] += 1
            X[i, :] = X[i, :] / L[i, i]
        return X

    def eigh(self, A):
        """eigenvalues (ascending) and orthonormal eigenvectors of the symmetric A to working precision:
        np.linalg.eigh in double, then Ogita-Aishima refinement (RefSyEv)"""
        n = A.shape[0]
        w, X = np.linalg.eigh(self.f64(A))
        X = self.arr(X)
        I = self.eye(n)
        for _ in range(self.iters):
            R = I - X.T @ X
            S = X.T @ A @ X
            lam = np.array([S[i, i] / (1 - R[i, i]) for i in range(n)], dtype=A.dtype)
            Sd, Rd, lf = self.f64(S), self.f64(R), self.f64(lam)
            delta = 2 * (np.linalg.norm(Sd - np.diag(lf)) + np.linalg.norm(self.f64(A)) * np.linalg.norm(Rd))
            E = self.arr(np.zeros((n, n)))
            for i in range(n):
                for j in range(n):
                    if i != j and abs(lf[j] - lf[i]) > delta:
                        E[i, j] = (S[i, j] + lam[j] * R[i, j]) / (lam[j] - lam[i])
                    else:
                        E[i, j] = R[i, j] / 2
            X = X + X @ E
        R = I - X.T @ X
        S = X.T @ A @ X
        lam = np.array([S[i, i] / (1 - R[i, i]) for i in range(n)], dtype=A.dtype)
        o = np.argsort(self.f64(lam), kind="stable")
        return lam[o], X[:, o]


@dataclass
class PsdRef:
    n: int
    lam: np.ndarray        # NT lambda, descending (double)
    W: np.ndarray          # W_nt = R R' (double)
    R: np.ndarray          # L1 V Lambda^-1/2 in the sign convention of the reference's eigenvectors (extended)
    Rinv: np.ndarray       # Lambda^1/2 V' L1^-1 (extended)
    lam_x: np.ndarray      # lambda (extended)
    Lz: np.ndarray         # chol(Z), chol(S) (extended), for the step length
    Ls: np.ndarray
    zmin: float            # smallest eigenvalue of Z and the sum of its positive eigenvalues
    zpos: float
    condS: float
    condZ: float
    ext: Ext


def psd_reference(s, z, n, use_mp=None):
    """NT scaling of one PSD cone from the svec points s, z"""
    e = Ext(n, use_mp)
    S, Z = e.smat(s, n), e.smat(z, n)
    L1, L2 = e.chol(S), e.chol(Z)
    ev, V = e.eigh(L1.T @ Z @ L1)          # = M'M with M = L2' L1: eigenvalues lambda^2
    ev, V = ev[::-1], V[:, ::-1]
    lam = e.sqrt(ev)
    R = L1 @ V / e.sqrt(lam)[None, :]
    Rinv = (e.sqrt(lam)[:, None] * V.T) @ e.tri_inv(L1)
    zev, _ = e.eigh(Z)
    sev, _ = e.eigh(S)
    zf, sf = e.f64(zev), e.f64(sev)
    return PsdRef(n, e.f64(lam), e.f64(R @ R.T), R, Rinv, lam, L2, L1, float(zf[0]), float(zf[zf > 0].sum()),
                  float(sf[-1] / sf[0]), float(zf[-1] / zf[0]), e)


def psd_maxstep(ref, side, d, amax):
    """largest alpha <= amax with X + alpha dX PSD (X = Z for side 'z', S for 's'); d an svec direction"""
    e = ref.ext
    L = ref.Lz if side == "z" else ref.Ls
    Li = e.tri_inv(L)
    ev, _ = e.eigh(Li @ e.smat(d, ref.n) @ Li.T)
    mn = ev[0]
    if not mn < 0:
        return amax
    return min(amax, float(-1 / mn))


def psd_eig(x, n):
    """eigenvalues of smat(x) to working precision (margins of an arbitrary symmetric point)"""
    e = Ext(n)
    ev, _ = e.eigh(e.smat(x, n))
    return e.f64(ev)


def psd_shift(ref, dz, ds, sigmamu):
    """(W^-T ds) o (W dz) - sigmamu I in the reference's frame, as an svec (double), and the extended W^-T ds, W dz"""
    e, n = ref.ext, ref.n
    Y = ref.R.T @ e.smat(dz, n) @ ref.R
    X = ref.Rinv @ e.smat(ds, n) @ ref.Rinv.T
    Sh = (X @ Y + Y @ X) / 2 - e.eye(n) * e.arr(sigmamu)
    return e.f64(e.svec(Sh))


def psd_ds_residual(ref, out, ds, D):
    """lambda o (W^-T out) - D ds D in extended precision (D: the device frame's column signs), svec (double)"""
    e, n = ref.ext, ref.n
    X = ref.Rinv @ e.smat(out, n) @ ref.Rinv.T
    lam = ref.lam_x
    P = (lam[:, None] * X + X * lam[None, :]) / 2
    Dd = e.arr(np.outer(D, D))
    return e.f64(e.svec(P - Dd * e.smat(ds, n)))


def svec_index(n):
    """(row, col) of each svec slot: column-major upper triangle"""
    return (np.array([r for c in range(n) for r in range(c + 1)]), np.array([c for c in range(n) for r in range(c + 1)]))


def skron_error(Hs, W, chunk=256):
    """max |Hs - H| / max |H| for the packed upper triangle Hs of one PSD cone's block, where H = skron(W, W) is the
    matrix of X -> W X W on svec space: H[(i,j),(k,l)] = (W_ik W_jl + W_il W_jk) c_(i,j) c_(k,l) / 2, c = sqrt2 off the
    diagonal and 1 on it.  Column chunks keep the n = 128 block (8256^2 / 2 entries) out of memory at once."""
    r, c = svec_index(W.shape[0])
    N = len(r)
    cf = np.where(r == c, 1.0, math.sqrt(2.0))
    err = big = 0.0
    for q0 in range(0, N, chunk):
        q = np.arange(q0, min(N, q0 + chunk))
        p = np.arange(q[-1] + 1)
        H = (W[r[p][:, None], r[q][None, :]] * W[c[p][:, None], c[q][None, :]] +
             W[r[p][:, None], c[q][None, :]] * W[c[p][:, None], r[q][None, :]]) * (cf[p][:, None] * cf[q][None, :] / 2)
        got = np.zeros_like(H)
        for t, qq in enumerate(q):
            got[:qq + 1, t] = Hs[qq * (qq + 1) // 2: qq * (qq + 1) // 2 + qq + 1]
        mask = p[:, None] <= q[None, :]
        err = max(err, float(np.max(np.abs(got - H)[mask])))
        big = max(big, float(np.max(np.abs(H)[mask])))
    return err / big


# ------------------------------------------------------------------------------------------------------- SOC (mpmath)
def _m(x):
    return [mp.mpf(float(v)) for v in x]


def _dot(a, b):
    return mp.fsum(x * y for x, y in zip(a, b))


@dataclass
class SocRef:
    eta: object
    w: list                # normalised w (w0 = sqrt(1 + |w1|^2))
    lam: list
    condH: float


def soc_reference(s, z):
    s, z = _m(s), _m(z)
    zres = z[0] ** 2 - _dot(z[1:], z[1:])
    sres = s[0] ** 2 - _dot(s[1:], s[1:])
    zs, ss = mp.sqrt(zres), mp.sqrt(sres)
    eta = mp.sqrt(ss / zs)
    wb = [s[0] / ss + z[0] / zs] + [s[i] / ss - z[i] / zs for i in range(1, len(s))]
    wscale = mp.sqrt(wb[0] ** 2 - _dot(wb[1:], wb[1:]))
    w1 = [v / wscale for v in wb[1:]]
    w = [mp.sqrt(1 + _dot(w1, w1))] + w1
    g = wscale / 2
    sq = mp.sqrt(ss * zs)
    den = s[0] / ss + z[0] / zs + 2 * g
    ca, cb = (g + z[0] / zs) / ss, (g + s[0] / ss) / zs
    lam = [g * sq] + [(ca * s[i] + cb * z[i]) / den * sq for i in range(1, len(s))]
    return SocRef(eta, w, lam, float((w[0] + mp.sqrt(w[0] ** 2 - 1)) ** 4))


def soc_W(ref, x, inverse=False):
    """W x or W^-1 x (socone.rs's fast products), exact"""
    x = _m(x) if not isinstance(x[0], mp.mpf) else x
    w = ref.w
    w1x1 = _dot(w[1:], x[1:])
    if not inverse:
        c = x[0] + w1x1 / (1 + w[0])
        return [ref.eta * (w[0] * x[0] + w1x1)] + [ref.eta * (x[i] + c * w[i]) for i in range(1, len(x))]
    c = -x[0] + w1x1 / (1 + w[0])
    return [(w[0] * x[0] - w1x1) / ref.eta] + [(x[i] + c * w[i]) / ref.eta for i in range(1, len(x))]


def soc_H(ref, x):
    """H x = eta^2 (2 w w' - J) x"""
    x = _m(x)
    a = 2 * _dot(ref.w, x)
    e2 = ref.eta ** 2
    return [e2 * (a * ref.w[0] - x[0])] + [e2 * (a * ref.w[i] + x[i]) for i in range(1, len(x))]


def circ(x, y):
    return [_dot(x, y)] + [x[0] * y[i] + y[0] * x[i] for i in range(1, len(x))]


def soc_dot_cond(s, z):
    """componentwise condition number of s'z: (|s0 z0| + sum |s1_i z1_i|) / |s'z|"""
    s, z = np.asarray(s, dtype=float), np.asarray(z, dtype=float)
    return float(max(1.0, np.sum(np.abs(s * z)) / abs(_dot(_m(s), _m(z)))))


def soc_margin(z):
    z = _m(z)
    return float(z[0] - mp.sqrt(_dot(z[1:], z[1:])))


def soc_maxstep(x, y, amax):
    """largest alpha <= amax with x + alpha y in the SOC, for x in its interior (exact)"""
    x, y = _m(x), _m(y)
    a = y[0] ** 2 - _dot(y[1:], y[1:])
    b = 2 * (x[0] * y[0] - _dot(x[1:], y[1:]))
    c = x[0] ** 2 - _dot(x[1:], x[1:])
    best = mp.mpf(amax)
    if y[0] < 0:
        best = min(best, -x[0] / y[0])
    if a == 0:
        if b < 0:
            best = min(best, -c / b)
    else:
        disc = b * b - 4 * a * c
        if disc >= 0:
            for r in ((-b - mp.sqrt(disc)) / (2 * a), (-b + mp.sqrt(disc)) / (2 * a)):
                if r > 0:
                    best = min(best, r)
    return float(best)


def on_boundary(d, scale=1.0):
    """(5, 3, 4, 0, ...) * scale (a power of two): exactly on the boundary, residual exactly 0 in double"""
    v = np.zeros(d)
    v[0], v[1] = (5.0, 3.0) if d > 2 else (1.0, 1.0)
    if d > 2:
        v[2] = 4.0
    return v * scale


def soc_directions(rng, x, amax, gap=1e-9):
    """(label, y) per branch of the reference's SOC step-length component (socone.rs) for the interior x:
      inside     y in the cone: a > 0, b > 0, no bound (amax)
      opposite   y = -x / 2: a > 0, b < 0, d = 0 in exact arithmetic, < 0 or >= 0 after rounding; the x0 / y0 cap binds
      a==0       y exactly on the boundary of the cone, pointing in (amax)
      two-roots  a random y with y0 < 0
      near-amax  the two-roots y scaled so that the bound is amax (1 - gap)
    (d < 0 needs a > 0 with b < 0, i.e. -y in the cone, where x + alpha y leaves the cone: a real root.  It only occurs
    by rounding, as in `opposite`.)"""
    d = len(x)
    out = [("inside", np.concatenate([[1.0], np.zeros(d - 1)]) * abs(x[0])), ("opposite", -x / 2),
           ("a==0", on_boundary(d, 2.0 ** math.floor(math.log2(abs(x[0]) + 1e-300))))]
    y = rng.standard_normal(d) * abs(x[0])
    y[0] = -abs(y[0])
    out.append(("two-roots", y))
    a_exact = soc_maxstep(x, y, np.inf)
    out.append(("near-amax", y * (a_exact / (amax * (1 - gap)))))
    return out
