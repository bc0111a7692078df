"""Cone lists at the block shapes the KKT layer (solver.cu, KKTDevice) dispatches on, small problems around them, the
interior points of the opening and of the late iterations, and two references for K x = b.  No GPU:
tests/test_kkt_shapes_cpu.py checks the cases and the references, tests/test_kkt_shapes_gpu.py holds the device to them.

Shapes (the constants restate solver.cu / cones_nonsym.cu / vec.cuh):
  SOC      dimensions 2..4 are dense Hs blocks, 5 and up the sparse expansion (two extra rows); k_sparse_soc_fill runs
           one 128-thread CTA per entry of soc_list and returns at once on a dense cone
  PSD      the Hs block is dense and goes through map_Hs; n <= 56 is computed in shared memory, 57 and up in the global
           scratch arena
  exp/pow  3x3 packed blocks, 128 cones per CTA (NS_GRID)
  genpow   k_gp_kkt_fill, 128 cones per CTA (GP_GRID), one thread walking all rows of its cone: q, r, p columns and the
           constant diagonal (-1, -1, +1) of the three extension rows
  diagonal the static regulariser eps = constant + proportional * max |diag K| comes from a grid-stride reduction over
           296 x 256 threads: row 75 776 starts a second pass

Regimes: `opening` (the points of the first iterations), `late` (mu = 1e-9: nonnegative s / z over 1e+-8, SOC margins
1e-6 z0, PSD scalings with eigenvalues over 1e+-4, the nonsymmetric cones on their central path).  Several late
matrices are too ill-conditioned for a double LU to refine from, so the solve tests use the opening points and the
late ones of the SOC lists only.

References:
  ext_solve   K x = b for the full N x N matrix: an LU of K in double (scipy splu), refined with residuals computed in
              np.longdouble until a correction falls below 2^-60 of the solution
  refine      the reference's KKT solve (directldlkktsolver.rs, regularize_and_refactor and iterative_refinement) in
              double: static regularisation of the diagonal, an LDL' of the oracle's (QDLDL) on a given permutation,
              refinement against the unregularised K with the same acceptance rule"""
import functools
from dataclasses import dataclass, field

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import cone_shapes as cs
import nonsym_shapes as ns

LD = np.longdouble
SOC_NO_EXPANSION_MAX_SIZE = 4          # problem_setup.cpp: larger SOCs get the sparse expansion
SOC_NT = 128                           # solver.cu: threads of k_sparse_soc_fill
NS_BLOCK = 128                         # cones_nonsym.cu: cones per CTA of NS_GRID / GP_GRID
RED_PASS = cs.RED_BLOCKS * cs.RED_THREADS    # 75 776 rows per grid-stride pass of k_max_nonneg
PSD_SMEM_MAX = 56                      # the largest PSD cone whose kernels work in shared memory
MU_LATE = 1e-9
REGIMES = ["opening", "late"]
EMU_MAX_N = 3000                       # the emulated build's dense LDL stand-in


def rows(kind, d):
    return ns.rows(kind, d)


def expansion(kind, d):
    """extension rows of one cone"""
    return 2 if kind == "soc" and d > SOC_NO_EXPANSION_MAX_SIZE else 3 if kind == "genpow" else 0


@dataclass
class Case:
    name: str
    cones: list
    reaches: str
    n: int = 8
    P: str = "rand"          # "rand" or "zero" (an LP)
    solve: bool = True       # small enough for the dense-ish references of the solve tests
    peak_last: bool = False  # the largest |diagonal| of K sits in its last row (the reduction cases)

    @property
    def m(self):
        return sum(rows(k, d) for k, d in self.cones)

    @property
    def p(self):
        return sum(expansion(k, d) for k, d in self.cones)

    @property
    def N(self):
        return self.n + self.m + self.p

    @property
    def symmetric(self):
        return all(k in ("zero", "nonneg", "soc", "psd") for k, _ in self.cones)

    @property
    def emu(self):
        """runs on the emulated build's dense stand-in"""
        return self.N <= EMU_MAX_N


def _gp(d1, d2, j):
    return ("genpow", (ns._gp_alphas(d1, j), d2))


def _gps(count, d1, d2):
    return [_gp(d1, d2, j) for j in range(count)]


CASES = [
    Case("soc-dense", [("soc", 2), ("soc", 3), ("soc", 4)], "dense Hs blocks only: every k_sparse_soc_fill CTA returns"),
    Case("soc-sparse", [("soc", d) for d in (5, 127, 128, 129, 257)], "sparse expansion, 1..3 strided passes of 128"),
    Case("soc-5000", [("soc", 5000)], "one expansion column pair of 5000 rows", solve=True),
    Case("soc5-x2000", [("soc", 5)] * 2000, "2000 CTAs, one per soc_list entry"),
    Case("soc-alternating", [("soc", d) for d in (2, 5, 3, 6, 4, 129, 3, 7, 2, 130)],
         "dense and sparse alternating: the soc_list index is not the sparse-cone index"),
    Case("psd-1-2-4", [("psd", 1), ("psd", 2), ("psd", 4)], "smallest blocks, shared memory"),
    Case("psd-32", [("psd", 32)], "shared memory, one row per lane"),
    Case("psd-33", [("psd", 33)], "shared memory, two rows per lane"),
    Case("psd-56", [("psd", 56)], "largest shared-memory cone"),
    Case("psd-57", [("psd", 57)], "global scratch, smallest"),
    Case("psd-96", [("psd", 96)], "global scratch, three rows per lane", solve=False),
]
CASES += [Case(f"ns-{c}", ns._interleaved(c), f"{(c + NS_BLOCK - 1) // NS_BLOCK} CTA(s) of 3x3 blocks")
          for c in (1, 127, 128, 129)]
CASES += [Case(f"gp-{c}-{d1}x{d2}", _gps(c, d1, d2), f"k_gp_kkt_fill, {(c + NS_BLOCK - 1) // NS_BLOCK} CTA(s)")
          for d1, d2 in ((2, 1), (7, 40)) for c in (1, 127, 128, 129)]
CASES += [
    Case("gp-long", [_gp(2, 3000, 0)], "one thread walks 3002 rows"),
    Case("gp+soc", [_gp(2, 2, 0), ("soc", 6), ("nonneg", 2), _gp(3, 5, 1), ("soc", 130), ("soc", 3)],
         "both expansion fills in one update (p > 3 ngp)"),
    Case("zero+nonneg", [("zero", 3), ("nonneg", 20)], "structural zeros on the diagonal"),
    Case("m0", [], "no constraints: K = P", n=12),
    Case("lp", [("nonneg", 30), ("soc", 5), ("soc", 3)], "P = 0: zeros on the diagonal of the (1,1) block", P="zero"),
    Case("all", [("zero", 2), ("nonneg", 4), ("soc", 3), ("soc", 7), ("psd", 3), ("exp", 3), ("pow", 0.3),
                 _gp(2, 2, 0), ("psd", 1), ("soc", 5), ("pow", 0.9), _gp(3, 1, 2)], "every cone type at once"),
]
CASES += [Case(f"diag-{N}", [("nonneg", N - 10)], "eps's k_max_nonneg across its grid-stride pass", n=10, peak_last=True)
          for N in (RED_PASS - 1, RED_PASS, RED_PASS + 1)]
BY_NAME = {c.name: c for c in CASES}
NAMES = [c.name for c in CASES]


# ------------------------------------------------------------------------------------------------------------ problem
@functools.lru_cache(maxsize=None)
def problem(name):
    """(P, q, A, b) of the case: P random and positive definite (or zero), A with every row touched"""
    case = BY_NAME[name]
    n, m = case.n, case.m
    rng = np.random.default_rng(CASES.index(case) + 1)
    if case.P == "zero":
        P = sp.csc_matrix((n, n))
    else:
        F = sp.random(n, n, density=0.4, random_state=rng) + sp.identity(n)
        P = sp.triu(F @ F.T / n + 0.1 * sp.identity(n), format="csc")
    i = np.arange(m)
    r = np.concatenate([i, i])
    c = np.concatenate([i % n, (7 * i + 3) % n])
    v = np.concatenate([1.0 + 0.5 * rng.random(m), 0.5 * rng.standard_normal(m)])
    A = sp.csc_matrix((v, (r, c)), shape=(m, n))
    A.sum_duplicates()
    return P, rng.standard_normal(n), A, np.zeros(m)


# ------------------------------------------------------------------------------------------------------------- points
def _nonneg(rng, d, regime):
    if regime == "opening":
        return rng.uniform(0.5, 2.0, d), rng.uniform(0.5, 2.0, d)
    s = np.sqrt(MU_LATE) * 10.0 ** rng.uniform(-4, 4, d)        # s / z over 1e+-8
    return s, MU_LATE / s * (1 + 0.1 * rng.random(d))


def _psd(rng, n, regime):
    if regime == "opening":
        return cs.psd_pair(rng, n, regime)
    Q = cs._orth(rng, n)
    sig = np.sqrt(MU_LATE) * np.logspace(-4, 4, n)[rng.permutation(n)]     # W's eigenvalues over 1e+-4
    S = Q @ np.diag(sig) @ Q.T
    Z = Q @ np.diag(MU_LATE / sig * (1 + 0.1 * rng.random(n))) @ Q.T
    return (S + S.T) / 2, (Z + Z.T) / 2


def point(name, regime, seed=0):
    """(s, z, mu): a point in the interior of every cone of the case, and the mu the nonsymmetric scalings are given"""
    case = BY_NAME[name]
    rng = np.random.default_rng(1000 * seed + 10 * CASES.index(case) + REGIMES.index(regime))
    ss, zz, mus, cnt = [], [], [], {}
    for j, (kind, d) in enumerate(case.cones):
        if kind == "zero":
            s, z = np.zeros(d), np.zeros(d)
        elif kind == "nonneg":
            s, z = _nonneg(rng, d, regime)
        elif kind == "soc":
            s, z = cs.soc_pair(rng, d, regime, 0)        # late: margin 1e-6 z0, nearly complementary
        elif kind == "psd":
            S, Z = _psd(rng, d, regime)
            s, z = cs.svec(S), cs.svec(Z)
        else:
            k = cnt.get(kind, 0)
            cnt[kind] = k + 1
            dd = (tuple(d[0]), d[1]) if kind == "genpow" else d
            s, z, mu = ns._point(kind, dd, regime, (k + seed) % 8)
            mus.append(mu)
        ss.append(s); zz.append(z)
    s = np.concatenate(ss) if ss else np.zeros(0)
    z = np.concatenate(zz) if zz else np.zeros(0)
    if case.peak_last:      # s / z in [1/4, 4], and 1e6 (1 + seed)^2 in the last row: the largest |diagonal| of K
        t = 1.0 if regime == "opening" else np.sqrt(MU_LATE)
        s, z = t * rng.uniform(0.5, 2.0, case.m), t * rng.uniform(0.5, 2.0, case.m)
        s[-1], z[-1] = t * 1e3 * (1 + seed), t * 1e-3 / (1 + seed)
    mu = mus[0] if mus else (float(s @ z) / max(case.m, 1) if case.m else 1.0)
    return s, z, mu


# ------------------------------------------------------------------------------------------------------ references
def full(N, cp, rv, nz):
    """the symmetric N x N matrix of a triu-stored K"""
    U = sp.csc_matrix((nz, rv, cp), shape=(N, N))
    return (U + sp.triu(U, 1, format="csc").T).tocsc()


def residual_ld(K, x, b):
    """b - K x in longdouble (K a scipy matrix of doubles; the products are exact in longdouble's wider mantissa only
    up to rounding at 2^-64)"""
    C = K.tocoo()
    r = np.asarray(b, dtype=LD).copy()
    np.subtract.at(r, C.row, C.data.astype(LD) * np.asarray(x, dtype=LD)[C.col])
    return r


def ext_solve(K, b, max_iter=60):
    """x with K x = b to about 2^-60 relative: splu in double, refined with longdouble residuals.  -> (x, converged)"""
    lu = spla.splu(sp.csc_matrix(K), permc_spec="COLAMD", diag_pivot_thresh=1.0)
    x = lu.solve(np.asarray(b, dtype=np.float64)).astype(LD)
    for _ in range(max_iter):
        d = lu.solve(residual_ld(K, x, b).astype(np.float64))
        x += d.astype(LD)
        if not np.all(np.isfinite(d)):
            return x, False
        if np.max(np.abs(d), initial=0.0) <= 2.0 ** -60 * float(np.max(np.abs(x), initial=0.0)):
            return x, True
    return x, False


def regulariser(diag, st):
    """eps of _compute_regularizer: constant + proportional * max |diag K|"""
    return st.static_regularization_constant + st.static_regularization_proportional * float(np.max(np.abs(diag), initial=0.0))


def shifted(nz, diag_idx, dsigns, eps):
    out = nz.copy()
    out[diag_idx] = nz[diag_idx] + np.where(dsigns == 1, eps, -eps)
    return out


@dataclass
class Refined:
    x: np.ndarray
    ok: bool
    n_solve: int
    eps: float
    steps: list = field(default_factory=list)     # norm of the residual after each accepted or rejected step


def refine(N, cp, rv, nz, dsigns, diag_idx, perm, st, b):
    """the reference's KKT solve of K x = b (nz: K's unregularised values, triu CSC) with the settings st"""
    import oracle
    eps = regulariser(nz[diag_idx], st) if st.static_regularization_enable else 0.0
    vals = shifted(nz, diag_idx, dsigns, eps) if st.static_regularization_enable else nz
    f = oracle.QDLDL((N, N), cp, rv, vals, perm, dsigns=dsigns, regularize_eps=st.dynamic_regularization_eps,
                     regularize_delta=st.dynamic_regularization_delta)
    x = f.solve(b)
    out = Refined(x, True, 1, eps)
    if not st.iterative_refinement_enable:
        out.ok = bool(np.all(np.isfinite(x)))
        return out
    K = full(N, cp, rv, nz)
    normb = np.max(np.abs(b), initial=0.0)
    e = b - K @ x
    norme = np.max(np.abs(e), initial=0.0)
    if not np.isfinite(norme):
        out.ok = False
        return out
    for _ in range(st.iterative_refinement_max_iter):
        if norme <= st.iterative_refinement_abstol + st.iterative_refinement_reltol * normb:
            break
        last = norme
        dx = f.solve(e) + x
        out.n_solve += 1
        e = b - K @ dx
        norme = np.max(np.abs(e), initial=0.0)
        out.steps.append(norme)
        if not np.isfinite(norme):
            out.ok = False
            return out
        if last / norme < st.iterative_refinement_stop_ratio:
            if last / norme > 1.0:
                x = dx
            break
        x = dx
    out.x = x
    return out
