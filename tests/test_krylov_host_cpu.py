"""The host state machine of cldl_solve_gmres (csrc/ldl_krylov.cpp) on dense matrices, without a CUDA runtime:
tests/host_harness/krylov_host.cpp implements its vector operations with plain loops, K dense and the preconditioner a
dense P = (K + E)^-1, x0 = P b.
- convergence within rank(E) + 1 steps (plus a small slack) for E of rank 1 to 8, x against numpy.linalg.solve;
- the Givens estimate |g_k| of each cycle against ||b - K x||_2 of the x the cycle formed;
- several cycles when the restart length is below the steps needed;
- the stagnation stop: K = diag(1, -1), P = 2 I, b = (-3, 1), m = 1, where r0 = (3, 3) is orthogonal to K P r0;
- a breakdown forced by tol = 0 (the Krylov space of I - E P is invariant after at most rank(E) + 1 steps);
- max_iter = 0, tol = 0 with max_iter steps, and an operation's error code passed on."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "clarabel.rs_b200", "csrc")
EPS = np.finfo(np.float64).eps
CAP = 256


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("krylov") / "krylov_host.so")
    cc = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I" + CSRC, "-o", so,
                         os.path.join(ROOT, "tests", "host_harness", "krylov_host.cpp"),
                         os.path.join(CSRC, "ldl_krylov.cpp")], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    L = C.CDLL(so)
    L.fgmres_c.restype = C.c_int
    return L


def _pd(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def run(lib, K, P, b, m, max_iter=100, tol=EPS, fail_at=-1):
    n = K.shape[0]
    K, P, b = (np.ascontiguousarray(a, dtype=np.float64) for a in (K, P, b))
    oi, od = np.zeros(5, np.int32), np.zeros(2)
    x, est, rn = np.empty(n), np.full(CAP, np.nan), np.full(CAP, np.nan)
    rc = lib.fgmres_c(n, _pd(K), _pd(P), _pd(b), m, max_iter, C.c_double(tol), fail_at,
                      oi.ctypes.data_as(C.POINTER(C.c_int)), _pd(od), _pd(x), _pd(est), _pd(rn), CAP)
    info = dict(zip(("iterations", "cycles", "analyses", "breakdowns", "nest"), map(int, oi)))
    info.update(omega1=od[0], omega2=od[1], estimates=est[:info["nest"]], rnorms=rn[:info["analyses"]])
    return rc, info, x


def omega(K, x, b):
    """omega1 + omega2 of x (the header's definitions), for the plain solve"""
    n = K.shape[0]
    r = b - K @ x
    kx = np.abs(K) @ np.abs(x)
    rmax = np.max(np.abs(K), axis=1)
    xn = np.max(np.abs(x))
    den1, den2 = kx + np.abs(b), kx + rmax * xn
    in1 = den1 > 1000 * n * EPS * (rmax * xn + np.abs(b))
    o1 = np.max(np.abs(r[in1]) / den1[in1]) if in1.any() else 0.0
    q = ~in1 & ((den2 != 0) | (r != 0))
    o2 = np.max(np.abs(r[q]) / den2[q]) if q.any() else 0.0
    return o1 + o2


def problem(rank, n=60, seed=0):
    """K symmetric indefinite and well conditioned, E symmetric of the given rank (orthonormal directions, |eigenvalues|
    0.5 to 2, either sign), P = (K + E)^-1"""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    K = (Q * np.r_[rng.uniform(1, 4, n // 2), -rng.uniform(1, 4, n - n // 2)]) @ Q.T
    U, _ = np.linalg.qr(rng.standard_normal((n, rank)))
    E = U @ np.diag(rng.uniform(0.5, 2, rank) * rng.choice([-1.0, 1.0], rank)) @ U.T
    return K, np.linalg.inv(K + E), rng.standard_normal(n)


@pytest.mark.parametrize("rank", range(1, 9))
def test_converges_within_rank_plus_one_steps(lib, rank):
    K, P, b = problem(rank, seed=rank)
    rc, info, x = run(lib, K, P, b, m=20)
    w0 = omega(K, P @ b, b)
    print("rank %d: %d steps, %d cycles, omega %.2e (x0 %.2e)" % (rank, info["iterations"], info["cycles"],
                                                                 info["omega1"] + info["omega2"], w0))
    assert rc == 0 and w0 > 1e-6
    assert info["omega1"] + info["omega2"] <= EPS
    assert info["iterations"] <= rank + 1 + 1 and info["cycles"] == 1
    xs = np.linalg.solve(K, b)
    assert np.max(np.abs(x - xs)) <= 1e-12 * np.max(np.abs(xs))
    assert omega(K, x, b) <= 4 * EPS


@pytest.mark.parametrize("m", [1, 3, 5])
def test_several_cycles_and_the_givens_estimate(lib, m):
    K, P, b = problem(8, seed=11)
    rc, info, x = run(lib, K, P, b, m=m, max_iter=400)
    assert rc == 0 and info["cycles"] >= 2 and info["omega1"] + info["omega2"] <= EPS
    # each corrected cycle's estimate against the residual of the x it formed (analysis c + 1), while that residual
    # is well above rounding
    est, rn = info["estimates"], info["rnorms"][1:]
    big = rn > 1e-8 * np.linalg.norm(b)
    assert big.sum() >= 2
    assert np.max(np.abs(est[big] - rn[big]) / rn[big]) <= 1e-8
    assert np.all(np.diff(info["rnorms"][: big.sum() + 1]) < 0)


def test_stagnation_stop(lib):
    K, P, b = np.diag([1.0, -1.0]), 2 * np.eye(2), np.array([-3.0, 1.0])
    rc, info, x = run(lib, K, P, b, m=1)
    assert rc == 0 and info["cycles"] == 1 and info["iterations"] == 1 and info["analyses"] == 2
    assert np.array_equal(x, np.array([-6.0, 2.0]))       # x0 = P b, r0 = (3, 3): no progress, x0 returned
    assert info["omega1"] + info["omega2"] == omega(K, x, b) > 0.5


@pytest.mark.parametrize("rank", [1, 4])
def test_breakdown_and_tol_zero(lib, rank):
    K, P, b = problem(rank, seed=20 + rank)
    rc, info, x = run(lib, K, P, b, m=30, max_iter=200, tol=0.0)
    assert rc == 0 and info["breakdowns"] >= 1
    assert info["iterations"] >= rank + 1 and info["iterations"] < 200      # stops at stagnation
    assert info["omega1"] + info["omega2"] <= EPS
    rc, info7, _ = run(lib, *problem(8, seed=11), m=30, max_iter=7, tol=0.0)
    assert rc == 0 and info7["iterations"] == 7 and info7["cycles"] == 1 and info7["breakdowns"] == 0


def test_max_iter_zero_returns_x0(lib):
    K, P, b = problem(3, seed=5)
    rc, info, x = run(lib, K, P, b, m=10, max_iter=0)
    assert rc == 0 and info["iterations"] == info["cycles"] == 0 and info["analyses"] == 1
    assert np.max(np.abs(x - P @ b)) <= 1e-13 * np.max(np.abs(x))          # x0 = P b, summed in the harness' order
    assert info["omega1"] + info["omega2"] == pytest.approx(omega(K, x, b), rel=1e-10)


def test_error_code_passed_on(lib):
    K, P, b = problem(3, seed=5)
    rc, info, _ = run(lib, K, P, b, m=10, fail_at=2)
    assert rc == 7 and info["iterations"] == 2
