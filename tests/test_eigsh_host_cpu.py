"""The host state machine of cldl_eigsh (csrc/ldl_eig.cpp) on dense operators, without a CUDA runtime:
tests/host_harness/eig_host.cpp implements its vector operations with plain loops on T = (A - sigma M)^-1 M.
- the cyclic Jacobi eigensolve against numpy.linalg.eigh on random symmetric, tridiagonal and arrowhead matrices;
- full thick-restart runs against dense eigenvalues, identity and generalised M, with restarts;
- locking and ordering: converged pairs come first, each group ascending in 1/theta, status 0 at max_restarts;
- deflation: an invariant Krylov space (beta = 0) continued by fresh vectors;
- M not positive definite (status -1) and an operation's error code passed on."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "clarabel.rs_b200", "csrc")
EPS = np.finfo(np.float64).eps


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("eig") / "eig_host.so")
    cc = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I" + CSRC, "-o", so,
                         os.path.join(ROOT, "tests", "host_harness", "eig_host.cpp"), os.path.join(CSRC, "ldl_eig.cpp")],
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return C.CDLL(so)


def _pd(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def jacobi(lib, A):
    m = A.shape[0]
    A = np.ascontiguousarray(A, dtype=np.float64)
    th, Y = np.empty(m), np.empty((m, m))
    lib.eig_jacobi_c(m, _pd(A), _pd(th), _pd(Y))
    return th, Y


def run(lib, T, M, nev, ncv, max_restarts=300, tol=0.0, nr=16, seed=0, fail_at=-1):
    n = T.shape[0]
    R = np.asfortranarray(np.random.default_rng(seed).standard_normal((n, nr)))
    T = np.ascontiguousarray(T)
    Mc = None if M is None else np.ascontiguousarray(M)
    oi = np.zeros(5, np.int32)
    th, X = np.full(nev, np.nan), np.zeros((n, nev), order="F")
    lib.eig_run_c.restype = C.c_int
    rc = lib.eig_run_c(n, _pd(T), None if Mc is None else _pd(Mc), _pd(R), nr, nev, ncv, max_restarts, C.c_double(tol),
                       fail_at, oi.ctypes.data_as(C.POINTER(C.c_int)), _pd(th), _pd(X))
    return rc, dict(zip(("status", "nconv", "restarts", "applies", "deflations"), map(int, oi))), th, X


def _lap(nx, ny):
    T1 = lambda k: 2 * np.eye(k) - np.eye(k, k=1) - np.eye(k, k=-1)
    return np.kron(np.eye(ny), T1(nx)) + np.kron(T1(ny), np.eye(nx))


@pytest.mark.parametrize("kind", ["random", "tridiagonal", "arrowhead", "graded"])
@pytest.mark.parametrize("m", [1, 2, 7, 40])
def test_jacobi_against_numpy(lib, kind, m):
    rng = np.random.default_rng(m)
    if kind == "random":
        A = rng.standard_normal((m, m)); A = A + A.T
    elif kind == "tridiagonal":
        A = np.diag(rng.standard_normal(m)) + np.diag(rng.standard_normal(m - 1), 1) + np.diag(np.zeros(m - 1), -1)
        A = np.triu(A) + np.triu(A, 1).T
    elif kind == "arrowhead":
        A = np.diag(rng.standard_normal(m))
        A[:-1, -1] = A[-1, :-1] = rng.standard_normal(m - 1)
    else:
        d = 10.0 ** -np.arange(m)
        A = np.outer(d, d) * (rng.standard_normal((m, m)) * 0.1) + np.diag(d * d)
        A = A + A.T
    th, Y = jacobi(lib, A)
    ref = np.linalg.eigvalsh(A)
    scale = max(np.max(np.abs(ref)), 1e-300)
    assert np.max(np.abs(np.sort(th) - ref)) <= 50 * m * EPS * scale
    assert np.max(np.abs(Y.T @ Y - np.eye(m))) <= 50 * m * EPS
    assert np.max(np.abs(A @ Y - Y * th)) <= 50 * m * EPS * scale
    assert (th, Y)[0].tobytes() == jacobi(lib, A)[0].tobytes()


@pytest.mark.parametrize("sigma,nev", [(0.0, 1), (0.0, 6), (0.0, 32), (3.3, 6), (3.3, 12)])
def test_thick_restart_against_dense_eigenvalues(lib, sigma, nev):
    A = _lap(13, 9)
    n = A.shape[0]
    T = np.linalg.inv(A - sigma * np.eye(n))
    ex = np.linalg.eigvalsh(A)
    rc, info, th, X = run(lib, T, None, nev, min(n, max(2 * nev + 1, 20)))
    assert rc == 0 and info["status"] == 1 and info["nconv"] == nev
    lam = sigma + 1.0 / th
    near = np.sort(ex[np.argsort(np.abs(ex - sigma), kind="stable")[:nev]])
    assert np.max(np.abs(lam - near)) <= 1e-12 * np.max(np.abs(ex))
    assert np.all(np.diff(lam) >= 0)
    assert np.max(np.abs(X.T @ X - np.eye(nev))) <= 1e-13
    assert np.max(np.abs(A @ X - X * lam)) <= 1e-11


def test_generalised_with_restarts(lib):
    rng = np.random.default_rng(3)
    n = 60
    Q = rng.standard_normal((n, n))
    M = Q @ Q.T / n + np.eye(n)
    A = _lap(6, 10)
    import scipy.linalg as sla
    ex = sla.eigh(A, M, eigvals_only=True)
    rc, info, th, X = run(lib, np.linalg.solve(A, M), M, 5, 12)
    assert rc == 0 and info["status"] == 1 and info["restarts"] > 0
    assert np.max(np.abs(1.0 / th - ex[:5])) <= 1e-12 * ex[-1]
    assert np.max(np.abs(X.T @ M @ X - np.eye(5))) <= 1e-13


def test_locking_and_ordering_when_not_all_converge(lib):
    """max_restarts 0: the converged wanted pairs come first, then the others, each ascending in 1/theta; the
    converged ones stay converged when restarts are allowed"""
    A = _lap(20, 15)
    n = A.shape[0]
    T = np.linalg.inv(A)
    rc, info, th, X = run(lib, T, None, 8, 17, max_restarts=0)
    assert rc == 0 and info["status"] == 0 and 0 < info["nconv"] < 8
    k = info["nconv"]
    assert np.all(np.diff(1.0 / th[:k]) >= 0) and np.all(np.diff(1.0 / th[k:]) >= 0)
    ex = np.linalg.eigvalsh(A)
    for t in th[:k]:                 # each converged pair is an eigenvalue to its tolerance
        assert np.min(np.abs(1.0 / t - ex)) <= 1e-10
    rc, info2, th2, _ = run(lib, T, None, 8, 17)
    assert info2["status"] == 1 and info2["restarts"] > 0
    assert np.max(np.abs(1.0 / th2 - ex[:8])) <= 1e-12 * ex[-1]


def test_deflation_of_an_invariant_krylov_space(lib):
    B = np.diag(np.arange(1.0, 6.0) * 1.5) + np.diag(-0.4 * np.ones(4), 1) + np.diag(-0.4 * np.ones(4), -1)
    A = np.kron(np.eye(3), B)                    # triple eigenvalues: Krylov spaces of dimension 5
    rc, info, th, X = run(lib, np.linalg.inv(A), None, 3, 12)
    assert rc == 0 and info["status"] == 1 and info["deflations"] >= 2
    mu = np.linalg.eigvalsh(B)[0]
    assert np.max(np.abs(1.0 / th - mu)) <= 1e-13
    assert np.max(np.abs(X.T @ X - np.eye(3))) <= 1e-13


@pytest.mark.parametrize("n", [2, 3, 5])
def test_basis_is_the_whole_space(lib, n):
    A = _lap(n, 1)
    rc, info, th, X = run(lib, np.linalg.inv(A), None, n - 1, n)
    assert rc == 0 and info["status"] == 1 and info["restarts"] == 0 and info["applies"] == n
    assert np.max(np.abs(np.sort(1.0 / th) - np.linalg.eigvalsh(A)[:n - 1])) <= 1e-13


def test_m_not_positive_definite_and_errors_passed_on(lib):
    A = _lap(5, 4)
    n = A.shape[0]
    rc, info, th, _ = run(lib, np.linalg.inv(A), -np.eye(n), 2, 8)
    assert rc == 0 and info["status"] == -1 and info["nconv"] == 0 and np.all(np.isnan(th))
    rc, info, _, _ = run(lib, np.linalg.inv(A), None, 2, 8, fail_at=3)
    assert rc == 7
