"""The interior-point solver's host set-up (csrc/problem_setup.cpp) built with g++ against no CUDA runtime and checked
against the oracle and scipy: the KKT structure, the inf-bound presolve and its reverse, the Ruiz scalings bit for bit,
the symmetric and transposed CSR forms with their value maps, and the length of a caller's KKT permutation.
tests/host_harness/problem_setup_driver.cpp runs the set-up on one problem and writes out what it built."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
CSRC = os.path.join(ROOT, "clarabel.rs_b200", "csrc")

import clarabel_rs_b200 as cb  # noqa: E402
import oracle  # noqa: E402
import ref_problems as rp  # noqa: E402
import test_oracle_nonsym as ns  # noqa: E402
from helpers import workloads  # noqa: E402
from test_api_checks_cpu import equilibration_data  # noqa: E402


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("setup") / "problem_setup_driver")
    srcs = [os.path.join(ROOT, "tests", "host_harness", "problem_setup_driver.cpp"), os.path.join(CSRC, "problem_setup.cpp")]
    # the library's flags for its host sources (Makefile): the same arithmetic as the product
    cc = subprocess.run(["g++", "-O3", "-std=c++17", "-Wall", "-I" + CSRC, "-o", exe] + srcs, capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def _presolve_case(idx, cones):     # tests/presolve.rs
    n = 3
    P = sp.identity(n, format="csc")
    A = (2.0 * sp.vstack([sp.identity(n), -sp.identity(n)])).tocsc()
    b = np.ones(2 * n)
    b[idx] = 1e30
    return P, np.array([3., -2., 1.]), A, b, cones


def _genpow_mix():
    cones = [("nonneg", 5), ("genpow", ([0.2, 0.3, 0.5], 2)), ("soc", 9), ("genpow", ([0.5, 0.5], 1)), ("exp", 3),
             ("soc", 3), ("genpow", ([1.0], 4)), ("pow", 0.3)]
    m = 5 + 5 + 9 + 3 + 3 + 3 + 5 + 3
    rng = np.random.default_rng(0)
    A = sp.random(m, 12, density=0.3, random_state=3, format="csc") + \
        sp.vstack([sp.identity(12), sp.csc_matrix((m - 12, 12))]).tocsc()
    return sp.identity(12, format="csc"), rng.standard_normal(12), A, rng.standard_normal(m), cones


def _user_perm():       # a presolved row next to generalised power cones
    P, c, A, b, cones = ns.genpow_data()
    b = np.concatenate([b, [1e30, 2.0]])
    A = sp.vstack([A, sp.csc_matrix(np.array([[1., 0, 0, 0, 0, 0], [0, 1., 0, 0, 0, 0]]))]).tocsc()
    return P, c, A, b, cones + [("nonneg", 2)]


def _equilibration_case(kind):    # tests/equilibration_bounds.rs
    P, c, A, b, cones = equilibration_data()
    P, A = P.copy(), A.copy()
    if kind == "lower":
        P.data[0] = 1e-15
    elif kind == "upper":
        A.data[0] = 1e15
    else:
        A.data[:] = 0.0
    return P, c, A, b, cones


def _workload(name):
    if name == "entropy_power_mix":
        pr = workloads.entropy_power_mix(40, 20, n_eq=3, seed=6)
    elif name == "portfolio":
        pr = workloads.portfolio_socp(n_assets=120, n_soc=6, soc_dim=9, block=30, seed=7)
    elif name == "sdp":
        pr = workloads.block_sdp(n=60, n_psd=4, psd_dim=4, nnz_per_row=3, window=20, n_nonneg=10, seed=4)
    else:               # the mixed block SDP of tests/test_zz_equilibration_gpu.py
        pr = workloads.block_sdp(n=60, n_psd=3, psd_dim=4, nnz_per_row=3, window=20, n_nonneg=10, seed=4)
    return pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"]


PRESOLVED = {"presolve1": [3], "presolve2": [4], "presolve3": [0, 1, 2], "presolve_all": list(range(6))}
PROBLEMS = {
    "qp": rp.basic_qp, "lp": rp.basic_lp, "socp": rp.basic_socp, "hs35": rp.hs35, "box_qp3": rp.box_qp3,
    "exp": ns.expcone_data, "mixed": ns.mixed_conic_data, "genpow": ns.genpow_data, "genpow_mix": _genpow_mix,
    "entropy_power_mix": lambda: _workload("entropy_power_mix"), "portfolio": lambda: _workload("portfolio"),
    "sdp": lambda: _workload("sdp"), "mixed_sdp": lambda: _workload("mixed_sdp"),
    "presolve1": lambda: _presolve_case([3], [("nonneg", 3), ("nonneg", 3)]),
    "presolve2": lambda: _presolve_case([4], [("zero", 2), ("nonneg", 4)]),
    "presolve3": lambda: _presolve_case([0, 1, 2], [("nonneg", 3), ("nonneg", 3)]),
    "presolve_all": lambda: _presolve_case(list(range(6)), [("nonneg", 3), ("nonneg", 3)]),
    "user_perm": _user_perm,
    "equilibrate_lower": lambda: _equilibration_case("lower"), "equilibrate_upper": lambda: _equilibration_case("upper"),
    "equilibrate_zero_rows": lambda: _equilibration_case("zero"),
}


def _inputs(P, A):
    """P and A as the product's constructor passes them on (CudaSolver.__init__)"""
    P = sp.triu(sp.csc_matrix(P), format="csc")
    A = sp.csc_matrix(A)
    P.sort_indices()
    A.sort_indices()
    return P, A


def _run(driver, tmp_path, P, q, A, b, cones, perm=None, infbound=1e20):
    P, A = _inputs(P, A)
    n, m = P.shape[0], A.shape[0]
    st = cb.default_settings()
    u64 = lambda a: np.ascontiguousarray(a, dtype=np.uint64)
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    galpha = [a for k, d in cones if k == "genpow" for a in d[0]]
    perm = [] if perm is None else perm
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        np.array([n, m, P.nnz, A.nnz, len(cones), len(galpha), st.presolve_enable, st.equilibrate_enable,
                  st.equilibrate_max_iter, len(perm)], dtype=np.int64).tofile(f)
        f64([infbound, st.equilibrate_min_scaling, st.equilibrate_max_scaling]).tofile(f)
        for a in (u64(P.indptr), u64(P.indices), f64(P.data), f64(q), u64(A.indptr), u64(A.indices), f64(A.data), f64(b)):
            a.tofile(f)
        np.array([cb.CONE_CODES[k] for k, _ in cones], dtype=np.int64).tofile(f)
        u64([3 if k in ("exp", "pow") else (len(d[0]) if k == "genpow" else d) for k, d in cones]).tofile(f)
        f64([float(d) if k == "pow" else 0.0 for k, d in cones]).tofile(f)
        u64([int(d[1]) if k == "genpow" else 0 for k, d in cones]).tofile(f)
        f64(galpha).tofile(f)
        u64(perm).tofile(f)
    r = subprocess.run([driver, fin, fout], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    out, raw, i = {}, open(fout, "rb").read(), 0
    while i < len(raw):
        ln = int(np.frombuffer(raw, np.int32, 1, i)[0]); i += 4
        key = raw[i:i + ln].decode(); i += ln
        dt = np.float64 if raw[i:i + 1] == b"f" else np.int64; i += 1
        cnt = int(np.frombuffer(raw, np.int64, 1, i)[0]); i += 8
        out[key] = np.frombuffer(raw, dt, cnt, i); i += 8 * cnt
    assert out["rc"][0] == 0, out["rc"]
    return out


@pytest.fixture(scope="module")
def results(driver, tmp_path_factory):
    res = {}
    for name, make in PROBLEMS.items():
        args = make()
        perm = None
        if name == "user_perm":         # n + rows left after the presolve + 3 expansion columns per GenPow cone
            perm = np.arange(6 + (8 + 1) + 6)[::-1].copy()
        res[name] = (args, _run(driver, tmp_path_factory.mktemp(name), *args, perm=perm))
    return res


@pytest.mark.parametrize("name", list(PROBLEMS))
def test_kkt_structure_equals_the_oracles(results, name):
    args, d = results[name]
    ora = oracle.IPM(*args)
    N, cp, rv, _, ds = ora.kkt()
    assert d["K.N"][0] == N and d["m_reduced"][0] == ora.m_reduced
    assert np.array_equal(d["K.Kp"], cp) and np.array_equal(d["K.Ki"], rv) and np.array_equal(d["K.dsigns"], ds)


@pytest.mark.parametrize("name", list(PROBLEMS))
def test_equilibration_is_bitwise_the_oracles(results, name):
    args, d = results[name]
    do, eo, co = oracle.IPM(*args).equilibration()
    assert np.array_equal(d["eq.d"], do) and np.array_equal(d["eq.e"], eo) and d["eq.c"][0] == co


def test_equilibration_bounds(results):
    st = cb.default_settings()
    for name in ("equilibrate_lower", "equilibrate_upper"):
        d, e = results[name][1]["eq.d"], results[name][1]["eq.e"]
        assert d.min() >= st.equilibrate_min_scaling and e.min() >= st.equilibrate_min_scaling, name
        assert d.max() <= st.equilibrate_max_scaling and e.max() <= st.equilibrate_max_scaling, name
    assert np.all(results["equilibrate_zero_rows"][1]["eq.e"] == 1.0)


@pytest.mark.parametrize("name", list(PRESOLVED))
def test_presolve_drops_the_infinite_rows_and_reverse_puts_them_back(results, name):
    args, d = results[name]
    m = args[2].shape[0]
    dropped = np.isin(np.arange(m), PRESOLVED[name])
    assert np.array_equal(d["keep"].astype(bool), ~dropped)
    assert d["m_reduced"][0] == m - dropped.sum()
    assert d["A.rowval"].size == 0 or d["A.rowval"].max() < d["m_reduced"][0]
    # an iterate of ones with t = 1: the kept rows unscale, the dropped ones get s = bound and z = 0
    e, c = d["eq.e"], d["eq.c"][0]
    z, s = d["sol.z"], d["sol.s"]
    assert np.all(z[dropped] == 0.0) and np.all(s[dropped] == 1e20)
    assert np.array_equal(z[~dropped], e * (1.0 / c)) and np.array_equal(s[~dropped], 1.0 / e)
    assert np.array_equal(d["sol.x"], d["eq.d"])


@pytest.mark.parametrize("name", list(PROBLEMS))
def test_transposes_rebuild_their_matrices(results, name):
    _, d = results[name]
    n = len(d["P.colptr"]) - 1
    m = int(d["m_reduced"][0])
    P = sp.csc_matrix((d["P.nzval"], d["P.rowval"], d["P.colptr"]), shape=(n, n))
    full = (P + P.T - sp.diags(P.diagonal())).tocsr()
    Ps = sp.csr_matrix((d["P.nzval"][d["Psym.src"]], d["Psym.col"], d["Psym.rowptr"]), shape=(n, n))
    assert (Ps != full).nnz == 0 and Ps.has_sorted_indices
    A = sp.csc_matrix((d["A.nzval"], d["A.rowval"], d["A.colptr"]), shape=(m, n))
    Ac = sp.csr_matrix((d["A.nzval"][d["Acsr.src"]], d["Acsr.col"], d["Acsr.rowptr"]), shape=(m, n))
    assert (Ac != A.tocsr()).nnz == 0 and Ac.nnz == A.nnz
    # K with distinct values, so that a wrong source position cannot go unnoticed
    N, Kp, Ki = int(d["K.N"][0]), d["K.Kp"], d["K.Ki"]
    kv = np.arange(1.0, len(Ki) + 1.0)
    K = sp.csc_matrix((kv, Ki, Kp), shape=(N, N))
    Kfull = (K + K.T - sp.diags(K.diagonal())).tocsr()
    Ks = sp.csr_matrix((kv[d["Ksym.src"]], d["Ksym.col"], d["Ksym.rowptr"]), shape=(N, N))
    assert (Ks != Kfull).nnz == 0 and Ks.nnz == 2 * len(Ki) - N


def test_caller_permutation_has_the_length_of_the_assembled_system(results):
    _, d = results["user_perm"]
    N = int(d["K.N"][0])
    assert N == 6 + (8 + 1) + 6 and d["m_reduced"][0] == 9
    assert np.array_equal(d["kkt_perm"], np.arange(N)[::-1])
