"""tests/golden/*.json (the reference's end-to-end known answers, see tests/golden/README.md) through the CPU oracle
(not gpu) and through the CUDA path (gpu)."""
import glob
import importlib.util
import json
import os

import numpy as np
import pytest

import clarabel_rs_b200 as cb
import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
FILES = sorted(glob.glob(os.path.join(HERE, "golden", "*.json")))
_spec = importlib.util.spec_from_file_location("jsonio", os.path.join(os.path.dirname(cb.pkg.__file__), "jsonio.py"))
jsonio = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(jsonio)


def _check(r, exp):
    assert r["status"] == exp["status"], (r["status"], exp)
    if "x" in exp:
        assert np.linalg.norm(r["x"] - np.asarray(exp["x"])) <= exp["x_tol"], (r["x"], exp)
    if "obj" in exp:
        assert abs(r["obj_val"] - exp["obj"]) <= exp["obj_tol"], (r["obj_val"], exp)


def test_fixture_set_is_complete():
    assert len(FILES) >= 14
    for f in FILES:
        exp = json.load(open(f))["expected"]
        assert exp["source"] and exp["status"]


@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f)[:-5] for f in FILES])
def test_oracle_reaches_the_reference_answer(path):
    d = jsonio.load_problem(path)
    exp = json.load(open(path))["expected"]
    ipm = oracle.IPM(d["P"], d["q"], d["A"], d["b"], d["cones"], settings=oracle.default_settings(**d["settings"]) if d["settings"] else None)
    ipm.set_perm(np.arange(ipm.N))
    _check(ipm.solve(), exp)


@pytest.mark.gpu
@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f)[:-5] for f in FILES])
def test_device_reaches_the_reference_answer(path):
    d = jsonio.load_problem(path)
    exp = json.load(open(path))["expected"]
    dev = cb.CudaSolver(d["P"], d["q"], d["A"], d["b"], d["cones"], settings=cb.default_settings(**d["settings"]) if d["settings"] else None)
    r = dev.solve()
    if os.path.basename(path) == "mixed_conic_dual_strategy.json":
        # the apex of every cone is the optimum (see tests/test_oracle_nonsym.py::test_iteration_count_under_last_bit_noise):
        # the optimum must be reached, the status label is not stable under last-bit differences
        assert r["status"] in ("Solved", "AlmostSolved", "InsufficientProgress") and abs(r["info"].cost_primal - exp["obj"]) <= 1e-6
        return
    _check(r, exp)
    ora = oracle.IPM(d["P"], d["q"], d["A"], d["b"], d["cones"], settings=oracle.default_settings(**d["settings"]) if d["settings"] else None)
    ora.set_perm(dev.kkt_perm())
    ro = ora.solve()
    assert r["status"] == ro["status"]
    if all(k in ("zero", "nonneg", "soc", "psd") for k, _ in d["cones"]):
        assert r["iterations"] == ro["iterations"]          # symmetric cones: identical iteration counts
    else:
        # nonsymmetric cones: the iteration count is not stable under last-bit differences of the cone arithmetic
        # (tests/test_oracle_nonsym.py::test_iteration_count_under_last_bit_noise)
        assert r["iterations"] <= 2 * ro["iterations"] + 10
