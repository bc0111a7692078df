"""Termination callbacks and verbose output of the device solver (core/solver.rs set_termination_callback(_c),
default/info_print.rs, src/io/mod.rs print targets), following the reference's tests/callbacks.rs and
tests/print_streams.rs.  tests/test_callbacks_print_cpu.py runs this module against the CUDA-on-CPU emulated build."""
import ctypes as C
import io

import numpy as np
import pytest
import scipy.sparse as sp

import clarabel_rs_b200 as cb
from helpers import workloads
from ref_problems import basic_qp

pytestmark = pytest.mark.gpu


def univariate(settings=None):
    """the 1-variable problem of tests/callbacks.rs and tests/print_streams.rs: P = I, q = 0, A = I, b = 1, x >= ..."""
    I1 = sp.identity(1, format="csc")
    return cb.CudaSolver(I1, [0.0], I1, [1.0], [("nonneg", 1)], settings)


def stop_at_3(info):
    return info.iterations >= 3


# ------------------------------------------------------------------------------------------ tests/callbacks.rs
def test_callbacks():
    s = univariate()
    s.set_termination_callback(stop_at_3)
    r = s.solve()
    assert r["status"] == "CallbackTerminated" and r["iterations"] == 3
    s.unset_termination_callback()
    assert s.solve()["status"] == "Solved"
    always = cb.CALLBACK_FN(lambda info, data: 1)           # a C callback: terminate immediately
    s.set_termination_callback_c(always)
    r = s.solve()
    assert r["status"] == "CallbackTerminated" and r["iterations"] == 0


def test_callbacks_with_state():
    s = univariate()
    s.set_termination_callback(stop_at_3)
    assert s.solve()["status"] == "CallbackTerminated"
    s.unset_termination_callback()
    assert s.solve()["status"] == "Solved"

    class State(C.Structure):
        _fields_ = [("counter", C.c_int)]

    def with_state(info, data):
        st = C.cast(data, C.POINTER(State)).contents
        st.counter += 1
        return 1 if st.counter >= 3 else 0

    state = State(-1)
    fn = cb.CALLBACK_FN(with_state)
    s.set_termination_callback_c(fn, C.cast(C.pointer(state), C.c_void_p))
    r = s.solve()
    assert r["status"] == "CallbackTerminated" and r["iterations"] == 3
    assert state.counter == 3


def test_callback_status_keeps_the_current_iterate():
    """the solution of a stopped solve is the iterate the callback saw, unscaled like any other ending"""
    P, q, A, b, cones = basic_qp()
    seen = []
    s = cb.CudaSolver(P, q, A, b, cones)
    s.set_termination_callback(lambda info: seen.append(info.cost_primal) or info.iterations >= 4)
    r = s.solve()
    assert r["status"] == "CallbackTerminated" and r["iterations"] == 4
    assert r["info"].cost_primal == seen[-1]
    full = cb.CudaSolver(P, q, A, b, cones).solve()
    assert full["iterations"] > 4 and not np.array_equal(r["x"], full["x"])
    assert np.all(np.isfinite(r["x"])) and np.max(np.abs(r["x"] - full["x"])) < 1.0


# ------------------------------------------------------------------------- the callback sees the reported numbers
FIELDS = ("iterations", "mu", "step_length", "sigma", "res_primal", "res_dual", "gap_abs")


def problems():
    pr = workloads.random_sparse_qp(n=150, m=300, nnz_per_row=3, seed=5, window=20)
    return {"basic_qp": basic_qp(), "random_sparse_qp": (pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"])}


@pytest.mark.parametrize("name", ["basic_qp", "random_sparse_qp"])
def test_callback_sees_the_trace_bit_for_bit(name):
    P, q, A, b, cones = problems()[name]
    s = cb.CudaSolver(P, q, A, b, cones)
    plain = s.solve()
    rows = []
    s.set_termination_callback(lambda info: rows.append(tuple(getattr(info, f) for f in FIELDS)) and False)
    r = s.solve()
    assert r["status"] == plain["status"] == "Solved" and r["iterations"] == plain["iterations"]
    assert [row[0] for row in rows] == list(range(len(rows))) and len(rows) == r["iterations"] + 1
    assert np.array_equal(np.array([row[1:] for row in rows]), s.trace)      # mu, alpha, sigma, pres, dres, gap
    for k in ("x", "z", "s"):
        assert np.array_equal(r[k], plain[k]), k


# ------------------------------------------------------------------------------------ tests/print_streams.rs
def test_print_to_buffer():
    s = univariate(cb.default_settings(verbose=1))
    s.print_to_buffer()
    s.solve()
    assert "Clarabel.rs" in s.get_print_buffer()
    assert "Clarabel.rs" in s.get_print_buffer()        # reading does not clear it


def test_print_to_file_and_stream_receive_the_same_text(tmp_path):
    path = tmp_path / "out.txt"
    a = univariate(cb.default_settings(verbose=1))
    a.print_to_file(str(path))
    a.solve()
    text = path.read_text()
    assert "Clarabel.rs" in text
    b = univariate(cb.default_settings(verbose=1))
    st = io.StringIO()
    b.print_to_stream(st)
    b.solve()
    strip = lambda t: [l for l in t.splitlines() if not l.startswith("solve time")]
    assert strip(st.getvalue()) == strip(text)
    a.solve()                                               # the file target appends
    assert path.read_text().count("Clarabel.rs") == 2


def test_print_to_sink(capfd):
    s = univariate(cb.default_settings(verbose=1))
    s.print_to_sink()
    s.solve()
    out, err = capfd.readouterr()
    assert out == "" and err == ""
    with pytest.raises(cb.BackendError):
        s.get_print_buffer()


def test_print_to_stdout(capfd):
    s = univariate(cb.default_settings(verbose=1))
    s.print_to_stdout()
    s.solve()
    out, _ = capfd.readouterr()
    assert "Clarabel.rs" in out and "Terminated with status = Solved" in out


# ----------------------------------------------------------------------------------------------- the table
def row_text(info):
    nums = [f"{info.cost_primal:+.4e}", f"{info.cost_dual:+.4e}", f"{min(info.gap_abs, info.gap_rel):.2e}",
            f"{info.res_primal:.2e}", f"{info.res_dual:.2e}", f"{info.ktratio:.2e}", f"{info.mu:.2e}"]
    step = f"{info.step_length:.2e}  " if info.iterations > 0 else " ------   "
    return f"{info.iterations:>3}  " + "".join(v + "  " for v in nums) + step


@pytest.mark.parametrize("name", ["basic_qp", "random_sparse_qp"])
def test_table_rows_are_the_callback_info(name):
    P, q, A, b, cones = problems()[name]
    s = cb.CudaSolver(P, q, A, b, cones, cb.default_settings(verbose=1))
    s.print_to_buffer()
    seen = []
    s.set_termination_callback(lambda info: seen.append(row_text(info)) and False)
    r = s.solve()
    lines = s.get_print_buffer().splitlines()
    h = next(i for i, l in enumerate(lines) if l.startswith("iter    pcost"))
    assert set(lines[h + 1]) == {"-"}
    end = next(i for i in range(h + 2, len(lines)) if set(lines[i]) == {"-"})
    table = lines[h + 2:end]
    assert [int(l.split()[0]) for l in table] == list(range(r["iterations"] + 1))
    assert table == seen
    assert lines[end + 1] == "Terminated with status = " + r["status"]
    assert lines[end + 2].startswith("solve time = ")
    text = "\n".join(lines)
    for key in ("problem:", "  variables     = %d" % s.n, "  constraints   = %d" % s.m, "  nnz(A)        = %d" % A.nnz,
                "linear algebra: direct / cudaldl, precision: 64 bit", "Nonnegative = "):
        assert key in text, key


# ------------------------------------------------------------------------------------------------ off means off
def test_default_settings_print_nothing(capfd):
    P, q, A, b, cones = basic_qp()
    s = cb.CudaSolver(P, q, A, b, cones)
    assert s.settings.verbose == 0
    assert s.solve()["status"] == "Solved"
    out, err = capfd.readouterr()
    assert out == "" and err == ""
    s.update_settings(verbose=1)                            # no rebuild of the handle
    s.solve()
    out, _ = capfd.readouterr()
    assert "Terminated with status = Solved" in out


def test_features_launch_no_kernels():
    P, q, A, b, cones = problems()["random_sparse_qp"]
    s = cb.CudaSolver(P, q, A, b, cones)
    c0 = cb.launch_count()
    r0 = s.solve()
    off = cb.launch_count() - c0
    s.update_settings(verbose=1)
    s.print_to_buffer()
    s.set_termination_callback(lambda info: False)
    c1 = cb.launch_count()
    r1 = s.solve()
    assert cb.launch_count() - c1 == off and r1["iterations"] == r0["iterations"]
    assert "Terminated with status = Solved" in s.get_print_buffer()


# ----------------------------------------------------------------------------------------------- Python errors
def test_exception_in_callback_is_raised_by_solve():
    P, q, A, b, cones = basic_qp()
    s = cb.CudaSolver(P, q, A, b, cones)

    def boom(info):
        if info.iterations == 2:
            raise ValueError("stop here")
        return False

    s.set_termination_callback(boom)
    with pytest.raises(ValueError, match="stop here"):
        s.solve()
    s.unset_termination_callback()
    assert s.solve()["status"] == "Solved"
