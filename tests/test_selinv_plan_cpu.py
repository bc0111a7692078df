"""The selected-inversion plan (build_selinv_plan in csrc/ldl_plan.cpp) built on the host, without a CUDA runtime, and
checked for what k_selinv relies on:
- every entry (r1, r2), r1 >= r2, of every front's Z_RR resolves through the gather maps to the panel position whose
  row and column really are (r1, r2) -- in the front that owns column r2, inside that front's panel;
- every task comes after the task that completes its parent's Z panel (co-resident CTAs spin on that flag: a task
  queued before its dependency can deadlock the kernel), a pivot-block task after all row tasks of its front, and
  the row-task counters match the queue;
- the caller-order map sends every stored entry of the caller's upper triangle to the panel position of that entry
  in the permuted order, and no two entries to the same position.
tests/host_harness/selinv_plan_driver.cpp builds the plan with g++ and writes it out.  The matrices are the LDL shape
matrices of tests/ldl_shapes.py (every front shape the kernels dispatch on) and random KKT matrices."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
CSRC = os.path.join(ROOT, "clarabel.rs_b200", "csrc")

import ldl_shapes  # noqa: E402
from helpers import workloads  # noqa: E402

SI_RB = 64


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("selinv") / "selinv_plan_driver")
    srcs = [os.path.join(ROOT, "tests", "host_harness", "selinv_plan_driver.cpp")] + \
           [os.path.join(CSRC, f) for f in ("ldl_plan.cpp", "symbolic.cpp", "ordering.cpp")]
    cc = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-I" + CSRC, "-o", exe] + srcs,
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def _matrix(name):
    if name in ("big_fronts", "child_records"):
        sh = getattr(ldl_shapes, name)()
        return sh.N, sh.cp, sh.rv, np.asarray(sh.perm, dtype=np.int32)
    if name == "random_qp":
        pr = workloads.random_sparse_qp(n=2000, m=4000, nnz_per_row=5, seed=1, window=200)
    else:
        pr = workloads.block_angular_qp(n=8000, nblocks=8, nlink=100, link_blocks=4, seed=3)
    N, cp, rv, _, _ = workloads.kkt_triu(pr["P"], pr["A"], np.full(pr["A"].shape[0], 1e-3))
    return N, cp, rv, None


_PLANS = {}


def _run(driver, tmp_path, name):
    if name not in _PLANS:
        _PLANS[name] = _build(driver, tmp_path, name)
    return _PLANS[name]


def _build(driver, tmp_path, name):
    N, cp, rv, perm = _matrix(name)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        np.array([N, len(rv), perm is not None], dtype=np.int64).tofile(f)
        np.asarray(cp, dtype=np.int64).tofile(f)
        np.asarray(rv, dtype=np.int32).tofile(f)
        if perm is not None:
            perm.tofile(f)
    r = subprocess.run([driver, fin, fout], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    out, raw, i = {}, open(fout, "rb").read(), 0
    while i < len(raw):
        ln = int(np.frombuffer(raw, np.int32, 1, i)[0]); i += 4
        key = raw[i:i + ln].decode(); i += ln
        cnt = int(np.frombuffer(raw, np.int64, 1, i)[0]); i += 8
        out[key] = np.frombuffer(raw, np.int64, cnt, i); i += 8 * cnt
    return N, np.asarray(cp), np.asarray(rv), out


class Panels:
    """decodes an offset into the factor's panel storage to (front, global row, global column)"""

    def __init__(self, d):
        self.first, self.rowptr, self.rows = d["sym.sn_first"], d["sym.sn_rowptr"], d["sym.sn_rows"]
        self.off = d["sym.panel_off"]
        self.ns, self.nr = np.diff(self.first), np.diff(self.rowptr)

    def decode(self, pos):
        a = np.searchsorted(self.off, pos, side="right") - 1
        ld = self.ns[a] + self.nr[a]
        loc = pos - self.off[a]
        assert (loc >= 0).all() and (loc < ld * self.ns[a]).all(), "offset outside every panel"
        c, r = loc // ld, loc % ld
        col = self.first[a] + c
        piv = r < self.ns[a]
        row = np.where(piv, self.first[a] + r, self.rows[np.where(piv, 0, self.rowptr[a] + r - self.ns[a])])
        return a, row, col


NAMES = ["big_fronts", "child_records", "random_qp", "block_angular"]


@pytest.mark.parametrize("name", NAMES)
def test_gathers_resolve_to_their_entries(driver, tmp_path, name):
    _, _, _, d = _run(driver, tmp_path, name)
    P = Panels(d)
    col, seg, segpos = d["col"], d["seg"], d["segpos"]
    first = P.first
    owner = np.searchsorted(first, np.arange(first[-1]), side="right") - 1
    n_checked = 0
    for s in range(len(P.ns)):
        nr, rp = int(P.nr[s]), int(P.rowptr[s])
        if nr == 0:
            continue
        R = P.rows[rp:rp + nr]
        I, K = np.tril_indices(nr)          # i >= k
        pos = col[rp + K] + segpos[seg[rp + K] + I]
        a, row, c = P.decode(pos)
        assert np.array_equal(c, R[K]) and np.array_equal(row, R[I]), (name, s)
        assert np.array_equal(a, owner[R[K]]), (name, s)
        n_checked += pos.size
    assert n_checked > 0
    print("%s: %d gathered entries checked, %d segment positions" % (name, n_checked, segpos.size))


@pytest.mark.parametrize("name", NAMES)
def test_every_task_comes_after_its_dependencies(driver, tmp_path, name):
    _, _, _, d = _run(driver, tmp_path, name)
    kind, s, parent, r0, r1, nr = d["t.kind"], d["t.s"], d["t.parent"], d["t.r0"], d["t.r1"], d["t.nr"]
    nsup = len(d["sym.sn_parent"])
    assert np.array_equal(parent, d["sym.sn_parent"][s])
    done_at = np.full(nsup, -1)            # task that completes the front's Z panel
    rows_seen = np.zeros(nsup, np.int64)
    row_cover = {}
    for t in range(len(kind)):
        k, f = int(kind[t]), int(s[t])
        if k in (0, 1):
            p = int(parent[t])
            assert p < 0 or 0 <= done_at[p] < t, (name, t, "queued before its parent completes")
        if k == 0:
            assert nr[t] <= SI_RB and r0[t] == 0 and r1[t] == nr[t]
        if k == 1:
            assert nr[t] > SI_RB and done_at[f] < 0
            rows_seen[f] += 1
            row_cover.setdefault(f, []).append((int(r0[t]), int(r1[t])))
        if k == 2:
            assert rows_seen[f] == d["rows_left"][f] > 0, (name, t)
        if k in (0, 2):
            assert done_at[f] < 0, (name, f, "completed twice")
            done_at[f] = t
    assert (done_at >= 0).all(), "a front without a task"
    assert np.array_equal(rows_seen, d["rows_left"])
    for f, blocks in row_cover.items():     # the row tasks tile the front's rows
        blocks.sort()
        assert blocks[0][0] == 0 and blocks[-1][1] == d["sym.sn_rowptr"][f + 1] - d["sym.sn_rowptr"][f]
        assert all(b[1] == c[0] and b[1] - b[0] <= SI_RB for b, c in zip(blocks, blocks[1:]))


@pytest.mark.parametrize("name", NAMES)
def test_caller_order_map_hits_each_entry_once(driver, tmp_path, name):
    N, cp, rv, d = _run(driver, tmp_path, name)
    P = Panels(d)
    pos = d["caller_pos"]
    assert pos.size == len(rv) and (pos >= 0).all()
    assert np.unique(pos).size == pos.size
    iperm = np.empty(N, np.int64)
    iperm[d["sym.perm"]] = np.arange(N)
    cols = np.repeat(np.arange(N), np.diff(cp))
    pi, pj = iperm[rv], iperm[cols]
    _, row, col = P.decode(pos)
    assert np.array_equal(row, np.maximum(pi, pj)) and np.array_equal(col, np.minimum(pi, pj))
