"""The update plans (build_updown_plan in csrc/ldl_plan.cpp) built on the host, without a CUDA runtime:
- the reached fronts are the union of the columns' paths to the root, in the level order of the full queue;
- each front's mask names exactly the columns whose path passes through it;
- tasks: one per front with at most DF_RB rows below the pivot block, else a pivot-block task then row tasks of DF_RB
  rows covering the rows in order; pend counts the reached children, rows_left the row tasks; every wait (children
  before a front, the pivot block before its rows) is on a task queued earlier, and slots stay within the bound;
- the pass width UD_PASS is 8 and the task record 32 bytes;
- the host steps grow with the reached fronts and the columns, not with n.
tests/host_harness/updown_plan_driver.cpp builds the plans with g++ and writes them out.  The matrices are the LDL
shape matrices of tests/ldl_shapes.py and KKT matrices, one of C2's size."""
import math
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

NF = 8
K_KIND, K_S, K_LI, K_PLI, K_MASK, K_R0, K_R1, K_SLOT = range(NF)


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("updown") / "updown_plan_driver")
    srcs = [os.path.join(ROOT, "tests", "host_harness", "updown_plan_driver.cpp")] + \
           [os.path.join(CSRC, f) for f in ("ldl_plan.cpp", "symbolic.cpp", "ordering.cpp")]
    cc = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-I" + CSRC, "-o", exe] + srcs,
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def _matrix(name):
    if name in ("big_fronts", "child_records"):
        sh = getattr(ldl_shapes, name)()
        return sh.N, sh.cp, sh.rv, np.asarray(sh.perm, dtype=np.int32)
    if name == "c2":
        pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    else:
        pr = workloads.random_sparse_qp(n=2000, m=4000, nnz_per_row=5, seed=1, window=200)
    N, cp, rv, _, _ = workloads.kkt_triu(pr["P"], pr["A"], np.full(pr["A"].shape[0], 1e-3))
    return N, cp, rv, None


def _sets(N, rng):
    """first rows of the columns (permuted): one column, 3 and 8 at random, 8 in the first columns (leaves), in the
    root separator, and 8 with repeats"""
    out = [rng.choice(N, size=k, replace=False) for k in (1, 3, 8)]
    out += [np.arange(8), np.arange(N - 8, N), np.array([5, 5, 9, 5, 1, 9, 9, 2]) % N]
    return [np.asarray(q, np.int32) for q in out]


_PLANS = {}


def _run(driver, tmp_path, name):
    if name not in _PLANS:
        N, cp, rv, perm = _matrix(name)
        sets = _sets(N, np.random.default_rng(1))
        fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
        with open(fin, "wb") as f:
            np.array([N, len(rv), perm is not None, len(sets)], dtype=np.int64).tofile(f)
            np.asarray(cp, dtype=np.int64).tofile(f)
            np.asarray(rv, dtype=np.int32).tofile(f)
            if perm is not None:
                perm.tofile(f)
            for q in sets:
                np.array([q.size], np.int64).tofile(f)
                q.tofile(f)
        r = subprocess.run([driver, fin, fout], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
        d, raw, i = {}, open(fout, "rb").read(), 0
        while i < len(raw):
            ln = int(np.frombuffer(raw, np.int32, 1, i)[0]); i += 4
            k = raw[i:i + ln].decode(); i += ln
            cnt = int(np.frombuffer(raw, np.int64, 1, i)[0]); i += 8
            d[k] = np.frombuffer(raw, np.int64, cnt, i); i += 8 * cnt
        for k in list(d):
            if k.endswith("tasks"):
                d[k] = d[k].reshape(-1, NF)
        _PLANS[name] = (N, sets, d)
    return _PLANS[name]


def _paths(d, firsts):
    first, parent = d["sym.sn_first"], d["sym.sn_parent"]
    col2sn = np.repeat(np.arange(len(first) - 1), np.diff(first))
    mask = {}
    for r, c in enumerate(firsts):
        s = int(col2sn[c])
        while s >= 0:
            mask[s] = mask.get(s, 0) | (1 << r)
            s = int(parent[s])
    return mask


NAMES = ["big_fronts", "child_records", "kkt", "c2"]


def test_pass_width_and_record():
    with open(os.path.join(CSRC, "ldl_plan.h")) as f:
        src = f.read()
    assert "#define UD_PASS 8 " in src


@pytest.mark.parametrize("name", NAMES)
def test_closure_masks_tasks_and_waits(driver, tmp_path, name):
    N, sets, d = _run(driver, tmp_path, name)
    ud_pass, rb, rec, bound = d["const"].tolist()
    assert ud_pass == 8 and rec == 32 and rb == 128
    parent, level, rowptr = d["sym.sn_parent"], d["sym.sn_level"], d["sym.sn_rowptr"]
    for qi, firsts in enumerate(sets):
        q = "q%d." % qi
        reached, mask, T, cnt = d[q + "reached"], d[q + "mask"], d[q + "tasks"], d[q + "cnt"]
        nslots = int(d[q + "stats"][0])
        want = _paths(d, firsts)
        assert set(reached.tolist()) == set(want) and len(set(reached.tolist())) == reached.size
        assert all((level[a], a) < (level[b], b) for a, b in zip(reached, reached[1:]))
        assert [want[int(s)] for s in reached] == mask.tolist()
        r = reached.size
        li = {int(s): i for i, s in enumerate(reached)}
        pend, rows_left, done = cnt[:r], cnt[r:2 * r], cnt[2 * r:]
        assert not done.any()
        exp_pend = np.zeros(r, np.int64)
        for s in reached:
            p = int(parent[s])
            if p >= 0:
                exp_pend[li[p]] += 1
        assert np.array_equal(pend, exp_pend)
        # the tasks of each front, in queue order
        head = {}        # front -> queue index of its kind 0 / 1 task
        last = {}        # front -> queue index of its last task
        t = 0
        slots = set()
        for i, s in enumerate(reached):
            s = int(s)
            nr = int(rowptr[s + 1] - rowptr[s])
            tk = T[t]
            assert tk[K_S] == s and tk[K_LI] == i and tk[K_MASK] == mask[i]
            assert tk[K_PLI] == (li[int(parent[s])] if parent[s] >= 0 else -1)
            head[s] = t
            if nr <= rb:
                assert tk[K_KIND] == 0 and (tk[K_R0], tk[K_R1]) == (0, nr) and rows_left[i] == 0
                last[s] = t
                t += 1
                continue
            assert tk[K_KIND] == 1 and 0 <= tk[K_SLOT] < nslots and tk[K_SLOT] not in slots
            slots.add(int(tk[K_SLOT]))
            t += 1
            r0 = 0
            while r0 < nr:
                tr = T[t]
                assert tr[K_KIND] == 2 and tr[K_S] == s and tr[K_SLOT] == tk[K_SLOT] and tr[K_MASK] == mask[i]
                assert (tr[K_R0], tr[K_R1]) == (r0, min(nr, r0 + rb))
                r0 = tr[K_R1]
                t += 1
            assert rows_left[i] == math.ceil(nr / rb)
            last[s] = t - 1
        assert t == len(T) and nslots <= bound
        # every front's head waits on its reached children, which all finish earlier in the queue
        for s in reached:
            p = int(parent[s])
            if p >= 0:
                assert last[int(s)] < head[p]


@pytest.mark.parametrize("name", ["kkt", "c2"])
def test_host_work_grows_with_the_reached_fronts(driver, tmp_path, name):
    N, sets, d = _run(driver, tmp_path, name)
    for qi, firsts in enumerate(sets):
        q = "q%d." % qi
        r, nt = d[q + "reached"].size, len(d[q + "tasks"])
        work = int(d[q + "stats"][2])
        bound = 4 * (firsts.size * r + r * math.log2(r + 2) + nt)
        assert work <= bound, (name, qi, work, bound)
    one = int(d["q0.stats"][2])
    assert d["q0.reached"].size < len(d["sym.sn_parent"]) and one < N / 100, (one, N)
