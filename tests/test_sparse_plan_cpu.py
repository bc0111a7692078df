"""The pruned solve plans (build_pruned_plan in csrc/ldl_plan.cpp) built on the host, without a CUDA runtime, and
checked against the full solve plan they derive from:
- the reached fronts are exactly the upward closure of the index set's fronts in sn_parent;
- every task of a reached wide front equals its full-plan record except for the remapped index fields (the parent's
  head task, and the chain child's tasks -- shifted when the child is reached, dropped when it is not);
- no task waits on a task outside its plan or later in the queue (co-resident CTAs spin on those flags: a wait on a
  later task can deadlock the sweep), and the backward waits name reached fronts;
- pend counts the reached non-chain children that have tasks;
- with every index, the pruned plan equals the full plan field for field;
- the host steps of a call grow with the fronts it reaches and the index list, not with n.
tests/host_harness/sparse_plan_driver.cpp builds the plans with g++ and writes them out.  The matrices are the LDL
shape matrices of tests/ldl_shapes.py (every front shape the sweeps dispatch on) and random KKT matrices; the slab
capacity is the one an H100 gets (8266 doubles) and a small one that splits more fronts into row tasks."""
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

NF = 20                      # values per task record
F_KIND, F_S, F_CNT, F_DEP0, F_DEP1, F_DEP2, F_NRT, F_BOWNER, F_PTASK, F_NOTIFY = 0, 1, 2, 10, 11, 12, 13, 14, 17, 19
REMAPPED = [F_DEP0, F_DEP1, F_DEP2, F_PTASK]
SIZES = [1, 2, 17, 200]


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("sparse") / "sparse_plan_driver")
    srcs = [os.path.join(ROOT, "tests", "host_harness", "sparse_plan_driver.cpp")] + \
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


def _sets(N, rng):
    """index sets (permuted columns): sizes 1..200 at random, a run at the start (a leaf), the last columns (the root
    separator), one with repeats, and every column"""
    out = [rng.choice(N, size=k, replace=False) for k in SIZES]
    out += [np.arange(5), np.arange(N - 5, N), np.array([7, 7, 3, 7]) % N, np.arange(N)]
    return [np.asarray(q, np.int32) for q in out]


_PLANS = {}


def _run(driver, tmp_path, name, cap):
    key = (name, cap)
    if key not in _PLANS:
        N, cp, rv, perm = _matrix(name)
        sets = _sets(N, np.random.default_rng(1))
        fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
        with open(fin, "wb") as f:
            np.array([N, len(rv), perm is not None, cap, len(sets)], dtype=np.int64).tofile(f)
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
        _PLANS[key] = (N, sets, d)
    return _PLANS[key]


def _closure(d, cols):
    first, parent = d["sym.sn_first"], d["sym.sn_parent"]
    col2sn = np.repeat(np.arange(len(first) - 1), np.diff(first))
    seen = set()
    for c in cols:
        s = int(col2sn[c])
        while s >= 0 and s not in seen:
            seen.add(s)
            s = int(parent[s])
    return seen


CASES = [(m, c) for m in ("big_fronts", "child_records", "random_qp", "block_angular") for c in (8266, 1024)]


@pytest.mark.parametrize("name,cap", CASES)
def test_pruned_plans_against_the_full_plan(driver, tmp_path, name, cap):
    N, sets, d = _run(driver, tmp_path, name, cap)
    parent, level = d["sym.sn_parent"], d["sym.sn_level"]
    nsup = len(parent)
    FT, f2t_full = d["full.tasks"], d["full.front2task"]
    for qi, cols in enumerate(sets):
        q = "q%d." % qi
        reached, T, pend, fronts = d[q + "reached"], d[q + "tasks"], d[q + "pend"], d[q + "fronts"]
        # the closure, in queue order
        assert set(reached.tolist()) == _closure(d, cols) and len(set(reached.tolist())) == reached.size
        assert all((level[a], a) < (level[b], b) for a, b in zip(reached, reached[1:]))
        rset = set(reached.tolist())
        pairs = d[q + "f2t"].reshape(-1, 2)
        f2t = dict((int(s), int(t)) for s, t in pairs)
        assert set(f2t) == {s for s in rset if f2t_full[s] >= 0}
        for lst in ("leaf1", "leafn", "leafw"):
            assert d[q + lst].tolist() == [s for s in d["full." + lst].tolist() if s in rset]
        expect_pend = np.zeros(len(T), np.int64)
        for t in range(len(T)):
            if T[t, F_KIND] == 0:
                for s in fronts[T[t, F_S]:T[t, F_S] + T[t, F_CNT]]:
                    assert f2t[int(s)] == t and f2t_full[s] >= 0 and FT[f2t_full[s], F_KIND] == 0
                    p = int(parent[s])
                    if p >= 0:
                        assert f2t[p] > t, "a narrow front's parent queued before it"
                        expect_pend[f2t[p]] += 1
                continue
            s = int(T[t, F_S])
            h = f2t[s]
            full_t = f2t_full[s] + (t - h)
            o = FT[full_t]
            keep = [i for i in range(NF) if i not in REMAPPED]
            assert np.array_equal(T[t, keep], o[keep]), (name, qi, t)
            p = int(parent[s])
            assert T[t, F_PTASK] == (f2t[p] if p >= 0 else -1)
            if T[t, F_PTASK] >= 0:
                assert T[t, F_PTASK] > t
            if t == h and p >= 0 and o[F_NOTIFY]:
                expect_pend[f2t[p]] += 1
            if o[F_DEP1] >= o[F_DEP0]:
                c = int(FT[o[F_DEP0], F_S])
                if c in rset:
                    sh = f2t[c] - f2t_full[c]
                    assert (T[t, F_DEP0], T[t, F_DEP1]) == (o[F_DEP0] + sh, o[F_DEP1] + sh)
                    assert T[t, F_DEP2] == (o[F_DEP2] + sh if o[F_DEP2] >= 0 else o[F_DEP2])
                    assert 0 <= T[t, F_DEP0] <= T[t, F_DEP1] < t and T[t, F_DEP2] < t
                    assert all(T[u, F_S] == c and T[u, F_KIND] != 0 for u in range(T[t, F_DEP0], max(T[t, F_DEP1], T[t, F_DEP2]) + 1))
                else:
                    assert (T[t, F_DEP0], T[t, F_DEP1], T[t, F_DEP2]) == (0, -1, -1)
            else:
                assert T[t, F_DEP1] < T[t, F_DEP0]
            # backward: the slab's first row belongs to a reached front whose head comes later in the queue
            b = int(T[t, F_BOWNER])
            if b >= 0:
                assert b in rset and f2t.get(b, -1) > t or (b in rset and f2t_full[b] < 0)
        assert np.array_equal(pend, expect_pend), (name, qi)


@pytest.mark.parametrize("name,cap", CASES)
def test_every_index_gives_the_full_plan(driver, tmp_path, name, cap):
    N, sets, d = _run(driver, tmp_path, name, cap)
    q = "q%d." % (len(sets) - 1)
    nt = len(d["full.tasks"])
    assert np.array_equal(d[q + "tasks"], d["full.tasks"])
    assert np.array_equal(d[q + "pend"], d["full.cnt_init"][:nt])
    assert np.array_equal(d[q + "fronts"], d["full.fronts"])
    for lst in ("leaf1", "leafn", "leafw"):
        assert np.array_equal(d[q + lst], d["full." + lst])
    f2t = np.full(len(d["full.front2task"]), -1)
    pairs = d[q + "f2t"].reshape(-1, 2)
    f2t[pairs[:, 0]] = pairs[:, 1]
    assert np.array_equal(f2t, d["full.front2task"])


@pytest.mark.parametrize("name", ["random_qp", "block_angular"])
def test_host_work_grows_with_the_reached_fronts(driver, tmp_path, name):
    N, sets, d = _run(driver, tmp_path, name, 8266)
    for qi, cols in enumerate(sets):
        q = "q%d." % qi
        r, nt = d[q + "reached"].size, len(d[q + "tasks"])
        work = int(d[q + "stats"][1])
        bound = 4 * (r * math.log2(r + 2) + cols.size + nt + r)
        assert work <= bound, (name, qi, work, bound)
    one = int(d["q0.stats"][1])
    assert d["q0.reached"].size < len(d["sym.sn_parent"]) and one < N / 10, (one, N)
