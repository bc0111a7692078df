"""The LDL factorisation and solve plans (csrc/ldl_plan.cpp) built on the host, without a CUDA runtime, and checked
for the conditions the persistent kernels rely on:
- every dependency of a task sits earlier in the queue (co-resident CTAs spin on their dependencies: a task queued
  before one it waits for can deadlock the kernel), and the dependency counters start at the right values;
- contributions to one destination are listed in a fixed order (child_list order), so sums are bit-reproducible;
- sharded, a rank's owned subtrees come before the replicated top part, and the ranks together cover the unsharded
  plan's fronts exactly once.
tests/host_harness/ldl_plan_driver.cpp builds the plans with g++ and writes them out."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
CSRC = os.path.join(ROOT, "clarabel.rs_b200", "csrc")

from helpers import workloads  # noqa: E402


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("plan") / "ldl_plan_driver")
    srcs = [os.path.join(ROOT, "tests", "host_harness", "ldl_plan_driver.cpp")] + \
           [os.path.join(CSRC, f) for f in ("ldl_plan.cpp", "symbolic.cpp", "ordering.cpp")]
    cc = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-I" + CSRC, "-o", exe] + srcs,
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def _kkt(name):
    perm = None
    if name == "c2_small":
        pr = workloads.random_sparse_qp(n=4000, m=8000, nnz_per_row=5, seed=1, window=200)
    elif name == "block_angular_small":
        pr = workloads.block_angular_qp(n=40_000, nblocks=8, nlink=300, link_blocks=4, seed=3)
    elif name == "portfolio_socp":
        pr = workloads.portfolio_socp(n_assets=600, n_soc=20, soc_dim=26, block=60, seed=2)
    else:   # grouped PSD: the ordering contracts every PSD block's rows into one vertex (what cipm_create does)
        import clarabel_rs_b200 as cb
        pr = workloads.block_sdp(n=2000, n_psd=40, psd_dim=10, nnz_per_row=6, window=200, n_nonneg=200, seed=4)
    N, cp, rv, _, ds = workloads.kkt_triu(pr["P"], pr["A"], np.full(pr["A"].shape[0], 1e-3))
    if name == "grouped_psd":
        perm = np.asarray(cb.order_groups(N, cp, rv, pr["cones"], pr["P"].shape[0]), dtype=np.int32)
    return N, cp, rv, perm


def _run(driver, tmp_path, name, nranks):
    N, cp, rv, perm = _kkt(name)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        np.array([N, len(rv), nranks, perm is not None], dtype=np.int64).tofile(f)
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
    return out


class Tree:
    def __init__(self, d):
        self.first, self.rowptr, self.parent = d["sym.sn_first"], d["sym.sn_rowptr"], d["sym.sn_parent"]
        self.level, self.cptr, self.clist, self.upd_off = d["sym.sn_level"], d["sym.child_ptr"], d["sym.child_list"], d["sym.upd_off"]
        self.nsup = len(self.parent)
        self.ns = np.diff(self.first)
        self.nr = np.diff(self.rowptr)

    def kids(self, s):
        return self.clist[self.cptr[s]:self.cptr[s + 1]]


def check_factor(T, d, p):
    """the factor queue of one view (prefix p): order, counters, sorted small-child lists; returns the fronts with tasks
    of the owned phase and of the top phase"""
    kind, s, d0, d1 = d[p + "f.kind"], d[p + "f.s"], d[p + "f.d0"], d[p + "f.d1"]
    a, e0, e1 = d[p + "f.a"], d[p + "f.e0"], d[p + "f.e1"]
    nt = len(kind)
    cnt = d[p + "f.cnt_init"].reshape(4, T.nsup)
    pend, rows_left, tiles_left = cnt[0], cnt[2], cnt[3]
    assert not cnt[1].any()
    first, last = {}, {}
    for i, f in enumerate(s):
        first.setdefault(int(f), i)
        last[int(f)] = i
    has_tasks = np.zeros(T.nsup, bool)
    has_tasks[list(first)] = True
    assert len(set(s[kind == 0]) & set(s[kind != 0])) == 0
    for f, i0 in first.items():
        assert kind[i0] in (0, 1) and (kind[i0] == 1 or last[f] == i0), f     # an F task, or a D task first
        # all tasks of every queued child before the parent's first task
        for c in T.kids(f):
            if has_tasks[c]:
                assert last[int(c)] < i0, (f, c)
        # pend = children with tasks on this rank
        assert pend[f] == has_tasks[T.kids(f)].sum(), f
    for f in set(s[kind == 1].tolist()):
        idx = np.nonzero(s == f)[0]
        ks = kind[idx]
        D, R, Tt = idx[ks == 1], idx[ks == 2], idx[ks == 3]
        assert len(D) == 1 and len(R) >= 1 and len(Tt) >= 1
        assert D[0] < R.min() and R.max() < Tt.min(), f           # D before its R tasks, every R before the T tasks
        assert rows_left[f] == len(R) and tiles_left[f] == len(Tt), f
        assert (np.sort(a[R]) == np.arange(len(R))).all()
    assert (rows_left[~np.isin(np.arange(T.nsup), s[kind == 1])] == 0).all()
    assert (tiles_left[~np.isin(np.arange(T.nsup), s[kind == 1])] == 0).all()
    assert (d0 <= d1).all() and (e0 <= e1).all()
    # small-child lists: sorted by dst inside each key, equal dst in child_list order
    big_pos, tile_base = d[p + "f.big_pos"], d[p + "f.tile_base"]
    owner_of_key = {"panel": np.argsort(np.where(big_pos >= 0, big_pos, T.nsup + 1))[:(big_pos >= 0).sum()]}
    tb = np.nonzero(tile_base >= 0)[0]
    tb = tb[np.argsort(tile_base[tb])]
    ntile = [(int(-(-T.nr[f] // 64)) * int(-(-T.nr[f] // 64) + 1)) // 2 for f in tb]
    owner_of_key["tile"] = np.concatenate([np.full(k, f) for f, k in zip(tb, ntile)]) if len(tb) else np.zeros(0, int)
    for which in ("panel", "tile"):
        ptr, src, dst = d[p + "f.sc_%s_ptr" % which], d[p + "f.sc_%s_src" % which], d[p + "f.sc_%s_dst" % which]
        assert len(ptr) == len(owner_of_key[which]) + 1
        for k in range(len(ptr) - 1):
            lo, hi = ptr[k], ptr[k + 1]
            if hi == lo:
                continue
            f = owner_of_key[which][k]
            dd, ss = dst[lo:hi], src[lo:hi]
            assert (np.diff(dd) >= 0).all(), (which, k)
            kids = T.kids(f)
            kids = kids[T.nr[kids] > 0]
            starts = T.upd_off[kids]
            order = np.argsort(starts)
            pos_in_list = order[np.searchsorted(starts[order], ss, side="right") - 1]   # child of each entry
            same = np.diff(dd) == 0
            assert (np.diff(pos_in_list)[same] > 0).all(), (which, k)
    own = set(s[:int(d[p + "f.ntask_owned"][0])].tolist())
    top = set(s[int(d[p + "f.ntask_owned"][0]):].tolist())
    return own, top


def check_level0(T, d, p, mine):
    """the level-0 launches cover this rank's level-0 fronts that k_factor_df does not factor, each once"""
    segs, lt = d[p + "l0.segs"].reshape(-1, 3), d[p + "l0.level_tasks"]
    launched = np.concatenate([lt[b:b + c] for _, b, c in segs]) if len(segs) else np.zeros(0, np.int64)
    big = (T.nr >= 96) & (T.ns <= 64)
    want = np.nonzero((T.level == 0) & ~big & mine)[0]
    assert len(np.unique(launched)) == len(launched) and sorted(launched) == sorted(want)
    assert sorted(lt) == list(range(T.nsup))


def check_solve(T, d, p):
    kind, s, cnt = d[p + "s.kind"], d[p + "s.s"], d[p + "s.cnt"]
    dep0, dep1, dep2, bslot, ptask = d[p + "s.dep0"], d[p + "s.dep1"], d[p + "s.dep2"], d[p + "s.bslot"], d[p + "s.ptask"]
    fronts, f2t = d[p + "s.fronts"], d[p + "s.front2task"]
    nt = len(kind)
    task_fronts = []
    for i in range(nt):
        fr = fronts[s[i]:s[i] + cnt[i]] if kind[i] == 0 else ([s[i]] if kind[i] == 1 else [])
        task_fronts.append(fr)
        for f in fr:
            assert f2t[f] == i
        if kind[i] != 0:
            if dep1[i] >= 0:
                assert 0 <= dep0[i] <= dep1[i] < i, i
                if kind[i] == 1:
                    assert dep1[i] <= dep2[i] < i, i
            assert ptask[i] == -1 or ptask[i] > i, i
            assert ptask[i] == -1 or ptask[i] == f2t[T.parent[s[i]]]
    rows = kind == 2
    assert len(np.unique(bslot[rows])) == rows.sum()
    # every front exactly once across the leaf lists and the tasks
    listed = np.concatenate([d[p + "s.leaf1"], d[p + "s.leafn"], d[p + "s.leafw"]] + [np.asarray(f, np.int64) for f in task_fronts])
    assert len(np.unique(listed)) == len(listed)
    # pend = non-chain children that have tasks; chain child of a wide front: a wide child whose rows are the whole front
    wide = T.ns > 8
    chain = np.full(T.nsup, -1)
    for c in range(T.nsup):
        q = T.parent[c]
        if q >= 0 and wide[c] and wide[q] and chain[q] < 0 and T.nr[c] == T.ns[q] + T.nr[q]:
            chain[q] = c
    pend = np.zeros(nt, np.int64)
    for c in range(T.nsup):
        q = T.parent[c]
        if q >= 0 and f2t[c] >= 0 and chain[q] != c:
            pend[f2t[q]] += 1
    assert (d[p + "s.cnt_init"][:nt] == pend).all()
    # gather lists in child_list order
    gptr, gsrc = d[p + "s.gat_ptr"], d[p + "s.gat_src"]
    child_of_row = np.searchsorted(T.rowptr, gsrc[:gptr[-1]], side="right") - 1
    rank_in_parent = np.empty(T.nsup, np.int64)
    for q in range(T.nsup):
        rank_in_parent[T.kids(q)] = np.arange(len(T.kids(q)))
    r = rank_in_parent[child_of_row]
    slot_start = np.zeros(len(r), bool)
    slot_start[gptr[:-1][gptr[:-1] < len(r)]] = True
    assert ((np.diff(r) > 0) | slot_start[1:]).all()
    listed = [np.asarray(f, np.int64) for f in task_fronts[:int(d[p + "s.ntask_owned"][0])]]
    own = set(np.concatenate(listed).tolist()) if listed else set()
    listed = [np.asarray(f, np.int64) for f in task_fronts[int(d[p + "s.ntask_owned"][0]):]]
    top = set(np.concatenate(listed).tolist()) if listed else set()
    return own, top, set(np.concatenate([d[p + "s.leaf1"], d[p + "s.leafn"], d[p + "s.leafw"]]).tolist())


CASES = ["c2_small", "block_angular_small", "grouped_psd", "portfolio_socp"]


@pytest.mark.parametrize("nranks", [2, 3])
@pytest.mark.parametrize("name", CASES)
def test_plans_keep_the_conditions_the_kernels_rely_on(driver, tmp_path, name, nranks):
    d = _run(driver, tmp_path, name, nranks)
    T = Tree(d)
    f_own, f_top = check_factor(T, d, "u.")
    s_own, s_top, s_leaves = check_solve(T, d, "u.")
    check_level0(T, d, "u.", np.ones(T.nsup, bool))
    assert not f_top and not s_top
    f_all, s_all = f_own, s_own
    assert len(f_all) > 0 and len(s_all) > 0
    owner = d["owner"]
    f_cover, s_cover, leaves = [], [], set()
    for r in range(nranks):
        fo, ft = check_factor(T, d, "r%d." % r)
        so, st, sl = check_solve(T, d, "r%d." % r)
        check_level0(T, d, "r%d." % r, (owner == r) | (owner < 0))
        assert all(owner[f] == r for f in fo) and all(owner[f] == r for f in so)
        assert all(owner[f] == -1 for f in ft) and all(owner[f] == -1 for f in st)
        f_cover += list(fo) + (list(ft) if r == 0 else [])
        s_cover += list(so) + (list(st) if r == 0 else [])
        leaves |= sl
        # the other ranks see the same top part
        assert ft == check_factor(T, d, "r0.")[1] and st == check_solve(T, d, "r0.")[1]
    assert sorted(f_cover) == sorted(f_all)
    assert sorted(s_cover) == sorted(s_all)
    assert leaves == s_leaves


def test_the_plans_exercise_every_task_kind(driver, tmp_path):
    d = _run(driver, tmp_path, "block_angular_small", 1)
    assert set(d["u.f.kind"].tolist()) == {0, 1, 2, 3}
    assert set(d["u.s.kind"].tolist()) == {0, 1, 2}
    assert len(d["u.f.sc_panel_src"]) > 1 and len(d["u.f.sc_tile_src"]) > 1
