"""The matrices of tests/ldl_shapes.py reach every front shape at which the LDL^T's factor and solve kernels switch
code paths.  Their plans are built on the host (tests/host_harness/ldl_plan_driver.cpp, with the shared-memory caps
cldl_create derives on an H100) and read back: every target below must be hit, so that tests/test_ldl_shapes_gpu.py,
which runs the same matrices on the device, is known to exercise it.  The plans also pass the structural checks of
test_ldl_plan_cpu.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ldl_shapes  # noqa: E402
from test_ldl_plan_cpu import Tree, check_factor, check_level0, check_solve, driver  # noqa: E402,F401

BIG_NR, PB_MAXNS, SMALL_NS, DF_RB, TS, SV_MAXROWS, DF_ENT_FAST, DF_DCAP = 96, 64, 8, 128, 64, 256, 512, 32
SV_CAP = 8266       # solve slab (doubles) on an H100, as in the driver
LEVEL_CLASSES = [1024, 5632, 28800]   # k_factor_level shared-memory classes (doubles), the last one the H100's cap


def _plans(driver, tmp_path, sh):
    fin, fout = str(tmp_path / (sh.name + ".in")), str(tmp_path / (sh.name + ".out"))
    with open(fin, "wb") as f:
        np.array([sh.N, len(sh.rv), 1, 1], dtype=np.int64).tofile(f)
        np.asarray(sh.cp, dtype=np.int64).tofile(f)
        np.asarray(sh.rv, dtype=np.int32).tofile(f)
        np.asarray(sh.perm, dtype=np.int32).tofile(f)
    r = subprocess.run([driver, fin, fout], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-3000:]
    out, raw, i = {}, open(fout, "rb").read(), 0
    while i < len(raw):
        ln = int(np.frombuffer(raw, np.int32, 1, i)[0]); i += 4
        key = raw[i:i + ln].decode(); i += ln
        cnt = int(np.frombuffer(raw, np.int64, 1, i)[0]); i += 8
        out[key] = np.frombuffer(raw, np.int64, cnt, i); i += 8 * cnt
    return out


def targets_hit(T, d):
    """{target: hit} over one matrix's plans"""
    hit = {}
    add = lambda k, v: hit.__setitem__(k, hit.get(k, False) or bool(v))
    # ---- level 0 ----
    segs = d["u.l0.segs"].reshape(-1, 3)
    add("l0: k_factor_leaf1", any(s[0] and s[2] > 0 for s in segs))
    lt = d["u.l0.level_tasks"]
    for leaf1, base, cnt in segs:
        if leaf1:
            continue
        p = [(T.ns[f] + T.nr[f]) * T.ns[f] for f in lt[base:base + cnt]]
        for c, cap in enumerate(LEVEL_CLASSES):
            lo = LEVEL_CLASSES[c - 1] if c else 0
            add("l0: k_factor_level class %d" % c, any(lo < x <= cap for x in p))
    # ---- k_factor_df ----
    kind, s, ns, nr = d["u.f.kind"], d["u.f.s"], d["u.f.ns"], d["u.f.nr"]
    d0, d1, e0, e1, ndense, a = d["u.f.d0"], d["u.f.d1"], d["u.f.e0"], d["u.f.e1"], d["u.f.ndense"], d["u.f.a"]
    assert (ns == T.ns[s]).all() and (nr == T.nr[s]).all()
    D, R, Tt, F = kind == 1, kind == 2, kind == 3, kind == 0
    add("df: big front at level 0", (D & (T.level[s] == 0)).any())
    add("df: F task", F.any())
    add("df: F task nr 95", (F & (nr == 95)).any())
    add("df: F task nr 0 (root)", (F & (nr == 0)).any())
    for x in (1, 2, 3, 4, 5, 8, 9, 63, 64):
        add("df: D ns %d" % x, (D & (ns == x)).any())
    for m in range(4):
        add("df: D ns%%4 == %d" % m, (D & (ns % 4 == m)).any())
        add("df: T ns%%4 == %d" % m, (Tt & (ns % 4 == m)).any())
    for x in (96, 97, 127, 128, 129, 255, 256, 257):
        add("df: big nr %d" % x, (D & (nr == x)).any())
    for m in (0, 1, 63):
        add("df: big nr%%64 == %d" % m, (D & (nr % 64 == m)).any())
    last_r = R & (a == (nr + DF_RB - 1) // DF_RB - 1)
    add("df: R last block partial", (last_r & (nr % DF_RB != 0)).any())
    add("df: R last block full", (last_r & (nr % DF_RB == 0)).any())
    add("df: T partial tile", (Tt & (nr % TS != 0)).any())
    add("df: T full tiles only", (Tt & (nr % TS == 0)).any())
    contig, recs = d["u.f.rec.contig"], d1 - d0
    for c in range(4):
        add("df: child record contig %d" % c, (contig == c).any())
    use_sc = (recs > ndense) | (e1 > e0)
    add("df: T ndense > 0 without use_sc", (Tt & (ndense > 0) & ~use_sc).any())
    add("df: T ndense > 0 with use_sc", (Tt & (ndense > 0) & use_sc).any())
    add("df: panel small-child list > 512 (df_apply_sorted)", ((D | R) & (e1 - e0 > DF_ENT_FAST)).any())
    add("df: tile small-child list > 512 (df_apply_sorted)", (Tt & (e1 - e0 > DF_ENT_FAST)).any())
    add("df: > 32 child records in one task", (recs > DF_DCAP).any())
    # ---- solves ----
    add("sv: leaf1", len(d["u.s.leaf1"]))
    add("sv: leafn", len(d["u.s.leafn"]))
    add("sv: leafw", len(d["u.s.leafw"]))
    add("sv: k_invert_pivots (wide fronts)", len(d["u.s.wide"]))
    skind, snr, sns, r0, r1, nrt = d["u.s.kind"], d["u.s.nr"], d["u.s.ns"], d["u.s.r0"], d["u.s.r1"], d["u.s.nrt"]
    narrow = d["u.s.fronts"]
    add("sv: narrow front nr <= 256", (T.nr[narrow] <= SV_MAXROWS).any())
    add("sv: narrow front nr > 256", (T.nr[narrow] > SV_MAXROWS).any())
    head = skind == 1
    add("sv: wide head only", (head & (nrt == 0)).any())
    add("sv: wide partial slab", (head & (r1 < snr)).any())
    add("sv: wide row tasks", (skind == 2).any())
    fits = sns * (sns + snr) + 1 <= SV_CAP
    add("sv: row task past SV_MAXROWS rows of a fitting panel", (head & fits & (snr > SV_MAXROWS) & (nrt > 0)).any())
    wide = T.ns > SMALL_NS
    chain = [c for c in range(T.nsup) if T.parent[c] >= 0 and wide[c] and wide[T.parent[c]]
             and T.nr[c] == T.ns[T.parent[c]] + T.nr[T.parent[c]]]
    add("sv: chain child", len(chain))
    return hit


# Targets of the table no matrix here can reach, and why.
UNREACHABLE = {
    # k_factor_level with the panel in global memory needs a level-0 front that is not big ((ns + nr) ns > 28800
    # doubles with nr < 96 or ns > 64); panels are at most 64 columns wide (cldl_create caps max_panel at 64), so the
    # widest such panel is (64 + 95) 64 = 10176 doubles
    "l0: k_factor_level class 3 (panel in global memory)",
}


@pytest.fixture(scope="module")
def coverage(driver, tmp_path_factory):
    tmp = tmp_path_factory.mktemp("shapes")
    hit = {}
    for sh in ldl_shapes.all_shapes():
        d = _plans(driver, tmp, sh)
        T = Tree(d)
        check_factor(T, d, "u.")
        check_solve(T, d, "u.")
        check_level0(T, d, "u.", np.ones(T.nsup, bool))
        for k, v in targets_hit(T, d).items():
            hit.setdefault(k, []).append(sh.name) if v else hit.setdefault(k, [])
    return hit


def test_every_kernel_path_is_reached(coverage):
    for k in sorted(coverage):
        print("%-60s %s" % (k, ", ".join(coverage[k]) or "-"))
    missed = sorted(k for k, v in coverage.items() if not v)
    assert not missed, missed
    assert not UNREACHABLE & set(coverage)


def test_the_generator_builds_quasidefinite_matrices():
    for sh in ldl_shapes.all_shapes():
        assert sorted(sh.perm) == list(range(sh.N))
        cols = np.repeat(np.arange(sh.N), np.diff(sh.cp))
        assert (sh.rv <= cols).all() and (np.diff(sh.cp) > 0).all()
        K = sh.dense()
        dg = np.diag(K)
        assert (np.abs(dg) > np.abs(K).sum(axis=1) - np.abs(dg)).all()    # strictly diagonally dominant
        assert (np.sign(dg) == sh.ds).all()
