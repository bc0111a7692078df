"""The host analysis of Schur complement handles (analyse_schur in csrc/symbolic.cpp, build_schur_plan and the plan
builders in csrc/ldl_plan.cpp) built without a CUDA runtime and checked for what the device relies on:
- the permutation ends with the Schur set S, and no front holds columns of both B and S;
- the rows of every cut root (a B front whose parent is in S) lie in S;
- no S front is in a level-0 launch, a factor or solve task of the B phase, a level-0 solve list, or the B-only
  backward queue, and every B front is in one of them;
- every wait of the B-only backward queue is on a B front whose task it runs after (the queue runs in reverse);
- the K_SS map and the cut-root maps together reach each entry of the permuted lower triangle of the output as often
  as the matrix's entries and the cut roots' rows say;
- without a Schur set the analysis and every plan are field for field those of the previous analysis code:
  tests/golden/schur/plain_digests.json holds SHA-256 digests written by the parent commit's build of this driver.
tests/host_harness/schur_plan_driver.cpp builds the plans with g++ and writes them out."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
CSRC = os.path.join(ROOT, "clarabel.rs_b200", "csrc")
GOLDEN = os.path.join(ROOT, "tests", "golden", "schur", "plain_digests.json")

import ldl_shapes  # noqa: E402
from helpers import workloads  # noqa: E402


def build_driver(exe, csrc=CSRC, extra=()):
    srcs = [os.path.join(ROOT, "tests", "host_harness", "schur_plan_driver.cpp")] + \
           [os.path.join(csrc, f) for f in ("ldl_plan.cpp", "symbolic.cpp", "ordering.cpp")]
    cc = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-I" + csrc, "-o", exe] + list(extra) + srcs,
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return build_driver(str(tmp_path_factory.mktemp("schur") / "schur_plan_driver"))


def matrix(name):
    """(N, colptr, rowval, perm or None)"""
    if name in ("big_fronts", "child_records"):
        sh = getattr(ldl_shapes, name)()
        return sh.N, np.asarray(sh.cp), np.asarray(sh.rv), np.asarray(sh.perm, dtype=np.int32)
    if name == "random_qp":
        pr = workloads.random_sparse_qp(n=2000, m=4000, nnz_per_row=5, seed=1, window=200)
    else:
        pr = workloads.block_angular_qp(n=8000, nblocks=8, nlink=100, link_blocks=4, seed=3)
    N, cp, rv, _, _ = workloads.kkt_triu(pr["P"], pr["A"], np.full(pr["A"].shape[0], 1e-3))
    return N, cp, rv, None


def with_island(N, cp, rv, m=5):
    """the matrix plus a dense m x m block joined to nothing: its indices have no edge to the rest"""
    cols = [rv[cp[j]:cp[j + 1]] for j in range(N)] + [np.arange(N, N + j + 1) for j in range(m)]
    cp2 = np.concatenate([[0], np.cumsum([c.size for c in cols])])
    return N + m, cp2, np.concatenate(cols)


def run(driver, tmp_path, N, cp, rv, perm=None, schur=()):
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        np.array([N, len(rv), perm is not None, len(schur)], dtype=np.int64).tofile(f)
        np.asarray(cp, dtype=np.int64).tofile(f)
        np.asarray(rv, dtype=np.int32).tofile(f)
        if perm is not None:
            np.asarray(perm, dtype=np.int32).tofile(f)
        np.asarray(schur, dtype=np.int32).tofile(f)
    r = subprocess.run([driver, fin, fout], capture_output=True, text=True, timeout=600)
    if r.returncode != 0:
        return r.returncode
    out, raw, i = {}, open(fout, "rb").read(), 0
    while i < len(raw):
        ln = int(np.frombuffer(raw, np.int32, 1, i)[0]); i += 4
        key = raw[i:i + ln].decode(); i += ln
        cnt = int(np.frombuffer(raw, np.int64, 1, i)[0]); i += 8
        out[key] = np.frombuffer(raw, np.int64, cnt, i); i += 8 * cnt
    return out


def digests(d):
    return {k: hashlib.sha256(np.ascontiguousarray(v, np.int64).tobytes()).hexdigest() for k, v in sorted(d.items())}


NAMES = ["big_fronts", "child_records", "random_qp", "block_angular"]


def schur_sets(name, N, perm):
    """name -> Schur set (caller indices, in output order)"""
    rng = np.random.default_rng(5)
    sets = {"random": rng.choice(N, size=max(2, N // 10), replace=False),
            "one": np.array([N // 2]),
            "all_but_one": rng.permutation(np.delete(np.arange(N), N // 3))}
    if name == "block_angular":
        sets["linking_rows"] = np.arange(N - 100, N)
    elif perm is not None:
        sets["last_of_perm"] = np.asarray(perm[-40:])     # the last columns of the given ordering: its top separator
    return sets


# SVTask words: kind s cnt f | ns nr r0 r1 | poff(2) rp(2) | dep0 dep1 dep2 nrt | bowner bslot pure ptask | cuoff(2) | notify pad
SV_WORDS, SV_KIND, SV_S, SV_CNT, SV_BOWNER = 24, 0, 1, 2, 16
# DFTask words: kind s a b ...
DF_WORDS = 16


def check_schur(d, N, S, perm_given=None):
    k = len(S)
    sf = N - k
    perm = d["sym.perm"]
    assert sorted(perm[sf:]) == sorted(S), "the permutation does not end with S"
    if perm_given is not None:
        assert np.array_equal(perm[sf:], perm_given[sf:]) or sorted(perm[sf:]) == sorted(S)
    first, rowptr, rows, par = d["sym.sn_first"], d["sym.sn_rowptr"], d["sym.sn_rows"], d["sym.sn_parent"]
    nsup = len(par)
    isS = first[:-1] >= sf
    assert ((first[1:] <= sf) | isS).all(), "a front holds columns of B and of S"
    owner = d["sc.owner"]
    assert np.array_equal(owner, np.where(isS, -1, 0))
    cut = [s for s in range(nsup) if not isS[s] and par[s] >= 0 and isS[par[s]]]
    assert list(d["sc.cut"]) == cut
    for c in cut:
        assert (rows[rowptr[c]:rowptr[c + 1]] >= sf).all(), ("cut root rows outside S", c)
    assert (isS[par[isS]] | (par[isS] < 0)).all(), "an S front with a B parent"

    # the queues of the B phase
    seen = np.zeros(nsup, bool)
    segs = d["l0.segs"].reshape(-1, 5)
    lt = d["l0.level_tasks"]
    for leaf1, base, count, _, _ in segs:
        fr = lt[base:base + count]
        assert not isS[fr].any(), "an S front in a level-0 launch"
        seen[fr] = True
    ft = d["fp.tasks"].reshape(-1, DF_WORDS)[:int(d["fp.ntask_owned"][0])]
    assert not isS[ft[:, 1]].any(), "an S front in a factor task of the B phase"
    seen[ft[:, 1]] = True
    assert seen[~isS].all() and not seen[isS].any(), "a B front that is never factored"
    nto = int(d["sp.scalars"][2])
    svt = d["sp.tasks"].reshape(-1, SV_WORDS)[:nto]
    fronts = d["sp.fronts"]
    solved = np.zeros(nsup, bool)
    for t in svt:
        fr = fronts[t[SV_S]:t[SV_S] + t[SV_CNT]] if t[SV_KIND] == 0 else [t[SV_S]]
        assert not isS[fr].any(), "an S front in a solve task of the B phase"
        solved[fr] = True
    for lst in ("sp.leaf1", "sp.leafn", "sp.leafw"):
        assert not isS[d[lst]].any(), "an S front in a level-0 solve list"
        solved[d[lst]] = True
    assert solved[~isS].all()

    # the B-only backward queue: runs from its last task to its first
    bwd = d["sc.bwd"].reshape(-1, SV_WORDS)
    assert np.array_equal(bwd[:, :16], svt[:, :16]) and np.array_equal(bwd[:, 17:], svt[:, 17:])
    bpar = d["sc.bparent"]
    assert np.array_equal(bpar, np.where(np.isin(np.arange(nsup), cut), -1, par))
    f2t = d["sp.front2task"]
    for q, t in enumerate(bwd):
        waits = []
        if t[SV_KIND] == 0:
            waits = [bpar[s] for s in fronts[t[SV_S]:t[SV_S] + t[SV_CNT]] if bpar[s] >= 0]
        elif t[SV_BOWNER] >= 0:
            waits = [t[SV_BOWNER]]
        for w in waits:
            assert not isS[w], ("the backward queue waits on an S front", q)
            assert f2t[w] > q, ("a backward task runs before the front it waits on", q, w)

    # the output maps: count how often each output entry of the permuted lower triangle is reached
    spos = d["sc.spos"]
    assert sorted(spos) == list(range(k)) and np.array_equal(np.asarray(S)[spos], perm[sf:])
    hits = np.zeros(k * k, np.int64)
    kp, kd = d["sc.kss_ptr"], d["sc.kss_dst"]
    for j in range(k):
        dst = kd[kp[j]:kp[j + 1]]
        assert (dst // k == spos[j]).all()
        np.add.at(hits, dst, 1)
    rp_, rb = d["sc.rec_ptr"], d["sc.rec_b"]
    for j in range(k):
        for r in range(rp_[j], rp_[j + 1]):
            R = rows[d["sc.rec_rp"][r]:d["sc.rec_rp"][r] + d["sc.rec_nr"][r]]
            assert R[rb[r]] == sf + j
            np.add.at(hits, spos[j] * k + spos[R[rb[r]:] - sf], 1)
    return hits, cut


def expected_hits(N, cp, rv, d, S, cut):
    """from the caller's pattern and the cut roots' rows, independently of the maps"""
    k = len(S)
    sf = N - k
    ip = np.empty(N, np.int64)
    ip[d["sym.perm"]] = np.arange(N)
    out_of = np.full(N, -1)
    out_of[np.asarray(S)] = np.arange(k)
    cols = np.repeat(np.arange(N), np.diff(cp))
    a, b = ip[rv], ip[cols]
    inS = (a >= sf) & (b >= sf)
    lo, hi = np.minimum(a, b)[inS], np.maximum(a, b)[inS]
    exp = np.zeros(k * k, np.int64)
    np.add.at(exp, out_of[d["sym.perm"][lo]] * k + out_of[d["sym.perm"][hi]], 1)
    rowptr, rows = d["sym.sn_rowptr"], d["sym.sn_rows"]
    for c in cut:
        R = rows[rowptr[c]:rowptr[c + 1]] - sf
        I, J = np.tril_indices(R.size)
        o = out_of[d["sym.perm"][sf + R]]
        np.add.at(exp, o[J] * k + o[I], 1)
    return exp


@pytest.mark.parametrize("name", NAMES)
def test_schur_analysis_and_plans(driver, tmp_path, name):
    N, cp, rv, perm = matrix(name)
    for sname, S in schur_sets(name, N, perm).items():
        pg = None
        if perm is not None:          # a given permutation: S moved to its end, B in the given order
            inS = np.isin(perm, S)
            pg = np.concatenate([perm[~inS], S]).astype(np.int32)
        d = run(driver, tmp_path, N, cp, rv, pg, S)
        assert isinstance(d, dict), (name, sname, d)
        hits, cut = check_schur(d, N, list(S), pg)
        assert np.array_equal(hits, expected_hits(N, cp, rv, d, list(S), cut)), (name, sname)
        print("%s / %s: |S| %d, %d cut roots, %d fronts" % (name, sname, len(S), len(cut), len(d["sym.sn_parent"])))


def test_s_without_edges_to_b(driver, tmp_path):
    N, cp, rv, _ = matrix("random_qp")
    N2, cp2, rv2 = with_island(N, cp, rv)
    S = np.arange(N, N2)
    d = run(driver, tmp_path, N2, cp2, rv2, None, S)
    hits, cut = check_schur(d, N2, list(S))
    assert cut == [] and (d["sc.rec_ptr"] == 0).all()
    exp = expected_hits(N2, cp2, rv2, d, list(S), cut)
    assert np.array_equal(hits, exp) and exp.reshape(5, 5)[np.tril_indices(5)[1], np.tril_indices(5)[0]].all()


def test_refusals(driver, tmp_path):
    N, cp, rv, perm = matrix("child_records")
    assert run(driver, tmp_path, N, cp, rv, None, [0, 0]) == 3            # duplicate
    assert run(driver, tmp_path, N, cp, rv, None, [N]) == 3               # out of range
    assert run(driver, tmp_path, N, cp, rv, None, np.arange(N)) == 3      # B empty
    assert run(driver, tmp_path, N, cp, rv, perm, [int(perm[0])]) == 3    # the given permutation does not end with S


@pytest.mark.parametrize("name", NAMES)
def test_without_a_schur_set_the_analysis_is_unchanged(driver, tmp_path, name):
    N, cp, rv, perm = matrix(name)
    got = digests(run(driver, tmp_path, N, cp, rv, perm))
    want = json.load(open(GOLDEN))[name]
    assert got == want, [k for k in want if got.get(k) != want[k]]
