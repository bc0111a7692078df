"""Schur complement handles (CudaLDLSolver(..., schur=S), cldl_create_schur): the dense complement
Sc = K_SS - K_SB K_BB^-1 K_BS and the two partial solves, against extended-precision references.

(a) The matrices of tests/ldl_shapes.py with a random Schur set and with the last columns of their ordering (the top
separator), given permutation and ordering of their own.  Reference: X = K_BB^-1 K_BS from an LU of K_BB, refined
once with the residual in np.longdouble, Sc* = K_SS - K_SB X in longdouble.  Error: max |Sc - Sc*| divided by
eps (|K_SS| + |K_SB| |K_BB^-1| |K_BS|) (1-norms).
(b) C4 at 1/25 of its size with S = the linking rows: the same error, with K_BB^-1 applied by a sparse LU and its norm
estimated.
(c) The regularised-pivot matrices of tests/test_ldl_shapes_gpu.py with S at the end of the ordering (the regularised
pivot in B): the complement of K + E_B, E_B the corrections of a dense longdouble LDL^T with the device's pivot rule,
and the exact regularisation count and inertia of B.
(d) condensation, x_S = Sc^-1 w_S in longdouble on the host, expansion: the normwise backward error of x against K.
Also: S with no edge to B gives K_SS bit for bit; two refactors give the same bits; Sc follows value updates at the
next refactor and not before; the refusals.

Worst values measured on an H100 (SXM, 80 GB HBM3, 700 W power limit; the host-emulated build gives the same (a)
and (c) figures to three digits):
  (a) 2.0e-2 (child_records, separator)   (b) 6.9e-3   (c) 8.8e-6 (D pivot 0)   (d) 6.9e-17
The thresholds below keep a margin of at least 100x to these."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import clarabel_rs_b200 as cb
import ldl_shapes

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
LD = np.longdouble
SC_TOL = 5.0          # (a), (b), (c): error / (eps (|K_SS| + |K_SB| |K_BB^-1| |K_BS|))
BWD_TOL = 2e-14       # (d): normwise backward error


def _full(N, cp, rv, nz):
    K = sp.csc_matrix((nz, rv, cp), shape=(N, N))
    return (K + sp.triu(K, 1).T).tocsc()


def _reference(K, S, E=None):
    """(Sc* in longdouble, error scale) for the dense or sparse symmetric K and Schur set S (output order)"""
    N = K.shape[0]
    B = np.setdiff1d(np.arange(N), S)
    if E is not None:
        K = (K + sp.diags(E)).tocsc()
    KBB, KBS, KSS = K[B][:, B].tocsc(), K[B][:, S].toarray(), K[S][:, S].toarray()
    lu = spla.splu(KBB)
    X = lu.solve(KBS)
    R = KBS.astype(LD) - _ld_matmul(KBB.tocsr(), X)
    X = X.astype(LD) + lu.solve(np.asarray(R, np.float64)).astype(LD)
    Sc = KSS.astype(LD) - _ld_matmul(K[S][:, B].tocsr(), X)
    inv_norm = spla.onenormest(spla.LinearOperator(KBB.shape, matvec=lu.solve, rmatvec=lambda v: lu.solve(v, trans="T")))
    scale = np.abs(KSS).sum(axis=0).max() + np.abs(KBS).sum(axis=0).max() ** 2 * inv_norm
    return Sc, float(scale)


def _ld_matmul(Kcsr, X, chunk=16):
    """K X with the products and sums in longdouble"""
    out = np.zeros((Kcsr.shape[0], X.shape[1]), LD)
    Kc = Kcsr.tocoo()
    data = Kc.data.astype(LD)[:, None]
    for c0 in range(0, X.shape[1], chunk):
        np.add.at(out[:, c0:c0 + chunk], Kc.row, data * X[Kc.col, c0:c0 + chunk].astype(LD))
    return out


def _err(Sc, ref, scale):
    return float(np.max(np.abs(Sc.astype(LD) - ref))) / (EPS * scale)


def _with_s_last(perm, S):
    inS = np.isin(perm, S)
    return np.concatenate([np.asarray(perm)[~inS], S])


def _sets(sh):
    rng = np.random.default_rng(7)
    return {"random": rng.choice(sh.N, size=40, replace=False), "separator": np.asarray(sh.perm[-48:])}


@pytest.mark.parametrize("name", [f.__name__ for f in (ldl_shapes.big_fronts, ldl_shapes.child_records)])
def test_shape_matrices_against_the_extended_precision_complement(name):
    sh = getattr(ldl_shapes, name)()
    K = _full(sh.N, sh.cp, sh.rv, sh.nz)
    for sname, S in _sets(sh).items():
        for perm in (_with_s_last(sh.perm, S), None):
            s = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=perm, schur=S)
            assert s.refactor()
            assert s.linear_solver_info().regularize_count == 0
            Sc = s.schur_complement()
            assert Sc.shape == (len(S), len(S)) and np.array_equal(Sc, Sc.T)
            ref, scale = _reference(K, S)
            err = _err(Sc, ref, scale)
            print("%s / %s / %s: error %.2e" % (name, sname, "given" if perm is not None else "ordered", err))
            assert err <= SC_TOL, (name, sname, err)
            _check_partial_solves(s, K, S, np.random.default_rng(3))
            s.close()


def _check_partial_solves(s, K, S, rng):
    """(d): condense, solve the complement in longdouble, expand; returns the backward error"""
    N = K.shape[0]
    Kc = K.tocsr()
    Sc = s.schur_complement()
    worst = 0.0
    for b in (rng.standard_normal(N), rng.choice([-1.0, 1.0], N) * 10.0 ** rng.uniform(-4, 4, N)):
        w = s.schur_reduce(b)
        xS = np.linalg.solve(Sc, w)
        for _ in range(2):
            r = w.astype(LD) - Sc.astype(LD) @ xS.astype(LD)
            xS = xS + np.linalg.solve(Sc, np.asarray(r, np.float64))
        x = s.schur_expand(xS)
        assert np.array_equal(x[S], xS)
        res = b.astype(LD) - _ld_matmul(Kc, x[:, None])[:, 0]
        knorm = float(np.abs(Kc).sum(axis=1).max())
        be = float(np.max(np.abs(res))) / (knorm * np.max(np.abs(x)) + np.max(np.abs(b)))
        worst = max(worst, be)
        assert be <= BWD_TOL, be
    print("  partial solves: backward error %.2e" % worst)
    return worst


def test_reduced_c4_linking_rows():
    import factor_digest
    c = factor_digest.reduced_c4()
    S = np.arange(c.N - 200, c.N)            # the linking rows
    s = cb.CudaLDLSolver(c.N, c.cp, c.rv, c.nz, c.ds, schur=S)
    assert s.refactor()
    assert s.linear_solver_info().regularize_count == 0
    K = _full(c.N, c.cp, c.rv, c.nz)
    ref, scale = _reference(K, S)
    err = _err(s.schur_complement(), ref, scale)
    print("c4_reduced: error %.2e" % err)
    assert err <= SC_TOL, err
    _check_partial_solves(s, K, S, np.random.default_rng(4))


def _ldl_reference(Kp, sp_, eps=1e-13, delta=2e-7):
    A = Kp.astype(LD).copy()
    n = A.shape[0]
    d0, d = np.zeros(n, LD), np.zeros(n, LD)
    for k in range(n):
        d0[k] = d[k] = A[k, k]
        if d[k] * sp_[k] < eps:
            d[k] = delta * sp_[k]
        l = A[k + 1:, k] / d[k]
        A[k + 1:, k + 1:] -= np.outer(l, A[k, k + 1:])
    return d0, d


@pytest.mark.parametrize("group,j", ldl_shapes.REG_SITES)
def test_regularised_pivot_in_b(group, j):
    sh = ldl_shapes.regularised(group, j)
    S = np.asarray(sh.perm[-20:])
    s = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, schur=S)
    assert s.refactor()
    p = s.perm()
    sf = sh.N - len(S)
    d0, d = _ldl_reference(sh.dense()[np.ix_(p[:sf], p[:sf])], sh.ds[p[:sf]].astype(LD))
    info = s.linear_solver_info()
    assert info.regularize_count == int((d != d0).sum()) >= 1
    assert info.positive_inertia == int((d > 0).sum())
    E = np.zeros(sh.N)
    E[p[:sf]] = np.asarray(d - d0, np.float64)
    ref, scale = _reference(_full(sh.N, sh.cp, sh.rv, sh.nz), S, E)
    err = _err(s.schur_complement(), ref, scale)
    print("reg %s %d: error %.2e" % (group, j, err))
    assert err <= SC_TOL, (group, j, err)


def _island():
    """a small KKT matrix plus a 6 x 6 symmetric block joined to nothing"""
    from helpers import small_kkt
    N, cp, rv, nz, ds = small_kkt(60, 40, seed=2)
    m = 6
    rng = np.random.default_rng(8)
    M = rng.standard_normal((m, m))
    M = M + M.T + 8 * np.eye(m)
    cols_r = [rv[cp[j]:cp[j + 1]] for j in range(N)] + [np.arange(N, N + j + 1) for j in range(m)]
    cols_v = [nz[cp[j]:cp[j + 1]] for j in range(N)] + [M[:j + 1, j] for j in range(m)]
    cp2 = np.concatenate([[0], np.cumsum([c.size for c in cols_r])])
    return N + m, cp2, np.concatenate(cols_r), np.concatenate(cols_v), np.concatenate([ds, np.ones(m, np.int8)]), M


def test_s_without_edges_to_b_gives_k_ss_bit_for_bit():
    N, cp, rv, nz, ds, M = _island()
    S = np.arange(N - 6, N)[::-1]
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, schur=S)
    assert s.refactor()
    assert np.array_equal(s.schur_complement().view(np.uint64), M[np.ix_(S - (N - 6), S - (N - 6))].view(np.uint64))


def test_repeatable_and_follows_value_updates_at_the_next_refactor():
    sh = ldl_shapes.big_fronts()
    S = _sets(sh)["random"]
    s = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=_with_s_last(sh.perm, S), schur=S)
    assert s.refactor()
    Sc1 = s.schur_complement()
    assert s.refactor()
    assert np.array_equal(Sc1.view(np.uint64), s.schur_complement().view(np.uint64))
    nz = sh.nz.copy()
    diag = np.nonzero(sh.rv == np.repeat(np.arange(sh.N), np.diff(sh.cp)))[0]
    nz[diag] *= 2.0
    s.update_values(diag, nz[diag])
    assert np.array_equal(Sc1.view(np.uint64), s.schur_complement().view(np.uint64))
    assert s.refactor()
    ref, scale = _reference(_full(sh.N, sh.cp, sh.rv, nz), S)
    assert _err(s.schur_complement(), ref, scale) <= SC_TOL


def test_refusals():
    sh = ldl_shapes.child_records()
    args = (sh.N, sh.cp, sh.rv, sh.nz, sh.ds)
    for bad in ([], [0, 0], [sh.N], np.arange(sh.N)):
        with pytest.raises(cb.BackendError, match="BadArgument"):
            cb.CudaLDLSolver(*args, schur=bad)
    with pytest.raises(cb.BackendError, match="InvalidPermutation"):
        cb.CudaLDLSolver(*args, perm=sh.perm, schur=[int(sh.perm[0])])
    with pytest.raises(cb.BackendError, match="BadArgument"):
        cb.CudaLDLSolver(*args, schur=[1], shard_nranks=2, shard_rank=0)
    S = np.asarray(sh.perm[-10:])
    s = cb.CudaLDLSolver(*args, perm=sh.perm, schur=S)
    b = np.ones(sh.N)
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.schur_complement()
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.schur_reduce(b)
    assert s.refactor()
    with pytest.raises(cb.BackendError, match="BadArgument"):
        s.schur_expand(np.zeros(len(S)))           # no condensation since the refactor
    with pytest.raises(cb.BackendError, match="BadArgument"):
        s.solve(b)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        s.selected_inverse()
    vp = cb.lib().cldl_shard_refactor_phase_dev
    assert vp(s._h, 0) == cb.CLDL_E_ARG
    s.schur_reduce(b)
    s.schur_expand(np.zeros(len(S)))
    with pytest.raises(cb.BackendError, match="BadArgument"):
        s.schur_expand(np.zeros(len(S)))           # the condensation was consumed
    s.close()
    t = cb.CudaLDLSolver(*args, perm=sh.perm)
    assert t.refactor()
    t.nschur = 1
    for call in (lambda: t.schur_complement(), lambda: t.schur_reduce(b), lambda: t.schur_expand(np.zeros(1))):
        with pytest.raises(cb.BackendError, match="BadArgument"):
            call()
    t.close()
