"""Pruned solves (CudaLDLSolver.solve_sparse / inverse_entries, cldl_solve_sparse(_dev) / cldl_inverse_entries).

Bitwise: the entries a pruned solve returns compare equal (==) to the same entries of solve() on the densified b, for
sparse and dense b and x, on the matrices of tests/ldl_shapes.py (every front shape the sweeps dispatch on) and on
matrices that regularise pivots, with index sets of size 1, 2, 17 and n inside one leaf, in the root separator only
and spread over the tree.  inverse_entries(i, j) equals solve(e_j)[i].
Accuracy: entries of (K + E)^-1 on and off K's pattern against the dense inverse refined in np.longdouble, and on the
pattern against selected_inverse(), at SHAPE_TOL eps cond_1(K).
Also: the refusals, two calls giving the same bits, the factor and a later solve() unchanged, and a C2-sized case."""
import ctypes as C
import hashlib
import os
import zlib

import numpy as np
import pytest
import scipy.sparse as sp

import clarabel_rs_b200 as cb
import ldl_shapes

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
LD = np.longdouble
SHAPE_TOL = 5.0
SIZES = [1, 2, 17, "n"]
WHERE = ["leaf", "root", "spread"]


def _solver(sh):
    return cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm)


def _index_set(s, size, where, rng):
    """caller indices: permuted positions from the start (the first front in postorder is a leaf), from the end (the
    root separator) or drawn at random"""
    n = s.n
    k = n if size == "n" else size
    p = s.perm()
    if where == "leaf":
        pos = np.arange(k)
    elif where == "root":
        pos = np.arange(n - k, n)
    else:
        pos = rng.choice(n, size=k, replace=False)
    return p[pos]


def _same(a, b):
    return a.shape == b.shape and bool(np.all(a == b))


def _check_all_combinations(s, rng, bidx, widx):
    n = s.n
    bv = rng.standard_normal(bidx.size)
    bd = np.zeros(n)
    bd[bidx] = bv
    full = s.solve(bd)
    assert _same(s.solve_sparse((bidx, bv), widx), full[widx])          # sparse b, sparse x
    st = s.sparse_stats()
    assert st["fronts_fwd"] >= 1 and st["fronts_bwd"] >= 1
    assert _same(s.solve_sparse((bidx, bv)), full)                      # sparse b, dense x
    assert _same(s.solve_sparse(bd, widx), full[widx])                  # dense b, sparse x
    assert _same(s.solve_sparse(bd), full)                              # dense b, dense x


SHAPES = [f.__name__ for f in (ldl_shapes.big_fronts, ldl_shapes.child_records)]


@pytest.mark.parametrize("where", WHERE)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("name", SHAPES)
def test_bitwise_equal_to_the_full_solve(name, size, where):
    sh = getattr(ldl_shapes, name)()
    s = _solver(sh)
    assert s.refactor()
    rng = np.random.default_rng(zlib.crc32(f"{name}-{size}-{where}".encode()))
    bidx = _index_set(s, size, where, rng)
    # the wanted set: the same kind of set, elsewhere for "spread", with a duplicate
    widx = _index_set(s, size, where, rng)
    widx = np.concatenate([widx, widx[:1]])
    _check_all_combinations(s, rng, bidx, widx)
    s.close()


@pytest.mark.parametrize("group,j", ldl_shapes.REG_SITES)
def test_bitwise_on_regularised_matrices(group, j):
    sh = ldl_shapes.regularised(group, j)
    s = _solver(sh)
    assert s.refactor()
    assert s.linear_solver_info().regularize_count >= 1
    rng = np.random.default_rng(7)
    for size in (1, 17):
        for where in WHERE:
            _check_all_combinations(s, rng, _index_set(s, size, where, rng), _index_set(s, size, "spread", rng))
    s.close()


def _ld_matmul(Kcsr, X, chunk=128):
    out = np.empty((Kcsr.shape[0], X.shape[1]), LD)
    data = Kcsr.data.astype(LD)[:, None]
    for c0 in range(0, X.shape[1], chunk):
        prod = data * X[Kcsr.indices, c0:c0 + chunk].astype(LD)
        out[:, c0:c0 + chunk] = np.add.reduceat(prod, Kcsr.indptr[:-1], axis=0)
    return out


def _sym(sh):
    K = sp.csc_matrix((sh.nz, sh.rv, sh.cp), shape=(sh.N, sh.N))
    return (K + sp.triu(K, 1).T).tocsr()


def _inverse_reference(Kcsr):
    Kd = Kcsr.toarray()
    X = np.linalg.inv(Kd)
    R = np.eye(Kd.shape[0], dtype=LD) - _ld_matmul(Kcsr, X)
    return X.astype(LD) + (X @ np.asarray(R, np.float64)).astype(LD), np.linalg.cond(Kd, 1)


@pytest.mark.parametrize("name", SHAPES)
def test_inverse_entries_accuracy_and_bitwise(name):
    sh = getattr(ldl_shapes, name)()
    s = _solver(sh)
    assert s.refactor()
    assert s.linear_solver_info().regularize_count == 0
    n = sh.N
    ref, cond = _inverse_reference(_sym(sh))
    scale = float(np.max(np.abs(ref)))
    rng = np.random.default_rng(5)
    # off the pattern: random positions, duplicates and both triangles; on the pattern: every stored entry
    rows = rng.integers(0, n, 300)
    cols = rng.integers(0, n, 300)
    rows, cols = np.concatenate([rows, rows[:3], cols[:5]]), np.concatenate([cols, cols[:3], rows[:5]])
    z = s.inverse_entries(rows, cols)
    err = float(np.max(np.abs(z.astype(LD) - ref[rows, cols]))) / scale / (EPS * cond)
    print("%s: off-pattern error / (eps cond_1) %.2e (cond_1 %.1e)" % (name, err, cond))
    assert err <= SHAPE_TOL, err
    pr = sh.rv.astype(np.int64)
    pc = np.repeat(np.arange(n), np.diff(sh.cp))
    zp = s.inverse_entries(pr, pc)
    err_p = float(np.max(np.abs(zp.astype(LD) - ref[pr, pc]))) / scale / (EPS * cond)
    assert err_p <= SHAPE_TOL, err_p
    Z = s.selected_inverse().tocoo()
    zsel = s.inverse_entries(Z.row, Z.col)
    assert float(np.max(np.abs(zsel - Z.data))) / scale / (EPS * cond) <= SHAPE_TOL
    # bitwise: inverse_entries(i, j) == solve(e_j)[i] for a few columns
    for j in rng.choice(n, 5, replace=False):
        e = np.zeros(n)
        e[j] = 1.0
        x = s.solve(e)
        ri = rng.choice(n, 40, replace=False)
        assert _same(s.inverse_entries(ri, np.full(ri.size, j)), x[ri])
        # the same column paired with another one in the two-column sweep
        j2 = (j + n // 2) % n
        both = s.inverse_entries(np.concatenate([ri, ri]), np.concatenate([np.full(ri.size, j), np.full(ri.size, j2)]))
        assert _same(both[:ri.size], x[ri])
    s.close()


def _factor_bytes(s):
    info = s.linear_solver_info()
    L, D, Dinv = np.empty(info.nnzL_stored), np.empty(s.n), np.empty(s.n)
    f = cb.lib().cldl_get_factor
    f.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * 3
    f.restype = C.c_int
    assert f(s._h, *(a.ctypes.data_as(C.POINTER(C.c_double)) for a in (L, D, Dinv))) == 0
    return [hashlib.sha256(a.tobytes()).hexdigest() for a in (L, D, Dinv)]


def test_repeatable_and_leaves_the_factor_and_solves_unchanged():
    sh = ldl_shapes.big_fronts()
    s = _solver(sh)
    assert s.refactor()
    rng = np.random.default_rng(3)
    b = rng.standard_normal(sh.N)
    before, x0 = _factor_bytes(s), s.solve(b)
    bi = rng.choice(sh.N, 9, replace=False)
    bv = rng.standard_normal(9)
    wi = rng.choice(sh.N, 11, replace=False)
    x1 = s.solve_sparse((bi, bv), wi)
    x2 = s.solve_sparse((bi, bv), wi)
    assert np.array_equal(x1.view(np.uint64), x2.view(np.uint64))
    z1 = s.inverse_entries(wi, np.full(11, bi[0]))
    z2 = s.inverse_entries(wi, np.full(11, bi[0]))
    assert np.array_equal(z1.view(np.uint64), z2.view(np.uint64))
    assert _factor_bytes(s) == before
    assert np.array_equal(s.solve(b).view(np.uint64), x0.view(np.uint64))
    # nb = 0 gives zeros
    assert np.all(s.solve_sparse((np.zeros(0, np.int64), np.zeros(0)), wi) == 0.0)
    s.close()


def test_device_pointer_form():
    import torch
    dev = torch.device("cpu") if os.environ.get("CLARABEL_EMU") == "1" else torch.device("cuda", 0)
    sh = ldl_shapes.child_records()
    s = _solver(sh)
    assert s.refactor()
    rng = np.random.default_rng(4)
    bi = rng.choice(sh.N, 17, replace=False)
    bv = rng.standard_normal(17)
    wi = rng.choice(sh.N, 17, replace=False)
    bd = np.zeros(sh.N)
    bd[bi] = bv
    full = s.solve(bd)
    db = torch.tensor(bv, dtype=torch.float64, device=dev)
    dx = torch.empty(17, dtype=torch.float64, device=dev)
    dxf = torch.empty(sh.N, dtype=torch.float64, device=dev)
    if dev.type == "cuda":
        torch.cuda.synchronize()
    for _ in range(3):      # the pinned buffers are reused in turn
        s.solve_sparse_dev(bi, db.data_ptr(), 17, wi, dx.data_ptr())
        s.solve_sparse_dev(bi, db.data_ptr(), 17, None, dxf.data_ptr())
        if dev.type == "cuda":
            torch.cuda.ExternalStream(s.stream_ptr()).synchronize()
        assert _same(dx.cpu().numpy(), full[wi])
        assert _same(dxf.cpu().numpy(), full)
    s.close()


def test_refusals():
    sh = ldl_shapes.child_records()
    s = _solver(sh)
    one = (np.array([0]), np.array([1.0]))
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.solve_sparse(one)
    with pytest.raises(cb.BackendError, match="NotFactored"):
        s.inverse_entries([0], [0])
    assert s.refactor()
    with pytest.raises(cb.BackendError, match="BadArgument"):
        s.solve_sparse((np.array([sh.N]), np.array([1.0])))
    with pytest.raises(cb.BackendError, match="BadArgument"):
        s.solve_sparse(one, [sh.N])
    with pytest.raises(cb.BackendError, match="BadArgument"):
        s.solve_sparse((np.array([3, 5, 3]), np.ones(3)))
    with pytest.raises(cb.BackendError, match="BadArgument"):
        s.inverse_entries([0], [sh.N])
    with pytest.raises(cb.BackendError, match="BadArgument"):
        s.inverse_entries([sh.N], [0])
    t = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm, shard_nranks=2, shard_rank=0)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        t.solve_sparse(one)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        t.inverse_entries([0], [0])
    t.close()
    u = cb.CudaLDLSolver(sh.N, sh.cp, sh.rv, sh.nz, sh.ds, schur=[sh.N - 1, sh.N - 2])
    assert u.refactor()
    with pytest.raises(cb.BackendError, match="BadArgument"):
        u.solve_sparse(one)
    with pytest.raises(cb.BackendError, match="BadArgument"):
        u.inverse_entries([0], [0])
    u.close()
    s.close()


def test_c2_sized_kkt():
    from helpers import workloads
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
    s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=cb.ORDER_ND)
    assert s.refactor()
    rng = np.random.default_rng(2)
    for nb, nx in ((1, 10), (100, 10), (10, None)):
        bi = rng.choice(N, nb, replace=False)
        bv = rng.standard_normal(nb)
        wi = None if nx is None else rng.choice(N, nx, replace=False)
        bd = np.zeros(N)
        bd[bi] = bv
        full = s.solve(bd)
        x = s.solve_sparse((bi, bv), wi)
        assert _same(x, full if wi is None else full[wi])
        st = s.sparse_stats()
        assert st["fronts_fwd"] < s.linear_solver_info().n_supernodes
    j = int(rng.integers(N))
    e = np.zeros(N)
    e[j] = 1.0
    ri = rng.choice(N, 50, replace=False)
    assert _same(s.inverse_entries(ri, np.full(50, j)), s.solve(e)[ri])
    s.close()
