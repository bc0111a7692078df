"""The stored factor of the device LDL^T on a fixed set of matrices, reduced to a digest: SHA-256 of the bytes of the
front panels (as the solves read them, inverted pivot blocks included), of D and of 1/D, plus the regularisation count
and the positive inertia.  tests/golden/ldl/factor_digests.json holds the digests of a build whose kernels are known good;
tests/test_level0_factor_gpu.py asserts equality, bit for bit.  scripts/make_factor_digests.py writes the file."""
import ctypes as C
import hashlib

import numpy as np

import clarabel_rs_b200 as cb
import ldl_shapes


class Case:
    def __init__(self, name, N, cp, rv, nz, ds, perm=None, ordering=cb.ORDER_BEST):
        self.name, self.N, self.cp, self.rv, self.nz, self.ds, self.perm, self.ordering = name, N, cp, rv, nz, ds, perm, ordering


def _shape_case(sh):
    return Case(sh.name, sh.N, sh.cp, sh.rv, sh.nz, sh.ds, perm=sh.perm)


def reduced_c4():
    """the block-angular QP of the benchmark's C4 at 1/25 of its size (KKT at a random diagonal scaling)"""
    from helpers import workloads
    pr = workloads.block_angular_qp(n=40_000, nblocks=16, nlink=200, link_blocks=8, seed=3)
    hd = np.random.default_rng(0).uniform(0.5, 2.0, pr["A"].shape[0])
    N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], hd)
    return Case("c4_reduced", N, cp, rv, nz, ds)


def cases():
    out = [_shape_case(sh) for sh in ldl_shapes.all_shapes()]
    out += [_shape_case(ldl_shapes.regularised(g, j)) for g, j in ldl_shapes.REG_SITES]
    out.append(reduced_c4())
    return out


def case(name):
    """one case of cases(), built alone"""
    if name == "c4_reduced":
        return reduced_c4()
    if name.startswith("reg_"):
        g, j = name[4:].rsplit("_", 1)
        return _shape_case(ldl_shapes.regularised(g, int(j)))
    return _shape_case(getattr(ldl_shapes, name)())


def solver(case):
    return cb.CudaLDLSolver(case.N, case.cp, case.rv, case.nz, case.ds, perm=case.perm, ordering=case.ordering)


def digest(s):
    """refactor s and return the digest of what it stored"""
    assert s.refactor()
    info = s.linear_solver_info()
    L = np.empty(info.nnzL_stored, np.float64)
    D = np.empty(s.n, np.float64)
    Dinv = np.empty(s.n, np.float64)
    lib = cb.lib()
    f = lib.cldl_get_factor
    f.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * 3
    f.restype = C.c_int
    rc = f(s._h, L.ctypes.data_as(C.POINTER(C.c_double)), D.ctypes.data_as(C.POINTER(C.c_double)),
           Dinv.ctypes.data_as(C.POINTER(C.c_double)))
    assert rc == 0, rc
    return {"L": hashlib.sha256(L.tobytes()).hexdigest(), "D": hashlib.sha256(D.tobytes()).hexdigest(),
            "Dinv": hashlib.sha256(Dinv.tobytes()).hexdigest(),
            "regularize_count": int(info.regularize_count), "positive_inertia": int(info.positive_inertia)}
