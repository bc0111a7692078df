"""clarabel.rs_b200 -- GPU-native KKT backend (host-side Python mirror).

The product is the C-ABI shared library ``libclarabel_b200.so`` (CUDA, sm_90a;
see ``include/clarabel_b200.h``).  This module is the thin ctypes binding used
by the tests and the bench; it mirrors the reference's plugin interface names:

* ``CudaLDLSolver``      <-> ``trait DirectLDLSolver`` + the qdldl adapter
  (/root/reference/src/solver/core/kktsolvers/direct/quasidef/mod.rs:14-26,
  .../ldlsolvers/qdldl.rs:19-107): ``update_values / scale_values /
  offset_values / refactor / solve / linear_solver_info``.
* ``SymbolicAnalysis``   host-only view of the ordering / supernodal analysis.

There is NO CPU fallback: if the shared library is missing, or no CUDA device
is present when a device object is constructed, this raises.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBPATH = os.path.join(_HERE, "libclarabel_b200.so")
_lib = None


class BadInputData(ValueError):
    """SolverError::BadInputData (src/solver/core/traits.rs): what DefaultSolver::new returns for inconsistent data"""


def cone_nvars(kind, d):
    """SupportedConeT::nvars (supportedcone.rs:54-71)"""
    if kind in ("exp", "pow"):
        return 3
    if kind == "psd":
        return int(d) * (int(d) + 1) // 2
    if kind == "genpow":
        return len(d[0]) + int(d[1])
    return int(d)


def get_infinity():
    """get_infinity (src/utils/infbounds.rs)"""
    L = _lib2()
    L.cipm_get_infinity.restype = C.c_double
    return float(L.cipm_get_infinity())


def set_infinity(v):
    L = _lib2()
    L.cipm_set_infinity.argtypes = [C.c_double]
    L.cipm_set_infinity.restype = None
    L.cipm_set_infinity(float(v))


def default_infinity():
    L = _lib2()
    L.cipm_default_infinity.restype = None
    L.cipm_default_infinity()


def check_dimensions(P, q, A, b, cones):
    """check_dimensions of DefaultSolver::new (implementations/default/solver.rs:129-159): same tests, same order,
    same messages; pinned by tests/api_dimension_checks.rs"""
    m, n = len(b), len(q)
    p = sum(cone_nvars(k, d) for k, d in cones)
    if m != A.shape[0]:
        raise BadInputData("A and b incompatible dimensions")
    if p != m:
        raise BadInputData("Constraint dimensions inconsistent with size of cones")
    if n != A.shape[1]:
        raise BadInputData("A and q incompatible dimensions")
    if n != P.shape[1]:
        raise BadInputData("P and q incompatible dimensions")
    if P.shape[0] != P.shape[1]:
        raise BadInputData("P not square")


class DataUpdateError(ValueError):
    """DataUpdateError (data_updating.rs:9-33): PresolveIsActive, BadVectorDimension, BadFormat"""


class BackendError(RuntimeError):
    pass


CLDL_OK = 0
CLDL_E_DIM, CLDL_E_EMPTY_COLUMN, CLDL_E_NOT_TRIU = -1, -2, -3
CLDL_E_ZERO_PIVOT, CLDL_E_BAD_PERM = -4, -5
CLDL_E_CUDA, CLDL_E_ARG, CLDL_E_NOT_FACTORED = -20, -21, -22
ORDER_AMD, ORDER_ND, ORDER_BEST = 1, 2, 3

_ERRNAMES = {
    -1: "IncompatibleDimension", -2: "EmptyColumn", -3: "NotUpperTriangular",
    -4: "ZeroPivot", -5: "InvalidPermutation", -20: "CudaFailure (no device / runtime error)",
    -21: "BadArgument", -22: "NotFactored",
}


class cldl_opts(C.Structure):
    _fields_ = [
        ("regularize_eps", C.c_double),
        ("regularize_delta", C.c_double),
        ("regularize_enable", C.c_int32),
        ("amd_dense_scale", C.c_double),
        ("ordering", C.c_int32),
        ("device", C.c_int32),
        ("max_panel", C.c_int32),
        ("nd_leaf", C.c_int32),
        ("shard_nranks", C.c_int32),
        ("shard_rank", C.c_int32),
    ]


# cldl_allgather_fn: int (*)(void* ctx, const double* d_send, double* d_recv, uint64_t count)
ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64)


class cldl_info_t(C.Structure):
    _fields_ = [
        ("name", C.c_char * 16),
        ("threads", C.c_uint32),
        ("direct", C.c_int32),
        ("nnzA", C.c_uint64),
        ("nnzL", C.c_uint64),
        ("nnzL_stored", C.c_uint64),
        ("regularize_count", C.c_uint64),
        ("positive_inertia", C.c_uint64),
        ("n_supernodes", C.c_uint64),
        ("n_levels", C.c_uint64),
        ("flops", C.c_double),
        ("ordering_used", C.c_int32),
    ]


# every symbol declared in include/clarabel_b200.h (checked by tests/test_abi.py)
EXPORTED_SYMBOLS = [
    "cldl_default_opts", "cldl_create", "cldl_destroy", "cldl_update_values",
    "cldl_scale_values", "cldl_offset_values", "cldl_refactor", "cldl_solve",
    "cldl_info", "cldl_get_perm", "cldl_update_values_dev", "cldl_set_values_dev",
    "cldl_refactor_dev", "cldl_solve_dev", "cldl_sync_status", "cldl_stream",
    "cldl_values_dev", "cldl_time_refactor_ms", "cldl_time_solve_ms",
    "cldl_selected_inverse", "cldl_selected_inverse_dev",
    "cldl_create_schur", "cldl_schur_complement", "cldl_schur_complement_dev", "cldl_schur_reduce",
    "cldl_schur_reduce_dev", "cldl_schur_expand", "cldl_schur_expand_dev",
    "cldl_logdet", "cldl_adjoint_solve", "cldl_adjoint_solve_dev",
]


def lib() -> C.CDLL:
    """Load the CUDA shared library; fail loudly when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIBPATH):
        raise BackendError(
            f"{_LIBPATH} not found: build it with `make` (or __graft_entry__.build()); "
            "this backend has no CPU fallback")
    L = C.CDLL(_LIBPATH)
    u64p, f64p, i8p, i32p = (C.POINTER(C.c_uint64), C.POINTER(C.c_double),
                             C.POINTER(C.c_int8), C.POINTER(C.c_int32))
    vp = C.c_void_p
    L.cldl_default_opts.argtypes = [C.POINTER(cldl_opts)]
    L.cldl_default_opts.restype = None
    L.cldl_create.argtypes = [C.POINTER(vp), C.c_uint64, u64p, u64p, f64p, i8p,
                              C.POINTER(cldl_opts), u64p]
    L.cldl_create.restype = C.c_int
    L.cldl_destroy.argtypes = [vp]
    L.cldl_destroy.restype = None
    L.cldl_update_values.argtypes = [vp, u64p, f64p, C.c_uint64]
    L.cldl_scale_values.argtypes = [vp, u64p, C.c_uint64, C.c_double]
    L.cldl_offset_values.argtypes = [vp, u64p, C.c_uint64, C.c_double, i8p]
    L.cldl_refactor.argtypes = [vp]
    L.cldl_solve.argtypes = [vp, f64p, f64p]
    L.cldl_info.argtypes = [vp, C.POINTER(cldl_info_t)]
    L.cldl_info.restype = None
    L.cldl_get_perm.argtypes = [vp, u64p]
    L.cldl_update_values_dev.argtypes = [vp, vp, vp, C.c_uint64]
    L.cldl_set_values_dev.argtypes = [vp, vp]
    L.cldl_refactor_dev.argtypes = [vp]
    L.cldl_solve_dev.argtypes = [vp, vp, vp]
    L.cldl_sync_status.argtypes = [vp]
    L.cldl_stream.argtypes = [vp]
    L.cldl_stream.restype = vp
    L.cldl_values_dev.argtypes = [vp]
    L.cldl_values_dev.restype = vp
    L.cldl_time_refactor_ms.argtypes = [vp, C.c_int]
    L.cldl_time_refactor_ms.restype = C.c_double
    L.cldl_time_solve_ms.argtypes = [vp, C.c_int]
    L.cldl_time_solve_ms.restype = C.c_double
    L.cldl_shard_refactor_phase_dev.argtypes = [vp, C.c_int]
    L.cldl_shard_solve_phase_dev.argtypes = [vp, vp, vp, C.c_int]
    L.cldl_shard_count.argtypes = [vp, C.c_int, C.c_int]
    L.cldl_shard_count.restype = C.c_uint64
    L.cldl_shard_pack_dev.argtypes = [vp, C.c_int, vp, vp]
    L.cldl_shard_unpack_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp]
    L.cldl_shard_counts.argtypes = [vp, u64p]
    L.cldl_set_transport.argtypes = [vp, ALLGATHER_FN, vp]
    L.cldl_copy_dev.argtypes = [vp, vp, C.c_uint64]
    # host-only symbolic API
    L.csym_analyse.argtypes = [C.POINTER(vp), C.c_uint64, u64p, u64p, u64p, C.c_int,
                               C.c_double, C.c_int, C.c_int]
    L.csym_free.argtypes = [vp]
    L.csym_free.restype = None
    L.csym_scalar.argtypes = [vp, C.c_int]
    L.csym_scalar.restype = C.c_int64
    L.csym_flops.argtypes = [vp, C.c_int]
    L.csym_flops.restype = C.c_double
    L.csym_array.argtypes = [vp, C.c_int, C.POINTER(C.c_int64), C.c_int64]
    L.csym_array.restype = C.c_int64
    L.csym_order.argtypes = [C.c_uint64, u64p, u64p, C.c_int, C.c_double, C.c_int, u64p]
    _lib = L
    return L


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _check(rc, what):
    if rc < 0:
        raise BackendError(f"{what} failed: {_ERRNAMES.get(rc, rc)}")
    return rc


@dataclass
class LinearSolverInfo:
    """Mirror of kktsolvers/mod.rs:24-38 plus factorisation counters."""
    name: str
    threads: int
    direct: bool
    nnzA: int
    nnzL: int
    nnzL_stored: int
    regularize_count: int
    positive_inertia: int
    n_supernodes: int
    n_levels: int
    flops: float
    ordering_used: int


class CudaLDLSolver:
    """Device LDL^T backend with the ``DirectLDLSolver`` method set.

    ``KKT`` is (n, colptr, rowval, nzval) of the upper-triangular CSC KKT matrix.
    Constructor arguments follow ``ldlsolvers/config.rs:19-20``:
    (KKT, Dsigns, settings, perm).
    """

    required_matrix_shape = "triu"  # DirectLDLSolverReqs, ldlsolvers/qdldl.rs:54-56

    def __init__(self, n, colptr, rowval, nzval, dsigns, *, perm=None,
                 regularize_eps=1e-13, regularize_delta=2e-7, regularize_enable=True,
                 amd_dense_scale=1.5, ordering=ORDER_BEST, device=0, max_panel=0, nd_leaf=0,
                 shard_nranks=0, shard_rank=0, schur=None):
        """``schur``: a Schur set (caller indices, in the order the complement's rows and columns take) makes a Schur
        complement handle: ``refactor()`` factors the other indices only, and ``schur_complement()``,
        ``schur_reduce()`` and ``schur_expand()`` replace ``solve()`` (see cldl_create_schur)."""
        L = lib()
        self._L = L
        self.n = int(n)
        o = cldl_opts()
        L.cldl_default_opts(C.byref(o))
        o.shard_nranks, o.shard_rank = int(shard_nranks), int(shard_rank)
        o.regularize_eps, o.regularize_delta = regularize_eps, regularize_delta
        o.regularize_enable = 1 if regularize_enable else 0
        o.amd_dense_scale, o.ordering, o.device = amd_dense_scale, ordering, device
        o.max_panel, o.nd_leaf = max_panel, nd_leaf
        cp, rv, nz = _u64(colptr), _u64(rowval), _f64(nzval)
        ds = np.ascontiguousarray(dsigns, dtype=np.int8)
        pm = _u64(perm) if perm is not None else None
        h = C.c_void_p()
        self.nschur = 0
        if schur is None:
            rc = L.cldl_create(C.byref(h), self.n, _p(cp, C.c_uint64), _p(rv, C.c_uint64),
                               _p(nz, C.c_double), _p(ds, C.c_int8), C.byref(o),
                               _p(pm, C.c_uint64) if pm is not None else None)
            _check(rc, "cldl_create")
        else:
            si = np.asarray(schur, dtype=np.int64).ravel()
            if si.size == 0 or (si < 0).any():
                raise BackendError("cldl_create_schur failed: BadArgument")
            si = _u64(si)
            f = L.cldl_create_schur
            f.argtypes = [C.POINTER(C.c_void_p), C.c_uint64] + [C.POINTER(C.c_uint64)] * 2 + \
                [C.POINTER(C.c_double), C.POINTER(C.c_int8), C.POINTER(cldl_opts), C.POINTER(C.c_uint64), C.c_uint64,
                 C.POINTER(C.c_uint64)]
            f.restype = C.c_int
            rc = f(C.byref(h), self.n, _p(cp, C.c_uint64), _p(rv, C.c_uint64), _p(nz, C.c_double), _p(ds, C.c_int8),
                   C.byref(o), _p(pm, C.c_uint64) if pm is not None else None, si.size, _p(si, C.c_uint64))
            _check(rc, "cldl_create_schur")
            self.nschur = int(si.size)
        self._h = h
        self._pattern = (cp, rv)

    def close(self):
        if getattr(self, "_h", None):
            self._L.cldl_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_transport(self, transport):
        """install the all-gather of a sharded handle (e.g. TorchDistTransport): refactor() / solve() then run their
        phases and exchanges themselves"""
        self._transport = transport
        _check(self._L.cldl_set_transport(self._h, transport.fn, None), "set_transport")

    # --- DirectLDLSolver trait ---
    def update_values(self, index, values):
        idx, v = _u64(index), _f64(values)
        assert idx.shape == v.shape
        _check(self._L.cldl_update_values(self._h, _p(idx, C.c_uint64), _p(v, C.c_double), idx.size),
               "update_values")

    def scale_values(self, index, scale):
        idx = _u64(index)
        _check(self._L.cldl_scale_values(self._h, _p(idx, C.c_uint64), idx.size, float(scale)),
               "scale_values")

    def offset_values(self, index, offset, signs):
        idx = _u64(index)
        sg = np.ascontiguousarray(signs, dtype=np.int8)
        assert idx.size == sg.size  # qdldl.rs:167
        _check(self._L.cldl_offset_values(self._h, _p(idx, C.c_uint64), idx.size, float(offset),
                                          _p(sg, C.c_int8)), "offset_values")

    def refactor(self) -> bool:
        return bool(_check(self._L.cldl_refactor(self._h), "refactor"))

    def solve(self, b):
        b = _f64(b)
        assert b.size == self.n  # qdldl.rs:121
        x = np.empty_like(b)
        _check(self._L.cldl_solve(self._h, _p(x, C.c_double), _p(b, C.c_double)), "solve")
        return x

    def linear_solver_info(self) -> LinearSolverInfo:
        i = cldl_info_t()
        self._L.cldl_info(self._h, C.byref(i))
        return LinearSolverInfo(i.name.decode(), i.threads, bool(i.direct), i.nnzA, i.nnzL,
                                i.nnzL_stored, i.regularize_count, i.positive_inertia,
                                i.n_supernodes, i.n_levels, i.flops, i.ordering_used)

    def perm(self):
        p = np.empty(self.n, dtype=np.uint64)
        _check(self._L.cldl_get_perm(self._h, _p(p, C.c_uint64)), "get_perm")
        return p.astype(np.int64)

    def selected_inverse(self):
        """Selected inversion: the entries of (K + E)^-1 at the stored entries of the upper-triangular matrix passed
        to the constructor, diagonal included, as a ``scipy.sparse.csc_matrix`` with that pattern.  K + E is the
        matrix the last ``refactor()`` factored, E its dynamic regularisation (``regularize_count`` pivots).

        Valid after a ``refactor()`` that returned True; raises BackendError (NotFactored) otherwise and
        (BadArgument) on a sharded handle.  Computed on the GPU in one pass over the factor, about the work of a
        refactor.  The first call allocates device memory that stays until ``close()``: one more array of
        ``nnzL_stored`` doubles (the inverse in the factor's panel layout), the gather maps (about 12 bytes per row
        index of the factor plus the segment positions) and nnzA doubles and int64s for the caller-order map and
        result.  The factor and later solves are unchanged."""
        import scipy.sparse as sps
        f = self._L.cldl_selected_inverse
        f.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        f.restype = C.c_int
        cp, rv = self._pattern
        out = np.empty(rv.size, np.float64)
        _check(f(self._h, _p(out, C.c_double)), "selected_inverse")
        return sps.csc_matrix((out, rv.astype(np.int64), cp.astype(np.int64)), shape=(self.n, self.n))

    def slogdet(self):
        """(sign, logabsdet) of K + E, the matrix the last ``refactor()`` factored (E its dynamic regularisation), from
        the factor's pivots: logabsdet = sum log|d_k|, sign = (-1)^(negative pivots).  On a Schur handle, of
        K_BB + E_B.  BackendError (NotFactored) before a refactor that returned True, (BadArgument) on a sharded
        handle (see cldl_logdet)."""
        f = self._L.cldl_logdet
        f.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int32)]
        f.restype = C.c_int
        ld, sg = C.c_double(), C.c_int32()
        _check(f(self._h, C.byref(ld), C.byref(sg)), "logdet")
        return int(sg.value), float(ld.value)

    def adjoint_solve(self, g, x):
        """The adjoint of x = K^-1 b for an output gradient g: (gb, gvals) with gb = (K + E)^-1 g (n values) and gvals
        the gradient of <g, x> with respect to the stored upper-triangle values, -(gb_i x_j + x_i gb_j) off the
        diagonal and -gb_i x_i on it, as a ``scipy.sparse.csc_matrix`` with the constructor's pattern.  ``x`` is the
        solution being differentiated (``solve(b)`` on the current factor).  BackendError (NotFactored) before a
        refactor that returned True, (BadArgument) on a Schur or sharded handle (see cldl_adjoint_solve)."""
        import scipy.sparse as sps
        f = self._L.cldl_adjoint_solve
        f.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * 4
        f.restype = C.c_int
        g, x = _f64(g), _f64(x)
        assert g.size == self.n and x.size == self.n
        cp, rv = self._pattern
        gb, gv = np.empty(self.n, np.float64), np.empty(rv.size, np.float64)
        _check(f(self._h, _p(g, C.c_double), _p(x, C.c_double), _p(gb, C.c_double), _p(gv, C.c_double)),
               "adjoint_solve")
        return gb, sps.csc_matrix((gv, rv.astype(np.int64), cp.astype(np.int64)), shape=(self.n, self.n))

    # --- Schur complement handles (constructed with schur=...) ---
    def _schur_call(self, name, *args):
        f = getattr(self._L, name)
        f.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * len(args)
        f.restype = C.c_int
        _check(f(self._h, *(_p(a, C.c_double) for a in args)), name[5:])

    def schur_complement(self):
        """The dense Schur complement K_SS - K_SB K_BB^-1 K_BS assembled by the last ``refactor()`` (which must have
        returned True), as a (k, k) array in the order of the Schur set.  With regularisation it is the complement of
        K + E_B, E_B the dynamic regularisation of B's pivots.  BackendError (NotFactored) before such a refactor,
        (BadArgument) on a handle without a Schur set."""
        k = self.nschur
        out = np.empty(k * k, np.float64)
        self._schur_call("cldl_schur_complement", out)
        return out.reshape((k, k), order="F")

    def schur_reduce(self, b):
        """Condensation: w_S = b_S - K_SB K_BB^-1 b_B (b: n values in the caller's order; w_S in the Schur set's
        order)."""
        b = _f64(b)
        assert b.size == self.n
        w = np.empty(self.nschur, np.float64)
        self._schur_call("cldl_schur_reduce", w, b)
        return w

    def schur_expand(self, xS):
        """Expansion: the whole solution x (n values) from x_S solving Sc x_S = w_S, for the b of the last
        ``schur_reduce``.  Each expansion consumes its condensation: BackendError (BadArgument) without one since the
        last refactor or expansion."""
        xS = _f64(xS)
        assert xS.size == self.nschur
        x = np.empty(self.n, np.float64)
        self._schur_call("cldl_schur_expand", x, xS)
        return x

    # --- device-side helpers (bench) ---
    def time_refactor_ms(self, reps):
        return self._L.cldl_time_refactor_ms(self._h, int(reps))

    def time_solve_ms(self, reps):
        return self._L.cldl_time_solve_ms(self._h, int(reps))

    def sync_status(self):
        return self._L.cldl_sync_status(self._h)

    def solve_dev(self, d_x_ptr, d_b_ptr):
        _check(self._L.cldl_solve_dev(self._h, C.c_void_p(d_x_ptr), C.c_void_p(d_b_ptr)), "solve_dev")

    def refactor_dev(self):
        _check(self._L.cldl_refactor_dev(self._h), "refactor_dev")

    def set_values_dev(self, d_ptr):
        _check(self._L.cldl_set_values_dev(self._h, C.c_void_p(d_ptr)), "set_values_dev")

    def selected_inverse_dev(self, d_out_ptr):
        f = self._L.cldl_selected_inverse_dev
        f.argtypes = [C.c_void_p, C.c_void_p]
        f.restype = C.c_int
        _check(f(self._h, C.c_void_p(d_out_ptr)), "selected_inverse_dev")

    def adjoint_solve_dev(self, d_g_ptr, d_x_ptr, d_gb_ptr, d_gvals_ptr):
        """device pointers; d_x_ptr / d_gvals_ptr may be None (gb only)"""
        f = self._L.cldl_adjoint_solve_dev
        f.argtypes = [C.c_void_p] * 5
        f.restype = C.c_int
        _check(f(self._h, C.c_void_p(d_g_ptr), C.c_void_p(d_x_ptr), C.c_void_p(d_gb_ptr), C.c_void_p(d_gvals_ptr)),
               "adjoint_solve_dev")

    def stream_ptr(self):
        return self._L.cldl_stream(self._h)


_SYM_ARRAYS = ["perm", "parent", "colcount", "sn_first", "sn_rowptr", "sn_rows", "sn_parent",
               "sn_level", "child_ptr", "child_list", "rel", "panel_off", "upd_off", "asm_ptr",
               "asm_src", "asm_dst", "level_ptr", "level_tasks", "iperm"]


class SymbolicAnalysis:
    """Host-only ordering + supernodal analysis (no GPU needed)."""

    def __init__(self, n, colptr, rowval, *, perm=None, ordering=ORDER_BEST,
                 amd_dense_scale=1.5, max_panel=0, nd_leaf=0):
        L = lib()
        cp, rv = _u64(colptr), _u64(rowval)
        pm = _u64(perm) if perm is not None else None
        h = C.c_void_p()
        rc = L.csym_analyse(C.byref(h), int(n), _p(cp, C.c_uint64), _p(rv, C.c_uint64),
                            _p(pm, C.c_uint64) if pm is not None else None,
                            0 if perm is not None else ordering, amd_dense_scale, max_panel, nd_leaf)
        if rc:
            raise BackendError(f"csym_analyse failed: {rc}")
        try:
            names = ["n", "nsup", "nlevels", "nnzL", "nnzL_stored", "upd_total", "ordering_used", "nnzA"]
            for k, nm in enumerate(names):
                setattr(self, nm, int(L.csym_scalar(h, k)))
            self.L_alloc = int(L.csym_scalar(h, 10))
            self.flops = L.csym_flops(h, 0)
            self.flops_stored = L.csym_flops(h, 1)
            for k, nm in enumerate(_SYM_ARRAYS):
                ln = L.csym_array(h, k, None, 0)
                a = np.empty(max(ln, 1), dtype=np.int64)
                L.csym_array(h, k, _p(a, C.c_int64), ln)
                setattr(self, nm, a[:ln])
        finally:
            L.csym_free(h)


class _DevBuf:
    """f64 device buffer for the sharded driver: a torch CUDA tensor, or (emulated build of the test-suite, where
    device memory is host memory) a numpy array."""

    def __init__(self, n, device, host=None):
        n = max(int(n), 1)
        self._torch = None
        if os.environ.get("CLARABEL_EMU") == "1":
            self.a = np.zeros(n) if host is None else np.ascontiguousarray(host, dtype=np.float64).copy()
            self.ptr = self.a.ctypes.data
        else:
            import torch
            self._torch = torch
            dev = torch.device("cuda", int(device))
            self.a = torch.zeros(n, dtype=torch.float64, device=dev) if host is None else \
                torch.as_tensor(np.ascontiguousarray(host, dtype=np.float64), device=dev).clone()
            self.ptr = self.a.data_ptr()
            # the fill / copy above runs on torch's stream, the library works on streams of its own that do not wait
            # for it: the buffer is handed out only when it is complete
            torch.cuda.synchronize(dev)

    def to(self, device):
        """copy on another device (same object when it already lives there / in the emulated build)"""
        if self._torch is None or self.a.device.index == int(device):
            return self
        out = _DevBuf.__new__(_DevBuf)
        out._torch = self._torch
        out.a = self.a.to(self._torch.device("cuda", int(device)))
        out.ptr = out.a.data_ptr()
        self._torch.cuda.synchronize(self.a.device)      # the peer copy is complete before a library stream reads it
        self._torch.cuda.synchronize(out.a.device)
        return out

    def numpy(self):
        return self.a.copy() if self._torch is None else self.a.cpu().numpy()


class ShardedLDLGroup:
    """ONE factorisation split over several ranks, all driven from this process (SURVEY 8e).

    Every rank is its own handle (`cldl_opts.shard_rank`), on its own GPU when `devices` names several, on the same
    GPU otherwise (which exercises exactly the same phases and exchanges -- the way the single-GPU test box checks the
    sharded path).  The exchanges between the phases are device-to-device copies here; with one process per GPU they
    are `torch.distributed` all-gathers of the same packed buffers (`ShardedLDLRank`).
    """

    def __init__(self, n, colptr, rowval, nzval, dsigns, nranks, devices=None, **kw):
        self.n, self.nranks = int(n), int(nranks)
        self.devices = list(devices) if devices is not None else [0] * self.nranks
        self.ranks = [CudaLDLSolver(n, colptr, rowval, nzval, dsigns, device=self.devices[r], shard_nranks=self.nranks,
                                    shard_rank=r, **kw) for r in range(self.nranks)]
        self._L = self.ranks[0]._L

    def _sync_streams(self):
        if os.environ.get("CLARABEL_EMU") != "1":
            import torch
            for d in set(self.devices):
                torch.cuda.synchronize(d)

    def _exchange(self, what, xs=None):
        L = self._L
        bufs = []
        for r, s in enumerate(self.ranks):
            cnt = int(L.cldl_shard_count(s._h, what, r))
            b = _DevBuf(cnt, self.devices[r])
            _check(L.cldl_shard_pack_dev(s._h, what, b.ptr, xs[r].ptr if xs else None), "shard_pack")
            bufs.append(b)
        self._sync_streams()
        for g, s in enumerate(self.ranks):
            for r in range(self.nranks):
                if r != g:
                    src = bufs[r].to(self.devices[g])
                    _check(L.cldl_shard_unpack_dev(s._h, what, r, src.ptr, xs[g].ptr if xs else None), "shard_unpack")
        self._sync_streams()

    def refactor(self):
        L = self._L
        for s in self.ranks:
            _check(L.cldl_shard_refactor_phase_dev(s._h, 0), "refactor phase 0")
        self._exchange(0)
        for s in self.ranks:
            _check(L.cldl_shard_refactor_phase_dev(s._h, 1), "refactor phase 1")
        ok = True
        for s in self.ranks:
            ok = bool(_check(L.cldl_sync_status(s._h), "sync_status")) and ok
        return ok

    def solve(self, b):
        L = self._L
        bs = [_DevBuf(self.n, d, host=b) for d in self.devices]
        xs = [_DevBuf(self.n, d) for d in self.devices]
        for s, x, bb in zip(self.ranks, xs, bs):
            _check(L.cldl_shard_solve_phase_dev(s._h, x.ptr, bb.ptr, 0), "solve phase 0")
        self._exchange(1)
        for s, x, bb in zip(self.ranks, xs, bs):
            _check(L.cldl_shard_solve_phase_dev(s._h, x.ptr, bb.ptr, 1), "solve phase 1")
        self._exchange(2, xs)
        return [x.numpy()[:self.n] for x in xs]

    def counts(self):
        """global (regularize_count, positive_inertia): owned parts of every rank + the top part once"""
        out = []
        for s in self.ranks:
            c = np.zeros(4, dtype=np.uint64)
            _check(self._L.cldl_shard_counts(s._h, _p(c, C.c_uint64)), "shard_counts")
            out.append(c.astype(np.int64))
        top = out[0][2:] - out[0][:2]
        tot = sum(c[:2] for c in out) + top
        return int(tot[0]), int(tot[1])

    def perm(self):
        return self.ranks[0].perm()

    def close(self):
        for s in self.ranks:
            s.close()


class TorchDistTransport:
    """The all-gather a sharded handle calls between its phases, over `torch.distributed` (NCCL on GPUs; gloo on host
    memory in the emulated build of the test-suite).  Keep the object alive as long as the handle uses it."""

    def __init__(self, device=0):
        import torch
        import torch.distributed as dist
        self._torch, self._dist, self.device = torch, dist, device
        self.world = dist.get_world_size()
        self.emu = os.environ.get("CLARABEL_EMU") == "1"
        self._send = self._recv = None
        self.calls = 0
        self.fn = ALLGATHER_FN(self._call)

    def _call(self, ctx, d_send, d_recv, count):
        try:
            torch, n = self._torch, int(count)
            self.calls += 1
            if self.emu:      # device memory is host memory: wrap the library's buffers directly
                send = torch.from_numpy(np.ctypeslib.as_array(C.cast(d_send, C.POINTER(C.c_double)), shape=(n,)))
                recv = torch.from_numpy(np.ctypeslib.as_array(C.cast(d_recv, C.POINTER(C.c_double)), shape=(n * self.world,)))
                self._dist.all_gather_into_tensor(recv, send)
                return 0
            if self._send is None or self._send.numel() < n:
                dev = torch.device("cuda", self.device)
                self._send = torch.empty(n + n // 4 + 64, dtype=torch.float64, device=dev)
                self._recv = torch.empty(self._send.numel() * self.world, dtype=torch.float64, device=dev)
            L = lib()
            L.cldl_copy_dev(self._send.data_ptr(), d_send, 8 * n)
            self._dist.all_gather_into_tensor(self._recv[:n * self.world], self._send[:n])
            torch.cuda.synchronize(self.device)
            L.cldl_copy_dev(d_recv, self._recv.data_ptr(), 8 * n * self.world)
            return 0
        except Exception as e:                     # never let an exception cross the C boundary
            import sys
            print("[clarabel_b200] transport failed:", repr(e), file=sys.stderr)
            return -1


def loaded_nccl_path():
    """Path of the libnccl this process has mapped (torch's bundled one once torch.distributed runs on NCCL), or None."""
    try:
        for line in open("/proc/self/maps"):
            if "libnccl" in line and ".so" in line:
                return line.split()[-1]
    except OSError:
        pass
    return None


def nccl_direct_setup(set_fn, handle, nranks, rank, device):
    """Give a sharded handle its own NCCL communicator (cldl_set_nccl / cipm_set_nccl), so that its all-gathers are
    stream-ordered calls issued by the library -- no Python callback, no host synchronisation per exchange.  Rank 0 draws
    the unique id, `torch.distributed` (already initialised by the launcher) broadcasts it.  Returns False (and leaves
    the handle to a callback transport) when the job does not run on NCCL or CB_SHARD_TRANSPORT=torch asks for the
    callback path."""
    import torch
    import torch.distributed as dist
    if os.environ.get("CB_SHARD_TRANSPORT", "nccl") == "torch" or os.environ.get("CLARABEL_EMU") == "1":
        return False
    if not (dist.is_available() and dist.is_initialized() and dist.get_backend() == "nccl"):
        return False
    L = lib()
    idt = torch.zeros(128, dtype=torch.uint8, device=torch.device("cuda", device))
    dist.all_reduce(idt)                              # makes sure NCCL itself is up (and its library mapped) on every rank
    path = loaded_nccl_path()
    pb = path.encode() if path else None
    idb = (C.c_ubyte * 128)()
    if rank == 0:
        L.cldl_nccl_unique_id.argtypes = [C.c_char_p, C.POINTER(C.c_ubyte)]
        _check(L.cldl_nccl_unique_id(pb, idb), "cldl_nccl_unique_id")
        idt = torch.tensor(list(idb), dtype=torch.uint8, device=torch.device("cuda", device))
    dist.broadcast(idt, src=0)
    torch.cuda.synchronize(device)
    idb = (C.c_ubyte * 128)(*[int(v) for v in idt.cpu().tolist()])
    set_fn.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_ubyte), C.c_int, C.c_int]
    _check(set_fn(handle, pb, idb, int(nranks), int(rank)), "set_nccl")
    return True


class ShardedLDLRank:
    """One rank of a sharded factorisation in a `torch.distributed` job (one process per GPU; NCCL over NVLink, or
    gloo on host buffers in the emulated build of the test-suite).  The exchanges between the phases are all-gathers of
    the packed contributions, padded to the largest one: update matrices of the cut roots per refactor, their update
    vectors per solve, and the solution entries every rank computed -- the all-gather of x the north star names."""

    def __init__(self, n, colptr, rowval, nzval, dsigns, device=0, **kw):
        import torch.distributed as dist
        self._dist = dist
        self.rank, self.nranks = dist.get_rank(), dist.get_world_size()
        self.n, self.device = int(n), device
        self.solver = CudaLDLSolver(n, colptr, rowval, nzval, dsigns, device=device, shard_nranks=self.nranks,
                                    shard_rank=self.rank, **kw)
        self._L = self.solver._L
        self._counts = [[int(self._L.cldl_shard_count(self.solver._h, w, r)) for r in range(self.nranks)] for w in range(3)]
        # on NCCL the library issues the all-gathers itself, stream-ordered (cldl_set_nccl); otherwise (gloo in the CPU
        # tests, CB_SHARD_TRANSPORT=torch) this class moves the packed buffers through torch.distributed
        self.nccl_direct = nccl_direct_setup(self._L.cldl_set_nccl, self.solver._h, self.nranks, self.rank, device)

    def _tensor(self, buf):
        import torch
        return buf.a if buf._torch is not None else torch.from_numpy(buf.a)

    def _exchange(self, what, x=None):
        import torch
        L, h = self._L, self.solver._h
        mx = max(max(self._counts[what]), 1)
        mine = _DevBuf(mx, self.device)
        _check(L.cldl_shard_pack_dev(h, what, mine.ptr, x.ptr if x is not None else None), "shard_pack")
        if mine._torch is not None:
            torch.cuda.synchronize(self.device)
        allb = _DevBuf(mx * self.nranks, self.device)
        self._dist.all_gather_into_tensor(self._tensor(allb), self._tensor(mine))
        if mine._torch is not None:
            torch.cuda.synchronize(self.device)      # the collective runs on NCCL's stream; the unpack kernels on the library's
        for r in range(self.nranks):
            if r != self.rank:
                _check(L.cldl_shard_unpack_dev(h, what, r, allb.ptr + 8 * mx * r, x.ptr if x is not None else None), "shard_unpack")
        if mine._torch is not None:
            torch.cuda.synchronize(self.device)

    def refactor(self):
        L, h = self._L, self.solver._h
        if self.nccl_direct:
            _check(L.cldl_refactor_dev(h), "refactor")
            return bool(_check(L.cldl_sync_status(h), "sync_status"))
        _check(L.cldl_shard_refactor_phase_dev(h, 0), "refactor phase 0")
        self._exchange(0)
        _check(L.cldl_shard_refactor_phase_dev(h, 1), "refactor phase 1")
        return bool(_check(L.cldl_sync_status(h), "sync_status"))

    def solve(self, b):
        L, h = self._L, self.solver._h
        bb, x = _DevBuf(self.n, self.device, host=b), _DevBuf(self.n, self.device)
        if self.nccl_direct:
            _check(L.cldl_solve_dev(h, x.ptr, bb.ptr), "solve")
            _check(L.cldl_sync_status(h), "sync_status")
            return x.numpy()[:self.n]
        _check(L.cldl_shard_solve_phase_dev(h, x.ptr, bb.ptr, 0), "solve phase 0")
        self._exchange(1)
        _check(L.cldl_shard_solve_phase_dev(h, x.ptr, bb.ptr, 1), "solve phase 1")
        self._exchange(2, x)
        return x.numpy()[:self.n]

    def close(self):
        self.solver.close()


def shard_plan(sym, nranks):
    """Subtree-to-rank mapping of one factorisation (SURVEY 8e; csrc/symbolic.h ShardPlan): owner[s] = rank that
    factors front s, -1 for the replicated top part; plus the flop split, what crosses ranks per refactor / solve and
    the modelled speed-up  total / (largest rank share + top)."""
    L = lib()
    nsup = int(sym.nsup)
    owner = np.empty(max(nsup, 1), dtype=np.int64)
    stats = np.zeros(8)
    f, rp, par = (np.ascontiguousarray(a, dtype=np.int64) for a in (sym.sn_first, sym.sn_rowptr, sym.sn_parent))
    rc = L.csym_shard_plan(nsup, _p(f, C.c_int64), _p(rp, C.c_int64), _p(par, C.c_int64), int(nranks),
                           _p(owner, C.c_int64), _p(stats, C.c_double))
    if rc:
        raise BackendError(f"csym_shard_plan failed: {rc}")
    keys = ["total_flops", "top_flops", "max_rank_flops", "min_rank_flops", "exchange_doubles", "exchange_vec",
            "top_levels", "model_speedup"]
    return dict(owner=owner[:nsup], **dict(zip(keys, stats.tolist())))


def order(n, colptr, rowval, kind=ORDER_AMD, dense_scale=1.5, nd_leaf=200):
    L = lib()
    cp, rv = _u64(colptr), _u64(rowval)
    out = np.empty(int(n), dtype=np.uint64)
    rc = L.csym_order(int(n), _p(cp, C.c_uint64), _p(rv, C.c_uint64), kind, dense_scale, nd_leaf,
                      _p(out, C.c_uint64))
    if rc:
        raise BackendError("ordering failed")
    return out.astype(np.int64)


def order_groups(N, colptr, rowval, cones, n, ordering=ORDER_BEST):
    """Host-only ordering of a KKT matrix whose cone list has dense Hs blocks (PSD cones, SOC cones kept dense): every
    block is one group of KKT vertices (rows n + offset .. of the cone), contracted for the ordering and eliminated
    first (csrc/symbolic.cpp order_with_groups -- what cipm_create does internally)."""
    L = lib()
    group = np.full(int(N), -1, dtype=np.int32)
    off, g = int(n), 0
    for kind, d in cones:
        rows = cone_nvars(kind, d)
        if kind == "psd":
            group[off:off + rows] = g
            g += 1
        off += rows
    cp, rv = _u64(colptr), _u64(rowval)
    out = np.empty(int(N), dtype=np.uint64)
    L.csym_order_groups.argtypes = [C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.c_int32, C.c_int, C.POINTER(C.c_uint64)]
    rc = L.csym_order_groups(int(N), _p(cp, C.c_uint64), _p(rv, C.c_uint64), group.ctypes.data_as(C.POINTER(C.c_int32)), g, ordering, _p(out, C.c_uint64))
    if rc < 0:
        raise BackendError("grouped ordering failed")
    return out.astype(np.int64)


# ===========================================================================
# Level 2: device-resident solver (cipm_* / ckkt_* / ccone_*)
# ===========================================================================
CONE_CODES = {"zero": 0, "nonneg": 1, "soc": 2, "psd": 3, "exp": 4, "pow": 5, "genpow": 6}
SCALING_PRIMAL_DUAL, SCALING_DUAL = 0, 1
STATUS_NAMES = ["Unsolved", "Solved", "PrimalInfeasible", "DualInfeasible", "AlmostSolved",
                "AlmostPrimalInfeasible", "AlmostDualInfeasible", "MaxIterations", "MaxTime",
                "NumericalError", "InsufficientProgress", "CallbackTerminated"]
# cipm_set_print_target kinds (print_to_stdout / _sink / _buffer / _file / _stream)
PRINT_STDOUT, PRINT_SINK, PRINT_BUFFER, PRINT_FILE, PRINT_STREAM = 0, 1, 2, 3, 4


class cipm_settings(C.Structure):
    """DefaultSettings fields read by the path (default/settings.rs:30-193)."""
    _fields_ = [
        ("max_iter", C.c_int32), ("time_limit", C.c_double), ("max_step_fraction", C.c_double),
        ("tol_gap_abs", C.c_double), ("tol_gap_rel", C.c_double), ("tol_feas", C.c_double),
        ("tol_infeas_abs", C.c_double), ("tol_infeas_rel", C.c_double), ("tol_ktratio", C.c_double),
        ("reduced_tol_gap_abs", C.c_double), ("reduced_tol_gap_rel", C.c_double),
        ("reduced_tol_feas", C.c_double), ("reduced_tol_infeas_abs", C.c_double),
        ("reduced_tol_infeas_rel", C.c_double), ("reduced_tol_ktratio", C.c_double),
        ("equilibrate_enable", C.c_int32), ("equilibrate_max_iter", C.c_int32),
        ("equilibrate_min_scaling", C.c_double), ("equilibrate_max_scaling", C.c_double),
        ("min_terminate_step_length", C.c_double),
        ("static_regularization_enable", C.c_int32),
        ("static_regularization_constant", C.c_double),
        ("static_regularization_proportional", C.c_double),
        ("dynamic_regularization_enable", C.c_int32),
        ("dynamic_regularization_eps", C.c_double), ("dynamic_regularization_delta", C.c_double),
        ("iterative_refinement_enable", C.c_int32),
        ("iterative_refinement_reltol", C.c_double), ("iterative_refinement_abstol", C.c_double),
        ("iterative_refinement_max_iter", C.c_int32),
        ("iterative_refinement_stop_ratio", C.c_double),
        ("linesearch_backtrack_step", C.c_double), ("min_switch_step_length", C.c_double),
        ("presolve_enable", C.c_int32),
        ("verbose", C.c_int32),
    ]


class cipm_info(C.Structure):
    _fields_ = [
        ("status", C.c_int32), ("iterations", C.c_uint32),
        ("cost_primal", C.c_double), ("cost_dual", C.c_double), ("res_primal", C.c_double),
        ("res_dual", C.c_double), ("res_primal_inf", C.c_double), ("res_dual_inf", C.c_double),
        ("gap_abs", C.c_double), ("gap_rel", C.c_double), ("ktratio", C.c_double), ("mu", C.c_double),
        ("step_length", C.c_double), ("sigma", C.c_double),
        ("solve_time", C.c_double), ("device_ms", C.c_double),
        ("t_kkt_update", C.c_double), ("t_kkt_solve", C.c_double), ("t_scale_cones", C.c_double),
        ("n_refactor", C.c_uint64), ("n_ldl_solve", C.c_uint64), ("n_ir_steps", C.c_uint64),
        ("regularize_count", C.c_uint64),
        ("nnzK", C.c_uint64), ("nnzL", C.c_uint64), ("kkt_dim", C.c_uint64),
    ]

    @property
    def status_name(self):
        return STATUS_NAMES[self.status]


# cipm_callback_fn: int (*)(const cipm_info* info, void* user_data); nonzero = stop
CALLBACK_FN = C.CFUNCTYPE(C.c_int, C.POINTER(cipm_info), C.c_void_p)
# cipm_write_fn: int (*)(void* ctx, const char* buf, uint64_t len)
WRITE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64)


EXPORTED_SYMBOLS += [
    "cipm_default_settings", "cipm_create", "cipm_destroy", "cipm_solve", "cipm_get_info",
    "cipm_get_solution", "cipm_trace", "cipm_iter_ms", "cipm_launch_count", "cipm_time_ms", "cipm_kkt_dim", "cipm_kkt_nnz", "cipm_get_kkt",
    "cipm_get_kkt_perm", "cipm_ldl_info", "cipm_update_data", "ckkt_update", "ckkt_setrhs", "ckkt_solve", "ckkt_update_P",
    "ckkt_update_A", "ckkt_get_values", "ccone_set_identity_scaling", "ccone_update_scaling",
    "ccone_Hs_len", "ccone_get_Hs", "ccone_mul_Hs", "ccone_affine_ds", "ccone_combined_ds_shift",
    "ccone_ds_from_dz_offset", "ccone_step_length", "ccone_margins", "ccone_scaled_unit_shift",
    "cipm_create_ex", "ccone_is_symmetric", "ccone_unit_initialization", "ccone_update_scaling_ex",
    "ccone_affine_ds_ex", "ccone_compute_barrier", "cipm_m_reduced", "cipm_get_equilibration", "cipm_get_infinity", "cipm_set_infinity", "cipm_default_infinity", "cipm_test_spmv", "cipm_test_vec", "cipm_create_gp",
    "cldl_shard_refactor_phase_dev", "cldl_shard_solve_phase_dev", "cldl_shard_count", "cldl_shard_pack_dev",
    "cldl_shard_unpack_dev", "cldl_shard_counts", "cipm_abi_sizes", "cldl_set_transport", "cipm_set_transport",
    "cldl_copy_dev", "cipm_update_settings", "cipm_set_termination_callback", "cipm_unset_termination_callback",
    "cipm_set_print_target", "cipm_get_print_buffer", "cipm_derivative", "cipm_adjoint_derivative",
]

_l2_ready = False


def _lib2():
    # (argtypes of the level-2 entry points; cipm_collective_count returns uint64)
    global _l2_ready
    L = lib()
    if _l2_ready:
        return L
    vp, u64p, f64p, i8p = C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_double), C.POINTER(C.c_int8)
    L.cipm_default_settings.argtypes = [C.POINTER(cipm_settings)]
    L.cipm_default_settings.restype = None
    L.cipm_create.argtypes = [C.POINTER(vp), C.c_uint64, C.c_uint64, u64p, u64p, f64p, f64p, u64p, u64p, f64p,
                              f64p, C.c_uint64, C.POINTER(C.c_int32), u64p, C.POINTER(cipm_settings),
                              C.POINTER(cldl_opts), u64p]
    L.cipm_create_ex.argtypes = [C.POINTER(vp), C.c_uint64, C.c_uint64, u64p, u64p, f64p, f64p, u64p, u64p, f64p,
                                 f64p, C.c_uint64, C.POINTER(C.c_int32), u64p, f64p, C.POINTER(cipm_settings),
                                 C.POINTER(cldl_opts), u64p]
    L.cipm_create_gp.argtypes = [C.POINTER(vp), C.c_uint64, C.c_uint64, u64p, u64p, f64p, f64p, u64p, u64p, f64p,
                                 f64p, C.c_uint64, C.POINTER(C.c_int32), u64p, f64p, u64p, f64p, C.POINTER(cipm_settings),
                                 C.POINTER(cldl_opts), u64p]
    L.ccone_is_symmetric.argtypes = [vp]
    L.ccone_unit_initialization.argtypes = [vp, f64p, f64p]
    L.ccone_update_scaling_ex.argtypes = [vp, f64p, f64p, C.c_double, C.c_int]
    L.ccone_affine_ds_ex.argtypes = [vp, f64p, f64p]
    L.ccone_compute_barrier.argtypes = [vp, f64p, f64p, f64p, f64p, C.c_double, f64p]
    L.cipm_set_transport.argtypes = [vp, ALLGATHER_FN, vp]
    L.cipm_update_settings.argtypes = [vp, C.POINTER(cipm_settings)]
    L.cipm_destroy.argtypes = [vp]
    L.cipm_destroy.restype = None
    L.cipm_solve.argtypes = [vp]
    L.cipm_get_info.argtypes = [vp, C.POINTER(cipm_info)]
    L.cipm_get_info.restype = None
    L.cipm_get_solution.argtypes = [vp, f64p, f64p, f64p]
    L.cipm_trace.argtypes = [vp, f64p, C.c_uint64]
    L.cipm_trace.restype = C.c_uint64
    L.cipm_iter_ms.argtypes = [vp, f64p, C.c_uint64]
    L.cipm_iter_ms.restype = C.c_uint64
    L.cipm_launch_count.argtypes = []
    L.cipm_launch_count.restype = C.c_uint64
    L.cipm_collective_count.argtypes = [C.c_void_p]
    L.cipm_collective_count.restype = C.c_uint64
    L.cipm_time_ms.argtypes = [vp, C.c_int, C.c_int]
    L.cipm_time_ms.restype = C.c_double
    for nm in ["cipm_kkt_dim", "cipm_kkt_nnz", "ccone_Hs_len", "cipm_m_reduced"]:
        getattr(L, nm).argtypes = [vp]
        getattr(L, nm).restype = C.c_uint64
    L.cipm_get_kkt.argtypes = [vp, u64p, u64p, f64p, i8p]
    L.cipm_get_equilibration.argtypes = [vp, f64p, f64p, C.POINTER(C.c_double)]
    L.cipm_get_equilibration.restype = C.c_int
    L.cipm_get_kkt_perm.argtypes = [vp, u64p]
    L.cipm_ldl_info.argtypes = [vp, C.POINTER(cldl_info_t)]
    L.cipm_ldl_info.restype = None
    L.ckkt_update.argtypes = [vp]
    L.ckkt_setrhs.argtypes = [vp, f64p, f64p]
    L.ckkt_solve.argtypes = [vp, f64p, f64p]
    L.cipm_update_data.argtypes = [vp, f64p, f64p, f64p, f64p]
    L.cipm_update_data.restype = C.c_int
    L.ckkt_update_P.argtypes = [vp, f64p]
    L.ckkt_update_A.argtypes = [vp, f64p]
    L.ckkt_get_values.argtypes = [vp, f64p]
    L.ccone_set_identity_scaling.argtypes = [vp]
    L.ccone_update_scaling.argtypes = [vp, f64p, f64p]
    L.ccone_get_Hs.argtypes = [vp, f64p]
    L.ccone_mul_Hs.argtypes = [vp, f64p, f64p]
    L.ccone_affine_ds.argtypes = [vp, f64p]
    L.ccone_combined_ds_shift.argtypes = [vp, f64p, f64p, f64p, C.c_double]
    L.ccone_ds_from_dz_offset.argtypes = [vp, f64p, f64p, f64p]
    L.ccone_step_length.argtypes = [vp, f64p, f64p, f64p, f64p, C.c_double, f64p]
    L.ccone_margins.argtypes = [vp, f64p, f64p, f64p]
    L.ccone_scaled_unit_shift.argtypes = [vp, f64p, C.c_double, C.c_int]
    L.cipm_set_termination_callback.argtypes = [vp, CALLBACK_FN, vp]
    L.cipm_unset_termination_callback.argtypes = [vp]
    L.cipm_set_print_target.argtypes = [vp, C.c_int, C.c_char_p, WRITE_FN, vp]
    L.cipm_get_print_buffer.argtypes = [vp, C.c_char_p, C.c_uint64]
    L.cipm_get_print_buffer.restype = C.c_int64
    L.cipm_derivative.argtypes = [vp, f64p, f64p, f64p, f64p, f64p, f64p, f64p]
    L.cipm_adjoint_derivative.argtypes = [vp, f64p, f64p, f64p, f64p, f64p, f64p, f64p]
    _l2_ready = True
    return L


def default_settings(**kw):
    s = cipm_settings()
    _lib2().cipm_default_settings(C.byref(s))
    for k, v in kw.items():
        setattr(s, k, v)
    return s


class CudaSolver:
    """Device interior-point solver: mirrors ``DefaultSolver::new(P,q,A,b,cones,settings)``
    and ``solve()`` (default/solver.rs:57-126, core/solver.rs:242-465).

    P: scipy sparse (symmetric or upper triangle; converted to triu like
    problemdata.rs:79-81); A: scipy sparse; cones: list of (kind, dim) with kind in
    {"zero", "nonneg", "soc", "psd"}, ("exp", 3) for an ExponentialConeT(),
    ("pow", alpha) for a PowerConeT(alpha) and ("genpow", (alphas, dim2)) for a
    GenPowerConeT(alphas, dim2).

    With ``shard=(nranks, rank)``, ranks other than 0 run with ``verbose`` off, so that one table is printed per
    solve; ``print_all_ranks=True`` leaves every rank's setting as given.
    """

    def __init__(self, P, q, A, b, cones, settings=None, *, ordering=ORDER_BEST, kkt_perm=None,
                 device=0, max_panel=0, nd_leaf=0, shard=None, transport=None, print_all_ranks=False):
        import scipy.sparse as sp
        L = _lib2()
        self._L = L
        self._callback = None        # ctypes objects the library holds pointers to: alive while installed
        self._print_fn = None
        self._pending_exc = None     # an exception raised inside a callback or a stream write, re-raised by solve()
        self._stamp = 0              # counts solves and data updates (autograd.py: the backward pass checks it)
        self._quiet_rank = shard is not None and int(shard[1]) != 0 and not print_all_ranks
        P, A = sp.csc_matrix(P), sp.csc_matrix(A)
        check_dimensions(P, q, A, b, cones)
        P = sp.triu(P, format="csc")
        P.sort_indices()
        A.sort_indices()
        self.n, self.m = P.shape[0], A.shape[0]
        self.settings = self._rank_settings(settings if settings is not None else default_settings())
        o = cldl_opts()
        L.cldl_default_opts(C.byref(o))
        o.ordering, o.device, o.max_panel, o.nd_leaf = ordering, device, max_panel, nd_leaf
        if shard is not None:      # (nranks, rank): this process is one rank of a factorisation split over several GPUs
            o.shard_nranks, o.shard_rank = int(shard[0]), int(shard[1])
        ct = np.ascontiguousarray([CONE_CODES[k] for k, _ in cones], dtype=np.int32)
        cd = _u64([3 if k in ("exp", "pow") else (len(d[0]) if k == "genpow" else d) for k, d in cones])
        cpar = _f64([float(d) if k == "pow" else 0.0 for k, d in cones])
        gdim2 = _u64([int(d[1]) if k == "genpow" else 0 for k, d in cones])
        galpha = _f64([a for k, d in cones if k == "genpow" for a in d[0]] or [0.0])
        Pp, Pi, Px = _u64(P.indptr), _u64(P.indices), _f64(P.data)
        Ap, Ai, Ax = _u64(A.indptr), _u64(A.indices), _f64(A.data)
        qq, bb = _f64(q), _f64(b)
        pm = _u64(kkt_perm) if kkt_perm is not None else None
        h = C.c_void_p()
        rc = L.cipm_create_gp(C.byref(h), self.n, self.m, _p(Pp, C.c_uint64), _p(Pi, C.c_uint64), _p(Px, C.c_double),
                              _p(qq, C.c_double), _p(Ap, C.c_uint64), _p(Ai, C.c_uint64), _p(Ax, C.c_double),
                              _p(bb, C.c_double), len(cones), ct.ctypes.data_as(C.POINTER(C.c_int32)),
                              _p(cd, C.c_uint64), _p(cpar, C.c_double), _p(gdim2, C.c_uint64), _p(galpha, C.c_double),
                              C.byref(self.settings), C.byref(o), _p(pm, C.c_uint64) if pm is not None else None)
        _check(rc, "cipm_create_gp")
        self._h = h
        # for the (index, values) update form.  P is this constructor's own upper-triangle copy, so its arrays are kept as
        # they are; q, b and A's values may alias the caller's arrays (which the caller is free to overwrite) and are copied
        self._cur = {"P": Px, "q": qq.copy(), "A": Ax.copy(), "b": bb.copy()}
        # sparsity patterns for the matrix form of update_data (index arrays only; no copies: a caller that rewrites the
        # index arrays of the matrix it passed in has a different matrix)
        self._pattern = {"P": (P.indptr, P.indices), "A": (A.indptr, A.indices)}
        self._shape = {"P": P.shape, "A": A.shape}
        self.N = int(L.cipm_kkt_dim(h))
        self.m_reduced = int(L.cipm_m_reduced(h))    # rows left after the inf-bound presolve
        if shard is not None:
            # every rank runs the same interior-point iterations on identical data; the factorisation and the
            # triangular solves are split and meet through this all-gather
            self.nccl_direct = transport is None and nccl_direct_setup(L.cipm_set_nccl, h, shard[0], shard[1], device)
            if not self.nccl_direct:
                self._transport = transport if transport is not None else TorchDistTransport(device)
                _check(L.cipm_set_transport(h, self._transport.fn, None), "cipm_set_transport")

    def test_spmv(self, which, y, x, a, b):
        """kernel-level check: which = 0  a P x + b y, 1  a A x + b y, 2  a A' x + b y on the handle's (equilibrated) data"""
        y, x = _f64(y).copy(), _f64(x)
        self._L.cipm_test_spmv.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double, C.c_double]
        _check(self._L.cipm_test_spmv(self._h, which, _p(y, C.c_double), _p(x, C.c_double), a, b), "cipm_test_spmv")
        return y

    def test_vec(self, what, x, v=None):
        """kernel-level check: what = 0  ||x||, 1  ||x||_inf, 2  ||x .* v||, 3  <x, v>"""
        x = _f64(x)
        v = _f64(v) if v is not None else x
        out = C.c_double(0.0)
        self._L.cipm_test_vec.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_uint64, C.POINTER(C.c_double)]
        xx, vv = (x if x.size else np.zeros(1)), (v if v.size else np.zeros(1))
        _check(self._L.cipm_test_vec(self._h, what, _p(xx, C.c_double), _p(vv, C.c_double), x.size, C.byref(out)), "cipm_test_vec")
        return out.value

    def equilibration(self):
        """(d, e, c) of DefaultProblemData::equilibration (problemdata.rs:229-312)"""
        d, e, c = np.zeros(max(self.n, 1)), np.zeros(max(self.m_reduced, 1)), C.c_double(0.0)
        _check(self._L.cipm_get_equilibration(self._h, _p(d, C.c_double), _p(e, C.c_double), C.byref(c)), "cipm_get_equilibration")
        return d[:self.n], e[:self.m_reduced], c.value

    def update_settings(self, **kw):
        """Solver::update_settings (core/solver.rs:207-211); construction-time fields may not change"""
        s = cipm_settings.from_buffer_copy(self.settings)
        for k, v in kw.items():
            setattr(s, k, v)
        s = self._rank_settings(s)
        _check(self._L.cipm_update_settings(self._h, C.byref(s)), "cipm_update_settings")
        self.settings = s

    def _rank_settings(self, s):
        if self._quiet_rank and s.verbose:
            s = cipm_settings.from_buffer_copy(s)
            s.verbose = 0
        return s

    # ---- termination callback (core/solver.rs: set_termination_callback / _c, unset_termination_callback) ----
    def set_termination_callback(self, fn):
        """`fn(info) -> bool` is called once per pass of the iteration loop with a copy of the current `cipm_info`;
        True ends the solve with status CallbackTerminated.  An exception raised by `fn` ends the solve too, and
        solve() raises it.  On a sharded solver every rank installs its own callback."""
        def call(pinfo, _user_data):
            try:
                return 1 if fn(cipm_info.from_buffer_copy(pinfo.contents)) else 0
            except BaseException as e:         # never let an exception cross the C boundary
                if self._pending_exc is None:
                    self._pending_exc = e
                return 1
        self.set_termination_callback_c(CALLBACK_FN(call))

    def set_termination_callback_c(self, cfn, user_data=None):
        """a C callback: a `CALLBACK_FN` (int (*)(const cipm_info*, void*)) and the pointer handed to it"""
        _check(self._L.cipm_set_termination_callback(self._h, cfn, user_data), "cipm_set_termination_callback")
        self._callback = (cfn, user_data)

    def unset_termination_callback(self):
        _check(self._L.cipm_unset_termination_callback(self._h), "cipm_unset_termination_callback")
        self._callback = None

    # ---- print targets (io/mod.rs: ConfigurablePrintTarget); output only appears with settings.verbose ----
    def _set_print(self, kind, path=None, fn=None):
        _check(self._L.cipm_set_print_target(self._h, kind, path, fn if fn is not None else WRITE_FN(), None),
               "cipm_set_print_target")
        self._print_fn = fn

    def print_to_stdout(self):
        self._set_print(PRINT_STDOUT)

    def print_to_file(self, path):
        """append the output to the file at `path`"""
        self._set_print(PRINT_FILE, path=os.fsencode(path))

    def print_to_stream(self, stream):
        """hand the output to `stream.write(str)`"""
        def write(_ctx, buf, n):
            try:
                stream.write(C.string_at(buf, n).decode("utf-8", "replace"))
                return 0
            except BaseException as e:
                if self._pending_exc is None:
                    self._pending_exc = e
                return -1
        self._set_print(PRINT_STREAM, fn=WRITE_FN(write))

    def print_to_sink(self):
        self._set_print(PRINT_SINK)

    def print_to_buffer(self):
        """collect the output in the solver (a fresh, empty buffer); read it with get_print_buffer()"""
        self._set_print(PRINT_BUFFER)

    def get_print_buffer(self):
        n = int(self._L.cipm_get_print_buffer(self._h, None, 0))
        if n < 0:
            raise BackendError("Print buffering is not configured.")
        buf = C.create_string_buffer(max(n, 1))
        self._L.cipm_get_print_buffer(self._h, buf, n)
        return buf.raw[:n].decode("utf-8", "replace")

    def is_data_update_allowed(self):
        """DefaultSolver::is_data_update_allowed (data_updating.rs:165-180): not while the presolver has removed rows"""
        return self.m_reduced == self.m

    def update_data(self, P=None, q=None, A=None, b=None):
        """DefaultSolver::update_data (data_updating.rs:68-163): new values on the same sparsity patterns; the
        symbolic analysis, the device plans and the equilibration scalings of the handle are reused.  Every argument
        takes the reference's three forms: a matrix / full vector, the vector of nonzero values, or a pair
        `(index, values)` that overwrites single entries (`zip(&index, &values)` there); `None` or an empty
        sequence leaves that part alone."""
        if not self.is_data_update_allowed():
            raise DataUpdateError("PresolveIsActive")
        new_values = self._new_values
        Pv, qv = new_values(P, self._cur["P"], True), new_values(q, self._cur["q"], False)
        Av, bv = new_values(A, self._cur["A"], False), new_values(b, self._cur["b"], False)
        f = lambda a: _p(a, C.c_double) if a is not None else None
        _check(self._L.cipm_update_data(self._h, f(Pv), f(qv), f(Av), f(bv)), "cipm_update_data")
        self._stamp += 1
        for k, v in (("P", Pv), ("q", qv), ("A", Av), ("b", bv)):
            if v is not None:
                self._cur[k] = v.copy()

    def _new_values(self, arg, current, triu):
        """the values update_data and the derivatives take: a matrix on the stored pattern (P: its upper triangle), a
        full vector, or a pair (index, values) that overwrites single entries of `current`; None or an empty sequence is
        None"""
        import scipy.sparse as sp
        if arg is None:
            return None
        if sp.issparse(arg):
            M = sp.csc_matrix(sp.triu(arg, format="csc") if triu else arg)
            M.sort_indices()
            # CscMatrix::is_equal_sparsity (algebra/csc/core.rs:436-445): same pattern, not just the same count
            ip, ix = self._pattern["P" if triu else "A"]
            if M.shape != self._shape["P" if triu else "A"] or not (np.array_equal(M.indptr, ip) and np.array_equal(M.indices, ix)):
                raise DataUpdateError("SparsityPattern")
            v = _f64(M.data)
        elif isinstance(arg, tuple) and len(arg) == 2 and not np.isscalar(arg[0]):
            idx, val = np.asarray(arg[0], dtype=np.int64), _f64(arg[1])
            if idx.size == 0:
                return None
            v = current.copy()
            v[idx] = val
        else:
            v = _f64(arg)
            if v.size == 0:
                return None
        if v.size != current.size:
            raise DataUpdateError("BadVectorDimension" if current.ndim == 1 else "BadFormat")
        return v

    # ---- derivatives of the solution at the last solve (cipm_derivative / cipm_adjoint_derivative) ----
    def _derivative_rc(self, rc, what):
        if rc == CLDL_E_ARG:
            if not self.is_data_update_allowed():
                raise BackendError(f"{what}: the presolve removed rows of this problem; derivatives are not available")
            raise BackendError(f"{what}: needs a solve that ended Solved or AlmostSolved, with no data update since")
        if rc == CLDL_E_NOT_FACTORED:
            raise BackendError(f"{what}: the cone scaling or the factorisation of the KKT matrix failed at the solution")
        _check(rc, what)

    def derivative(self, dP=None, dq=None, dA=None, db=None):
        """Forward derivative at the last solve: (dx, dz, ds) for the data perturbation (dP, dq, dA, db).  dP and dA
        take the forms of update_data (matrix on the stored pattern, value vector, or (index, values) pairs of a
        perturbation that is zero elsewhere); None = zero.  See include/clarabel_b200.h for the linear system solved."""
        zero = {k: np.zeros_like(v) for k, v in self._cur.items()}
        Pv, qv = self._new_values(dP, zero["P"], True), self._new_values(dq, zero["q"], False)
        Av, bv = self._new_values(dA, zero["A"], False), self._new_values(db, zero["b"], False)
        dx, dz, ds = np.zeros(max(self.n, 1)), np.zeros(max(self.m, 1)), np.zeros(max(self.m, 1))
        f = lambda a: _p(a, C.c_double) if a is not None else None
        self._derivative_rc(self._L.cipm_derivative(self._h, f(Pv), f(qv), f(Av), f(bv), f(dx), f(dz), f(ds)),
                            "derivative")
        return dx[:self.n], dz[:self.m], ds[:self.m]

    def adjoint_derivative(self, dx=None, dz=None, ds=None):
        """Adjoint derivative at the last solve: the gradients of <dx, x> + <dz, z> + <ds, s> w.r.t. the data, as
        dict(P=csc on P's stored upper triangle, q=..., A=csc on A's stored pattern, b=...).  None = zero."""
        import scipy.sparse as sp

        def vec(a, n):
            if a is None:
                return None
            v = _f64(a)
            if v.size != n:
                raise DataUpdateError("BadVectorDimension")
            return v
        gx, gz, gs = vec(dx, self.n), vec(dz, self.m), vec(ds, self.m)
        nP, nA = self._cur["P"].size, self._cur["A"].size
        gP, gq, gA, gb = np.zeros(max(nP, 1)), np.zeros(max(self.n, 1)), np.zeros(max(nA, 1)), np.zeros(max(self.m, 1))
        f = lambda a: _p(a, C.c_double) if a is not None else None
        self._derivative_rc(self._L.cipm_adjoint_derivative(self._h, f(gx), f(gz), f(gs), f(gP), f(gq), f(gA), f(gb)),
                            "adjoint_derivative")
        (Pp, Pi), (Ap, Ai) = self._pattern["P"], self._pattern["A"]
        return dict(P=sp.csc_matrix((gP[:nP], Pi.copy(), Pp.copy()), shape=self._shape["P"]), q=gq[:self.n],
                    A=sp.csc_matrix((gA[:nA], Ai.copy(), Ap.copy()), shape=self._shape["A"]), b=gb[:self.m])

    def close(self):
        if getattr(self, "_h", None):
            self._L.cipm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def solve(self):
        self._pending_exc = None
        self._stamp += 1
        rc = self._L.cipm_solve(self._h)
        exc, self._pending_exc = self._pending_exc, None
        if exc is not None:
            raise exc
        _check(rc, "cipm_solve")
        info = cipm_info()
        self._L.cipm_get_info(self._h, C.byref(info))
        x, z, s = np.zeros(max(self.n, 1)), np.zeros(max(self.m, 1)), np.zeros(max(self.m, 1))
        _check(self._L.cipm_get_solution(self._h, _p(x, C.c_double), _p(z, C.c_double), _p(s, C.c_double)),
               "cipm_get_solution")
        rows = int(self._L.cipm_trace(self._h, None, 0))
        tr = np.zeros((max(rows, 1), 6))
        self._L.cipm_trace(self._h, _p(tr.reshape(-1), C.c_double), rows)
        self.info, self.trace = info, tr[:rows]
        k = int(self._L.cipm_iter_ms(self._h, None, 0))
        it = np.zeros(max(k, 1))
        self._L.cipm_iter_ms(self._h, _p(it, C.c_double), k)
        self.iter_ms = it[:k]
        infeas = "Infeasible" in info.status_name
        return dict(status=info.status_name, iterations=int(info.iterations), x=x[:self.n], z=z[:self.m],
                    s=s[:self.m], obj_val=float("nan") if infeas else info.cost_primal,
                    obj_val_dual=float("nan") if infeas else info.cost_dual, info=info)

    def time_ms(self, which, reps):
        """which: 'refactor' | 'ldl_solve' | 'kkt_solve' (device time, CUDA events)."""
        return self._L.cipm_time_ms(self._h, {'refactor': 0, 'ldl_solve': 1, 'kkt_solve': 2}[which], int(reps))

    def kkt(self):
        N, nnz = self.N, int(self._L.cipm_kkt_nnz(self._h))
        cp, rv = np.zeros(N + 1, np.uint64), np.zeros(max(nnz, 1), np.uint64)
        nz, ds = np.zeros(max(nnz, 1)), np.zeros(N, np.int8)
        _check(self._L.cipm_get_kkt(self._h, _p(cp, C.c_uint64), _p(rv, C.c_uint64), _p(nz, C.c_double),
                                    _p(ds, C.c_int8)), "get_kkt")
        return N, cp.astype(np.int64), rv[:nnz].astype(np.int64), nz[:nnz], ds

    def kkt_perm(self):
        p = np.zeros(self.N, np.uint64)
        _check(self._L.cipm_get_kkt_perm(self._h, _p(p, C.c_uint64)), "get_kkt_perm")
        return p.astype(np.int64)

    def kkt_values(self):
        nz = np.zeros(max(int(self._L.cipm_kkt_nnz(self._h)), 1))
        _check(self._L.ckkt_get_values(self._h, _p(nz, C.c_double)), "kkt_values")
        return nz[:int(self._L.cipm_kkt_nnz(self._h))]

    def linear_solver_info(self):
        i = cldl_info_t()
        self._L.cipm_ldl_info(self._h, C.byref(i))
        return LinearSolverInfo(i.name.decode(), i.threads, bool(i.direct), i.nnzA, i.nnzL, i.nnzL_stored,
                                i.regularize_count, i.positive_inertia, i.n_supernodes, i.n_levels, i.flops,
                                i.ordering_used)

    # ---- KKTSolver trait ----
    def kkt_update(self):
        return bool(_check(self._L.ckkt_update(self._h), "ckkt_update"))

    def kkt_setrhs(self, rx, rz):
        rx, rz = _f64(rx), _f64(rz)
        _check(self._L.ckkt_setrhs(self._h, _p(rx, C.c_double), _p(rz, C.c_double)), "ckkt_setrhs")

    def kkt_solve(self):
        x, z = np.zeros(max(self.n, 1)), np.zeros(max(self.m, 1))
        ok = _check(self._L.ckkt_solve(self._h, _p(x, C.c_double), _p(z, C.c_double)), "ckkt_solve")
        return bool(ok), x[:self.n], z[:self.m]

    # ---- Cone trait ----
    def _m(self, a):
        a = _f64(a)
        assert a.size == self.m
        return a

    def cone_set_identity_scaling(self):
        _check(self._L.ccone_set_identity_scaling(self._h), "set_identity_scaling")

    def cone_update_scaling(self, s, z):
        s, z = self._m(s), self._m(z)
        return bool(_check(self._L.ccone_update_scaling(self._h, _p(s, C.c_double), _p(z, C.c_double)), "update_scaling"))

    def cone_is_symmetric(self):
        return bool(_check(self._L.ccone_is_symmetric(self._h), "is_symmetric"))

    def cone_unit_initialization(self):
        z, s = np.zeros(max(self.m, 1)), np.zeros(max(self.m, 1))
        _check(self._L.ccone_unit_initialization(self._h, _p(z, C.c_double), _p(s, C.c_double)), "unit_initialization")
        return z[:self.m], s[:self.m]

    def cone_update_scaling_ex(self, s, z, mu, strategy):
        s, z = self._m(s), self._m(z)
        return bool(_check(self._L.ccone_update_scaling_ex(self._h, _p(s, C.c_double), _p(z, C.c_double), float(mu),
                                                           int(strategy)), "update_scaling_ex"))

    def cone_affine_ds_ex(self, s):
        s = self._m(s)
        y = np.zeros(max(self.m, 1))
        _check(self._L.ccone_affine_ds_ex(self._h, _p(y, C.c_double), _p(s, C.c_double)), "affine_ds_ex")
        return y[:self.m]

    def cone_compute_barrier(self, z, s, dz, ds, alpha):
        a, b, c, d = self._m(z), self._m(s), self._m(dz), self._m(ds)
        out = C.c_double()
        _check(self._L.ccone_compute_barrier(self._h, _p(a, C.c_double), _p(b, C.c_double), _p(c, C.c_double),
                                             _p(d, C.c_double), float(alpha), C.byref(out)), "compute_barrier")
        return out.value

    def cone_get_Hs(self):
        ln = int(self._L.ccone_Hs_len(self._h))
        out = np.zeros(max(ln, 1))
        _check(self._L.ccone_get_Hs(self._h, _p(out, C.c_double)), "get_Hs")
        return out[:ln]

    def cone_mul_Hs(self, x):
        x = self._m(x)
        y = np.zeros(max(self.m, 1))
        _check(self._L.ccone_mul_Hs(self._h, _p(y, C.c_double), _p(x, C.c_double)), "mul_Hs")
        return y[:self.m]

    def cone_affine_ds(self):
        y = np.zeros(max(self.m, 1))
        _check(self._L.ccone_affine_ds(self._h, _p(y, C.c_double)), "affine_ds")
        return y[:self.m]

    def cone_combined_ds_shift(self, step_z, step_s, sigmamu):
        a, b = self._m(step_z), self._m(step_s)
        y = np.zeros(max(self.m, 1))
        _check(self._L.ccone_combined_ds_shift(self._h, _p(y, C.c_double), _p(a, C.c_double), _p(b, C.c_double),
                                               float(sigmamu)), "combined_ds_shift")
        return y[:self.m]

    def cone_ds_from_dz_offset(self, ds, z):
        a, b = self._m(ds), self._m(z)
        y = np.zeros(max(self.m, 1))
        _check(self._L.ccone_ds_from_dz_offset(self._h, _p(y, C.c_double), _p(a, C.c_double), _p(b, C.c_double)),
               "ds_from_dz_offset")
        return y[:self.m]

    def cone_step_length(self, dz, ds, z, s, amax=1.0):
        a, b, c, d = self._m(dz), self._m(ds), self._m(z), self._m(s)
        out = C.c_double()
        _check(self._L.ccone_step_length(self._h, _p(a, C.c_double), _p(b, C.c_double), _p(c, C.c_double),
                                         _p(d, C.c_double), float(amax), C.byref(out)), "step_length")
        return out.value

    def cone_margins(self, z):
        z = self._m(z)
        a, b = C.c_double(), C.c_double()
        _check(self._L.ccone_margins(self._h, _p(z, C.c_double), C.byref(a), C.byref(b)), "margins")
        return a.value, b.value

    def cone_scaled_unit_shift(self, z, alpha, primal):
        z = self._m(z).copy()
        _check(self._L.ccone_scaled_unit_shift(self._h, _p(z, C.c_double), float(alpha), 1 if primal else 0), "unit_shift")
        return z


def launch_count():
    return int(_lib2().cipm_launch_count())
