"""The device solver as a differentiable torch function.

    import clarabel_rs_b200                       # loads the package (as clarabel_rs_b200_pkg)
    from clarabel_rs_b200_pkg.autograd import solve

    x, z, s = solve(solver, P_values, q, A_values, b)

`solver` is a `CudaSolver` built once for the sparsity patterns of P (upper triangle) and A; the four inputs are float64
tensors of P's stored upper-triangle values, q, A's stored values (CSC order) and b.  The forward pass is
`update_data` + `solve` on those values; the backward pass is one `adjoint_derivative` at that solution (one cone
scaling update, one refactor and one refined KKT solve on the device, see include/clarabel_b200.h).  The outputs and
gradients are float64 tensors on the device of `q`.

A solve that does not end Solved or AlmostSolved raises.  The backward pass needs the handle to still hold the
solution of its forward pass: a later solve or data update on the same solver in between makes it raise.  torch is
imported by this module only.

The linear solve underneath, differentiable on its own (`SparseLDL`, one `CudaLDLSolver` on a fixed pattern):

    from clarabel_rs_b200_pkg.autograd import SparseLDL

    K = SparseLDL(n, colptr, rowval, dsigns)       # upper-triangular CSC pattern, diagonal included
    x = K.solve(values, b)                         # x = K^-1 b, differentiable in values and b
    sign, logabsdet = K.slogdet(values)            # differentiable in values
    X = K.sample(values, k, seed, mean=mu)         # k draws of N(mu, K^-1), differentiable in mu

`values` are the stored upper-triangle values (float64, the pattern's CSC order), b is (n,) or (n, k).  The backward
pass of `solve` is one adjoint solve on the forward pass's factor (gb = K^-1 g, and -(gb_i x_j + x_i gb_j) on the
pattern); that of `slogdet` is one selected inversion (Z = K^-1 on the pattern, 2 Z_ij off the diagonal, Z_ii on it).
The layer refactors only when it is handed values other than those of its current factor.
"""
import os

import numpy as np
import torch

from . import CudaLDLSolver, _check as _check_rc

_OK = ("Solved", "AlmostSolved")


def _np(t):
    return np.ascontiguousarray(t.detach().to("cpu", torch.float64).numpy())


class SolveFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, solver, P_values, q, A_values, b):
        solver.update_data(P=_np(P_values), q=_np(q), A=_np(A_values), b=_np(b))
        r = solver.solve()
        if r["status"] not in _OK:
            raise RuntimeError(f"solve ended {r['status']}: the solution map has no derivative there")
        ctx.solver, ctx.stamp = solver, solver._stamp
        ctx.devices = tuple(t.device for t in (P_values, q, A_values, b))
        dev = q.device
        return tuple(torch.from_numpy(np.array(v, dtype=np.float64)).to(dev) for v in (r["x"], r["z"], r["s"]))

    @staticmethod
    def backward(ctx, gx, gz, gs):
        solver = ctx.solver
        if solver._stamp != ctx.stamp:
            raise RuntimeError("the solver has solved again or taken new data since this forward pass")
        g = solver.adjoint_derivative(_np(gx), _np(gz), _np(gs))
        out = [torch.from_numpy(np.array(v, dtype=np.float64)).to(d)
               for v, d in zip((g["P"].data, g["q"], g["A"].data, g["b"]), ctx.devices)]
        return (None, *out)


def solve(solver, P_values, q, A_values, b):
    """(x, z, s) of the problem with the given data on `solver`'s patterns, differentiable in all four inputs"""
    return SolveFunction.apply(solver, P_values, q, A_values, b)


class SparseLDL:
    """x = K^-1 b and log|det K| for a sparse symmetric quasidefinite K on a fixed pattern, differentiable in K's stored
    values and in b, on the GPU's multifrontal LDL^T.

    n, colptr, rowval: K's upper triangle in CSC form, diagonal included; dsigns: the expected sign of every pivot
    (+1 / -1, as for `CudaLDLSolver`); perm: an optional fill-reducing permutation; device: the CUDA device.  The
    layer owns one `CudaLDLSolver` and refactors it only when it is handed values that differ (`torch.equal`) from
    those of its current factor, so `solve` then `slogdet` on the same values, or a forward pass and its backward pass,
    cost one refactor.  A backward pass whose forward values are no longer factored (another forward pass came in
    between) refactors from its own saved values.  `refactors` counts the refactors.

    A refactor whose verdict is 0 raises, and so does one that regularised a pivot (regularize_count > 0): the results
    would be those of K + E, and so would their derivatives.  Inputs are float64 tensors on the layer's device (CPU
    tensors under CLARABEL_EMU=1, where the emulated build's device memory is host memory)."""

    def __init__(self, n, colptr, rowval, dsigns, perm=None, device=0):
        self.n = int(n)
        cp = np.asarray(colptr, dtype=np.int64)
        rv = np.asarray(rowval, dtype=np.int64)
        self.nnz = int(rv.size)
        self.emu = os.environ.get("CLARABEL_EMU") == "1"
        self.device = torch.device("cpu") if self.emu else torch.device("cuda", int(device))
        self.solver = CudaLDLSolver(self.n, cp, rv, np.zeros(self.nnz), dsigns, perm=perm, device=int(device))
        col = np.repeat(np.arange(self.n), np.diff(cp))
        # d logabsdet / d v_ij = Z_ij + Z_ji = 2 Z_ij for a stored off-diagonal value (it stands for K_ij and K_ji)
        self._logdet_weight = torch.from_numpy(np.where(rv == col, 1.0, 2.0)).to(self.device)
        self._stream = None if self.emu else torch.cuda.ExternalStream(self.solver.stream_ptr(), device=self.device)
        self._values = None       # copy of the values of the handle's current factor (None: no valid factor)
        self.refactors = 0

    def close(self):
        self.solver.close()

    # The library works on the handle's own stream (cldl_stream), torch on its current stream.  Every call below makes
    # two hand-offs:
    #  (1) before the handle reads a tensor torch wrote (values, b, g, x) or writes one torch allocated (outputs), the
    #      handle's stream waits for torch's stream;
    #  (2) after the handle's last write, torch's stream waits for the handle's stream, so that whatever torch does
    #      next (read the outputs, free or reuse the inputs' memory) comes after the handle's work.
    def _handle_waits_for_torch(self):
        if not self.emu:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.device))
            self._stream.wait_event(ev)

    def _torch_waits_for_handle(self):
        if not self.emu:
            ev = torch.cuda.Event()
            ev.record(self._stream)
            torch.cuda.current_stream(self.device).wait_event(ev)

    def _check(self, t, shape, what):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float64 or t.device != self.device:
            raise TypeError(f"{what} must be a float64 tensor on {self.device}")
        if tuple(t.shape[:1]) != shape:
            raise ValueError(f"{what} has shape {tuple(t.shape)}, expected ({shape[0]}, ...)")
        return t.detach().contiguous()

    def _factor(self, values):
        """make the handle's factor the factor of `values`, refactoring only when they differ from the current one"""
        v = self._check(values, (self.nnz,), "values")
        if v.dim() != 1:
            raise ValueError(f"values must have shape ({self.nnz},)")
        if self._values is not None and torch.equal(v, self._values):
            return
        self._values = None
        self._handle_waits_for_torch()                   # (1) v is complete
        self.solver.set_values_dev(v.data_ptr())
        self.solver.refactor_dev()
        verdict = self.solver.sync_status()              # synchronises the handle's stream: v has been read
        self.refactors += 1
        _check_rc(verdict, "refactor")
        if verdict == 0:
            raise RuntimeError("refactor failed: a non-finite pivot")
        reg = self.solver.linear_solver_info().regularize_count
        if reg > 0:
            raise RuntimeError(f"refactor regularised {reg} pivot(s): K is not quasidefinite with the given dsigns, "
                               "and the results and their derivatives would be those of K + E, not of K")
        self._values = v.clone()

    def _solve_cols(self, B):
        """X = K^-1 B column by column on the current factor; B (k, n) contiguous, X (k, n)"""
        X = torch.empty_like(B)
        self._handle_waits_for_torch()                   # (1)
        for j in range(B.shape[0]):
            self.solver.solve_dev(X[j].data_ptr(), B[j].data_ptr())
        self._torch_waits_for_handle()                   # (2)
        return X

    def _adjoint_cols(self, G, X, with_values):
        """GB = K^-1 G column by column, and the pattern gradient summed over the columns (None without with_values)"""
        GB = torch.empty_like(G)
        GV = torch.empty((G.shape[0], self.nnz), dtype=torch.float64, device=self.device) if with_values else None
        self._handle_waits_for_torch()                   # (1)
        for j in range(G.shape[0]):
            self.solver.adjoint_solve_dev(G[j].data_ptr(), X[j].data_ptr(), GB[j].data_ptr(),
                                          GV[j].data_ptr() if with_values else None)
        self._torch_waits_for_handle()                   # (2)
        return GB, (GV.sum(0) if with_values else None)

    def _selected_inverse(self):
        Z = torch.empty(self.nnz, dtype=torch.float64, device=self.device)
        self._handle_waits_for_torch()                   # (1)
        self.solver.selected_inverse_dev(Z.data_ptr())
        self._torch_waits_for_handle()                   # (2)
        return Z

    def solve(self, values, b):
        """x = K^-1 b; b (n,) or (n, k), whose k columns are k solves.  Differentiable in values and b."""
        return _LDLSolve.apply(self, values, b)

    def slogdet(self, values):
        """(sign, logabsdet) of K, as float64 scalar tensors; logabsdet is differentiable in values."""
        return _LDLSlogdet.apply(self, values)

    def sample(self, values, k, seed, mean=None, form="precision", offset=0):
        """k Gaussian draws as an (n, k) tensor: x ~ N(mean, K^-1) (form "precision", K a sparse precision matrix) or
        N(mean, K) (form "covariance"), from the handle's sampler (CudaLDLSolver.sample: Philox4x64-10 with key
        (seed, 0), draw c at stream position offset + c).  K must be positive semidefinite.  Differentiable in mean
        only: a reparameterised gradient in values would need the adjoint of the factorisation itself, so values that
        require grad raise."""
        if isinstance(values, torch.Tensor) and values.requires_grad:
            raise RuntimeError("sample is not differentiable in values: pass values.detach()")
        self._factor(values)
        k = int(k)
        X = torch.empty((k, self.n), dtype=torch.float64, device=self.device)    # column-major n x k
        self._handle_waits_for_torch()                   # (1)
        self.solver.sample_dev(k, int(seed), int(offset), None, X.data_ptr(), None, form=form)
        self._torch_waits_for_handle()                   # (2)
        X = X.t()
        if mean is None:
            return X
        return self._check_mean(mean) + X

    def _check_mean(self, mean):
        if not isinstance(mean, torch.Tensor) or mean.dtype != torch.float64 or mean.device != self.device:
            raise TypeError(f"mean must be a float64 tensor on {self.device}")
        if tuple(mean.shape) != (self.n,):
            raise ValueError(f"mean has shape {tuple(mean.shape)}, expected ({self.n},)")
        return mean.reshape(self.n, 1)


class _LDLSolve(torch.autograd.Function):
    @staticmethod
    def forward(ctx, layer, values, b):
        layer._factor(values)
        bb = layer._check(b, (layer.n,), "b")
        if bb.dim() not in (1, 2):
            raise ValueError("b must be (n,) or (n, k)")
        X = layer._solve_cols(bb.reshape(layer.n, -1).t().contiguous())
        ctx.layer, ctx.bdim = layer, bb.dim()
        ctx.save_for_backward(values, X)
        return X[0].clone() if bb.dim() == 1 else X.t().contiguous()

    @staticmethod
    def backward(ctx, gx):
        layer = ctx.layer
        values, X = ctx.saved_tensors
        layer._factor(values)          # refactors only if another forward pass factored other values since
        G = (gx.reshape(layer.n, 1) if ctx.bdim == 1 else gx).t().contiguous()
        GB, gvals = layer._adjoint_cols(G, X, ctx.needs_input_grad[1])
        gb = GB[0].clone() if ctx.bdim == 1 else GB.t().contiguous()
        return None, gvals, gb


class _LDLSlogdet(torch.autograd.Function):
    @staticmethod
    def forward(ctx, layer, values):
        layer._factor(values)
        sign, logabsdet = layer.solver.slogdet()
        ctx.layer = layer
        ctx.save_for_backward(values)
        s = torch.tensor(float(sign), dtype=torch.float64, device=layer.device)
        ctx.mark_non_differentiable(s)
        return s, torch.tensor(logabsdet, dtype=torch.float64, device=layer.device)

    @staticmethod
    def backward(ctx, gsign, glogabsdet):
        layer = ctx.layer
        (values,) = ctx.saved_tensors
        layer._factor(values)
        return None, glogabsdet * layer._logdet_weight * layer._selected_inverse()
