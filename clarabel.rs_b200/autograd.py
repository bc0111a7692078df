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
"""
import numpy as np
import torch

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
