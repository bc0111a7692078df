"""Per-call time of CudaSolver.derivative / adjoint_derivative on the full-size C2 and C4 workloads.

Each call is timed with CUDA events around the call (it returns once its results are on the host), so the time includes
the host work of the call.  The "device part" printed is an estimate: the call time minus the time of ONE device-to-host
copy, into pageable numpy memory, of as many doubles as the call returns (adjoint: nnzP + n + nnzA + m; forward:
n + 2m).  The library makes up to four separate copies instead, and the host-to-device uploads of the inputs stay in
the estimate.
Prints the card's name and power limit first; a number means something only next to them.

    python scripts/derivative_time.py [--reps 5] [--configs C2,C4]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import clarabel_rs_b200 as cb  # noqa: E402
from helpers import workloads  # noqa: E402

CONFIGS = {
    "C2": lambda: workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200),
    "C4": lambda: workloads.block_angular_qp(),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def timed(fn, reps):
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), float(np.min(ms))


def copy_ms(count, reps):
    src = torch.randn(max(count, 1), dtype=torch.float64, device="cuda")
    dst = np.empty(max(count, 1))
    t = torch.from_numpy(dst)
    return timed(lambda: t.copy_(src), reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--configs", default="C2,C4")
    a = ap.parse_args()
    print(f"card: {card()}")
    rng = np.random.default_rng(0)
    for name in a.configs.split(","):
        pr = CONFIGS[name]()
        t0 = time.time()
        dev = cb.CudaSolver(pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"])
        r = dev.solve()
        print(f"{name}: n={dev.n} m={dev.m} status={r['status']} setup+solve {time.time() - t0:.1f} s, "
              f"refactor {dev.time_ms('refactor', 3):.2f} ms, KKT solve {dev.time_ms('kkt_solve', 3):.2f} ms")
        nP, nA = len(dev._cur["P"]), len(dev._cur["A"])
        d = rng.standard_normal(nP), rng.standard_normal(dev.n), rng.standard_normal(nA), rng.standard_normal(dev.m)
        g = rng.standard_normal(dev.n), rng.standard_normal(dev.m), rng.standard_normal(dev.m)
        dev.derivative(*d)                      # first call: scratch and position maps
        fwd = timed(lambda: dev.derivative(*d), a.reps)
        adj = timed(lambda: dev.adjoint_derivative(*g), a.reps)
        cf = copy_ms(dev.n + 2 * dev.m, a.reps)
        ca = copy_ms(nP + dev.n + nA + dev.m, a.reps)
        print(f"{name}: derivative          {fwd[0]:8.2f} ms median ({fwd[1]:.2f} min); host copies {cf[0]:.2f} ms "
              f"-> device part estimate ~{fwd[0] - cf[0]:.2f} ms")
        print(f"{name}: adjoint_derivative  {adj[0]:8.2f} ms median ({adj[1]:.2f} min); host copies of "
              f"nnzP + n + nnzA + m = {nP + dev.n + nA + dev.m} doubles {ca[0]:.2f} ms -> device part estimate "
              f"~{adj[0] - ca[0]:.2f} ms")
        dev.close()


if __name__ == "__main__":
    main()
