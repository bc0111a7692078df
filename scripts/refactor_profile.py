"""Per-kernel device time of one numeric refactor of a workload's KKT matrix (c2 | c4), with torch.profiler (CUDA
activities).  Two refactors warm up, then `reps` refactors are traced; every launch of one refactor is reported by its
position in the launch sequence (the level-0 size classes are separate launches of one kernel), averaged over the reps.
Usage: python scripts/refactor_profile.py c4 [reps] [trace_dir]"""
import collections
import json
import os
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import clarabel_rs_b200 as cb  # noqa: E402
from helpers import workloads  # noqa: E402

which = sys.argv[1] if len(sys.argv) > 1 else "c4"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
if which == "c2":
    pr = workloads.random_sparse_qp(n=100_000, m=200_000, nnz_per_row=5, seed=1, window=200)
    ordering = cb.ORDER_ND
else:
    pr = workloads.block_angular_qp(seed=3)
    ordering = cb.ORDER_BEST
N, cp, rv, nz, ds = workloads.kkt_triu(pr["P"], pr["A"], np.random.default_rng(0).uniform(0.5, 2, pr["A"].shape[0]))
s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=ordering)
for _ in range(2):
    assert s.refactor()
torch.cuda.synchronize()
l0 = cb.launch_count()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(reps):
        assert s.refactor()
    torch.cuda.synchronize()
launches = (cb.launch_count() - l0) / reps
kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith("Memcpy")
        and not e.name.startswith("Memset")]
kern.sort(key=lambda e: e.time_range.start)
per = len(kern) // reps
assert per * reps == len(kern), (len(kern), reps)
rows = collections.OrderedDict()
for r in range(reps):
    for i, e in enumerate(kern[r * per:(r + 1) * per]):
        rows.setdefault((i, e.name), []).append(e.time_range.elapsed_us())
total = 0.0
out = []
for (i, name), t in rows.items():
    short = name.split("(")[0]
    out.append({"pos": i, "kernel": short, "us": float(np.mean(t)), "us_min": float(np.min(t)), "us_max": float(np.max(t))})
    total += float(np.mean(t))
    print("%3d  %-40s %9.1f us  (min %.1f, max %.1f)" % (i, short, np.mean(t), np.min(t), np.max(t)))
print("kernels per refactor %d, launches counted %.0f, kernel time %.1f us" % (per, launches, total))
res = {"workload": which, "reps": reps, "kernels_per_refactor": per, "kernel_us": total, "launches": out,
       "device": torch.cuda.get_device_name(0)}
if len(sys.argv) > 3:
    os.makedirs(sys.argv[3], exist_ok=True)
    with open(os.path.join(sys.argv[3], "refactor_profile_%s.json" % which), "w") as fp:
        json.dump(res, fp, indent=1)
