#!/bin/bash
# Memory check of the product's kernels without a GPU: the emulated build (tests/emu) compiled with AddressSanitizer.
# Device buffers, shared-memory slots and dynamic shared memory are heap blocks there, so an out-of-bounds access of a
# kernel is reported like compute-sanitizer's memcheck would; -fsanitize=alignment stops at a vector-type access (int2, int4,
# double2) through a pointer the device would reject as misaligned.  Run from the repo root after `make`:  bash scripts/emu_asan.sh
set -e
mkdir -p /tmp/cb_asan
g++ -O1 -g -fsanitize=address,alignment -fno-sanitize-recover=alignment -fno-omit-frame-pointer -march=x86-64-v3 -ffp-contract=fast -std=c++17 -fPIC -shared -pthread \
  -Wno-unknown-pragmas -Itests/emu/include -Itests/emu/gen -Iinclude -Iclarabel.rs_b200/csrc -o /tmp/cb_asan/libclarabel_emu_asan.so \
  tests/emu/gen/cones.cpp tests/emu/gen/cones_psd.cpp tests/emu/gen/cones_nonsym.cpp tests/emu/gen/solver.cpp tests/emu/gen/ldl.cpp \
  tests/emu/cuda_emu.cpp clarabel.rs_b200/csrc/*.cpp
cat > /tmp/cb_asan/run.py <<'PY'
import sys, os, numpy as np
os.environ["CLARABEL_EMU"] = "1"
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import clarabel_rs_b200 as cb
cb.pkg._LIBPATH = "/tmp/cb_asan/libclarabel_emu_asan.so"
from helpers import small_kkt, workloads
import test_oracle_nonsym as ns
N, cp, rv, nz, ds = small_kkt(600, 1000, seed=1, window=30, k=3)
s = cb.CudaLDLSolver(N, cp, rv, nz, ds, ordering=cb.ORDER_ND, nd_leaf=40); assert s.refactor()
b = np.random.default_rng(0).standard_normal(N); x = s.solve(b); print("ldl ok", flush=True)
g = cb.ShardedLDLGroup(N, cp, rv, nz, ds, 3, ordering=cb.ORDER_ND, nd_leaf=40); assert g.refactor()
print("sharded ldl bitwise equal:", np.array_equal(g.solve(b)[0], x), flush=True)
for name, data in [("mixed", ns.mixed_conic_data()), ("genpow", ns.genpow_data()), ("exp", ns.expcone_data())]:
    r = cb.CudaSolver(*data).solve(); print(name, r["status"], r["iterations"], flush=True)
pr = workloads.portfolio_socp(n_assets=120, n_soc=6, soc_dim=9, block=30, seed=7)
print("socp", cb.CudaSolver(pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"]).solve()["status"], flush=True)
pr = workloads.block_sdp(n=60, n_psd=4, psd_dim=5, nnz_per_row=3, window=20, n_nonneg=10, seed=4)
print("sdp", cb.CudaSolver(pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"]).solve()["status"], flush=True)
ne = 40 * 41 // 2
import scipy.sparse as sp
print("psd40", cb.CudaSolver(sp.identity(ne, format="csc"), np.ones(ne), -sp.identity(ne, format="csc"), np.zeros(ne), [("psd", 40)]).solve()["status"], flush=True)
pr = workloads.random_sparse_qp(n=400, m=800, nnz_per_row=4, seed=2, window=30)
print("qp", cb.CudaSolver(pr["P"], pr["q"], pr["A"], pr["b"], pr["cones"], ordering=cb.ORDER_ND, nd_leaf=60).solve()["status"], flush=True)
PY
UBSAN_OPTIONS=print_stacktrace=1 ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0:halt_on_error=1 LD_PRELOAD=$(gcc -print-file-name=libasan.so) python /tmp/cb_asan/run.py
echo "asan run finished without a report"
