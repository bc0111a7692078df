// Device-resident KKT solver and interior-point driver (sm_90a) + ckkt_* /
// ccone_* / cipm_* C-ABI (include/clarabel_b200.h).
//
// The set-up on the host (input checks, presolve, equilibration, KKT assembly) is in problem_setup.{h,cpp}.
//
// What it replaces in the reference (all file:line under /root/reference/src):
//   KKTDevice::init        directldlkktsolver.rs:392-405
//   KKTDevice::update      directldlkktsolver.rs:134-158, 217-264, 324-329
//   KKTDevice::solve       directldlkktsolver.rs:168-189, 266-347 (iterative refinement)
//   k_csr_spmv             algebra/csc/matrix_math.rs:178-208, 261-343 (symv / gemv, as gathers)
//   IPM::*                 solver/core/solver.rs:242-465,525-665 and
//                          solver/implementations/default/{kktsystem,variables,residuals,info}.rs
//
// All vectors stay in HBM for the whole solve; the host only sees O(1) scalars
// per decision point (norms, dots, step lengths) through one pinned slot bank.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <new>
#include <vector>
#include <thread>

#include "../../include/clarabel_b200.h"
#include "cones.h"
#include "ipm_print.h"
#include "ldl_device.h"
#include "problem_setup.h"
#include "vec.cuh"

// the bound beyond which a constraint counts as absent (src/utils/infbounds.rs: INFINITY_DEFAULT = 1e20, process-wide,
// settable: get_infinity / set_infinity / default_infinity)
static std::atomic<double> g_infinity{1e20};

namespace cb {

#define SCK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { std::fprintf(stderr, "[clarabel_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return CLDL_E_CUDA; } } while (0)

static double wall() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// ---------------------------------------------------------------- sparse ops
struct CsrDev {
  int nrows = 0;
  const int* rowptr = nullptr;
  const int* col = nullptr;
  const double* val = nullptr;
};

// y = a*M*x + b*y, one thread per row (rows are short: ~5-30 entries)
__global__ void k_csr_spmv(CsrDev M, double* __restrict__ y, const double* __restrict__ x, double a, double b) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= M.nrows) return;
  double acc = 0.0;
  for (int p = M.rowptr[r]; p < M.rowptr[r + 1]; p++) acc += M.val[p] * x[M.col[p]];
  y[r] = (b == 0.0) ? a * acc : a * acc + b * y[r];
}
// e = b - K x with K's values gathered on the fly from csr_vals
__global__ void k_kkt_residual(CsrDev M, double* __restrict__ e, const double* __restrict__ b,
                               const double* __restrict__ x) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= M.nrows) return;
  double acc = 0.0;
  for (int p = M.rowptr[r]; p < M.rowptr[r + 1]; p++) acc += M.val[p] * x[M.col[p]];
  e[r] = b[r] - acc;
}
__global__ void k_gather(double* __restrict__ dst, const double* __restrict__ src, const int* __restrict__ idx, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}
__global__ void k_scatter(double* __restrict__ dst, const int* __restrict__ idx, const double* __restrict__ src, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[idx[i]] = src[i];
}
__global__ void k_diag_shift(double* __restrict__ vals, const int* __restrict__ didx, const double* __restrict__ diag,
                             const signed char* __restrict__ sg, const double* __restrict__ maxdiag,
                             double rconst, double rprop, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double eps = rconst + rprop * maxdiag[0];
  vals[didx[i]] = (sg[i] == 1) ? diag[i] + eps : diag[i] - eps;
}
// sparse SOC expansion values: columns -eta^2 u, -eta^2 v and the 2 extra diagonals
__global__ void k_sparse_soc_fill(ConeDev c, double* __restrict__ vals, const int* __restrict__ map_u,
                                  const int* __restrict__ map_v, const int* __restrict__ map_D) {
  const int id = c.soc_list[blockIdx.x];
  if (!c.sparse[id]) return;
  const int o = c.off[id], n = c.dim[id];
  const double e2 = c.eta[id] * c.eta[id];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    vals[map_u[o + i]] = c.u[o + i] * (-e2);
    vals[map_v[o + i]] = c.v[o + i] * (-e2);
  }
  if (threadIdx.x == 0) { vals[map_D[2 * id]] = -e2; vals[map_D[2 * id + 1]] = e2; }
}

// ------------------------------------------------------------- host helpers
static void dfree(const void* p) { if (p) cudaFree((void*)p); }

// scalar slots shared between device reductions and the host
enum Slot { S_NORMB = 0, S_NORME, S_MAXDIAG, S_QX, S_BZ, S_SZ, S_XPX, S_ALPHA, S_MARG0, S_MARG1,
            S_D0, S_D1, S_D2, S_D3, S_D4, S_D5, S_D6, S_D7, S_N0, S_N1, S_N2, S_N3, S_N4, S_N5, S_N6, S_N7,
            S_NORMB2, S_NORME2, S_BARR, S_BP0, S_BP1, S_BP2, S_BP3, S_BP4, S_SZSH, S_DMU, S_COUNT = 40 };

struct Scalars {
  double* d = nullptr;  // device [S_COUNT]
  double* h = nullptr;  // pinned host mirror
  cudaStream_t st = nullptr;
  int init(cudaStream_t s) {
    st = s;
    SCK(cudaMalloc((void**)&d, S_COUNT * sizeof(double)));
    SCK(cudaMemset(d, 0, S_COUNT * sizeof(double)));
    SCK(cudaMallocHost((void**)&h, S_COUNT * sizeof(double)));
    return 0;
  }
  void release() { if (d) cudaFree(d); if (h) cudaFreeHost(h); }
  int fetch() {
    SCK(cudaMemcpyAsync(h, d, S_COUNT * sizeof(double), cudaMemcpyDeviceToHost, st));
    SCK(cudaStreamSynchronize(st));
    return 0;
  }
};

// ----------------------------------------------------------- vector wrappers
struct Vec {
  cudaStream_t st;
  ReduceWS ws;
  void dot(const double* x, const double* y, int n, double* out) const {
    if (n == 0) { cudaMemsetAsync(out, 0, 8, st); return; }
    g_launches++;
    k_sum<<<red_grid(n), RED_THREADS, 0, st>>>(n, [=] __device__(int i) { return x[i] * y[i]; }, ws, out);
  }
  void norm_inf(const double* x, int n, double* out) const {
    cudaMemsetAsync(out, 0, 8, st);
    if (n == 0) return;
    g_launches++;
    k_max_nonneg<<<red_grid(n), RED_THREADS, 0, st>>>(n, [=] __device__(int i) { return x[i]; }, out);
  }
  // || x .* v ||_2 (norm_scaled, vecmath.rs:118-121), overflow-safe like the reference's stable_norm
  void norm_scaled(const double* x, const double* v, int n, double* out) const {
    if (n == 0) { cudaMemsetAsync(out, 0, 8, st); return; }
    g_launches++;
    k_norm2<<<red_grid(n), RED_THREADS, 0, st>>>(n, [=] __device__(int i) { return x[i] * v[i]; }, ws, out);
  }
  void norm(const double* x, int n, double* out) const {
    if (n == 0) { cudaMemsetAsync(out, 0, 8, st); return; }
    g_launches++;
    k_norm2<<<red_grid(n), RED_THREADS, 0, st>>>(n, [=] __device__(int i) { return x[i]; }, ws, out);
  }
  void axpby(double* y, double a, const double* x, double b, int n) const {  // y = a x + b y
    if (n == 0) return;
    g_launches++;
    k_map<<<(n + 255) / 256, 256, 0, st>>>(n, [=] __device__(int i) { y[i] = a * x[i] + b * y[i]; });
  }
  void waxpby(double* w, double a, const double* x, double b, const double* y, int n) const {
    if (n == 0) return;
    g_launches++;
    k_map<<<(n + 255) / 256, 256, 0, st>>>(n, [=] __device__(int i) { w[i] = a * x[i] + b * y[i]; });
  }
  void scale_copy(double* y, double a, const double* x, int n) const {  // y = a x
    if (n == 0) return;
    g_launches++;
    k_map<<<(n + 255) / 256, 256, 0, st>>>(n, [=] __device__(int i) { y[i] = a * x[i]; });
  }
  void copy(double* y, const double* x, int n) const {
    if (n) cudaMemcpyAsync(y, x, (size_t)n * 8, cudaMemcpyDeviceToDevice, st);
  }
  void zero(double* y, int n) const { if (n) cudaMemsetAsync(y, 0, (size_t)n * 8, st); }
};

// --------------------------------------------------------------- KKT solver
// the device half of a KKT assembly (the host copies stay for tests / get_kkt)
class KKTDevice : public KKTAssembly {
 public:
  int n = 0, m = 0, p = 0;
  cipm_settings set{};
  ConeSet* cones = nullptr;
  LDLObject ldl;
  cudaStream_t st = nullptr;
  Scalars* sc = nullptr;
  Vec V{};
  std::vector<double> Kx;   // host copy of the values: P and A, zeros elsewhere
  int *d_map_gqr = nullptr, *d_map_gp = nullptr, *d_map_gD = nullptr;
  // device
  int *d_map_P = nullptr, *d_map_A = nullptr, *d_map_Hs = nullptr, *d_map_u = nullptr, *d_map_v = nullptr,
      *d_map_D = nullptr, *d_map_diag = nullptr;
  signed char* d_dsigns = nullptr;
  int *d_srow = nullptr, *d_scol = nullptr, *d_sidx = nullptr;  // full symmetric CSR of K
  double* d_sval = nullptr;
  int64_t nnzS = 0;
  double *d_Hs = nullptr, *d_x = nullptr, *d_b = nullptr, *d_w1 = nullptr, *d_w2 = nullptr;
  double *d_x2 = nullptr, *d_b2 = nullptr, *d_w1b = nullptr, *d_w2b = nullptr;   // second right-hand side in flight
  int64_t n_refactor = 0, n_ldl_solve = 0, n_ir_steps = 0;

  int set_PA_values(const HostCsc& P, const HostCsc& A);
  int init(const HostCsc& P, const HostCsc& A, ConeSet* cs, const cipm_settings& s, const cldl_opts& lo,
           const int* perm, cudaStream_t stream_unused, Scalars* scal);
  void release();
  int update();                                      // -> 1 ok / 0 failed / <0 error
  void setrhs(const double* rx, const double* rz);
  void setrhs2(const double* rx, const double* rz);  // right-hand side of the second system of solve2
  int solve(double* lhsx, double* lhsz);             // -> 1 ok / 0 failed / <0 error
  // two systems with the same matrix at once (rhs from setrhs / setrhs2): the LDL sweeps of both run
  // concurrently on two streams, iterative refinement proceeds in lockstep with one host round trip per round
  int solve2(double* ax, double* az, double* bx, double* bz);
  void update_vals(const int* d_map, const double* d_src, int len);
  CsrDev symK() const { CsrDev M; M.nrows = N; M.rowptr = d_srow; M.col = d_scol; M.val = d_sval; return M; }
};

int KKTDevice::init(const HostCsc& P, const HostCsc& A, ConeSet* cs, const cipm_settings& s, const cldl_opts& lo,
                    const int* perm, cudaStream_t, Scalars* scal) {
  n = P.n; m = A.m; p = cs->p; cones = cs; set = s; sc = scal;
  int rc = assemble_kkt(P, A, *cones, *this);
  if (rc) return rc;
  Kx.assign(nnzK, 0.0);
  cb_tmark("kkt: assemble");
  cldl_opts o = lo;
  o.regularize_eps = s.dynamic_regularization_eps;
  o.regularize_delta = s.dynamic_regularization_delta;
  o.regularize_enable = 1;  // the reference adapter ignores dynamic_regularization_enable (ldlsolvers/qdldl.rs:38)
  // Dense cone blocks (PSD, dense SOC): contract every block to one vertex for the ordering, unless the caller fixed
  // the permutation.
  std::vector<int> perm_grp;
  if (!perm && ngroups > 0) {
    SymbolicOptions so;
    so.ordering = o.ordering ? o.ordering : ORDER_BEST;
    if (o.nd_leaf > 0) so.nd_leaf = o.nd_leaf;
    if (o.max_panel > 0) so.max_panel = o.max_panel > CB_PB_MAXNS ? CB_PB_MAXNS : o.max_panel;
    int kind = 0;
    rc = order_with_groups(N, Kp.data(), Ki.data(), group.data(), ngroups, so, perm_grp, &kind);
    if (rc) return CLDL_E_ARG;
    perm = perm_grp.data();
  }
  // full symmetric CSR of K with an index into the value array (used by iterative refinement): only needs the
  // assembled pattern, so it is built and uploaded on a host thread next to the ordering / symbolic analysis
  int rc_csr = 0;
  const int devid = lo.device;
  auto build_sym_csr = [&]() -> int {
    if (cudaSetDevice(devid) != cudaSuccess) return CLDL_E_CUDA;
    const CsrMap S = triu_to_sym_csr(N, Kp.data(), Ki.data());
    nnzS = S.rowptr[N];
    SCK(upload(&d_srow, S.rowptr)); SCK(upload(&d_scol, S.col)); SCK(upload(&d_sidx, S.src));
    SCK(cudaMalloc((void**)&d_sval, (size_t)(nnzS ? nnzS : 1) * 8));
    return 0;
  };
  std::thread th_csr([&]() { rc_csr = build_sym_csr(); });
  struct ThJoin { std::thread* t; ~ThJoin() { if (t->joinable()) t->join(); } } th_csr_guard{&th_csr};
  rc = ldl.init(N, Kp.data(), Ki.data(), Kx.data(), dsigns.data(), o, perm);
  if (rc) return rc;
  st = ldl.stream;
  V.st = st;
  V.ws = cones->ws;
  th_csr.join();
  if (rc_csr) return rc_csr;
  std::vector<signed char> ds8(dsigns.begin(), dsigns.end());
  SCK(upload(&d_map_P, map_P)); SCK(upload(&d_map_A, map_A)); SCK(upload(&d_map_Hs, map_Hs));
  SCK(upload(&d_map_u, map_u)); SCK(upload(&d_map_v, map_v)); SCK(upload(&d_map_D, map_D));
  SCK(upload(&d_map_diag, map_diag)); SCK(upload(&d_dsigns, ds8));
  SCK(upload(&d_map_gqr, map_gqr)); SCK(upload(&d_map_gp, map_gp)); SCK(upload(&d_map_gD, map_gD));
  SCK(cudaMalloc((void**)&d_Hs, (size_t)(cones->nHs ? cones->nHs : 1) * 8));
  SCK(cudaMalloc((void**)&d_x, (size_t)N * 8)); SCK(cudaMalloc((void**)&d_b, (size_t)N * 8));
  SCK(cudaMalloc((void**)&d_w1, (size_t)N * 8)); SCK(cudaMalloc((void**)&d_w2, (size_t)N * 8));
  SCK(cudaMalloc((void**)&d_x2, (size_t)N * 8)); SCK(cudaMalloc((void**)&d_b2, (size_t)N * 8));
  SCK(cudaMalloc((void**)&d_w1b, (size_t)N * 8)); SCK(cudaMalloc((void**)&d_w2b, (size_t)N * 8));
  SCK(cudaMemset(d_x, 0, (size_t)N * 8)); SCK(cudaMemset(d_b, 0, (size_t)N * 8));
  return 0;
}

int KKTDevice::set_PA_values(const HostCsc& P, const HostCsc& A) {
  for (size_t q = 0; q < map_P.size(); q++) Kx[map_P[q]] = P.nzval[q];
  for (size_t q = 0; q < map_A.size(); q++) Kx[map_A[q]] = A.nzval[q];
  SCK(cudaMemcpyAsync(ldl.dev.vals, Kx.data(), (size_t)nnzK * 8, cudaMemcpyHostToDevice, st));
  SCK(cudaStreamSynchronize(st));
  return 0;
}

void KKTDevice::release() {
  dfree(d_map_P); dfree(d_map_A); dfree(d_map_Hs); dfree(d_map_u); dfree(d_map_v); dfree(d_map_D); dfree(d_map_gqr); dfree(d_map_gp); dfree(d_map_gD);
  dfree(d_map_diag); dfree(d_dsigns); dfree(d_srow); dfree(d_scol); dfree(d_sidx); dfree(d_sval);
  dfree(d_Hs); dfree(d_x); dfree(d_b); dfree(d_w1); dfree(d_w2);
  dfree(d_x2); dfree(d_b2); dfree(d_w1b); dfree(d_w2b);
  ldl.release();
}

void KKTDevice::update_vals(const int* d_map, const double* d_src, int len) {
  if (len) { g_launches++; k_scatter<<<(len + 255) / 256, 256, 0, st>>>(ldl.dev.vals, d_map, d_src, len); }
}

int KKTDevice::update() {
  double* vals = ldl.dev.vals;
  // -W'W blocks straight into the KKT value array (get_Hs + negate + scatter)
  cones->get_Hs(d_Hs, true);
  update_vals(d_map_Hs, d_Hs, cones->nHs);
  const bool soc_exp = cones->p > 3 * (int)cones->gp_list.size();
  g_launches += (soc_exp ? 1 : 0) + (nnzS > 0) + (set.static_regularization_enable ? 3 : 0);
  if (soc_exp)
    k_sparse_soc_fill<<<cones->dev.nsoc, 128, 0, st>>>(cones->dev, vals, d_map_u, d_map_v, d_map_D);
  cones->gp_kkt_fill(vals, d_map_gqr, d_map_gp, d_map_gD);
  // refresh the symmetric-CSR values used by iterative refinement (un-regularised K)
  if (nnzS) k_gather<<<(unsigned)((nnzS + 255) / 256), 256, 0, st>>>(d_sval, vals, d_sidx, (int)nnzS);
  // static regularisation (directldlkktsolver.rs:217-264): keep the true diagonal in w1
  if (set.static_regularization_enable) {
    k_gather<<<(N + 255) / 256, 256, 0, st>>>(d_w1, vals, d_map_diag, N);
    V.norm_inf(d_w1, N, sc->d + S_MAXDIAG);
    k_diag_shift<<<(N + 255) / 256, 256, 0, st>>>(vals, d_map_diag, d_w1, d_dsigns, sc->d + S_MAXDIAG,
                                                   set.static_regularization_constant,
                                                   set.static_regularization_proportional, N);
  }
  int rc = ldl.refactor_async();
  n_refactor++;
  if (rc) return rc;
  if (set.static_regularization_enable) k_scatter<<<(N + 255) / 256, 256, 0, st>>>(vals, d_map_diag, d_w1, N);
  rc = ldl.sync_status();
  if (rc < 0) return rc;
  return rc;
}

void KKTDevice::setrhs(const double* rx, const double* rz) {
  V.copy(d_b, rx, n);
  V.copy(d_b + n, rz, m);
  V.zero(d_b + n + m, p);
}

int KKTDevice::solve(double* lhsx, double* lhsz) {
  int rc = ldl.solve_async(d_x, d_b);
  n_ldl_solve++;
  if (rc) return rc;
  double *x = d_x, *dx = d_w2, *e = d_w1;
  bool ok = true;
  const CsrDev K = symK();
  const unsigned grid = (N + 127) / 128;
  if (set.iterative_refinement_enable) {
    V.norm_inf(d_b, N, sc->d + S_NORMB);
    g_launches++;
    k_kkt_residual<<<grid, 128, 0, st>>>(K, e, d_b, x);
    V.norm_inf(e, N, sc->d + S_NORME);
    if ((rc = sc->fetch())) return rc;
    const double normb = sc->h[S_NORMB];
    double norme = sc->h[S_NORME];
    if (!std::isfinite(norme)) ok = false;
    for (int it = 0; ok && it < set.iterative_refinement_max_iter; it++) {
      if (norme <= set.iterative_refinement_abstol + set.iterative_refinement_reltol * normb) break;
      const double last = norme;
      if ((rc = ldl.solve_async(dx, e))) return rc;
      n_ldl_solve++; n_ir_steps++;
      V.axpby(dx, 1.0, x, 1.0, N);
      g_launches++;
      k_kkt_residual<<<grid, 128, 0, st>>>(K, e, d_b, dx);
      V.norm_inf(e, N, sc->d + S_NORME);
      if ((rc = sc->fetch())) return rc;
      norme = sc->h[S_NORME];
      if (!std::isfinite(norme)) { ok = false; break; }
      const double ratio = last / norme;
      if (ratio < set.iterative_refinement_stop_ratio) {
        if (ratio > 1.0) std::swap(x, dx);
        break;
      }
      std::swap(x, dx);
    }
    if (x != d_x) { d_w2 = d_x; d_x = x; }
  } else {
    V.norm_inf(d_x, N, sc->d + S_NORME);
    if ((rc = sc->fetch())) return rc;
    ok = std::isfinite(sc->h[S_NORME]);
  }
  if (!ok) return 0;
  if (lhsx) V.copy(lhsx, d_x, n);
  if (lhsz) V.copy(lhsz, d_x + n, m);
  return 1;
}

void KKTDevice::setrhs2(const double* rx, const double* rz) {
  V.copy(d_b2, rx, n);
  V.copy(d_b2 + n, rz, m);
  V.zero(d_b2 + n + m, p);
}

int KKTDevice::solve2(double* ax, double* az, double* bx, double* bz) {
  if (!set.iterative_refinement_enable || !ldl.use_dataflow) {   // plain path: one after the other
    int ok = solve(ax, az);
    if (ok != 1) return ok;
    std::swap(d_b, d_b2);
    ok = solve(bx, bz);
    std::swap(d_b, d_b2);
    return ok;
  }
  int rc;
  // per-system state: k = 0 uses (d_b, d_x, d_w1, d_w2), k = 1 the second set
  double* B[2] = {d_b, d_b2};
  double* X[2] = {d_x, d_x2};
  double* DX[2] = {d_w2, d_w2b};
  double* E[2] = {d_w1, d_w1b};
  const int SB[2] = {S_NORMB, S_NORMB2}, SE[2] = {S_NORME, S_NORME2};
  const CsrDev K = symK();
  const unsigned grid = (N + 127) / 128;
  // first solves, together
  if ((rc = ldl.solve_async(X[0], B[0], X[1], B[1]))) return rc;      // one sweep pair for both right-hand sides
  n_ldl_solve += 2;
  for (int k = 0; k < 2; k++) {
    V.norm_inf(B[k], N, sc->d + SB[k]);
    g_launches++;
    k_kkt_residual<<<grid, 128, 0, st>>>(K, E[k], B[k], X[k]);
    V.norm_inf(E[k], N, sc->d + SE[k]);
  }
  if ((rc = sc->fetch())) return rc;
  double normb[2] = {sc->h[SB[0]], sc->h[SB[1]]}, norme[2] = {sc->h[SE[0]], sc->h[SE[1]]};
  bool ok[2] = {true, true}, active[2] = {true, true};
  for (int k = 0; k < 2; k++) if (!std::isfinite(norme[k])) { ok[k] = false; active[k] = false; }
  for (int it = 0; it < set.iterative_refinement_max_iter; it++) {
    for (int k = 0; k < 2; k++)
      if (active[k] && norme[k] <= set.iterative_refinement_abstol + set.iterative_refinement_reltol * normb[k]) active[k] = false;
    if (!active[0] && !active[1]) break;
    const double last[2] = {norme[0], norme[1]};
    if (active[0] && active[1]) {
      if ((rc = ldl.solve_async(DX[0], E[0], DX[1], E[1]))) return rc;
    } else {
      const int k = active[0] ? 0 : 1;
      if ((rc = ldl.solve_async(DX[k], E[k]))) return rc;
    }
    for (int k = 0; k < 2; k++) {
      if (!active[k]) continue;
      n_ldl_solve++; n_ir_steps++;
      V.axpby(DX[k], 1.0, X[k], 1.0, N);
      g_launches++;
      k_kkt_residual<<<grid, 128, 0, st>>>(K, E[k], B[k], DX[k]);
      V.norm_inf(E[k], N, sc->d + SE[k]);
    }
    if ((rc = sc->fetch())) return rc;
    for (int k = 0; k < 2; k++) {
      if (!active[k]) continue;
      norme[k] = sc->h[SE[k]];
      if (!std::isfinite(norme[k])) { ok[k] = false; active[k] = false; continue; }
      const double ratio = last[k] / norme[k];
      if (ratio < set.iterative_refinement_stop_ratio) {
        if (ratio > 1.0) std::swap(X[k], DX[k]);
        active[k] = false;
        continue;
      }
      std::swap(X[k], DX[k]);
    }
  }
  // keep the buffer roles consistent for the next call (as in solve)
  if (X[0] != d_x) { d_w2 = d_x; d_x = X[0]; }
  if (X[1] != d_x2) { d_w2b = d_x2; d_x2 = X[1]; }
  if (!ok[0] || !ok[1]) return 0;
  if (ax) V.copy(ax, d_x, n);
  if (az) V.copy(az, d_x + n, m);
  if (bx) V.copy(bx, d_x2, n);
  if (bz) V.copy(bz, d_x2 + n, m);
  return 1;
}

// ------------------------------------------------------- solution derivatives
// Elementwise kernels of IPM::derivative / IPM::adjoint_derivative.  The solver holds P̂ = cDPD, Â = EAD and the iterate
// (x̂, ŝ, ẑ, τ); the derivative system K = [P A'; A -H] of the caller's coordinates is solved as K̂ [a; b] = [c D r1; E r2]
// with [dx; dz] = [D a; E b / c] (DESIGN.md, "Solution derivatives").  Every output element is written by one thread.

// the final iterate in the caller's coordinates, xo = D x̂ / τ and zo = E ẑ / (c τ) (the arithmetic of
// cipm_get_solution), and normalised for the cone scaling, sn = ŝ / τ and zn = ẑ / τ
__global__ void k_deriv_point(int n, int m, const double* __restrict__ x, const double* __restrict__ s,
                              const double* __restrict__ z, const double* __restrict__ d, const double* __restrict__ e,
                              double tauinv, double cinv, double* __restrict__ xo, double* __restrict__ zo,
                              double* __restrict__ sn, double* __restrict__ zn) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) xo[i] = x[i] * d[i] * tauinv;
  if (i < m) { zo[i] = z[i] * e[i] * (tauinv * cinv); sn[i] = s[i] * tauinv; zn[i] = z[i] * tauinv; }
}
// forward right-hand side [c D r1; E r2], r1 = -(dq + dP x + dA' z), r2 = db - dA x
__global__ void k_deriv_rhs(int n, int m, double c, const double* __restrict__ d, const double* __restrict__ e,
                            const double* __restrict__ dq, const double* __restrict__ dPx, const double* __restrict__ dAtz,
                            const double* __restrict__ db, const double* __restrict__ dAx, double* __restrict__ r1,
                            double* __restrict__ r2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) r1[i] = -c * d[i] * (dq[i] + dPx[i] + dAtz[i]);
  if (i < m) r2[i] = e[i] * (db[i] - dAx[i]);
}
// forward solution in the caller's coordinates: dx = D a, dz = E b / c, ds = E⁻¹ (E r2 - Â a) = r2 - A dx
__global__ void k_deriv_unscale(int n, int m, double cinv, const double* __restrict__ d, const double* __restrict__ e,
                                const double* __restrict__ einv, const double* __restrict__ a,
                                const double* __restrict__ b, const double* __restrict__ r2a, double* __restrict__ dx,
                                double* __restrict__ dz, double* __restrict__ ds) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dx[i] = d[i] * a[i];
  if (i < m) { dz[i] = e[i] * b[i] * cinv; ds[i] = einv[i] * r2a[i]; }
}
// adjoint right-hand side [c D (gx - A' gs); E gz] before its Â' product: r1 = c D gx, r2 = E gz, t = E⁻¹ gs, after
// which r1 -= c Â' t  (A' gs = D⁻¹ Â' E⁻¹ gs)
__global__ void k_adj_rhs(int n, int m, double c, const double* __restrict__ d, const double* __restrict__ e,
                          const double* __restrict__ einv, const double* __restrict__ gx, const double* __restrict__ gz,
                          const double* __restrict__ gs, double* __restrict__ r1, double* __restrict__ r2,
                          double* __restrict__ t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) r1[i] = c * d[i] * gx[i];
  if (i < m) { r2[i] = e[i] * gz[i]; t[i] = einv[i] * gs[i]; }
}
// adjoint solution in the caller's coordinates: u = D a, w = E b / c + gs; the gradients w.r.t. q and b are -u and w
__global__ void k_adj_unscale(int n, int m, double cinv, const double* __restrict__ d, const double* __restrict__ e,
                              const double* __restrict__ a, const double* __restrict__ b, const double* __restrict__ gs,
                              double* __restrict__ u, double* __restrict__ gq, double* __restrict__ w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { const double ui = d[i] * a[i]; u[i] = ui; gq[i] = -ui; }
  if (i < m) w[i] = e[i] * b[i] * cinv + gs[i];
}
// gradient on the stored pattern of A (CSC, the caller's order): -(z_i u_j + w_i x_j); one warp per column
__global__ void k_grad_A(int n, const int* __restrict__ colptr, const int* __restrict__ rowval,
                         const double* __restrict__ x, const double* __restrict__ u, const double* __restrict__ z,
                         const double* __restrict__ w, double* __restrict__ g) {
  const int j = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (j >= n) return;
  const double xj = x[j], uj = u[j];
  for (int p = colptr[j] + lane; p < colptr[j + 1]; p += 32) {
    const int i = rowval[p];
    g[p] = -(z[i] * uj + w[i] * xj);
  }
}

// ------------------------------------------------------------------ the IPM
enum { IST_UNSOLVED = 0, IST_SOLVED, IST_PINF, IST_DINF, IST_ALMOST_SOLVED, IST_ALMOST_PINF, IST_ALMOST_DINF,
       IST_MAXIT, IST_MAXTIME, IST_NUMERR, IST_INSUFF, IST_CALLBACK };

class IPM {
 public:
  int n = 0, m = 0;
  int mfull = 0;                 // rows of the caller's problem (m = rows left after the inf-bound presolve)
  double setup_time = 0.0;       // seconds spent in cipm_create: the reference's time limit runs on setup + solve
  double infbound = 1e20;        // the infinity bound at construction (presolver.rs:51,150): what reverse_presolve writes into s, whatever set_infinity did since
  std::vector<char> keep;        // presolve row mask over the caller's rows, empty = nothing dropped
  cipm_settings set{};
  HostCsc P, A;  // equilibrated copies (host)
  std::vector<double> q, b;
  Equilibration eq;
  double normq = 0, normb = 0;
  CsrMap hPsym, hAcsr;   // patterns of Psym and Acsr, and where their values sit in P's and A's CSC arrays
  ConeSet cones;
  KKTDevice kkt;
  Scalars sc;
  Vec V{};
  cudaStream_t st = nullptr;
  // device problem data
  CsrDev Psym, Acsr, Atcsr;
  int *dPr = nullptr, *dPc = nullptr, *dAr = nullptr, *dAc = nullptr, *dAtr = nullptr, *dAtc = nullptr;
  double *dPv = nullptr, *dAv = nullptr, *dAtv = nullptr;
  double *dq = nullptr, *db = nullptr, *dd = nullptr, *ddinv = nullptr, *de = nullptr, *deinv = nullptr;
  // iterate, steps, residuals (device)
  double *x = nullptr, *s = nullptr, *z = nullptr, *lx = nullptr, *ls = nullptr, *lz = nullptr;
  double *rhx = nullptr, *rhs_ = nullptr, *rhz = nullptr, *px = nullptr, *ps = nullptr, *pz = nullptr;
  double *rx = nullptr, *rz = nullptr, *rx_inf = nullptr, *rz_inf = nullptr, *Px = nullptr;
  double *x1 = nullptr, *z1 = nullptr, *x2 = nullptr, *z2 = nullptr, *workx = nullptr, *workz = nullptr,
         *work_conic = nullptr, *tmpn = nullptr;
  double tau = 1, kap = 1, ltau = 0, lkap = 0, rtau = 1, rhtau = 0, rhkap = 0, ptau = 1, pkap = 1;
  double dot_qx = 0, dot_bz = 0, dot_sz = 0, dot_xPx = 0, quad_x2 = 0, q_x2 = 0, b_z2 = 0;
  cipm_info info{};
  double prev_cost_primal = 0, prev_cost_dual = 0, prev_res_primal = 0, prev_res_dual = 0, prev_gap_abs = 0,
         prev_gap_rel = 0;
  std::vector<double> trace;
  std::vector<cudaEvent_t> iter_ev;   // one event at the start of every iteration
  std::vector<double> iter_ms;        // ms since the start of solve()
  int n_iter_ev = 0;
  // termination callback and verbose output (core/solver.rs:297-313, default/info_print.rs)
  cipm_callback_fn cb_fn = nullptr;
  void* cb_data = nullptr;
  double* d_verdict = nullptr;   // sharded: [this rank's verdict, every rank's verdict] on the device ...
  double* h_verdict = nullptr;   // ... and its pinned host mirror
  PrintTarget out;
  PrintSetup psetup;

  int init(int n_, int m_, const uint64_t* Pp, const uint64_t* Pi, const double* Pxv, const double* q_,
           const uint64_t* Ap, const uint64_t* Ai, const double* Axv, const double* b_, uint64_t ncones,
           const int32_t* ctype, const uint64_t* cdim, const cipm_settings& s, const cldl_opts& lo,
           const uint64_t* perm, const double* cparam = nullptr, const uint64_t* gp_dim2 = nullptr,
           const double* gp_alpha = nullptr);
  void release();
  int upload_problem();
  int solve();
  // pieces
  void spmv(const CsrDev& M, double* y, const double* xx, double a, double bb) {
    if (M.nrows) g_launches++;
    if (M.nrows) k_csr_spmv<<<(M.nrows + 127) / 128, 128, 0, st>>>(M, y, xx, a, bb);
  }
  int residuals_update();
  void info_update(double t0);
  void check_convergence(double tga, double tgr, double tf, double tia, double tir, double tkt, int s1, int s2, int s3);
  bool check_termination(int iter);
  int kkt_update(bool with_affine = false);
  int update_data(const double* Pnz, const double* qv, const double* Anz, const double* bv);
  bool affine_presolved = false;
  bool pair_solves = std::getenv("CB_NO_PAIRED_SOLVES") == nullptr;
  int kkt_solve_step(bool combined);
  int solve_initial_point();
  int shift_to_interior(double* v, bool primal);
  int step_length(bool combined, double* alpha, int scaling = SCALING_PRIMAL_DUAL);
  int variables_barrier(double a, double* out);
  int report_pass(bool verbose, bool* stop);
  // derivatives of the solution at the last solve (DESIGN.md, "Solution derivatives").  Valid after a solve that ended
  // Solved / AlmostSolved until the data changes.  The scratch below is allocated by the first call.
  bool deriv_valid = false;
  struct DerivWS {
    int *map_Psym = nullptr, *map_Acsr = nullptr;   // hPsym.src, hAcsr.src
    int *Pcp = nullptr, *Pri = nullptr;             // P's upper triangle as CSC (the caller's order)
    double* arena = nullptr;
    double *xo, *vn0, *vn1, *vn2, *rn, *an, *on0, *on1;                  // length n
    double *zo, *sn, *zn, *vm0, *vm1, *vm2, *rm, *bm, *om0, *om1;        // length m
    double *vP, *vPs, *vA, *vAc;                    // values on P's triu pattern, Psym, A's CSC and Acsr patterns
    int nnzPs = 0;                                  // entries of Psym
  } dw;
  int derivative(const double* dPnz, const double* dqv, const double* dAnz, const double* dbv, double* dx, double* dz,
                 double* ds);
  int adjoint_derivative(const double* gx, const double* gz, const double* gs, double* gP, double* gq, double* gA,
                         double* gb);
  int deriv_prepare();
  int deriv_factor();
  int deriv_solve();
};

int IPM::upload_problem() {
  // A as CSR (A x) and A' as CSR (== A in CSC) ; P as full symmetric CSR
  hAcsr = csc_to_csr(A);
  SCK(upload(&dAr, hAcsr.rowptr)); SCK(upload(&dAc, hAcsr.col)); SCK(upload(&dAv, gather(A.nzval, hAcsr.src)));
  Acsr.nrows = m; Acsr.rowptr = dAr; Acsr.col = dAc; Acsr.val = dAv;
  std::vector<int> cp32(A.colptr.begin(), A.colptr.end());
  SCK(upload(&dAtr, cp32)); SCK(upload(&dAtc, A.rowval)); SCK(upload(&dAtv, A.nzval));
  Atcsr.nrows = n; Atcsr.rowptr = dAtr; Atcsr.col = dAtc; Atcsr.val = dAtv;
  hPsym = triu_to_sym_csr(n, P.colptr.data(), P.rowval.data());
  SCK(upload(&dPr, hPsym.rowptr)); SCK(upload(&dPc, hPsym.col)); SCK(upload(&dPv, gather(P.nzval, hPsym.src)));
  Psym.nrows = n; Psym.rowptr = dPr; Psym.col = dPc; Psym.val = dPv;
  SCK(upload(&dq, q)); SCK(upload(&db, b)); SCK(upload(&dd, eq.d)); SCK(upload(&ddinv, eq.dinv));
  SCK(upload(&de, eq.e)); SCK(upload(&deinv, eq.einv));
  return 0;
}

// DefaultSolver::update_data (implementations/default/data_updating.rs:68-163): new values on the same sparsity
// patterns go through the STORED equilibration (P <- c D P D, A <- E A D, q <- c D q, b <- E b), the KKT values are
// overwritten through the assembly maps, symbolic analysis and plans are kept.  Null pointer = unchanged.
int IPM::update_data(const double* Pnz, const double* qv, const double* Anz, const double* bv) {
  if (!keep.empty()) return CLDL_E_ARG;   // data updates are refused on a presolved problem (data_updating.rs:165-180)
  SCK(cudaSetDevice(kkt.ldl.device));
  deriv_valid = false;                    // the last solve no longer belongs to this data
  if (Pnz) {
    eq.scale_P(P, Pnz);
    const std::vector<double> val = gather(P.nzval, hPsym.src);
    if (!val.empty()) SCK(cudaMemcpy((void*)dPv, val.data(), val.size() * 8, cudaMemcpyHostToDevice));
  }
  if (Anz) {
    eq.scale_A(A, Anz);
    const std::vector<double> vv = gather(A.nzval, hAcsr.src);
    if (!vv.empty()) {
      SCK(cudaMemcpy((void*)dAv, vv.data(), vv.size() * 8, cudaMemcpyHostToDevice));
      SCK(cudaMemcpy((void*)dAtv, A.nzval.data(), A.nzval.size() * 8, cudaMemcpyHostToDevice));
    }
  }
  if (Pnz || Anz) {
    int rc = kkt.set_PA_values(P, A);     // kktsystem.update_P / update_A -> KKT value array
    if (rc) return rc;
  }
  if (qv) {
    normq = eq.scale_q(q, qv);
    if (n) SCK(cudaMemcpy((void*)dq, q.data(), (size_t)n * 8, cudaMemcpyHostToDevice));
  }
  if (bv) {
    normb = eq.scale_b(b, bv);
    if (m) SCK(cudaMemcpy((void*)db, b.data(), (size_t)m * 8, cudaMemcpyHostToDevice));
  }
  SCK(cudaDeviceSynchronize());      // pageable-memory copies above: landed before anything on the solver's streams reads them
  return 0;
}

int IPM::init(int n_, int m_, const uint64_t* Pp, const uint64_t* Pi, const double* Pxv, const double* q_,
              const uint64_t* Ap, const uint64_t* Ai, const double* Axv, const double* b_, uint64_t ncones,
              const int32_t* ctype, const uint64_t* cdim, const cipm_settings& s_, const cldl_opts& lo,
              const uint64_t* perm, const double* cparam, const uint64_t* gp_dim2, const double* gp_alpha) {
  n = n_; m = m_; set = s_;
  // checked before a device is touched
  int rc = check_csc(Pp, Pi, (uint64_t)n, n, true);
  if (rc || (rc = check_csc(Ap, Ai, (uint64_t)m, n, false))) return rc;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    std::fprintf(stderr, "[clarabel_b200] no CUDA device: this backend has no CPU fallback\n");
    return CLDL_E_CUDA;
  }
  SCK(cudaSetDevice(lo.device));
  P = host_csc(n, n, Pp, Pi, Pxv);
  A = host_csc(m, n, Ap, Ai, Axv);
  q.assign(q_, q_ + n); b.assign(b_, b_ + m);
  std::vector<ConeSpec> cs;
  if ((rc = collapse_cones(ctype, cdim, ncones, cs, cparam, gp_dim2, gp_alpha))) return rc;
  cones.ns_amin = set.min_terminate_step_length; cones.ns_step = set.linesearch_backtrack_step;
  if (lo.shard_nranks > 1) pair_solves = false;   // a sharded factorisation runs its exchanges on one solve context
  infbound = g_infinity.load();
  mfull = m;
  if ((rc = presolve(cs, A, b, infbound, set.presolve_enable != 0, keep))) return rc;
  m = A.m;
  ConeLayout layout;
  if ((rc = cone_layout(cs, layout))) return rc;
  std::vector<int> kperm;
  if (perm) kperm = kkt_perm(perm, n, m, layout);
  normq = 0; for (double v : q) normq = std::max(normq, std::fabs(v));
  normb = 0; for (double v : b) normb = std::max(normb, std::fabs(v));
  // cone set needs a stream: borrow the LDL's once it exists -> create ours first
  SCK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  cb_tmark(nullptr);
  if ((rc = cones.init(layout, st))) return rc;
  cb_tmark("ipm: cone set init");
  // Ruiz equilibration only rescales values: it runs on a host thread next to the pattern work of the KKT
  // layer (assembly maps, ordering, symbolic analysis, plans); the values go in afterwards
  if ((rc = sc.init(st))) return rc;
  {
    // ... and so does the upload of the scaled problem data (CSR forms of A, A', P and the vectors), which only
    // needs the equilibrated values
    int rc_up = 0;
    const int devid = lo.device;
    std::thread th([this, &rc_up, devid]() {
      eq = equilibrate(P, A, q, b, cones, set);
      rc_up = cudaSetDevice(devid) == cudaSuccess ? upload_problem() : CLDL_E_CUDA;
    });
    // joined on every way out of this scope: an exception from kkt.init (std::bad_alloc of a host vector) with the
    // thread still joinable would end the process in std::terminate
    struct Join { std::thread& t; ~Join() { if (t.joinable()) t.join(); } } th_guard{th};
    rc = kkt.init(P, A, &cones, set, lo, perm ? kperm.data() : nullptr, st, &sc);
    th.join();
    if (rc || rc_up) { cudaStreamDestroy(st); st = nullptr; return rc ? rc : rc_up; }      // the temporary stream does not leak on the error paths
    if ((rc = kkt.set_PA_values(P, A))) { cudaStreamDestroy(st); st = nullptr; return rc; }
  }
  cb_tmark("ipm: equilibrate + upload problem || kkt init");
  // single stream for everything: adopt the LDL object's stream
  cudaStreamDestroy(st);
  st = kkt.st;
  cones.stream = st; sc.st = st; V.st = st; V.ws = cones.ws;
  cb_tmark("ipm: kkt init total");
  auto al = [&](double** pp, int len) { return cudaMalloc((void**)pp, (size_t)(len ? len : 1) * 8) == cudaSuccess && cudaMemset(*pp, 0, (size_t)(len ? len : 1) * 8) == cudaSuccess; };
  bool ok = al(&x, n) && al(&s, m) && al(&z, m) && al(&lx, n) && al(&ls, m) && al(&lz, m) && al(&rhx, n) &&
            al(&rhs_, m) && al(&rhz, m) && al(&px, n) && al(&ps, m) && al(&pz, m) && al(&rx, n) && al(&rz, m) &&
            al(&rx_inf, n) && al(&rz_inf, m) && al(&Px, n) && al(&x1, n) && al(&z1, m) && al(&x2, n) && al(&z2, m) &&
            al(&workx, n) && al(&workz, m) && al(&work_conic, m) && al(&tmpn, n);
  if (!ok) return CLDL_E_CUDA;
  std::memset(&info, 0, sizeof(info));
  info.nnzK = (uint64_t)kkt.nnzK;
  info.nnzL = (uint64_t)kkt.ldl.S.nnzL_simplicial;
  info.kkt_dim = (uint64_t)kkt.N;
  // what the verbose configuration block reports (info_print.rs: print_configuration / print_settings)
  psetup.n = n; psetup.m = m; psetup.nnzP = P.colptr[n]; psetup.nnzA = A.colptr[n];
  psetup.presolve_removed = mfull - m;
  psetup.cones.clear();
  for (const ConeSpec& c : cones.cones) psetup.cones.emplace_back(c.type, (int64_t)c.dim);
#ifdef CB_EMU   /* host build of the test suite (tests/emu): no device to name */
  psetup.device = "CUDA-on-CPU emulator";
#else
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, lo.device) == cudaSuccess) psetup.device = prop.name;
#endif
  return 0;
}

void IPM::release() {
  for (const void* p_ : {(const void*)dPr, (const void*)dPc, (const void*)dAr, (const void*)dAc, (const void*)dAtr,
                         (const void*)dAtc, (const void*)dPv, (const void*)dAv, (const void*)dAtv, (const void*)dq,
                         (const void*)db, (const void*)dd, (const void*)ddinv, (const void*)de, (const void*)deinv,
                         (const void*)x, (const void*)s, (const void*)z, (const void*)lx, (const void*)ls,
                         (const void*)lz, (const void*)rhx, (const void*)rhs_, (const void*)rhz, (const void*)px,
                         (const void*)ps, (const void*)pz, (const void*)rx, (const void*)rz, (const void*)rx_inf,
                         (const void*)rz_inf, (const void*)Px, (const void*)x1, (const void*)z1, (const void*)x2,
                         (const void*)z2, (const void*)workx, (const void*)workz, (const void*)work_conic,
                         (const void*)tmpn})
    dfree(p_);
  for (auto ev : iter_ev) cudaEventDestroy(ev);
  dfree(dw.map_Psym); dfree(dw.map_Acsr); dfree(dw.Pcp); dfree(dw.Pri); dfree(dw.arena);
  dfree(d_verdict);
  if (h_verdict) cudaFreeHost(h_verdict);
  cones.release();
  sc.release();
  kkt.release();
}

int IPM::residuals_update() {
  // residuals.rs:69-111
  V.dot(dq, x, n, sc.d + S_QX);
  V.dot(db, z, m, sc.d + S_BZ);
  V.dot(s, z, m, sc.d + S_SZ);
  spmv(Psym, Px, x, 1.0, 0.0);
  if (n == 0) V.zero(Px, n);
  V.dot(x, Px, n, sc.d + S_XPX);
  if (m) spmv(Atcsr, rx_inf, z, -1.0, 0.0); else V.zero(rx_inf, n);
  V.copy(rz_inf, s, m);
  spmv(Acsr, rz_inf, x, 1.0, 1.0);
  V.waxpby(rx, -1.0, Px, -tau, dq, n);
  V.axpby(rx, 1.0, rx_inf, 1.0, n);
  V.waxpby(rz, 1.0, rz_inf, -tau, db, m);
  // norms for info.update (info.rs:112-180): sums of squares, roots on the host
  V.norm_scaled(x, dd, n, sc.d + S_N0);
  V.norm_scaled(z, de, m, sc.d + S_N1);
  V.norm_scaled(s, deinv, m, sc.d + S_N2);
  V.norm_scaled(rx_inf, ddinv, n, sc.d + S_N3);
  V.norm_scaled(Px, ddinv, n, sc.d + S_N4);
  V.norm_scaled(rz_inf, deinv, m, sc.d + S_N5);
  V.norm_scaled(rz, deinv, m, sc.d + S_N6);
  V.norm_scaled(rx, ddinv, n, sc.d + S_N7);
  int rc = sc.fetch();
  if (rc) return rc;
  dot_qx = sc.h[S_QX]; dot_bz = sc.h[S_BZ]; dot_sz = sc.h[S_SZ]; dot_xPx = sc.h[S_XPX];
  rtau = dot_qx + dot_bz + kap + dot_xPx / tau;
  return 0;
}

void IPM::info_update(double t0) {
  const double tinv = 1.0 / tau, cinv = 1.0 / eq.c;
  const double xPx2 = dot_xPx * tinv * tinv / 2.0;
  info.cost_primal = (dot_qx * tinv + xPx2) * cinv;
  info.cost_dual = (-dot_bz * tinv - xPx2) * cinv;
  double normx = sc.h[S_N0], normz = sc.h[S_N1] * cinv, norms = sc.h[S_N2];
  info.res_primal_inf = (sc.h[S_N3] * cinv) / std::fmax(1.0, normz);
  info.res_dual_inf = std::fmax(sc.h[S_N4] / std::fmax(1.0, normx),
                                sc.h[S_N5] / std::fmax(1.0, normx + norms));
  normx *= tinv; normz *= tinv; norms *= tinv;
  info.res_primal = sc.h[S_N6] * tinv / std::fmax(1.0, normb + normx + norms);
  info.res_dual = sc.h[S_N7] * tinv * cinv / std::fmax(1.0, normq + normx + normz);
  info.gap_abs = std::fabs(info.cost_primal - info.cost_dual);
  info.gap_rel = info.gap_abs / std::fmax(1.0, std::fmin(std::fabs(info.cost_primal), std::fabs(info.cost_dual)));
  info.ktratio = kap * tinv;
  info.solve_time = wall() - t0;
}

void IPM::check_convergence(double tga, double tgr, double tf, double tia, double tir, double tkt, int s1, int s2, int s3) {
  const bool solved = ((info.gap_abs < tga) || (info.gap_rel < tgr)) && (info.res_primal < tf) && (info.res_dual < tf);
  if (info.ktratio <= 1.0 && solved) info.status = s1;
  else if (info.ktratio > (1.0 / tkt) * 1000.0) {
    if ((dot_bz < -tia) && (info.res_primal_inf < -tir * dot_bz)) info.status = s2;
    else if ((dot_qx < -tia) && (info.res_dual_inf < -tir * dot_qx)) info.status = s3;
  }
}

bool IPM::check_termination(int iter) {
  check_convergence(set.tol_gap_abs, set.tol_gap_rel, set.tol_feas, set.tol_infeas_abs, set.tol_infeas_rel,
                    set.tol_ktratio, IST_SOLVED, IST_PINF, IST_DINF);
  if (info.status == IST_UNSOLVED && iter > 1 &&
      (info.res_dual > prev_res_dual || info.res_primal > prev_res_primal)) {
    if (info.ktratio < 2.220446049250313e-16 * 100.0 &&
        (prev_gap_abs < set.tol_gap_abs || prev_gap_rel < set.tol_gap_rel))
      info.status = IST_INSUFF;
    if (info.ktratio < 1.0) {
      if ((info.res_dual > set.tol_feas * 100.0 && info.res_dual > prev_res_dual * 100.0) ||
          (info.res_primal > set.tol_feas * 100.0 && info.res_primal > prev_res_primal * 100.0))
        info.status = IST_INSUFF;
    }
  }
  if (info.status == IST_UNSOLVED) {
    if (set.max_iter == (int32_t)info.iterations) info.status = IST_MAXIT;
    else if (info.solve_time + setup_time > set.time_limit) info.status = IST_MAXTIME;   // timers.total_time() = setup + solve (solver.rs:447-452, info.rs:46-60)
  }
  return info.status != IST_UNSOLVED;
}

int IPM::kkt_update(bool with_affine) {
  // kktsystem.rs:108-125, 266-278.  with_affine: the affine step's system (kktsystem.rs:127-150) does not depend
  // on the constant-rhs solution, so both go through the factorisation together (KKTDevice::solve2); the
  // arithmetic per system is the one of two separate solves.
  const double t = wall();
  int ok = kkt.update();
  affine_presolved = false;
  if (ok == 1) {
    V.scale_copy(workx, -1.0, dq, n);
    kkt.setrhs(workx, db);
    if (with_affine) {
      V.copy(workx, rhx, n);
      V.copy(work_conic, s, m);
      V.waxpby(workz, 1.0, work_conic, -1.0, rhz, m);
      kkt.setrhs2(workx, workz);
      ok = kkt.solve2(x2, z2, x1, z1);
      affine_presolved = ok == 1;
    } else {
      ok = kkt.solve(x2, z2);
    }
    if (ok == 1) {
      // constants of the delta-tau formula that only depend on (x2, z2)
      spmv(Psym, tmpn, x2, 1.0, 0.0);
      if (n == 0) V.zero(tmpn, n);
      V.dot(x2, tmpn, n, sc.d + S_D0);
      V.dot(dq, x2, n, sc.d + S_D1);
      V.dot(db, z2, m, sc.d + S_D2);
      int rc = sc.fetch();
      if (rc) return rc;
      quad_x2 = sc.h[S_D0]; q_x2 = sc.h[S_D1]; b_z2 = sc.h[S_D2];
    }
  }
  info.t_kkt_update += wall() - t;
  return ok;
}

int IPM::kkt_solve_step(bool combined) {
  // kktsystem.rs:127-209
  const double t0 = wall();
  if (!combined && affine_presolved) {
    affine_presolved = false;      // (x1, z1) and work_conic = s were produced together with the constant-rhs solve
  } else {
    V.copy(workx, rhx, n);
    if (!combined) V.copy(work_conic, s, m);
    else cones.ds_from_dz_offset(work_conic, rhs_, z);
    V.waxpby(workz, 1.0, work_conic, -1.0, rhz, m);
    kkt.setrhs(workx, workz);
    int ok = kkt.solve(x1, z1);
    if (ok != 1) { info.t_kkt_solve += wall() - t0; return ok; }
  }
  // xi = x / tau ;  2 xi'P x1  and  (xi - x2)'P(xi - x2)
  double* xi = workx;
  V.scale_copy(xi, 1.0 / tau, x, n);
  spmv(Psym, tmpn, x1, 1.0, 0.0);
  if (n == 0) V.zero(tmpn, n);
  V.dot(xi, tmpn, n, sc.d + S_D3);
  V.dot(dq, x1, n, sc.d + S_D4);
  V.dot(db, z1, m, sc.d + S_D5);
  V.axpby(xi, -1.0, x2, 1.0, n);
  spmv(Psym, tmpn, xi, 1.0, 0.0);
  if (n == 0) V.zero(tmpn, n);
  V.dot(xi, tmpn, n, sc.d + S_D6);
  int rc = sc.fetch();
  if (rc) return rc;
  const double tau_num = rhtau - rhkap / tau + sc.h[S_D4] + sc.h[S_D5] + 2.0 * sc.h[S_D3];
  double tau_den = kap / tau - q_x2 - b_z2;
  tau_den += sc.h[S_D6] - quad_x2;
  ltau = tau_num / tau_den;
  V.waxpby(lx, 1.0, x1, ltau, x2, n);
  V.waxpby(lz, 1.0, z1, ltau, z2, m);
  cones.mul_Hs(ls, lz);
  V.axpby(ls, -1.0, work_conic, -1.0, m);
  lkap = -(rhkap + kap * ltau) / tau;
  info.t_kkt_solve += wall() - t0;
  return 1;
}

int IPM::solve_initial_point() {
  // kktsystem.rs:211-259
  int ok;
  if (P.colptr[n] == 0) {
    V.zero(workx, n);
    V.copy(workz, db, m);
    kkt.setrhs(workx, workz);
    ok = kkt.solve(x, s);
    V.axpby(s, 0.0, s, -1.0, m);
    if (ok != 1) return ok;
    V.scale_copy(workx, -1.0, dq, n);
    V.zero(workz, m);
    kkt.setrhs(workx, workz);
    ok = kkt.solve(nullptr, z);
  } else {
    V.scale_copy(workx, -1.0, dq, n);
    V.copy(workz, db, m);
    kkt.setrhs(workx, workz);
    ok = kkt.solve(x, z);
    V.scale_copy(s, -1.0, z, m);
  }
  return ok;
}

int IPM::shift_to_interior(double* v, bool primal) {
  // variables.rs:231-256
  cones.margins(v, sc.d + S_MARG0);
  int rc = sc.fetch();
  if (rc) return rc;
  const double minm = sc.h[S_MARG0], posm = sc.h[S_MARG1];
  double target = (posm * 0.1) / (double)cones.degree;
  if (!(target > 1.0)) target = 1.0;
  if (minm <= 0.0) { cones.scaled_unit_shift(v, -minm, primal); cones.scaled_unit_shift(v, target, primal); }
  else if (minm < target) cones.scaled_unit_shift(v, target - minm, primal);
  else cones.scaled_unit_shift(v, 0.0, primal);
  return 0;
}

int IPM::variables_barrier(double a, double* out) {
  // variables.rs:205-228
  const double central_coef = (double)(cones.degree + 1);
  const double cur_tau = tau + a * ltau, cur_kap = kap + a * lkap;
  const double *zz = z, *ss = s, *dz = lz, *ds = ls;
  if (m) {
    g_launches++;
    k_sum<<<red_grid(m), RED_THREADS, 0, st>>>(m, [=] __device__(int i) { return (ss[i] + a * ds[i]) * (zz[i] + a * dz[i]); },
                                              V.ws, sc.d + S_SZSH);
  } else SCK(cudaMemsetAsync(sc.d + S_SZSH, 0, 8, st));
  cones.compute_barrier(z, s, lz, ls, a, sc.d + S_BP0, sc.d + S_BARR);   // S_BP0..S_BP4: scratch
  int rc = sc.fetch();
  if (rc) return rc;
  auto lsafe = [](double v) { return v <= 0.0 ? -INFINITY : std::log(v); };
  const double mu_a = (sc.h[S_SZSH] + cur_tau * cur_kap) / central_coef;
  *out = central_coef * lsafe(mu_a) - lsafe(cur_tau) - lsafe(cur_kap) + sc.h[S_BARR];
  return 0;
}

int IPM::step_length(bool combined, double* alpha, int scaling) {
  // variables.rs:117-154, core/solver.rs:548-584
  const double at = ltau < 0.0 ? -tau / ltau : 1.7976931348623157e308;
  const double ak = lkap < 0.0 ? -kap / lkap : 1.7976931348623157e308;
  double a = std::fmin(std::fmin(at, ak), 1.0);
  if (m > 0) {
    SCK(cudaMemcpyAsync(sc.d + S_ALPHA, &a, 8, cudaMemcpyHostToDevice, st));
    cones.step_length(lz, ls, z, s, sc.d + S_ALPHA);
    int rc = sc.fetch();
    if (rc) return rc;
    a = sc.h[S_ALPHA];
  }
  if (combined) a *= set.max_step_fraction;
  if (!cones.all_symmetric && combined && scaling == SCALING_DUAL) {
    // backtrack_step_to_barrier (core/solver.rs:570-584)
    for (int it = 0; it < 50; it++) {
      double barrier = 0.0;
      int rc = variables_barrier(a, &barrier);
      if (rc) return rc;
      if (barrier < 1.0) break;
      a = set.linesearch_backtrack_step * a;
    }
  }
  *alpha = a;
  return 0;
}

int IPM::solve() {
  SCK(cudaSetDevice(kkt.ldl.device));
  int iter = 0, rc;
  double sigma = 1.0, alpha = 0.0, mu = 0.0;
  const double t0 = wall();
  info.status = IST_UNSOLVED; info.iterations = 0;
  deriv_valid = false;
  info.t_kkt_update = info.t_kkt_solve = info.t_scale_cones = 0;
  kkt.n_refactor = kkt.n_ldl_solve = kkt.n_ir_steps = 0;
  trace.clear();
  cudaEvent_t e0 = kkt.ldl.ev0, e1 = kkt.ldl.ev1;
  // printing and the termination callback only read host copies of the info: with both off a pass costs one branch
  const bool verbose = set.verbose != 0, hooks = verbose || cb_fn != nullptr;
  if (verbose) out.write(print_banner() + print_configuration(psetup, set) + print_header());
  SCK(cudaEventRecord(e0, st));

  // default start (core/solver.rs:525-541)
  if (cones.all_symmetric) {
    cones.set_identity_scaling();
    if ((rc = kkt_update()) < 0) return rc;
    if ((rc = solve_initial_point()) < 0) return rc;
    if ((rc = shift_to_interior(s, true))) return rc;
    if ((rc = shift_to_interior(z, false))) return rc;
  } else {
    cones.unit_initialization(z, s);      // variables.rs:173-179
    V.zero(x, n);
  }
  tau = 1.0; kap = 1.0;
  // core/solver.rs:277-280: dual-only scaling from the start when a cone (GenPow) has no primal-dual one
  int scaling = cones.allows_primal_dual ? SCALING_PRIMAL_DUAL : SCALING_DUAL;
  const bool nonsym = !cones.all_symmetric;

  n_iter_ev = 0;
  for (;;) {
    if (n_iter_ev < 1024) {
      if ((int)iter_ev.size() <= n_iter_ev) { cudaEvent_t ev; SCK(cudaEventCreate(&ev)); iter_ev.push_back(ev); }
      SCK(cudaEventRecord(iter_ev[n_iter_ev++], st));
    }
    if ((rc = residuals_update())) return rc;
    mu = (dot_sz + tau * kap) / (double)(cones.degree + 1);
    info.mu = mu; info.step_length = alpha; info.sigma = sigma; info.iterations = (uint32_t)iter;
    info_update(t0);
    trace.resize((size_t)(iter + 1) * 6);     // one row per iteration; a strategy switch re-enters the same row
    { double* tr = trace.data() + (size_t)iter * 6; tr[0] = mu; tr[1] = alpha; tr[2] = sigma; tr[3] = info.res_primal; tr[4] = info.res_dual; tr[5] = info.gap_abs; }
    if (hooks) {   // the row, then the user's termination check (core/solver.rs:297-313)
      bool stop = false;
      if ((rc = report_pass(verbose, &stop))) return rc;
      if (stop) { info.status = IST_CALLBACK; break; }
    }
    if (check_termination(iter)) {
      if (info.status == IST_INSUFF) {  // recover the previous iterate (core/solver.rs:586-611)
        info.cost_primal = prev_cost_primal; info.cost_dual = prev_cost_dual;
        info.res_primal = prev_res_primal; info.res_dual = prev_res_dual;
        info.gap_abs = prev_gap_abs; info.gap_rel = prev_gap_rel;
        V.copy(x, px, n); V.copy(s, ps, m); V.copy(z, pz, m); tau = ptau; kap = pkap;
        // nonsymmetric problems get a second chance with the dual-only scaling
        if (nonsym && scaling == SCALING_PRIMAL_DUAL) { info.status = IST_UNSOLVED; scaling = SCALING_DUAL; continue; }
      }
      break;
    }
    const double ts = wall();
    SCK(cudaMemsetAsync(cones.dev.fail, 0, sizeof(int), st));
    cones.update_scaling(s, z, mu, scaling);
    int failflag = 0;
    if (cones.dev.nsoc || cones.dev.npsd || cones.dev.ngp) {  // only SOC / PSD / GenPow scalings can fail
      SCK(cudaMemcpyAsync(&failflag, cones.dev.fail, sizeof(int), cudaMemcpyDeviceToHost, st));
      SCK(cudaStreamSynchronize(st));
    }
    info.t_scale_cones += wall() - ts;
    if (failflag) { info.status = IST_NUMERR; break; }
    iter += 1;
    // affine right-hand side (variables.rs:67-78)
    V.copy(rhx, rx, n);
    V.copy(rhz, rz, m);
    cones.affine_ds(rhs_, s);
    rhtau = rtau; rhkap = tau * kap;
    int ok = kkt_update(pair_solves);
    if (ok < 0) return ok;
    if (ok == 1) { ok = kkt_solve_step(false); if (ok < 0) return ok; }
    if (ok == 1) {
      if ((rc = step_length(false, &alpha, scaling))) return rc;
      sigma = (1.0 - alpha) * (1.0 - alpha) * (1.0 - alpha);
      const double mm = iter > 1 ? 1.0 : alpha;
      const double dsm = sigma * mu;
      // combined right-hand side (variables.rs:80-115)
      V.scale_copy(rhx, 1.0 - sigma, rx, n);
      rhtau = (1.0 - sigma) * rtau;
      rhkap = -dsm + mm * ltau * lkap + tau * kap;
      if (mm != 1.0) V.axpby(lz, 0.0, lz, mm, m);
      cones.combined_ds_shift(rhz, lz, ls, dsm);
      V.axpby(rhs_, 1.0, rhz, 1.0, m);
      V.scale_copy(rhz, 1.0 - sigma, rz, m);
      ok = kkt_solve_step(true);
      if (ok < 0) return ok;
    }
    // strategy checkpoints (core/solver.rs:613-651)
    if (ok != 1 && nonsym && scaling == SCALING_PRIMAL_DUAL) { alpha = 0.0; scaling = SCALING_DUAL; continue; }
    if (ok != 1) { info.status = IST_NUMERR; alpha = 0.0; break; }
    if ((rc = step_length(true, &alpha, scaling))) return rc;
    if (nonsym && scaling == SCALING_PRIMAL_DUAL && alpha < set.min_switch_step_length) { alpha = 0.0; scaling = SCALING_DUAL; continue; }
    if (alpha <= std::fmax(0.0, set.min_terminate_step_length)) { info.status = IST_INSUFF; alpha = 0.0; break; }
    prev_cost_primal = info.cost_primal; prev_cost_dual = info.cost_dual;
    prev_res_primal = info.res_primal; prev_res_dual = info.res_dual;
    prev_gap_abs = info.gap_abs; prev_gap_rel = info.gap_rel;
    V.copy(px, x, n); V.copy(ps, s, m); V.copy(pz, z, m); ptau = tau; pkap = kap;
    V.axpby(x, alpha, lx, 1.0, n);
    V.axpby(s, alpha, ls, 1.0, m);
    V.axpby(z, alpha, lz, 1.0, m);
    tau += alpha * ltau; kap += alpha * lkap;
  }
  if (alpha == 0.0) {   // no final step: the scalars are captured again, and printed once more (core/solver.rs:444-448)
    info.mu = mu; info.step_length = alpha; info.sigma = sigma; info.iterations = (uint32_t)iter;
    if (verbose) out.write(print_row(info));
  }
  if (info.status == IST_NUMERR || info.status == IST_INSUFF || info.status == IST_MAXIT || info.status == IST_MAXTIME)
    check_convergence(set.reduced_tol_gap_abs, set.reduced_tol_gap_rel, set.reduced_tol_feas,
                      set.reduced_tol_infeas_abs, set.reduced_tol_infeas_rel, set.reduced_tol_ktratio,
                      IST_ALMOST_SOLVED, IST_ALMOST_PINF, IST_ALMOST_DINF);
  SCK(cudaEventRecord(e1, st));
  SCK(cudaEventSynchronize(e1));
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  info.device_ms = ms;
  iter_ms.assign(n_iter_ev + 1, 0.0);
  for (int i = 0; i < n_iter_ev; i++) { float t = 0; cudaEventElapsedTime(&t, e0, iter_ev[i]); iter_ms[i] = t; }
  iter_ms[n_iter_ev] = ms;
  info.solve_time = wall() - t0;
  info.n_refactor = (uint64_t)kkt.n_refactor;
  info.n_ldl_solve = (uint64_t)kkt.n_ldl_solve;
  info.n_ir_steps = (uint64_t)kkt.n_ir_steps;
  info.regularize_count = kkt.ldl.regularize_count;
  deriv_valid = info.status == IST_SOLVED || info.status == IST_ALMOST_SOLVED;
  if (verbose) out.write(print_footer(info));
  return 0;
}

// ------------------------------------------------------- solution derivatives
// First derivative call: position maps from the caller's CSC orders to Psym / Acsr, P's triu pattern on the device and
// one scratch arena.  A handle that never differentiates allocates none of it.
int IPM::deriv_prepare() {
  if (dw.arena) return 0;
  // what an earlier call that failed half way uploaded is freed, not overwritten
  for (int** p : {&dw.map_Psym, &dw.map_Acsr, &dw.Pcp, &dw.Pri}) { dfree(*p); *p = nullptr; }
  std::vector<int> pcp(P.colptr.begin(), P.colptr.end());
  SCK(upload(&dw.map_Psym, hPsym.src)); SCK(upload(&dw.map_Acsr, hAcsr.src));
  SCK(upload(&dw.Pcp, pcp)); SCK(upload(&dw.Pri, P.rowval));
  const size_t nnzP = (size_t)P.colptr[n], nnzA = (size_t)A.colptr[n], nnzPs = hPsym.src.size();
  const size_t total = 8 * (size_t)n + 10 * (size_t)m + nnzP + nnzPs + 2 * nnzA;
  double* a = nullptr;
  SCK(cudaMalloc((void**)&a, total * 8));
  dw.arena = a;
  for (double** p : {&dw.xo, &dw.vn0, &dw.vn1, &dw.vn2, &dw.rn, &dw.an, &dw.on0, &dw.on1}) { *p = a; a += n; }
  for (double** p : {&dw.zo, &dw.sn, &dw.zn, &dw.vm0, &dw.vm1, &dw.vm2, &dw.rm, &dw.bm, &dw.om0, &dw.om1}) { *p = a; a += m; }
  dw.vP = a; a += nnzP;
  dw.vPs = a; a += nnzPs;
  dw.vA = a; a += nnzA;
  dw.vAc = a;
  dw.nnzPs = (int)nnzPs;
  return 0;
}

// Steps 1-3 of both derivative calls: the final iterate normalised by τ, the cone scaling H at it (NT scaling on the
// symmetric cones, μ∇²f*(z) with μ = <s, z> / ν on the others), the KKT values, static regularisation and refactor.
int IPM::deriv_factor() {
  if (!deriv_valid || !keep.empty()) return CLDL_E_ARG;
  SCK(cudaSetDevice(kkt.ldl.device));
  int rc = deriv_prepare();
  if (rc) return rc;
  g_launches++;
  k_deriv_point<<<(std::max(n, m) + 255) / 256, 256, 0, st>>>(n, m, x, s, z, dd, de, 1.0 / tau, 1.0 / eq.c, dw.xo, dw.zo,
                                                              dw.sn, dw.zn);
  double mu = 0.0;
  if (!cones.all_symmetric) {
    V.dot(dw.sn, dw.zn, m, sc.d + S_DMU);
    if ((rc = sc.fetch())) return rc;
    mu = sc.h[S_DMU] / (double)cones.degree;
  }
  SCK(cudaMemsetAsync(cones.dev.fail, 0, sizeof(int), st));
  cones.update_scaling(dw.sn, dw.zn, mu, SCALING_DUAL);
  if (cones.dev.nsoc || cones.dev.npsd || cones.dev.ngp) {
    int failflag = 0;
    SCK(cudaMemcpyAsync(&failflag, cones.dev.fail, sizeof(int), cudaMemcpyDeviceToHost, st));
    SCK(cudaStreamSynchronize(st));
    if (failflag) return CLDL_E_NOT_FACTORED;
  }
  rc = kkt.update();
  if (rc < 0) return rc;
  return rc == 1 ? 0 : CLDL_E_NOT_FACTORED;
}

// K̂ [an; bm] = [rn; rm], refined against the unregularised K̂
int IPM::deriv_solve() {
  kkt.setrhs(dw.rn, dw.rm);
  const int ok = kkt.solve(dw.an, dw.bm);
  if (ok < 0) return ok;
  return ok == 1 ? 0 : CLDL_E_NOT_FACTORED;
}

// host -> device on the solver's stream; NULL = zero
static int deriv_upload(double* dst, const double* src, size_t len, cudaStream_t st) {
  if (len == 0) return 0;
  if (src) SCK(cudaMemcpyAsync(dst, src, len * 8, cudaMemcpyHostToDevice, st));
  else SCK(cudaMemsetAsync(dst, 0, len * 8, st));
  return 0;
}
// device -> host on the solver's stream; NULL = not wanted
static int deriv_download(double* dst, const double* src, size_t len, cudaStream_t st) {
  if (dst && len) SCK(cudaMemcpyAsync(dst, src, len * 8, cudaMemcpyDeviceToHost, st));
  return 0;
}

int IPM::derivative(const double* dPnz, const double* dqv, const double* dAnz, const double* dbv, double* dxo,
                    double* dzo, double* dso) {
  int rc = deriv_factor();
  if (rc) return rc;
  const size_t nnzP = (size_t)P.colptr[n], nnzA = (size_t)A.colptr[n];
  const unsigned grid = (std::max(n, m) + 255) / 256;
  if ((rc = deriv_upload(dw.vn0, dqv, n, st)) || (rc = deriv_upload(dw.vm0, dbv, m, st))) return rc;
  // dP x: the caller's values gathered into Psym order, then Psym's product
  if (dPnz && dw.nnzPs) {
    if ((rc = deriv_upload(dw.vP, dPnz, nnzP, st))) return rc;
    g_launches++;
    k_gather<<<(dw.nnzPs + 255) / 256, 256, 0, st>>>(dw.vPs, dw.vP, dw.map_Psym, dw.nnzPs);
    CsrDev M = Psym;
    M.val = dw.vPs;
    spmv(M, dw.vn1, dw.xo, 1.0, 0.0);
  } else {
    V.zero(dw.vn1, n);
  }
  // dA' z on A's own CSC (Atcsr's pattern) and dA x through the values gathered into Acsr order
  if (dAnz && nnzA) {
    if ((rc = deriv_upload(dw.vA, dAnz, nnzA, st))) return rc;
    CsrDev Mt = Atcsr;
    Mt.val = dw.vA;
    spmv(Mt, dw.vn2, dw.zo, 1.0, 0.0);
    g_launches++;
    k_gather<<<(unsigned)((nnzA + 255) / 256), 256, 0, st>>>(dw.vAc, dw.vA, dw.map_Acsr, (int)nnzA);
    CsrDev M = Acsr;
    M.val = dw.vAc;
    spmv(M, dw.vm1, dw.xo, 1.0, 0.0);
  } else {
    V.zero(dw.vn2, n);
    V.zero(dw.vm1, m);
  }
  g_launches++;
  k_deriv_rhs<<<grid, 256, 0, st>>>(n, m, eq.c, dd, de, dw.vn0, dw.vn1, dw.vn2, dw.vm0, dw.vm1, dw.rn, dw.rm);
  if ((rc = deriv_solve())) return rc;
  spmv(Acsr, dw.rm, dw.an, -1.0, 1.0);     // E r2 - Â a
  g_launches++;
  k_deriv_unscale<<<grid, 256, 0, st>>>(n, m, 1.0 / eq.c, dd, de, deinv, dw.an, dw.bm, dw.rm, dw.on0, dw.om0, dw.om1);
  if ((rc = deriv_download(dxo, dw.on0, n, st)) || (rc = deriv_download(dzo, dw.om0, m, st)) ||
      (rc = deriv_download(dso, dw.om1, m, st)))
    return rc;
  SCK(cudaStreamSynchronize(st));
  return 0;
}

int IPM::adjoint_derivative(const double* gx, const double* gz, const double* gs, double* gPo, double* gqo,
                            double* gAo, double* gbo) {
  int rc = deriv_factor();
  if (rc) return rc;
  const size_t nnzP = (size_t)P.colptr[n], nnzA = (size_t)A.colptr[n];
  const unsigned grid = (std::max(n, m) + 255) / 256;
  if ((rc = deriv_upload(dw.vn0, gx, n, st)) || (rc = deriv_upload(dw.vm0, gz, m, st)) ||
      (rc = deriv_upload(dw.vm1, gs, m, st)))
    return rc;
  g_launches++;
  k_adj_rhs<<<grid, 256, 0, st>>>(n, m, eq.c, dd, de, deinv, dw.vn0, dw.vm0, dw.vm1, dw.rn, dw.rm, dw.vm2);
  if (m) spmv(Atcsr, dw.rn, dw.vm2, -eq.c, 1.0);
  if ((rc = deriv_solve())) return rc;
  g_launches++;
  k_adj_unscale<<<grid, 256, 0, st>>>(n, m, 1.0 / eq.c, dd, de, dw.an, dw.bm, dw.vm1, dw.on0, dw.on1, dw.om0);
  const unsigned wgrid = (unsigned)((n + 7) / 8);   // 8 warps of 256 threads: one column each
  if (nnzP) {
    g_launches++;
    k_grad_P<<<wgrid, 256, 0, st>>>(n, dw.Pcp, dw.Pri, dw.xo, dw.on0, dw.vP);
  }
  if (nnzA) {
    g_launches++;
    k_grad_A<<<wgrid, 256, 0, st>>>(n, dAtr, dAtc, dw.xo, dw.on0, dw.zo, dw.om0, dw.vA);
  }
  if ((rc = deriv_download(gPo, dw.vP, nnzP, st)) || (rc = deriv_download(gqo, dw.on1, n, st)) ||
      (rc = deriv_download(gAo, dw.vA, nnzA, st)) || (rc = deriv_download(gbo, dw.om0, m, st)))
    return rc;
  SCK(cudaStreamSynchronize(st));
  return 0;
}

// One pass's row and the termination callback.  On a sharded solver every rank runs the same passes: the verdicts of
// all ranks are all-gathered, and all stop when any asked to, so that no rank is left waiting in a collective.
int IPM::report_pass(bool verbose, bool* stop) {
  if (verbose) out.write(print_row(info));
  *stop = false;
  if (!cb_fn) return 0;
  const bool mine = cb_fn(&info, cb_data) != 0;
  LDLObject& L = kkt.ldl;
  if (!L.sharded() || !L.has_transport()) { *stop = mine; return 0; }
  const int R = L.shard_nranks;
  if (!d_verdict) {
    SCK(cudaMalloc((void**)&d_verdict, (size_t)(1 + R) * sizeof(double)));
    SCK(cudaMallocHost((void**)&h_verdict, (size_t)(1 + R) * sizeof(double)));
  }
  h_verdict[0] = mine ? 1.0 : 0.0;
  SCK(cudaMemcpyAsync(d_verdict, h_verdict, sizeof(double), cudaMemcpyHostToDevice, st));
  int rc = L.allgather(d_verdict, d_verdict + 1, 1);
  if (rc) return rc;
  SCK(cudaMemcpyAsync(h_verdict + 1, d_verdict + 1, (size_t)R * sizeof(double), cudaMemcpyDeviceToHost, st));
  SCK(cudaStreamSynchronize(st));
  for (int r = 0; r < R; r++) *stop = *stop || h_verdict[1 + r] != 0.0;
  return 0;
}

}  // namespace cb

// ===========================================================================
// C ABI
// ===========================================================================
using cb::IPM;

struct cipm_handle { IPM ipm; };

extern "C" {

void cipm_default_settings(cipm_settings* s) {
  s->max_iter = 200; s->time_limit = INFINITY; s->max_step_fraction = 0.99;
  s->tol_gap_abs = 1e-8; s->tol_gap_rel = 1e-8; s->tol_feas = 1e-8;
  s->tol_infeas_abs = 1e-8; s->tol_infeas_rel = 1e-8; s->tol_ktratio = 1e-6;
  s->reduced_tol_gap_abs = 5e-5; s->reduced_tol_gap_rel = 5e-5; s->reduced_tol_feas = 1e-4;
  s->reduced_tol_infeas_abs = 5e-12; s->reduced_tol_infeas_rel = 5e-5; s->reduced_tol_ktratio = 1e-4;
  s->equilibrate_enable = 1; s->equilibrate_max_iter = 10;
  s->equilibrate_min_scaling = 1e-4; s->equilibrate_max_scaling = 1e4;
  s->min_terminate_step_length = 1e-4;
  s->static_regularization_enable = 1; s->static_regularization_constant = 1e-8;
  s->static_regularization_proportional = 2.220446049250313e-16 * 2.220446049250313e-16;
  s->dynamic_regularization_enable = 1; s->dynamic_regularization_eps = 1e-13;
  s->dynamic_regularization_delta = 2e-7;
  s->iterative_refinement_enable = 1; s->iterative_refinement_reltol = 1e-13;
  s->iterative_refinement_abstol = 1e-12; s->iterative_refinement_max_iter = 10;
  s->iterative_refinement_stop_ratio = 5.0;
  s->linesearch_backtrack_step = 0.8; s->min_switch_step_length = 0.1;
  s->presolve_enable = 1;
  s->verbose = 0;   // the reference prints by default; a library call below other code stays silent unless asked
}

int cipm_create(cipm_t** out, uint64_t n, uint64_t m, const uint64_t* P_colptr, const uint64_t* P_rowval,
                const double* P_nzval, const double* q, const uint64_t* A_colptr, const uint64_t* A_rowval,
                const double* A_nzval, const double* b, uint64_t ncones, const int32_t* cone_types,
                const uint64_t* cone_dims, const cipm_settings* settings, const cldl_opts* ldl_opts,
                const uint64_t* kkt_perm_or_null) {
  return cipm_create_gp(out, n, m, P_colptr, P_rowval, P_nzval, q, A_colptr, A_rowval, A_nzval, b, ncones, cone_types,
                        cone_dims, nullptr, nullptr, nullptr, settings, ldl_opts, kkt_perm_or_null);
}

int cipm_create_ex(cipm_t** out, uint64_t n, uint64_t m, const uint64_t* P_colptr, const uint64_t* P_rowval,
                   const double* P_nzval, const double* q, const uint64_t* A_colptr, const uint64_t* A_rowval,
                   const double* A_nzval, const double* b, uint64_t ncones, const int32_t* cone_types,
                   const uint64_t* cone_dims, const double* cone_params, const cipm_settings* settings,
                   const cldl_opts* ldl_opts, const uint64_t* kkt_perm_or_null) {
  return cipm_create_gp(out, n, m, P_colptr, P_rowval, P_nzval, q, A_colptr, A_rowval, A_nzval, b, ncones, cone_types,
                        cone_dims, cone_params, nullptr, nullptr, settings, ldl_opts, kkt_perm_or_null);
}

int cipm_create_gp(cipm_t** out, uint64_t n, uint64_t m, const uint64_t* P_colptr, const uint64_t* P_rowval,
                   const double* P_nzval, const double* q, const uint64_t* A_colptr, const uint64_t* A_rowval,
                   const double* A_nzval, const double* b, uint64_t ncones, const int32_t* cone_types,
                   const uint64_t* cone_dims, const double* cone_params, const uint64_t* genpow_dim2,
                   const double* genpow_alpha, const cipm_settings* settings, const cldl_opts* ldl_opts,
                   const uint64_t* kkt_perm_or_null) {
  if (!out) return CLDL_E_ARG;
  *out = nullptr;
  if (n == 0 || n > 0x7fffffffu || m > 0x7fffffffu) return CLDL_E_DIM;
  cipm_settings s;
  if (settings) s = *settings; else cipm_default_settings(&s);
  cldl_opts lo;
  if (ldl_opts) lo = *ldl_opts; else cldl_default_opts(&lo);
  cipm_handle* h = new (std::nothrow) cipm_handle();
  if (!h) return CLDL_E_ARG;
  const double t_create0 = cb::wall();
  int rc = h->ipm.init((int)n, (int)m, P_colptr, P_rowval, P_nzval, q, A_colptr, A_rowval, A_nzval, b, ncones,
                       cone_types, cone_dims, s, lo, kkt_perm_or_null, cone_params, genpow_dim2, genpow_alpha);
  if (rc) { h->ipm.release(); delete h; return rc; }
  h->ipm.setup_time = cb::wall() - t_create0;
  *out = h;
  return CLDL_OK;
}

// Solver::update_settings (core/solver.rs:207-211): every field may change except the ones that only act at
// construction (settings.rs:307-335: equilibration parameters, presolve_enable)
int cipm_update_settings(cipm_t* h, const cipm_settings* s) {
  if (!h || !s) return CLDL_E_ARG;
  IPM& I = h->ipm;
  const cipm_settings& p = I.set;
  if (s->equilibrate_enable != p.equilibrate_enable || s->equilibrate_max_iter != p.equilibrate_max_iter ||
      s->equilibrate_min_scaling != p.equilibrate_min_scaling || s->equilibrate_max_scaling != p.equilibrate_max_scaling ||
      s->presolve_enable != p.presolve_enable)
    return CLDL_E_ARG;
  I.set = *s;
  I.kkt.set = *s;
  I.cones.ns_amin = s->min_terminate_step_length; I.cones.ns_step = s->linesearch_backtrack_step;
  return CLDL_OK;
}

int cipm_set_nccl(cipm_t* h, const char* libpath, const unsigned char* id128, int nranks, int rank) {
  return h ? h->ipm.kkt.ldl.set_nccl(libpath, id128, nranks, rank) : CLDL_E_ARG;
}
uint64_t cipm_collective_count(const cipm_t* h) { return h ? h->ipm.kkt.ldl.n_collectives : 0; }
int cipm_set_transport(cipm_t* h, cldl_allgather_fn fn, void* ctx) {
  if (!h) return CLDL_E_ARG;
  h->ipm.kkt.ldl.transport = fn; h->ipm.kkt.ldl.transport_ctx = ctx;
  return CLDL_OK;
}

void cipm_destroy(cipm_t* h) {
  if (!h) return;
  h->ipm.release();
  delete h;
}

int cipm_solve(cipm_t* h) { return h ? h->ipm.solve() : CLDL_E_ARG; }

// set_termination_callback_c / unset_termination_callback (core/solver.rs); on a sharded handle every rank makes the
// call, since a solve with a callback all-gathers every rank's verdict once per pass
int cipm_set_termination_callback(cipm_t* h, cipm_callback_fn fn, void* user_data) {
  if (!h || !fn) return CLDL_E_ARG;
  h->ipm.cb_fn = fn; h->ipm.cb_data = user_data;
  return CLDL_OK;
}
int cipm_unset_termination_callback(cipm_t* h) {
  if (!h) return CLDL_E_ARG;
  h->ipm.cb_fn = nullptr; h->ipm.cb_data = nullptr;
  return CLDL_OK;
}

int cipm_set_print_target(cipm_t* h, int kind, const char* path, cipm_write_fn fn, void* ctx) {
  return h ? h->ipm.out.set(kind, path, fn, ctx) : CLDL_E_ARG;
}
int64_t cipm_get_print_buffer(cipm_t* h, char* out, uint64_t cap) {
  if (!h || h->ipm.out.kind != CIPM_PRINT_BUFFER) return CLDL_E_ARG;
  const std::string& b = h->ipm.out.buffer;
  if (out) std::memcpy(out, b.data(), std::min<uint64_t>(cap, b.size()));
  return (int64_t)b.size();
}

void cipm_get_info(const cipm_t* h, cipm_info* out) { if (h && out) *out = h->ipm.info; }

int cipm_get_solution(cipm_t* h, double* x, double* z, double* s) {
  // unscale (variables.rs:262-285, solution.rs:68-111)
  if (!h) return CLDL_E_ARG;
  IPM& I = h->ipm;
  if (cudaSetDevice(I.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;
  const int st = I.info.status;
  const bool infeas = st == cb::IST_PINF || st == cb::IST_DINF || st == cb::IST_ALMOST_PINF || st == cb::IST_ALMOST_DINF;
  const double scaleinv = infeas ? 1.0 / I.kap : 1.0 / I.tau;
  std::vector<double> hx(I.n), hz(I.m), hs(I.m);
  if (I.n && cudaMemcpy(hx.data(), I.x, (size_t)I.n * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return CLDL_E_CUDA;
  if (I.m && cudaMemcpy(hz.data(), I.z, (size_t)I.m * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return CLDL_E_CUDA;
  if (I.m && cudaMemcpy(hs.data(), I.s, (size_t)I.m * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return CLDL_E_CUDA;
  cb::unscale_solution(I.eq, I.keep, I.infbound, scaleinv, I.n, I.mfull, hx.data(), hz.data(), hs.data(), x, z, s);
  return CLDL_OK;
}

uint64_t cipm_trace(const cipm_t* h, double* out, uint64_t cap_rows) {
  if (!h) return 0;
  const uint64_t rows = h->ipm.trace.size() / 6;
  if (out) for (uint64_t i = 0; i < std::min(rows, cap_rows) * 6; i++) out[i] = h->ipm.trace[i];
  return rows;
}

uint64_t cipm_iter_ms(const cipm_t* h, double* out, uint64_t cap) {
  if (!h) return 0;
  const uint64_t n = h->ipm.iter_ms.size();
  if (out) for (uint64_t i = 0; i < std::min(n, cap); i++) out[i] = h->ipm.iter_ms[i];
  return n;
}
uint64_t cipm_launch_count(void) { return cb::g_launches.load(std::memory_order_relaxed); }
// sizes of the structs that cross the ABI, so that a binding can check its own mirror: {cldl_opts, cldl_info_t, cipm_settings, cipm_info}
void cipm_abi_sizes(uint64_t* out4) { out4[0] = sizeof(cldl_opts); out4[1] = sizeof(cldl_info_t); out4[2] = sizeof(cipm_settings); out4[3] = sizeof(cipm_info); }

// which: 0 = numeric refactor, 1 = one LDL solve (fwd+bwd), 2 = one KKTSolver::solve incl. iterative
// refinement, on whatever values / right-hand side the handle currently holds.  CUDA events on the stream.
double cipm_time_ms(cipm_t* h, int which, int reps) {
  if (!h || reps <= 0) return -1.0;
  IPM& I = h->ipm;
  cb::LDLObject& o = I.kkt.ldl;
  if (cudaSetDevice(o.device) != cudaSuccess) return -1.0;
  cudaStreamSynchronize(o.stream);
  cudaEventRecord(o.ev0, o.stream);
  for (int r = 0; r < reps; r++) {
    if (which == 0) o.refactor_async();
    else if (which == 1) o.solve_async(I.kkt.d_w2, I.kkt.d_b);
    else if (I.kkt.solve(nullptr, nullptr) < 0) return -1.0;
  }
  cudaEventRecord(o.ev1, o.stream);
  cudaEventSynchronize(o.ev1);
  float ms = 0;
  cudaEventElapsedTime(&ms, o.ev0, o.ev1);
  return (double)ms / reps;
}

double cipm_get_infinity(void) { return g_infinity.load(); }
void cipm_set_infinity(double v) { g_infinity.store(v); }
void cipm_default_infinity(void) { g_infinity.store(1e20); }
uint64_t cipm_m_reduced(const cipm_t* h) { return h ? (uint64_t)h->ipm.m : 0; }

// DefaultProblemData::equilibration (problemdata.rs:229-312): d [n], e [cipm_m_reduced] and the cost scaling c
int cipm_get_equilibration(const cipm_t* h, double* d, double* e, double* c) {
  if (!h) return CLDL_E_ARG;
  const cb::IPM& I = h->ipm;
  if (d) for (int i = 0; i < I.n; i++) d[i] = I.eq.d[i];
  if (e) for (int i = 0; i < I.m; i++) e[i] = I.eq.e[i];
  if (c) *c = I.eq.c;
  return CLDL_OK;
}
uint64_t cipm_kkt_dim(const cipm_t* h) { return h ? (uint64_t)h->ipm.kkt.N : 0; }
uint64_t cipm_kkt_nnz(const cipm_t* h) { return h ? (uint64_t)h->ipm.kkt.nnzK : 0; }

int cipm_get_kkt(const cipm_t* h, uint64_t* colptr, uint64_t* rowval, double* nzval, int8_t* dsigns) {
  if (!h) return CLDL_E_ARG;
  const cb::KKTDevice& K = h->ipm.kkt;
  for (int j = 0; j <= K.N; j++) colptr[j] = (uint64_t)K.Kp[j];
  for (int64_t q = 0; q < K.nnzK; q++) { rowval[q] = (uint64_t)K.Ki[q]; nzval[q] = K.Kx[q]; }
  for (int j = 0; j < K.N; j++) dsigns[j] = K.dsigns[j];
  return CLDL_OK;
}

int cipm_get_kkt_perm(const cipm_t* h, uint64_t* perm) {
  if (!h) return CLDL_E_ARG;
  for (int k = 0; k < h->ipm.kkt.N; k++) perm[k] = (uint64_t)h->ipm.kkt.ldl.S.perm[k];
  return CLDL_OK;
}

void cipm_ldl_info(const cipm_t* h, cldl_info_t* info) {
  if (!h || !info) return;
  const cb::LDLObject& o = h->ipm.kkt.ldl;
  std::memset(info, 0, sizeof(*info));
  std::strncpy(info->name, "cudaldl", sizeof(info->name) - 1);
  info->direct = 1;
  info->nnzA = (uint64_t)o.nnzA; info->nnzL = (uint64_t)o.S.nnzL_simplicial; info->nnzL_stored = (uint64_t)o.S.nnzL_stored;
  info->regularize_count = o.regularize_count; info->positive_inertia = o.positive_inertia;
  info->n_supernodes = (uint64_t)o.S.nsup; info->n_levels = (uint64_t)o.S.nlevels; info->flops = o.S.flops_stored;
  info->ordering_used = o.S.ordering_used;
}

// ---- KKTSolver trait (kktsolvers/mod.rs:7-19) on the handle's KKT object; host buffers ----
// cudaMemcpy from pageable host memory returns once the data is STAGED; the DMA to the device may still be in flight, and
// the kernels that consume it run on non-blocking streams that do not wait for the default stream -- so the copy is
// completed here (a flaky dot product in tests/test_zz_algebra_gpu.py was exactly this race)
static int h2d(double* d, const double* h, size_t n) {
  if (n == 0) return 0;
  if (cudaMemcpy(d, h, n * 8, cudaMemcpyHostToDevice) != cudaSuccess) return CLDL_E_CUDA;
  return cudaDeviceSynchronize() == cudaSuccess ? 0 : CLDL_E_CUDA;
}
static int d2h(double* h, const double* d, size_t n) { return n == 0 || cudaMemcpy(h, d, n * 8, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : CLDL_E_CUDA; }

int ckkt_update(cipm_t* h) {
  if (!h) return CLDL_E_ARG;
  if (cudaSetDevice(h->ipm.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;
  return h->ipm.kkt.update();
}
int ckkt_setrhs(cipm_t* h, const double* rhsx, const double* rhsz) {
  if (!h) return CLDL_E_ARG;
  IPM& I = h->ipm;
  if (cudaSetDevice(I.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;
  cudaStreamSynchronize(I.st);
  if (h2d(I.workx, rhsx, I.n) || h2d(I.workz, rhsz, I.m)) return CLDL_E_CUDA;
  I.kkt.setrhs(I.workx, I.workz);
  return CLDL_OK;
}
int ckkt_solve(cipm_t* h, double* lhsx, double* lhsz) {
  if (!h) return CLDL_E_ARG;
  IPM& I = h->ipm;
  if (cudaSetDevice(I.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;
  int ok = I.kkt.solve(I.x1, I.z1);
  if (ok != 1) return ok;
  cudaStreamSynchronize(I.st);
  if ((lhsx && d2h(lhsx, I.x1, I.n)) || (lhsz && d2h(lhsz, I.z1, I.m))) return CLDL_E_CUDA;
  return 1;
}
// The sparse products and reductions of the iteration body on caller data, for kernel-level parity tests
// (algebra/csc/matrix_math.rs, algebra/vecmath.rs; the reference's own known answers are in src/algebra/tests).
// which: 0  y = a P x + b y (P symmetric, the handle's equilibrated copy), 1  y = a A x + b y, 2  y = a A' x + b y
int cipm_test_spmv(cipm_t* h, int which, double* y, const double* x, double a, double b) {
  if (!h || which < 0 || which > 2) return CLDL_E_ARG;
  IPM& I = h->ipm;
  if (cudaSetDevice(I.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;
  const int ny = which == 1 ? I.m : I.n, nx = which == 1 ? I.n : (which == 2 ? I.m : I.n);
  double *dy = nullptr, *dx = nullptr;
  if (cudaMalloc((void**)&dy, (size_t)(ny ? ny : 1) * 8) != cudaSuccess || cudaMalloc((void**)&dx, (size_t)(nx ? nx : 1) * 8) != cudaSuccess) return CLDL_E_CUDA;
  int rc = (h2d(dy, y, ny) || h2d(dx, x, nx)) ? CLDL_E_CUDA : CLDL_OK;
  if (!rc) {
    I.spmv(which == 0 ? I.Psym : (which == 1 ? I.Acsr : I.Atcsr), dy, dx, a, b);
    cudaStreamSynchronize(I.st);
    rc = d2h(y, dy, ny) ? CLDL_E_CUDA : CLDL_OK;
  }
  cudaFree(dy); cudaFree(dx);
  return rc;
}
// what: 0  ||x||_2, 1  ||x||_inf (NaN propagates), 2  ||x .* v||_2, 3  <x, v>
int cipm_test_vec(cipm_t* h, int what, const double* x, const double* v, uint64_t n, double* out) {
  if (!h || !out || what < 0 || what > 3) return CLDL_E_ARG;
  IPM& I = h->ipm;
  if (cudaSetDevice(I.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;
  double *dx = nullptr, *dv = nullptr, *dout = nullptr;
  const size_t nb = (size_t)(n ? n : 1) * 8;
  if (cudaMalloc((void**)&dx, nb) != cudaSuccess || cudaMalloc((void**)&dv, nb) != cudaSuccess || cudaMalloc((void**)&dout, 8) != cudaSuccess) return CLDL_E_CUDA;
  int rc = (h2d(dx, x, n) || h2d(dv, v ? v : x, n)) ? CLDL_E_CUDA : CLDL_OK;
  if (!rc) {
    if (what == 0) I.V.norm(dx, (int)n, dout);
    else if (what == 1) I.V.norm_inf(dx, (int)n, dout);
    else if (what == 2) I.V.norm_scaled(dx, dv, (int)n, dout);
    else I.V.dot(dx, dv, (int)n, dout);
    cudaStreamSynchronize(I.st);
    rc = d2h(out, dout, 1) ? CLDL_E_CUDA : CLDL_OK;
  }
  cudaFree(dx); cudaFree(dv); cudaFree(dout);
  return rc;
}
int cipm_update_data(cipm_t* h, const double* P_nzval, const double* q, const double* A_nzval, const double* b) {
  if (!h) return CLDL_E_ARG;
  return h->ipm.update_data(P_nzval, q, A_nzval, b);
}
// derivatives at the last solve (DESIGN.md, "Solution derivatives"); host buffers, NULL input = zero, NULL output = not
// wanted.  Collective on a sharded handle: the refactor and the solve run the LDL's exchanges.
int cipm_derivative(cipm_t* h, const double* dP_nzval, const double* dq, const double* dA_nzval, const double* db,
                    double* dx, double* dz, double* ds) {
  if (!h) return CLDL_E_ARG;
  return h->ipm.derivative(dP_nzval, dq, dA_nzval, db, dx, dz, ds);
}
int cipm_adjoint_derivative(cipm_t* h, const double* gx, const double* gz, const double* gs, double* gP_nzval,
                            double* gq, double* gA_nzval, double* gb) {
  if (!h) return CLDL_E_ARG;
  return h->ipm.adjoint_derivative(gx, gz, gs, gP_nzval, gq, gA_nzval, gb);
}
int ckkt_update_P(cipm_t* h, const double* P_nzval_scaled) {
  if (!h) return CLDL_E_ARG;
  IPM& I = h->ipm;
  if (cudaSetDevice(I.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;
  I.deriv_valid = false;     // K no longer holds the data of the last solve
  const size_t len = I.kkt.map_P.size();
  double* tmp = nullptr;
  if (cudaMalloc((void**)&tmp, (len ? len : 1) * 8) != cudaSuccess) return CLDL_E_CUDA;
  int rc = h2d(tmp, P_nzval_scaled, len);
  if (!rc) { I.kkt.update_vals(I.kkt.d_map_P, tmp, (int)len); cudaStreamSynchronize(I.st); }
  cudaFree(tmp);
  return rc;
}
int ckkt_update_A(cipm_t* h, const double* A_nzval_scaled) {
  if (!h) return CLDL_E_ARG;
  IPM& I = h->ipm;
  if (cudaSetDevice(I.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;
  I.deriv_valid = false;     // K no longer holds the data of the last solve
  const size_t len = I.kkt.map_A.size();
  double* tmp = nullptr;
  if (cudaMalloc((void**)&tmp, (len ? len : 1) * 8) != cudaSuccess) return CLDL_E_CUDA;
  int rc = h2d(tmp, A_nzval_scaled, len);
  if (!rc) { I.kkt.update_vals(I.kkt.d_map_A, tmp, (int)len); cudaStreamSynchronize(I.st); }
  cudaFree(tmp);
  return rc;
}
int ckkt_get_values(cipm_t* h, double* nzval_out) {
  if (!h) return CLDL_E_ARG;
  IPM& I = h->ipm;
  if (cudaSetDevice(I.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;
  cudaStreamSynchronize(I.st);
  return d2h(nzval_out, I.kkt.ldl.dev.vals, (size_t)I.kkt.nnzK);
}

// ---- Cone trait (cones/mod.rs:42-154) on the handle's composite cone; host buffers of length m ----
#define CONE_PRE                                                                                 \
  if (!h) return CLDL_E_ARG;                                                                     \
  IPM& I = h->ipm;                                                                               \
  if (cudaSetDevice(I.kkt.ldl.device) != cudaSuccess) return CLDL_E_CUDA;                        \
  cudaStreamSynchronize(I.st);                                                                   \
  const size_t m = (size_t)I.m;

int ccone_set_identity_scaling(cipm_t* h) { CONE_PRE (void)m; I.cones.set_identity_scaling(); return cudaStreamSynchronize(I.st) == cudaSuccess ? 0 : CLDL_E_CUDA; }
int ccone_update_scaling(cipm_t* h, const double* s, const double* z) {
  CONE_PRE
  if (h2d(I.ps, s, m) || h2d(I.pz, z, m)) return CLDL_E_CUDA;
  cudaMemsetAsync(I.cones.dev.fail, 0, sizeof(int), I.st);
  I.cones.update_scaling(I.ps, I.pz);
  int fail = 0;
  cudaStreamSynchronize(I.st);
  if (cudaMemcpy(&fail, I.cones.dev.fail, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return CLDL_E_CUDA;
  return fail ? 0 : 1;
}
int ccone_update_scaling_ex(cipm_t* h, const double* s, const double* z, double mu, int strategy) {
  CONE_PRE
  if (h2d(I.ps, s, m) || h2d(I.pz, z, m)) return CLDL_E_CUDA;
  cudaMemsetAsync(I.cones.dev.fail, 0, sizeof(int), I.st);
  I.cones.update_scaling(I.ps, I.pz, mu, strategy);
  int fail = 0;
  cudaStreamSynchronize(I.st);
  if (cudaMemcpy(&fail, I.cones.dev.fail, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return CLDL_E_CUDA;
  return fail ? 0 : 1;
}
int ccone_unit_initialization(cipm_t* h, double* z, double* s) {
  CONE_PRE
  I.cones.unit_initialization(I.pz, I.ps);
  cudaStreamSynchronize(I.st);
  return d2h(z, I.pz, m) || d2h(s, I.ps, m) ? CLDL_E_CUDA : 0;
}
int ccone_affine_ds_ex(cipm_t* h, double* ds, const double* s) {
  CONE_PRE
  if (h2d(I.pz, s, m)) return CLDL_E_CUDA;
  I.cones.affine_ds(I.ps, I.pz);
  cudaStreamSynchronize(I.st);
  return d2h(ds, I.ps, m);
}
int ccone_compute_barrier(cipm_t* h, const double* z, const double* s, const double* dz, const double* ds,
                          double alpha, double* barrier_out) {
  CONE_PRE
  if (h2d(I.ps, z, m) || h2d(I.pz, s, m) || h2d(I.workz, dz, m) || h2d(I.work_conic, ds, m)) return CLDL_E_CUDA;
  I.cones.compute_barrier(I.ps, I.pz, I.workz, I.work_conic, alpha, I.sc.d + cb::S_BP0, I.sc.d + cb::S_BARR);
  cudaStreamSynchronize(I.st);
  return d2h(barrier_out, I.sc.d + cb::S_BARR, 1);
}
int ccone_is_symmetric(const cipm_t* h) { return h ? (h->ipm.cones.all_symmetric ? 1 : 0) : CLDL_E_ARG; }
uint64_t ccone_Hs_len(const cipm_t* h) { return h ? (uint64_t)h->ipm.cones.nHs : 0; }
int ccone_get_Hs(cipm_t* h, double* Hs) {
  CONE_PRE (void)m;
  I.cones.get_Hs(I.kkt.d_Hs, false);
  cudaStreamSynchronize(I.st);
  return d2h(Hs, I.kkt.d_Hs, (size_t)I.cones.nHs);
}
int ccone_mul_Hs(cipm_t* h, double* y, const double* x) {
  CONE_PRE
  if (h2d(I.ps, x, m)) return CLDL_E_CUDA;
  I.cones.mul_Hs(I.pz, I.ps);
  cudaStreamSynchronize(I.st);
  return d2h(y, I.pz, m);
}
int ccone_affine_ds(cipm_t* h, double* ds) {
  CONE_PRE
  I.cones.affine_ds(I.ps);
  cudaStreamSynchronize(I.st);
  return d2h(ds, I.ps, m);
}
int ccone_combined_ds_shift(cipm_t* h, double* shift, const double* step_z, const double* step_s, double sigmamu) {
  CONE_PRE
  if (h2d(I.ps, step_z, m) || h2d(I.pz, step_s, m)) return CLDL_E_CUDA;
  I.cones.combined_ds_shift(I.work_conic, I.ps, I.pz, sigmamu);
  cudaStreamSynchronize(I.st);
  return d2h(shift, I.work_conic, m);
}
int ccone_ds_from_dz_offset(cipm_t* h, double* out, const double* ds, const double* z) {
  CONE_PRE
  if (h2d(I.ps, ds, m) || h2d(I.pz, z, m)) return CLDL_E_CUDA;
  I.cones.ds_from_dz_offset(I.work_conic, I.ps, I.pz);
  cudaStreamSynchronize(I.st);
  return d2h(out, I.work_conic, m);
}
int ccone_step_length(cipm_t* h, const double* dz, const double* ds, const double* z, const double* s,
                      double alpha_max, double* alpha_out) {
  CONE_PRE
  if (h2d(I.ps, dz, m) || h2d(I.pz, ds, m) || h2d(I.workz, z, m) || h2d(I.work_conic, s, m)) return CLDL_E_CUDA;
  if (cudaMemcpy(I.sc.d + cb::S_ALPHA, &alpha_max, 8, cudaMemcpyHostToDevice) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) return CLDL_E_CUDA;
  I.cones.step_length(I.ps, I.pz, I.workz, I.work_conic, I.sc.d + cb::S_ALPHA);
  cudaStreamSynchronize(I.st);
  return d2h(alpha_out, I.sc.d + cb::S_ALPHA, 1);
}
int ccone_margins(cipm_t* h, const double* z, double* min_margin, double* pos_margin) {
  CONE_PRE
  if (h2d(I.ps, z, m)) return CLDL_E_CUDA;
  I.cones.margins(I.ps, I.sc.d + cb::S_MARG0);
  cudaStreamSynchronize(I.st);
  double t[2];
  if (d2h(t, I.sc.d + cb::S_MARG0, 2)) return CLDL_E_CUDA;
  *min_margin = t[0]; *pos_margin = t[1];
  return 0;
}
int ccone_scaled_unit_shift(cipm_t* h, double* z, double alpha, int primal) {
  CONE_PRE
  if (h2d(I.ps, z, m)) return CLDL_E_CUDA;
  I.cones.scaled_unit_shift(I.ps, alpha, primal != 0);
  cudaStreamSynchronize(I.st);
  return d2h(z, I.ps, m);
}

}  // extern "C"
