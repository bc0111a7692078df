// TEST INFRASTRUCTURE ONLY -- the emulated build's stand-in for clarabel.rs_b200/csrc/ldl.cu.
//
// Same LDLObject interface (csrc/ldl_device.h), same ordering / symbolic analysis (csrc/{ordering,symbolic}.cpp, so
// the permutation handed to the oracle is the product's), but the numeric part is a DENSE host LDL^T of the permuted
// KKT matrix with the product's pivot rule: D[k]*sign < eps  =>  D[k] = delta*sign, counted (qdldl.rs:645-651), in
// elimination order.  This lets tests/test_emu_cpu.py run the IPM driver, the KKT layer and every cone kernel of the
// product on a CPU (small problems only: O(N^3)).  The multifrontal kernels themselves are NOT exercised here; they
// have their own GPU parity tests (tests/test_ldl_gpu.py).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "ldl_device.h"

namespace cb {

std::atomic<unsigned long long> g_launches{0};

namespace {
struct Dense {
  std::vector<int64_t> Ap;
  std::vector<int32_t> Ai;
  std::vector<signed char> ds;    // caller order
  std::vector<double> L;          // n x n column major, unit lower
  std::vector<double> D, Dinv;
};
Dense* dense_of(LDLObject* o) { return reinterpret_cast<Dense*>(o->d_bx); }   // d_bx is otherwise unused here
}  // namespace

int LDLObject::init(int n_, const int64_t* Ap, const int32_t* Ai, const double* Ax, const int8_t* dsigns,
                    const cldl_opts& o, const int* perm_in) {
  n = n_;
  opts = o;
  device = o.device;
  if (n > 3000) { std::fprintf(stderr, "[emu] dense LDL stand-in: N = %d is too large\n", n); return CLDL_E_DIM; }
  SymbolicOptions so;
  so.ordering = o.ordering ? o.ordering : ORDER_BEST;
  so.amd_dense_scale = o.amd_dense_scale > 0 ? o.amd_dense_scale : 1.5;
  if (o.max_panel > 0) so.max_panel = o.max_panel > CB_PB_MAXNS ? CB_PB_MAXNS : o.max_panel;
  if (o.nd_leaf > 0) so.nd_leaf = o.nd_leaf;
  int rc = analyse(n, Ap, Ai, perm_in, so, S);
  if (rc == -2) return CLDL_E_EMPTY_COLUMN;
  if (rc == -3) return CLDL_E_NOT_TRIU;
  if (rc == -5) return CLDL_E_BAD_PERM;
  if (rc) return CLDL_E_ARG;
  if (own.stream(&stream, cudaStreamNonBlocking) || own.event(&ev0) || own.event(&ev1))
    return CLDL_E_CUDA;
  nnzA = Ap[n];
  if (own.alloc(&dev.vals, (size_t)nnzA)) return CLDL_E_CUDA;
  std::memcpy(dev.vals, Ax, (size_t)nnzA * sizeof(double));
  dev.reg_enable = o.regularize_enable; dev.reg_eps = o.regularize_eps; dev.reg_delta = o.regularize_delta;
  Dense* d = new Dense();
  d->Ap.assign(Ap, Ap + n + 1);
  d->Ai.assign(Ai, Ai + nnzA);
  d->ds.resize(n);
  for (int k = 0; k < n; k++) d->ds[k] = dsigns ? (signed char)dsigns[k] : (signed char)1;
  d->L.assign((size_t)n * n, 0.0); d->D.assign(n, 0.0); d->Dinv.assign(n, 0.0);
  d_bx = reinterpret_cast<double*>(d);
  use_dataflow = false;
  factored = false;
  return CLDL_OK;
}

void LDLObject::release() {
  delete dense_of(this);
  d_bx = nullptr;
}

static int g_nonfinite = 0, g_zeropiv = 0;

int LDLObject::refactor_async() {
  Dense* d = dense_of(this);
  const int N = n;
  std::vector<double>& M = d->L;           // permuted matrix, overwritten by L (unit lower) below the diagonal
  std::fill(M.begin(), M.end(), 0.0);
  for (int c = 0; c < N; c++)
    for (int64_t p = d->Ap[c]; p < d->Ap[c + 1]; p++) {
      const int a = S.iperm[d->Ai[p]], b = S.iperm[c];
      const int i = a > b ? a : b, j = a > b ? b : a;     // lower triangle (i >= j)
      M[(size_t)j * N + i] += dev.vals[p];
    }
  regularize_count = 0; positive_inertia = 0; g_nonfinite = 0; g_zeropiv = 0;
  for (int k = 0; k < N; k++) {
    double dk = M[(size_t)k * N + k];
    const double sgn = (double)d->ds[S.perm[k]];
    if (dev.reg_enable && dk * sgn < dev.reg_eps) { dk = dev.reg_delta * sgn; regularize_count++; }
    if (dk == 0.0) g_zeropiv = 1;
    if (dk > 0.0) positive_inertia++;
    d->D[k] = dk; d->Dinv[k] = 1.0 / dk;
    if (!std::isfinite(d->Dinv[k])) g_nonfinite = 1;
    double* colk = &M[(size_t)k * N];
    for (int i = k + 1; i < N; i++) colk[i] *= d->Dinv[k];           // L(:,k)
    for (int j = k + 1; j < N; j++) {
      const double ljk = colk[j] * dk;                               // = original M(j,k)
      if (ljk == 0.0) continue;
      double* colj = &M[(size_t)j * N];
      for (int i = j; i < N; i++) colj[i] -= colk[i] * ljk;
    }
  }
  factored = true;
  return CLDL_OK;
}

int LDLObject::sync_status() {
  if (g_zeropiv && !dev.reg_enable) return CLDL_E_ZERO_PIVOT;
  return g_nonfinite ? 0 : 1;
}


int LDLObject::solve_async(double* d_x, const double* d_b, double* d_x1, const double* d_b1) {
  if (!factored) return CLDL_E_NOT_FACTORED;
  if (d_x1) { int rc = solve_async(d_x1, d_b1, nullptr, nullptr); if (rc) return rc; }
  Dense* d = dense_of(this);
  const int N = n;
  std::vector<double> y(N);
  for (int k = 0; k < N; k++) y[k] = d_b[S.perm[k]];
  for (int k = 0; k < N; k++) {                                       // L y = b
    const double yk = y[k];
    const double* colk = &d->L[(size_t)k * N];
    for (int i = k + 1; i < N; i++) y[i] -= colk[i] * yk;
  }
  for (int k = 0; k < N; k++) y[k] *= d->Dinv[k];
  for (int k = N - 1; k >= 0; k--) {                                  // L' x = y
    const double* colk = &d->L[(size_t)k * N];
    double acc = y[k];
    for (int i = k + 1; i < N; i++) acc -= colk[i] * y[i];
    y[k] = acc;
  }
  for (int k = 0; k < N; k++) d_x[S.perm[k]] = y[k];
  return CLDL_OK;
}

int LDLObject::set_nccl(const char*, const unsigned char*, int, int) { return CLDL_E_ARG; }
int LDLObject::refactor_phase_async(int) { return CLDL_E_ARG; }
int LDLObject::solve_phase_async(double*, const double*, int) { return CLDL_E_ARG; }
uint64_t LDLObject::shard_count(int, int) const { return 0; }
int LDLObject::shard_pack(int, double*, const double*) { return CLDL_E_ARG; }
int LDLObject::shard_seglist(int, int, const long long**, int*) { return CLDL_E_ARG; }
int LDLObject::shard_unpack(int, int, const double*, double*) { return CLDL_E_ARG; }
int LDLObject::ensure_tmp(size_t) { return 0; }
int LDLObject::stage_index(const uint64_t*, uint64_t) { return 0; }

}  // namespace cb

// Level-1 entry points referenced by solver.cu
extern "C" void cldl_default_opts(cldl_opts* o) {
  std::memset(o, 0, sizeof(*o));
  o->regularize_eps = 1e-13; o->regularize_delta = 2e-7; o->regularize_enable = 1; o->amd_dense_scale = 1.5;
  o->ordering = CLDL_ORDER_BEST;
}
// The Level-1 C entry points are not part of the emulated build (they wrap the multifrontal kernels); they exist so
// that the Python loader finds every symbol, and refuse.
extern "C" {
int cldl_create(cldl_t** out, uint64_t, const uint64_t*, const uint64_t*, const double*, const int8_t*, const cldl_opts*, const uint64_t*) { if (out) *out = nullptr; return CLDL_E_CUDA; }
void cldl_destroy(cldl_t*) {}
int cldl_update_values(cldl_t*, const uint64_t*, const double*, uint64_t) { return CLDL_E_CUDA; }
int cldl_scale_values(cldl_t*, const uint64_t*, uint64_t, double) { return CLDL_E_CUDA; }
int cldl_offset_values(cldl_t*, const uint64_t*, uint64_t, double, const int8_t*) { return CLDL_E_CUDA; }
int cldl_refactor(cldl_t*) { return CLDL_E_CUDA; }
int cldl_solve(cldl_t*, double*, const double*) { return CLDL_E_CUDA; }
void cldl_info(const cldl_t*, cldl_info_t*) {}
int cldl_get_perm(const cldl_t*, uint64_t*) { return CLDL_E_CUDA; }
int cldl_update_values_dev(cldl_t*, const int32_t*, const double*, uint64_t) { return CLDL_E_CUDA; }
int cldl_set_values_dev(cldl_t*, const double*) { return CLDL_E_CUDA; }
int cldl_refactor_dev(cldl_t*) { return CLDL_E_CUDA; }
int cldl_solve_dev(cldl_t*, double*, const double*) { return CLDL_E_CUDA; }
int cldl_sync_status(cldl_t*) { return CLDL_E_CUDA; }
void* cldl_stream(cldl_t*) { return nullptr; }
double* cldl_values_dev(cldl_t*) { return nullptr; }
double cldl_time_refactor_ms(cldl_t*, int) { return -1.0; }
double cldl_time_solve_ms(cldl_t*, int) { return -1.0; }
int cldl_shard_refactor_phase_dev(cldl_t*, int) { return CLDL_E_CUDA; }
int cldl_shard_solve_phase_dev(cldl_t*, double*, const double*, int) { return CLDL_E_CUDA; }
uint64_t cldl_shard_count(const cldl_t*, int, int) { return 0; }
int cldl_shard_pack_dev(cldl_t*, int, double*, const double*) { return CLDL_E_CUDA; }
int cldl_shard_unpack_dev(cldl_t*, int, int, const double*, double*) { return CLDL_E_CUDA; }
int cldl_shard_counts(const cldl_t*, uint64_t*) { return CLDL_E_CUDA; }
int cldl_set_transport(cldl_t*, cldl_allgather_fn, void*) { return CLDL_E_CUDA; }
int cldl_copy_dev(void* d, const void* s, uint64_t n) { if (n) std::memmove(d, s, (size_t)n); return 0; }
}
