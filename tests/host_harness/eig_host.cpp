// The thick-restart Lanczos of cldl_eigsh (csrc/ldl_eig.cpp) on dense matrices, for tests/test_eigsh_host_cpu.py: the
// EigOps are plain loops, T a dense n x n matrix (the test passes (A - sigma M)^-1 M), M dense or the identity, the
// random vectors the columns of a matrix the test passes.  Built with g++ by the test, loaded with ctypes.
#include <cmath>
#include <cstring>
#include <vector>

#include "ldl_eig.h"

using namespace cb;

namespace {
struct DenseOps final : EigOps {
  int n, ncv;
  const double *T, *M, *R;     // row-major n x n; M NULL = identity; R n x nr column-major
  int nr;
  std::vector<double> V, w, Mw, h[2], s;
  int fail_at = -1;            // apply() of this call count returns error 7 (error propagation)
  int calls = 0;

  void mw() {
    if (!M) { Mw = w; return; }
    for (int i = 0; i < n; i++) {
      double a = 0.0;
      for (int k = 0; k < n; k++) a += M[(size_t)i * n + k] * w[k];
      Mw[i] = a;
    }
  }
  double* col(int j) { return V.data() + (size_t)j * n; }
  int apply(int j) override {
    if (calls++ == fail_at) return 7;
    const double* v = col(j);
    for (int i = 0; i < n; i++) {
      double a = 0.0;
      for (int k = 0; k < n; k++) a += T[(size_t)i * n + k] * v[k];
      w[i] = a;
    }
    return 0;
  }
  int random(uint64_t draw) override {
    if ((int)draw >= nr) return 8;
    std::memcpy(w.data(), R + (size_t)draw * n, (size_t)n * sizeof(double));
    return 0;
  }
  int mdots(int j, int slot) override {
    mw();
    for (int c = 0; c < j; c++) {
      double a = 0.0;
      for (int i = 0; i < n; i++) a += col(c)[i] * Mw[i];
      h[slot][c] = a;
    }
    return 0;
  }
  int update(int j, int slot) override {
    for (int i = 0; i < n; i++) {
      double a = 0.0;
      for (int c = 0; c < j; c++) a += col(c)[i] * h[slot][c];
      w[i] -= a;
    }
    return 0;
  }
  int mnorm2(int slot) override {
    mw();
    double a = 0.0;
    for (int i = 0; i < n; i++) a += w[i] * Mw[i];
    s[slot] = a;
    return 0;
  }
  int store(int j, int slot) override {
    const double d = s[slot] > 0.0 ? std::sqrt(s[slot]) : 0.0;
    for (int i = 0; i < n; i++) col(j)[i] = d > 0.0 ? w[i] / d : 0.0;
    return 0;
  }
  int combine(int m, int k, const double* S) override {
    std::vector<double> Y((size_t)n * k, 0.0);
    for (int c = 0; c < k; c++)
      for (int i = 0; i < n; i++) {
        double a = 0.0;
        for (int p = 0; p < m; p++) a += col(p)[i] * S[(size_t)c * m + p];
        Y[(size_t)c * n + i] = a;
      }
    std::memcpy(V.data(), Y.data(), Y.size() * sizeof(double));
    return 0;
  }
  int copy(int dst, int src) override {
    std::memcpy(col(dst), col(src), (size_t)n * sizeof(double));
    return 0;
  }
  int fetch(int j, double out[5]) override {
    out[0] = h[0][j]; out[1] = h[1][j]; out[2] = s[0]; out[3] = s[1]; out[4] = s[2];
    return 0;
  }
};
}  // namespace

extern "C" {

void eig_jacobi_c(int m, const double* A, double* theta, double* Y) {
  std::vector<double> a(A, A + (size_t)m * m), th, y;
  eig_jacobi(m, a, th, y);
  std::memcpy(theta, th.data(), (size_t)m * sizeof(double));
  std::memcpy(Y, y.data(), (size_t)m * m * sizeof(double));
}

// out_i: status, nconv, restarts, applies, deflations; theta nev values; X n x nev column-major
int eig_run_c(int n, const double* T, const double* M, const double* R, int nr, int nev, int ncv, int max_restarts,
              double tol, int fail_at, int* out_i, double* theta, double* X) {
  DenseOps o;
  o.n = n; o.ncv = ncv; o.T = T; o.M = M; o.R = R; o.nr = nr; o.fail_at = fail_at;
  o.V.assign((size_t)n * (ncv + 1), 0.0);
  o.w.assign(n, 0.0); o.Mw.assign(n, 0.0);
  o.h[0].assign(ncv + 1, 0.0); o.h[1].assign(ncv + 1, 0.0);
  o.s.assign(3, 0.0);
  EigResult r;
  const int rc = lanczos_run(o, n, nev, ncv, max_restarts, tol, M == nullptr, r);
  out_i[0] = r.status; out_i[1] = r.nconv; out_i[2] = r.restarts; out_i[3] = (int)r.applies; out_i[4] = (int)r.deflations;
  for (size_t c = 0; c < r.theta.size(); c++) theta[c] = r.theta[c];
  std::memcpy(X, o.V.data(), (size_t)n * nev * sizeof(double));
  return rc;
}
}
