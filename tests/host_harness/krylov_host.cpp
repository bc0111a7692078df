// The restarted FGMRES of cldl_solve_gmres (csrc/ldl_krylov.cpp) on dense matrices, for tests/test_krylov_host_cpu.py:
// the KrylovOps are plain loops, K a dense n x n matrix, the preconditioner a dense matrix P applied as z = P v (the
// test passes P = (K + E)^-1), x0 = P b, and the analysis the componentwise backward errors of cldl_solve_refined.
// Built with g++ by the test, loaded with ctypes.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "ldl_krylov.h"

using namespace cb;

namespace {
struct DenseOps final : KrylovOps {
  int n, m;
  const double *K, *P, *b;     // row-major n x n
  std::vector<double> V, Z, w, x, xbest, r, h[2], s;
  std::vector<double> rnorms;  // ||b - K x||_2 at every analysis
  int fail_at = -1;            // precondition() of this call count returns error 7 (error propagation)
  int calls = 0;

  double* col(std::vector<double>& B, int j) { return B.data() + (size_t)j * n; }
  void matvec(const double* A, const double* v, double* out) {
    for (int i = 0; i < n; i++) {
      double a = 0.0;
      for (int k = 0; k < n; k++) a += A[(size_t)i * n + k] * v[k];
      out[i] = a;
    }
  }
  int residual() override { w = r; return 0; }
  int precondition(int j) override {
    if (calls++ == fail_at) return 7;
    matvec(P, col(V, j), col(Z, j));
    return 0;
  }
  int apply(int j) override { matvec(K, col(Z, j), w.data()); return 0; }
  int dots(int j, int slot) override {
    for (int c = 0; c < j; c++) {
      double a = 0.0;
      for (int i = 0; i < n; i++) a += col(V, c)[i] * w[i];
      h[slot][c] = a;
    }
    return 0;
  }
  int update(int j, int slot) override {
    for (int i = 0; i < n; i++) {
      double a = 0.0;
      for (int c = 0; c < j; c++) a += col(V, c)[i] * h[slot][c];
      w[i] -= a;
    }
    return 0;
  }
  int norm2(int slot) override {
    double a = 0.0;
    for (int i = 0; i < n; i++) a += w[i] * w[i];
    s[slot] = a;
    return 0;
  }
  int store(int j, int slot) override {
    const double d = s[slot] > 0.0 ? std::sqrt(s[slot]) : 0.0;
    for (int i = 0; i < n; i++) col(V, j)[i] = d > 0.0 ? w[i] / d : 0.0;
    return 0;
  }
  int correct(int k, const double* y) override {
    for (int i = 0; i < n; i++) {
      double a = 0.0;
      for (int c = 0; c < k; c++) a += col(Z, c)[i] * y[c];
      x[i] = xbest[i] + a;
    }
    return 0;
  }
  int keep() override { xbest = x; return 0; }
  int analyse(double om[2]) override {
    double xn = 0.0, rn = 0.0;
    for (int i = 0; i < n; i++) xn = std::fmax(xn, std::fabs(x[i]));
    matvec(K, x.data(), r.data());
    om[0] = om[1] = 0.0;
    for (int i = 0; i < n; i++) {
      r[i] = b[i] - r[i];
      rn += r[i] * r[i];
      double kx = 0.0, rmax = 0.0;
      for (int k = 0; k < n; k++) {
        const double a = std::fabs(K[(size_t)i * n + k]);
        kx += a * std::fabs(x[k]);
        rmax = std::fmax(rmax, a);
      }
      const double ab = std::fabs(b[i]), ar = std::fabs(r[i]), den1 = kx + ab, den2 = kx + rmax * xn;
      if (den1 > 1000.0 * n * DBL_EPSILON * (rmax * xn + ab)) om[0] = std::fmax(om[0], ar / den1);
      else if (den2 != 0.0 || ar != 0.0) om[1] = std::fmax(om[1], ar / den2);
    }
    rnorms.push_back(std::sqrt(rn));
    return 0;
  }
  int fetch(int j, double* h0, double* h1, double out[4]) override {
    for (int i = 0; i < j; i++) { h0[i] = h[0][i]; h1[i] = h[1][i]; }
    for (int q = 0; q < 4; q++) out[q] = s[q];
    return 0;
  }
};
}  // namespace

extern "C" {

// out_i: iterations, cycles, analyses, breakdowns, number of estimates; out_d: omega1, omega2 of the returned x.
// x: the returned x; est: the per-cycle estimates (cap entries at most); rnorm: ||b - K x||_2 at every analysis
int fgmres_c(int n, const double* K, const double* P, const double* b, int m, int max_iter, double tol, int fail_at,
             int* out_i, double* out_d, double* x, double* est, double* rnorm, int cap) {
  DenseOps o;
  o.n = n; o.m = m; o.K = K; o.P = P; o.b = b; o.fail_at = fail_at;
  o.V.assign((size_t)n * (m + 1), 0.0);
  o.Z.assign((size_t)n * m, 0.0);
  o.w.assign(n, 0.0); o.r.assign(n, 0.0); o.x.assign(n, 0.0);
  o.h[0].assign(m + 1, 0.0); o.h[1].assign(m + 1, 0.0);
  o.s.assign(4, 0.0);
  o.matvec(P, b, o.x.data());       // x0: the "plain solve" with the preconditioner
  o.xbest = o.x;
  KrylovResult res;
  const int rc = fgmres_run(o, m, max_iter, tol, res);
  out_i[0] = (int)res.iterations; out_i[1] = (int)res.cycles; out_i[2] = (int)res.analyses;
  out_i[3] = (int)res.breakdowns; out_i[4] = (int)res.estimates.size();
  out_d[0] = res.omega1; out_d[1] = res.omega2;
  std::memcpy(x, o.xbest.data(), (size_t)n * sizeof(double));
  for (size_t c = 0; c < res.estimates.size() && (int)c < cap; c++) est[c] = res.estimates[c];
  for (size_t c = 0; c < o.rnorms.size() && (int)c < cap; c++) rnorm[c] = o.rnorms[c];
  return rc;
}
}
