// Restarted flexible GMRES: the host state machine of cldl_solve_gmres (see ldl_krylov.h).
//
// Within a cycle, with beta = ||r||_2 and v_0 = r / beta, step j forms z_j = K~^-1 v_j and w = K z_j, orthogonalises w
// against v_0 .. v_j by classical Gram-Schmidt twice (h_{i,j} = the two passes' coefficients summed) and stores
// v_{j+1} = w / h_{j+1,j}.  Then K Z_k = V_{k+1} H_k holds to rounding whatever K~ is, so x_best + Z_k y with y the
// least-squares solution of H_k y ~ beta e_1 has residual norm |g_k|, the last entry of the rotated right-hand side
// (Saad 1993).  The rotations, the least-squares solve and every stopping test run here in double precision, in one
// fixed order, so the iteration takes the same path on the same values.
#include "ldl_krylov.h"

#include <cmath>

namespace cb {

namespace {

// the Givens rotation (c, s) with [c s; -s c] [a; b] = [rho; 0]
void givens(double a, double b, double* c, double* s) {
  if (b == 0.0) { *c = 1.0; *s = 0.0; return; }
  if (std::fabs(b) > std::fabs(a)) {
    const double t = a / b, u = 1.0 / std::sqrt(1.0 + t * t);
    *s = u; *c = u * t;
  } else {
    const double t = b / a, u = 1.0 / std::sqrt(1.0 + t * t);
    *c = u; *s = u * t;
  }
}

bool finite_all(const double* v, int k) {
  for (int i = 0; i < k; i++)
    if (!std::isfinite(v[i])) return false;
  return true;
}

}  // namespace

int fgmres_run(KrylovOps& ops, int m, int max_iter, double tol, KrylovResult& out) {
  out = KrylovResult();
  double om[2];
  if (int rc = ops.analyse(om)) return rc;
  out.analyses++;
  if (int rc = ops.keep()) return rc;
  double w = om[0] + om[1];
  out.omega1 = om[0];
  out.omega2 = om[1];
  // R: the rotated Hessenberg matrix, column-major (m + 1) x m; g: the rotated beta e_1
  std::vector<double> R((size_t)(m + 1) * m), cs(m), sn(m), g(m + 1), y(m), h0(m + 1), h1(m + 1);
  while (std::isfinite(w) && w > tol && (int)out.iterations < max_iter) {
    const double wc = w;
    if (int rc = ops.residual()) return rc;
    if (int rc = ops.norm2(3)) return rc;
    if (int rc = ops.store(0, 3)) return rc;
    double beta = 0.0;
    int k = 0;                 // steps of the cycle that enter the least-squares problem
    for (int j = 0; j < m && (int)out.iterations < max_iter; j++) {
      if (int rc = ops.precondition(j)) return rc;
      if (int rc = ops.apply(j)) return rc;
      if (int rc = ops.norm2(2)) return rc;
      for (int pass = 0; pass < 2; pass++) {
        if (int rc = ops.dots(j + 1, pass)) return rc;
        if (int rc = ops.update(j + 1, pass)) return rc;
        if (int rc = ops.norm2(pass)) return rc;
      }
      if (int rc = ops.store(j + 1, 1)) return rc;
      double s[4];
      if (int rc = ops.fetch(j + 1, h0.data(), h1.data(), s)) return rc;
      out.iterations++;
      if (j == 0) {
        beta = std::sqrt(s[3]);
        g[0] = beta;
      }
      double* col = R.data() + (size_t)j * (m + 1);
      for (int i = 0; i <= j; i++) col[i] = h0[i] + h1[i];
      const double hn = std::sqrt(s[1]), kz = std::sqrt(s[2]);
      col[j + 1] = hn;
      if (!(beta > 0.0) || !std::isfinite(beta) || !finite_all(col, j + 2) || !std::isfinite(kz)) break;
      for (int i = 0; i < j; i++) {
        const double a = col[i], b = col[i + 1];
        col[i] = cs[i] * a + sn[i] * b;
        col[i + 1] = -sn[i] * a + cs[i] * b;
      }
      givens(col[j], col[j + 1], &cs[j], &sn[j]);
      col[j] = cs[j] * col[j] + sn[j] * col[j + 1];
      col[j + 1] = 0.0;
      g[j + 1] = -sn[j] * g[j];
      g[j] = cs[j] * g[j];
      k = j + 1;
      if (hn <= 0x1p-40 * kz) { out.breakdowns++; break; }     // the solution lies in the space
      if (std::fabs(g[j + 1]) <= tol / wc * beta) break;
    }
    out.cycles++;
    if (k == 0) break;         // nothing to correct with: x stays, so omega1 + omega2 is not lowered
    for (int i = k - 1; i >= 0; i--) {
      double a = g[i];
      for (int l = i + 1; l < k; l++) a -= R[(size_t)l * (m + 1) + i] * y[l];
      y[i] = a / R[(size_t)i * (m + 1) + i];
    }
    if (int rc = ops.correct(k, y.data())) return rc;
    if (int rc = ops.analyse(om)) return rc;
    out.analyses++;
    out.estimates.push_back(std::fabs(g[k]));
    const double wn = om[0] + om[1];
    if (wn < w) {              // the earlier iterate on a tie
      if (int rc = ops.keep()) return rc;
      out.omega1 = om[0];
      out.omega2 = om[1];
    }
    if (!(wn < wc)) break;     // not lowered, or not finite
    w = wn;
  }
  return 0;
}

}  // namespace cb
