// Thick-restart Lanczos: the host state machine of cldl_eigsh (see ldl_eig.h).
//
// After a restart with k kept Ritz pairs the projected matrix H (m x m, m = ncv) is
//     [ diag(theta_kept)  s        ]      s_i = beta_m y_{m-1,i}, the old residual's coupling to kept pair i,
//     [ s^T               tridiag  ]      the Lanczos steps j = k .. m-1 fill the tridiagonal part,
// and T V_m = V_m H + beta_m v_m e_m^T holds with v_m the normalised residual (column m of V).  Each step
// orthogonalises w = T v_j against every basis vector by classical Gram-Schmidt, twice, so only alpha_j and beta_j
// enter H.  When the second pass removes more than 30% of what the first left (ARPACK's DGKS test), or what is left is
// below 2^-40 of ||T v_j||_M, w is rounding noise: T's Krylov space is invariant, beta_j = 0 and a fresh random vector
// continues the basis.
#include "ldl_eig.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <numeric>

namespace cb {

void eig_jacobi(int m, std::vector<double>& A, std::vector<double>& theta, std::vector<double>& Y) {
  Y.assign((size_t)m * m, 0.0);
  for (int i = 0; i < m; i++) Y[(size_t)i * m + i] = 1.0;
  for (int sweep = 0; sweep < 100; sweep++) {
    int rotations = 0;
    for (int p = 0; p < m - 1; p++)
      for (int q = p + 1; q < m; q++) {
        const double apq = A[(size_t)p * m + q], app = A[(size_t)p * m + p], aqq = A[(size_t)q * m + q];
        if (!(std::fabs(apq) > DBL_EPSILON * std::sqrt(std::fabs(app * aqq)))) continue;
        rotations++;
        // Rutishauser's rotation: t = tan of the angle that zeroes a_pq, the smaller root
        const double th = (aqq - app) / (2.0 * apq);
        const double t = std::fabs(th) > 1e150 ? 0.5 / th
                                               : (th >= 0.0 ? 1.0 : -1.0) / (std::fabs(th) + std::sqrt(th * th + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int r = 0; r < m; r++) {          // columns p and q
          const double ap = A[(size_t)r * m + p], aq = A[(size_t)r * m + q];
          A[(size_t)r * m + p] = c * ap - s * aq;
          A[(size_t)r * m + q] = s * ap + c * aq;
        }
        for (int r = 0; r < m; r++) {          // rows p and q
          const double ap = A[(size_t)p * m + r], aq = A[(size_t)q * m + r];
          A[(size_t)p * m + r] = c * ap - s * aq;
          A[(size_t)q * m + r] = s * ap + c * aq;
        }
        A[(size_t)p * m + q] = A[(size_t)q * m + p] = 0.0;
        for (int r = 0; r < m; r++) {
          const double yp = Y[(size_t)r * m + p], yq = Y[(size_t)r * m + q];
          Y[(size_t)r * m + p] = c * yp - s * yq;
          Y[(size_t)r * m + q] = s * yp + c * yq;
        }
      }
    if (!rotations) break;
  }
  theta.resize(m);
  for (int i = 0; i < m; i++) theta[i] = A[(size_t)i * m + i];
}

namespace {

// w orthogonalised twice against v_0 .. v_{j-1} (none when j = 0) and stored as v_j.  out = h0[row], h1[row] and the
// squared M-norms of w after pass 1 (s0), after pass 2 (s1) and before either (s2).
int orth_store(EigOps& ops, int j, int row, double out[5]) {
  if (int rc = ops.mnorm2(2)) return rc;
  if (j == 0) {
    if (int rc = ops.store(0, 2)) return rc;
    return ops.fetch(row, out);
  }
  for (int pass = 0; pass < 2; pass++) {
    if (int rc = ops.mdots(j, pass)) return rc;
    if (int rc = ops.update(j, pass)) return rc;
    if (int rc = ops.mnorm2(pass)) return rc;
  }
  if (int rc = ops.store(j, 1)) return rc;
  return ops.fetch(row, out);
}

bool kept_norm(double n0sq, double n1sq, double n2sq) {
  return n2sq > 0.717 * 0.717 * n1sq && n2sq > 0x1p-80 * n0sq;
}

struct Lanczos {
  EigOps& ops;
  int n, m;
  bool ident;
  EigResult& res;
  uint64_t draws = 0;
  bool failed = false;         // M-norm <= 0 (status -1) or a non-finite value (status 0)
  // Only the norms of vectors that are not noise decide status -1: a fresh draw's, and that of T v_j, both with M w
  // from a product.  After the passes z = M w is carried along (z -= MV h), and at rounding level w^T z may come out
  // negative for a positive definite M: that w is noise and is deflated.

  // v_j = a fresh random vector orthogonal to v_0 .. v_{j-1} (j < m <= n, so the complement is not empty); three
  // draws at most (a draw inside the span is as likely as hitting a hyperplane), the last one kept when its M-norm is
  // positive.  A draw orthogonalised against fewer than n vectors keeps a real component, so a norm^2 <= 0 left after
  // three draws comes from M, not from rounding: status -1.
  int fresh(int j) {
    double o[5];
    for (int attempt = 0; attempt < 3; attempt++) {
      if (int rc = ops.random(draws++)) return rc;
      if (int rc = orth_store(ops, j, 0, o)) return rc;
      if (j == 0) o[2] = o[3] = o[4];          // no Gram-Schmidt passes: s0 and s1 were not written
      if (!std::isfinite(o[2]) || !std::isfinite(o[3]) || !std::isfinite(o[4])) { failed = true; res.status = 0; return 0; }
      if (!(o[4] > 0.0)) { failed = true; res.status = -1; return 0; }
      if (j == 0 || kept_norm(o[4], o[2], o[3])) return 0;
    }
    if (!ident && !(o[3] > 0.0)) { failed = true; res.status = -1; }
    return 0;
  }

  // Lanczos step j: alpha_j and beta_j (0 at an invariant subspace, v_{j+1} then fresh)
  int step(int j, double* alpha, double* beta) {
    if (int rc = ops.apply(j)) return rc;
    res.applies++;
    double o[5];
    if (int rc = orth_store(ops, j + 1, j, o)) return rc;
    *alpha = o[0] + o[1];
    if (!std::isfinite(*alpha) || !std::isfinite(o[2]) || !std::isfinite(o[3]) || !std::isfinite(o[4])) {
      failed = true; res.status = 0; return 0;
    }
    if (!ident && o[4] < 0.0) { failed = true; res.status = -1; return 0; }
    if (kept_norm(o[4], o[2], o[3])) { *beta = std::sqrt(o[3]); return 0; }
    *beta = 0.0;
    res.deflations++;
    return j + 1 < m ? fresh(j + 1) : 0;     // at j + 1 = m the residual is not needed: beta_m = 0 converges every pair
  }
};

}  // namespace

int lanczos_run(EigOps& ops, int n, int nev, int ncv, int max_restarts, double tol, bool m_identity, EigResult& out) {
  out = EigResult();
  const int m = ncv;
  if (!(tol > 0.0)) tol = DBL_EPSILON;
  Lanczos L{ops, n, m, m_identity, out};
  if (int rc = L.fresh(0)) return rc;
  if (L.failed) return 0;
  std::vector<double> H((size_t)m * m, 0.0), A, theta, Y;
  std::vector<int> order(m);
  double beta_m = 0.0;
  int k = 0, nconv = 0;
  auto conv = [&](int i) { return std::fabs(beta_m * Y[(size_t)(m - 1) * m + i]) <= tol * std::fabs(theta[i]); };
  for (;;) {
    for (int j = k; j < m; j++) {
      double a = 0.0, b = 0.0;
      if (int rc = L.step(j, &a, &b)) return rc;
      if (L.failed) return 0;
      H[(size_t)j * m + j] = a;
      if (j + 1 < m) H[(size_t)j * m + j + 1] = H[(size_t)(j + 1) * m + j] = b;
      else beta_m = b;
    }
    A = H;
    eig_jacobi(m, A, theta, Y);
    // wanted: largest |theta| first; ties by theta, then by index, so the order is a function of the values alone
    std::iota(order.begin(), order.end(), 0);
    std::sort(order.begin(), order.end(), [&](int a, int b) {
      const double fa = std::fabs(theta[a]), fb = std::fabs(theta[b]);
      if (fa != fb) return fa > fb;
      if (theta[a] != theta[b]) return theta[a] > theta[b];
      return a < b;
    });
    nconv = 0;
    for (int i = 0; i < nev; i++) nconv += conv(order[i]) ? 1 : 0;
    if (nconv >= nev) { out.status = 1; break; }
    if (out.restarts >= max_restarts) { out.status = 0; break; }
    // keep the nev wanted pairs and up to half the rest, more as more have converged (ARPACK's dsaup2)
    const int kk = std::min(m - 1, nev + std::min(nconv, (m - nev) / 2));
    std::vector<double> S((size_t)m * kk);
    for (int c = 0; c < kk; c++)
      for (int r = 0; r < m; r++) S[(size_t)c * m + r] = Y[(size_t)r * m + order[c]];
    if (int rc = ops.combine(m, kk, S.data())) return rc;
    if (int rc = ops.copy(kk, m)) return rc;
    std::fill(H.begin(), H.end(), 0.0);
    for (int c = 0; c < kk; c++) {
      H[(size_t)c * m + c] = theta[order[c]];
      H[(size_t)c * m + kk] = H[(size_t)kk * m + c] = beta_m * Y[(size_t)(m - 1) * m + order[c]];
    }
    k = kk;
    out.restarts++;
  }
  // the returned pairs: the converged wanted ones, then the rest of the wanted, each group ascending in 1/theta (which
  // is ascending in sigma + 1/theta)
  std::vector<int> sel(order.begin(), order.begin() + nev);
  std::stable_sort(sel.begin(), sel.end(), [&](int a, int b) {
    const bool ca = conv(a), cb = conv(b);
    if (ca != cb) return ca;
    return 1.0 / theta[a] < 1.0 / theta[b];
  });
  std::vector<double> S((size_t)m * nev);
  out.theta.resize(nev);
  for (int c = 0; c < nev; c++) {
    out.theta[c] = theta[sel[c]];
    for (int r = 0; r < m; r++) S[(size_t)c * m + r] = Y[(size_t)r * m + sel[c]];
  }
  out.nconv = nconv;
  return ops.combine(m, nev, S.data());
}

}  // namespace cb
