// Restarted right-preconditioned flexible GMRES (Saad 1993) for K x = b with a preconditioner K~ close to K.
// cldl_solve_gmres runs it with K the handle's current values and K~ the factor of the last refactor (static pivoting,
// perhaps regularised, perhaps of older values).  Host-only code: the iteration is written against KrylovOps, a small
// set of operations on an n x (m + 1) basis V, an n x m block Z = K~^-1 V, a work vector w and the iterates, so that it
// runs unchanged on the GPU (LDLObject::solve_gmres) and on dense matrices in a CPU test.
#pragma once
#include <cstdint>
#include <vector>

namespace cb {

constexpr int KRYLOV_MAX_RESTART = 512;     // the basis operations are those of cldl_eigsh (EIG_MAX_NCV)

// The operations the iteration is written in.  There are two iterates: x, the one being formed, and x_best, the one
// kept (the output).  At the start both are x0.  Results of dots and norm2 go to slots on the implementation's side and
// are read back together by fetch(), so that an implementation may queue a whole Arnoldi step and wait once.  Slots:
// h0, h1 (m + 1 values each) for the two Gram-Schmidt passes, s0 .. s3 for squared norms.  Every call returns 0 or a
// nonzero error code that the iteration passes on.
class KrylovOps {
 public:
  virtual ~KrylovOps() = default;
  virtual int residual() = 0;                         // w = r, the residual b - K x of the last analysis
  virtual int precondition(int j) = 0;                // z_j = K~^-1 v_j, column j of Z
  virtual int apply(int j) = 0;                       // w = K z_j
  virtual int dots(int j, int slot) = 0;              // h_slot[0, j) = V[:, 0, j)^T w
  virtual int update(int j, int slot) = 0;            // w -= V[:, 0, j) h_slot
  virtual int norm2(int slot) = 0;                    // s_slot = w^T w
  virtual int store(int j, int slot) = 0;             // v_j = w / sqrt(s_slot), or 0 when s_slot <= 0
  virtual int correct(int k, const double* y) = 0;    // x = x_best + Z[:, 0, k) y
  virtual int keep() = 0;                             // x_best = x, with the analysis of x
  virtual int analyse(double omega[2]) = 0;           // waits; omega = omega1, omega2 of x; keeps x's residual
  virtual int fetch(int j, double* h0, double* h1, double s[4]) = 0;   // waits; h0, h1 = j values of the slots
};

struct KrylovResult {
  uint32_t iterations = 0;     // Arnoldi steps (each one preconditioner solve and one product with K)
  uint32_t cycles = 0;
  uint32_t analyses = 0;       // x0's included
  uint32_t breakdowns = 0;     // cycles ended by h_{j+1,j} <= 2^-40 ||K z_j||_2
  double omega1 = 0.0, omega2 = 0.0;   // of x_best
  std::vector<double> estimates;       // per corrected cycle: its Givens estimate |g_k| of ||b - K x||_2 at its end
};

// FGMRES(m) from x0 (already x and x_best; its analysis is the first operation).  A cycle starts from the residual of
// the last analysis and ends after m steps, at max_iter steps in all, at a breakdown, at a non-finite value (that step
// is not used) or when |g_{j+1}| <= (tol / omega_c) beta, omega_c = omega1 + omega2 at its start; then y solves the
// least-squares problem and x = x_best + Z y is analysed, kept when its omega1 + omega2 is smaller.  The call stops at
// omega1 + omega2 <= tol, after max_iter steps, at a non-finite omega, or when a cycle did not lower omega1 + omega2
// below omega_c.  1 <= m <= KRYLOV_MAX_RESTART, max_iter >= 0, tol >= 0.  Returns 0 or the first error code of an
// operation.
int fgmres_run(KrylovOps& ops, int m, int max_iter, double tol, KrylovResult& out);

}  // namespace cb
