// Thick-restart Lanczos (Wu and Simon 2000) for the eigenvalues of largest magnitude of an operator T that is
// self-adjoint in the inner product <x, y>_M = x^T M y, M positive definite.  cldl_eigsh runs it on
// T = (A - sigma M)^-1 M.  Host-only code: the iteration is written against EigOps, a small set of operations on an
// n x (ncv + 1) basis V and a work vector w, so that it runs unchanged on the GPU (LDLObject::eigsh, ldl_eig.cuh) and on
// dense matrices in a CPU test.
#pragma once
#include <cstdint>
#include <vector>

namespace cb {

constexpr int EIG_MAX_NCV = 512;

// The operations the iteration is written in.  Results of mdots and mnorm2 go to slots on the implementation's side and
// are read back together by fetch(), so that an implementation may queue a whole Lanczos step and wait once.  Slots:
// h0, h1 (ncv + 1 values each) for the two Gram-Schmidt passes, s0, s1, s2 for squared norms.  Every call returns 0 or
// a nonzero error code that the iteration passes on.
class EigOps {
 public:
  virtual ~EigOps() = default;
  virtual int apply(int j) = 0;                       // w = T v_j
  virtual int random(uint64_t draw) = 0;              // w = the draw-th random vector of the seed
  virtual int mdots(int j, int slot) = 0;             // h_slot[0, j) = V[:, 0, j)^T M w
  virtual int update(int j, int slot) = 0;            // w -= V[:, 0, j) h_slot
  virtual int mnorm2(int slot) = 0;                   // s_slot = w^T M w
  virtual int store(int j, int slot) = 0;             // v_j = w / sqrt(s_slot), or 0 when s_slot <= 0
  virtual int combine(int m, int k, const double* S) = 0;   // V[:, 0, k) = V[:, 0, m) S, S m x k column-major
  virtual int copy(int dst, int src) = 0;             // v_dst = v_src
  virtual int fetch(int j, double out[5]) = 0;        // waits; out = h0[j], h1[j], s0, s1, s2
};

struct EigResult {
  int status = 0;              // 1 all nev converged, 0 not within max_restarts (or a non-finite value), -1 M-norm <= 0
  int nconv = 0;               // converged among the returned pairs (they come first)
  int restarts = 0;
  uint32_t applies = 0;        // products with T
  uint32_t deflations = 0;     // invariant subspaces met (beta = 0, a fresh random vector)
  std::vector<double> theta;   // nev Ritz values of T: converged first, each group in ascending 1/theta
};

// Symmetric eigensolve of the m x m matrix A (row-major, overwritten) by cyclic Jacobi: rotations in row order (p < q),
// each one taken when |a_pq| > eps sqrt(|a_pp a_qq|), sweeps until one takes none (or 100 sweeps).  theta[i] = the
// eigenvalues (A's diagonal at the end), Y (row-major m x m) the eigenvectors in its columns.  Deterministic.
void eig_jacobi(int m, std::vector<double>& A, std::vector<double>& theta, std::vector<double>& Y);

// The nev eigenvalues of largest |theta| of T on an n-dimensional space, with an ncv-column basis (nev < ncv <= n,
// ncv <= EIG_MAX_NCV).  Convergence: |beta_m y_{m-1,i}| <= tol |theta_i| (ARPACK's test), tol 0 = machine eps.
// m_identity: the norms are Euclidean (a norm^2 < 0 cannot come from M then).  On return with status 0 or 1 the first
// nev columns of V hold the Ritz vectors of out.theta, in its order.  Returns 0 or the first error code of an operation.
int lanczos_run(EigOps& ops, int n, int nev, int ncv, int max_restarts, double tol, bool m_identity, EigResult& out);

}  // namespace cb
