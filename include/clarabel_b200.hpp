// clarabel_b200.hpp -- header-only C++ face of the C ABI in clarabel_b200.h, shaped like the reference's own types so
// that host code written against Clarabel.rs reads the same:
//
//   reference (Rust)                                               here
//   ---------------------------------------------------------------------------------------------------------------
//   trait DirectLDLSolver  (kktsolvers/direct/quasidef/mod.rs:14-26) cb200::DirectLDLSolver
//     update_values / scale_values / offset_values / solve / refactor   same names, same argument meaning
//   LinearSolverInfo       (kktsolvers/mod.rs:24-38)                 cb200::LinearSolverInfo (= cldl_info_t)
//   CscMatrix<T>           (algebra/csc/core.rs)                     cb200::CscMatrix (borrowed view: m, n, colptr, rowval, nzval)
//   SupportedConeT<T>      (cones/supportedcone.rs:17-52)            cb200::SupportedConeT + ZeroConeT(..) ... GenPowerConeT(..)
//   DefaultSettings<T>     (default/settings.rs)                     cb200::DefaultSettings (= cipm_settings, defaults filled)
//   DefaultSolver::new / solve / solution / info (default/solver.rs:57-126, core/solver.rs:242-465)
//                                                                    cb200::DefaultSolver
//   DefaultSolver::update_data (data_updating.rs:68-163)             DefaultSolver::update_data
//
// Errors: constructors throw cb200::SolverError (the reference returns Err(SolverError) / panics); methods that return
// bool in the reference return bool here.  Nothing in this header computes: every call goes to the CUDA library.
#pragma once
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "clarabel_b200.h"

namespace cb200 {

struct SolverError : std::runtime_error {
  int code;
  SolverError(const std::string& what, int c) : std::runtime_error(what + " (code " + std::to_string(c) + ")"), code(c) {}
};
inline void check(int rc, const char* what) { if (rc < 0) throw SolverError(what, rc); }

// borrowed CSC view with the reference's field names; indices are usize = uint64_t
struct CscMatrix {
  uint64_t m = 0, n = 0;
  const uint64_t* colptr = nullptr;
  const uint64_t* rowval = nullptr;
  const double* nzval = nullptr;
  uint64_t nnz() const { return colptr ? colptr[n] : 0; }
};

using LinearSolverInfo = cldl_info_t;

// ---------------------------------------------------------------------------------------------------- Level 1
class DirectLDLSolver {
 public:
  // ctor signature of ldlsolvers/config.rs:19-20: (KKT triu CSC, Dsigns, settings subset, optional permutation)
  DirectLDLSolver(const CscMatrix& kkt, const int8_t* dsigns, const cldl_opts* opts = nullptr,
                  const uint64_t* perm = nullptr) {
    check(cldl_create(&h_, kkt.n, kkt.colptr, kkt.rowval, kkt.nzval, dsigns, opts, perm), "cldl_create");
    n_ = kkt.n;
  }
  ~DirectLDLSolver() { if (h_) cldl_destroy(h_); }
  DirectLDLSolver(const DirectLDLSolver&) = delete;
  DirectLDLSolver& operator=(const DirectLDLSolver&) = delete;
  DirectLDLSolver(DirectLDLSolver&& o) noexcept : h_(o.h_), n_(o.n_) { o.h_ = nullptr; }

  void update_values(const uint64_t* index, const double* values, uint64_t len) { check(cldl_update_values(h_, index, values, len), "update_values"); }
  void scale_values(const uint64_t* index, uint64_t len, double scale) { check(cldl_scale_values(h_, index, len, scale), "scale_values"); }
  void offset_values(const uint64_t* index, uint64_t len, double offset, const int8_t* signs) { check(cldl_offset_values(h_, index, len, offset, signs), "offset_values"); }
  // x <- K^-1 b, b untouched (ldlsolvers/qdldl.rs:93-97)
  void solve(double* x, const double* b) { check(cldl_solve(h_, x, b), "solve"); }
  bool refactor() { const int rc = cldl_refactor(h_); check(rc, "refactor"); return rc == 1; }
  LinearSolverInfo linear_solver_info() const { LinearSolverInfo i; cldl_info(h_, &i); return i; }
  std::vector<uint64_t> perm() const { std::vector<uint64_t> p(n_); check(cldl_get_perm(h_, p.data()), "get_perm"); return p; }
  cldl_t* handle() { return h_; }

 private:
  cldl_t* h_ = nullptr;
  uint64_t n_ = 0;
};

// ---------------------------------------------------------------------------------------------------- cones
struct SupportedConeT {
  int32_t tag;                  // CIPM_CONE_*
  uint64_t dim;                 // rows (PSD: matrix dimension; GenPow: len(alpha))
  double alpha = 0.0;           // PowerConeT exponent
  std::vector<double> alphas;   // GenPowerConeT exponents
  uint64_t dim2 = 0;            // GenPowerConeT dim2
};
inline SupportedConeT ZeroConeT(uint64_t d) { return {CIPM_CONE_ZERO, d, 0.0, {}, 0}; }
inline SupportedConeT NonnegativeConeT(uint64_t d) { return {CIPM_CONE_NONNEG, d, 0.0, {}, 0}; }
inline SupportedConeT SecondOrderConeT(uint64_t d) { return {CIPM_CONE_SOC, d, 0.0, {}, 0}; }
inline SupportedConeT PSDTriangleConeT(uint64_t d) { return {CIPM_CONE_PSD, d, 0.0, {}, 0}; }
inline SupportedConeT ExponentialConeT() { return {CIPM_CONE_EXP, 3, 0.0, {}, 0}; }
inline SupportedConeT PowerConeT(double a) { return {CIPM_CONE_POW, 3, a, {}, 0}; }
inline SupportedConeT GenPowerConeT(std::vector<double> a, uint64_t dim2) {
  const uint64_t d = a.size();
  return {CIPM_CONE_GENPOW, d, 0.0, std::move(a), dim2};
}

struct DefaultSettings : cipm_settings {
  DefaultSettings() { cipm_default_settings(this); }
};

enum class SolverStatus : int32_t {
  Unsolved = CIPM_UNSOLVED, Solved = CIPM_SOLVED, PrimalInfeasible = CIPM_PRIMAL_INFEASIBLE,
  DualInfeasible = CIPM_DUAL_INFEASIBLE, AlmostSolved = CIPM_ALMOST_SOLVED,
  AlmostPrimalInfeasible = CIPM_ALMOST_PRIMAL_INFEASIBLE, AlmostDualInfeasible = CIPM_ALMOST_DUAL_INFEASIBLE,
  MaxIterations = CIPM_MAX_ITERATIONS, MaxTime = CIPM_MAX_TIME, NumericalError = CIPM_NUMERICAL_ERROR,
  InsufficientProgress = CIPM_INSUFFICIENT_PROGRESS, CallbackTerminated = CIPM_CALLBACK_TERMINATED
};

// DefaultSolution (default/solution.rs:12-40)
struct DefaultSolution {
  std::vector<double> x, z, s;
  SolverStatus status = SolverStatus::Unsolved;
  double obj_val = NAN, obj_val_dual = NAN;
  uint32_t iterations = 0;
  double r_prim = NAN, r_dual = NAN, solve_time = 0.0;
};

// ---------------------------------------------------------------------------------------------------- Level 2
class DefaultSolver {
 public:
  DefaultSolution solution;
  cipm_info info{};

  // DefaultSolver::new(P, q, A, b, cones, settings) (default/solver.rs:57-126); P upper triangular
  DefaultSolver(const CscMatrix& P, const double* q, const CscMatrix& A, const double* b,
                const std::vector<SupportedConeT>& cones, const DefaultSettings& settings = DefaultSettings(),
                const cldl_opts* ldl_opts = nullptr) {
    std::vector<int32_t> tags;
    std::vector<uint64_t> dims, dim2;
    std::vector<double> params, alphas;
    for (const auto& c : cones) {
      tags.push_back(c.tag); dims.push_back(c.dim); params.push_back(c.alpha); dim2.push_back(c.dim2);
      alphas.insert(alphas.end(), c.alphas.begin(), c.alphas.end());
    }
    if (alphas.empty()) alphas.push_back(0.0);
    // the part of check_dimensions (default/solver.rs:129-159) that can be seen through raw q / b pointers; the cone
    // sizes against A.m are checked by cipm_create_gp
    if (A.n != P.n) throw std::invalid_argument("A and q incompatible dimensions");
    if (P.m != P.n) throw std::invalid_argument("P not square");
    n_ = P.n; m_ = A.m;
    check(cipm_create_gp(&h_, P.n, A.m, P.colptr, P.rowval, P.nzval, q, A.colptr, A.rowval, A.nzval, b, cones.size(),
                         tags.data(), dims.data(), params.data(), dim2.data(), alphas.data(), &settings, ldl_opts, nullptr),
          "cipm_create_gp");
  }
  ~DefaultSolver() { if (h_) cipm_destroy(h_); }
  DefaultSolver(const DefaultSolver&) = delete;
  DefaultSolver& operator=(const DefaultSolver&) = delete;

  // IPSolver::solve (core/solver.rs:242-465) + solution post-processing (default/solution.rs:68-111)
  void solve() {
    check(cipm_solve(h_), "cipm_solve");
    cipm_get_info(h_, &info);
    solution.x.assign(n_, 0.0); solution.z.assign(m_, 0.0); solution.s.assign(m_, 0.0);
    check(cipm_get_solution(h_, solution.x.data(), solution.z.data(), solution.s.data()), "cipm_get_solution");
    solution.status = static_cast<SolverStatus>(info.status);
    const bool infeasible = info.status == CIPM_PRIMAL_INFEASIBLE || info.status == CIPM_DUAL_INFEASIBLE ||
                            info.status == CIPM_ALMOST_PRIMAL_INFEASIBLE || info.status == CIPM_ALMOST_DUAL_INFEASIBLE;
    solution.obj_val = infeasible ? NAN : info.cost_primal;
    solution.obj_val_dual = infeasible ? NAN : info.cost_dual;
    solution.iterations = info.iterations;
    solution.r_prim = info.res_primal; solution.r_dual = info.res_dual; solution.solve_time = info.solve_time;
  }
  // DefaultSolver::update_data (data_updating.rs:68-163): nullptr = unchanged; false = refused (presolved problem)
  bool update_data(const double* P_nzval, const double* q, const double* A_nzval, const double* b) {
    return cipm_update_data(h_, P_nzval, q, A_nzval, b) == 0;
  }
  // DefaultProblemData::equilibration (problemdata.rs:229-312): d [n], e [rows left after the presolve], c
  void equilibration(std::vector<double>& d, std::vector<double>& e, double& c) const {
    d.assign(n_, 0.0); e.assign(cipm_m_reduced(h_), 0.0);
    check(cipm_get_equilibration(h_, d.data(), e.data(), &c), "cipm_get_equilibration");
  }
  LinearSolverInfo linear_solver_info() const { LinearSolverInfo i; cipm_ldl_info(h_, &i); return i; }
  cipm_t* handle() { return h_; }

 private:
  cipm_t* h_ = nullptr;
  uint64_t n_ = 0, m_ = 0;
};

}  // namespace cb200
