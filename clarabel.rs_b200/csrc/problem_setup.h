// Set-up of the interior-point solver on the host: the input checks, cone collapsing and the cone layout, the inf-bound
// presolve and its reverse, Ruiz equilibration, the KKT assembly and the sparse transposes the device solver reads.
// Host-only code: no CUDA runtime, so the set-up can be built and checked without a device.
//
// What it replaces in the reference (all file:line under /root/reference/src):
//   check_csc            algebra/csc/core.rs (CscMatrix::check_format)
//   collapse_cones       solver/core/cones/supportedcone.rs:105-161
//   presolve             solver/implementations/default/presolver.rs:75-125, 157-204, problemdata.rs:86-93, 130-131
//   equilibrate          solver/implementations/default/problemdata.rs:229-312
//   assemble_kkt         solver/core/kktsolvers/direct/quasidef/kkt_assembly.rs:20-183, datamaps.rs:112-221, 350-405
#pragma once
#include <cstdint>
#include <vector>

#include "../../include/clarabel_b200.h"

namespace cb {

enum { CT_ZERO = 0, CT_NONNEG = 1, CT_SOC = 2, CT_PSD = 3, CT_EXP = 4, CT_POW = 5, CT_GENPOW = 6 };
constexpr int SOC_NO_EXPANSION_MAX_SIZE = 4;  // socone.rs:46
constexpr int CB_PSD_MAX_N = 128;             // Hs block of one cone: tri(tri(128)) = 3.4e7 entries

// dim = number of rows the cone occupies (numel); psd_n = matrix dimension of a PSD cone
// param: exponent of a power cone; alphas: exponents of a generalised power cone (dim = alphas.size() + dim2)
struct ConeSpec { int type; int dim; int psd_n = 0; double param = 0.0; std::vector<double> alphas; };

struct HostCsc {
  int m = 0, n = 0;
  std::vector<int64_t> colptr;
  std::vector<int> rowval;
  std::vector<double> nzval;
};

// A caller's CSC arrays as CscMatrix::check_format sees them: column pointers start at 0 and never decrease, row indices
// are below `rows` and strictly increasing inside a column (sorted, no duplicates), and with triu no entry lies below
// the diagonal.  The assembly relies on it (the diagonal of a P column is its LAST entry, kkt_assembly.rs:20-60) and
// the equilibration indexes vectors by row: an unchecked caller would get a silently wrong KKT matrix or a write out
// of bounds.  Returns 0, CLDL_E_ARG, CLDL_E_DIM (row out of range) or CLDL_E_NOT_TRIU.
int check_csc(const uint64_t* colptr, const uint64_t* rowval, uint64_t rows, int cols, bool triu);
// a copy of checked CSC arrays
HostCsc host_csc(int m, int n, const uint64_t* colptr, const uint64_t* rowval, const double* nzval);

// collapse like SupportedConeT::new_collapsed; CLDL_E_ARG on an unknown type or invalid dimension / exponent
int collapse_cones(const int32_t* types, const uint64_t* dims, uint64_t n, std::vector<ConeSpec>& out,
                   const double* params = nullptr, const uint64_t* gp_dim2 = nullptr, const double* gp_alpha = nullptr);

// b capped at the infinity bound and, when enabled, the inf-bound presolve: the rows of nonnegative cones whose bound is
// beyond it (b was capped at it, which still compares as beyond) leave A, b and their cone.  keep is the mask over the
// caller's rows, left empty when no row is dropped.  CLDL_E_DIM when the cones do not cover A's rows.
int presolve(std::vector<ConeSpec>& cones, HostCsc& A, std::vector<double>& b, double infbound, bool enable,
             std::vector<char>& keep);

// Where every cone sits in the rows, in the flat Hs vector and in the KKT matrix: computed once from the collapsed
// (and presolved) cone list; the device cone set uploads it and the KKT assembly reads it.
struct ConeLayout {
  std::vector<ConeSpec> cones;
  std::vector<int> off, boff;      // [cone] first row, first entry of the Hs block
  std::vector<int> sparse_flag;    // [cone] 1: second-order cone in sparse expanded form
  std::vector<char> diag_block;    // [cone] 1: diagonal Hs block of dim entries, 0: packed upper triangle
  std::vector<int> pdim;           // [cone] expansion columns of the KKT matrix (2 sparse SOC, 3 GenPow, else 0)
  std::vector<int> soc_list, psd_list, ns_list, gp_list;   // cone ids per class (ns: exponential and 3-D power)
  int m = 0, nHs = 0, degree = 0, p = 0;   // p = expansion columns in all
  bool all_symmetric = true;
  bool allows_primal_dual = true;  // false as soon as a generalised power cone is present (genpowcone.rs:108-110)
};
// CLDL_E_ARG when the Hs vector would not be indexable by int
int cone_layout(const std::vector<ConeSpec>& cones, ConeLayout& L);

// The caller's KKT permutation (kkt_dim = n + m + L.p entries) as int
std::vector<int> kkt_perm(const uint64_t* perm, int n, int m, const ConeLayout& L);

// Ruiz scaling: P <- c D P D, A <- E A D, q <- c D q, b <- E b
struct Equilibration {
  std::vector<double> d, dinv, e, einv;
  double c = 1.0;
  // new values on the stored patterns, scaled like the set-up data (data_updating.rs:68-163)
  void scale_P(HostCsc& P, const double* v) const;
  void scale_A(HostCsc& A, const double* v) const;
  double scale_q(std::vector<double>& q, const double* v) const;   // -> ||q||_inf of the caller's q
  double scale_b(std::vector<double>& b, const double* v) const;   // -> ||b||_inf of the caller's b
};
// Ruiz equilibration of P, A, q and b in place (problemdata.rs:229-312)
Equilibration equilibrate(HostCsc& P, HostCsc& A, std::vector<double>& q, std::vector<double>& b, const ConeLayout& L,
                          const cipm_settings& s);

// The solution in the caller's coordinates from the device iterate (variables.rs:262-285, solution.rs:68-111),
// x = D x̂ / t, z = E ẑ / (c t), s = E⁻¹ ŝ / t with t = 1 / scaleinv, and the reverse presolve (presolver.rs:127-150):
// rows the presolve dropped get s = infbound and z = 0.  z and s have one entry per caller row.
void unscale_solution(const Equilibration& eq, const std::vector<char>& keep, double infbound, double scaleinv, int n,
                      int mfull, const double* hx, const double* hz, const double* hs, double* x, double* z, double* s);

// A CSR form of a CSC matrix: row pointers, columns, and src[k] = position of the k-th entry's value in the CSC arrays
struct CsrMap { std::vector<int> rowptr, col, src; };
CsrMap csc_to_csr(const HostCsc& M);
// the full symmetric CSR of an upper-triangular CSC matrix (P, the KKT matrix): an off-diagonal entry appears twice,
// at (i, j) and at (j, i), both with the same src
CsrMap triu_to_sym_csr(int n, const int64_t* colptr, const int* rowval);
// v[idx[k]] for every k
std::vector<double> gather(const std::vector<double>& v, const std::vector<int>& idx);

// The KKT matrix's upper triangle and where every value comes from.  Layout contract (SURVEY 8a): cols 0..n = triu(P) +
// structural diagonal; cols n..n+m = A' block then the cone's Hs entries; cols n+m.. = expansion columns (sparse SOC: v
// first, u second; GenPow: q|r, p) then their diagonal entries.  The diagonal is the last entry of every column.
struct KKTAssembly {
  int N = 0;
  int64_t nnzK = 0;
  std::vector<int64_t> Kp;
  std::vector<int> Ki;
  std::vector<int8_t> dsigns;
  std::vector<int> map_P, map_A, map_Hs, map_u, map_v, map_D, map_diag;
  std::vector<int> map_gqr, map_gp, map_gD;   // generalised power cones: q|r rows, p rows (by row), 3 diagonals per cone
  // dense cone blocks (PSD, dense SOC of more than 8 rows): group of every column for order_with_groups, or -1
  std::vector<int> group;
  int ngroups = 0;
};
// from the patterns of P (upper triangle) and A; CLDL_E_DIM when K has more entries than an int indexes
int assemble_kkt(const HostCsc& P, const HostCsc& A, const ConeLayout& L, KKTAssembly& K);

}  // namespace cb
