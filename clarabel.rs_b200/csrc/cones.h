// Device cone engine (internal header): Zero / Nonnegative / second-order / PSD-triangle cones and the
// nonsymmetric exponential and 3-D power cones.
//
// Device counterpart of the reference's `Cone` trait and CompositeCone dispatch
// (/root/reference/src/solver/core/cones/mod.rs:42-154, compositecone.rs:197-352).
// The reference loops over cones sequentially on one thread; here every
// operation is one batched launch per cone *class*: an elementwise kernel over
// all rows (row tags select Zero / Nonnegative semantics) plus one CTA per
// second-order cone with block reductions for its dot products and norms.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "problem_setup.h"
#include "vec.cuh"

namespace cb {

enum { SCALING_PRIMAL_DUAL = 0, SCALING_DUAL = 1 };   // ScalingStrategy (cones/mod.rs)

struct ConeDev {
  int ncones = 0, m = 0, nsoc = 0;
  const int* type = nullptr;
  const int* off = nullptr;
  const int* dim = nullptr;
  const int* boff = nullptr;     // offset of the cone's Hs block
  const int* sparse = nullptr;   // 1 if sparse-expanded SOC
  const int* soc_list = nullptr; // cone ids of the SOC cones
  const signed char* rowtag = nullptr;  // [m] cone type of every row
  double* w = nullptr;    // [m]
  double* lam = nullptr;  // [m]
  double* eta = nullptr;  // [ncones]
  double* u = nullptr;    // [m] sparse SOC data
  double* v = nullptr;    // [m]
  double* dd = nullptr;   // [ncones]
  int* fail = nullptr;    // scaling failure flag
  // PSD triangle cones (matrix dimension <= CB_PSD_MAX_N)
  int npsd = 0;
  const int* psd_list = nullptr;   // cone ids
  const int* psd_n = nullptr;      // [ncones] matrix dimension (0 for other cones)
  const long long* psd_moff = nullptr;  // [ncones] offset into the n x n matrix arenas
  double *psd_R = nullptr, *psd_Rinv = nullptr, *psd_RRt = nullptr;
  double* psd_ws = nullptr;        // global scratch (8 matrices per cone) when the matrices do not fit shared memory
  double* psd_bar = nullptr;       // one matrix per cone for the barrier's Cholesky
  // exponential / 3-D power cones (cones_nonsym.cu): state in structure-of-arrays form, component j of the
  // k-th nonsymmetric cone at [j*nns + k]
  int nns = 0;
  const int* ns_list = nullptr;      // cone ids
  const double* ns_alpha = nullptr;  // [nns] exponent of a power cone
  double *ns_Hd = nullptr, *ns_Hs = nullptr;     // [6*nns] dual Hessian, scaling block (packed triu)
  double *ns_grad = nullptr, *ns_z = nullptr;    // [3*nns] dual gradient, z at the scaling point
  int* ns_jmax = nullptr;            // backtracking count of the composite step length
  // generalised power cones (cones_nonsym.cu): per-row state in m-length arrays (q in a cone's first dim1 rows of
  // gp_qr, r in the rest), per-cone scalars in [ngp] arrays
  int ngp = 0;
  const int* gp_list = nullptr;      // cone ids
  const int* gp_dim1 = nullptr;      // [ngp]
  const double* gp_alpha = nullptr;  // [m]
  const double* gp_psi = nullptr;    // [ngp]
  double *gp_grad = nullptr, *gp_p = nullptr, *gp_qr = nullptr, *gp_d1 = nullptr, *gp_zc = nullptr;   // [m]
  double *gp_d2 = nullptr, *gp_mu = nullptr;                                                            // [ngp]
};

// the device half of a cone layout
class ConeSet : public ConeLayout {
 public:
  DevOwner own;       // every buffer behind dev, ws and the scratch below
  ConeDev dev;
  cudaStream_t stream = nullptr;
  ReduceWS ws;
  const int* row2blk_dev = nullptr;  // row -> slot in the flat Hs vector (diagonal-block cones)
  double* d_pmin = nullptr;
  double* d_psum = nullptr;

  int init(const ConeLayout& layout, cudaStream_t st);   // uploads the layout

  void set_identity_scaling();
  // failure -> dev.fail; mu and the scaling strategy only matter to the nonsymmetric cones
  void update_scaling(const double* s, const double* z, double mu = 0.0, int strategy = SCALING_PRIMAL_DUAL);
  void get_Hs(double* Hs, bool negate);
  void mul_Hs(double* y, const double* x);
  void affine_ds(double* ds, const double* s = nullptr);   // s: current iterate, read by the nonsymmetric cones
  void combined_ds_shift(double* shift, double* step_z, double* step_s, double sigmamu);
  void ds_from_dz_offset(double* out, const double* ds, const double* z);
  // alpha slot must be pre-set to alpha_max by the caller (device double)
  void step_length(const double* dz, const double* ds, const double* z, const double* s, double* alpha_slot);
  // out2[0] = min margin, out2[1] = sum of positive margins
  void margins(const double* z, double* out2);
  void scaled_unit_shift(double* z, double alpha, bool primal);

  // nonsymmetric pieces (cones_nonsym.cu)
  int gp_prepare();
  // the three KKT columns + diagonal entries of every generalised power cone (datamaps.rs:314-337)
  void gp_kkt_fill(double* vals, const int* map_qr, const int* map_p, const int* map_D);
  double ns_amin = 1e-4, ns_step = 0.8;   // min_terminate_step_length, linesearch_backtrack_step
  int ns_prepare(const std::vector<double>& alpha_per_cone);
  void unit_initialization(double* z, double* s);
  void ns_update_scaling(const double* s, const double* z, double mu, int strategy);
  void ns_get_Hs(double* Hs, double sign);
  void ns_mul_Hs(double* y, const double* x);
  void ns_copy_rows(double* out, const double* in);
  void ns_combined_shift(double* shift, const double* step_z, const double* step_s, double sigmamu);
  void ns_step_length(const double* dz, const double* ds, const double* z, const double* s, double* alpha_slot);
  // out[0] = sum of the cones' barrier functions at (z + alpha dz, s + alpha ds); partial = 5 doubles of scratch
  void compute_barrier(const double* z, const double* s, const double* dz, const double* ds, double alpha,
                       double* partial, double* out);

  // PSD pieces (cones_psd.cu)
  int psd_nmax = 0, psd_numel_max = 0, psd_warps = 4;
  long long psd_mat_total = 0;     // sum of n^2 over the PSD cones
  int psd_prepare();
  void psd_set_identity();
  void psd_update_scaling(const double* s, const double* z);
  void psd_get_Hs(double* Hs, double sign);
  void psd_apply(int op, double* out, double* a, double* b, double scalar);
  void psd_step_length(const double* dz, const double* ds, double* alpha_slot);
  void psd_margins(const double* z, double* pmin, double* psum);
};

}  // namespace cb
