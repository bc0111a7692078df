// Exponential and 3-D power cone kernels (sm_90a): one thread per cone.  See cones_nonsym.cuh for the per-cone
// arithmetic and the reference map, cones.h for the cone engine these methods belong to.
//
// Layout: cone k of the nns nonsymmetric cones owns rows off[id]..off[id]+2 of the m-vectors and entries
// boff[id]..boff[id]+5 of the flat Hs vector (packed upper triangle, the KKT block order of
// kkt_assembly.rs:107-183).  Per-cone state (dual Hessian, Hs, dual gradient, scaling-point z) is kept in
// structure-of-arrays form, component j of cone k at [j*nns + k]: thread k and thread k+1 touch adjacent doubles.
//
// The composite step length (compositecone.rs:289-332) threads one running alpha through the cones in order;
// every cone shortens it by whole multiples of the backtracking factor, so the result is alpha0 * step^J with
// J the largest per-cone count: cones count independently, an integer atomicMax combines them (order
// independent, hence reproducible), and one thread rebuilds alpha with the same sequence of multiplications.
#include "cones.h"
#include "cones_nonsym.cuh"

#include <cstdio>

namespace cb {

using ns3::Sym3;

namespace {

__host__ __device__ inline ns3::View view(const ConeDev& c) {
  return ns3::View{c.nns, c.ns_list, c.type, c.off, c.boff, c.ns_alpha, c.ns_Hd, c.ns_Hs, c.ns_grad, c.ns_z};
}
#define NS_THREAD                                            \
  const int k = blockIdx.x * blockDim.x + threadIdx.x;       \
  if (k >= c.nns) return;                                    \
  const ns3::View v = view(c);

__global__ void k_ns_unit_init(ConeDev c, double* __restrict__ z, double* __restrict__ s) {
  NS_THREAD
  ns3::body_unit_init(v, k, z, s);
}
__global__ void k_ns_update_scaling(ConeDev c, const double* __restrict__ s, const double* __restrict__ z, double mu,
                                    int strategy) {
  NS_THREAD
  ns3::body_update_scaling(v, k, s, z, mu, strategy);
}
__global__ void k_ns_get_Hs(ConeDev c, double* __restrict__ Hs, double sign) {
  NS_THREAD
  ns3::body_get_Hs(v, k, Hs, sign);
}
__global__ void k_ns_mul_Hs(ConeDev c, double* __restrict__ y, const double* __restrict__ x) {
  NS_THREAD
  ns3::body_mul_Hs(v, k, y, x);
}
__global__ void k_ns_copy_rows(ConeDev c, double* __restrict__ out, const double* __restrict__ in) {
  NS_THREAD
  ns3::body_copy_rows(v, k, out, in);
}
__global__ void k_ns_combined_shift(ConeDev c, double* __restrict__ shift, const double* __restrict__ step_z,
                                    const double* __restrict__ step_s, double sigmamu) {
  NS_THREAD
  ns3::body_combined_shift(v, k, shift, step_z, step_s, sigmamu);
}
// *alpha is the step the symmetric cones allow; the largest backtracking count goes to *jmax
__global__ void k_ns_step_count(ConeDev c, const double* __restrict__ dz, const double* __restrict__ ds,
                                const double* __restrict__ z, const double* __restrict__ s,
                                const double* __restrict__ alpha, double a_min, double step, int* jmax) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  int j = 0;
  if (k < c.nns) j = ns3::body_step_count(view(c), k, dz, ds, z, s, *alpha, a_min, step);
  __syncwarp();
  for (int o = 16; o > 0; o >>= 1) { const int t = __shfl_xor_sync(0xffffffffu, j, o); j = t > j ? t : j; }
  if ((threadIdx.x & 31) == 0 && j > 0) atomicMax(jmax, j);
}
// ---- generalised power cones: thread k = cone k, loops over the cone's rows ----
__host__ __device__ inline gp::View gview(const ConeDev& c) {
  return gp::View{c.ngp, c.gp_list, c.off, c.dim, c.boff, c.gp_dim1, c.gp_alpha, c.gp_psi,
                  c.gp_grad, c.gp_p, c.gp_qr, c.gp_d1, c.gp_zc, c.gp_d2, c.gp_mu};
}
#define GP_THREAD                                            \
  const int k = blockIdx.x * blockDim.x + threadIdx.x;       \
  if (k >= c.ngp) return;                                    \
  const gp::View v = gview(c);

__global__ void k_gp_unit_init(ConeDev c, double* __restrict__ z, double* __restrict__ s) {
  GP_THREAD
  gp::body_unit_init(v, k, z, s);
}
__global__ void k_gp_update_scaling(ConeDev c, const double* __restrict__ z, double mu) {
  GP_THREAD
  if (!gp::body_update_scaling(v, k, z, mu)) atomicExch(c.fail, 1);
}
__global__ void k_gp_get_Hs(ConeDev c, double* __restrict__ Hs, double sign) {
  GP_THREAD
  gp::body_get_Hs(v, k, Hs, sign);
}
__global__ void k_gp_mul_Hs(ConeDev c, double* __restrict__ y, const double* __restrict__ x) {
  GP_THREAD
  gp::body_mul_Hs(v, k, y, x);
}
__global__ void k_gp_copy_rows(ConeDev c, double* __restrict__ out, const double* __restrict__ in) {
  GP_THREAD
  gp::body_copy_rows(v, k, out, in);
}
__global__ void k_gp_combined_shift(ConeDev c, double* __restrict__ shift, double sigmamu) {
  GP_THREAD
  gp::body_combined_shift(v, k, shift, sigmamu);
}
__global__ void k_gp_kkt_fill(ConeDev c, double* __restrict__ vals, const int* __restrict__ map_qr,
                              const int* __restrict__ map_p, const int* __restrict__ map_D) {
  GP_THREAD
  gp::body_kkt_fill(v, k, vals, map_qr, map_p, map_D);
}
__global__ void k_gp_step_count(ConeDev c, const double* __restrict__ dz, const double* __restrict__ ds,
                                const double* __restrict__ z, const double* __restrict__ s,
                                const double* __restrict__ alpha, double a_min, double step, int* jmax) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  int j = 0;
  if (k < c.ngp) j = gp::body_step_count(gview(c), k, dz, ds, z, s, *alpha, a_min, step);
  __syncwarp();
  for (int o = 16; o > 0; o >>= 1) { const int t = __shfl_xor_sync(0xffffffffu, j, o); j = t > j ? t : j; }
  if ((threadIdx.x & 31) == 0 && j > 0) atomicMax(jmax, j);
}

__global__ void k_ns_step_final(double* alpha, int* jmax, double step) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    *alpha = ns3::body_step_final(*alpha, *jmax, step);
    *jmax = 0;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------- host side
#define NCK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { std::fprintf(stderr, "[clarabel_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return -20; } } while (0)
#define NS_GRID ((dev.nns + 127) / 128)

int ConeSet::ns_prepare(const std::vector<double>& alpha_per_cone) {
  dev.nns = (int)ns_list.size();
  if (dev.nns == 0) return 0;
  std::vector<double> al(ns_list.size());
  for (size_t k = 0; k < ns_list.size(); k++) al[k] = alpha_per_cone[ns_list[k]];
  NCK(own.upload(&dev.ns_list, ns_list));
  NCK(own.upload(&dev.ns_alpha, al));
  const size_t n = ns_list.size();
  NCK(own.alloc(&dev.ns_Hd, 6 * n)); NCK(own.alloc(&dev.ns_Hs, 6 * n));
  NCK(own.alloc(&dev.ns_grad, 3 * n)); NCK(own.alloc(&dev.ns_z, 3 * n));
  NCK(cudaMemset(dev.ns_Hd, 0, 6 * n * 8)); NCK(cudaMemset(dev.ns_Hs, 0, 6 * n * 8));
  NCK(cudaMemset(dev.ns_grad, 0, 3 * n * 8)); NCK(cudaMemset(dev.ns_z, 0, 3 * n * 8));
  NCK(own.alloc(&dev.ns_jmax, 1));
  NCK(cudaMemset(dev.ns_jmax, 0, sizeof(int)));
  return 0;
}
#define GP_GRID ((dev.ngp + 127) / 128)
int ConeSet::gp_prepare() {
  dev.ngp = (int)gp_list.size();
  if (dev.ngp == 0) return 0;
  const size_t n = gp_list.size(), mm = (size_t)(m ? m : 1);
  std::vector<int> d1(n);
  std::vector<double> psi(n), al(mm, 0.0);
  for (size_t k = 0; k < n; k++) {
    const ConeSpec& c = cones[gp_list[k]];
    d1[k] = (int)c.alphas.size();
    double sq = 0.0;
    for (size_t i = 0; i < c.alphas.size(); i++) { al[off[gp_list[k]] + i] = c.alphas[i]; sq += c.alphas[i] * c.alphas[i]; }
    psi[k] = 1.0 / sq;                       // genpowcone.rs:56
  }
  NCK(own.upload(&dev.gp_list, gp_list)); NCK(own.upload(&dev.gp_dim1, d1));
  NCK(own.upload(&dev.gp_alpha, al)); NCK(own.upload(&dev.gp_psi, psi));
  for (double** q : {&dev.gp_grad, &dev.gp_p, &dev.gp_qr, &dev.gp_d1, &dev.gp_zc}) {
    NCK(own.alloc(q, mm)); NCK(cudaMemset(*q, 0, mm * 8));
  }
  for (double** q : {&dev.gp_d2, &dev.gp_mu}) { NCK(own.alloc(q, n)); NCK(cudaMemset(*q, 0, n * 8)); }
  if (!dev.ns_jmax) { NCK(own.alloc(&dev.ns_jmax, 1)); NCK(cudaMemset(dev.ns_jmax, 0, sizeof(int))); }
  return 0;
}
void ConeSet::gp_kkt_fill(double* vals, const int* map_qr, const int* map_p, const int* map_D) {
  if (!dev.ngp) return;
  g_launches++;
  k_gp_kkt_fill<<<GP_GRID, 128, 0, stream>>>(dev, vals, map_qr, map_p, map_D);
}

// Cone::unit_initialization of the whole composite cone (compositecone.rs:217-221): zero everything, add the
// unit element of every symmetric cone (e for NN / SOC / PSD, nothing for the zero cone), set the nonsymmetric ones
void ConeSet::unit_initialization(double* z, double* s) {
  if (m == 0) return;
  cudaMemsetAsync(z, 0, (size_t)m * 8, stream);
  cudaMemsetAsync(s, 0, (size_t)m * 8, stream);
  scaled_unit_shift(s, 1.0, true);
  scaled_unit_shift(z, 1.0, false);
  if (dev.nns) { g_launches++; k_ns_unit_init<<<NS_GRID, 128, 0, stream>>>(dev, z, s); }
  if (dev.ngp) { g_launches++; k_gp_unit_init<<<GP_GRID, 128, 0, stream>>>(dev, z, s); }
}
void ConeSet::ns_update_scaling(const double* s, const double* z, double mu, int strategy) {
  if (dev.nns) { g_launches++; k_ns_update_scaling<<<NS_GRID, 128, 0, stream>>>(dev, s, z, mu, strategy); }
  if (dev.ngp) { g_launches++; k_gp_update_scaling<<<GP_GRID, 128, 0, stream>>>(dev, z, mu); }
}
void ConeSet::ns_get_Hs(double* Hs, double sign) {
  if (dev.nns) { g_launches++; k_ns_get_Hs<<<NS_GRID, 128, 0, stream>>>(dev, Hs, sign); }
  if (dev.ngp) { g_launches++; k_gp_get_Hs<<<GP_GRID, 128, 0, stream>>>(dev, Hs, sign); }
}
void ConeSet::ns_mul_Hs(double* y, const double* x) {
  if (dev.nns) { g_launches++; k_ns_mul_Hs<<<NS_GRID, 128, 0, stream>>>(dev, y, x); }
  if (dev.ngp) { g_launches++; k_gp_mul_Hs<<<GP_GRID, 128, 0, stream>>>(dev, y, x); }
}
void ConeSet::ns_copy_rows(double* out, const double* in) {
  if (dev.nns) { g_launches++; k_ns_copy_rows<<<NS_GRID, 128, 0, stream>>>(dev, out, in); }
  if (dev.ngp) { g_launches++; k_gp_copy_rows<<<GP_GRID, 128, 0, stream>>>(dev, out, in); }
}
void ConeSet::ns_combined_shift(double* shift, const double* step_z, const double* step_s, double sigmamu) {
  if (dev.nns) { g_launches++; k_ns_combined_shift<<<NS_GRID, 128, 0, stream>>>(dev, shift, step_z, step_s, sigmamu); }
  if (dev.ngp) { g_launches++; k_gp_combined_shift<<<GP_GRID, 128, 0, stream>>>(dev, shift, sigmamu); }
}
void ConeSet::ns_step_length(const double* dz, const double* ds, const double* z, const double* s, double* alpha_slot) {
  if (!dev.nns && !dev.ngp) return;
  if (dev.nns) { g_launches++; k_ns_step_count<<<NS_GRID, 128, 0, stream>>>(dev, dz, ds, z, s, alpha_slot, ns_amin, ns_step, dev.ns_jmax); }
  if (dev.ngp) { g_launches++; k_gp_step_count<<<GP_GRID, 128, 0, stream>>>(dev, dz, ds, z, s, alpha_slot, ns_amin, ns_step, dev.ns_jmax); }
  g_launches++;
  k_ns_step_final<<<1, 32, 0, stream>>>(alpha_slot, dev.ns_jmax, ns_step);
}

// Cone::compute_barrier summed over all cones (compositecone.rs:334-345) into out[0]; deterministic two-level
// sums per cone class.  partial = 4 device doubles of scratch.
void ConeSet::compute_barrier(const double* z, const double* s, const double* dz, const double* ds, double alpha,
                              double* partial, double* out) {
  const ConeDev c = dev;
  cudaMemsetAsync(partial, 0, 5 * 8, stream);
  if (m) {
    g_launches++;
    k_sum<<<red_grid(m), RED_THREADS, 0, stream>>>(m, [=] __device__(int i) {
      if (c.rowtag[i] != CT_NONNEG) return 0.0;
      return -ns3::lsafe((s[i] + alpha * ds[i]) * (z[i] + alpha * dz[i]));     // nonnegativecone.rs:155-166
    }, ws, partial + 0);
  }
  if (c.nsoc) {
    g_launches++;
    k_sum<<<red_grid(c.nsoc), RED_THREADS, 0, stream>>>(c.nsoc, [=] __device__(int k) {
      const int id = c.soc_list[k], o = c.off[id];
      return ns3::soc_barrier(z + o, s + o, dz + o, ds + o, c.dim[id], alpha);
    }, ws, partial + 1);
  }
  if (c.npsd) {
    g_launches++;
    k_sum<<<red_grid(c.npsd), RED_THREADS, 0, stream>>>(c.npsd, [=] __device__(int k) {
      const int id = c.psd_list[k], o = c.off[id], n = c.psd_n[id];
      double* W = c.psd_bar + c.psd_moff[id];
      return ns3::psd_neg_logdet(z + o, dz + o, n, alpha, W) + ns3::psd_neg_logdet(s + o, ds + o, n, alpha, W);
    }, ws, partial + 2);
  }
  if (c.nns) {
    g_launches++;
    const ns3::View v = view(c);
    k_sum<<<red_grid(c.nns), RED_THREADS, 0, stream>>>(c.nns, [=] __device__(int k) {
      return ns3::body_barrier(v, k, z, s, dz, ds, alpha);
    }, ws, partial + 3);
  }
  if (c.ngp) {
    g_launches++;
    const gp::View v = gview(c);
    k_sum<<<red_grid(c.ngp), RED_THREADS, 0, stream>>>(c.ngp, [=] __device__(int k) {
      return gp::body_barrier(v, k, z, s, dz, ds, alpha);
    }, ws, partial + 4);
  }
  g_launches++;
  k_map<<<1, 32, 0, stream>>>(1, [=] __device__(int) {
    out[0] = (((partial[0] + partial[1]) + partial[2]) + partial[3]) + partial[4];
  });
}

}  // namespace cb
