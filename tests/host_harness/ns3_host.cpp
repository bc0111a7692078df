// TEST INFRASTRUCTURE ONLY -- never part of the product library.
//
// Compiles the per-cone thread bodies of clarabel.rs_b200/csrc/cones_nonsym.cuh with g++ and runs "thread k" for
// k = 0..n-1 in a loop, so that the CPU test-suite (tests/test_nonsym_host.py) can compare exactly the code the
// CUDA kernels of cones_nonsym.cu execute against the oracle without a GPU.  The kernels themselves only add the
// thread index, the warp/atomic max of the backtracking counts and the deterministic sums of vec.cuh.
#include <cstdint>
#include <vector>

#include "../../clarabel.rs_b200/csrc/cones_nonsym.cuh"

using namespace cb::ns3;

extern "C" {

struct ns3h {
  int ncones, m, nHs;
  std::vector<int> type, off, boff, dim, psd_n, list;
  std::vector<double> alpha, Hd, Hs, grad, zc;
  View v;
};

// types: 0 zero 1 nonneg 2 soc 3 psd 4 exp 5 pow; dims = rows of each cone (psd: matrix dimension)
ns3h* ns3h_new(int ncones, const int32_t* types, const int64_t* dims, const double* params) {
  ns3h* h = new ns3h();
  h->ncones = ncones; h->m = 0; h->nHs = 0;
  for (int k = 0; k < ncones; k++) {
    const int t = types[k];
    int rows = (int)dims[k];
    if (t == 3) { h->psd_n.push_back(rows); rows = rows * (rows + 1) / 2; } else h->psd_n.push_back(0);
    if (t == 4 || t == 5) rows = 3;
    const bool diag = t == 0 || t == 1 || (t == 2 && rows > 4);
    h->type.push_back(t); h->off.push_back(h->m); h->boff.push_back(h->nHs); h->dim.push_back(rows);
    h->m += rows; h->nHs += diag ? rows : rows * (rows + 1) / 2;
    if (t == 4 || t == 5) { h->list.push_back(k); h->alpha.push_back(params ? params[k] : 0.5); }
  }
  const size_t n = h->list.size();
  h->Hd.assign(6 * n, 0.0); h->Hs.assign(6 * n, 0.0); h->grad.assign(3 * n, 0.0); h->zc.assign(3 * n, 0.0);
  h->v = View{(int)n, h->list.data(), h->type.data(), h->off.data(), h->boff.data(), h->alpha.data(),
              h->Hd.data(), h->Hs.data(), h->grad.data(), h->zc.data()};
  return h;
}
void ns3h_free(ns3h* h) { delete h; }
int ns3h_m(const ns3h* h) { return h->m; }
int ns3h_nHs(const ns3h* h) { return h->nHs; }
int ns3h_n(const ns3h* h) { return h->v.n; }

void ns3h_unit_init(ns3h* h, double* z, double* s) { for (int k = 0; k < h->v.n; k++) body_unit_init(h->v, k, z, s); }
void ns3h_update_scaling(ns3h* h, const double* s, const double* z, double mu, int strategy) {
  for (int k = 0; k < h->v.n; k++) body_update_scaling(h->v, k, s, z, mu, strategy);
}
void ns3h_get_Hs(ns3h* h, double* Hs, double sign) { for (int k = 0; k < h->v.n; k++) body_get_Hs(h->v, k, Hs, sign); }
void ns3h_mul_Hs(ns3h* h, double* y, const double* x) { for (int k = 0; k < h->v.n; k++) body_mul_Hs(h->v, k, y, x); }
void ns3h_copy_rows(ns3h* h, double* out, const double* in) { for (int k = 0; k < h->v.n; k++) body_copy_rows(h->v, k, out, in); }
void ns3h_combined_shift(ns3h* h, double* shift, const double* step_z, const double* step_s, double sigmamu) {
  for (int k = 0; k < h->v.n; k++) body_combined_shift(h->v, k, shift, step_z, step_s, sigmamu);
}
// the composite step: max of the per-cone counts, then the shared sequence of multiplications
double ns3h_step_length(ns3h* h, const double* dz, const double* ds, const double* z, const double* s, double alpha_sym,
                        double a_min, double step) {
  int jmax = 0;
  for (int k = 0; k < h->v.n; k++) {
    const int j = body_step_count(h->v, k, dz, ds, z, s, alpha_sym, a_min, step);
    if (j > jmax) jmax = j;
  }
  return body_step_final(alpha_sym, jmax, step);
}
// barrier terms of the nonsymmetric, second-order and PSD cones (the nonnegative rows are a plain -log sum)
double ns3h_barrier(ns3h* h, const double* z, const double* s, const double* dz, const double* ds, double al) {
  double b = 0.0;
  for (int k = 0; k < h->v.n; k++) b += body_barrier(h->v, k, z, s, dz, ds, al);
  std::vector<double> W(32 * 32);
  for (int k = 0; k < h->ncones; k++) {
    const int o = h->off[k];
    if (h->type[k] == 1)
      for (int i = 0; i < h->dim[k]; i++) b += -lsafe((s[o + i] + al * ds[o + i]) * (z[o + i] + al * dz[o + i]));
    else if (h->type[k] == 2) b += soc_barrier(z + o, s + o, dz + o, ds + o, h->dim[k], al);
    else if (h->type[k] == 3)
      b += psd_neg_logdet(z + o, dz + o, h->psd_n[k], al, W.data()) + psd_neg_logdet(s + o, ds + o, h->psd_n[k], al, W.data());
  }
  return b;
}
double ns3h_wright_omega(double z) { return wright_omega(z); }
// the primal gradient update_scaling forms at the rows of every exponential / power cone (g is m long)
void ns3h_grad_primal(ns3h* h, const double* s, double* g) {
  for (int k = 0; k < h->v.n; k++) {
    const int id = h->list[k], o = h->off[id];
    if (h->type[id] == KIND_EXP) exp_grad_primal(s + o, g + o); else pow_grad_primal(s + o, h->alpha[k], g + o);
  }
}

// ---------------------------------------------------------------- generalised power cones (namespace cb::gp)
struct gph {
  int ncones, m, nHs;
  std::vector<int> type, off, boff, dim, list, dim1;
  std::vector<double> alpha, psi, grad, p, qr, d1, zc, d2, mu;
  std::vector<int> map_qr, map_p, map_D;
  cb::gp::View v;
};
// types as above plus 6 = genpow: dims[k] = len(alpha), dim2[k], exponents concatenated in alphas
gph* gph_new(int ncones, const int32_t* types, const int64_t* dims, const int64_t* dim2, const double* alphas) {
  gph* h = new gph();
  h->ncones = ncones; h->m = 0; h->nHs = 0;
  int cur = 0;
  std::vector<std::vector<double>> al(ncones);
  for (int k = 0; k < ncones; k++) {
    const int t = types[k];
    int rows = (int)dims[k];
    if (t == 3) rows = rows * (rows + 1) / 2;
    if (t == 4 || t == 5) rows = 3;
    if (t == 6) { al[k].assign(alphas + cur, alphas + cur + dims[k]); cur += (int)dims[k]; rows = (int)(dims[k] + dim2[k]); }
    const bool diag = t == 0 || t == 1 || (t == 2 && rows > 4) || t == 6;
    h->type.push_back(t); h->off.push_back(h->m); h->boff.push_back(h->nHs); h->dim.push_back(rows);
    h->m += rows; h->nHs += diag ? rows : rows * (rows + 1) / 2;
    if (t == 6) { h->list.push_back(k); h->dim1.push_back((int)dims[k]); }
  }
  const size_t n = h->list.size(), m = (size_t)h->m;
  h->alpha.assign(m, 0.0); h->psi.assign(n, 0.0);
  for (size_t k = 0; k < n; k++) {
    double sq = 0.0;
    const int id = h->list[k];
    for (size_t i = 0; i < al[id].size(); i++) { h->alpha[h->off[id] + i] = al[id][i]; sq += al[id][i] * al[id][i]; }
    h->psi[k] = 1.0 / sq;
  }
  for (auto* vv : {&h->grad, &h->p, &h->qr, &h->d1, &h->zc}) vv->assign(m, 0.0);
  h->d2.assign(n, 0.0); h->mu.assign(n, 0.0);
  h->v = cb::gp::View{(int)n, h->list.data(), h->off.data(), h->dim.data(), h->boff.data(), h->dim1.data(),
                      h->alpha.data(), h->psi.data(), h->grad.data(), h->p.data(), h->qr.data(), h->d1.data(),
                      h->zc.data(), h->d2.data(), h->mu.data()};
  return h;
}
void gph_free(gph* h) { delete h; }
int gph_m(const gph* h) { return h->m; }
int gph_nHs(const gph* h) { return h->nHs; }
void gph_unit_init(gph* h, double* z, double* s) { for (int k = 0; k < h->v.n; k++) cb::gp::body_unit_init(h->v, k, z, s); }
int gph_update_scaling(gph* h, const double* z, double mu) {
  int ok = 1;
  for (int k = 0; k < h->v.n; k++) if (!cb::gp::body_update_scaling(h->v, k, z, mu)) ok = 0;
  return ok;
}
void gph_get_Hs(gph* h, double* Hs, double sign) { for (int k = 0; k < h->v.n; k++) cb::gp::body_get_Hs(h->v, k, Hs, sign); }
void gph_mul_Hs(gph* h, double* y, const double* x) { for (int k = 0; k < h->v.n; k++) cb::gp::body_mul_Hs(h->v, k, y, x); }
void gph_copy_rows(gph* h, double* out, const double* in) { for (int k = 0; k < h->v.n; k++) cb::gp::body_copy_rows(h->v, k, out, in); }
void gph_combined_shift(gph* h, double* shift, double sigmamu) { for (int k = 0; k < h->v.n; k++) cb::gp::body_combined_shift(h->v, k, shift, sigmamu); }
double gph_step_length(gph* h, const double* dz, const double* ds, const double* z, const double* s, double alpha_sym,
                       double a_min, double step) {
  int jmax = 0;
  for (int k = 0; k < h->v.n; k++) {
    const int j = cb::gp::body_step_count(h->v, k, dz, ds, z, s, alpha_sym, a_min, step);
    if (j > jmax) jmax = j;
  }
  return body_step_final(alpha_sym, jmax, step);
}
double gph_barrier(gph* h, const double* z, const double* s, const double* dz, const double* ds, double al) {
  double b = 0.0;
  for (int k = 0; k < h->v.n; k++) b += cb::gp::body_barrier(h->v, k, z, s, dz, ds, al);
  return b;
}
// the primal gradient the primal barrier is formed from, at the rows of every generalised power cone (g is m long)
void gph_grad_primal(gph* h, const double* s, double* g) {
  std::vector<double> zero(h->m, 0.0);
  for (int k = 0; k < h->v.n; k++) {
    const int id = h->list[k], o = h->off[id], n = h->dim[id], d1 = h->dim1[k];
    double nw;
    const double x = cb::gp::primal_grad_scalar(h->v, k, s, zero.data(), 0.0, &nw);
    const bool far = nw > EPS;
    for (int i = 0; i < d1; i++) {
      const double a = h->alpha[o + i];
      g[o + i] = far ? -(1.0 + a + a * x * nw) / s[o + i] : -(1.0 + a) / s[o + i];
    }
    for (int i = d1; i < n; i++) g[o + i] = far ? (x / nw) * s[o + i] : 0.0;
  }
}
// values the three expansion columns and their diagonals would receive: out_qr[m], out_p[m], out_D[3*n]
void gph_kkt_values(gph* h, double* out_qr, double* out_p, double* out_D) {
  const int m = h->m, n = h->v.n;
  std::vector<double> vals((size_t)2 * m + 3 * n, 0.0);
  std::vector<int> mq(m), mp(m), mD(3 * n);
  for (int i = 0; i < m; i++) { mq[i] = i; mp[i] = m + i; }
  for (int i = 0; i < 3 * n; i++) mD[i] = 2 * m + i;
  for (int k = 0; k < n; k++) cb::gp::body_kkt_fill(h->v, k, vals.data(), mq.data(), mp.data(), mD.data());
  for (int i = 0; i < m; i++) { out_qr[i] = vals[i]; out_p[i] = vals[m + i]; }
  for (int i = 0; i < 3 * n; i++) out_D[i] = vals[2 * m + i];
}

}  // extern "C"
