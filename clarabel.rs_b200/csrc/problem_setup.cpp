// Set-up of the interior-point solver on the host.  See problem_setup.h.
#include "problem_setup.h"

#include <algorithm>
#include <cmath>

namespace cb {

int check_csc(const uint64_t* cp, const uint64_t* ri, uint64_t rows, int cols, bool triu) {
  if (!cp || cp[0] != 0) return CLDL_E_ARG;
  for (int j = 0; j < cols; j++) if (cp[j + 1] < cp[j]) return CLDL_E_ARG;
  if (cp[cols] > 0 && !ri) return CLDL_E_ARG;
  for (int j = 0; j < cols; j++)
    for (uint64_t t = cp[j]; t < cp[j + 1]; t++) {
      if (ri[t] >= rows) return CLDL_E_DIM;
      if (t > cp[j] && ri[t] <= ri[t - 1]) return CLDL_E_ARG;
      if (triu && ri[t] > (uint64_t)j) return CLDL_E_NOT_TRIU;
    }
  return 0;
}

HostCsc host_csc(int m, int n, const uint64_t* cp, const uint64_t* ri, const double* v) {
  HostCsc M;
  M.m = m; M.n = n;
  M.colptr.assign(cp, cp + n + 1); M.rowval.assign(ri, ri + cp[n]); M.nzval.assign(v, v + cp[n]);
  return M;
}

int collapse_cones(const int32_t* types, const uint64_t* dims, uint64_t n, std::vector<ConeSpec>& out,
                   const double* params, const uint64_t* gp_dim2, const double* gp_alpha) {
  out.clear();
  uint64_t k = 0, gp_cursor = 0;
  // rows a cone occupies; exponential / power cones are three rows whatever dims[] says (supportedcone.rs:54-71)
  auto numel = [](int t, uint64_t d) -> uint64_t { return t == CT_PSD ? d * (d + 1) / 2 : (t == CT_EXP || t == CT_POW) ? 3 : (t == CT_GENPOW ? (d ? d : 1) : d); };
  while (k < n) {
    const int t = types[k];
    if (t < 0 || t > CT_GENPOW) return CLDL_E_ARG;
    if (t == CT_GENPOW) {   // GenPowerConeT(alpha, dim2): dims[k] = len(alpha) (supportedcone.rs:44, genpowcone.rs:41-49)
      if (!gp_dim2 || !gp_alpha || dims[k] < 1) return CLDL_E_ARG;
      const uint64_t d1 = dims[k], d2 = gp_dim2[k];
      ConeSpec cs{t, (int)(d1 + d2), 0, 0.0, std::vector<double>(gp_alpha + gp_cursor, gp_alpha + gp_cursor + d1)};
      gp_cursor += d1;
      double sum = 0.0;
      for (double a : cs.alphas) { if (!(a > 0.0)) return CLDL_E_ARG; sum += a; }
      if (!(std::fabs(1.0 - sum) < 2.220446049250313e-16 * (double)d1 * 0.5 + 1e-300)) return CLDL_E_ARG;
      out.push_back(cs);
      k++;
      continue;
    }
    if (t == CT_EXP || t == CT_POW) {   // 3 rows each, never merged (supportedcone.rs:105-161)
      const double a = (t == CT_POW && params) ? params[k] : 0.0;
      if (t == CT_POW && !(a > 0.0 && a < 1.0)) return CLDL_E_ARG;
      out.push_back({t, 3, 0, a, {}});
      k++;
      continue;
    }
    const uint64_t d = dims[k];
    if (numel(t, d) == 0) { k++; continue; }
    const bool coll = (t == CT_NONNEG) || ((t == CT_SOC || t == CT_PSD) && d == 1);
    if (coll) {
      uint64_t tot = (t == CT_NONNEG) ? d : 1;
      k++;
      while (k < n) {
        const int t2 = types[k];
        const uint64_t d2 = dims[k];
        if (numel(t2, d2) != 0) {
          if (t2 == CT_NONNEG) tot += d2;
          else if ((t2 == CT_SOC || t2 == CT_PSD) && d2 == 1) tot += 1;
          else break;
        }
        k++;
      }
      out.push_back({CT_NONNEG, (int)tot, 0, 0.0, {}});
    } else {
      if (t == CT_SOC && d < 2) return CLDL_E_ARG;
      if (t == CT_PSD) { if (d > (uint64_t)CB_PSD_MAX_N) return CLDL_E_ARG; out.push_back({t, (int)(d * (d + 1) / 2), (int)d, 0.0, {}}); }
      else out.push_back({t, (int)d, 0, 0.0, {}});
      k++;
    }
  }
  return 0;
}

int presolve(std::vector<ConeSpec>& cones, HostCsc& A, std::vector<double>& b, double infbound, bool enable,
             std::vector<char>& keep) {
  keep.clear();
  int64_t rows = 0;
  for (const ConeSpec& c : cones) rows += c.dim;
  if (rows != A.m) return CLDL_E_DIM;
  for (double& v : b) v = std::min(v, infbound);
  if (!enable) return 0;
  const int m = A.m, n = A.n;
  const double thr = (1.0 - 2.220446049250313e-16 * 10.0) * infbound;
  std::vector<char> kp(m, 1);
  int mred = m, r = 0;
  for (const ConeSpec& c : cones) {
    if (c.type == CT_NONNEG) { for (int i = 0; i < c.dim; i++, r++) if (b[r] > thr) { kp[r] = 0; mred--; } }
    else r += c.dim;
  }
  if (mred == m) return 0;
  std::vector<ConeSpec> cs;
  r = 0;
  for (const ConeSpec& c : cones) {
    if (c.type == CT_NONNEG) {
      int nk = 0;
      for (int i = 0; i < c.dim; i++) nk += kp[r + i];
      if (nk > 0) { ConeSpec c2 = c; c2.dim = nk; cs.push_back(c2); }
    } else {
      cs.push_back(c);
    }
    r += c.dim;
  }
  cones.swap(cs);
  std::vector<int> rowmap(m, -1);
  int nr = 0;
  for (int i = 0; i < m; i++) if (kp[i]) rowmap[i] = nr++;
  int64_t w = 0;
  for (int j = 0; j < n; j++) {
    const int64_t b0 = A.colptr[j];
    A.colptr[j] = w;
    for (int64_t t = b0; t < A.colptr[j + 1]; t++)
      if (rowmap[A.rowval[t]] >= 0) { A.rowval[w] = rowmap[A.rowval[t]]; A.nzval[w] = A.nzval[t]; w++; }
  }
  A.colptr[n] = w; A.rowval.resize(w); A.nzval.resize(w); A.m = mred;
  for (int i = 0; i < m; i++) if (kp[i]) b[rowmap[i]] = b[i];
  b.resize(mred);
  keep.swap(kp);
  return 0;
}

int cone_layout(const std::vector<ConeSpec>& cs, ConeLayout& L) {
  const int nc = (int)cs.size();
  L = ConeLayout();
  L.cones = cs;
  L.off.assign(nc, 0); L.boff.assign(nc, 0); L.sparse_flag.assign(nc, 0); L.diag_block.assign(nc, 0); L.pdim.assign(nc, 0);
  for (int k = 0; k < nc; k++) {
    const ConeSpec& c = cs[k];
    const bool sp = c.type == CT_SOC && c.dim > SOC_NO_EXPANSION_MAX_SIZE;
    const bool diag = c.type == CT_ZERO || c.type == CT_NONNEG || sp || c.type == CT_GENPOW;
    const long long blk = diag ? (long long)c.dim : (long long)c.dim * (c.dim + 1) / 2;
    if ((long long)L.nHs + blk > 2000000000LL) return CLDL_E_ARG;
    L.off[k] = L.m; L.boff[k] = L.nHs;
    L.sparse_flag[k] = sp ? 1 : 0;
    L.diag_block[k] = diag ? 1 : 0;
    L.pdim[k] = sp ? 2 : (c.type == CT_GENPOW ? 3 : 0);
    L.p += L.pdim[k];
    L.nHs += (int)blk;
    L.m += c.dim;
    const bool ns3c = c.type == CT_EXP || c.type == CT_POW;
    const bool gpc = c.type == CT_GENPOW;
    L.degree += c.type == CT_ZERO ? 0 : (c.type == CT_NONNEG ? c.dim : (c.type == CT_PSD ? c.psd_n : (ns3c ? 3 : (gpc ? (int)c.alphas.size() + 1 : 1))));
    if (ns3c) { L.ns_list.push_back(k); L.all_symmetric = false; }
    if (gpc) { L.gp_list.push_back(k); L.all_symmetric = false; L.allows_primal_dual = false; }
    if (c.type == CT_SOC) L.soc_list.push_back(k);
    if (c.type == CT_PSD) L.psd_list.push_back(k);
  }
  return 0;
}

std::vector<int> kkt_perm(const uint64_t* perm, int n, int m, const ConeLayout& L) {
  std::vector<int> out((size_t)n + m + L.p);
  for (size_t k = 0; k < out.size(); k++) out[k] = (int)perm[k];
  return out;
}

void Equilibration::scale_P(HostCsc& P, const double* v) const {
  for (int j = 0; j < P.n; j++)
    for (int64_t t = P.colptr[j]; t < P.colptr[j + 1]; t++) P.nzval[t] = v[t] * d[P.rowval[t]] * d[j] * c;
}
void Equilibration::scale_A(HostCsc& A, const double* v) const {
  for (int j = 0; j < A.n; j++)
    for (int64_t t = A.colptr[j]; t < A.colptr[j + 1]; t++) A.nzval[t] = v[t] * e[A.rowval[t]] * d[j];
}
double Equilibration::scale_q(std::vector<double>& q, const double* v) const {
  double norm = 0;
  for (size_t i = 0; i < q.size(); i++) { q[i] = v[i] * d[i] * c; norm = std::max(norm, std::fabs(q[i] * dinv[i])); }
  return norm / c;                         // problemdata.rs:147-189: unscaled norm recomputed from the scaled data
}
double Equilibration::scale_b(std::vector<double>& b, const double* v) const {
  double norm = 0;
  for (size_t i = 0; i < b.size(); i++) { b[i] = v[i] * e[i]; norm = std::max(norm, std::fabs(b[i] * einv[i])); }
  return norm;
}

Equilibration equilibrate(HostCsc& P, HostCsc& A, std::vector<double>& q, std::vector<double>& b, const ConeLayout& L,
                          const cipm_settings& s) {
  const int n = P.n, m = A.m;
  Equilibration eq;
  std::vector<double>&d = eq.d, &e = eq.e, &dw = eq.dinv, &ew = eq.einv;
  double& c = eq.c;
  d.assign(n, 1.0); dw.assign(n, 1.0); e.assign(m, 1.0); ew.assign(m, 1.0);
  if (!s.equilibrate_enable) return eq;
  const double smin = s.equilibrate_min_scaling, smax = s.equilibrate_max_scaling;
  auto clip = [](double v, double lo, double hi) { return v < lo ? lo : (v > hi ? hi : v); };
  auto scale_data = [&](const double* dd_, const double* ee_) {
    if (dd_) {
      for (int col = 0; col < n; col++)
        for (int64_t t = P.colptr[col]; t < P.colptr[col + 1]; t++) P.nzval[t] *= dd_[P.rowval[t]] * dd_[col];
      for (int col = 0; col < n; col++)
        for (int64_t t = A.colptr[col]; t < A.colptr[col + 1]; t++) A.nzval[t] *= ee_[A.rowval[t]] * dd_[col];
      for (int i = 0; i < n; i++) q[i] *= dd_[i];
    } else {
      for (int64_t t = 0; t < A.colptr[n]; t++) A.nzval[t] *= ee_[A.rowval[t]];
    }
    for (int i = 0; i < m; i++) b[i] *= ee_[i];
  };
  for (int it = 0; it < s.equilibrate_max_iter; it++) {
    std::fill(dw.begin(), dw.end(), 0.0);
    for (int i = 0; i < n; i++)
      for (int64_t t = P.colptr[i]; t < P.colptr[i + 1]; t++) {
        const double v = std::fabs(P.nzval[t]);
        const int r = P.rowval[t];
        dw[i] = std::max(dw[i], v); dw[r] = std::max(dw[r], v);
      }
    for (int i = 0; i < n; i++)
      for (int64_t t = A.colptr[i]; t < A.colptr[i + 1]; t++) dw[i] = std::max(dw[i], std::fabs(A.nzval[t]));
    std::fill(ew.begin(), ew.end(), 0.0);
    for (int64_t t = 0; t < A.colptr[n]; t++) ew[A.rowval[t]] = std::max(ew[A.rowval[t]], std::fabs(A.nzval[t]));
    for (auto& v : dw) { if (v == 0.0) v = 1.0; v = 1.0 / std::sqrt(v); }
    for (auto& v : ew) { if (v == 0.0) v = 1.0; v = 1.0 / std::sqrt(v); }
    for (int i = 0; i < n; i++) dw[i] = clip(dw[i], smin / d[i], smax / d[i]);
    for (int i = 0; i < m; i++) ew[i] = clip(ew[i], smin / e[i], smax / e[i]);
    scale_data(dw.data(), ew.data());
    for (int i = 0; i < n; i++) d[i] *= dw[i];
    for (int i = 0; i < m; i++) e[i] *= ew[i];
    double meanP = 0.0, infq = 0.0;
    for (int i = 0; i < n; i++) {
      double v = 0.0;
      for (int64_t t = P.colptr[i]; t < P.colptr[i + 1]; t++) v = std::max(v, std::fabs(P.nzval[t]));
      meanP += v;
    }
    meanP = n ? meanP / n : 0.0;
    for (int i = 0; i < n; i++) infq = std::max(infq, std::fabs(q[i]));
    if (meanP != 0.0 && infq != 0.0) {
      const double ct = clip(1.0 / std::max(infq, meanP), smin / c, smax / c);
      for (auto& v : P.nzval) v *= ct;
      for (auto& v : q) v *= ct;
      c *= ct;
    }
  }
  bool changed = false;
  std::fill(ew.begin(), ew.end(), 1.0);
  for (size_t k = 0; k < L.cones.size(); k++)
    if (L.cones[k].type != CT_ZERO && L.cones[k].type != CT_NONNEG) {  // scalar scaling inside the other cones (socone.rs:97-101, psdtrianglecone.rs:98-101, expcone.rs:71-74, powcone.rs:63-66)
      const int o = L.off[k], dm = L.cones[k].dim;
      double mean = 0.0;
      for (int i = 0; i < dm; i++) mean += e[o + i];
      mean /= dm;
      for (int i = 0; i < dm; i++) ew[o + i] = (1.0 / e[o + i]) * mean;
      changed = true;
    }
  if (changed) { scale_data(nullptr, ew.data()); for (int i = 0; i < m; i++) e[i] *= ew[i]; }
  for (int i = 0; i < n; i++) dw[i] = 1.0 / d[i];
  for (int i = 0; i < m; i++) ew[i] = 1.0 / e[i];
  return eq;
}

void unscale_solution(const Equilibration& eq, const std::vector<char>& keep, double infbound, double scaleinv, int n,
                      int mfull, const double* hx, const double* hz, const double* hs, double* x, double* z, double* s) {
  const double cinv = 1.0 / eq.c;
  for (int i = 0; i < n; i++) x[i] = hx[i] * eq.d[i] * scaleinv;
  for (int i = 0, r = 0; i < mfull; i++) {
    if (keep.empty() || keep[i]) { z[i] = hz[r] * eq.e[r] * (scaleinv * cinv); s[i] = hs[r] * eq.einv[r] * scaleinv; r++; }
    else { z[i] = 0.0; s[i] = infbound; }
  }
}

CsrMap csc_to_csr(const HostCsc& M) {
  CsrMap R;
  R.rowptr.assign(M.m + 1, 0);
  const int64_t nnz = M.colptr[M.n];
  for (int64_t t = 0; t < nnz; t++) R.rowptr[M.rowval[t] + 1]++;
  for (int i = 0; i < M.m; i++) R.rowptr[i + 1] += R.rowptr[i];
  R.col.resize(nnz); R.src.resize(nnz);
  std::vector<int> pos(R.rowptr.begin(), R.rowptr.end() - 1);
  for (int j = 0; j < M.n; j++)
    for (int64_t t = M.colptr[j]; t < M.colptr[j + 1]; t++) {
      const int d = pos[M.rowval[t]]++;
      R.col[d] = j; R.src[d] = (int)t;
    }
  return R;
}

CsrMap triu_to_sym_csr(int n, const int64_t* colptr, const int* rowval) {
  CsrMap R;
  R.rowptr.assign(n + 1, 0);
  for (int j = 0; j < n; j++)
    for (int64_t t = colptr[j]; t < colptr[j + 1]; t++) { R.rowptr[rowval[t] + 1]++; if (rowval[t] != j) R.rowptr[j + 1]++; }
  for (int i = 0; i < n; i++) R.rowptr[i + 1] += R.rowptr[i];
  R.col.resize(R.rowptr[n]); R.src.resize(R.rowptr[n]);
  std::vector<int> pos(R.rowptr.begin(), R.rowptr.end() - 1);
  for (int j = 0; j < n; j++)
    for (int64_t t = colptr[j]; t < colptr[j + 1]; t++) {
      const int i = rowval[t];
      R.col[pos[i]] = j; R.src[pos[i]++] = (int)t;
      if (i != j) { R.col[pos[j]] = i; R.src[pos[j]++] = (int)t; }
    }
  return R;
}

std::vector<double> gather(const std::vector<double>& v, const std::vector<int>& idx) {
  std::vector<double> out(idx.size());
  for (size_t k = 0; k < idx.size(); k++) out[k] = v[idx[k]];
  return out;
}

int assemble_kkt(const HostCsc& P, const HostCsc& A, const ConeLayout& L, KKTAssembly& K) {
  const int n = P.n, m = A.m, nc = (int)L.cones.size(), N = n + m + L.p;
  K.N = N;
  std::vector<int64_t> cnt(N + 1, 0);
  auto has_diag = [&](int i) {
    return P.colptr[i] != P.colptr[i + 1] && P.rowval[P.colptr[i + 1] - 1] == i;
  };
  for (int i = 0; i < n; i++) cnt[i] += P.colptr[i + 1] - P.colptr[i] + (has_diag(i) ? 0 : 1);
  for (int64_t q = 0; q < A.colptr[n]; q++) cnt[n + A.rowval[q]] += 1;
  for (int k = 0, pcol = n + m; k < nc; pcol += L.pdim[k], k++) {
    const ConeSpec& c = L.cones[k];
    const int row = n + L.off[k];
    for (int i = 0; i < c.dim; i++) cnt[row + i] += L.diag_block[k] ? 1 : i + 1;
    if (L.sparse_flag[k]) { cnt[pcol] += c.dim + 1; cnt[pcol + 1] += c.dim + 1; }
    if (c.type == CT_GENPOW) {   // q, r, p columns + their diagonal entries (datamaps.rs:264-287)
      const int d1 = (int)c.alphas.size();
      cnt[pcol] += d1 + 1; cnt[pcol + 1] += c.dim - d1 + 1; cnt[pcol + 2] += c.dim + 1;
    }
  }
  std::vector<int64_t>& Kp = K.Kp;
  Kp.assign(N + 1, 0);
  for (int j = 0; j < N; j++) Kp[j + 1] = Kp[j] + cnt[j];
  K.nnzK = Kp[N];
  if (K.nnzK > 0x7fffffff) return CLDL_E_DIM;
  std::vector<int>& Ki = K.Ki;
  Ki.assign(K.nnzK, 0);
  std::vector<int64_t> nxt(Kp.begin(), Kp.end() - 1);
  K.map_P.assign(P.colptr[n], 0);
  K.map_A.assign(A.colptr[n], 0);
  K.map_Hs.assign(L.nHs, 0);
  K.map_u.assign(m ? m : 1, 0);
  K.map_v.assign(m ? m : 1, 0);
  K.map_D.assign(2 * (nc ? nc : 1), 0);
  K.map_gqr.assign(m ? m : 1, 0); K.map_gp.assign(m ? m : 1, 0); K.map_gD.assign(3 * (L.gp_list.size() ? L.gp_list.size() : 1), 0);
  K.dsigns.assign(N, 1);
  for (int i = 0; i < n; i++) {
    for (int64_t q = P.colptr[i]; q < P.colptr[i + 1]; q++) {
      int64_t d = nxt[i]++;
      Ki[d] = P.rowval[q]; K.map_P[q] = (int)d;
    }
    if (!has_diag(i)) { int64_t d = nxt[i]++; Ki[d] = i; }
  }
  for (int i = 0; i < A.n; i++)
    for (int64_t q = A.colptr[i]; q < A.colptr[i + 1]; q++) {
      const int col = n + A.rowval[q];
      int64_t d = nxt[col]++;
      Ki[d] = i; K.map_A[q] = (int)d;
    }
  for (int i = n; i < n + m; i++) K.dsigns[i] = -1;
  int gpk = 0;
  for (int k = 0, pcol = n + m; k < nc; pcol += L.pdim[k], k++) {
    const ConeSpec& c = L.cones[k];
    const int row = n + L.off[k], o = L.off[k];
    int* blk = K.map_Hs.data() + L.boff[k];
    if (L.diag_block[k]) {
      for (int i = 0; i < c.dim; i++) { int64_t d = nxt[row + i]++; Ki[d] = row + i; blk[i] = (int)d; }
    } else {
      int kk = 0;
      for (int col = row; col < row + c.dim; col++)
        for (int r = row; r <= col; r++) { int64_t d = nxt[col]++; Ki[d] = r; blk[kk++] = (int)d; }
    }
    if (L.sparse_flag[k]) {
      for (int i = 0; i < c.dim; i++) { int64_t d = nxt[pcol]++; Ki[d] = row + i; K.map_v[o + i] = (int)d; }
      for (int i = 0; i < c.dim; i++) { int64_t d = nxt[pcol + 1]++; Ki[d] = row + i; K.map_u[o + i] = (int)d; }
      for (int i = 0; i < 2; i++) { int64_t d = nxt[pcol + i]++; Ki[d] = pcol + i; K.map_D[2 * k + i] = (int)d; }
      K.dsigns[pcol] = -1;
    }
    if (c.type == CT_GENPOW) {   // datamaps.rs:289-312: q rows [0, dim1), r rows [dim1, dim), p all rows
      const int d1 = (int)c.alphas.size();
      for (int i = 0; i < d1; i++) { int64_t d = nxt[pcol]++; Ki[d] = row + i; K.map_gqr[o + i] = (int)d; }
      for (int i = d1; i < c.dim; i++) { int64_t d = nxt[pcol + 1]++; Ki[d] = row + i; K.map_gqr[o + i] = (int)d; }
      for (int i = 0; i < c.dim; i++) { int64_t d = nxt[pcol + 2]++; Ki[d] = row + i; K.map_gp[o + i] = (int)d; }
      for (int i = 0; i < 3; i++) { int64_t d = nxt[pcol + i]++; Ki[d] = pcol + i; K.map_gD[3 * gpk + i] = (int)d; }
      gpk++;
      K.dsigns[pcol] = -1; K.dsigns[pcol + 1] = -1;   // datamaps.rs:252-254
    }
  }
  K.map_diag.resize(N);
  for (int j = 0; j < N; j++) K.map_diag[j] = (int)(Kp[j + 1] - 1);
  // dense cone blocks: every block is contracted to one vertex for the ordering (order_with_groups in symbolic.cpp)
  K.group.assign(N, -1);
  K.ngroups = 0;
  for (int k = 0; k < nc; k++) {
    if (L.diag_block[k] || L.cones[k].dim <= 8) continue;
    for (int i = 0; i < L.cones[k].dim; i++) K.group[n + L.off[k] + i] = K.ngroups;
    K.ngroups++;
  }
  return 0;
}

}  // namespace cb
