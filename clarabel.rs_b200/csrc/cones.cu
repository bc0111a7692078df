// Device cone kernels (sm_90a).  See cones.h.
//
// Per-function reference map (all under /root/reference/src/solver/core/cones):
//   Nonnegative  nonnegativecone.rs:58-166, 177-195
//   Zero         zerocone.rs:53-131
//   SOC          socone.rs:104-287 (scaling, Hs, mul_Hs, ds offset), :360-382 (Jordan ops),
//                :421-495 (step length), :504-530 (fast W / W^-1 products)
//   shift        symmetric_common.rs:53-84
#include "cones.h"

#include <cmath>
#include <cstdio>

namespace cb {

#define SOC_NT 128

// ---------------------------------------------------------------- elementwise
__global__ void k_ew_set_identity(ConeDev c) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.m) return;
  const int t = c.rowtag[i];
  if (t == CT_NONNEG) c.w[i] = 1.0;
  else if (t == CT_SOC) { c.w[i] = 0.0; c.u[i] = 0.0; c.v[i] = 0.0; }
}
__global__ void k_soc_set_identity(ConeDev c) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= c.nsoc) return;
  const int id = c.soc_list[k];
  c.w[c.off[id]] = 1.0;
  c.eta[id] = 1.0;
  if (c.sparse[id]) { c.dd[id] = 0.5; c.u[c.off[id]] = 0.70710678118654752440; }
}

__global__ void k_ew_update_scaling(ConeDev c, const double* __restrict__ s, const double* __restrict__ z) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.m) return;
  if (c.rowtag[i] == CT_NONNEG) {
    const double si = s[i], zi = z[i];
    c.lam[i] = sqrt(si * zi);
    c.w[i] = sqrt(si / zi);
  }
}

__global__ void k_ew_get_Hs(ConeDev c, double* __restrict__ Hs, double sign, const int* __restrict__ row2blk) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.m) return;
  const int t = c.rowtag[i];
  if (t == CT_ZERO) Hs[row2blk[i]] = sign * 0.0;
  else if (t == CT_NONNEG) { const double w = c.w[i]; Hs[row2blk[i]] = sign * (w * w); }
}

__global__ void k_ew_mul_Hs(ConeDev c, double* __restrict__ y, const double* __restrict__ x) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.m) return;
  const int t = c.rowtag[i];
  if (t == CT_ZERO) y[i] = 0.0;
  else if (t == CT_NONNEG) { const double w = c.w[i]; y[i] = w * (w * x[i]); }
}

__global__ void k_ew_affine_ds(ConeDev c, double* __restrict__ ds) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.m) return;
  const int t = c.rowtag[i];
  if (t == CT_ZERO) ds[i] = 0.0;
  else if (t == CT_NONNEG) { const double l = c.lam[i]; ds[i] = l * l; }
}

__global__ void k_ew_combined_shift(ConeDev c, double* __restrict__ shift, double* __restrict__ sz,
                                    double* __restrict__ ss, double sigmamu) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.m) return;
  const int t = c.rowtag[i];
  if (t == CT_ZERO) shift[i] = 0.0;
  else if (t == CT_NONNEG) {
    const double w = c.w[i];
    const double a = sz[i] * w, b = ss[i] / w;
    sz[i] = a; ss[i] = b;
    shift[i] = b * a + (-sigmamu);
  }
}

__global__ void k_ew_ds_offset(ConeDev c, double* __restrict__ out, const double* __restrict__ ds,
                               const double* __restrict__ z) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.m) return;
  const int t = c.rowtag[i];
  if (t == CT_ZERO) out[i] = 0.0;
  else if (t == CT_NONNEG) out[i] = ds[i] / z[i];
}

__global__ void __launch_bounds__(RED_THREADS)
k_ew_step_length(ConeDev c, const double* __restrict__ dz, const double* __restrict__ ds,
                 const double* __restrict__ z, const double* __restrict__ s, double* alpha) {
  double a = INFINITY;
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < c.m; i += gridDim.x * RED_THREADS) {
    if (c.rowtag[i] != CT_NONNEG) continue;
    const double dzi = dz[i], dsi = ds[i];
    if (dzi < 0.0) a = fmin(a, -z[i] / dzi);
    if (dsi < 0.0) a = fmin(a, -s[i] / dsi);
  }
  a = warp_min(a);
  if ((threadIdx.x & 31) == 0 && a < INFINITY) atomic_min_nonneg(alpha, fmax(a, 0.0));
}

__global__ void k_ew_unit_shift(ConeDev c, double* __restrict__ z, double alpha, int primal) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.m) return;
  const int t = c.rowtag[i];
  if (t == CT_ZERO) { if (primal) z[i] = 0.0; }
  else if (t == CT_NONNEG) z[i] += alpha;
}
__global__ void k_soc_unit_shift(ConeDev c, double* __restrict__ z, double alpha) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < c.nsoc) z[c.off[c.soc_list[k]]] += alpha;
}

// margins: per-block partial (min, possum) for NN rows; SOC cones handled by k_soc_margins
__global__ void __launch_bounds__(RED_THREADS)
k_ew_margins(ConeDev c, const double* __restrict__ z, double* pmin, double* psum) {
  __shared__ double sh[32];
  double mn = INFINITY, sm = 0.0;
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < c.m; i += gridDim.x * RED_THREADS) {
    if (c.rowtag[i] != CT_NONNEG) continue;
    const double zi = z[i];
    mn = fmin(mn, zi);
    sm += fmax(zi, 0.0);
  }
  sm = block_sum(sm, sh);
  mn = warp_min(mn);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = mn;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m2 = INFINITY;
    for (int w = 0; w < RED_THREADS / 32; w++) m2 = fmin(m2, sh[w]);
    pmin[blockIdx.x] = m2;
    psum[blockIdx.x] = sm;
  }
}
// one CTA per SOC cone: margin = z0 - ||z1||
__global__ void __launch_bounds__(SOC_NT) k_soc_margins(ConeDev c, const double* __restrict__ z, double* pmin, double* psum) {
  __shared__ double sh[32];
  const int id = c.soc_list[blockIdx.x];
  const int o = c.off[id], n = c.dim[id];
  Blue3 q{0.0, 0.0, 0.0};     // z[1..].norm() is the reference's overflow-safe norm (socone.rs:105, vecmath.rs:206-226)
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) blue_add(q, z[o + i]);
  q.big = block_sum(q.big, sh);
  q.med = block_sum(q.med, sh);
  q.sml = block_sum(q.sml, sh);
  if (threadIdx.x == 0) {
    const double a = z[o] - blue_norm(q);
    pmin[blockIdx.x] = a;
    psum[blockIdx.x] = fmax(a, 0.0);
  }
}
__global__ void k_margins_final(const double* pmin, const double* psum, int n1, int n2, double* out2) {
  // single thread: fixed summation order
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double mn = 1.7976931348623157e308, sm = 0.0;   // T::max_value() start, compositecone.rs:197-205
  for (int i = 0; i < n1 + n2; i++) { mn = fmin(mn, pmin[i]); sm += psum[i]; }
  out2[0] = mn; out2[1] = sm;
}

// ------------------------------------------------------------------- SOC CTAs
__device__ __forceinline__ double soc_res_from(double z0, double sumsq1) {
  const double t = sqrt(sumsq1);
  return (z0 - t) * (z0 + t);
}

__global__ void __launch_bounds__(SOC_NT) k_soc_update_scaling(ConeDev c, const double* __restrict__ s_, const double* __restrict__ z_) {
  __shared__ double sh[32];
  const int id = c.soc_list[blockIdx.x];
  const int o = c.off[id], n = c.dim[id];
  const double* s = s_ + o; const double* z = z_ + o;
  double* w = c.w + o; double* lam = c.lam + o;
  double qz = 0.0, qs = 0.0;
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) { qz += z[i] * z[i]; qs += s[i] * s[i]; }
  qz = block_sum(qz, sh);
  qs = block_sum(qs, sh);
  const double rz = soc_res_from(z[0], qz), rs = soc_res_from(s[0], qs);
  const double zscale = rz > 0.0 ? sqrt(rz) : 0.0, sscale = rs > 0.0 ? sqrt(rs) : 0.0;
  if (zscale == 0.0 || sscale == 0.0) { if (threadIdx.x == 0) atomicExch(c.fail, 1); return; }
  const double eta = sqrt(sscale / zscale);
  const double sinv = 1.0 / sscale, mz = -(1.0 / zscale);
  // w = s/sscale + J z/zscale  (unnormalised)
  double qw = 0.0;
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) { const double wi = mz * z[i] + s[i] * sinv; w[i] = wi; qw += wi * wi; }
  qw = block_sum(qw, sh);
  const double w0u = s[0] * sinv + z[0] / zscale;
  const double rw = soc_res_from(w0u, qw);
  const double wscale = rw > 0.0 ? sqrt(rw) : 0.0;
  if (wscale == 0.0) { if (threadIdx.x == 0) atomicExch(c.fail, 1); return; }
  const double winv = 1.0 / wscale;
  double w1sq = 0.0;
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) { const double wi = w[i] * winv; w[i] = wi; w1sq += wi * wi; }
  w1sq = block_sum(w1sq, sh);
  const double w0 = sqrt(1.0 + w1sq);
  const double g = 0.5 * wscale;
  const double ca = (g + z[0] / zscale) / sscale, cb = (g + s[0] / sscale) / zscale;
  const double den = 1.0 / (s[0] / sscale + z[0] / zscale + 2.0 * g);
  const double sq = sqrt(sscale * zscale);
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) lam[i] = ((ca * s[i] + cb * z[i]) * den) * sq;
  const bool sp = c.sparse[id] != 0;
  double u1 = 0.0, v1 = 0.0, dval = 0.0, u0 = 0.0;
  if (sp) {
    const double alpha = 2.0 * w0;
    const double wsq = w0 * w0 + w1sq;
    const double wsqinv = 1.0 / wsq;
    dval = 0.5 * wsqinv;
    u0 = sqrt(wsq - dval);
    u1 = alpha / u0;
    v1 = sqrt(2.0 * (2.0 + wsqinv) / (2.0 * wsq - wsqinv));
    for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) { const double wi = w[i]; c.u[o + i] = u1 * wi; c.v[o + i] = v1 * wi; }
  }
  if (threadIdx.x == 0) {
    w[0] = w0; lam[0] = g * sq; c.eta[id] = eta;
    if (sp) { c.dd[id] = dval; c.u[o] = u0; c.v[o] = 0.0; }
  }
}

__global__ void __launch_bounds__(SOC_NT) k_soc_get_Hs(ConeDev c, double* __restrict__ Hs, double sign) {
  const int id = c.soc_list[blockIdx.x];
  const int o = c.off[id], n = c.dim[id];
  double* H = Hs + c.boff[id];
  const double e2 = c.eta[id] * c.eta[id];
  if (c.sparse[id]) {
    const double d = c.dd[id];
    for (int i = threadIdx.x; i < n; i += SOC_NT) H[i] = sign * (i == 0 ? e2 * d : e2);
  } else {
    // dense packed triu, column major (socone.rs:229-244); n <= 4
    const double* w = c.w + o;
    if (threadIdx.x == 0) {
      H[0] = sign * (((1.4142135623730951 * w[0] - 1.0) * (1.4142135623730951 * w[0] + 1.0)) * e2);
      int h = 1;
      for (int col = 1; col < n; col++)
        for (int row = 0; row <= col; row++) {
          double v = 2.0 * w[row] * w[col];
          if (row == col) v += 1.0;
          H[h++] = sign * (v * e2);
        }
    }
  }
}

__global__ void __launch_bounds__(SOC_NT) k_soc_mul_Hs(ConeDev c, double* __restrict__ y_, const double* __restrict__ x_) {
  __shared__ double sh[32];
  const int id = c.soc_list[blockIdx.x];
  const int o = c.off[id], n = c.dim[id];
  const double* w = c.w + o; const double* x = x_ + o; double* y = y_ + o;
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += SOC_NT) a += w[i] * x[i];
  a = block_sum(a, sh);
  const double cc = a * 2.0, e2 = c.eta[id] * c.eta[id];
  for (int i = threadIdx.x; i < n; i += SOC_NT) {
    const double xi = (i == 0) ? -x[0] : x[i];
    y[i] = (cc * w[i] + xi) * e2;
  }
}

__global__ void __launch_bounds__(SOC_NT) k_soc_affine_ds(ConeDev c, double* __restrict__ ds_) {
  __shared__ double sh[32];
  const int id = c.soc_list[blockIdx.x];
  const int o = c.off[id], n = c.dim[id];
  const double* l = c.lam + o; double* ds = ds_ + o;
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += SOC_NT) a += l[i] * l[i];
  a = block_sum(a, sh);
  const double l0 = l[0];
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) ds[i] = l0 * l[i] + l0 * l[i];
  if (threadIdx.x == 0) ds[0] = a;
}

__global__ void __launch_bounds__(SOC_NT)
k_soc_combined_shift(ConeDev c, double* __restrict__ shift_, double* __restrict__ sz_, double* __restrict__ ss_, double sigmamu) {
  __shared__ double sh[32];
  const int id = c.soc_list[blockIdx.x];
  const int o = c.off[id], n = c.dim[id];
  const double* w = c.w + o;
  double* sz = sz_ + o; double* ss = ss_ + o; double* shift = shift_ + o;
  const double eta = c.eta[id], w0 = w[0];
  double zz = 0.0, zs = 0.0;
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) { zz += w[i] * sz[i]; zs += w[i] * ss[i]; }
  zz = block_sum(zz, sh);
  zs = block_sum(zs, sh);
  const double z0 = sz[0], s0 = ss[0];
  const double cz = z0 + zz / (1.0 + w0);          // W  (socone.rs:507-516)
  const double cs = -s0 + zs / (1.0 + w0);         // W^-1 (socone.rs:521-530)
  const double Wz0 = eta * (w0 * z0 + zz);
  const double Ws0 = (1.0 / eta) * (w0 * s0 - zs);
  __syncthreads();
  double dot = 0.0;
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) {
    const double a = (eta * cz) * w[i] + eta * sz[i];
    const double b = ((1.0 / eta) * cs) * w[i] + (1.0 / eta) * ss[i];
    sz[i] = a; ss[i] = b;
    dot += b * a;
    shift[i] = Ws0 * a + Wz0 * b;   // circ_op(x, y=ss, z=sz): x1 = y0*z1 + z0*y1
  }
  dot = block_sum(dot, sh);
  if (threadIdx.x == 0) {
    sz[0] = Wz0; ss[0] = Ws0;
    shift[0] = (dot + Ws0 * Wz0) + (-sigmamu);
  }
}

__global__ void __launch_bounds__(SOC_NT)
k_soc_ds_offset(ConeDev c, double* __restrict__ out_, const double* __restrict__ ds_, const double* __restrict__ z_) {
  __shared__ double sh[32];
  const int id = c.soc_list[blockIdx.x];
  const int o = c.off[id], n = c.dim[id];
  const double* w = c.w + o; const double* l = c.lam + o;
  const double* ds = ds_ + o; const double* z = z_ + o; double* out = out_ + o;
  double qz = 0.0, lds = 0.0, wds = 0.0;
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) { qz += z[i] * z[i]; lds += l[i] * ds[i]; wds += w[i] * ds[i]; }
  qz = block_sum(qz, sh);
  lds = block_sum(lds, sh);
  wds = block_sum(wds, sh);
  const double resz = soc_res_from(z[0], qz);
  const double eta = c.eta[id];
  const double cc = (l[0] * ds[0] - lds) / resz;
  const double linv = 1.0 / l[0];
  const double f = wds / (1.0 + w[0]);
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) out[i] = ((-z[i]) * cc + eta * (ds[i] + f * w[i])) * linv;
  if (threadIdx.x == 0) out[0] = (z[0] * cc + eta * wds) * linv;
}

__device__ double soc_step_component(double x0, double y0, double qx, double qy, double xy1, double amax) {
  // socone.rs:421-495
  if (x0 >= 0.0 && y0 < 0.0) amax = fmin(amax, -x0 / y0);
  const double a = soc_res_from(y0, qy);
  const double b = 2.0 * (x0 * y0 - xy1);
  const double c = fmax(0.0, soc_res_from(x0, qx));
  const double d = b * b - 4.0 * a * c;
  if ((a > 0.0 && b > 0.0) || d < 0.0) return amax;
  if (a == 0.0) return amax;
  if (c == 0.0) return a >= 0.0 ? amax : 0.0;
  const double t = b >= 0.0 ? (-b - sqrt(d)) : (-b + sqrt(d));
  double r1 = (2.0 * c) / t, r2 = t / (2.0 * a);
  if (r1 < 0.0) r1 = INFINITY;
  if (r2 < 0.0) r2 = INFINITY;
  return fmin(amax, fmin(r1, r2));
}

__global__ void __launch_bounds__(SOC_NT)
k_soc_step_length(ConeDev c, const double* __restrict__ dz_, const double* __restrict__ ds_,
                  const double* __restrict__ z_, const double* __restrict__ s_, double* alpha) {
  __shared__ double sh[32];
  const int id = c.soc_list[blockIdx.x];
  const int o = c.off[id], n = c.dim[id];
  const double* dz = dz_ + o; const double* ds = ds_ + o; const double* z = z_ + o; const double* s = s_ + o;
  double qz = 0, qdz = 0, zdz = 0, qs = 0, qds = 0, sds = 0;
  for (int i = 1 + threadIdx.x; i < n; i += SOC_NT) {
    qz += z[i] * z[i]; qdz += dz[i] * dz[i]; zdz += z[i] * dz[i];
    qs += s[i] * s[i]; qds += ds[i] * ds[i]; sds += s[i] * ds[i];
  }
  qz = block_sum(qz, sh); qdz = block_sum(qdz, sh); zdz = block_sum(zdz, sh);
  qs = block_sum(qs, sh); qds = block_sum(qds, sh); sds = block_sum(sds, sh);
  if (threadIdx.x == 0) {
    const double amax = *((volatile double*)alpha);
    const double az = soc_step_component(z[0], dz[0], qz, qdz, zdz, amax);
    const double as = soc_step_component(s[0], ds[0], qs, qds, sds, amax);
    atomic_min_nonneg(alpha, fmax(fmin(az, as), 0.0));
  }
}

// --------------------------------------------------------------------- host
#define CCK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { std::fprintf(stderr, "[clarabel_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return -20; } } while (0)

int ConeSet::init(const ConeLayout& layout, cudaStream_t st) {
  static_cast<ConeLayout&>(*this) = layout;
  stream = st;
  const std::vector<ConeSpec>& cs = cones;
  const int nc = (int)cs.size();
  std::vector<int> type(nc), dim(nc);
  for (int k = 0; k < nc; k++) { type[k] = cs[k].type; dim[k] = cs[k].dim; }
  std::vector<signed char> tag(m);
  std::vector<int> row2blk(m, 0);
  for (int k = 0; k < nc; k++)
    for (int i = 0; i < cs[k].dim; i++) {
      tag[off[k] + i] = (signed char)cs[k].type;
      row2blk[off[k] + i] = boff[k] + i;  // valid for diagonal-block cones
    }
  dev.ncones = nc; dev.m = m; dev.nsoc = (int)soc_list.size();
  CCK(upload(&dev.type, type)); CCK(upload(&dev.off, off)); CCK(upload(&dev.dim, dim)); CCK(upload(&dev.boff, boff));
  CCK(upload(&dev.sparse, sparse_flag)); CCK(upload(&dev.soc_list, soc_list)); CCK(upload(&dev.rowtag, tag));
  CCK(upload(&row2blk_dev, row2blk));
  const size_t mm = (size_t)(m ? m : 1), cc = (size_t)(nc ? nc : 1);
  CCK(cudaMalloc((void**)&dev.w, mm * 8)); CCK(cudaMalloc((void**)&dev.lam, mm * 8));
  CCK(cudaMalloc((void**)&dev.u, mm * 8)); CCK(cudaMalloc((void**)&dev.v, mm * 8));
  CCK(cudaMalloc((void**)&dev.eta, cc * 8)); CCK(cudaMalloc((void**)&dev.dd, cc * 8));
  CCK(cudaMalloc((void**)&dev.fail, sizeof(int)));
  CCK(cudaMemset(dev.w, 0, mm * 8)); CCK(cudaMemset(dev.lam, 0, mm * 8));
  CCK(cudaMemset(dev.u, 0, mm * 8)); CCK(cudaMemset(dev.v, 0, mm * 8));
  CCK(cudaMemset(dev.eta, 0, cc * 8)); CCK(cudaMemset(dev.dd, 0, cc * 8));
  CCK(cudaMemset(dev.fail, 0, sizeof(int)));
  CCK(cudaMalloc((void**)&ws.partials, (size_t)(RED_BLOCKS + 64) * 4 * 8));
  CCK(cudaMalloc((void**)&ws.counter, sizeof(unsigned)));
  CCK(cudaMemset(ws.counter, 0, sizeof(unsigned)));
  {
    std::vector<int> pn(nc, 0);
    std::vector<long long> mo(nc, 0);
    long long tot = 0;
    psd_nmax = 0; psd_numel_max = 0;
    for (int k = 0; k < nc; k++)
      if (cs[k].type == CT_PSD) {
        pn[k] = cs[k].psd_n; mo[k] = tot; tot += (long long)cs[k].psd_n * cs[k].psd_n;
        if (cs[k].psd_n > psd_nmax) psd_nmax = cs[k].psd_n;
        if (cs[k].dim > psd_numel_max) psd_numel_max = cs[k].dim;
      }
    dev.npsd = (int)psd_list.size();
    CCK(upload(&dev.psd_list, psd_list)); CCK(upload(&dev.psd_n, pn)); CCK(upload(&dev.psd_moff, mo));
    const size_t tb = (size_t)(tot ? tot : 1) * 8;
    psd_mat_total = tot;
    CCK(cudaMalloc((void**)&dev.psd_R, tb)); CCK(cudaMalloc((void**)&dev.psd_Rinv, tb)); CCK(cudaMalloc((void**)&dev.psd_RRt, tb));
    CCK(cudaMalloc((void**)&dev.psd_bar, tb));
    CCK(cudaMemset(dev.psd_R, 0, tb)); CCK(cudaMemset(dev.psd_Rinv, 0, tb)); CCK(cudaMemset(dev.psd_RRt, 0, tb));
    if (dev.npsd && psd_prepare()) return -20;
  }
  {
    std::vector<double> al(nc, 0.0);
    for (int k = 0; k < nc; k++) al[k] = cs[k].param;
    if (ns_prepare(al)) return -20;
    if (gp_prepare()) return -20;
  }
  const size_t np = (size_t)RED_BLOCKS + soc_list.size() + psd_list.size() + 8;
  CCK(cudaMalloc((void**)&d_pmin, np * 8)); CCK(cudaMalloc((void**)&d_psum, np * 8));
  return 0;
}

void ConeSet::release() {
  auto fr = [](const void* p) { if (p) cudaFree((void*)p); };
  fr(dev.type); fr(dev.off); fr(dev.dim); fr(dev.boff); fr(dev.sparse); fr(dev.soc_list); fr(dev.rowtag);
  fr(dev.w); fr(dev.lam); fr(dev.u); fr(dev.v); fr(dev.eta); fr(dev.dd); fr(dev.fail);
  fr(ws.partials); fr(ws.counter); fr(row2blk_dev); fr(d_pmin); fr(d_psum);
  fr(dev.psd_list); fr(dev.psd_n); fr(dev.psd_moff); fr(dev.psd_R); fr(dev.psd_Rinv); fr(dev.psd_RRt); fr(dev.psd_ws); fr(dev.psd_bar);
  ns_release();
  gp_release();
}

#define EW_GRID ((m + 255) / 256)

void ConeSet::set_identity_scaling() {
  if (m == 0) return;
  g_launches += 1 + (dev.nsoc ? 1 : 0);
  k_ew_set_identity<<<EW_GRID, 256, 0, stream>>>(dev);
  if (dev.nsoc) k_soc_set_identity<<<(dev.nsoc + 127) / 128, 128, 0, stream>>>(dev);
  psd_set_identity();
}
void ConeSet::update_scaling(const double* s, const double* z, double mu, int strategy) {
  if (m == 0) return;
  g_launches += 1 + (dev.nsoc ? 1 : 0);
  k_ew_update_scaling<<<EW_GRID, 256, 0, stream>>>(dev, s, z);
  if (dev.nsoc) k_soc_update_scaling<<<dev.nsoc, SOC_NT, 0, stream>>>(dev, s, z);
  psd_update_scaling(s, z);
  ns_update_scaling(s, z, mu, strategy);
}
void ConeSet::get_Hs(double* Hs, bool negate) {
  if (m == 0) return;
  g_launches += 1 + (dev.nsoc ? 1 : 0);
  const double sg = negate ? -1.0 : 1.0;
  k_ew_get_Hs<<<EW_GRID, 256, 0, stream>>>(dev, Hs, sg, row2blk_dev);
  if (dev.nsoc) k_soc_get_Hs<<<dev.nsoc, SOC_NT, 0, stream>>>(dev, Hs, sg);
  psd_get_Hs(Hs, sg);
  ns_get_Hs(Hs, sg);
}
void ConeSet::mul_Hs(double* y, const double* x) {
  if (m == 0) return;
  g_launches += 1 + (dev.nsoc ? 1 : 0);
  k_ew_mul_Hs<<<EW_GRID, 256, 0, stream>>>(dev, y, x);
  if (dev.nsoc) k_soc_mul_Hs<<<dev.nsoc, SOC_NT, 0, stream>>>(dev, y, x);
  psd_apply(0, y, const_cast<double*>(x), nullptr, 0.0);
  ns_mul_Hs(y, x);
}
void ConeSet::affine_ds(double* ds, const double* s) {
  if (m == 0) return;
  g_launches += 1 + (dev.nsoc ? 1 : 0);
  k_ew_affine_ds<<<EW_GRID, 256, 0, stream>>>(dev, ds);
  if (dev.nsoc) k_soc_affine_ds<<<dev.nsoc, SOC_NT, 0, stream>>>(dev, ds);
  psd_apply(1, ds, nullptr, nullptr, 0.0);
  if (s) ns_copy_rows(ds, s);      // expcone.rs:135-137
}
void ConeSet::combined_ds_shift(double* shift, double* step_z, double* step_s, double sigmamu) {
  if (m == 0) return;
  g_launches += 1 + (dev.nsoc ? 1 : 0);
  k_ew_combined_shift<<<EW_GRID, 256, 0, stream>>>(dev, shift, step_z, step_s, sigmamu);
  if (dev.nsoc) k_soc_combined_shift<<<dev.nsoc, SOC_NT, 0, stream>>>(dev, shift, step_z, step_s, sigmamu);
  psd_apply(2, shift, step_z, step_s, sigmamu);
  ns_combined_shift(shift, step_z, step_s, sigmamu);
}
void ConeSet::ds_from_dz_offset(double* out, const double* ds, const double* z) {
  if (m == 0) return;
  g_launches += 1 + (dev.nsoc ? 1 : 0);
  k_ew_ds_offset<<<EW_GRID, 256, 0, stream>>>(dev, out, ds, z);
  if (dev.nsoc) k_soc_ds_offset<<<dev.nsoc, SOC_NT, 0, stream>>>(dev, out, ds, z);
  psd_apply(3, out, const_cast<double*>(ds), nullptr, 0.0);
  ns_copy_rows(out, ds);           // expcone.rs:150-152
}
void ConeSet::step_length(const double* dz, const double* ds, const double* z, const double* s, double* alpha_slot) {
  if (m == 0) return;
  g_launches += 1 + (dev.nsoc ? 1 : 0);
  k_ew_step_length<<<red_grid(m), RED_THREADS, 0, stream>>>(dev, dz, ds, z, s, alpha_slot);
  if (dev.nsoc) k_soc_step_length<<<dev.nsoc, SOC_NT, 0, stream>>>(dev, dz, ds, z, s, alpha_slot);
  psd_step_length(dz, ds, alpha_slot);
  ns_step_length(dz, ds, z, s, alpha_slot);   // symmetric cones first, nonsymmetric last (compositecone.rs:289-332)
}
void ConeSet::margins(const double* z, double* out2) {
  const int g = m ? red_grid(m) : 0;
  g_launches += 1 + (g ? 1 : 0) + (dev.nsoc ? 1 : 0);
  if (g) k_ew_margins<<<g, RED_THREADS, 0, stream>>>(dev, z, d_pmin, d_psum);
  if (dev.nsoc) k_soc_margins<<<dev.nsoc, SOC_NT, 0, stream>>>(dev, z, d_pmin + g, d_psum + g);
  psd_margins(z, d_pmin + g + dev.nsoc, d_psum + g + dev.nsoc);
  k_margins_final<<<1, 32, 0, stream>>>(d_pmin, d_psum, g, dev.nsoc + dev.npsd, out2);
}
void ConeSet::scaled_unit_shift(double* z, double alpha, bool primal) {
  if (m == 0) return;
  g_launches += 1 + (dev.nsoc ? 1 : 0);
  k_ew_unit_shift<<<EW_GRID, 256, 0, stream>>>(dev, z, alpha, primal ? 1 : 0);
  if (dev.nsoc) k_soc_unit_shift<<<(dev.nsoc + 127) / 128, 128, 0, stream>>>(dev, z, alpha);
  psd_apply(4, z, nullptr, nullptr, alpha);
}

}  // namespace cb
