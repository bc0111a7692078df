// Iterative refinement and error analysis of solves with the multifrontal LDL^T (included by ldl.cu; the host loop
// is LDLObject::solve_refined, the estimator LDLObject::condest).
//
// K is the symmetric matrix of the handle's current values: the caller's upper triangle mirrored into a full CSR
// whose entries point back into `vals` (src), so value updates since the last refactor are seen.  For an iterate x,
// with r = b - K x (Arioli, Demmel and Duff 1989; MUMPS RINFOG(7..8)):
//     den1_i = (|K||x|)_i + |b_i|,   den2_i = (|K||x|)_i + ||K_i||_inf ||x||_inf,
//     tau_i = 1000 n eps (||K_i||_inf ||x||_inf + |b_i|),   I1 = {i : den1_i > tau_i},  I2 the rest,
//     omega1 = max_I1 |r_i| / den1_i,   omega2 = max_I2 |r_i| / den2_i   (den2_i = r_i = 0 counts 0).
// Sums run in a fixed order (a warp's strided lanes, then a fixed shuffle tree) and every maximum is exact, so two calls
// give the same bits.  No floating-point atomics.
#define RF_NT 256                  // 8 rows per block in k_refine_residual
#define RF_NVEC 6                  // work vectors of n doubles (LDLObject::solve_refined)
#define RF_NOMEGA 5                // maxima of k_refine_omega

// the scalars of one call, in LDLObject::d_rf_ws after the reduction partials
enum { RF_XN = 0, RF_KN, RF_W1, RF_W2, RF_RINF, RF_HAS1, RF_HAS2, RF_EST, RF_CNT, RF_J, RF_VJ, RF_VJL, RF_NS = 16 };

// One warp per row i of the mirrored CSR: r_i = b_i - (K x)_i, kx_i = (|K||x|)_i, rmax_i = ||K_i||_inf and, when rsum
// is not null, rsum_i = sum_j |K_ij| (for ||K||_inf).  Lanes take entries p = rowptr[i] + lane + 32 k, then the shuffle
// tree of warp_sum / warp_max: one order for any row length, dense rows (arrow, linking rows) included.
__global__ void __launch_bounds__(RF_NT) k_refine_residual(int n, const int* __restrict__ rowptr,
                                                           const int* __restrict__ col, const int* __restrict__ src,
                                                           const double* __restrict__ vals,
                                                           const double* __restrict__ x, const double* __restrict__ b,
                                                           double* __restrict__ r, double* __restrict__ kx,
                                                           double* __restrict__ rmax, double* __restrict__ rsum) {
  const int i = (int)((blockIdx.x * (unsigned)RF_NT + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;                  // whole warps
  double s = 0.0, a = 0.0, m = 0.0, t = 0.0;
  for (int p = rowptr[i] + lane; p < rowptr[i + 1]; p += 32) {
    const double v = vals[src[p]], xv = x[col[p]];
    s += v * xv;
    a += fabs(v) * fabs(xv);
    m = fmax(m, fabs(v));
    t += fabs(v);
  }
  s = warp_sum(s);
  a = warp_sum(a);
  m = warp_max(m);
  if (rsum) t = warp_sum(t);
  if (lane == 0) {
    r[i] = b[i] - s;
    kx[i] = a;
    rmax[i] = m;
    if (rsum) rsum[i] = t;
  }
}

// den1, den2 and the category of row i at an iterate with ||x||_inf = xn; c = 1000 n eps
struct RfRow { double den1, den2; bool in1; };
__device__ __forceinline__ RfRow rf_row(int i, const double* kx, const double* rmax, const double* b, double xn, double c) {
  const double ab = fabs(b[i]), rx = rmax[i] * xn;
  RfRow w;
  w.den1 = kx[i] + ab;
  w.den2 = kx[i] + rx;
  w.in1 = w.den1 > c * (rx + ab);
  return w;
}

// a non-negative double or NaN as a key whose unsigned order is the values' order with NaN above +inf, so that the
// maximum of keys is the NaN-propagating maximum (the ordering atomic_max_nonneg relies on)
__device__ __forceinline__ unsigned long long rf_key(double v) {
  return v != v ? 0x7ff8000000000000ull : (unsigned long long)__double_as_longlong(v);
}
__device__ __forceinline__ unsigned long long rf_warp_max(unsigned long long k) {
  __syncwarp();
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, k, o); k = t > k ? t : k; }
  return k;
}

// out[RF_W1 ..] = omega1, omega2, ||r||_inf, [I1 non-empty], [I2 non-empty] at the iterate of k_refine_residual, with
// ||x||_inf read from xn.  k_sum's two levels: per-block maxima in ws.partials (one row of RED_BLOCKS per value), the
// last block to finish folds them in index order.
__global__ void __launch_bounds__(RED_THREADS) k_refine_omega(int n, const double* __restrict__ r,
                                                              const double* __restrict__ kx,
                                                              const double* __restrict__ rmax,
                                                              const double* __restrict__ b, const double* __restrict__ xn,
                                                              double c, ReduceWS ws, double* __restrict__ out) {
  __shared__ unsigned long long sh[RF_NOMEGA][RED_THREADS / 32];
  __shared__ bool last;
  const double xnv = *xn;
  unsigned long long m[RF_NOMEGA] = {0, 0, 0, 0, 0};
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += gridDim.x * RED_THREADS) {
    const RfRow w = rf_row(i, kx, rmax, b, xnv, c);
    const double ar = fabs(r[i]);
    double o1 = 0.0, o2 = 0.0;
    if (w.in1) o1 = ar / w.den1;
    else if (w.den2 != 0.0 || ar != 0.0) o2 = ar / w.den2;
    const unsigned long long k1 = rf_key(o1), k2 = rf_key(o2), k3 = rf_key(ar);
    m[0] = k1 > m[0] ? k1 : m[0];
    m[1] = k2 > m[1] ? k2 : m[1];
    m[2] = k3 > m[2] ? k3 : m[2];
    if (w.in1) m[3] = rf_key(1.0); else m[4] = rf_key(1.0);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int v = 0; v < RF_NOMEGA; v++) {
    const unsigned long long k = rf_warp_max(m[v]);
    if (lane == 0) sh[v][wid] = k;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int v = 0; v < RF_NOMEGA; v++) {
      unsigned long long k = 0;
      for (int w = 0; w < RED_THREADS / 32; w++) k = sh[v][w] > k ? sh[v][w] : k;
      ws.partials[v * RED_BLOCKS + blockIdx.x] = __longlong_as_double((long long)k);
    }
    __threadfence();
    const unsigned t = atomicInc(ws.counter, gridDim.x - 1);
    last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x < RF_NOMEGA) {
    __threadfence();
    unsigned long long k = 0;
    for (int i = 0; i < (int)gridDim.x; i++) {
      const unsigned long long q = (unsigned long long)__double_as_longlong(((volatile double*)ws.partials)[threadIdx.x * RED_BLOCKS + i]);
      k = q > k ? q : k;
    }
    out[threadIdx.x] = __longlong_as_double((long long)k);
  }
}

// The estimator's argmax: out[RF_J] = the smallest j with |v_j| = max_i |v_i|, out[RF_VJ] = |v_j|, in k_sum's two
// levels; each block keeps the first index of its maximum, and the last block folds the blocks in index order.  (A NaN
// is never larger, so it is not chosen unless every entry is NaN; the estimate is then NaN through its 1-norm.)
__global__ void __launch_bounds__(RED_THREADS) k_refine_argmax(int n, const double* __restrict__ v, ReduceWS ws,
                                                               double* __restrict__ out) {
  __shared__ double shv[RED_THREADS];
  __shared__ int shi[RED_THREADS];
  __shared__ bool last;
  double bv = -1.0;
  int bi = n;
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += gridDim.x * RED_THREADS) {
    const double a = fabs(v[i]);
    if (a > bv) { bv = a; bi = i; }            // ascending i: the first index of the thread's maximum
  }
  shv[threadIdx.x] = bv;
  shi[threadIdx.x] = bi;
  __syncthreads();
  for (int s = RED_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const double ov = shv[threadIdx.x + s];
      const int oi = shi[threadIdx.x + s];
      if (ov > shv[threadIdx.x] || (ov == shv[threadIdx.x] && oi < shi[threadIdx.x])) { shv[threadIdx.x] = ov; shi[threadIdx.x] = oi; }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    ws.partials[blockIdx.x] = shv[0];
    ws.partials[RED_BLOCKS + blockIdx.x] = (double)shi[0];
    __threadfence();
    const unsigned t = atomicInc(ws.counter, gridDim.x - 1);
    last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    double mv = -1.0, mi = (double)n;
    for (int k = 0; k < (int)gridDim.x; k++) {   // blocks own interleaved index ranges: ties go to the smaller index
      const double pv = ((volatile double*)ws.partials)[k], pi = ((volatile double*)ws.partials)[RED_BLOCKS + k];
      if (pv > mv || (pv == mv && pi < mi)) { mv = pv; mi = pi; }
    }
    out[RF_J] = mi;
    out[RF_VJ] = mv;
  }
}
