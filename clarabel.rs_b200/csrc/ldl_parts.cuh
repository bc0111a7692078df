// The factor's parts (cldl_solve_part, cldl_mul_part, cldl_get_factor_csc, cldl_sample): products with L and L^T, the
// factor in compressed-column form and the standard normals of the sampler (device code, included by ldl.cu).
//
// P (K + E) P^T = L D L^T; every vector here is in permuted (elimination) order.  A front s owns the pivots f .. f+ns-1
// and the rows sn_rows[rp .. rp+nr) below them (ascending, all > f+ns-1); its panel is (ns+nr) x ns column-major in
// d.L, L21 below the pivot block.  Wide pivot blocks (ns > CB_SOLVE_SMALL_NS) hold M = L11^-1 in their strictly lower
// triangle (ldl_solve.cuh): a product with L11 is then a substitution with M, and the export recovers L11 = M^-1 with
// pivot_inverse, the factorisation's own routine.  Every sum has a fixed order and there are no floating-point atomics:
// repeated calls give the same bits, and a column gives the same bits whatever else the call computes.
#pragma once

#define PT_NT 128           /* threads per front of the product and export kernels */
#define PT_LDA 65           /* leading dimension of a recovered pivot block in shared memory */

// butterfly sum over the warp, fixed order; every lane gets the total
__device__ __forceinline__ double pt_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// y = L^T x, one CTA per front, no dependencies between fronts:  y_S = L11^T x_S + L21^T x_R.
// L21^T x_R: warp w takes the columns w, w + 4, ..., lanes run down a column (coalesced), one butterfly per column.
// L11^T x_S: narrow, thread j sums x_j + L11[j+1..][j] x_S in ascending order; wide, warp 0 solves M^T z = x_S by back
// substitution (z_j = x_j - sum_{i>j} M[i][j] z_i, j descending).
__global__ void __launch_bounds__(PT_NT) k_pt_ltmul(LDLDev d, const double* __restrict__ x, double* __restrict__ y) {
  __shared__ double sx[CB_PB_MAXNS], st[CB_PB_MAXNS];
  const int s = blockIdx.x;
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const double* __restrict__ P = d.L + d.panel_off[s];
  const int* __restrict__ rows = d.sn_rows + rp;
  if (tid < ns) sx[tid] = x[f + tid];
  for (int j = w; j < ns; j += PT_NT / 32) {
    const double* __restrict__ col = P + (long long)j * ld + ns;
    double acc = 0.0;
    for (int a = lane; a < nr; a += 32) acc += col[a] * x[rows[a]];
    __syncwarp();
    acc = pt_warp_sum(acc);
    if (lane == 0) st[j] = acc;
  }
  __syncthreads();
  if (ns > CB_SOLVE_SMALL_NS) {
    if (w == 0) {
      for (int j = ns - 1; j >= 0; j--) {
        const double* __restrict__ col = P + (long long)j * ld;
        double acc = 0.0;
        for (int i = j + 1 + lane; i < ns; i += 32) acc += col[i] * sx[i];
        __syncwarp();
        acc = pt_warp_sum(acc);
        if (lane == 0) sx[j] = sx[j] - acc;
        __syncwarp();
      }
    }
    __syncthreads();
    if (tid < ns) y[f + tid] = sx[tid] + st[tid];
  } else if (tid < ns) {
    const double* __restrict__ col = P + (long long)tid * ld;
    double z = sx[tid];
    for (int i = tid + 1; i < ns; i++) z += col[i] * sx[i];
    y[f + tid] = z + st[tid];
  }
}

// y = L x, first half, one CTA per front:  y_S = L11 x_S and w[rp + a] = (L21 x_S)[a], the front's contribution to row
// sn_rows[rp + a] (w is laid out like the solves' update vectors).  L11 x_S: narrow, thread i sums x_i + L11[i][..i-1]
// x_S in ascending order; wide, warp 0 solves M y_S = x_S by forward substitution.  L21 x_S: thread a sums over the
// columns in ascending order.
__global__ void __launch_bounds__(PT_NT) k_pt_lmul_front(LDLDev d, const double* __restrict__ x, double* __restrict__ y,
                                                         double* __restrict__ w) {
  __shared__ double sx[CB_PB_MAXNS], sy[CB_PB_MAXNS];
  const int s = blockIdx.x;
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr, tid = threadIdx.x, lane = tid & 31;
  const double* __restrict__ P = d.L + d.panel_off[s];
  if (tid < ns) sx[tid] = x[f + tid];
  __syncthreads();
  for (int a = tid; a < nr; a += PT_NT) {
    const double* __restrict__ row = P + ns + a;
    double acc = 0.0;
    for (int j = 0; j < ns; j++) acc += row[(long long)j * ld] * sx[j];
    w[rp + a] = acc;
  }
  if (ns > CB_SOLVE_SMALL_NS) {
    if (tid < 32) {
      for (int i = 0; i < ns; i++) {
        double acc = 0.0;
        for (int j = lane; j < i; j += 32) acc += P[(long long)j * ld + i] * sy[j];
        __syncwarp();
        acc = pt_warp_sum(acc);
        if (lane == 0) sy[i] = sx[i] - acc;
        __syncwarp();
      }
    }
    __syncthreads();
    if (tid < ns) y[f + tid] = sy[tid];
  } else if (tid < ns) {
    double z = sx[tid];
    for (int j = 0; j < tid; j++) z += P[(long long)j * ld + tid] * sx[j];
    y[f + tid] = z;
  }
}

// y = L x, second half, one thread per row:  y_i += the fronts' contributions to row i, in ascending position in w
// (FactorParts in ldl_plan.h: row_ptr / row_pos)
__global__ void k_pt_lmul_rows(int n, const long long* __restrict__ ptr, const long long* __restrict__ pos,
                               const double* __restrict__ w, double* __restrict__ y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc = y[i];
  for (long long e = ptr[i]; e < ptr[i + 1]; e++) acc += w[pos[e]];
  y[i] = acc;
}

// L strictly lower in compressed-column form, permuted order, rows ascending: column f + j of front s is the pivot
// block's rows f+j+1 .. f+ns-1, then sn_rows[rp ..].  L21 and narrow pivot blocks are copied as stored; a wide pivot
// block's L11 is recovered from M = L11^-1 in shared memory by pivot_inverse (the refactor's routine, applied to M).
// Warp w writes the columns w, w + 4, ...; rowval or Lx may be NULL.
__global__ void __launch_bounds__(PT_NT) k_pt_csc(LDLDev d, const unsigned long long* __restrict__ colptr,
                                                  unsigned long long* __restrict__ rowval, double* __restrict__ Lx) {
  __shared__ double sA[CB_PB_MAXNS * PT_LDA];
  const int s = blockIdx.x;
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const double* __restrict__ P = d.L + d.panel_off[s];
  const int* __restrict__ rows = d.sn_rows + rp;
  const bool wide = ns > CB_SOLVE_SMALL_NS;
  if (wide) {
    for (int idx = tid; idx < ns * ns; idx += PT_NT) {
      const int j = idx / ns, i = idx - j * ns;
      if (i > j) sA[j * PT_LDA + i] = P[(long long)j * ld + i];
    }
    __syncthreads();
    pivot_inverse<PT_NT>(sA, PT_LDA, ns);
    __syncthreads();
    pivot_inverse_place<PT_NT>(sA, PT_LDA, ns);
    __syncthreads();
  }
  for (int j = w; j < ns; j += PT_NT / 32) {
    const unsigned long long base = colptr[f + j];
    const int nt = ns - 1 - j;
    for (int t = lane; t < nt + nr; t += 32) {
      if (t < nt) {
        const int i = j + 1 + t;
        if (rowval) rowval[base + t] = (unsigned long long)(f + i);
        if (Lx) Lx[base + t] = wide ? sA[j * PT_LDA + i] : P[(long long)j * ld + i];
      } else {
        const int a = t - nt;
        if (rowval) rowval[base + t] = (unsigned long long)rows[a];
        if (Lx) Lx[base + t] = P[(long long)j * ld + ns + a];
      }
    }
  }
}

// ---- standard normals: Philox4x64-10 (Salmon, Moraes, Dror, Shaw, SC 2011; numpy.random.Philox) and Box-Muller ----
__device__ __forceinline__ unsigned long long pt_mulhi(unsigned long long a, unsigned long long b) {
#ifdef CB_EMU
  return (unsigned long long)(((unsigned __int128)a * b) >> 64);
#else
  return __umul64hi(a, b);
#endif
}
__device__ __forceinline__ void pt_sincospi(double x, double* s, double* c) {
#ifdef CB_EMU
  *s = std::sin(M_PI * x);
  *c = std::cos(M_PI * x);
#else
  sincospi(x, s, c);
#endif
}
// ten rounds of Philox4x64 on counter c with key k (Random123's philox4x64_R(10, c, k))
__device__ __forceinline__ void pt_philox(unsigned long long c[4], unsigned long long k0, unsigned long long k1) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    const unsigned long long a0 = 0xD2E7470EE14C6C93ull * c[0], h0 = pt_mulhi(0xD2E7470EE14C6C93ull, c[0]);
    const unsigned long long a1 = 0xCA5A826395121157ull * c[2], h1 = pt_mulhi(0xCA5A826395121157ull, c[2]);
    const unsigned long long n0 = h1 ^ c[1] ^ k0, n2 = h0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = a1; c[2] = n2; c[3] = a0;
    k0 += 0x9E3779B97F4A7C15ull;
    k1 += 0xBB67AE8584CAA73Bull;
  }
}
// z[4 j .. 4 j + 3] (rows below n only) for the draw at stream position `col`: counter (j, col, 0, 0), key (seed, 0);
// u = (r >> 11) 2^-53, Box-Muller on (1 - u0, u1) and (1 - u2, u3):  sqrt(-2 ln(1 - u0)) (cos, sin)(2 pi u1), ...
__global__ void k_pt_normals(int n, unsigned long long seed, unsigned long long col, double* __restrict__ z) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (4 * (long long)j >= n) return;
  unsigned long long c[4] = {(unsigned long long)j, col, 0ull, 0ull};
  pt_philox(c, seed, 0ull);
  double v[4];
#pragma unroll
  for (int p = 0; p < 2; p++) {
    const double u0 = (double)(c[2 * p] >> 11) * 0x1.0p-53, u1 = (double)(c[2 * p + 1] >> 11) * 0x1.0p-53;
    const double rad = sqrt(-2.0 * log(1.0 - u0));
    double sn, cs;
    pt_sincospi(2.0 * u1, &sn, &cs);
    v[2 * p] = rad * cs;
    v[2 * p + 1] = rad * sn;
  }
#pragma unroll
  for (int q = 0; q < 4; q++)
    if (4 * j + q < n) z[4 * j + q] = v[q];
}

// ---- per-entry operations ----
// y = s x with s = a (root 0) or sqrt|a| (root 1); x NULL stands for ones.  a is D or 1/D, both 0 at null pivots.
__global__ void k_pt_diag(int n, int root, const double* __restrict__ a, const double* x, double* y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double s = root ? sqrt(fabs(a[i])) : a[i];
  y[i] = x ? s * x[i] : s;
}
// x[perm[k]] = b[k] (x = P^T b)
__global__ void k_pt_permute_out(int n, const int* __restrict__ perm, const double* __restrict__ b, double* __restrict__ x) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) x[perm[k]] = b[k];
}
// x += mu
__global__ void k_pt_add(int n, const double* __restrict__ mu, double* __restrict__ x) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = x[i] + mu[i];
}
