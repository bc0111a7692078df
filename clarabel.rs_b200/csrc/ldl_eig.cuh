// Krylov basis operations of cldl_eigsh (included by ldl.cu; the iteration is lanczos_run in ldl_eig.cpp, the driver
// LDLObject::eigsh).  The basis V is n x (ncv + 1), column-major with leading dimension n; MV = M V beside it when M is
// not the identity.  Tall-skinny FP64, memory bound.  Every sum has a fixed order and there are no floating-point
// atomics, so two calls give the same bits.
#define EIG_CB_NT 128              // k_eig_combine: rows per block (one per thread)
#define EIG_CB_COLS 8              // output columns per block, held in registers
#define EIG_CB_P 64                // rows of S per shared-memory tile

// h[c] = sum_i V[i, c] z[i] for c < j.  k_sum's two levels: each block sums its rows (grid-stride) for four columns at a
// time and writes one partial per column to part[c * RED_BLOCKS + block]; the last block to finish folds each column's
// partials in block order.
__global__ void __launch_bounds__(RED_THREADS) k_eig_dots(int n, int j, const double* __restrict__ V,
                                                          const double* __restrict__ z, double* __restrict__ part,
                                                          unsigned* __restrict__ counter, double* __restrict__ h) {
  __shared__ double sh[32];
  __shared__ bool last;
  for (int c0 = 0; c0 < j; c0 += 4) {
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    const int nc = j - c0 < 4 ? j - c0 : 4;
    for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += gridDim.x * RED_THREADS) {
      const double zi = z[i];
#pragma unroll
      for (int q = 0; q < 4; q++)
        if (q < nc) acc[q] += V[(size_t)(c0 + q) * n + i] * zi;
    }
    for (int q = 0; q < nc; q++) {
      const double s = block_sum(acc[q], sh);
      if (threadIdx.x == 0) part[(size_t)(c0 + q) * RED_BLOCKS + blockIdx.x] = s;
    }
  }
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned t = atomicInc(counter, gridDim.x - 1);
    last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int c = 0; c < j; c++) {
    double a = 0.0;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += RED_THREADS) a += ((volatile double*)part)[(size_t)c * RED_BLOCKS + b];
    a = block_sum(a, sh);
    if (threadIdx.x == 0) h[c] = a;
  }
}

// w -= V[:, 0, j) h and, when z is not null, z -= MV[:, 0, j) h: one thread per row, columns in ascending order
__global__ void __launch_bounds__(256) k_eig_update(int n, int j, const double* __restrict__ V,
                                                    const double* __restrict__ MV, const double* __restrict__ h,
                                                    double* __restrict__ w, double* __restrict__ z) {
  __shared__ double hs[EIG_MAX_NCV + 1];
  for (int c = threadIdx.x; c < j; c += blockDim.x) hs[c] = h[c];
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int c = 0; c < j; c++) s += V[(size_t)c * n + i] * hs[c];
  w[i] -= s;
  if (z) {
    double t = 0.0;
    for (int c = 0; c < j; c++) t += MV[(size_t)c * n + i] * hs[c];
    z[i] -= t;
  }
}

// Y = V[:, 0, m) S with S m x k column-major, Y n x k: a block takes EIG_CB_NT rows and EIG_CB_COLS columns of Y, S
// passes through shared memory in tiles of EIG_CB_P rows, each output sums over p in ascending order
__global__ void __launch_bounds__(EIG_CB_NT) k_eig_combine(int n, int m, int k, const double* __restrict__ V,
                                                           const double* __restrict__ S, double* __restrict__ Y) {
  __shared__ double ss[EIG_CB_P][EIG_CB_COLS];
  const int i = blockIdx.x * EIG_CB_NT + threadIdx.x, c0 = blockIdx.y * EIG_CB_COLS;
  double acc[EIG_CB_COLS];
#pragma unroll
  for (int c = 0; c < EIG_CB_COLS; c++) acc[c] = 0.0;
  for (int p0 = 0; p0 < m; p0 += EIG_CB_P) {
    __syncthreads();
    for (int t = threadIdx.x; t < EIG_CB_P * EIG_CB_COLS; t += EIG_CB_NT) {
      const int p = t % EIG_CB_P, c = t / EIG_CB_P;
      ss[p][c] = (p0 + p < m && c0 + c < k) ? S[(size_t)(c0 + c) * m + p0 + p] : 0.0;
    }
    __syncthreads();
    if (i < n) {
      const int pe = m - p0 < EIG_CB_P ? m - p0 : EIG_CB_P;
      for (int p = 0; p < pe; p++) {
        const double v = V[(size_t)(p0 + p) * n + i];
#pragma unroll
        for (int c = 0; c < EIG_CB_COLS; c++) acc[c] += v * ss[p][c];
      }
    }
  }
  if (i >= n) return;
#pragma unroll
  for (int c = 0; c < EIG_CB_COLS; c++)
    if (c0 + c < k) Y[(size_t)(c0 + c) * n + i] = acc[c];
}
