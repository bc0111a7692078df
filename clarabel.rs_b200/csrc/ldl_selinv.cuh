// Selected inversion of the multifrontal LDL^T (included by ldl.cu): Z = (K + E)^-1 at every position of the
// factor's panels, K + E the regularised matrix that was factored, in the permuted order.
//
// For a front with pivots S and rows R (Takahashi; the supernodal form of Lin et al.'s SelInv), with Li = L_SS^-1
// (unit lower) and W = L_RS Li:
//     Z_RS = -Z_RR W = -(Z_RR L_RS) Li
//     Z_SS = Li^T D_S^-1 Li + W^T Z_RR W = Li^T (D_S^-1 Li - L_RS^T Z_RS)
// Z_RR is gathered from the ancestors' Z panels through the plan's maps (SelinvPlan in ldl_plan.h), so a front needs
// its parent's Z panel and nothing else: one persistent kernel runs the queue from the root down, every task spinning
// on its dependency (the parent's `done` flag, or its own front's row tasks) as the dataflow factorisation does.
// Z panels written inside the launch are read with ld.global.cg.  Every sum has a fixed order (the tile products keep
// their k order, the scalar sums run in index order), so two calls give the same bits.
//
// Shared memory of a task (doubles): Li [SI_RB][SI_LD] | A [SI_RB][SI_RB] | B [SI_RB][SI_RB] | 1/D [CB_PB_MAXNS].
// A and B hold the operands of one 64-deep slice of a tile product (k-major); afterwards the product goes to the
// same space as a [64][SI_LD] column-major block.
#define SI_NT 256
#define SI_LD (SI_RB + 1)
#define SI_SMEM_DOUBLES (SI_RB * SI_LD + 2 * SI_RB * SI_RB + CB_PB_MAXNS)
static_assert(SI_RB == TS && CB_PB_MAXNS <= SI_RB, "the selected-inversion tiles are the factorisation's 64 x 64 tiles");

// C[r][c] += sum_k A[k][r] B[k][c] over k < kn (kn a multiple of 4; operand rows kn.. are never read).  The thread's
// 4 x 4 entries of the 64 x 64 tile are (SI_OWN_R(i), SI_OWN_C(j)): on the device the ones mma.sync.m8n8k4 leaves in
// its registers (the ownership of the factorisation's T tasks), in the host build of the test suite a plain 4 x 4
// register tile with the same k order.
#ifdef CB_EMU
#define SI_OWN_R(i) ((threadIdx.x & 15) + 16 * (i))
#define SI_OWN_C(j) ((threadIdx.x >> 4) + 16 * (j))
#else
#define SI_OWN_R(i) (((threadIdx.x >> 5) & 1) * 32 + 8 * (i) + ((threadIdx.x & 31) >> 2))
#define SI_OWN_C(j) ((threadIdx.x >> 6) * 16 + 8 * ((j) >> 1) + 2 * (threadIdx.x & 3) + ((j) & 1))
#endif
__device__ __forceinline__ void si_tile_product(const double* __restrict__ sA, const double* __restrict__ sB, int kn,
                                                double (&acc)[4][4]) {
#ifdef CB_EMU   /* host build of the test suite: the same product with scalar FMAs */
  for (int k = 0; k < kn; k++) {
    double a[4], b[4];
    for (int i = 0; i < 4; i++) { a[i] = sA[k * SI_RB + SI_OWN_R(i)]; b[i] = sB[k * SI_RB + SI_OWN_C(i)]; }
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) acc[i][j] += a[i] * b[j];
  }
#else
  // FP64 tensor path, as in dff_tile: acc[i][2 jj + h] is fragment (i, jj), element h
  const int lk = threadIdx.x & 3, lr = (threadIdx.x & 31) >> 2;
  const int r0w = ((threadIdx.x >> 5) & 1) * 32, c0w = (threadIdx.x >> 6) * 16;
#pragma unroll 2
  for (int k = 0; k < kn; k += 4) {
    double a[4], b[2];
#pragma unroll
    for (int i = 0; i < 4; i++) a[i] = sA[(k + lk) * SI_RB + r0w + 8 * i + lr];
#pragma unroll
    for (int j = 0; j < 2; j++) b[j] = sB[(k + lk) * SI_RB + c0w + 8 * j + lr];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 2; j++)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                     : "+d"(acc[i][2 * j]), "+d"(acc[i][2 * j + 1]) : "d"(a[i]), "d"(b[j]));
  }
#endif
}

// the tile product's registers to a [64][SI_LD] column-major block (entry (r, c) at c * SI_LD + r)
__device__ __forceinline__ void si_tile_store(double* __restrict__ sC, const double (&acc)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) sC[SI_OWN_C(j) * SI_LD + SI_OWN_R(i)] = acc[i][j];
}

// Li = L_SS^-1 into sLi (column c at sLi[c * SI_LD ..], strictly lower part; the unit diagonal is implicit).  Fronts
// with more than CB_SOLVE_SMALL_NS pivots store it in their panel; narrower ones store L_SS and thread c substitutes
// column c (X[c] = 1, X[i] = -sum_{k = c .. i-1} L[i][k] X[k]).
__device__ __forceinline__ void si_load_linv(const LDLDev& d, const SITask& tk, double* sLi) {
  const int ns = tk.ns, ld = ns + tk.nr;
  const double* P = d.L + tk.poff;
  if (ns > CB_SOLVE_SMALL_NS) {
    for (int idx = threadIdx.x; idx < ns * ns; idx += SI_NT) {
      const int c = idx / ns, m = idx - c * ns;
      if (m > c) sLi[c * SI_LD + m] = P[(long long)c * ld + m];
    }
  } else if ((int)threadIdx.x < ns) {
    const int c = threadIdx.x;
    double x[CB_SOLVE_SMALL_NS];
    x[c] = 1.0;
    for (int i = c + 1; i < ns; i++) {
      double acc = 0.0;
      for (int k = c; k < i; k++) acc += P[(long long)k * ld + i] * x[k];
      x[i] = -acc;
      sLi[c * SI_LD + i] = x[i];
    }
  }
}

// Z_RR entry (R[i], R[k]) of the task's front, i and k front-local row indices
__device__ __forceinline__ double si_zrr(const SIPlan& q, long long rp, int i, int k) {
  const long long t = rp + (i >= k ? k : i);
  const int o = i >= k ? i : k;
  return __ldcg(q.Z + q.col[t] + q.segpos[q.seg[t] + o]);
}

// rows [r0, r1) of Z_RS = -(Z_RR L_RS) Li: the 64-row block of Y = Z_RR L_RS is one tile product over the front's
// rows (64 at a time: Z_RR gathered into A, L_RS into B), then each entry of Z_RS is a scalar sum over Li's column
__device__ void si_rows(const LDLDev& d, const SIPlan& q, const SITask& tk, double* sm) {
  double* sLi = sm;
  double* sA = sm + SI_RB * SI_LD;
  double* sB = sA + SI_RB * SI_RB;
  const int tid = threadIdx.x;
  const int ns = tk.ns, nr = tk.nr, ld = ns + nr, r0 = tk.r0, nb = tk.r1 - tk.r0;
  const double* P = d.L + tk.poff;
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.0;
  for (int k0 = 0; k0 < nr; k0 += SI_RB) {
    const int kn = min(SI_RB, nr - k0), kn4 = (kn + 3) & ~3;
    __syncthreads();   // the previous slice's operands are consumed
    for (int idx = tid; idx < kn4 * SI_RB; idx += SI_NT) {
      const int k = idx / SI_RB, i = idx - k * SI_RB;
      sA[idx] = (k < kn && i < nb) ? si_zrr(q, tk.rp, r0 + i, k0 + k) : 0.0;
      sB[idx] = (k < kn && i < ns) ? P[(long long)i * ld + ns + k0 + k] : 0.0;
    }
    __syncthreads();
    si_tile_product(sA, sB, kn4, acc);
  }
  __syncthreads();
  double* sY = sA;     // Y block, column c at sY[c * SI_LD ..]
  si_tile_store(sY, acc);
  __syncthreads();
  double* Z = q.Z + tk.poff;
  for (int idx = tid; idx < SI_RB * ns; idx += SI_NT) {
    const int c = idx / SI_RB, i = idx - c * SI_RB;
    if (i >= nb) continue;
    double y = sY[c * SI_LD + i];
    for (int m = c + 1; m < ns; m++) y += sY[m * SI_LD + i] * sLi[c * SI_LD + m];
    Z[(long long)c * ld + ns + r0 + i] = 0.0 - y;
  }
}

// Z_SS = Li^T (D^-1 Li - M), M = L_RS^T Z_RS (one tile product over the front's rows, Z_RS as the row tasks stored
// it); both triangles of the pivot block are written
__device__ void si_diag(const LDLDev& d, const SIPlan& q, const SITask& tk, double* sm) {
  double* sLi = sm;
  double* sA = sm + SI_RB * SI_LD;
  double* sB = sA + SI_RB * SI_RB;
  double* sDi = sB + SI_RB * SI_RB;
  const int tid = threadIdx.x;
  const int ns = tk.ns, nr = tk.nr, ld = ns + nr;
  const double* P = d.L + tk.poff;
  double* Z = q.Z + tk.poff;
  if (tid < ns) sDi[tid] = d.Dinv[tk.f + tid];
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.0;
  for (int k0 = 0; k0 < nr; k0 += SI_RB) {
    const int kn = min(SI_RB, nr - k0), kn4 = (kn + 3) & ~3;
    __syncthreads();
    for (int idx = tid; idx < kn4 * SI_RB; idx += SI_NT) {
      const int k = idx / SI_RB, c = idx - k * SI_RB;
      const bool on = k < kn && c < ns;
      sA[idx] = on ? P[(long long)c * ld + ns + k0 + k] : 0.0;
      sB[idx] = on ? __ldcg(Z + (long long)c * ld + ns + k0 + k) : 0.0;
    }
    __syncthreads();
    si_tile_product(sA, sB, kn4, acc);
  }
  __syncthreads();
  double* sT = sA;     // M, then T = D^-1 Li - M, column b at sT[b * SI_LD ..]
  si_tile_store(sT, acc);
  __syncthreads();
  for (int idx = tid; idx < ns * ns; idx += SI_NT) {
    const int b = idx / ns, m = idx - b * ns;
    const double li = m == b ? 1.0 : m > b ? sLi[b * SI_LD + m] : 0.0;
    sT[b * SI_LD + m] = sDi[m] * li - sT[b * SI_LD + m];
  }
  __syncthreads();
  for (int idx = tid; idx < ns * ns; idx += SI_NT) {
    const int b = idx / ns, a = idx - b * ns;
    if (a < b) continue;
    double z = sT[b * SI_LD + a];
    for (int m = a + 1; m < ns; m++) z += sLi[a * SI_LD + m] * sT[b * SI_LD + m];
    Z[(long long)b * ld + a] = z;
    if (a != b) Z[(long long)a * ld + b] = z;
  }
}

__global__ void __launch_bounds__(SI_NT, 2) k_selinv(LDLDev d, SIPlan q) {
  extern __shared__ __align__(16) double sism[];
  __shared__ __align__(16) int s_task[12];
  __shared__ int s_qi;
  const int tid = threadIdx.x;
  for (;;) {
    __syncthreads();
    if (tid == 0) {
      const int qi = atomicAdd(q.qhead, 1);
      s_qi = qi < q.ntask ? qi : -1;
    }
    __syncthreads();
    const int qi = s_qi;
    if (qi < 0) break;
    if (tid < 3) reinterpret_cast<int4*>(s_task)[tid] = q.tasks[3 * (size_t)qi + tid];
    __syncthreads();
    const SITask& tk = *reinterpret_cast<const SITask*>(s_task);
    const int kind = tk.kind, s = tk.s;
    if (tid == 0) {
      if (kind == 2) df_wait_zero(q.rows_left + s);
      else if (tk.parent >= 0) df_wait_set(q.done + tk.parent);
      __threadfence();
    }
    __syncthreads();
    si_load_linv(d, tk, sism);
    if (kind != 2) si_rows(d, q, tk, sism);
    if (kind == 1) {
      __syncthreads();
      if (tid == 0) { __threadfence(); atomicSub(q.rows_left + s, 1); }
      continue;
    }
    __syncthreads();   // kind 0: the front's Z_RS is stored
    si_diag(d, q, tk, sism);
    __syncthreads();
    if (tid == 0) { __threadfence(); atomicExch(q.done + s, 1); }
  }
}
#undef SI_OWN_R
#undef SI_OWN_C

// Z at the caller's entries: out[p] = Z[pos[p]], p in the caller's CSC order
__global__ void k_selinv_gather(const long long* __restrict__ pos, const double* __restrict__ Z, double* __restrict__ out,
                                long long n) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) out[p] = __ldcg(Z + pos[p]);
}
