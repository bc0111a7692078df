// Rank-k updates of the factor (cldl_updown; device code, included by ldl.cu).  The plan (UpdownPlan, ldl_plan.h)
// is the upward closure of a pass's columns; k_updown runs it as one persistent dataflow kernel with the progress
// discipline of k_factor_df: tasks are claimed in queue order through an atomic head and only wait on tasks queued
// before them.  The recurrence is Gill, Golub, Murray and Saunders' method C1 for L D L^T + alpha w w^T, per pivot
// column j in elimination order and per column r of the pass in ascending r:
//     p = w[j];  dbar = d_j + alpha_r p^2;  beta = alpha_r p / dbar;  alpha_r <- alpha_r d_j / dbar;  d_j <- dbar
//     rows i below j:  w[i] -= p L_ij;  L_ij += beta w[i]
// A step with p = 0 changes nothing and is skipped.  No floating-point atomics: the bits do not depend on the
// schedule.
#pragma once

#define UD_NT DF_RB        /* threads of a k_updown CTA: one per row of a row task */
#define UD_LDA 65          /* leading dimension of the pivot block in shared memory */

struct UDPlanDev {
  int ntask = 0, n = 0;
  const int4* tasks = nullptr;      // 2 x int4 per task: UDTask
  int* pend = nullptr;              // [reached] reached children still running
  int* rows_left = nullptr;         // [reached] row tasks still running
  int* done = nullptr;              // [reached] 1 when the pivot block's (p, beta) are published
  int* qhead = nullptr;
  double* alpha = nullptr;          // [UD_PASS]
  double* w = nullptr;              // [UD_PASS][n] permuted work vectors
  double* pb = nullptr;             // [slot][CB_PB_MAXNS][UD_PASS] (p, beta)
  int* stat = nullptr;              // UD_FAIL, UD_ZERO, UD_DPOS
};
enum { UD_FAIL = 0, UD_ZERO = 1, UD_DPOS = 2, UD_NSTAT = 4 };

// v = vals[pos[t]] plus, in list order (ascending column r), (sigma[r] * wv[a]) * wv[b], each operation rounded once
__global__ void k_ud_values(int npos, const int* __restrict__ pos, const int* __restrict__ ptr, const int* __restrict__ c,
                            const double* __restrict__ sigma, const double* __restrict__ wv, double* __restrict__ vals) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= npos) return;
  double v = vals[pos[t]];
  for (int e = ptr[t]; e < ptr[t + 1]; e++) {
#ifdef CB_EMU    /* the host build contracts a * b + c into an fma; the volatile stores keep one rounding each */
    volatile double a = sigma[c[3 * e]] * wv[c[3 * e + 1]];
    volatile double b = a * wv[c[3 * e + 2]];
    v = v + b;
#else
    v = __dadd_rn(v, __dmul_rn(__dmul_rn(sigma[c[3 * e]], wv[c[3 * e + 1]]), wv[c[3 * e + 2]]));
#endif
  }
  vals[pos[t]] = v;
}

// the work vectors at the pivots of the reached fronts, for the columns of their masks: zero (one warp per front)
__global__ void __launch_bounds__(256) k_ud_zero(LDLDev d, int count, const int* __restrict__ fronts,
                                                 const int* __restrict__ mask, int n, double* __restrict__ w) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= count) return;
  const int s = fronts[i], f = d.sn_first[s], ns = d.sn_first[s + 1] - f;
  for (int r = 0; r < UD_PASS; r++)
    if ((mask[i] >> r) & 1)
      for (int j = lane; j < ns; j += 32) w[(size_t)r * n + f + j] = 0.0;
}

// w[r][pos] = wv[src] for the (r, pos, src) triples of the pass
__global__ void k_ud_scatter(int cnt, const int* __restrict__ e, const double* __restrict__ wv, int n, double* __restrict__ w) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < cnt) w[(size_t)e[3 * t] * n + e[3 * t + 1]] = wv[e[3 * t + 2]];
}

// The pivot block of front s: its L11 in shared memory (wide fronts store L11^-1: recovered by pivot_inverse, and
// inverted again at the end), the recurrence run by warp 0 with lane l owning pivot rows l and l + 32 (p reaches the
// lanes by shuffle, every lane computes the scalars alike), (p, beta) per (pivot, column) left in sPB.  Each updated
// pivot gets the verdict of the refactor's pivot site: not finite, or with regularisation the sign test, or with a
// null-pivot threshold |dbar| <= tol fails; an exact zero with regularisation off is a zero pivot; the change of the
// positive count is summed in an int.
__device__ void ud_pivots(const LDLDev& d, const UDPlanDev& q, const UDTask& tk, double* sA, double* sPB) {
  const int tid = threadIdx.x, s = tk.s;
  const int f = d.sn_first[s], ns = d.sn_first[s + 1] - f;
  const int ld = ns + (int)(d.sn_rowptr[s + 1] - d.sn_rowptr[s]);
  double* P = d.L + d.panel_off[s];
  const bool wide = ns > CB_SOLVE_SMALL_NS;
  for (int idx = tid; idx < ns * ns; idx += UD_NT) {
    const int j = idx / ns, i = idx - j * ns;
    sA[j * UD_LDA + i] = P[(long long)j * ld + i];
  }
  __syncthreads();
  if (wide) {
    pivot_inverse<UD_NT>(sA, UD_LDA, ns);
    __syncthreads();
    pivot_inverse_place<UD_NT>(sA, UD_LDA, ns);
    __syncthreads();
  }
  if (tid < 32) {
    const int lane = tid;
    const unsigned m = (unsigned)tk.mask;
    double w0[UD_PASS], w1[UD_PASS], al[UD_PASS];
#pragma unroll
    for (int r = 0; r < UD_PASS; r++) {
      const bool on = (m >> r) & 1;
      w0[r] = on && lane < ns ? __ldcg(q.w + (size_t)r * q.n + f + lane) : 0.0;
      w1[r] = on && lane + 32 < ns ? __ldcg(q.w + (size_t)r * q.n + f + lane + 32) : 0.0;
      al[r] = on ? __ldcg(q.alpha + r) : 0.0;
    }
    int fail = 0, zero = 0, dpos = 0;
    for (int j = 0; j < ns; j++) {
      const double d0 = d.D[f + j];
      double dj = d0;
      bool upd = false;
      double* cj = sA + j * UD_LDA;
#pragma unroll
      for (int r = 0; r < UD_PASS; r++) {
        double p = 0.0, beta = 0.0;
        if ((m >> r) & 1) {
          p = __shfl_sync(0xffffffffu, j < 32 ? w0[r] : w1[r], j & 31);
          if (p != 0.0) {
            const double ap = al[r] * p;
            const double db = dj + ap * p;
            beta = ap / db;
            al[r] = al[r] * dj / db;
            dj = db;
            upd = true;
            if (lane > j && lane < ns) { const double l = cj[lane]; w0[r] -= p * l; cj[lane] = l + beta * w0[r]; }
            if (lane + 32 > j && lane + 32 < ns) { const double l = cj[lane + 32]; w1[r] -= p * l; cj[lane + 32] = l + beta * w1[r]; }
          }
        }
        if (lane == 0) { sPB[2 * (j * UD_PASS + r)] = p; sPB[2 * (j * UD_PASS + r) + 1] = beta; }
      }
      if (upd && lane == 0) {
        const double inv = 1.0 / dj;
        if (!isfinite(dj) || !isfinite(inv)) fail = 1;
        if (d.reg_enable && dj * (double)d.dsigns[f + j] < d.reg_eps) fail = 1;
        if (d.null_tol > 0.0 && fabs(dj) <= d.null_tol) fail = 1;
        if (!d.reg_enable && dj == 0.0) zero = 1;
        dpos += (dj > 0.0 ? 1 : 0) - (d0 > 0.0 ? 1 : 0);
        d.D[f + j] = dj;
        d.Dinv[f + j] = inv;
        cj[j] = dj;
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int r = 0; r < UD_PASS; r++)
        if ((m >> r) & 1) q.alpha[r] = al[r];
      if (fail) atomicExch(q.stat + UD_FAIL, 1);
      if (zero) atomicExch(q.stat + UD_ZERO, 1);
      if (dpos) atomicAdd(q.stat + UD_DPOS, dpos);
    }
  }
  __syncthreads();
  if (wide) {
    pivot_inverse<UD_NT>(sA, UD_LDA, ns);
    __syncthreads();
    pivot_inverse_place<UD_NT>(sA, UD_LDA, ns);
    __syncthreads();
  }
  for (int idx = tid; idx < ns * ns; idx += UD_NT) {
    const int j = idx / ns, i = idx - j * ns;
    if (i >= j) P[(long long)j * ld + i] = sA[j * UD_LDA + i];
  }
  if (tk.kind == 1)
    for (int idx = tid; idx < ns * UD_PASS * 2; idx += UD_NT) q.pb[(size_t)tk.slot * CB_PB_MAXNS * UD_PASS * 2 + idx] = sPB[idx];
}

// rows [r0, r1) below the pivot block, one thread each: the columns' work-vector entries in registers, the row of L21
// read and written once per pivot
__device__ void ud_rows(const LDLDev& d, const UDPlanDev& q, const UDTask& tk, const double* sPB) {
  const int i = tk.r0 + (int)threadIdx.x;
  if (i >= tk.r1) return;
  const int s = tk.s;
  const int f = d.sn_first[s], ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int ld = ns + (int)(d.sn_rowptr[s + 1] - rp);
  const int row = d.sn_rows[rp + i];
  const unsigned m = (unsigned)tk.mask;
  double w[UD_PASS];
#pragma unroll
  for (int r = 0; r < UD_PASS; r++) w[r] = (m >> r) & 1 ? __ldcg(q.w + (size_t)r * q.n + row) : 0.0;
  double* pl = d.L + d.panel_off[s] + ns + i;
  for (int j = 0; j < ns; j++) {
    double l = pl[(long long)j * ld];
#pragma unroll
    for (int r = 0; r < UD_PASS; r++) {
      const double p = sPB[2 * (j * UD_PASS + r)];
      if (((m >> r) & 1) && p != 0.0) {
        w[r] -= p * l;
        l += sPB[2 * (j * UD_PASS + r) + 1] * w[r];
      }
    }
    pl[(long long)j * ld] = l;
  }
#pragma unroll
  for (int r = 0; r < UD_PASS; r++)
    if ((m >> r) & 1) q.w[(size_t)r * q.n + row] = w[r];
}

__global__ void __launch_bounds__(UD_NT) k_updown(LDLDev d, UDPlanDev q) {
  __shared__ double sA[CB_PB_MAXNS * UD_LDA];
  __shared__ double sPB[CB_PB_MAXNS * UD_PASS * 2];
  __shared__ __align__(16) int s_task[8];
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
    if (tid < 2) reinterpret_cast<int4*>(s_task)[tid] = q.tasks[2 * (size_t)qi + tid];
    __syncthreads();
    const UDTask tk = *reinterpret_cast<const UDTask*>(s_task);
    if (tk.kind != 2) {
      if (tid == 0) { df_wait_zero(q.pend + tk.li); __threadfence(); }
      __syncthreads();
      ud_pivots(d, q, tk, sA, sPB);
      __syncthreads();
      if (tk.kind == 0) {
        ud_rows(d, q, tk, sPB);
        __syncthreads();
        if (tid == 0) { __threadfence(); if (tk.pli >= 0) atomicSub(q.pend + tk.pli, 1); }
      } else if (tid == 0) {
        __threadfence();
        atomicExch(q.done + tk.li, 1);
      }
    } else {
      if (tid == 0) { df_wait_set(q.done + tk.li); __threadfence(); }
      __syncthreads();
      const int ns = d.sn_first[tk.s + 1] - d.sn_first[tk.s];
      for (int idx = tid; idx < ns * UD_PASS * 2; idx += UD_NT)
        sPB[idx] = __ldcg(q.pb + (size_t)tk.slot * CB_PB_MAXNS * UD_PASS * 2 + idx);
      __syncthreads();
      ud_rows(d, q, tk, sPB);
      __syncthreads();
      if (tid == 0) {
        __threadfence();
        if (atomicSub(q.rows_left + tk.li, 1) == 1 && tk.pli >= 0) atomicSub(q.pend + tk.pli, 1);
      }
    }
  }
}
