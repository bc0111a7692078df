// Triangular solves of the multifrontal LDL^T (device code, included by ldl.cu).
//
//   x <- b[perm];  forward: L y = x (leaves -> root);  backward: x = L^-T D^-1 y (root -> leaves);  out[perm] <- x
//   (reference: qdldl.rs:116-138 solve, :708-719 _lsolve, :737-752 _dltsolve -- column by column on one thread)
//
// Layout the sweeps rely on.  A front s with ns pivots and nr rows below stores its panel (ns+nr) x ns column-major
// in d.L.  For wide fronts (ns > CB_SOLVE_SMALL_NS) the strictly lower triangle of the pivot block holds
// L11^-1 (unit diagonal implied), written by the factorisation where it has the pivot block: the ns dependent
// substitution steps of a pivot block become one ns x ns matrix-vector product.  Narrow fronts keep L11.
//
// Schedule.  Tree level 0 has no dependencies: its narrow fronts are swept by plain kernels before (forward) and
// after (backward) the dataflow kernel -- one THREAD per single-column front, one warp per front otherwise.
// Everything else is ONE persistent kernel per sweep; CTAs pull 96-byte task records from a queue in level order:
//   narrow batch   up to 8 narrow fronts, one warp each (substitution in registers / global memory)
//   head           one wide front: pivot block + its first rh rows.  The slab (<= cap doubles) goes to shared memory
//                  with cp.async BEFORE the task waits for its dependencies, so the wait hides the load
//   rows           a further slab of rows of a wide front whose panel exceeds cap: several CTAs stream one front
// Dependencies are counters / flags in global memory (release: stores -> __syncthreads -> one thread fences and
// sets the flag; acquire: one thread spins, fences, __syncthreads, consumers read with ld.global.cg).  A chain
// child (rows(c) = cols(p) + rows(p)) is followed slab by slab: the parent's head starts as soon as the child's
// tasks covering the parent's pivot rows are done.  Every sum has a fixed order: no floating-point atomics, two
// solves of the same right-hand side are bit-identical, and a right-hand side gives the same bits whether it is
// swept alone (NR = 1) or next to a second one (NR = 2: the panels are read once for both).
#pragma once

#include "ldl_solve_plan.h"

__device__ __forceinline__ void sv_cp8(double* smem_dst, const double* gsrc) {
#ifdef CB_EMU
  *smem_dst = *gsrc;
#else
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
#endif
}
__device__ __forceinline__ void sv_cp16(double* smem_dst, const double* gsrc) {   // both 16-byte aligned; bypasses L1
#ifdef CB_EMU
  smem_dst[0] = gsrc[0]; smem_dst[1] = gsrc[1];
#else
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
#endif
}
// ---- TMA bulk copy (cp.async.bulk, completion on an mbarrier): a panel that fits the slab is ONE contiguous block of
// global memory, so one thread hands the whole transfer to the copy engine -- no per-element instructions, no
// registers, no L1.  dst / src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void sv_mbar_init(unsigned long long* mbar) {
#ifndef CB_EMU
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((unsigned)__cvta_generic_to_shared(mbar)) : "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}
__device__ __forceinline__ void sv_bulk_load(double* smem_dst, const double* gsrc, unsigned bytes, unsigned long long* mbar) {
#ifdef CB_EMU
  for (unsigned i = 0; i < bytes / 8; i++) smem_dst[i] = gsrc[i];
#else
  const unsigned mb = (unsigned)__cvta_generic_to_shared(mbar);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // earlier generic-proxy reads of the slab are ordered before the engine's writes
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc), "r"(bytes), "r"(mb) : "memory");
#endif
}
__device__ __forceinline__ void sv_mbar_wait(unsigned long long* mbar, unsigned phase) {
#ifndef CB_EMU
  const unsigned mb = (unsigned)__cvta_generic_to_shared(mbar);
  unsigned ok = 0;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(mb), "r"(phase) : "memory");
  } while (!ok);
#endif
}
__device__ __forceinline__ void sv_cp_commit_wait() {
#ifndef CB_EMU
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
#endif
}

// ---- narrow fronts (ns <= CB_SOLVE_SMALL_NS): one warp, substitution ----
__device__ void df_fwd_small(const LDLDev& d, double* __restrict__ u, int s, double* __restrict__ xp, int lane) {
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr;
  const double* __restrict__ P = d.L + d.panel_off[s];
  double* us = u + rp;
  const int* __restrict__ gp = d.gat_ptr + (f + rp);
  for (int p = lane; p < ld; p += 32) {
    double acc = 0.0;
    for (int e = gp[p]; e < gp[p + 1]; e++) acc += __ldcg(u + d.gat_src[e]);
    if (p < ns) xp[f + p] += acc; else us[p - ns] = acc;
  }
  __syncwarp();
  for (int j = 0; j + 1 < ns; j++) {
    const double xj = xp[f + j];
    for (int i = j + 1 + lane; i < ns; i += 32) xp[f + i] -= P[(long long)j * ld + i] * xj;
    __syncwarp();
  }
  for (int a = lane; a < nr; a += 32) {
    double acc = 0.0;
    for (int j = 0; j < ns; j++) acc += P[(long long)j * ld + ns + a] * xp[f + j];
    us[a] -= acc;
  }
}

__device__ void df_bwd_small(const LDLDev& d, int s, double* __restrict__ xp, double* __restrict__ out, int lane) {
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr;
  const double* __restrict__ P = d.L + d.panel_off[s];
  const int* __restrict__ rows = d.sn_rows + rp;
  if (nr <= 8 * 32) {
    // the ancestors' solution entries this front needs are fetched once (index -> value is a dependent pair of loads)
    double xv[8];
#pragma unroll
    for (int q8 = 0; q8 < 8; q8++) {
      const int a = lane + 32 * q8;
      xv[q8] = a < nr ? __ldcg(xp + rows[a]) : 0.0;
    }
    for (int j = 0; j < ns; j++) {
      const double* __restrict__ cj = P + (long long)j * ld + ns;
      double acc = 0.0;
#pragma unroll
      for (int q8 = 0; q8 < 8; q8++) {
        const int a = lane + 32 * q8;
        if (a < nr) acc += cj[a] * xv[q8];
      }
      __syncwarp();
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) xp[f + j] = xp[f + j] * d.Dinv[f + j] - acc;
    }
  } else {
    for (int j = 0; j < ns; j++) {
      const double* __restrict__ cj = P + (long long)j * ld + ns;
      double acc = 0.0;
      for (int a = lane; a < nr; a += 32) acc += cj[a] * __ldcg(xp + rows[a]);
      __syncwarp();   // lanes leave the strided loop at different trip counts: reconverge before the shuffles
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) xp[f + j] = xp[f + j] * d.Dinv[f + j] - acc;
    }
  }
  __syncwarp();
  for (int j = ns - 1; j > 0; j--) {
    const double xj = xp[f + j];
    for (int i = lane; i < j; i += 32) xp[f + i] -= P[(long long)i * ld + j] * xj;
    __syncwarp();
  }
  for (int j = lane; j < ns; j += 32) out[d.perm[f + j]] = xp[f + j];
}

// ---- tree level 0, narrow fronts: no dependencies, plain kernels around the dataflow sweep ----
// single-column leaves: one thread per front (ones[] lists them)
template <int NR>
__global__ void __launch_bounds__(256) k_fwd_leaf1(LDLDev d, const int* __restrict__ ones, int count, SVRhs r) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const int s = ones[i];
  const int f = d.sn_first[s];
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const double* __restrict__ P = d.L + d.panel_off[s] + 1;
#pragma unroll
  for (int h = 0; h < NR; h++) {
    const double x = r.xp[h][f];
    double* us = r.u[h] + rp;
    for (int a = 0; a < nr; a++) us[a] = -(P[a] * x);
  }
}
template <int NR>
__global__ void __launch_bounds__(256) k_bwd_leaf1(LDLDev d, const int* __restrict__ ones, int count, SVRhs r) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const int s = ones[i];
  const int f = d.sn_first[s];
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const double* __restrict__ P = d.L + d.panel_off[s] + 1;
  const int* __restrict__ rows = d.sn_rows + rp;
  const double di = d.Dinv[f];
  const int pf = d.perm[f];
#pragma unroll
  for (int h = 0; h < NR; h++) {
    double acc = 0.0;
    for (int a = 0; a < nr; a++) acc += P[a] * r.xp[h][rows[a]];
    const double x = r.xp[h][f] * di - acc;
    r.xp[h][f] = x;
    r.out[h][pf] = x;
  }
}
// other narrow leaves: one warp per front
template <int NR, bool FWD>
__global__ void __launch_bounds__(256) k_leaf_small(LDLDev d, const int* __restrict__ list, int count, SVRhs r) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= count) return;
  const int s = list[w];
#pragma unroll
  for (int h = 0; h < NR; h++) {
    if (FWD) df_fwd_small(d, r.u[h], s, r.xp[h], lane);
    else df_bwd_small(d, s, r.xp[h], r.out[h], lane);
    __syncwarp();
  }
}

// wide leaves (ns > CB_SOLVE_SMALL_NS, no children): one CTA of 128 threads per front, straight from global memory --
// nothing to wait for, nothing to gather; many CTAs per SM hide the latency.  Same arithmetic, in the same order, as a
// head task of the dataflow kernel would do for the front.
#define SV_LEAF_NT 128
#define SV_POLL 64          /* thread of a sweep CTA that polls the dependencies (thread 0 publishes the previous task meanwhile) */
template <int NR>
__global__ void __launch_bounds__(SV_LEAF_NT) k_fwd_leafw(LDLDev d, const int* __restrict__ list, int count, SVRhs r) {
  __shared__ double sb[NR * CB_PB_MAXNS], sy[NR * CB_PB_MAXNS];
  {
  const int s = list[blockIdx.x];
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr, tid = threadIdx.x;
  const double* __restrict__ P = d.L + d.panel_off[s];
  __syncthreads();            // the previous front's readers of sb / sy are done
  if (tid < ns) {
#pragma unroll
    for (int h = 0; h < NR; h++) sb[h * CB_PB_MAXNS + tid] = r.xp[h][f + tid] + 0.0;
  }
  __syncthreads();
  if (tid < ns) {
    double y[NR];
#pragma unroll
    for (int h = 0; h < NR; h++) y[h] = sb[h * CB_PB_MAXNS + tid];
    for (int j = 0; j < tid; j++) {
      const double l = P[(long long)j * ld + tid];
#pragma unroll
      for (int h = 0; h < NR; h++) y[h] += l * sb[h * CB_PB_MAXNS + j];
    }
#pragma unroll
    for (int h = 0; h < NR; h++) { sy[h * CB_PB_MAXNS + tid] = y[h]; r.xp[h][f + tid] = y[h]; }
  }
  __syncthreads();
  for (int a = tid; a < nr; a += SV_LEAF_NT) {
    double acc[NR];
#pragma unroll
    for (int h = 0; h < NR; h++) acc[h] = 0.0;
    const double* __restrict__ col = P + ns + a;
    for (int j = 0; j < ns; j++) {
      const double l = col[(long long)j * ld];
#pragma unroll
      for (int h = 0; h < NR; h++) acc[h] += l * sy[h * CB_PB_MAXNS + j];
    }
#pragma unroll
    for (int h = 0; h < NR; h++) r.u[h][rp + a] = 0.0 - acc[h];
  }
  }
}
// backward: warp w owns the columns j = w, w + 4, ...; lanes run down a column (coalesced), one butterfly per column
template <int NR>
__global__ void __launch_bounds__(SV_LEAF_NT) k_bwd_leafw(LDLDev d, const int* __restrict__ list, int count, SVRhs r, int nr_max) {
  extern __shared__ double lw_smem[];
  double* sx = lw_smem;                        // NR * nr_max: x at the front's rows
  double* st = sx + NR * nr_max;               // NR * 64
  __shared__ double s0[NR * CB_PB_MAXNS];      // D^-1 y of the pivots, then the solution (written out together at the end)
  {
  const int s = list[blockIdx.x];
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const double* __restrict__ P = d.L + d.panel_off[s];
  const int* __restrict__ rows = d.sn_rows + rp;
  __syncthreads();            // the previous front's readers of the shared vectors are done
  for (int a = tid; a < nr; a += SV_LEAF_NT) {
    const int ri = rows[a];
#pragma unroll
    for (int h = 0; h < NR; h++) sx[h * nr_max + a] = r.xp[h][ri];
  }
  if (tid < ns) {
    const double di = d.Dinv[f + tid];
#pragma unroll
    for (int h = 0; h < NR; h++) s0[h * CB_PB_MAXNS + tid] = r.xp[h][f + tid] * di;
  }
  __syncthreads();
  for (int j = w; j < ns; j += SV_LEAF_NT / 32) {
    const double* __restrict__ col = P + (long long)j * ld + ns;
    double acc[NR];
#pragma unroll
    for (int h = 0; h < NR; h++) acc[h] = 0.0;
    for (int a = lane; a < nr; a += 32) {
      const double l = col[a];
#pragma unroll
      for (int h = 0; h < NR; h++) acc[h] += l * sx[h * nr_max + a];
    }
    __syncwarp();
#pragma unroll
    for (int h = 0; h < NR; h++) {
      double t = acc[h];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (lane == 0) st[h * CB_PB_MAXNS + j] = s0[h * CB_PB_MAXNS + j] - t;
    }
  }
  __syncthreads();
  // x1 = L11^-T t: column i of the inverse below its diagonal, lanes down the column
  for (int i = w; i < ns; i += SV_LEAF_NT / 32) {
    const double* __restrict__ col = P + (long long)i * ld;
    double acc[NR];
#pragma unroll
    for (int h = 0; h < NR; h++) acc[h] = 0.0;
    for (int j = i + 1 + lane; j < ns; j += 32) {
      const double l = col[j];
#pragma unroll
      for (int h = 0; h < NR; h++) acc[h] += l * st[h * CB_PB_MAXNS + j];
    }
    __syncwarp();
#pragma unroll
    for (int h = 0; h < NR; h++) {
      double t = acc[h];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (lane == 0) s0[h * CB_PB_MAXNS + i] = st[h * CB_PB_MAXNS + i] + t;
    }
  }
  __syncthreads();
  if (tid < ns) {
    const int pf = d.perm[f + tid];
#pragma unroll
    for (int h = 0; h < NR; h++) { const double x = s0[h * CB_PB_MAXNS + tid]; r.xp[h][f + tid] = x; r.out[h][pf] = x; }
  }
  }
}

// ---- the dataflow sweep ----
// Flags and counters between CTAs.  Publishing: all threads store their results, __syncthreads, then ONE thread issues
// a release operation at device scope (st.release / red.release: the ordering travels with the operation, the thread
// does not stall on a fence and is free for the next task at once).  Consuming: one thread polls with ld.acquire,
// __syncthreads, then everybody reads (ld.global.cg: L1 is not coherent).
__device__ __forceinline__ int sv_ld_acquire(const int* p) {
#ifdef CB_EMU
  return *(volatile const int*)p;
#else
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ void sv_set_release(int* p) {          // *p = 1
#ifdef CB_EMU
  __threadfence(); atomicExch(p, 1);
#else
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(1) : "memory");
#endif
}
__device__ __forceinline__ void sv_dec_release(int* p) {          // *p -= 1, result not needed
#ifdef CB_EMU
  __threadfence(); atomicSub(p, 1);
#else
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(-1) : "memory");
#endif
}
__device__ __forceinline__ int sv_dec_acq_rel(int* p) {           // returns the value before the decrement
#ifdef CB_EMU
  __threadfence(); return atomicSub(p, 1);
#else
  int v;
  asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], %2;" : "=r"(v) : "l"(p), "r"(-1) : "memory");
  return v;
#endif
}
__device__ __forceinline__ void sv_wait_zero(const int* p) {
  unsigned ns = 20;
  while (sv_ld_acquire(p) > 0) { __nanosleep(ns); if (ns < 320) ns <<= 1; }
}
__device__ __forceinline__ void sv_wait_set(const int* p) {
  unsigned ns = 20;
  while (sv_ld_acquire(p) == 0) { __nanosleep(ns); if (ns < 320) ns <<= 1; }
}

// slab -> shared memory, column-major with leading dimension lds: columns [0, ns), `rows` panel rows starting at src0.
// lds has the parity of ld and the slab starts at an element whose parity is that of src0's offset in d.L (see
// sv_lds / boff at the call site), so source and destination of every column are 16-byte aligned at the same
// elements: the body of a column goes in 16-byte cp.async.cg pieces (L2 only), a leading / trailing single in 8 bytes.
__device__ __forceinline__ void sv_stage(double* sl, int boff, const double* __restrict__ src0, int ld, int ns, int rows, int lds) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = warp; j < ns; j += SV_NT / 32) {
    const double* __restrict__ src = src0 + (long long)j * ld;
    double* dst = sl + j * lds;
    const int i0 = (boff + j * lds) & 1;                 // first element of the column that is 16-byte aligned
    if (i0 && lane == 0 && rows > 0) sv_cp8(dst, src);
    const int npairs = (rows - i0) >> 1;
    for (int t = lane; t < npairs; t += 32) sv_cp16(dst + i0 + 2 * t, src + i0 + 2 * t);
    if (((rows - i0) & 1) && rows > i0 && lane == 31) sv_cp8(dst + rows - 1, src + rows - 1);
  }
}

template <bool FWD, int NR>
__global__ void __launch_bounds__(SV_NT, SV_MINB) k_solve2(LDLDev d, SVPlan q, SVRhs r, int cap) {
  extern __shared__ __align__(16) double sv_smem[];
  double* slab = sv_smem;                       // cap doubles (+ 2 of slack: a bulk copy is rounded up to 16 bytes)
  double* sw = slab + cap + 2;                  // NR * 64: gathered right-hand side of the pivot block / D^-1 y - sums
  double* sy = sw + NR * CB_PB_MAXNS;           // NR * 64: pivot solution
  double* sx = sy + NR * CB_PB_MAXNS;           // NR * SV_MAXROWS: backward, x at the slab's rows
  double* sred = sx + NR * SV_MAXROWS;          // NR * 4 * 64: backward, partial column sums of the four row quarters
  // The queue is read one task ahead: the next index and its 96-byte record are fetched by warp 1 while the current
  // task computes (an atomic + a dependent load, ~1.5 us of pure latency otherwise).  The fetch is issued only AFTER
  // the current task's dependency wait: a task that is being held back must not hold a second one back with it.
  // Holding a fetched task for the few microseconds of a compute phase is safe: dependencies point to earlier queue
  // positions only.
  __shared__ int4 s_rec[2][6];
  __shared__ int s_task[2];
  __shared__ __align__(8) unsigned long long s_mbar;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int cur = 0;
  unsigned mph = 0;                              // phase of the bulk-copy barrier: flips with every bulk copy (all threads see the same tasks)
  if (tid == 0) sv_mbar_init(&s_mbar);
  if (tid == 0) s_task[0] = atomicAdd(&q.qhead[FWD ? 0 : 1], 1);
  __syncthreads();
  {
    const int q0 = s_task[0];
    if (q0 < q.ntask && tid < 6) s_rec[0][tid] = q.tasks[6 * (size_t)(FWD ? q0 : q.ntask - 1 - q0) + tid];
  }
  __syncthreads();
  // three steps, spread over the task so that no step waits for the previous one's memory round trip: index (atomic),
  // record (dependent load), record -> shared memory.  Warp 7 does it: its threads have the least other work.
  int fq = 0;
  int4 frec = make_int4(0, 0, 0, 0);
#define SV_FETCH1() do { if (tid == SV_NT - 32) fq = atomicAdd(&q.qhead[FWD ? 0 : 1], 1); } while (0)
#define SV_FETCH2()                                                                                     \
  do {                                                                                                  \
    if (warp == SV_NT / 32 - 1) {                                                                       \
      fq = __shfl_sync(0xffffffffu, fq, 0);                                                             \
      if (lane == 0) s_task[cur ^ 1] = fq;                                                              \
      if (fq < q.ntask && lane < 6) frec = q.tasks[6 * (size_t)(FWD ? fq : q.ntask - 1 - fq) + lane];   \
    }                                                                                                   \
  } while (0)
#define SV_FETCH3() do { if (warp == SV_NT / 32 - 1 && lane < 6 && fq < q.ntask) s_rec[cur ^ 1][lane] = frec; } while (0)
#define SV_FETCH_NEXT() do { SV_FETCH1(); SV_FETCH2(); SV_FETCH3(); } while (0)
  for (;;) {
    // no barrier here: every path below ends with a barrier that follows all reads of the slab and the vectors, and
    // what comes after it (thread 0 publishing the finished task) overlaps with the staging of the next one
    const int qi = s_task[cur];
    if (qi >= q.ntask) break;
    const int k = FWD ? qi : q.ntask - 1 - qi;
    unsigned long long* trk = q.trace ? q.trace + 4 * ((size_t)(FWD ? 0 : q.ntask) + k) : nullptr;
    if (trk && tid == 0) trk[0] = df_gtime();
    const SVTask& T = *reinterpret_cast<const SVTask*>(s_rec[cur]);
    const int kind = T.kind;
    if (kind == 0) {
      // ---------------- batch of narrow fronts ----------------
      const int first = T.s, cnt = T.cnt;
      if (FWD) {
        if (tid == SV_POLL) { sv_wait_zero(q.pend + k); if (trk) trk[1] = df_gtime(); }
        __syncthreads();
        SV_FETCH_NEXT();
        if (warp < cnt) {
#pragma unroll
          for (int h = 0; h < NR; h++) { df_fwd_small(d, r.u[h], q.fronts[first + warp], r.xp[h], lane); __syncwarp(); }
        }
        __syncthreads();
        if (tid < cnt) {
          const int p = q.parent[q.fronts[first + tid]];
          if (p >= 0) sv_dec_release(q.pend + q.front2task[p]);
        }
      } else {
        __syncthreads();
        SV_FETCH_NEXT();
        if (warp < cnt) {
          const int s = q.fronts[first + warp];
          if (lane == 0) { const int p = q.parent[s]; if (p >= 0) sv_wait_set(q.done + p); }
          __syncwarp();
#pragma unroll
          for (int h = 0; h < NR; h++) { df_bwd_small(d, s, r.xp[h], r.out[h], lane); __syncwarp(); }
          if (lane == 0) sv_set_release(q.done + s);
        }
        __syncthreads();
      }
      if (trk && tid == 0) trk[2] = df_gtime();
      cur ^= 1;
      continue;
    }
    // ---------------- wide front: head (pivot block + first rows) or a further slab of rows ----------------
    const int s = T.s, f = T.f, ns = T.ns, nr = T.nr, r0 = T.r0, r1 = T.r1;
    const int ld = ns + nr;
    const int rows = r1 - r0;                                   // rows of L21 in this slab (<= SV_MAXROWS = SV_NT)
    const bool head = kind == 1;
    const int srows = head ? ns + rows : rows;                  // rows of the staged slab
    const int l21 = head ? ns : 0;                              // where the L21 rows start inside the slab
    const double* __restrict__ P = d.L + T.poff;
    // in flight while the task waits below: the whole panel in one TMA bulk copy when it fits (it is contiguous),
    // otherwise the slab's piece of every column with 16-byte cp.async
    const bool contig = head && rows == nr;
    const int row0 = head ? 0 : ns + r0;
    const int lds = contig ? ld : sv_lds(srows, ld);
    const int boff = contig ? 0 : (int)((T.poff + row0) & 1);
    double* const sl = slab + boff;
    if (contig) { if (tid == SV_POLL) sv_bulk_load(slab, P, (unsigned)(((ns * ld + 1) & ~1) * 8), &s_mbar); }
    else sv_stage(sl, boff, P + row0, ld, ns, srows, lds);
#define SV_SLAB_WAIT() do { if (contig) { sv_mbar_wait(&s_mbar, mph); mph ^= 1; } else sv_cp_commit_wait(); } while (0)
    const long long rp = T.rp;
    if (FWD) {
      const int* __restrict__ gp = d.gat_ptr + (f + rp);
      const bool pure = T.pure != 0;
      const int nrt = T.nrt, dep0 = T.dep0, dep1 = T.dep1, dep2 = T.dep2, t_notify = T.notify, t_ptask = T.ptask;
      const long long cuoff = T.cuoff;
      const bool rows_late = head && dep2 > dep1;               // the rows' contributions arrive after the pivots' (chain child followed slab by slab)
      // static gather lists: ranges and the first two source indices of every destination are fetched before the wait
      int ga0 = 0, ga1 = 0, gai0 = 0, gai1 = 0, gb0 = 0, gb1 = 0, gbi0 = 0, gbi1 = 0;
      if (!pure) {
        if (head && tid < ns) { ga0 = gp[tid]; ga1 = gp[tid + 1]; }
        if (tid < rows) { gb0 = gp[ns + r0 + tid]; gb1 = gp[ns + r0 + tid + 1]; }
        if (ga1 > ga0) gai0 = d.gat_src[ga0];
        if (ga1 > ga0 + 1) gai1 = d.gat_src[ga0 + 1];
        if (gb1 > gb0) gbi0 = d.gat_src[gb0];
        if (gb1 > gb0 + 1) gbi1 = d.gat_src[gb0 + 1];
      }
      if (tid == SV_POLL) {     // not thread 0: that one may still be publishing the previous task
        if (head) sv_wait_zero(q.pend + k); else sv_wait_set(q.ydone + s);
        for (int t = dep0; t <= dep1; t++) sv_wait_set(q.tdone + t);
        if (trk) trk[1] = df_gtime();
      }
      __syncthreads();
      SV_FETCH1();
      // children's contributions to the slab's rows -> sx (phase B reads them with a different thread mapping)
      auto gather_rows = [&]() {
        if (tid < rows) {
#pragma unroll
          for (int h = 0; h < NR; h++) {
            double acc = 0.0;
            if (pure) acc = __ldcg(r.u[h] + cuoff + ns + r0 + tid);
            else {
              if (gb1 > gb0) acc += __ldcg(r.u[h] + gbi0);
              if (gb1 > gb0 + 1) acc += __ldcg(r.u[h] + gbi1);
              for (int e = gb0 + 2; e < gb1; e++) acc += __ldcg(r.u[h] + d.gat_src[e]);
            }
            sx[h * SV_MAXROWS + tid] = acc;
          }
        }
      };
      // the dot products of both phases are split four ways: thread (i, q) = (tid / 4, tid % 4) takes the terms
      // j = q, q + 4, ... of row i, the quad adds its partial sums with two shuffles (fixed order)
      const int qi_row = tid >> 2, qd = tid & 3;
      if (head) {
        // phase A: y1 = L11^-1 (b1 + children)
        if (tid < ns) {
#pragma unroll
          for (int h = 0; h < NR; h++) {
            double acc = 0.0;
            if (pure) acc = __ldcg(r.u[h] + cuoff + tid);
            else {
              if (ga1 > ga0) acc += __ldcg(r.u[h] + gai0);
              if (ga1 > ga0 + 1) acc += __ldcg(r.u[h] + gai1);
              for (int e = ga0 + 2; e < ga1; e++) acc += __ldcg(r.u[h] + d.gat_src[e]);
            }
            sw[h * CB_PB_MAXNS + tid] = r.xp[h][f + tid] + acc;
          }
        }
        if (!rows_late) gather_rows();          // issued now, consumed in phase B
        SV_SLAB_WAIT();
        __syncthreads();
        if (trk && tid == 0) trk[3] = df_gtime();
        {
          double y[NR];
#pragma unroll
          for (int h = 0; h < NR; h++) y[h] = 0.0;
          if (qi_row < ns) {
            for (int j = qd; j < qi_row; j += 4) {
              const double l = sl[j * lds + qi_row];
#pragma unroll
              for (int h = 0; h < NR; h++) y[h] += l * sw[h * CB_PB_MAXNS + j];
            }
          }
          __syncwarp();
#pragma unroll
          for (int h = 0; h < NR; h++) {
            y[h] += __shfl_xor_sync(0xffffffffu, y[h], 1);
            y[h] += __shfl_xor_sync(0xffffffffu, y[h], 2);
            if (qd == 0 && qi_row < ns) { const double v = sw[h * CB_PB_MAXNS + qi_row] + y[h]; sy[h * CB_PB_MAXNS + qi_row] = v; r.xp[h][f + qi_row] = v; }
          }
        }
        __syncthreads();
        SV_FETCH2();
        if (tid == 0) {
          if (nrt > 0) sv_set_release(q.ydone + s);
          if (rows_late) { for (int t = max(dep1 + 1, dep0); t <= dep2; t++) sv_wait_set(q.tdone + t); }
        }
        if (rows_late) { __syncthreads(); gather_rows(); __syncthreads(); }
      } else {
        if (tid < ns) {
#pragma unroll
          for (int h = 0; h < NR; h++) sy[h * CB_PB_MAXNS + tid] = __ldcg(r.xp[h] + f + tid);
        }
        gather_rows();
        SV_SLAB_WAIT();
        __syncthreads();
        SV_FETCH2();
      }
      // phase B: u[rows] = children - L21 y1, 64 rows per pass
      for (int base = 0; base < rows; base += SV_NT / 4) {
        const int a = base + qi_row;
        double acc[NR];
#pragma unroll
        for (int h = 0; h < NR; h++) acc[h] = 0.0;
        if (a < rows) {
          const double* __restrict__ col = sl + l21 + a;
          for (int j = qd; j < ns; j += 4) {
            const double l = col[j * lds];
#pragma unroll
            for (int h = 0; h < NR; h++) acc[h] += l * sy[h * CB_PB_MAXNS + j];
          }
        }
        __syncwarp();
#pragma unroll
        for (int h = 0; h < NR; h++) {
          acc[h] += __shfl_xor_sync(0xffffffffu, acc[h], 1);
          acc[h] += __shfl_xor_sync(0xffffffffu, acc[h], 2);
          if (qd == 0 && a < rows) r.u[h][rp + r0 + a] = sx[h * SV_MAXROWS + a] - acc[h];
        }
      }
      SV_FETCH3();
      __syncthreads();
      if (tid == 0) {
        sv_set_release(q.tdone + k);
        // a front that is one task needs no count of its tasks: the parent hears of it at once (no atomic round trip)
        if (nrt == 0) { if (t_notify && t_ptask >= 0) sv_dec_release(q.pend + t_ptask); }
        else if (sv_dec_acq_rel(q.fleft + s) == 1 && t_notify && t_ptask >= 0) sv_dec_release(q.pend + t_ptask);
        if (trk) trk[2] = df_gtime();
      }
    } else {
      // ---------------- backward ----------------
      const int* __restrict__ rowsi = d.sn_rows + rp + r0;
      const int nrt = T.nrt, bowner = T.bowner, bslot = T.bslot;
      const int ri = tid < rows ? rowsi[tid] : 0;               // static: before the wait
      const int pf = (head && tid < ns) ? d.perm[f + tid] : 0;
      const double di = (head && tid < ns) ? d.Dinv[f + tid] : 0.0;
      if (tid == SV_POLL) {
        if (head && nrt > 0) sv_wait_zero(q.bleft + s);
        if (bowner >= 0) sv_wait_set(q.done + bowner);
        if (trk) trk[1] = df_gtime();
      }
      __syncthreads();
      SV_FETCH1();
      if (tid < rows) {
#pragma unroll
        for (int h = 0; h < NR; h++) sx[h * SV_MAXROWS + tid] = __ldcg(r.xp[h] + ri);
      }
      double part[NR];                                          // head: sum of the row tasks' partial column sums (fixed order)
#pragma unroll
      for (int h = 0; h < NR; h++) part[h] = 0.0;
      if (head && tid < ns) {
#pragma unroll
        for (int h = 0; h < NR; h++) {
          sw[h * CB_PB_MAXNS + tid] = r.xp[h][f + tid] * di;
          for (int b = 0; b < nrt; b++) part[h] += __ldcg(q.bpart + h * q.bpart_stride + (long long)(bslot + b) * CB_PB_MAXNS + tid);
        }
      }
      SV_SLAB_WAIT();
      __syncthreads();
      {
        // column sums over the slab's rows: thread (j, quarter) walks rows quarter, quarter + 4, ...
        const int j = tid & (CB_PB_MAXNS - 1), qd = tid >> 6;
        double acc[NR];
#pragma unroll
        for (int h = 0; h < NR; h++) acc[h] = 0.0;
        if (j < ns) {
          const double* __restrict__ col = sl + j * lds + l21;
          for (int a = qd; a < rows; a += 4) {
            const double l = col[a];
#pragma unroll
            for (int h = 0; h < NR; h++) acc[h] += l * sx[h * SV_MAXROWS + a];
          }
        }
#pragma unroll
        for (int h = 0; h < NR; h++) sred[(h * 4 + qd) * CB_PB_MAXNS + j] = acc[h];
      }
      SV_FETCH2();
      __syncthreads();
      if (!head) {
        if (tid < ns) {
#pragma unroll
          for (int h = 0; h < NR; h++) {
            const double* sr = sred + h * 4 * CB_PB_MAXNS + tid;
            q.bpart[h * q.bpart_stride + (long long)bslot * CB_PB_MAXNS + tid] =
                ((sr[0] + sr[CB_PB_MAXNS]) + sr[2 * CB_PB_MAXNS]) + sr[3 * CB_PB_MAXNS];
          }
        }
        SV_FETCH3();
        __syncthreads();
        if (tid == 0) { sv_dec_release(q.bleft + s); if (trk) trk[2] = df_gtime(); }
      } else {
        if (tid < ns) {
#pragma unroll
          for (int h = 0; h < NR; h++) {
            const double* sr = sred + h * 4 * CB_PB_MAXNS + tid;
            sy[h * CB_PB_MAXNS + tid] = (sw[h * CB_PB_MAXNS + tid] - (((sr[0] + sr[CB_PB_MAXNS]) + sr[2 * CB_PB_MAXNS]) + sr[3 * CB_PB_MAXNS])) - part[h];
          }
        }
        __syncthreads();
        {
          // x1 = L11^-T t:  x1[i] = t[i] + sum_{j > i} Linv[j][i] t[j], four threads per row
          const int i = tid >> 2, qd4 = tid & 3;
          double x[NR];
#pragma unroll
          for (int h = 0; h < NR; h++) x[h] = 0.0;
          if (i < ns) {
            const double* __restrict__ col = sl + i * lds;
            for (int j = i + 1 + qd4; j < ns; j += 4) {
              const double l = col[j];
#pragma unroll
              for (int h = 0; h < NR; h++) x[h] += l * sy[h * CB_PB_MAXNS + j];
            }
          }
          __syncwarp();
#pragma unroll
          for (int h = 0; h < NR; h++) {
            x[h] += __shfl_xor_sync(0xffffffffu, x[h], 1);
            x[h] += __shfl_xor_sync(0xffffffffu, x[h], 2);
            if (qd4 == 0 && i < ns) sw[h * CB_PB_MAXNS + i] = sy[h * CB_PB_MAXNS + i] + x[h];
          }
        }
        __syncthreads();
        if (tid < ns) {
#pragma unroll
          for (int h = 0; h < NR; h++) { const double v = sw[h * CB_PB_MAXNS + tid]; r.xp[h][f + tid] = v; r.out[h][pf] = v; }
        }
        SV_FETCH3();
        __syncthreads();
        if (tid == 0) { sv_set_release(q.done + s); if (trk) trk[2] = df_gtime(); }
      }
    }
#undef SV_SLAB_WAIT
    cur ^= 1;
  }
#undef SV_FETCH_NEXT
#undef SV_FETCH1
#undef SV_FETCH2
#undef SV_FETCH3
}
