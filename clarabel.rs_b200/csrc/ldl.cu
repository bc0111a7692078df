// Device multifrontal LDL^T for quasidefinite KKT matrices (sm_90a) + the
// cldl_* C-ABI (include/clarabel_b200.h).
//
// What it replaces in the reference (all file:line under /root/reference):
//   numeric refactor  src/qdldl/qdldl.rs:469-669   (_factor_inner, up-looking, 1 thread)
//   solve             src/qdldl/qdldl.rs:116-138, 708-768 (permute, L, D L^T, ipermute)
//   value updates     src/qdldl/qdldl.rs:142-183
//   adapter           src/solver/core/kktsolvers/direct/quasidef/ldlsolvers/qdldl.rs
//
// Design (see DESIGN.md): host symbolic analysis builds a supernodal assembly
// tree of dense fronts.  A front's panel ((ns+nr) x ns, column major) lives in
// the compact factor storage, its update matrix (nr x nr) in a lifetime-managed
// arena.  Tree level 0 (leaves, no dependencies) is factored by plain launches
// (k_factor_leaf1, k_factor_level), everything above it by one persistent
// dataflow kernel (k_factor_df).  Per front: assemble (original entries +
// children's update matrices through relative indices), dense LDL^T of the
// pivot block with the reference's sign-aware dynamic regularisation rule
// (qdldl.rs:645-651) applied pivot by pivot in elimination order, panel
// scaling, Schur update.  No atomics on floating point data: every sum has a
// fixed order, so refactor/solve are bit-reproducible run to run.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <thread>
#include <vector>

#include "../../include/clarabel_b200.h"
#include "ldl_device.h"
#include "symbolic.h"
#include "vec.cuh"

namespace cb {

std::atomic<unsigned long long> g_launches{0};

// ---- NCCL on the handle's own stream -------------------------------------------------------------------------
// The all-gathers between the phases are stream-ordered NCCL calls: pack kernel -> ncclAllGather -> unpack kernels on
// `stream`, no host synchronisation in between.  The library is NOT linked against NCCL: the process that drives the
// ranks (one per GPU, torch.distributed) already has a libnccl mapped, and two different NCCL builds in one process
// do not mix -- so the binding passes the path of the one that is loaded and the five entry points are taken from it
// with dlsym.  Only these five, with their long-stable signatures, are used (no nccl.h: its version may differ).
typedef struct ncclComm* cb_ncclComm_t;
typedef struct { char internal[128]; } cb_ncclUniqueId;
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(cb_ncclUniqueId*) = nullptr;
  int (*CommInitRank)(cb_ncclComm_t*, int, cb_ncclUniqueId, int) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, cb_ncclComm_t, cudaStream_t) = nullptr;
  int (*CommDestroy)(cb_ncclComm_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi* nccl_api(const char* libpath) {
  static NcclApi api;
  static bool tried = false;
  if (api.lib) return &api;
  if (tried && !libpath) return nullptr;
  tried = true;
  void* h = dlopen(libpath && *libpath ? libpath : "libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) { std::fprintf(stderr, "[clarabel_b200] dlopen(%s) failed: %s\n", libpath ? libpath : "libnccl.so.2", dlerror()); return nullptr; }
  api.GetUniqueId = (int (*)(cb_ncclUniqueId*))dlsym(h, "ncclGetUniqueId");
  api.CommInitRank = (int (*)(cb_ncclComm_t*, int, cb_ncclUniqueId, int))dlsym(h, "ncclCommInitRank");
  api.AllGather = (int (*)(const void*, void*, size_t, int, cb_ncclComm_t, cudaStream_t))dlsym(h, "ncclAllGather");
  api.CommDestroy = (int (*)(cb_ncclComm_t))dlsym(h, "ncclCommDestroy");
  api.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
  if (!api.GetUniqueId || !api.CommInitRank || !api.AllGather || !api.CommDestroy) return nullptr;
  api.lib = h;
  return &api;
}


// ------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------

// Inverse of the unit lower triangular pivot block L11 of a front with more than CB_SOLVE_SMALL_NS pivots, for the
// solves (ldl_solve.cuh), computed where the factorisation has the block.  A: the pivot block, column major with
// leading dimension lda, L11 in its strictly lower triangle.  Thread j builds column j of X = L11^-1 by forward
// substitution on e_j (X[j][j] = 1, X[i][j] = -sum_{k=j..i-1} L[i][k] X[k][j], two interleaved partial sums) and
// keeps it in the upper triangle, X[i][j] at A[i * lda + j], while the other threads still read L11.
template <int NT>
__device__ __forceinline__ void pivot_inverse(double* A, int lda, int ns) {
  for (int j = threadIdx.x; j < ns; j += NT) {
    for (int i = j + 1; i < ns; i++) {
      double a0 = A[(long long)j * lda + i], a1 = 0.0;     // k = j term: L[i][j] * X[j][j]
      int k = j + 1;
      for (; k + 1 < i; k += 2) {
        a0 += A[(long long)k * lda + i] * A[(long long)k * lda + j];
        a1 += A[(long long)(k + 1) * lda + i] * A[(long long)(k + 1) * lda + j];
      }
      if (k < i) a0 += A[(long long)k * lda + i] * A[(long long)k * lda + j];
      A[(long long)i * lda + j] = -(a0 + a1);
    }
  }
}
// after pivot_inverse and a barrier: X moves to the strictly lower triangle, the upper triangle is zero again
template <int NT>
__device__ __forceinline__ void pivot_inverse_place(double* A, int lda, int ns) {
  for (int idx = threadIdx.x; idx < ns * ns; idx += NT) {
    const int j = idx / ns, i = idx - j * ns;
    if (i > j) {
      A[(long long)j * lda + i] = A[(long long)i * lda + j];
      A[(long long)i * lda + j] = 0.0;
    }
  }
}

// Tree level 0: one CTA per front with at least two pivots.  Level-0 fronts have no children: the panel is the
// front's own entries, and U = 0 - L21 D L21^T is written once.
//   pivot block  right-looking, one barrier per pivot: every thread reads the pivot after the barrier and applies the
//                sign test / regularisation itself; the columns are scaled (l = a / d) after the last pivot, since
//                no later pivot reads them
//   Schur        1 x 4 register tiles: a lane owns one row of U and four columns, a warp 32 rows
//   inverse      L11^-1 of a wide front, from the panel before it is stored (pivot_inverse)
// Inertia, regularisation, zero-pivot and non-finite flags: one atomic per counter per CTA.  Every entry receives
// the same operations in the same order as in a column-by-column factorisation, so the bits do not depend on the
// schedule.
template <int NT>
__global__ void __launch_bounds__(NT) k_factor_level(LDLDev d, int task_base, int smem_cap) {
  extern __shared__ double sm[];
  __shared__ double sD[CB_MAX_PANEL];
  __shared__ double sInv[CB_MAX_PANEL];
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nwarp = NT >> 5;
  const int s = d.level_tasks[task_base + blockIdx.x];
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr;
  double* __restrict__ P = d.L + d.panel_off[s];
  double* __restrict__ U = d.U + d.upd_off[s];
  const long long psz = (long long)ld * ns;
  const bool use_sm = psz <= (long long)smem_cap;
  double* W = use_sm ? sm : P;

  for (long long i = tid; i < psz; i += NT) W[i] = 0.0;
  __syncthreads();
  // original matrix entries (each lands in a distinct slot)
  for (long long e = d.asm_ptr[s] + tid; e < d.asm_ptr[s + 1]; e += NT)
    W[d.asm_dst[e]] = d.vals[d.asm_src[e]];

  int c_reg = 0, c_pos = 0, c_zero = 0, c_nonf = 0;
  for (int j = 0; j < ns; j++) {
    __syncthreads();    // column j is final: assembled, and updated by every earlier pivot
    const double* __restrict__ cj = W + (long long)j * ld;
    double dj = cj[j];
    bool reg = false;
    if (d.reg_enable) {
      const double sg = (double)d.dsigns[f + j];
      if (dj * sg < d.reg_eps) { dj = d.reg_delta * sg; reg = true; }
    }
    const double inv = 1.0 / dj;
    if (tid == 0) {
      c_reg += reg ? 1 : 0;
      c_pos += dj > 0.0 ? 1 : 0;
      if (dj == 0.0) c_zero = 1;
      if (!isfinite(inv)) c_nonf = 1;
      d.D[f + j] = dj;
      d.Dinv[f + j] = inv;
      sD[j] = dj;
      sInv[j] = inv;
    }
    for (int k = j + 1 + warp; k < ns; k += nwarp) {
      const double wk = cj[k] * inv;
      double* __restrict__ ck = W + (long long)k * ld;
      for (int i = k + lane; i < ld; i += 32) ck[i] -= cj[i] * wk;
    }
  }
  __syncthreads();
  for (int j = warp; j < ns; j += nwarp) {
    double* __restrict__ cj = W + (long long)j * ld;
    const double inv = sInv[j];
    if (lane == 0) cj[j] = sD[j];
    for (int i = j + 1 + lane; i < ld; i += 32) cj[i] *= inv;
  }
  if (tid == 0) {
    if (c_reg) atomicAdd(&d.status[ST_REGCOUNT], c_reg);
    if (c_pos) atomicAdd(&d.status[ST_POSINERTIA], c_pos);
    if (c_zero) atomicExch(&d.status[ST_ZEROPIV], 1);
    if (c_nonf) atomicExch(&d.status[ST_NONFINITE], 1);
  }
  __syncthreads();

  // Schur update of the lower triangle of U; warp items (column block of 4, 32-row chunk from the block's diagonal)
  {
    int it = 0;
    for (int b0 = 0; b0 < nr; b0 += 4)
      for (int a0 = b0; a0 < nr; a0 += 32, it++) {
        if (it % nwarp != warp) continue;
        const int a = a0 + lane;
        const bool on = a < nr;
        const int nb = min(4, nr - b0);      // columns b0 .. b0 + nb - 1; the others repeat the last one
        double acc[4] = {0.0, 0.0, 0.0, 0.0};
        const double* __restrict__ ck = W + ns;
        for (int k = 0; k < ns; k++, ck += ld) {
          const double la = on ? ck[a] : 0.0, dk = sD[k];
#pragma unroll
          for (int c = 0; c < 4; c++) acc[c] += la * (ck[b0 + min(c, nb - 1)] * dk);
        }
#pragma unroll
        for (int c = 0; c < 4; c++)
          if (on && b0 + c < nr && a >= b0 + c) U[(long long)(b0 + c) * nr + a] = 0.0 - acc[c];
      }
  }
  // the Schur update reads rows ns.. only: the inverse of the pivot block needs no barrier before it
  if (ns > CB_SOLVE_SMALL_NS) {
    pivot_inverse<NT>(W, ld, ns);
    __syncthreads();
    pivot_inverse_place<NT>(W, ld, ns);
  }
  if (use_sm) {
    __syncthreads();
    for (long long i = tid; i < psz; i += NT) P[i] = W[i];
  }
}

// Single-column leaves (no children: tree level 0; on KKT matrices these are the constraint rows eliminated first,
// 5e5 of them on config C4): ONE WARP per front instead of one CTA.  The column is assembled in a per-warp shared
// buffer, then the lanes store the panel and U = 0 - l (l d)^T (lower triangle) with consecutive lanes on consecutive
// addresses.  Same arithmetic as the fused kernel above does for such a front: d = a_jj (sign test, regularisation),
// l = a_:j / d.  The inertia / regularisation counters are aggregated per CTA before they touch global memory.
#define LEAF1_NT 256
#define LEAF1_MAXLD 128    /* level-0 fronts that are not big have fewer than CB_BIG_NR rows */
static_assert(LEAF1_MAXLD > CB_BIG_NR, "a level-0 column must fit the per-warp buffer");
__global__ void __launch_bounds__(LEAF1_NT) k_factor_leaf1(LDLDev d, int task_base, int count) {
  __shared__ double s_col[LEAF1_NT / 32][LEAF1_MAXLD];
  __shared__ int s_pos, s_reg;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * (LEAF1_NT / 32) + warp;
  if (threadIdx.x == 0) { s_pos = 0; s_reg = 0; }
  __syncthreads();
  if (i < count) {
    double* col = s_col[warp];
    const int s = d.level_tasks[task_base + i];
    const int f = d.sn_first[s];
    const long long rp = d.sn_rowptr[s];
    const int nr = (int)(d.sn_rowptr[s + 1] - rp);
    const int ld = 1 + nr;
    double* __restrict__ P = d.L + d.panel_off[s];
    double* __restrict__ U = d.U + d.upd_off[s];
    for (int a = lane; a < ld; a += 32) col[a] = 0.0;
    __syncwarp();
    for (long long e = d.asm_ptr[s] + lane; e < d.asm_ptr[s + 1]; e += 32) col[d.asm_dst[e]] = d.vals[d.asm_src[e]];
    __syncwarp();
    double dj = col[0];
    bool reg = false;
    if (d.reg_enable) {
      const double sg = (double)d.dsigns[f];
      if (dj * sg < d.reg_eps) { dj = d.reg_delta * sg; reg = true; }
    }
    const double inv = 1.0 / dj;
    if (lane == 0) {
      if (dj == 0.0) atomicExch(&d.status[ST_ZEROPIV], 1);
      if (!isfinite(inv)) atomicExch(&d.status[ST_NONFINITE], 1);
      if (dj > 0.0) atomicAdd(&s_pos, 1);
      if (reg) atomicAdd(&s_reg, 1);
      d.D[f] = dj;
      d.Dinv[f] = inv;
    }
    __syncwarp();
    for (int a = lane; a < ld; a += 32) {
      const double v = a == 0 ? dj : col[a] * inv;
      col[a] = v;
      P[a] = v;
    }
    __syncwarp();
    for (int idx = lane; idx < nr * nr; idx += 32) {
      const int b = idx / nr, a = idx - b * nr;
      if (a >= b) {
        const double t = col[1 + b] * dj;
        double acc = 0.0;
        acc += col[1 + a] * t;
        U[idx] = 0.0 - acc;
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_pos) atomicAdd(&d.status[ST_POSINERTIA], s_pos);
    if (s_reg) atomicAdd(&d.status[ST_REGCOUNT], s_reg);
  }
}

__global__ void k_permute_in(int n, const int* __restrict__ perm, const double* __restrict__ b,
                             double* __restrict__ xp) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) xp[k] = b[perm[k]];
}

// ------------------------------------------------------------------------
// Dataflow triangular solves: ONE persistent kernel per sweep.  CTAs pull tasks from a queue in
// topological (level) order; a task waits on a counter (forward: number of unfinished child fronts;
// backward: parent's done flag) instead of on a kernel boundary, so independent branches of the tree
// overlap across levels and a level never waits for its slowest front.  A task is one wide front
// (whole CTA) or a batch of up to 8 narrow fronts (one warp each).  Data that crosses fronts is read
// with ld.global.cg (L2), written once before its consumers are released (threadfence + atomic).
// No floating-point atomics: every sum has a fixed order, so results are bit-identical run to run.
// ------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long df_gtime() {
#ifdef CB_EMU   /* host build of the test suite (tests/emu): no device clock */
  return 0;
#else
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
#endif
}
__device__ __forceinline__ void df_wait_zero(volatile int* p) {
  unsigned ns = 20;
  while (*p > 0) { __nanosleep(ns); if (ns < 640) ns <<= 1; }
}
__device__ __forceinline__ void df_wait_set(volatile int* p) {
  unsigned ns = 20;
  while (*p == 0) { __nanosleep(ns); if (ns < 640) ns <<= 1; }
}

#include "ldl_solve.cuh"

// ------------------------------------------------------------------------
// Dataflow numeric factorisation: ONE persistent kernel for everything above tree level 0.
// Task kinds (queue in level order, so every dependency sits earlier in the queue):
//   F  small front, fused (as k_factor_level)                 waits: all children complete
//   D  big front: assemble + factor the ns x ns pivot block    waits: all children complete
//   R  big front: 256 rows below the pivot block (assemble + triangular solve)   waits: D
//   T  big front: one 64x64 tile of the update matrix (extend-add + Schur update) waits: all R of the front
// A front is complete when its last tile (or its F task) finishes; that releases its parent.  Data
// produced by other CTAs inside this kernel is read with ld.global.cg (L1 is not coherent across SMs and
// the update-matrix arena is recycled along the schedule).  Every sum has a fixed order, whatever the
// schedule: results are bit-identical run to run.
// ------------------------------------------------------------------------
#define DF_NT 256
#define DF_SMEM_DOUBLES (CB_PB_MAXNS * CB_PB_LD + 2 * CB_PB_MAXNS + CB_PB_MAXNS * 128)   /* 12544 doubles = 98 KB (R task); T needs 12352 */

__device__ __forceinline__ double ldcg_d(const double* p) { return __ldcg(p); }

// (src,dst) list sorted by dst, applied to `base` with an index filter/transform:
//   keep(dst) -> new index or -1.  One destination is only touched by one thread, in list order.
template <class Map>
__device__ __forceinline__ void df_apply_sorted(double* base, const double* __restrict__ U,
                                                const int* __restrict__ esrc, const int* __restrict__ edst,
                                                int e0, int e1, Map map) {
  const int cnt = e1 - e0;
  if (cnt <= 0) return;
  const int per = (cnt + DF_NT - 1) / DF_NT;
  int b = e0 + threadIdx.x * per, e = min(e1, b + per);
  if (b >= e1) return;
  if (b > e0) { while (b < e1 && edst[b] == edst[b - 1]) b++; }
  if (e < e1) { while (e < e1 && edst[e] == edst[e - 1]) e++; }
  int i = b;
  while (i < e) {
    const int dd = edst[i];
    double acc = 0.0;
    while (i < e && edst[i] == dd) { acc += __ldcg(U + esrc[i]); i++; }
    const long long t = map(dd);
    if (t >= 0) base[t] += acc;
  }
}

__shared__ int df_cur_qi;
#define DF_STAMP(q, slot) do { if ((q).trace && threadIdx.x == 0) (q).trace[10 * (size_t)df_cur_qi + (slot)] = df_gtime(); } while (0)
__device__ __forceinline__ void df_front_complete(const DFFactor& q, int s) {
  const int p = q.parent[s];
  if (p >= 0) atomicSub(q.pend + p, 1);
}

// ---- F: small front, everything fused (mirrors k_factor_level<256>) ----
__device__ void dff_small(const LDLDev& d, int s, double* sm, int* s_flag) {
  __shared__ double s_inv;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = DF_NT >> 5;
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr;
  double* P = d.L + d.panel_off[s];
  double* U = d.U + d.upd_off[s];
  const long long psz = (long long)ld * ns;
  double* sD = sm;                       // [CB_MAX_PANEL]
  double* Wsm = sm + CB_MAX_PANEL;
  const bool use_sm = psz <= (long long)(DF_SMEM_DOUBLES - CB_MAX_PANEL);
  double* W = use_sm ? Wsm : P;
  (void)s_flag;
  for (long long i = tid; i < psz; i += DF_NT) W[i] = 0.0;
  for (int b = warp; b < nr; b += nwarp)
    for (int a = b + lane; a < nr; a += 32) U[(long long)b * nr + a] = 0.0;
  __syncthreads();
  for (long long e = d.asm_ptr[s] + tid; e < d.asm_ptr[s + 1]; e += DF_NT) W[d.asm_dst[e]] = d.vals[d.asm_src[e]];
  __syncthreads();
  for (long long ci = d.child_ptr[s]; ci < d.child_ptr[s + 1]; ci++) {
    const int c = d.child_list[ci];
    const long long crp = d.sn_rowptr[c];
    const int nrc = (int)(d.sn_rowptr[c + 1] - crp);
    const double* Uc = d.U + d.upd_off[c];
    const int* __restrict__ relc = d.rel + crp;
    for (int b = warp; b < nrc; b += nwarp) {
      const int rb = relc[b];
      for (int a = b + lane; a < nrc; a += 32) {
        const int ra = relc[a];
        const double v = __ldcg(Uc + (long long)b * nrc + a);
        if (rb < ns) W[(long long)rb * ld + ra] += v;
        else U[(long long)(rb - ns) * nr + (ra - ns)] += v;
      }
    }
    __syncthreads();
  }
  int c_reg = 0, c_pos = 0, c_zero = 0, c_nonf = 0;
  for (int j = 0; j < ns; j++) {
    if (tid == 0) {
      double dj = W[(long long)j * ld + j];
      if (d.reg_enable) {
        const double sg = (double)d.dsigns[f + j];
        if (dj * sg < d.reg_eps) { dj = d.reg_delta * sg; c_reg++; }
      }
      if (dj == 0.0) c_zero = 1;
      if (dj > 0.0) c_pos++;
      const double inv = 1.0 / dj;
      if (!isfinite(inv)) c_nonf = 1;
      d.D[f + j] = dj;
      d.Dinv[f + j] = inv;
      W[(long long)j * ld + j] = dj;
      s_inv = inv;
      sD[j] = dj;
    }
    __syncthreads();
    const double inv = s_inv;
    const double* cj = W + (long long)j * ld;
    for (int k = j + 1 + warp; k < ns; k += nwarp) {
      const double wk = cj[k] * inv;
      double* ck = W + (long long)k * ld;
      for (int i = k + lane; i < ld; i += 32) ck[i] -= cj[i] * wk;
    }
    __syncthreads();
    double* cjw = W + (long long)j * ld;
    for (int i = j + 1 + tid; i < ld; i += DF_NT) cjw[i] *= inv;
  }
  __syncthreads();
  if (tid == 0) {
    if (c_reg) atomicAdd(&d.status[ST_REGCOUNT], c_reg);
    if (c_pos) atomicAdd(&d.status[ST_POSINERTIA], c_pos);
    if (c_zero) atomicExch(&d.status[ST_ZEROPIV], 1);
    if (c_nonf) atomicExch(&d.status[ST_NONFINITE], 1);
  }
  for (int b = warp; b < nr; b += nwarp)
    for (int a = b + lane; a < nr; a += 32) {
      double acc = 0.0;
      for (int k = 0; k < ns; k++) {
        const double* ck = W + (long long)k * ld + ns;
        acc += ck[a] * (ck[b] * sD[k]);
      }
      U[(long long)b * nr + a] -= acc;
    }
  // the Schur update reads rows ns.. only: the inverse of the pivot block needs no barrier before it
  if (ns > CB_SOLVE_SMALL_NS) {
    pivot_inverse<DF_NT>(W, ld, ns);
    __syncthreads();
    pivot_inverse_place<DF_NT>(W, ld, ns);
    __syncthreads();
  }
  if (use_sm) for (long long i = tid; i < psz; i += DF_NT) P[i] = W[i];
}

// ---- D, R and T tasks read their records (DFTask, DFChildRec: ldl_plan.h) by field ----
#define DF_DCAP 32          /* child records staged per round */
#define DF_REC_INTS ((int)(sizeof(DFChildRec) / sizeof(int)))
// an int field of a child record in global memory, loaded on its own: read through a DFChildRec lvalue, the record's
// 8-byte alignment lets the compiler pair neighbouring fields into 64-bit loads, which reschedules the tile task
#define DF_REC_INT(r, field) (reinterpret_cast<const int*>(r)[offsetof(DFChildRec, field) / sizeof(int)])

// One child's block added into a shared-memory target.  The 8 warps own the target COLUMNS (column & 7), so no
// two warps ever touch the same element and a warp meets the children in list order: sums keep a fixed order
// without barriers between children.  Inside a warp lane = (owned column, row phase): at most 8 of the <= 64
// target columns of a block belong to one warp.
template <int NH>
__device__ __forceinline__ void df_add_child(const LDLDev& d, const DFChildRec& ch, double* dst, int rowoff,
                                             int rstride, int coloff, int cstride) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int* __restrict__ relc = d.rel + ch.relp;
  const double* Uc = d.U + ch.uoff;
  __syncwarp();
  if (ch.contig == 3) {
    // rows and columns of the block are contiguous in the target (the previous panel of the same separator,
    // dense children): no index loads, warp-wide coalesced reads down the columns this warp owns
    const int r0 = ch.ra0 - rowoff - ch.a0, c0 = ch.rb0 - coloff - ch.b0;   // target row of a: r0 + a, column of b: c0 + b
    const int bfirst = ch.b0 + ((warp - (c0 + ch.b0)) & 7);
    const int a1 = ch.a1, b1 = ch.b1;
    for (int ab = ch.a0; ab < a1; ab += 32 * NH) {
      double v[8][NH];
#pragma unroll
      for (int c = 0; c < 8; c++) {
        const int b = bfirst + 8 * c;
#pragma unroll
        for (int h = 0; h < NH; h++) {
          const int a = ab + lane + 32 * h;
          v[c][h] = (b < b1 && a < a1 && a >= b) ? __ldcg(Uc + (long long)b * ch.nrc + a) : 0.0;
        }
      }
#pragma unroll
      for (int c = 0; c < 8; c++) {
        const int b = bfirst + 8 * c;
#pragma unroll
        for (int h = 0; h < NH; h++) {
          const int a = ab + lane + 32 * h;
          if (b < b1 && a < a1 && a >= b) dst[(r0 + a) * rstride + (c0 + b) * cstride] += v[c][h];
        }
      }
    }
    __syncwarp();
    return;
  }
  const int bl = ch.b0 + lane, bh = bl + 32;
  const int dc0 = bl < ch.b1 ? relc[bl] - coloff : -1;
  const int dc1 = bh < ch.b1 ? relc[bh] - coloff : -1;
  unsigned m0 = __ballot_sync(0xffffffffu, dc0 >= 0 && (dc0 & 7) == warp);
  unsigned m1 = __ballot_sync(0xffffffffu, dc1 >= 0 && (dc1 & 7) == warp);
  const int cnt0 = __popc(m0), cnt = cnt0 + __popc(m1);
  const int oc = lane >> 2, ar = lane & 3;
  int pos = -1;
  if (oc < cnt) {
    unsigned m = oc < cnt0 ? m0 : m1;
    const int skip = oc < cnt0 ? oc : oc - cnt0;
    for (int k = 0; k < skip; k++) m &= m - 1;
    pos = __ffs(m) - 1 + (oc < cnt0 ? 0 : 32);
  }
  const int srcl = pos < 0 ? 0 : (pos & 31);
  const int x0 = __shfl_sync(0xffffffffu, dc0, srcl), x1 = __shfl_sync(0xffffffffu, dc1, srcl);
  if (pos >= 0) {
    const int dcc = (pos < 32 ? x0 : x1) * cstride;
    const int b = ch.b0 + pos;
    const double* ucol = Uc + (long long)b * ch.nrc;
    const int a1 = ch.a1;
    for (int a = max(ch.a0, b) + ar; a < a1; a += 32) {
      double v[8];
      int r[8];
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const int aa = a + 4 * u;
        const bool ok = aa < a1;
        v[u] = ok ? __ldcg(ucol + aa) : 0.0;
        r[u] = ok ? relc[aa] : rowoff;
      }
#pragma unroll
      for (int u = 0; u < 8; u++)
        if (a + 4 * u < a1) dst[(r[u] - rowoff) * rstride + dcc] += v[u];
    }
  }
  __syncwarp();
}

// Sorted (src,dst) entries with the loads hoisted: df_ent_issue starts the loads at the top of a task (they
// overlap the panel / child-record loads), df_ent_apply adds them after the children, in list order, one
// destination per thread (same sums as df_apply_sorted).  Lists longer than 2*DF_NT take the plain path.
#define DF_ENT_FAST (2 * DF_NT)
struct DFEnt { int dd[2]; double v[2]; };
__device__ __forceinline__ void df_ent_issue(const double* __restrict__ U, const int* __restrict__ esrc,
                                             const int* __restrict__ edst, int e0, int e1, DFEnt& pe) {
  const int cnt = e1 - e0;
  pe.dd[0] = pe.dd[1] = -1;
  pe.v[0] = pe.v[1] = 0.0;
  if (cnt > DF_ENT_FAST) return;
  int src[2] = {0, 0};
#pragma unroll
  for (int u = 0; u < 2; u++) {
    const int i = threadIdx.x + u * DF_NT;
    if (i < cnt) { pe.dd[u] = edst[e0 + i]; src[u] = esrc[e0 + i]; }
  }
#pragma unroll
  for (int u = 0; u < 2; u++)
    if (threadIdx.x + u * DF_NT < cnt) pe.v[u] = __ldcg(U + src[u]);
}
template <class Map>
__device__ __forceinline__ void df_ent_apply(double* base, const double* __restrict__ U, const int* __restrict__ esrc,
                                             const int* __restrict__ edst, int e0, int e1, const DFEnt& pe,
                                             int* s_ed, double* s_ev, Map map) {
  const int cnt = e1 - e0;
  if (cnt <= 0) return;
  if (cnt > DF_ENT_FAST) { df_apply_sorted(base, U, esrc, edst, e0, e1, map); return; }
#pragma unroll
  for (int u = 0; u < 2; u++) {
    const int i = threadIdx.x + u * DF_NT;
    if (i < cnt) { s_ed[i] = pe.dd[u]; s_ev[i] = pe.v[u]; }
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < 2; u++) {
    int i = threadIdx.x + u * DF_NT;
    if (i < cnt) {
      const int dd = pe.dd[u];
      if (i == 0 || s_ed[i - 1] != dd) {
        double acc = 0.0;
        while (i < cnt && s_ed[i] == dd) { acc += s_ev[i]; i++; }
        const long long t = map(dd);
        if (t >= 0) base[t] += acc;
      }
    }
  }
}

// The front's own KKT entries (assembly map), 4 per thread in flight
template <class Put>
__device__ __forceinline__ void df_scatter_asm(const LDLDev& d, int s, Put put) {
  const long long e0 = d.asm_ptr[s], e1 = d.asm_ptr[s + 1];
  for (long long e = e0 + threadIdx.x; e < e1; e += 4 * DF_NT) {
    long long dst[4];
    int src[4];
    double v[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const long long ee = e + (long long)u * DF_NT;
      const bool ok = ee < e1;
      dst[u] = ok ? (long long)d.asm_dst[ee] : -1;
      src[u] = ok ? d.asm_src[ee] : 0;
    }
#pragma unroll
    for (int u = 0; u < 4; u++) v[u] = dst[u] >= 0 ? d.vals[src[u]] : 0.0;
#pragma unroll
    for (int u = 0; u < 4; u++) if (dst[u] >= 0) put(dst[u], v[u]);
  }
}

template <class F>
__device__ __forceinline__ void df_children(const DFFactor& q, int d0, int d1, int* s_desc, F f) {
  for (int base = d0; base < d1; base += DF_DCAP) {
    const int cnt = min(DF_DCAP, d1 - base);
    const int* src = reinterpret_cast<const int*>(q.recs);
    for (int i = threadIdx.x; i < cnt * DF_REC_INTS; i += DF_NT) s_desc[i] = src[(size_t)base * DF_REC_INTS + i];
    __syncthreads();
    const DFChildRec* rec = reinterpret_cast<const DFChildRec*>(s_desc);
    for (int k = 0; k < cnt; k++) f(rec[k]);
    __syncthreads();
  }
}

// ---- D: pivot block of a big front ----
// Assembly in shared memory, then a right-looking LDL^T with the block held in REGISTERS: thread (bi, bj)
// owns the 4x4 block (rows 4bi.., columns 4bj..) of the lower triangle; per pivot the owners of the pivot
// column publish it through a double-buffered shared column (one barrier per pivot), the owner of the diagonal
// element applies the sign test / regularisation and the reciprocal.
__device__ void dff_diag(const LDLDev& d, const DFFactor& q, const DFTask& tk, double* sm, int* s_desc, int* s_ed, double* s_ev) {
  double* sA = sm;                                     // [64][CB_PB_LD]
  double* sSign = sm + CB_PB_MAXNS * CB_PB_LD;         // [64]
  double* colbuf = sSign + CB_PB_MAXNS;                // [2][72]: column, then dj, 1/dj
  const int tid = threadIdx.x;
  const int s = tk.s, ns = tk.ns, nr = tk.nr, f = tk.f;
  const int ld = ns + nr;
  const long long poff = tk.poff;
  double* P = d.L + poff;
  DFEnt pe;
  df_ent_issue(d.U, d.sc_panel_src, d.sc_panel_dst, tk.e0, tk.e1, pe);
  for (int i = tid; i < CB_PB_MAXNS * CB_PB_LD; i += DF_NT) sA[i] = 0.0;
  if (tid < CB_PB_MAXNS) sSign[tid] = tid < ns ? (double)d.dsigns[f + tid] : 1.0;
  __syncthreads();
  df_scatter_asm(d, s, [&](long long dst, double v) {
    const int col = (int)(dst / ld), row = (int)(dst - (long long)col * ld);
    if (row < ns) sA[col * CB_PB_LD + row] = v;
  });
  __syncthreads();
  df_children(q, tk.d0, tk.d1, s_desc, [&](const DFChildRec& ch) { df_add_child<2>(d, ch, sA, 0, 1, 0, CB_PB_LD); });
  df_ent_apply(sA, d.U, d.sc_panel_src, d.sc_panel_dst, tk.e0, tk.e1, pe, s_ed, s_ev,
               [&](int dd) -> long long { const int col = dd / ld, row = dd - col * ld; return row < ns ? (long long)col * CB_PB_LD + row : -1; });
  __syncthreads();
  DF_STAMP(q, 4);
  const int bi = tid & 15, bj = tid >> 4;
  const bool active = bi >= bj;
  double a[4][4];
#pragma unroll
  for (int k = 0; k < 4; k++)
#pragma unroll
    for (int i = 0; i < 4; i++) a[i][k] = active ? sA[(4 * bj + k) * CB_PB_LD + 4 * bi + i] : 0.0;
  int c_reg = 0, c_pos = 0, c_zero = 0, c_nonf = 0;
  const int nJ = (ns + 3) >> 2;
  for (int J = 0; J < nJ; J++) {
#pragma unroll
    for (int jj = 0; jj < 4; jj++) {
      const int j = 4 * J + jj;
      if (j >= ns) break;
      double* buf = colbuf + (j & 1) * 72;
      if (bj == J && active) {
        if (bi == J) {
          double dj = a[jj][jj];
          if (d.reg_enable) {
            const double sg = sSign[j];
            if (dj * sg < d.reg_eps) { dj = d.reg_delta * sg; c_reg++; }
          }
          if (dj == 0.0) c_zero = 1;
          if (dj > 0.0) c_pos++;
          const double inv = __drcp_rn(dj);
          if (!isfinite(inv)) c_nonf = 1;
          a[jj][jj] = dj;
          buf[64] = dj;
          buf[65] = inv;
          d.D[f + j] = dj;
          d.Dinv[f + j] = inv;
        }
#pragma unroll
        for (int i = 0; i < 4; i++) buf[4 * bi + i] = a[i][jj];
      }
      __syncthreads();
      if (active && bj >= J) {
        const double inv = buf[65];
        double li[4];
#pragma unroll
        for (int i = 0; i < 4; i++) li[i] = buf[4 * bi + i];
        if (bj > J) {
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const double wk = buf[4 * bj + k] * inv;
#pragma unroll
            for (int i = 0; i < 4; i++) a[i][k] -= li[i] * wk;
          }
        } else {
#pragma unroll
          for (int k = jj + 1; k < 4; k++) {
            const double wk = buf[4 * bj + k] * inv;
#pragma unroll
            for (int i = 0; i < 4; i++) a[i][k] -= li[i] * wk;
          }
#pragma unroll
          for (int i = 0; i < 4; i++)
            if (4 * bi + i > j) a[i][jj] *= inv;
        }
      }
    }
  }
  if (c_reg) atomicAdd(&d.status[ST_REGCOUNT], c_reg);
  if (c_pos) atomicAdd(&d.status[ST_POSINERTIA], c_pos);
  if (c_zero) atomicExch(&d.status[ST_ZEROPIV], 1);
  if (c_nonf) atomicExch(&d.status[ST_NONFINITE], 1);
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int col = 4 * bj + k;
    if (col < ns) {
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int row = 4 * bi + i;
        if (row < ns) P[(long long)col * ld + row] = row >= col ? a[i][k] : 0.0;
      }
    }
  }
}

// ---- R: DF_RB rows below the pivot block: assemble in shared memory, wait for D, triangular solve ----
__device__ void dff_rows(const LDLDev& d, const DFFactor& q, const DFTask& tk, double* sm, int* s_desc, int* s_ed, double* s_ev) {
  double* sA = sm;                                     // [64][CB_PB_LD]  L11 (unit lower, column major)
  double* sDval = sm + CB_PB_MAXNS * CB_PB_LD;
  double* sDinv = sDval + CB_PB_MAXNS;
  double* sR = sDinv + CB_PB_MAXNS;                    // [64][DF_RB]  the rows, column major
  const int tid = threadIdx.x;
  const int s = tk.s, blk = tk.a, ns = tk.ns, nr = tk.nr, f = tk.f;
  const int ld = ns + nr;
  double* P = d.L + tk.poff;
  const int r0 = blk * DF_RB, r1 = min(nr, r0 + DF_RB);
  const int g0 = ns + r0, g1 = ns + r1;
  DFEnt pe;
  df_ent_issue(d.U, d.sc_panel_src, d.sc_panel_dst, tk.e0, tk.e1, pe);
  for (int i = tid; i < CB_PB_MAXNS * DF_RB; i += DF_NT) sR[i] = 0.0;
  __syncthreads();
  df_scatter_asm(d, s, [&](long long dst, double v) {
    const int col = (int)(dst / ld), row = (int)(dst - (long long)col * ld);
    if (row >= g0 && row < g1) sR[col * DF_RB + row - g0] = v;
  });
  __syncthreads();
  df_children(q, tk.d0, tk.d1, s_desc, [&](const DFChildRec& ch) { df_add_child<4>(d, ch, sR, g0, 1, 0, DF_RB); });
  df_ent_apply(sR, d.U, d.sc_panel_src, d.sc_panel_dst, tk.e0, tk.e1, pe, s_ed, s_ev,
               [&](int dd) -> long long { const int col = dd / ld, row = dd - col * ld; return (row >= g0 && row < g1) ? (long long)col * DF_RB + row - g0 : -1; });
  __syncthreads();
  DF_STAMP(q, 4);
  if (tid == 0) { df_wait_set(q.diag_done + s); __threadfence(); }
  __syncthreads();
  DF_STAMP(q, 5);
  for (int idx = tid; idx < ns * ns; idx += DF_NT) {
    const int j = idx / ns, i = idx - j * ns;
    sA[j * CB_PB_LD + i] = __ldcg(P + (long long)j * ld + i);
  }
  if (tid < ns) { sDval[tid] = __ldcg(d.D + f + tid); sDinv[tid] = __ldcg(d.Dinv + f + tid); }
  __syncthreads();
  constexpr int JB = 16;
  const int r = tid;
  if (r < r1 - r0) {
    double* prow = sR + r;
    for (int jb = 0; jb < ns; jb += JB) {
      const int nj = min(JB, ns - jb);
      double t[JB];
#pragma unroll
      for (int jj = 0; jj < JB; jj++) t[jj] = jj < nj ? prow[(jb + jj) * DF_RB] : 0.0;
      for (int kb = 0; kb < jb; kb += JB) {
#pragma unroll
        for (int kk = 0; kk < JB; kk++) {
          const double wk = prow[(kb + kk) * DF_RB] * sDval[kb + kk];
          const double2* lk2 = reinterpret_cast<const double2*>(sA + (kb + kk) * CB_PB_LD + jb);
#pragma unroll
          for (int j2 = 0; j2 < JB / 2; j2++) { const double2 l = lk2[j2]; t[2 * j2] -= wk * l.x; t[2 * j2 + 1] -= wk * l.y; }
        }
      }
#pragma unroll
      for (int jj = 0; jj < JB; jj++) {
        if (jj < nj) {
          const double* lk = sA + (jb + jj) * CB_PB_LD + jb;
#pragma unroll
          for (int j2 = jj + 1; j2 < JB; j2++) t[j2] -= t[jj] * lk[j2];
        }
      }
#pragma unroll
      for (int jj = 0; jj < JB; jj++) if (jj < nj) prow[(jb + jj) * DF_RB] = t[jj] * sDinv[jb + jj];
    }
  }
  __syncthreads();
  const int nrow = r1 - r0;
  for (int idx = tid; idx < ns * DF_RB; idx += DF_NT) {
    const int j = idx / DF_RB, rr = idx - j * DF_RB;
    if (rr < nrow) P[(long long)j * ld + g0 + rr] = sR[idx];
  }
}

// ---- the R task that finishes a wide big front: L11^-1 for the solves ----
// L11 has to stay in the panel until every R task of the front has read it; the last one to finish still holds it
// in shared memory (sA of dff_rows) and replaces it in the panel by its inverse.  T tasks and the parent never read
// L11, so this is off the critical path.
__device__ void dff_rows_invert(const LDLDev& d, const DFTask& tk, double* sm) {
  double* sA = sm;                                     // [64][CB_PB_LD]  L11, as dff_rows left it
  const int ns = tk.ns, ld = ns + tk.nr;
  double* P = d.L + tk.poff;
  pivot_inverse<DF_NT>(sA, CB_PB_LD, ns);
  __syncthreads();
  for (int idx = threadIdx.x; idx < ns * ns; idx += DF_NT) {
    const int j = idx / ns, i = idx - j * ns;
    if (i > j) P[(long long)j * ld + i] = sA[i * CB_PB_LD + j];
  }
}

// ---- T: one 64x64 tile of the update matrix ----
__device__ void dff_tile(const LDLDev& d, const DFFactor& q, const DFTask& tk, double* sm, int* s_desc, int* s_ed, double* s_ev) {
  double* sAt = sm;                      // [ns][TS]  L21 rows of tile-row I
  double* sBt = sm + TS * TS;            // [ns][TS]  L21 rows of tile-row J, scaled by D
  double* sC = sm + 2 * TS * TS;         // [TS][TS+1] children's contributions
  double* sD = sC + TS * (TS + 1);       // [ns]
  const int tid = threadIdx.x;
  const int ti = tk.a, tj = tk.b, ns = tk.ns, nr = tk.nr, f = tk.f;
  const int ld = ns + nr;
  const double* P = d.L + tk.poff;
  double* U = d.U + tk.uoff;
  const int i0 = ti * TS, j0 = tj * TS;
  const int ni = min(TS, nr - i0), nj = min(TS, nr - j0);
  // every independent load of the task is issued up front (sorted entries, child records, the whole K range
  // of both panels) so that the task pays ~3 dependent memory round trips instead of one per stage
  DFEnt pe;
  df_ent_issue(d.U, d.sc_tile_src, d.sc_tile_dst, tk.e0, tk.e1, pe);
  {
    // finished panels are immutable for the rest of the launch and start on sector boundaries, so they may
    // travel through L1: 8-byte cp.async straight into shared memory, no registers, no issue stall
    const int rr = tid & (TS - 1), kq = tid >> 6;
    const unsigned sa = (unsigned)__cvta_generic_to_shared(sAt), sb = (unsigned)__cvta_generic_to_shared(sBt);
    const unsigned za = rr < ni ? 8u : 0u, zb = rr < nj ? 8u : 0u;
    const double* pa = P + ns + i0 + (rr < ni ? rr : 0);
    const double* pb = P + ns + j0 + (rr < nj ? rr : 0);
#pragma unroll 4
    for (int k = kq; k < ns; k += 4) {
      const long long col = (long long)k * ld;
#ifdef CB_EMU   /* host build of the test suite: the copy with zero fill, done synchronously */
      (void)sa; (void)sb;
      sAt[k * TS + rr] = za ? pa[col] : 0.0;
      sBt[k * TS + rr] = zb ? pb[col] : 0.0;
    }
#else
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(sa + (unsigned)(k * TS + rr) * 8u), "l"(pa + col), "r"(za) : "memory");
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(sb + (unsigned)(k * TS + rr) * 8u), "l"(pb + col), "r"(zb) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
#endif
    if (tid < ns) sD[tid] = __ldcg(d.D + f + tid);
  }
  DF_STAMP(q, 6);
  // children that are contiguous in this tile (the previous panel of the same separator) are added in
  // registers, straight from their update matrix.  A thread owns 4 x 4 entries of the tile, (OWN_R(i), OWN_C(j)):
  // on the device the ones the tensor-core fragments of the product below leave in its registers (warp w: rows
  // 32 (w & 1) .., columns 16 (w >> 1) ..; lane: row lane / 4 of every 8 x 8 fragment, columns 2 (lane % 4), +1), in the
  // host build of the test suite rows tx + 16 i, columns ty + 16 j
#ifdef CB_EMU
  const int tx = tid & 15, ty = tid >> 4;
#define OWN_R(i) (tx + 16 * (i))
#define OWN_C(j) (ty + 16 * (j))
#else
  const int lk = tid & 3, lr = (tid & 31) >> 2, r0w = ((tid >> 5) & 1) * 32, c0w = (tid >> 6) * 16;
#define OWN_R(i) (r0w + 8 * (i) + lr)
#define OWN_C(j) (c0w + 8 * ((j) >> 1) + 2 * lk + ((j) & 1))
#endif
  double creg[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) creg[i][j] = 0.0;
  const int ndense = tk.ndense;
  for (int kd = 0; kd < ndense; kd++) {
    const DFChildRec* rec = q.recs + (size_t)(tk.d0 + kd);
    const long long uoff = rec->uoff;
    const int nrc = DF_REC_INT(rec, nrc), a0 = DF_REC_INT(rec, a0), a1 = DF_REC_INT(rec, a1), b0 = DF_REC_INT(rec, b0), b1 = DF_REC_INT(rec, b1);
    const int ra = a0 - (DF_REC_INT(rec, ra0) - (ns + i0)), rb = b0 - (DF_REC_INT(rec, rb0) - (ns + j0));   // child index = tile index + ra / rb
    const double* Uc = d.U + uoff;
    double v[4][4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int b = OWN_C(j) + rb;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int a = OWN_R(i) + ra;
        v[i][j] = (a >= a0 && a < a1 && b >= b0 && b < b1 && a >= b) ? __ldcg(Uc + (long long)b * nrc + a) : 0.0;
      }
    }
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 4; j++) creg[i][j] += v[i][j];
  }
  const bool use_sc = (tk.d1 - tk.d0 > ndense) || (tk.e1 > tk.e0);
  if (use_sc) {
    for (int idx = tid; idx < TS * (TS + 1); idx += DF_NT) sC[idx] = 0.0;
    __syncthreads();
    DF_STAMP(q, 7);
    df_children(q, tk.d0 + ndense, tk.d1, s_desc, [&](const DFChildRec& ch) { df_add_child<2>(d, ch, sC, ns + i0, TS + 1, ns + j0, 1); });
    DF_STAMP(q, 8);
    df_ent_apply(sC, d.U, d.sc_tile_src, d.sc_tile_dst, tk.e0, tk.e1, pe, s_ed, s_ev, [&](int dd) -> long long { return dd; });
  }
#ifndef CB_EMU
  asm volatile("cp.async.wait_group 0;" ::: "memory");
#endif
  __syncthreads();
  for (int idx = tid; idx < ns * TS; idx += DF_NT) sBt[idx] *= sD[idx >> 6];
#ifndef CB_EMU
  {   // the tensor-core product below walks K in steps of 4: rows ns .. of both operands count as zero
    const int ns4 = (ns + 3) & ~3;
    for (int idx = ns * TS + tid; idx < ns4 * TS; idx += DF_NT) { sAt[idx] = 0.0; sBt[idx] = 0.0; }
  }
#endif
  __syncthreads();
  DF_STAMP(q, 4);
#ifdef CB_EMU   /* host build of the test suite: the same product with scalar FMAs */
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.0;
#pragma unroll 4
  for (int k = 0; k < ns; k++) {
    double a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; i++) { a[i] = sAt[k * TS + tx + 16 * i]; b[i] = sBt[k * TS + ty + 16 * i]; }
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 4; j++) acc[i][j] += a[i] * b[j];
  }
#else
  // The 64 x 64 x ns product L21_I (D L21_J)^T on the FP64 tensor path: mma.sync.aligned.m8n8k4 (SASS DMMA) -- FP64
  // MMA on sm_90a is mma.sync only (wgmma has no FP64 kind).  On C5 these tiles ARE the dense Schur blocks of the PSD
  // cones' Hs blocks (the north star's "tensor cores only for the dense Schur blocks arising from SDP cones").
  // scripts/ubench/dmma_tile.cu compares it with the 4 x 4 FMA register tile on this tile shape.
  // Warp w owns rows 32 (w & 1) .., columns 16 (w >> 1) .. as 4 x 2 fragments of 8 x 8; the extend-add above and the store
  // below use the same ownership, so the product never leaves the registers.
  double c2[4][2][2];
  {
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 2; j++) { c2[i][j][0] = 0.0; c2[i][j][1] = 0.0; }
    const int ns4 = (ns + 3) & ~3;
#pragma unroll 2
    for (int k = 0; k < ns4; k += 4) {
      double a[4], b[2];
#pragma unroll
      for (int i = 0; i < 4; i++) a[i] = sAt[(k + lk) * TS + r0w + 8 * i + lr];
#pragma unroll
      for (int j = 0; j < 2; j++) b[j] = sBt[(k + lk) * TS + c0w + 8 * j + lr];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 2; j++)
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                       : "+d"(c2[i][j][0]), "+d"(c2[i][j][1]) : "d"(a[i]), "d"(b[j]));
    }
  }
#endif
  DF_STAMP(q, 5);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int rr = OWN_R(i);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int cc = OWN_C(j);
#ifdef CB_EMU
      const double prod = acc[i][j];
#else
      const double prod = c2[i][j >> 1][j & 1];
#endif
      if (rr < ni && cc < nj && (i0 + rr >= j0 + cc))
        U[(long long)(j0 + cc) * nr + (i0 + rr)] = (use_sc ? creg[i][j] + sC[rr * (TS + 1) + cc] : creg[i][j]) - prod;
    }
  }
#undef OWN_R
#undef OWN_C
}

__global__ void __launch_bounds__(DF_NT, 2) k_factor_df(LDLDev d, DFFactor q) {
  extern __shared__ __align__(16) double dfsm[];
  __shared__ __align__(16) int s_desc[DF_DCAP * DF_REC_INTS];
  __shared__ __align__(16) int s_task[16];
  __shared__ int s_ed[DF_ENT_FAST];
  __shared__ double s_ev[DF_ENT_FAST];
  __shared__ int s_last;
  const int tid = threadIdx.x;
  if (tid == 0) df_cur_qi = -1;
  for (;;) {
    __syncthreads();
    if (tid == 0) {
      if (q.trace && df_cur_qi >= 0) q.trace[10 * (size_t)df_cur_qi + 2] = df_gtime();
      const int qi = atomicAdd(q.qhead, 1);
      df_cur_qi = qi < q.ntask ? qi : -1;
      if (q.trace && df_cur_qi >= 0) {
        unsigned smid = 0;
#ifndef CB_EMU
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
#endif
        q.trace[10 * (size_t)qi] = df_gtime();
        q.trace[10 * (size_t)qi + 3] = smid;
      }
    }
    __syncthreads();
    const int qi = df_cur_qi;
    if (qi < 0) break;
    if (tid < 4) reinterpret_cast<int4*>(s_task)[tid] = q.tasks[4 * (size_t)qi + tid];
    __syncthreads();
    const DFTask& tk = *reinterpret_cast<const DFTask*>(s_task);
    const int kind = tk.kind, s = tk.s;
    if (kind == 0) {
      if (tid == 0) { df_wait_zero(q.pend + s); __threadfence(); if (q.trace) q.trace[10 * (size_t)qi + 1] = df_gtime(); }
      __syncthreads();
      dff_small(d, s, dfsm, nullptr);
      __syncthreads();
      if (tid == 0) { __threadfence(); df_front_complete(q, s); }
    } else if (kind == 1) {
      if (tid == 0) { df_wait_zero(q.pend + s); __threadfence(); if (q.trace) q.trace[10 * (size_t)qi + 1] = df_gtime(); }
      __syncthreads();
      dff_diag(d, q, tk, dfsm, s_desc, s_ed, s_ev);
      __syncthreads();
      if (tid == 0) { __threadfence(); atomicExch(q.diag_done + s, 1); }
    } else if (kind == 2) {
      // the row task needs the children's data as well as the pivot block: it waits on the children counter
      // first, assembles, and only then waits for the D task of the front
      if (tid == 0) { df_wait_zero(q.pend + s); __threadfence(); if (q.trace) q.trace[10 * (size_t)qi + 1] = df_gtime(); }
      __syncthreads();
      dff_rows(d, q, tk, dfsm, s_desc, s_ed, s_ev);
      __syncthreads();
      if (tid == 0) { __threadfence(); s_last = atomicSub(q.rows_left + s, 1) == 1; }
      __syncthreads();
      if (s_last && tk.ns > CB_SOLVE_SMALL_NS) dff_rows_invert(d, tk, dfsm);
    } else {
      if (tid == 0) { df_wait_zero(q.rows_left + s); __threadfence(); if (q.trace) q.trace[10 * (size_t)qi + 1] = df_gtime(); }
      __syncthreads();
      dff_tile(d, q, tk, dfsm, s_desc, s_ed, s_ev);
      __syncthreads();
      if (tid == 0) {
        __threadfence();
        if (atomicSub(q.tiles_left + s, 1) == 1) df_front_complete(q, s);
      }
    }
  }
}

#include "ldl_selinv.cuh"
#include "ldl_schur.cuh"

__global__ void k_update_values(double* __restrict__ vals, const int* __restrict__ idx,
                                const double* __restrict__ v, long long len) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < len) vals[idx[i]] = v[i];
}
__global__ void k_scale_values(double* __restrict__ vals, const int* __restrict__ idx, double s,
                               long long len) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < len) vals[idx[i]] *= s;
}
__global__ void k_offset_values(double* __restrict__ vals, const int* __restrict__ idx, double off,
                                const signed char* __restrict__ sg, long long len) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < len) {
    const int s = sg[i];
    if (s > 0) vals[idx[i]] += off;
    else if (s < 0) vals[idx[i]] -= off;
  }
}

// ------------------------------------------------------------------------
// host object
// ------------------------------------------------------------------------

#define CK(x)                                                                        \
  do {                                                                               \
    cudaError_t e_ = (x);                                                            \
    if (e_ != cudaSuccess) {                                                         \
      std::fprintf(stderr, "[clarabel_b200] CUDA error %s at %s:%d\n",              \
                   cudaGetErrorString(e_), __FILE__, __LINE__);                      \
      return CLDL_E_CUDA;                                                            \
    }                                                                                \
  } while (0)

int LDLObject::init(int n_, const int64_t* Ap, const int32_t* Ai, const double* Ax,
                    const int8_t* dsigns, const cldl_opts& o, const int* perm_in) {
  n = n_;
  opts = o;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    std::fprintf(stderr, "[clarabel_b200] no CUDA device: this backend has no CPU fallback\n");
    return CLDL_E_CUDA;
  }
  device = o.device;
  CK(cudaSetDevice(device));
  SymbolicOptions so;
  so.ordering = o.ordering ? o.ordering : ORDER_BEST;
  so.amd_dense_scale = o.amd_dense_scale > 0 ? o.amd_dense_scale : 1.5;
  if (o.max_panel > 0) so.max_panel = o.max_panel > CB_PB_MAXNS ? CB_PB_MAXNS : o.max_panel;
  if (o.nd_leaf > 0) so.nd_leaf = o.nd_leaf;
  cb_tmark(nullptr);
  schur = !schur_set.empty();
  int rc = schur ? analyse_schur(n, Ap, Ai, perm_in, schur_set, so, S) : analyse(n, Ap, Ai, perm_in, so, S);
  cb_tmark("ldl: ordering + symbolic");
  if (rc == -2) return CLDL_E_EMPTY_COLUMN;
  if (rc == -3) return CLDL_E_NOT_TRIU;
  if (rc == -5) return CLDL_E_BAD_PERM;
  if (rc) return CLDL_E_ARG;
  shard_nranks = o.shard_nranks > 1 ? o.shard_nranks : 1;
  shard_rank = o.shard_rank;
  if (schur && sharded()) return CLDL_E_ARG;
  if (schur) shard_rank = 0;
  if (sharded()) {
    if (shard_rank < 0 || shard_rank >= shard_nranks) return CLDL_E_ARG;
    std::vector<int> par(S.sn_parent);
    if (plan_shards(S.nsup, S.sn_first.data(), S.sn_rowptr.data(), par.data(), shard_nranks, shard)) return CLDL_E_ARG;
    shard_cut.assign(shard_nranks, {});
    shard_xidx.assign(shard_nranks, {});
    for (int s = 0; s < S.nsup; s++) {
      const int g = shard.owner[s];
      if (g < 0) continue;
      if (S.sn_parent[s] >= 0 && shard.owner[S.sn_parent[s]] < 0) shard_cut[g].push_back(s);
      for (int j = S.sn_first[s]; j < S.sn_first[s + 1]; j++) shard_xidx[g].push_back(S.perm[j]);
    }
  }
  // the plans' view of the fronts: a Schur handle is rank 0 of a split whose top part is S (never factored)
  const std::vector<int> owner = schur ? schur_owner(S, n - (int)schur_set.size()) : shard.owner;

  CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&stream_a, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&stream_b, cudaStreamNonBlocking));
  for (auto& e : ev_leaf) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  CK(cudaEventCreate(&ev0));
  CK(cudaEventCreate(&ev1));
  CK(cudaMallocHost((void**)&h_status, ST_COUNT * sizeof(int)));

  auto to_ll = [](const std::vector<int64_t>& v) { return std::vector<long long>(v.begin(), v.end()); };
  CK(upload(&dev.sn_first, S.sn_first));
  CK(upload(&dev.sn_rowptr, to_ll(S.sn_rowptr)));
  CK(upload(&dev.sn_rows, S.sn_rows));
  CK(upload(&dev.child_ptr, to_ll(S.child_ptr)));
  CK(upload(&dev.child_list, S.child_list));
  CK(upload(&dev.rel, S.rel));
  CK(upload(&dev.panel_off, to_ll(S.panel_off)));
  CK(upload(&dev.upd_off, to_ll(S.upd_off)));
  CK(upload(&dev.asm_ptr, to_ll(S.asm_ptr)));
  CK(upload(&dev.asm_src, S.asm_src));
  CK(upload(&dev.asm_dst, to_ll(S.asm_dst)));
  CK(upload(&dev.perm, S.perm));
  {
    std::vector<signed char> ds(n);
    for (int k = 0; k < n; k++) ds[k] = dsigns ? (signed char)dsigns[S.perm[k]] : (signed char)1;
    CK(upload(&dev.dsigns, ds));
  }
  nnzA = Ap[n];
  h_colptr.assign(Ap, Ap + n + 1);
  h_rowval.assign(Ai, Ai + nnzA);
  CK(cudaMalloc((void**)&dev.vals, (size_t)(nnzA ? nnzA : 1) * sizeof(double)));
  CK(cudaMemcpy(dev.vals, Ax, (size_t)nnzA * sizeof(double), cudaMemcpyHostToDevice));
  // The factor panels, the update-matrix arena and the update vectors are gigabytes (C4: 1.7 + 2.8 + 0.25 GB) and
  // cudaMalloc of that size takes a few tenths of a second: a helper thread allocates them while this one builds and
  // uploads the plans below (nothing in init touches these buffers; the first refactor does).  Joined before init returns.
  big_alloc_rc = 0;
  big_alloc = std::thread([this]() {
    if (cudaSetDevice(device) != cudaSuccess) { big_alloc_rc = 1; return; }
    const size_t nu = S.sn_rows.size() ? S.sn_rows.size() : 1;
    if (cudaMalloc((void**)&dev.L, ((size_t)(S.L_alloc ? S.L_alloc : 1) + 8) * sizeof(double)) != cudaSuccess ||   // + slack: a bulk copy of the last panel is rounded up to 16 bytes
        cudaMalloc((void**)&dev.U, (size_t)(S.upd_total ? S.upd_total : 1) * sizeof(double)) != cudaSuccess ||
        cudaMalloc((void**)&dev.u, nu * sizeof(double)) != cudaSuccess ||
        cudaMalloc((void**)&d_u2, nu * sizeof(double)) != cudaSuccess)
      big_alloc_rc = 1;
  });
  struct BigJoin { std::thread& t; ~BigJoin() { if (t.joinable()) t.join(); } } big_join{big_alloc};
  CK(cudaMalloc((void**)&dev.D, (size_t)n * sizeof(double)));
  CK(cudaMalloc((void**)&dev.Dinv, (size_t)n * sizeof(double)));
  CK(cudaMalloc((void**)&d_xp, (size_t)n * sizeof(double)));
  CK(cudaMalloc((void**)&d_xp2, (size_t)n * sizeof(double)));
  CK(cudaMalloc((void**)&d_bx, (size_t)2 * n * sizeof(double)));
  CK(cudaMalloc((void**)&dev.status, ST_COUNT * sizeof(int)));
  CK(cudaMemset(dev.status, 0, ST_COUNT * sizeof(int)));
  dev.reg_enable = o.regularize_enable;
  dev.reg_eps = o.regularize_eps;
  dev.reg_delta = o.regularize_delta;

  cb_tmark("ldl: uploads + device alloc");
  // plans (ldl_plan.cpp): the solve plan is built on a host thread beside the level-0 and factorisation plans
  int max_optin = 0, nsm = 0;
  CK(cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
  const int level_cap = (max_optin - 2048) / 8;  // doubles of the largest k_factor_level class
  // the solve slab size that goes with SV_MINB resident CTAs per SM (227 KB of shared memory per SM, 1 KB reserved per CTA)
  const size_t extra2 = (size_t)2 * (2 * CB_PB_MAXNS + SV_MAXROWS + 4 * CB_PB_MAXNS) * sizeof(double);   // NR = 2 vectors
  {
    const size_t per_cta = ((size_t)227 * 1024) / SV_MINB - 1024 - 64;
    sv_cap = (int)((per_cta - extra2) / sizeof(double)) - 2;
    sv_cap &= ~1;
    sv_cap = std::min(sv_cap, 16384);
  }
  SolvePlan sp;
  std::thread th_solve([&]() { sp = build_solve_plan(S, owner, shard_rank, sv_cap); });
  struct ThJoin { std::thread& t; ~ThJoin() { if (t.joinable()) t.join(); } } th_solve_guard{th_solve};
  Level0Plan l0 = build_level0_plan(S, owner, shard_rank, level_cap);
  FactorPlan fp = build_factor_plan(S, owner, shard_rank);
  th_solve.join();
  cb_tmark("ldl: plans");

  // tree level 0: plain launches
  CK(cudaFuncSetAttribute(k_factor_level<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, level_cap * 8));
  plan = std::move(l0.segs);
  CK(upload(&dev.level_tasks, l0.level_tasks));

  // dataflow factorisation (k_factor_df)
  CK(upload(&dev.sc_panel_src, fp.sc_panel_src));
  CK(upload(&dev.sc_panel_dst, fp.sc_panel_dst));
  CK(upload(&dev.sc_tile_src, fp.sc_tile_src));
  CK(upload(&dev.sc_tile_dst, fp.sc_tile_dst));
  if (std::getenv("CB_TIMING")) std::fprintf(stderr, "[cb timing]     factor plan: %zu tasks, %zu child records, %zu big fronts, %zu tiles\n",
                                              fp.tasks.size(), fp.recs.size(), fp.sc_panel_ptr.size() - 1, fp.sc_tile_ptr.size() - 1);
  dff.ntask = (int)fp.tasks.size();
  dff_ntask_owned = fp.ntask_owned;
  CK(upload(&dff.tasks, fp.tasks));
  CK(upload(&dff.recs, fp.recs));
  CK(upload(&d_dff_init, fp.cnt_init));
  CK(cudaMalloc((void**)&d_dff_cnt, fp.cnt_init.size() * sizeof(int) + 16));
  dff.pend = d_dff_cnt; dff.diag_done = d_dff_cnt + S.nsup; dff.rows_left = d_dff_cnt + 2 * (size_t)S.nsup;
  dff.tiles_left = d_dff_cnt + 3 * (size_t)S.nsup;
  CK(cudaMalloc((void**)&dff.qhead, sizeof(int)));
  CK(upload(&dff.parent, S.sn_parent));
  CK(upload(&dff.big_pos, fp.big_pos));
  CK(upload(&dff.tile_base, fp.tile_base));
  CK(cudaFuncSetAttribute(k_factor_df, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_SMEM_DOUBLES * 8));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_factor_df, DF_NT, (size_t)DF_SMEM_DOUBLES * 8));
  dff_grid = nsm * std::max(1, occ);
  dff_nsup4 = 4 * (size_t)S.nsup;
  if (std::getenv("CB_DF_TRACE") && dff.ntask > 0) {
    h_dff_tasks = fp.tasks;
    CK(cudaMalloc((void**)&dff.trace, (size_t)dff.ntask * 10 * sizeof(unsigned long long)));
    CK(cudaMemset(dff.trace, 0, (size_t)dff.ntask * 10 * sizeof(unsigned long long)));
  }

  // dataflow solves (ldl_solve.cuh)
  const int nt = (int)sp.tasks.size();
  sv_nwide = (int)sp.wide.size();
  sv_nleaf1 = (int)sp.leaf1.size(); sv_nleafn = (int)sp.leafn.size(); sv_nleafw = (int)sp.leafw.size();
  sv_leafw_nrmax = sp.leafw_nrmax;
  sv_leafw_grid = sv_nleafw;      // one CTA per front (a loop over fronts inside fewer CTAs was slower: 312 vs 189 us forward on C4)
  sv_ntask_owned = sp.ntask_owned;
  CK(upload(&dev.gat_ptr, sp.gat_ptr));
  CK(upload(&dev.gat_src, sp.gat_src));
  CK(upload(&d_sv_leaf1, sp.leaf1));
  CK(upload(&d_sv_leafn, sp.leafn));
  CK(upload(&d_sv_leafw, sp.leafw));
  CK(upload(&sv.fronts, sp.fronts));
  CK(upload(&sv.front2task, sp.front2task));
  CK(upload(&sv.parent, S.sn_parent));
  CK(upload(&sv.tasks, sp.tasks));
  // counters: [pend(nt) | fleft(nsup) | bleft(nsup)] are copied from their initial values before every solve,
  // [tdone(nt) | ydone(nsup) | done(nsup) | qhead(2)] are cleared
  sv_ninit = sp.cnt_init.size();
  sv_nzero = (size_t)nt + 2 * (size_t)S.nsup + 2;
  CK(upload(&d_sv_init, sp.cnt_init));
  CK(cudaMalloc((void**)&d_sv_cnt, (sv_ninit + sv_nzero) * sizeof(int)));
  sv.pend = d_sv_cnt; sv.fleft = d_sv_cnt + nt; sv.bleft = sv.fleft + S.nsup;
  sv.tdone = d_sv_cnt + sv_ninit; sv.ydone = sv.tdone + nt; sv.done = sv.ydone + S.nsup; sv.qhead = sv.done + S.nsup;
  sv.bpart_stride = (long long)(sp.nslots ? sp.nslots : 1) * CB_PB_MAXNS;
  CK(cudaMalloc((void**)&sv.bpart, (size_t)2 * sv.bpart_stride * sizeof(double)));
  sv.ntask = nt;
  // launch geometry: dynamic shared memory = slab + vectors for one or two right-hand sides
  for (int nr2 = 1; nr2 <= 2; nr2++)
    sv_smem[nr2 - 1] = ((size_t)sv_cap + 2 + (size_t)nr2 * (2 * CB_PB_MAXNS + SV_MAXROWS + 4 * CB_PB_MAXNS)) * sizeof(double);
  if ((rc = sv_configure())) return rc;
  const int sv_occ = sv_occupancy();
  if (sv_occ < 1) return CLDL_E_CUDA;
  sv_grid = nsm * sv_occ;
  use_dataflow = true;
  if (std::getenv("CB_DF_TRACE_SOLVE") && nt > 0) {
    CK(cudaMalloc((void**)&sv.trace, (size_t)nt * 8 * sizeof(unsigned long long)));
    CK(cudaMemset(sv.trace, 0, (size_t)nt * 8 * sizeof(unsigned long long)));
    h_sv_tasks = sp.tasks;
  }
  if (std::getenv("CB_TIMING") != nullptr) std::fprintf(stderr, "[cb timing]     solve plan: %d tasks (%d leaf columns, %d narrow leaves, %d wide leaves, %d wide fronts, %d row slabs), slab %d doubles, %d CTAs\n",
                                   nt, sv_nleaf1, sv_nleafn, sv_nleafw, sv_nwide, sp.nslots, sv_cap, sv_grid);
  cb_tmark("ldl: plan uploads");
  if (sharded()) {
    d_shard_xidx.assign(shard_nranks, nullptr);
    for (int w = 0; w < 2; w++) { d_shard_segs[w].assign(shard_nranks, nullptr); shard_nsegs[w].assign(shard_nranks, 0); }
    for (int g = 0; g < shard_nranks; g++) CK(upload(&d_shard_xidx[g], shard_xidx[g]));
  }
  if (schur && (rc = schur_setup(sp))) return rc;
  if (big_alloc.joinable()) big_alloc.join();
  if (big_alloc_rc) { std::fprintf(stderr, "[clarabel_b200] device allocation of the factor storage failed\n"); return CLDL_E_CUDA; }
  cb_tmark("ldl: big allocations joined");
  CK(cudaDeviceSynchronize());      // the uploads above are cudaMemcpy from pageable memory (staged, not necessarily landed); `stream` does not wait for the default stream
  factored = false;
  return CLDL_OK;
}

void LDLObject::release() {
  cudaSetDevice(device);
  for (auto& w : d_shard_segs) for (auto& p : w) if (p) { cudaFree(p); p = nullptr; }
  for (int* p : d_shard_xidx) if (p) cudaFree(p);
  d_shard_xidx.clear();
  if (nccl_comm) { if (NcclApi* a = nccl_api(nullptr)) a->CommDestroy((cb_ncclComm_t)nccl_comm); nccl_comm = nullptr; }
  if (d_xsend) { cudaFree(d_xsend); d_xsend = nullptr; }
  if (d_xrecv) { cudaFree(d_xrecv); d_xrecv = nullptr; }
  xbuf_cap = 0;
  auto fr = [](const void* p) { if (p) cudaFree((void*)p); };
  fr(dev.sn_first); fr(dev.sn_rowptr); fr(dev.sn_rows); fr(dev.child_ptr); fr(dev.child_list);
  fr(dev.rel); fr(dev.panel_off); fr(dev.upd_off); fr(dev.asm_ptr); fr(dev.asm_src);
  fr(dev.asm_dst); fr(dev.level_tasks); fr(dev.perm); fr(dev.dsigns); fr(dev.vals); fr(dev.L);
  fr(dev.U); fr(dev.D); fr(dev.Dinv); fr(dev.u); fr(dev.status); fr(d_xp); fr(d_bx);
  fr(d_tmp_idx); fr(d_tmp_val); fr(d_tmp_sgn); fr(sv.tasks); fr(sv.fronts); fr(sv.front2task); fr(sv.parent); fr(sv.bpart); fr(sv.trace); fr(d_sv_cnt); fr(d_sv_init); fr(d_sv_leaf1); fr(d_sv_leafn); fr(d_sv_leafw); fr(d_xp2); fr(d_u2); fr(dff.tasks); fr(dff.recs); fr(d_dff_init); fr(d_dff_cnt); fr(dff.qhead); fr(dff.parent); fr(dff.big_pos); fr(dff.tile_base); fr(dff.trace); fr(dev.gat_ptr); fr(dev.gat_src); fr(dev.sc_panel_src); fr(dev.sc_panel_dst); fr(dev.sc_tile_src); fr(dev.sc_tile_dst);
  fr(si.tasks); fr(si.col); fr(si.seg); fr(si.segpos); fr(si.Z); fr(d_si_pos); fr(d_si_init); fr(d_si_cnt); fr(d_si_out);
  fr(sv_bwd.tasks); fr(sv_bwd.parent); fr(d_sc_spos); fr(d_sc_kss_src); fr(d_sc_rec_ptr); fr(d_sc_kss_ptr); fr(d_sc_kss_dst);
  fr(d_sc_recs); fr(d_sc_out); fr(d_sc_vec);
  fr(d_adj_cp); fr(d_adj_rv); fr(d_adj_buf); fr(d_ld_ws); fr(d_ld_cnt);
  if (h_status) cudaFreeHost(h_status);
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  for (auto& e : ev_leaf) if (e) { cudaEventDestroy(e); e = nullptr; }
  if (stream_a) { cudaStreamDestroy(stream_a); stream_a = nullptr; }
  if (stream_b) { cudaStreamDestroy(stream_b); stream_b = nullptr; }
  if (stream) cudaStreamDestroy(stream);
}

// the start of every refactor: status, counters and queue head of k_factor_df reset, tree level 0 factored by the
// plain launches of `plan`
int LDLObject::refactor_level0() {
  CK(cudaMemsetAsync(dev.status, 0, ST_COUNT * sizeof(int), stream));
  CK(cudaMemcpyAsync(d_dff_cnt, d_dff_init, dff_nsup4 * sizeof(int), cudaMemcpyDeviceToDevice, stream));
  CK(cudaMemsetAsync(dff.qhead, 0, sizeof(int), stream));
  g_launches += plan.size();
  for (const LaunchSeg& g : plan) {
    if (g.leaf1) k_factor_leaf1<<<(g.count + LEAF1_NT / 32 - 1) / (LEAF1_NT / 32), LEAF1_NT, 0, stream>>>(dev, g.base, g.count);
    else if (g.threads == 64)
      k_factor_level<64><<<g.count, 64, (size_t)g.smem_doubles * 8, stream>>>(dev, g.base, g.smem_doubles);
    else
      k_factor_level<256><<<g.count, 256, (size_t)g.smem_doubles * 8, stream>>>(dev, g.base, g.smem_doubles);
  }
  return CLDL_OK;
}

int LDLObject::refactor_async() {
  if (sharded()) return has_transport() ? refactor_sharded() : CLDL_E_ARG;   // without a transport: the phase entry points
  CK(cudaSetDevice(device));
  factor_ok = false;
  schur_fwd = false;
  if (int rc = refactor_level0()) return rc;
  g_launches++;
  if (schur) {    // B's tasks only (they come first in the queue), then the complement from the cut roots
    DFFactor q = dff;
    q.ntask = dff_ntask_owned;
    k_factor_df<<<dff_grid, DF_NT, (size_t)DF_SMEM_DOUBLES * 8, stream>>>(dev, q);
    g_launches++;
    k_schur_assemble<<<schur_k, SC_NT, 0, stream>>>(dev.vals, dev.U, dev.sn_rows, schur_first, schur_k, d_sc_spos,
                                                     d_sc_kss_ptr, d_sc_kss_dst, d_sc_kss_src, d_sc_rec_ptr, d_sc_recs,
                                                     d_sc_out);
  } else {
    k_factor_df<<<dff_grid, DF_NT, (size_t)DF_SMEM_DOUBLES * 8, stream>>>(dev, dff);
  }
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(h_status, dev.status, ST_COUNT * sizeof(int), cudaMemcpyDeviceToHost, stream));
  factored = true;
  return CLDL_OK;
}

// the selected-inversion plan (ldl_plan.cpp) uploaded, Z panels and counters allocated: on the first call
int LDLObject::selinv_setup() {
  const SelinvPlan p = build_selinv_plan(S);
  si.ntask = (int)p.tasks.size();
  CK(upload(&si.tasks, p.tasks));
  CK(upload(&si.col, p.col));
  CK(upload(&si.seg, p.seg));
  CK(upload(&si.segpos, p.segpos));
  CK(upload(&d_si_pos, p.caller_pos));
  CK(upload(&d_si_init, p.rows_left));
  CK(cudaMalloc((void**)&d_si_cnt, (2 * (size_t)S.nsup + 1) * sizeof(int)));
  si.rows_left = d_si_cnt; si.done = d_si_cnt + S.nsup; si.qhead = d_si_cnt + 2 * (size_t)S.nsup;
  CK(cudaMalloc((void**)&si.Z, ((size_t)(S.L_alloc ? S.L_alloc : 1)) * sizeof(double)));
  CK(cudaFuncSetAttribute(k_selinv, cudaFuncAttributeMaxDynamicSharedMemorySize, SI_SMEM_DOUBLES * 8));
  int occ = 0, nsm = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_selinv, SI_NT, (size_t)SI_SMEM_DOUBLES * 8));
  CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
  if (occ < 1) return CLDL_E_CUDA;
  si_grid = nsm * occ;    // every CTA resident: a task only waits for tasks queued before it
  CK(cudaDeviceSynchronize());      // pageable uploads have landed before `stream` reads them
  return CLDL_OK;
}

int LDLObject::selected_inverse_async(double* d_out) {
  if (sharded() || schur) return CLDL_E_ARG;
  if (!factor_ok) return CLDL_E_NOT_FACTORED;
  CK(cudaSetDevice(device));
  if (!si.Z) {
    if (int rc = selinv_setup()) return rc;
  }
  CK(cudaMemcpyAsync(si.rows_left, d_si_init, (size_t)S.nsup * sizeof(int), cudaMemcpyDeviceToDevice, stream));
  CK(cudaMemsetAsync(si.done, 0, ((size_t)S.nsup + 1) * sizeof(int), stream));
  g_launches += 2;
  if (si.ntask) k_selinv<<<si_grid, SI_NT, (size_t)SI_SMEM_DOUBLES * 8, stream>>>(dev, si);
  if (nnzA) k_selinv_gather<<<(unsigned)((nnzA + 255) / 256), 256, 0, stream>>>(d_si_pos, si.Z, d_out, (long long)nnzA);
  CK(cudaGetLastError());
  return CLDL_OK;
}

// log|det(K + E)| as one deterministic sum of log|d_k| over the factored pivots (B's alone on a Schur handle); the sign
// from the negative-pivot count the refactor collected
int LDLObject::logdet(double* logabsdet, int32_t* sign) {
  if (sharded()) return CLDL_E_ARG;
  if (!factor_ok) return CLDL_E_NOT_FACTORED;
  CK(cudaSetDevice(device));
  if (!d_ld_ws) {
    CK(cudaMalloc((void**)&d_ld_ws, (RED_BLOCKS + 1) * sizeof(double)));
    CK(cudaMalloc((void**)&d_ld_cnt, sizeof(unsigned)));
    CK(cudaMemsetAsync(d_ld_cnt, 0, sizeof(unsigned), stream));   // k_sum's last block leaves it at 0 again
  }
  const int nf = schur ? schur_first : n;
  const double* D = dev.D;
  double* out = d_ld_ws + RED_BLOCKS;
  g_launches++;
  k_sum<<<red_grid(nf), RED_THREADS, 0, stream>>>(nf, [=] __device__(int k) { return log(fabs(D[k])); },
                                                  ReduceWS{d_ld_ws, d_ld_cnt}, out);
  CK(cudaGetLastError());
  double v = 0.0;
  CK(cudaMemcpyAsync(&v, out, sizeof(double), cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));
  *logabsdet = v;
  *sign = (((uint64_t)nf - positive_inertia) & 1) ? -1 : 1;
  return CLDL_OK;
}

// gb = (K + E)^-1 g by the solve's launch sequence, then (d_gvals non-null) the gradient of <g, x> on the caller's
// pattern by k_grad_P
int LDLObject::adjoint_async(const double* d_g, const double* d_x, double* d_gb, double* d_gvals) {
  if (sharded() || schur) return CLDL_E_ARG;
  if (!factor_ok) return CLDL_E_NOT_FACTORED;
  CK(cudaSetDevice(device));
  if (d_gvals && !d_adj_cp) {
    CK(upload(&d_adj_cp, h_colptr));
    CK(upload(&d_adj_rv, h_rowval));
    CK(cudaDeviceSynchronize());      // pageable uploads have landed before `stream` reads them
  }
  if (int rc = solve_async(d_gb, d_g)) return rc;
  if (d_gvals && nnzA) {
    g_launches++;
    k_grad_P<<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(n, d_adj_cp, d_adj_rv, d_x, d_gb, d_gvals);   // a warp per column
    CK(cudaGetLastError());
  }
  return CLDL_OK;
}

// the Schur plan (ldl_plan.cpp) uploaded and the complement allocated, at the end of init
int LDLObject::schur_setup(const SolvePlan& sp) {
  const SchurPlan p = build_schur_plan(S, schur_set, sp);
  schur_k = p.k;
  schur_first = p.first;
  for (int c : p.cut)     // their update matrices and vectors must hold S rows only
    if (S.sn_rowptr[c + 1] > S.sn_rowptr[c] && S.sn_rows[S.sn_rowptr[c]] < schur_first) return CLDL_E_ARG;
  const size_t kk = (size_t)schur_k * (size_t)schur_k;
  if (cudaMalloc((void**)&d_sc_out, kk * sizeof(double)) != cudaSuccess) {
    cudaGetLastError();
    d_sc_out = nullptr;
    std::fprintf(stderr, "[clarabel_b200] a Schur set of %d needs %zu bytes for the complement\n", schur_k, kk * sizeof(double));
    return CLDL_E_ARG;
  }
  CK(cudaMalloc((void**)&d_sc_vec, 2 * (size_t)schur_k * sizeof(double)));
  CK(upload(&d_sc_spos, p.spos));
  CK(upload(&d_sc_kss_ptr, p.kss_ptr));
  CK(upload(&d_sc_kss_dst, p.kss_dst));
  CK(upload(&d_sc_kss_src, p.kss_src));
  CK(upload(&d_sc_rec_ptr, p.rec_ptr));
  CK(upload(&d_sc_recs, p.recs));
  sv_bwd = sv;
  sv_bwd.ntask = (int)p.bwd.size();
  sv_bwd.tasks = nullptr;
  sv_bwd.parent = nullptr;
  sv_bwd.trace = nullptr;
  CK(upload(&sv_bwd.tasks, p.bwd.empty() ? std::vector<SVTask>(1) : p.bwd));
  CK(upload(&sv_bwd.parent, p.bparent));
  return CLDL_OK;
}

// condensation: permute b, forward over B (leaf kernels and the owned phase of the sweep), then w_S
int LDLObject::schur_reduce_async(double* d_wS, const double* d_b) {
  if (!schur) return CLDL_E_ARG;
  if (!factor_ok) return CLDL_E_NOT_FACTORED;
  CK(cudaSetDevice(device));
  SVRhs r;
  r.xp[0] = r.xp[1] = d_xp; r.u[0] = r.u[1] = dev.u; r.out[0] = r.out[1] = d_xp;
  g_launches += 2;
  k_permute_in<<<(n + 255) / 256, 256, 0, stream>>>(n, dev.perm, d_b, d_xp);
  if (int rc = sv_reset()) return rc;
  sv_leaves(true, 1, r);
  SVPlan qv = sv;
  qv.ntask = sv_ntask_owned;
  sv_sweep(true, 1, qv, r);
  k_schur_reduce<<<(schur_k + 255) / 256, 256, 0, stream>>>(schur_first, schur_k, d_sc_spos, d_sc_rec_ptr, d_sc_recs,
                                                             d_xp, dev.u, d_wS);
  CK(cudaGetLastError());
  schur_fwd = true;
  return CLDL_OK;
}

// expansion: x_S into the work vector (B's forward state from the last condensation), backward over B alone
int LDLObject::schur_expand_async(double* d_x, const double* d_xS) {
  if (!schur) return CLDL_E_ARG;
  if (!factor_ok) return CLDL_E_NOT_FACTORED;
  if (!schur_fwd) return CLDL_E_ARG;
  CK(cudaSetDevice(device));
  SVRhs r;
  r.xp[0] = r.xp[1] = d_xp; r.u[0] = r.u[1] = dev.u; r.out[0] = r.out[1] = d_x;
  g_launches++;
  k_schur_expand_in<<<(schur_k + 255) / 256, 256, 0, stream>>>(schur_first, schur_k, d_sc_spos, dev.perm, d_xS, d_xp, d_x);
  if (sv_bwd.ntask) sv_sweep(false, 1, sv_bwd, r);
  sv_leaves(false, 1, r);
  CK(cudaGetLastError());
  schur_fwd = false;     // the backward sweep overwrote the forward state
  return CLDL_OK;
}

int LDLObject::sync_status() {
  CK(cudaSetDevice(device));
  CK(cudaStreamSynchronize(stream));
  regularize_count = (uint64_t)h_status[ST_REGCOUNT];
  positive_inertia = (uint64_t)h_status[ST_POSINERTIA];
  if (dff.trace) {  // diagnostic: CB_DF_TRACE=<file> dumps the last refactor's task timeline
    std::vector<unsigned long long> tr((size_t)dff.ntask * 10);
    CK(cudaMemcpy(tr.data(), dff.trace, tr.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    if (FILE* fp = std::fopen(std::getenv("CB_DF_TRACE"), "wb")) {
      const long long nt = dff.ntask;
      std::fwrite(&nt, sizeof(nt), 1, fp);
      std::fwrite(h_dff_tasks.data(), sizeof(DFTask), (size_t)nt, fp);
      std::fwrite(tr.data(), sizeof(unsigned long long), tr.size(), fp);
      std::fclose(fp);
    }
  }
  if (h_status[ST_ZEROPIV] && !dev.reg_enable) return CLDL_E_ZERO_PIVOT;
  factor_ok = factored && !h_status[ST_NONFINITE];
  return h_status[ST_NONFINITE] ? 0 : 1;
}

// opt-in to the dynamic shared memory of the sweep kernels
int LDLObject::sv_configure() {
  CK(cudaFuncSetAttribute(k_solve2<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sv_smem[0]));
  CK(cudaFuncSetAttribute(k_solve2<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sv_smem[0]));
  CK(cudaFuncSetAttribute(k_solve2<true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sv_smem[1]));
  CK(cudaFuncSetAttribute(k_solve2<false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sv_smem[1]));
  return CLDL_OK;
}
int LDLObject::sv_occupancy() {
  // the two-right-hand-side instantiations need the most shared memory: they decide how many CTAs are co-resident
  int of = 0, ob = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&of, k_solve2<true, 2>, SV_NT, sv_smem[1]) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ob, k_solve2<false, 2>, SV_NT, sv_smem[1]) != cudaSuccess)
    return 0;
  return std::min(of, ob);
}

// one sweep kernel over the task queue as it stands (queue heads / counters are prepared by the caller)
void LDLObject::sv_sweep(bool fwd, int nrhs, const SVPlan& q, const SVRhs& r) {
  g_launches++;
  const size_t smem = sv_smem[nrhs - 1];
  if (fwd) { if (nrhs == 1) k_solve2<true, 1><<<sv_grid, SV_NT, smem, stream>>>(dev, q, r, sv_cap); else k_solve2<true, 2><<<sv_grid, SV_NT, smem, stream>>>(dev, q, r, sv_cap); }
  else { if (nrhs == 1) k_solve2<false, 1><<<sv_grid, SV_NT, smem, stream>>>(dev, q, r, sv_cap); else k_solve2<false, 2><<<sv_grid, SV_NT, smem, stream>>>(dev, q, r, sv_cap); }
}
// the level-0 fronts: before the forward sweep, after the backward sweep.  The three kernels touch disjoint fronts and
// none depends on another, so the two narrow-leaf kernels run on side streams next to the wide-leaf kernel
// (C4: 24 + 48 + 186 us one after the other -> ~190 us together)
void LDLObject::sv_leaves(bool fwd, int nrhs, const SVRhs& r) {
  const bool side = ((sv_nleaf1 ? 1 : 0) + (sv_nleafn ? 1 : 0) + (sv_nleafw ? 1 : 0)) > 1;
  cudaStream_t s1 = side ? stream_a : stream, sn = side ? stream_b : stream;
  if (side) {
    cudaEventRecord(ev_leaf[0], stream);
    cudaStreamWaitEvent(s1, ev_leaf[0], 0);
    cudaStreamWaitEvent(sn, ev_leaf[0], 0);
  }
  if (fwd) {
    if (sv_nleaf1) { g_launches++; if (nrhs == 1) k_fwd_leaf1<1><<<(sv_nleaf1 + 255) / 256, 256, 0, s1>>>(dev, d_sv_leaf1, sv_nleaf1, r); else k_fwd_leaf1<2><<<(sv_nleaf1 + 255) / 256, 256, 0, s1>>>(dev, d_sv_leaf1, sv_nleaf1, r); }
    if (sv_nleafn) { g_launches++; if (nrhs == 1) k_leaf_small<1, true><<<(sv_nleafn + 7) / 8, 256, 0, sn>>>(dev, d_sv_leafn, sv_nleafn, r); else k_leaf_small<2, true><<<(sv_nleafn + 7) / 8, 256, 0, sn>>>(dev, d_sv_leafn, sv_nleafn, r); }
    if (sv_nleafw) { g_launches++; if (nrhs == 1) k_fwd_leafw<1><<<sv_nleafw, SV_LEAF_NT, 0, stream>>>(dev, d_sv_leafw, sv_nleafw, r); else k_fwd_leafw<2><<<sv_nleafw, SV_LEAF_NT, 0, stream>>>(dev, d_sv_leafw, sv_nleafw, r); }
  } else {
    if (sv_nleafw) {
      g_launches++;
      const size_t sm = (size_t)nrhs * (sv_leafw_nrmax + CB_PB_MAXNS) * sizeof(double);
      if (nrhs == 1) k_bwd_leafw<1><<<sv_nleafw, SV_LEAF_NT, sm, stream>>>(dev, d_sv_leafw, sv_nleafw, r, sv_leafw_nrmax);
      else k_bwd_leafw<2><<<sv_nleafw, SV_LEAF_NT, sm, stream>>>(dev, d_sv_leafw, sv_nleafw, r, sv_leafw_nrmax);
    }
    if (sv_nleafn) { g_launches++; if (nrhs == 1) k_leaf_small<1, false><<<(sv_nleafn + 7) / 8, 256, 0, sn>>>(dev, d_sv_leafn, sv_nleafn, r); else k_leaf_small<2, false><<<(sv_nleafn + 7) / 8, 256, 0, sn>>>(dev, d_sv_leafn, sv_nleafn, r); }
    if (sv_nleaf1) { g_launches++; if (nrhs == 1) k_bwd_leaf1<1><<<(sv_nleaf1 + 255) / 256, 256, 0, s1>>>(dev, d_sv_leaf1, sv_nleaf1, r); else k_bwd_leaf1<2><<<(sv_nleaf1 + 255) / 256, 256, 0, s1>>>(dev, d_sv_leaf1, sv_nleaf1, r); }
  }
  if (side) {
    cudaEventRecord(ev_leaf[1], s1);
    cudaEventRecord(ev_leaf[2], sn);
    cudaStreamWaitEvent(stream, ev_leaf[1], 0);
    cudaStreamWaitEvent(stream, ev_leaf[2], 0);
  }
}
int LDLObject::sv_reset() {
  CK(cudaMemcpyAsync(d_sv_cnt, d_sv_init, sv_ninit * sizeof(int), cudaMemcpyDeviceToDevice, stream));
  CK(cudaMemsetAsync(d_sv_cnt + sv_ninit, 0, sv_nzero * sizeof(int), stream));
  return CLDL_OK;
}

// one right-hand side (d_x1 == nullptr) or two through the same sweeps (the panels are read once for both)
int LDLObject::solve_async(double* d_x, const double* d_b, double* d_x1, const double* d_b1) {
  const int nrhs = d_x1 ? 2 : 1;
  if (sharded()) {
    if (!has_transport()) return CLDL_E_ARG;
    int rc = solve_sharded(d_x, d_b);
    if (rc || nrhs == 1) return rc;
    return solve_sharded(d_x1, d_b1);
  }
  if (schur) return CLDL_E_ARG;   // S is never factored: schur_reduce_async / schur_expand_async
  if (!factored) return CLDL_E_NOT_FACTORED;
  CK(cudaSetDevice(device));
  SVRhs r;
  r.xp[0] = d_xp; r.u[0] = dev.u; r.out[0] = d_x;
  r.xp[1] = nrhs == 2 ? d_xp2 : d_xp; r.u[1] = nrhs == 2 ? d_u2 : dev.u; r.out[1] = nrhs == 2 ? d_x1 : d_x;
  g_launches += nrhs;
  k_permute_in<<<(n + 255) / 256, 256, 0, stream>>>(n, dev.perm, d_b, d_xp);
  if (nrhs == 2) k_permute_in<<<(n + 255) / 256, 256, 0, stream>>>(n, dev.perm, d_b1, d_xp2);
  int rc = sv_reset();
  if (rc) return rc;
  sv_leaves(true, nrhs, r);
  sv_sweep(true, nrhs, sv, r);
  sv_sweep(false, nrhs, sv, r);
  sv_leaves(false, nrhs, r);
  CK(cudaGetLastError());
  return CLDL_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// One factorisation on several GPUs (SURVEY 8e).  This object is one rank: it owns some subtrees of the assembly tree
// and replicates the top part above the cut.  Both dataflow queues list the owned tasks first, then the top tasks:
//   refactor phase 0  level-0 kernel + k_factor_df over the owned tasks
//            exchange the update matrix of every cut root goes to every rank (shard_pack / shard_unpack, what = 0)
//            phase 1  k_factor_df continues with the top tasks (queue head preset to the first of them)
//   solve    phase 0  permute b, forward sweep over the owned tasks
//            exchange update vectors of the cut roots (what = 1)
//            phase 1  forward sweep over the top tasks, backward sweep over everything (its dependencies point upwards)
//            exchange every rank's own x entries (what = 2): the all-gather of the solution the north star names
// The kernels are the single-GPU ones; only the host-side task lists, counter initialisation and launch sequence differ.
__global__ void k_gather_idx(int n, const int* __restrict__ idx, const double* __restrict__ x, double* __restrict__ buf) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) buf[i] = x[idx[i]];
}
__global__ void k_scatter_idx(int n, const int* __restrict__ idx, const double* __restrict__ buf, double* __restrict__ x) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[idx[i]] = buf[i];
}

int LDLObject::refactor_phase_async(int phase) {
  if (!sharded()) return CLDL_E_ARG;
  CK(cudaSetDevice(device));
  if (phase == 0) {
    if (int rc = refactor_level0()) return rc;
    DFFactor q = dff;
    q.ntask = dff_ntask_owned;
    g_launches++;
    k_factor_df<<<dff_grid, DF_NT, (size_t)DF_SMEM_DOUBLES * 8, stream>>>(dev, q);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(h_status, dev.status, ST_COUNT * sizeof(int), cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    shard_count_owned[0] = (uint64_t)h_status[ST_REGCOUNT];
    shard_count_owned[1] = (uint64_t)h_status[ST_POSINERTIA];
    factored = false;
    return CLDL_OK;
  }
  h_phase_start[0] = dff_ntask_owned;
  CK(cudaMemcpyAsync(dff.qhead, &h_phase_start[0], sizeof(int), cudaMemcpyHostToDevice, stream));
  g_launches++;
  k_factor_df<<<dff_grid, DF_NT, (size_t)DF_SMEM_DOUBLES * 8, stream>>>(dev, dff);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(h_status, dev.status, ST_COUNT * sizeof(int), cudaMemcpyDeviceToHost, stream));
  factored = true;
  return CLDL_OK;
}

int LDLObject::solve_phase_async(double* d_x, const double* d_b, int phase) {
  if (!sharded()) return CLDL_E_ARG;
  if (!factored) return CLDL_E_NOT_FACTORED;
  CK(cudaSetDevice(device));
  SVPlan qv = sv;
  SVRhs r;
  r.xp[0] = r.xp[1] = d_xp; r.u[0] = r.u[1] = dev.u; r.out[0] = r.out[1] = d_x;
  if (phase == 0) {
    g_launches++;
    k_permute_in<<<(n + 255) / 256, 256, 0, stream>>>(n, dev.perm, d_b, d_xp);
    int rc = sv_reset();
    if (rc) return rc;
    sv_leaves(true, 1, r);
    qv.ntask = sv_ntask_owned;
    sv_sweep(true, 1, qv, r);
  } else {
    h_phase_start[1] = sv_ntask_owned;
    CK(cudaMemcpyAsync(qv.qhead, &h_phase_start[1], sizeof(int), cudaMemcpyHostToDevice, stream));
    sv_sweep(true, 1, qv, r);
    sv_sweep(false, 1, qv, r);
    sv_leaves(false, 1, r);
  }
  CK(cudaGetLastError());
  return CLDL_OK;
}

int LDLObject::set_nccl(const char* libpath, const unsigned char* id128, int nranks, int rank) {
  if (!sharded() || nranks != shard_nranks || rank != shard_rank) return CLDL_E_ARG;
  NcclApi* a = nccl_api(libpath);
  if (!a) return CLDL_E_CUDA;
  CK(cudaSetDevice(device));
  cb_ncclUniqueId id;
  std::memcpy(id.internal, id128, 128);
  cb_ncclComm_t c = nullptr;
  const int r = a->CommInitRank(&c, nranks, id, rank);
  if (r != 0) { std::fprintf(stderr, "[clarabel_b200] ncclCommInitRank: %s\n", a->GetErrorString ? a->GetErrorString(r) : "error"); return CLDL_E_CUDA; }
  nccl_comm = c;
  nccl_allgather = a->AllGather; nccl_error = a->GetErrorString;
  return CLDL_OK;
}

// padded all-gather of one kind of contribution through the installed transport
int LDLObject::exchange(int what, double* d_x) {
  uint64_t cnt = 1;
  for (int r = 0; r < shard_nranks; r++) cnt = std::max(cnt, shard_count(what, r));
  if ((size_t)cnt > xbuf_cap) {
    if (d_xsend) cudaFree(d_xsend);
    if (d_xrecv) cudaFree(d_xrecv);
    xbuf_cap = (size_t)cnt + (size_t)cnt / 4 + 64;
    CK(cudaMalloc((void**)&d_xsend, xbuf_cap * sizeof(double)));
    CK(cudaMalloc((void**)&d_xrecv, xbuf_cap * (size_t)shard_nranks * sizeof(double)));
  }
  int rc = shard_pack(what, d_xsend, d_x);
  if (rc) return rc;
  if ((rc = allgather(d_xsend, d_xrecv, cnt))) return rc;
  for (int r = 0; r < shard_nranks; r++)
    if (r != shard_rank && (rc = shard_unpack(what, r, d_xrecv + (size_t)r * cnt, d_x))) return rc;
  return CLDL_OK;
}
int LDLObject::refactor_sharded() {
  int rc = refactor_phase_async(0);
  if (rc) return rc;
  if ((rc = exchange(0, nullptr))) return rc;
  return refactor_phase_async(1);
}
int LDLObject::solve_sharded(double* d_x, const double* d_b) {
  int rc = solve_phase_async(d_x, d_b, 0);
  if (rc) return rc;
  if ((rc = exchange(1, nullptr))) return rc;
  if ((rc = solve_phase_async(d_x, d_b, 1))) return rc;
  return exchange(2, d_x);
}

uint64_t LDLObject::shard_count(int what, int rank) const {
  if (!sharded() || rank < 0 || rank >= shard_nranks) return 0;
  if (what == 2) return (uint64_t)shard_xidx[rank].size();
  uint64_t t = 0;
  for (int c : shard_cut[rank]) {
    const uint64_t nr = (uint64_t)(S.sn_rowptr[c + 1] - S.sn_rowptr[c]);
    t += what == 0 ? nr * nr : nr;
  }
  return t;
}
// a list of contiguous segments copied by one launch (one CTA per segment): the cut roots' update matrices / vectors
// between the arena and the packed exchange buffer (64 separate cudaMemcpyAsync per exchange on C4 otherwise)
__global__ void k_copy_segs(const long long* __restrict__ seg, double* __restrict__ arena, double* __restrict__ buf, int to_buf) {
  const long long a = seg[3 * blockIdx.x], b = seg[3 * blockIdx.x + 1], len = seg[3 * blockIdx.x + 2];
  if (to_buf) for (long long i = threadIdx.x; i < len; i += blockDim.x) buf[b + i] = arena[a + i];
  else for (long long i = threadIdx.x; i < len; i += blockDim.x) arena[a + i] = buf[b + i];
}
int LDLObject::shard_seglist(int what, int rank, const long long** d_out, int* nseg) {
  auto& slot = d_shard_segs[what][rank];
  if (!slot) {
    std::vector<long long> h;
    long long off = 0;
    for (int c : shard_cut[rank]) {
      const long long nr = S.sn_rowptr[c + 1] - S.sn_rowptr[c];
      const long long len = what == 0 ? nr * nr : nr;
      if (len) { h.push_back(what == 0 ? (long long)S.upd_off[c] : (long long)S.sn_rowptr[c]); h.push_back(off); h.push_back(len); }
      off += len;
    }
    shard_nsegs[what][rank] = (int)(h.size() / 3);
    if (h.empty()) h.assign(3, 0);
    long long* dp = nullptr;
    CK(cudaMalloc((void**)&dp, h.size() * sizeof(long long)));
    CK(cudaMemcpy(dp, h.data(), h.size() * sizeof(long long), cudaMemcpyHostToDevice));
    CK(cudaDeviceSynchronize());
    slot = dp;
  }
  *d_out = slot; *nseg = shard_nsegs[what][rank];
  return CLDL_OK;
}
// my contribution -> d_buf (contiguous, in the order of shard_cut[rank] / shard_xidx[rank])
int LDLObject::shard_pack(int what, double* d_buf, const double* d_x) {
  if (!sharded()) return CLDL_E_ARG;
  CK(cudaSetDevice(device));
  if (what == 2) {
    const int cnt = (int)shard_xidx[shard_rank].size();
    if (cnt) { g_launches++; k_gather_idx<<<(cnt + 255) / 256, 256, 0, stream>>>(cnt, d_shard_xidx[shard_rank], d_x, d_buf); }
    return CLDL_OK;
  }
  const long long* segs = nullptr;
  int nseg = 0;
  int rc = shard_seglist(what, shard_rank, &segs, &nseg);
  if (rc) return rc;
  if (nseg) { g_launches++; k_copy_segs<<<nseg, 256, 0, stream>>>(segs, what == 0 ? dev.U : dev.u, d_buf, 1); }
  return CLDL_OK;
}
// rank `rank`'s contribution (as packed there) -> this rank's arena / update vectors / x
int LDLObject::shard_unpack(int what, int rank, const double* d_buf, double* d_x) {
  if (!sharded() || rank < 0 || rank >= shard_nranks) return CLDL_E_ARG;
  if (rank == shard_rank) return CLDL_OK;
  CK(cudaSetDevice(device));
  if (what == 2) {
    const int cnt = (int)shard_xidx[rank].size();
    if (cnt) { g_launches++; k_scatter_idx<<<(cnt + 255) / 256, 256, 0, stream>>>(cnt, d_shard_xidx[rank], d_buf, d_x); }
    return CLDL_OK;
  }
  const long long* segs = nullptr;
  int nseg = 0;
  int rc = shard_seglist(what, rank, &segs, &nseg);
  if (rc) return rc;
  if (nseg) { g_launches++; k_copy_segs<<<nseg, 256, 0, stream>>>(segs, what == 0 ? dev.U : dev.u, const_cast<double*>(d_buf), 0); }
  return CLDL_OK;
}

int LDLObject::ensure_tmp(size_t len) {
  if (len <= tmp_cap) return 0;
  CK(cudaSetDevice(device));
  if (d_tmp_idx) cudaFree(d_tmp_idx);
  if (d_tmp_val) cudaFree(d_tmp_val);
  if (d_tmp_sgn) cudaFree(d_tmp_sgn);
  tmp_cap = len + len / 2 + 256;
  CK(cudaMalloc((void**)&d_tmp_idx, tmp_cap * sizeof(int)));
  CK(cudaMalloc((void**)&d_tmp_val, tmp_cap * sizeof(double)));
  CK(cudaMalloc((void**)&d_tmp_sgn, tmp_cap));
  return 0;
}

int LDLObject::stage_index(const uint64_t* index, uint64_t len) {
  int rc = ensure_tmp(len);
  if (rc) return rc;
  h_idx.resize(len);
  for (uint64_t i = 0; i < len; i++) {
    if (index[i] >= (uint64_t)nnzA) return CLDL_E_ARG;
    h_idx[i] = (int)index[i];
  }
  CK(cudaMemcpyAsync(d_tmp_idx, h_idx.data(), len * sizeof(int), cudaMemcpyHostToDevice, stream));
  return 0;
}

}  // namespace cb

// ------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------
using cb::LDLObject;

struct cldl_handle { LDLObject obj; };

extern "C" {

void cldl_default_opts(cldl_opts* o) {
  std::memset(o, 0, sizeof(*o));
  o->regularize_eps = 1e-13;    // default/settings.rs:155-158
  o->regularize_delta = 2e-7;   // default/settings.rs:159-161
  o->regularize_enable = 1;
  o->amd_dense_scale = 1.5;
  o->ordering = CLDL_ORDER_BEST;
  o->device = 0;
  o->max_panel = 0;
  o->nd_leaf = 0;
}

int cldl_create(cldl_t** out, uint64_t n, const uint64_t* colptr, const uint64_t* rowval,
                const double* nzval, const int8_t* dsigns, const cldl_opts* opts,
                const uint64_t* perm_or_null) {
  if (!out) return CLDL_E_ARG;
  *out = nullptr;
  if (!colptr || !rowval || !nzval || n == 0 || n > 0x7fffffffu) return CLDL_E_DIM;
  cldl_opts o;
  if (opts) o = *opts; else cldl_default_opts(&o);
  uint64_t nnz = colptr[n];
  if (nnz > 0x7fffffffu) return CLDL_E_DIM;
  std::vector<int64_t> Ap(n + 1);
  std::vector<int32_t> Ai(nnz);
  for (uint64_t j = 0; j <= n; j++) Ap[j] = (int64_t)colptr[j];
  for (uint64_t p = 0; p < nnz; p++) {
    if (rowval[p] >= n) return CLDL_E_DIM;
    Ai[p] = (int32_t)rowval[p];
  }
  std::vector<int> perm;
  if (perm_or_null) {
    perm.resize(n);
    for (uint64_t k = 0; k < n; k++) {
      if (perm_or_null[k] >= n) return CLDL_E_BAD_PERM;
      perm[k] = (int)perm_or_null[k];
    }
  }
  cldl_handle* h = new (std::nothrow) cldl_handle();
  if (!h) return CLDL_E_ARG;
  int rc = h->obj.init((int)n, Ap.data(), Ai.data(), nzval, dsigns, o,
                       perm_or_null ? perm.data() : nullptr);
  if (rc != CLDL_OK) {
    h->obj.release();
    delete h;
    return rc;
  }
  *out = h;
  return CLDL_OK;
}

void cldl_destroy(cldl_t* h) {
  if (!h) return;
  h->obj.release();
  delete h;
}

int cldl_update_values(cldl_t* h, const uint64_t* index, const double* values, uint64_t len) {
  if (!h) return CLDL_E_ARG;
  if (len == 0) return CLDL_OK;
  LDLObject& o = h->obj;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  int rc = o.stage_index(index, len);
  if (rc) return rc;
  if (cudaMemcpyAsync(o.d_tmp_val, values, len * sizeof(double), cudaMemcpyHostToDevice, o.stream) != cudaSuccess)
    return CLDL_E_CUDA;
  cb::k_update_values<<<(unsigned)((len + 255) / 256), 256, 0, o.stream>>>(o.dev.vals, o.d_tmp_idx, o.d_tmp_val, (long long)len);
  return cudaStreamSynchronize(o.stream) == cudaSuccess ? CLDL_OK : CLDL_E_CUDA;
}

int cldl_scale_values(cldl_t* h, const uint64_t* index, uint64_t len, double scale) {
  if (!h) return CLDL_E_ARG;
  if (len == 0) return CLDL_OK;
  LDLObject& o = h->obj;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  int rc = o.stage_index(index, len);
  if (rc) return rc;
  cb::k_scale_values<<<(unsigned)((len + 255) / 256), 256, 0, o.stream>>>(o.dev.vals, o.d_tmp_idx, scale, (long long)len);
  return cudaStreamSynchronize(o.stream) == cudaSuccess ? CLDL_OK : CLDL_E_CUDA;
}

int cldl_offset_values(cldl_t* h, const uint64_t* index, uint64_t len, double offset,
                       const int8_t* signs) {
  if (!h || !signs) return CLDL_E_ARG;
  if (len == 0) return CLDL_OK;
  LDLObject& o = h->obj;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  int rc = o.stage_index(index, len);
  if (rc) return rc;
  if (cudaMemcpyAsync(o.d_tmp_sgn, signs, len, cudaMemcpyHostToDevice, o.stream) != cudaSuccess)
    return CLDL_E_CUDA;
  cb::k_offset_values<<<(unsigned)((len + 255) / 256), 256, 0, o.stream>>>(o.dev.vals, o.d_tmp_idx, offset, o.d_tmp_sgn, (long long)len);
  return cudaStreamSynchronize(o.stream) == cudaSuccess ? CLDL_OK : CLDL_E_CUDA;
}

int cldl_refactor(cldl_t* h) {
  if (!h) return CLDL_E_ARG;
  int rc = h->obj.refactor_async();
  if (rc) return rc;
  return h->obj.sync_status();
}

int cldl_solve(cldl_t* h, double* x, const double* b) {
  if (!h || !x || !b) return CLDL_E_ARG;
  LDLObject& o = h->obj;
  if (o.schur) return CLDL_E_ARG;
  if (!o.factored) return CLDL_E_NOT_FACTORED;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  size_t bytes = (size_t)o.n * sizeof(double);
  if (cudaMemcpyAsync(o.d_bx, b, bytes, cudaMemcpyHostToDevice, o.stream) != cudaSuccess) return CLDL_E_CUDA;
  int rc = o.solve_async(o.d_bx + o.n, o.d_bx);
  if (rc) return rc;
  if (cudaMemcpyAsync(x, o.d_bx + o.n, bytes, cudaMemcpyDeviceToHost, o.stream) != cudaSuccess) return CLDL_E_CUDA;
  if (cudaStreamSynchronize(o.stream) != cudaSuccess) return CLDL_E_CUDA;
  if (o.sv.trace) {   // diagnostic: CB_DF_TRACE_SOLVE=<file> dumps the last solve's task timeline (scripts/df_trace_solve.py)
    const long long nt = o.sv.ntask;
    std::vector<unsigned long long> tr((size_t)nt * 8);
    cudaMemcpy(tr.data(), o.sv.trace, tr.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
    if (FILE* fp = std::fopen(std::getenv("CB_DF_TRACE_SOLVE"), "wb")) {
      std::fwrite(&nt, sizeof(nt), 1, fp);
      std::fwrite(o.h_sv_tasks.data(), sizeof(cb::SVTask), (size_t)nt, fp);
      std::fwrite(tr.data(), sizeof(unsigned long long), tr.size(), fp);
      std::fclose(fp);
    }
  }
  return CLDL_OK;
}

void cldl_info(const cldl_t* h, cldl_info_t* info) {
  if (!h || !info) return;
  const LDLObject& o = h->obj;
  std::memset(info, 0, sizeof(*info));
  std::strncpy(info->name, "cudaldl", sizeof(info->name) - 1);
  info->threads = 0;
  info->direct = 1;
  info->nnzA = (uint64_t)o.nnzA;
  info->nnzL = (uint64_t)o.S.nnzL_simplicial;
  info->nnzL_stored = (uint64_t)o.S.nnzL_stored;
  info->regularize_count = o.regularize_count;
  info->positive_inertia = o.positive_inertia;
  info->n_supernodes = (uint64_t)o.S.nsup;
  info->n_levels = (uint64_t)o.S.nlevels;
  info->flops = o.S.flops_stored;
  info->ordering_used = o.S.ordering_used;
}

int cldl_get_perm(const cldl_t* h, uint64_t* perm_out) {
  if (!h || !perm_out) return CLDL_E_ARG;
  for (int k = 0; k < h->obj.n; k++) perm_out[k] = (uint64_t)h->obj.S.perm[k];
  return CLDL_OK;
}

int cldl_get_factor(const cldl_t* h, double* L_out, double* D_out, double* Dinv_out) {
  if (!h || !L_out || !D_out || !Dinv_out) return CLDL_E_ARG;
  const LDLObject& o = h->obj;
  if (!o.factored) return CLDL_E_NOT_FACTORED;
  if (cudaSetDevice(o.device) != cudaSuccess || cudaStreamSynchronize(o.stream) != cudaSuccess) return CLDL_E_CUDA;
  std::vector<double> all((size_t)o.S.L_alloc);
  if (cudaMemcpy(all.data(), o.dev.L, all.size() * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(D_out, o.dev.D, (size_t)o.n * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(Dinv_out, o.dev.Dinv, (size_t)o.n * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess)
    return CLDL_E_CUDA;
  // panels start on 32-byte boundaries in device memory; the padding between them is never written
  size_t pos = 0;
  for (int s = 0; s < o.S.nsup; s++) {
    const size_t ns = (size_t)(o.S.sn_first[s + 1] - o.S.sn_first[s]), nr = (size_t)(o.S.sn_rowptr[s + 1] - o.S.sn_rowptr[s]);
    std::memcpy(L_out + pos, all.data() + o.S.panel_off[s], (ns + nr) * ns * sizeof(double));
    pos += (ns + nr) * ns;
  }
  return CLDL_OK;
}

int cldl_selected_inverse(cldl_t* h, double* nzval_out) {
  if (!h || !nzval_out) return CLDL_E_ARG;
  LDLObject& o = h->obj;
  if (!o.sharded() && !o.schur && o.factor_ok && !o.d_si_out) {
    if (cudaSetDevice(o.device) != cudaSuccess ||
        cudaMalloc((void**)&o.d_si_out, (size_t)(o.nnzA ? o.nnzA : 1) * sizeof(double)) != cudaSuccess)
      return CLDL_E_CUDA;
  }
  int rc = o.selected_inverse_async(o.d_si_out);
  if (rc) return rc;
  if (cudaMemcpyAsync(nzval_out, o.d_si_out, (size_t)o.nnzA * sizeof(double), cudaMemcpyDeviceToHost, o.stream) != cudaSuccess ||
      cudaStreamSynchronize(o.stream) != cudaSuccess)
    return CLDL_E_CUDA;
  return CLDL_OK;
}
int cldl_selected_inverse_dev(cldl_t* h, double* d_nzval_out) {
  if (!h || !d_nzval_out) return CLDL_E_ARG;
  return h->obj.selected_inverse_async(d_nzval_out);
}

int cldl_logdet(cldl_t* h, double* logabsdet, int32_t* sign) {
  if (!h || !logabsdet || !sign) return CLDL_E_ARG;
  return h->obj.logdet(logabsdet, sign);
}

int cldl_adjoint_solve(cldl_t* h, const double* g, const double* x, double* gb, double* gvals) {
  if (!h || !g || !gb || (gvals && !x)) return CLDL_E_ARG;
  LDLObject& o = h->obj;
  if (o.sharded() || o.schur) return CLDL_E_ARG;
  if (!o.factor_ok) return CLDL_E_NOT_FACTORED;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  const size_t n = (size_t)o.n, nnz = (size_t)o.nnzA;
  if (!o.d_adj_buf && cudaMalloc((void**)&o.d_adj_buf, (3 * n + (nnz ? nnz : 1)) * sizeof(double)) != cudaSuccess) {
    o.d_adj_buf = nullptr;
    return CLDL_E_CUDA;
  }
  double *dg = o.d_adj_buf, *dx = dg + n, *dgb = dx + n, *dv = dgb + n;
  if (cudaMemcpyAsync(dg, g, n * sizeof(double), cudaMemcpyHostToDevice, o.stream) != cudaSuccess ||
      (gvals && cudaMemcpyAsync(dx, x, n * sizeof(double), cudaMemcpyHostToDevice, o.stream) != cudaSuccess))
    return CLDL_E_CUDA;
  int rc = o.adjoint_async(dg, dx, dgb, gvals ? dv : nullptr);
  if (rc) return rc;
  if (cudaMemcpyAsync(gb, dgb, n * sizeof(double), cudaMemcpyDeviceToHost, o.stream) != cudaSuccess ||
      (gvals && cudaMemcpyAsync(gvals, dv, nnz * sizeof(double), cudaMemcpyDeviceToHost, o.stream) != cudaSuccess) ||
      cudaStreamSynchronize(o.stream) != cudaSuccess)
    return CLDL_E_CUDA;
  return CLDL_OK;
}
int cldl_adjoint_solve_dev(cldl_t* h, const double* d_g, const double* d_x, double* d_gb, double* d_gvals) {
  if (!h || !d_g || !d_gb || (d_gvals && !d_x)) return CLDL_E_ARG;
  return h->obj.adjoint_async(d_g, d_x, d_gb, d_gvals);
}

int cldl_create_schur(cldl_t** out, uint64_t n, const uint64_t* colptr, const uint64_t* rowval,
                      const double* nzval, const int8_t* dsigns, const cldl_opts* opts,
                      const uint64_t* perm_or_null, uint64_t nschur, const uint64_t* schur_idx) {
  if (!out) return CLDL_E_ARG;
  *out = nullptr;
  if (!colptr || !rowval || !nzval || n == 0 || n > 0x7fffffffu) return CLDL_E_DIM;
  if (!schur_idx || nschur == 0 || nschur >= n) return CLDL_E_ARG;
  if (opts && opts->shard_nranks > 1) return CLDL_E_ARG;
  const uint64_t nnz = colptr[n];
  if (nnz > 0x7fffffffu) return CLDL_E_DIM;
  std::vector<int64_t> Ap(n + 1);
  std::vector<int32_t> Ai(nnz);
  for (uint64_t j = 0; j <= n; j++) Ap[j] = (int64_t)colptr[j];
  for (uint64_t p = 0; p < nnz; p++) {
    if (rowval[p] >= n) return CLDL_E_DIM;
    Ai[p] = (int32_t)rowval[p];
  }
  std::vector<int> perm;
  if (perm_or_null) {
    perm.resize(n);
    for (uint64_t k = 0; k < n; k++) {
      if (perm_or_null[k] >= n) return CLDL_E_BAD_PERM;
      perm[k] = (int)perm_or_null[k];
    }
  }
  std::vector<int> sidx(nschur);
  for (uint64_t i = 0; i < nschur; i++) {
    if (schur_idx[i] >= n) return CLDL_E_ARG;
    sidx[i] = (int)schur_idx[i];
  }
  cldl_opts o;
  if (opts) o = *opts; else cldl_default_opts(&o);
  cldl_handle* h = new (std::nothrow) cldl_handle();
  if (!h) return CLDL_E_ARG;
  h->obj.schur_set = std::move(sidx);
  int rc = h->obj.init((int)n, Ap.data(), Ai.data(), nzval, dsigns, o, perm_or_null ? perm.data() : nullptr);
  if (rc != CLDL_OK) {
    h->obj.release();
    delete h;
    return rc;
  }
  *out = h;
  return CLDL_OK;
}

int cldl_schur_complement_dev(cldl_t* h, double* d_out) {
  if (!h || !d_out) return CLDL_E_ARG;
  LDLObject& o = h->obj;
  if (!o.schur) return CLDL_E_ARG;
  if (!o.factor_ok) return CLDL_E_NOT_FACTORED;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  const size_t bytes = (size_t)o.schur_k * (size_t)o.schur_k * sizeof(double);
  return cudaMemcpyAsync(d_out, o.d_sc_out, bytes, cudaMemcpyDeviceToDevice, o.stream) == cudaSuccess ? CLDL_OK : CLDL_E_CUDA;
}
int cldl_schur_complement(cldl_t* h, double* out) {
  if (!h || !out) return CLDL_E_ARG;
  LDLObject& o = h->obj;
  if (!o.schur) return CLDL_E_ARG;
  if (!o.factor_ok) return CLDL_E_NOT_FACTORED;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  const size_t bytes = (size_t)o.schur_k * (size_t)o.schur_k * sizeof(double);
  if (cudaMemcpyAsync(out, o.d_sc_out, bytes, cudaMemcpyDeviceToHost, o.stream) != cudaSuccess ||
      cudaStreamSynchronize(o.stream) != cudaSuccess)
    return CLDL_E_CUDA;
  return CLDL_OK;
}
int cldl_schur_reduce_dev(cldl_t* h, double* d_wS, const double* d_b) {
  if (!h || !d_wS || !d_b) return CLDL_E_ARG;
  return h->obj.schur_reduce_async(d_wS, d_b);
}
int cldl_schur_reduce(cldl_t* h, double* wS, const double* b) {
  if (!h || !wS || !b) return CLDL_E_ARG;
  LDLObject& o = h->obj;
  if (!o.schur) return CLDL_E_ARG;
  if (!o.factor_ok) return CLDL_E_NOT_FACTORED;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  const size_t k = (size_t)o.schur_k;
  if (cudaMemcpyAsync(o.d_bx, b, (size_t)o.n * sizeof(double), cudaMemcpyHostToDevice, o.stream) != cudaSuccess) return CLDL_E_CUDA;
  int rc = o.schur_reduce_async(o.d_sc_vec, o.d_bx);
  if (rc) return rc;
  if (cudaMemcpyAsync(wS, o.d_sc_vec, k * sizeof(double), cudaMemcpyDeviceToHost, o.stream) != cudaSuccess ||
      cudaStreamSynchronize(o.stream) != cudaSuccess)
    return CLDL_E_CUDA;
  return CLDL_OK;
}
int cldl_schur_expand_dev(cldl_t* h, double* d_x, const double* d_xS) {
  if (!h || !d_x || !d_xS) return CLDL_E_ARG;
  return h->obj.schur_expand_async(d_x, d_xS);
}
int cldl_schur_expand(cldl_t* h, double* x, const double* xS) {
  if (!h || !x || !xS) return CLDL_E_ARG;
  LDLObject& o = h->obj;
  if (!o.schur) return CLDL_E_ARG;
  if (!o.factor_ok) return CLDL_E_NOT_FACTORED;
  if (!o.schur_fwd) return CLDL_E_ARG;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  const size_t k = (size_t)o.schur_k;
  if (cudaMemcpyAsync(o.d_sc_vec + k, xS, k * sizeof(double), cudaMemcpyHostToDevice, o.stream) != cudaSuccess) return CLDL_E_CUDA;
  int rc = o.schur_expand_async(o.d_bx + o.n, o.d_sc_vec + k);
  if (rc) return rc;
  if (cudaMemcpyAsync(x, o.d_bx + o.n, (size_t)o.n * sizeof(double), cudaMemcpyDeviceToHost, o.stream) != cudaSuccess ||
      cudaStreamSynchronize(o.stream) != cudaSuccess)
    return CLDL_E_CUDA;
  return CLDL_OK;
}

int cldl_update_values_dev(cldl_t* h, const int32_t* d_index, const double* d_values, uint64_t len) {
  if (!h) return CLDL_E_ARG;
  if (len == 0) return CLDL_OK;
  LDLObject& o = h->obj;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  cb::k_update_values<<<(unsigned)((len + 255) / 256), 256, 0, o.stream>>>(o.dev.vals, d_index, d_values, (long long)len);
  return CLDL_OK;
}

int cldl_set_values_dev(cldl_t* h, const double* d_nzval) {
  if (!h) return CLDL_E_ARG;
  LDLObject& o = h->obj;
  if (cudaSetDevice(o.device) != cudaSuccess) return CLDL_E_CUDA;
  return cudaMemcpyAsync(o.dev.vals, d_nzval, (size_t)o.nnzA * sizeof(double), cudaMemcpyDeviceToDevice, o.stream) == cudaSuccess
             ? CLDL_OK : CLDL_E_CUDA;
}

int cldl_refactor_dev(cldl_t* h) { return h ? h->obj.refactor_async() : CLDL_E_ARG; }
int cldl_solve_dev(cldl_t* h, double* d_x, const double* d_b) {
  return h ? h->obj.solve_async(d_x, d_b) : CLDL_E_ARG;
}
int cldl_sync_status(cldl_t* h) { return h ? h->obj.sync_status() : CLDL_E_ARG; }
// ---- one factorisation on several GPUs: device-pointer phase API (see clarabel_b200.h) ----
int cldl_shard_refactor_phase_dev(cldl_t* h, int phase) { return h ? h->obj.refactor_phase_async(phase) : CLDL_E_ARG; }
int cldl_shard_solve_phase_dev(cldl_t* h, double* d_x, const double* d_b, int phase) { return h ? h->obj.solve_phase_async(d_x, d_b, phase) : CLDL_E_ARG; }
uint64_t cldl_shard_count(const cldl_t* h, int what, int rank) { return h ? h->obj.shard_count(what, rank) : 0; }
int cldl_shard_pack_dev(cldl_t* h, int what, double* d_buf, const double* d_x) { return h ? h->obj.shard_pack(what, d_buf, d_x) : CLDL_E_ARG; }
int cldl_shard_unpack_dev(cldl_t* h, int what, int rank, const double* d_buf, double* d_x) { return h ? h->obj.shard_unpack(what, rank, d_buf, d_x) : CLDL_E_ARG; }
int cldl_nccl_unique_id(const char* libpath, unsigned char* id128) {
  cb::NcclApi* a = cb::nccl_api(libpath);
  if (!a || !id128) return CLDL_E_CUDA;
  cb::cb_ncclUniqueId id;
  if (a->GetUniqueId(&id) != 0) return CLDL_E_CUDA;
  std::memcpy(id128, id.internal, 128);
  return CLDL_OK;
}
int cldl_set_nccl(cldl_t* h, const char* libpath, const unsigned char* id128, int nranks, int rank) {
  return h ? h->obj.set_nccl(libpath, id128, nranks, rank) : CLDL_E_ARG;
}
int cldl_set_transport(cldl_t* h, cldl_allgather_fn fn, void* ctx) {
  if (!h) return CLDL_E_ARG;
  h->obj.transport = fn; h->obj.transport_ctx = ctx;
  return CLDL_OK;
}
int cldl_copy_dev(void* d_dst, const void* d_src, uint64_t bytes) {
  if (bytes == 0) return CLDL_OK;
  // a device-to-device cudaMemcpy is queued on the default stream and may return before it has run; the handles work
  // on non-blocking streams that do not wait for the default stream, so the copy is completed here
  if (cudaMemcpy(d_dst, d_src, (size_t)bytes, cudaMemcpyDeviceToDevice) != cudaSuccess) return CLDL_E_CUDA;
  return cudaStreamSynchronize(nullptr) == cudaSuccess ? CLDL_OK : CLDL_E_CUDA;
}
int cldl_shard_counts(const cldl_t* h, uint64_t* out4) {
  if (!h || !out4) return CLDL_E_ARG;
  out4[0] = h->obj.shard_count_owned[0]; out4[1] = h->obj.shard_count_owned[1];
  out4[2] = h->obj.regularize_count; out4[3] = h->obj.positive_inertia;
  return CLDL_OK;
}
void* cldl_stream(cldl_t* h) { return h ? (void*)h->obj.stream : nullptr; }
double* cldl_values_dev(cldl_t* h) { return h ? h->obj.dev.vals : nullptr; }

double cldl_time_refactor_ms(cldl_t* h, int reps) {
  if (!h || reps <= 0) return -1.0;
  LDLObject& o = h->obj;
  cudaSetDevice(o.device);
  cudaStreamSynchronize(o.stream);
  cudaEventRecord(o.ev0, o.stream);
  for (int r = 0; r < reps; r++) o.refactor_async();
  cudaEventRecord(o.ev1, o.stream);
  cudaEventSynchronize(o.ev1);
  float ms = 0;
  cudaEventElapsedTime(&ms, o.ev0, o.ev1);
  return (double)ms / reps;
}

double cldl_time_solve_ms(cldl_t* h, int reps) {
  if (!h || reps <= 0 || !h->obj.factored) return -1.0;
  LDLObject& o = h->obj;
  cudaSetDevice(o.device);
  cudaStreamSynchronize(o.stream);
  cudaEventRecord(o.ev0, o.stream);
  for (int r = 0; r < reps; r++) o.solve_async(o.d_bx + o.n, o.d_bx);
  cudaEventRecord(o.ev1, o.stream);
  cudaEventSynchronize(o.ev1);
  float ms = 0;
  cudaEventElapsedTime(&ms, o.ev0, o.ev1);
  return (double)ms / reps;
}

}  // extern "C"
