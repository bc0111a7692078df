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
// tree; every tree level is a batch of independent dense fronts.  A front's
// panel ((ns+nr) x ns, column major) lives in the compact factor storage, its
// update matrix (nr x nr) in a lifetime-managed arena.  Per level: assemble
// (original entries + children's update matrices through relative indices),
// dense LDL^T of the pivot block with the reference's sign-aware dynamic
// regularisation rule (qdldl.rs:645-651) applied pivot by pivot in elimination
// order, panel scaling, Schur update.  No atomics on floating point data:
// every sum has a fixed order, so refactor/solve are bit-reproducible run to run.
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

// Fused front kernel: one CTA per front.
template <int NT>
__global__ void __launch_bounds__(NT) k_factor_level(LDLDev d, int task_base, int smem_cap) {
  extern __shared__ double sm[];
  __shared__ double s_inv;
  __shared__ double sD[CB_MAX_PANEL];
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
  for (int b = warp; b < nr; b += nwarp)
    for (int a = b + lane; a < nr; a += 32) U[(long long)b * nr + a] = 0.0;
  __syncthreads();

  // original matrix entries (each lands in a distinct slot)
  for (long long e = d.asm_ptr[s] + tid; e < d.asm_ptr[s + 1]; e += NT)
    W[d.asm_dst[e]] = d.vals[d.asm_src[e]];
  __syncthreads();

  // extend-add of the children's update matrices, fixed child order
  for (long long ci = d.child_ptr[s]; ci < d.child_ptr[s + 1]; ci++) {
    const int c = d.child_list[ci];
    const long long crp = d.sn_rowptr[c];
    const int nrc = (int)(d.sn_rowptr[c + 1] - crp);
    const double* __restrict__ Uc = d.U + d.upd_off[c];
    const int* __restrict__ relc = d.rel + crp;
    for (int b = warp; b < nrc; b += nwarp) {
      const int rb = relc[b];
      for (int a = b + lane; a < nrc; a += 32) {
        const int ra = relc[a];
        const double v = Uc[(long long)b * nrc + a];
        if (rb < ns) W[(long long)rb * ld + ra] += v;
        else U[(long long)(rb - ns) * nr + (ra - ns)] += v;
      }
    }
    __syncthreads();
  }

  // dense LDL^T of the panel, right-looking, pivot order = elimination order
  for (int j = 0; j < ns; j++) {
    if (tid == 0) {
      double dj = W[(long long)j * ld + j];
      if (d.reg_enable) {
        const double sg = (double)d.dsigns[f + j];
        if (dj * sg < d.reg_eps) { dj = d.reg_delta * sg; atomicAdd(&d.status[ST_REGCOUNT], 1); }
      }
      if (dj == 0.0) atomicExch(&d.status[ST_ZEROPIV], 1);
      if (dj > 0.0) atomicAdd(&d.status[ST_POSINERTIA], 1);
      const double inv = 1.0 / dj;
      if (!isfinite(inv)) atomicExch(&d.status[ST_NONFINITE], 1);
      d.D[f + j] = dj;
      d.Dinv[f + j] = inv;
      W[(long long)j * ld + j] = dj;
      s_inv = inv;
      sD[j] = dj;
    }
    __syncthreads();
    const double inv = s_inv;
    const double* __restrict__ cj = W + (long long)j * ld;
    for (int k = j + 1 + warp; k < ns; k += nwarp) {
      const double wk = cj[k] * inv;
      double* __restrict__ ck = W + (long long)k * ld;
      for (int i = k + lane; i < ld; i += 32) ck[i] -= cj[i] * wk;
    }
    __syncthreads();
    double* cjw = W + (long long)j * ld;
    for (int i = j + 1 + tid; i < ld; i += NT) cjw[i] *= inv;
  }
  __syncthreads();

  // Schur update of the lower triangle of U
  for (int b = warp; b < nr; b += nwarp) {
    for (int a = b + lane; a < nr; a += 32) {
      double acc = 0.0;
      for (int k = 0; k < ns; k++) {
        const double* __restrict__ ck = W + (long long)k * ld + ns;
        acc += ck[a] * (ck[b] * sD[k]);
      }
      U[(long long)b * nr + a] -= acc;
    }
  }
  if (use_sm) {
    for (long long i = tid; i < psz; i += NT) P[i] = W[i];
  }
}

// Single-column leaves (no children: tree level 0; on KKT matrices these are the constraint rows eliminated first,
// 5e5 of them on config C4): ONE THREAD per front instead of one CTA.  Same arithmetic as the fused kernel above does
// for such a front: d = a_jj (sign test, regularisation), l = a_:j / d, U = 0 - l (l d)^T on the lower triangle.
// The inertia / regularisation counters are aggregated per warp before they touch global memory.
__global__ void __launch_bounds__(256) k_factor_leaf1(LDLDev d, int task_base, int count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool on = i < count;
  int pos = 0, reg = 0;
  if (on) {
    const int s = d.level_tasks[task_base + i];
    const int f = d.sn_first[s];
    const long long rp = d.sn_rowptr[s];
    const int nr = (int)(d.sn_rowptr[s + 1] - rp);
    const int ld = 1 + nr;
    double* __restrict__ P = d.L + d.panel_off[s];
    double* __restrict__ U = d.U + d.upd_off[s];
    for (int a = 0; a < ld; a++) P[a] = 0.0;
    for (long long e = d.asm_ptr[s]; e < d.asm_ptr[s + 1]; e++) P[d.asm_dst[e]] = d.vals[d.asm_src[e]];
    double dj = P[0];
    if (d.reg_enable) {
      const double sg = (double)d.dsigns[f];
      if (dj * sg < d.reg_eps) { dj = d.reg_delta * sg; reg = 1; }
    }
    if (dj == 0.0) atomicExch(&d.status[ST_ZEROPIV], 1);
    pos = dj > 0.0 ? 1 : 0;
    const double inv = 1.0 / dj;
    if (!isfinite(inv)) atomicExch(&d.status[ST_NONFINITE], 1);
    d.D[f] = dj;
    d.Dinv[f] = inv;
    P[0] = dj;
    for (int a = 1; a < ld; a++) P[a] *= inv;
    for (int b = 0; b < nr; b++) {
      const double t = P[1 + b] * dj;
      for (int a = b; a < nr; a++) {
        double acc = 0.0;
        acc += P[1 + a] * t;
        U[(long long)b * nr + a] = 0.0 - acc;
      }
    }
  }
  const unsigned mp = __ballot_sync(0xffffffffu, pos != 0), mr = __ballot_sync(0xffffffffu, reg != 0);
  if ((threadIdx.x & 31) == 0) {
    if (mp) atomicAdd(&d.status[ST_POSINERTIA], __popc(mp));
    if (mr) atomicAdd(&d.status[ST_REGCOUNT], __popc(mr));
  }
}

// ------------------------------------------------------------------------
// Big fronts: two kernels per level.
//   k_panel_big   : one CTA per front.  Assembles the ns panel columns (original
//                   entries + the children's update-matrix columns that fall inside
//                   the pivot block), factors the ns x ns pivot block in shared
//                   memory (same pivot-by-pivot regularisation rule), then solves
//                   the nr rows below it (one thread per row, rows independent).
//   k_update_tiles: one CTA per 64x64 tile of the front's update matrix:
//                   U_tile = sum_children extend-add  -  L21_I * D * L21_J^T
//                   with 4x4 register tiles; the extend-add is fused, so U is
//                   written exactly once and never zero-filled.
// ------------------------------------------------------------------------
#define PB_NT 256
#define TS 64
#define KC 32   /* pivots staged per chunk by k_update_tiles */

__device__ __forceinline__ int lower_bound_dev(const int* __restrict__ a, int n, int key) {
  int lo = 0, hi = n;
  while (lo < hi) { int mid = (lo + hi) >> 1; if (a[mid] < key) lo = mid + 1; else hi = mid; }
  return lo;
}

// Ordered compaction of the children of front s that satisfy `pred`: every thread
// evaluates up to one child per round; the surviving child ids are appended to
// s_list in child_list order (so sums keep a fixed order).  Returns the count.
template <class Pred>
__device__ __forceinline__ int compact_children(const LDLDev& d, int s, int* s_list, int cap, int* s_wcnt, Pred pred) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
  const long long c0 = d.child_ptr[s], c1 = d.child_ptr[s + 1];
  int total = 0;
  for (long long base = c0; base < c1; base += blockDim.x) {
    const long long ci = base + tid;
    int c = -1;
    bool ok = false;
    if (ci < c1) { c = d.child_list[ci]; ok = pred(c); }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_wcnt[warp] = __popc(bal);
    __syncthreads();
    int off = total;
    for (int w = 0; w < warp; w++) off += s_wcnt[w];
    int add = 0;
    for (int w = 0; w < nwarp; w++) add += s_wcnt[w];
    if (ok) {
      const int p = off + __popc(bal & ((1u << lane) - 1u));
      if (p < cap) s_list[p] = c;
    }
    total += add;
    __syncthreads();
  }
  return total;
}

// Adds U-arena values into `dst_base` through a (src,dst) entry list sorted by dst.  Every thread takes a
// contiguous slice; slice borders are moved forward to the next change of dst so that one destination is
// only ever touched by one thread, in list order (deterministic, no atomics, no barriers).
__device__ __forceinline__ void apply_sorted_entries(double* __restrict__ dst_base, const double* __restrict__ U,
                                                     const int* __restrict__ esrc, const int* __restrict__ edst,
                                                     int e0, int e1, int nthreads) {
  const int cnt = e1 - e0;
  if (cnt <= 0) return;
  const int per = (cnt + nthreads - 1) / nthreads;
  int b = e0 + threadIdx.x * per, e = min(e1, b + per);
  if (b >= e1) return;
  if (b > e0) { while (b < e1 && edst[b] == edst[b - 1]) b++; }
  if (e < e1) { while (e < e1 && edst[e] == edst[e - 1]) e++; }
  int i = b;
  while (i < e) {
    const int dd = edst[i];
    double acc = 0.0;
    while (i < e && edst[i] == dd) { acc += U[esrc[i]]; i++; }
    dst_base[dd] += acc;
  }
}

#define CB_CHILD_CAP 1024

__global__ void __launch_bounds__(PB_NT) k_panel_big(LDLDev d, const int* __restrict__ tasks, int task_off) {
  __shared__ __align__(16) double sA[CB_PB_MAXNS * CB_PB_LD];   // pivot block, column major, padded
  __shared__ double sDinv[CB_PB_MAXNS], sDval[CB_PB_MAXNS], sSign[CB_PB_MAXNS];
  __shared__ double s_inv;
  __shared__ int s_list[CB_CHILD_CAP];
  __shared__ int s_wcnt[PB_NT / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = PB_NT >> 5;
  const int s = tasks[blockIdx.x];
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr;
  double* __restrict__ P = d.L + d.panel_off[s];
  const long long psz = (long long)ld * ns;

  for (long long i = tid; i < psz; i += PB_NT) P[i] = 0.0;
  if (tid < ns) sSign[tid] = (double)d.dsigns[f + tid];
  const int ncontrib = compact_children(d, s, s_list, CB_CHILD_CAP, s_wcnt, [&](int c) { return d.child_nb[c] > 0 && !d.child_small[c]; });
  __syncthreads();
  for (long long e = d.asm_ptr[s] + tid; e < d.asm_ptr[s + 1]; e += PB_NT) P[d.asm_dst[e]] = d.vals[d.asm_src[e]];
  __syncthreads();
  const bool overflow = ncontrib > CB_CHILD_CAP;
  const int nloop = overflow ? (int)(d.child_ptr[s + 1] - d.child_ptr[s]) : ncontrib;
  for (int q = 0; q < nloop; q++) {
    const int c = overflow ? d.child_list[d.child_ptr[s] + q] : s_list[q];
    const int nb = d.child_nb[c];   // child columns landing inside the pivot block (host precomputed)
    if (nb == 0 || d.child_small[c]) continue;
    const long long crp = d.sn_rowptr[c];
    const int nrc = (int)(d.sn_rowptr[c + 1] - crp);
    const double* __restrict__ Uc = d.U + d.upd_off[c];
    const int* __restrict__ relc = d.rel + crp;
    for (int b = warp; b < nb; b += nwarp) {
      double* __restrict__ col = P + (long long)relc[b] * ld;
      const double* __restrict__ ucol = Uc + (long long)b * nrc;
      // destinations inside one child column are distinct: batch the read-modify-writes so that
      // 8 independent global round trips are in flight per lane
      int a = b + lane;
      for (; a + 7 * 32 < nrc; a += 8 * 32) {
        int r[8];
        double u[8], pv[8];
#pragma unroll
        for (int q = 0; q < 8; q++) { r[q] = relc[a + q * 32]; u[q] = ucol[a + q * 32]; }
#pragma unroll
        for (int q = 0; q < 8; q++) pv[q] = col[r[q]];
        asm volatile("" ::: "memory");
#pragma unroll
        for (int q = 0; q < 8; q++) col[r[q]] = pv[q] + u[q];
      }
      for (; a < nrc; a += 32) col[relc[a]] += ucol[a];
    }
    __syncthreads();
  }
  // all small children at once (sorted entry list, conflict free)
  apply_sorted_entries(P, d.U, d.sc_panel_src, d.sc_panel_dst, d.sc_panel_ptr[blockIdx.x + task_off],
                       d.sc_panel_ptr[blockIdx.x + task_off + 1], PB_NT);
  __syncthreads();
  // pivot block -> shared
  for (int idx = tid; idx < ns * ns; idx += PB_NT) {
    const int j = idx / ns, i = idx - j * ns;
    sA[j * CB_PB_LD + i] = P[(long long)j * ld + i];
  }
  __syncthreads();
  int c_reg = 0, c_pos = 0, c_zero = 0, c_nonf = 0;   // thread 0 only
  for (int j = 0; j < ns; j++) {
    if (tid == 0) {
      double dj = sA[j * CB_PB_LD + j];
      if (d.reg_enable) {
        const double sg = sSign[j];
        if (dj * sg < d.reg_eps) { dj = d.reg_delta * sg; c_reg++; }
      }
      if (dj == 0.0) c_zero = 1;
      if (dj > 0.0) c_pos++;
      const double inv = 1.0 / dj;
      if (!isfinite(inv)) c_nonf = 1;
      sDval[j] = dj;
      sA[j * CB_PB_LD + j] = dj;
      sDinv[j] = inv;
      s_inv = inv;
    }
    __syncthreads();
    const double inv = s_inv;
    const double* cj = sA + j * CB_PB_LD;
    for (int k = j + 1 + warp; k < ns; k += nwarp) {
      const double wk = cj[k] * inv;
      double* ck = sA + k * CB_PB_LD;
      for (int i = k + lane; i < ns; i += 32) ck[i] -= cj[i] * wk;
    }
    __syncthreads();
    for (int i = j + 1 + tid; i < ns; i += PB_NT) sA[j * CB_PB_LD + i] *= inv;
    // column j is final; the next pivot only reads column j+1
  }
  __syncthreads();
  if (tid == 0) {
    if (c_reg) atomicAdd(&d.status[ST_REGCOUNT], c_reg);
    if (c_pos) atomicAdd(&d.status[ST_POSINERTIA], c_pos);
    if (c_zero) atomicExch(&d.status[ST_ZEROPIV], 1);
    if (c_nonf) atomicExch(&d.status[ST_NONFINITE], 1);
  }
  if (tid < ns) { d.D[f + tid] = sDval[tid]; d.Dinv[f + tid] = sDinv[tid]; }
  // write the unit-lower pivot block back
  for (int idx = tid; idx < ns * ns; idx += PB_NT) {
    const int j = idx / ns, i = idx - j * ns;
    if (i >= j) P[(long long)j * ld + i] = sA[j * CB_PB_LD + i];
  }
  // rows below:  W L11^T = F21,  L21 = W D^-1.  One thread per row, 16 columns at a time in
  // registers; W of earlier column blocks is re-read from the panel (L21 * D), coalesced.
  constexpr int JB = 16;
  for (int r0 = 0; r0 < nr; r0 += PB_NT) {
    const int r = r0 + tid;
    if (r >= nr) continue;
    double* __restrict__ prow = P + ns + r;
    for (int jb = 0; jb < ns; jb += JB) {
      const int nj = min(JB, ns - jb);
      double t[JB];
#pragma unroll
      for (int jj = 0; jj < JB; jj++) t[jj] = jj < nj ? prow[(long long)(jb + jj) * ld] : 0.0;
      for (int kb = 0; kb < jb; kb += JB) {
        double wv[JB];
#pragma unroll
        for (int kk = 0; kk < JB; kk++) wv[kk] = prow[(long long)(kb + kk) * ld];   // 16 loads in flight
#pragma unroll
        for (int kk = 0; kk < JB; kk++) {
          const double wk = wv[kk] * sDval[kb + kk];
          const double2* lk2 = reinterpret_cast<const double2*>(sA + (kb + kk) * CB_PB_LD + jb);   // L11[jb+jj][k]
#pragma unroll
          for (int j2 = 0; j2 < JB / 2; j2++) {
            const double2 l = lk2[j2];
            t[2 * j2] -= wk * l.x;
            t[2 * j2 + 1] -= wk * l.y;
          }
        }
      }
#pragma unroll
      for (int jj = 0; jj < JB; jj++) {
        if (jj < nj) {
          const double* lk = sA + (jb + jj) * CB_PB_LD + jb;   // column jb+jj: rows jb+jj+1.. hold L11[.][jb+jj]
#pragma unroll
          for (int j2 = jj + 1; j2 < JB; j2++) t[j2] -= t[jj] * lk[j2];
        }
      }
#pragma unroll
      for (int jj = 0; jj < JB; jj++) if (jj < nj) prow[(long long)(jb + jj) * ld] = t[jj] * sDinv[jb + jj];
    }
  }
}

// tile descriptor: x = task, y = tile row, z = tile column (ti >= tj)
__global__ void __launch_bounds__(256) k_update_tiles(LDLDev d, const int4* __restrict__ tiles, int tile_off) {
  extern __shared__ double sm[];
  double* sAt = sm;                 // [KC][TS]   L21 rows of tile-row I   (KC pivots at a time)
  double* sBt = sm + KC * TS;        // [KC][TS]   L21 rows of tile-row J scaled by D
  double* sC = sm + 2 * KC * TS;     // [TS][TS+1] children's contributions
  const int4 td = tiles[blockIdx.x];
  const int s = td.x, ti = td.y, tj = td.z;
  const int tid = threadIdx.x;
  const int f = d.sn_first[s];
  const int ns = d.sn_first[s + 1] - f;
  const long long rp = d.sn_rowptr[s];
  const int nr = (int)(d.sn_rowptr[s + 1] - rp);
  const int ld = ns + nr;
  const double* __restrict__ P = d.L + d.panel_off[s];
  double* __restrict__ U = d.U + d.upd_off[s];
  const int i0 = ti * TS, j0 = tj * TS;
  const int ni = min(TS, nr - i0), nj = min(TS, nr - j0);

  for (int idx = tid; idx < TS * (TS + 1); idx += 256) sC[idx] = 0.0;
  __syncthreads();
  // extend-add (fixed child order; distinct destinations inside one child).  Only children whose
  // rows can reach both tile rows are visited.
  __shared__ int s_list[CB_CHILD_CAP];
  __shared__ int s_wcnt[8];
  const int ncontrib = compact_children(d, s, s_list, CB_CHILD_CAP, s_wcnt, [&](int c) {
    const int2 tr = d.child_trange[c];
    return !(ti < tr.x || ti > tr.y || tj < tr.x || tj > tr.y) && !d.child_small[c];
  });
  const bool overflow = ncontrib > CB_CHILD_CAP;
  const int nloop = overflow ? (int)(d.child_ptr[s + 1] - d.child_ptr[s]) : ncontrib;
  for (int q = 0; q < nloop; q++) {
    const int c = overflow ? d.child_list[d.child_ptr[s] + q] : s_list[q];
    if (overflow) {
      const int2 tr = d.child_trange[c];
      if (ti < tr.x || ti > tr.y || tj < tr.x || tj > tr.y || d.child_small[c]) continue;
    }
    const long long crp = d.sn_rowptr[c];
    const int nrc = (int)(d.sn_rowptr[c + 1] - crp);
    const int* __restrict__ relc = d.rel + crp;
    // first child row falling into tile row t is tp[t - tlo] (host precomputed, uniform loads)
    const int* __restrict__ tp = d.child_tptr + d.child_tptr_off[c];
    const int tlo = d.child_trange[c].x;
    const int a0 = tp[ti - tlo], a1 = tp[ti - tlo + 1], b0 = tp[tj - tlo], b1 = tp[tj - tlo + 1];
    const int na = a1 - a0, nb = b1 - b0;
    if (na > 0 && nb > 0) {
      const double* __restrict__ Uc = d.U + d.upd_off[c];
      for (int idx = tid; idx < na * nb; idx += 256) {
        const int bb = idx / na, aa = idx - bb * na;
        const int a = a0 + aa, b = b0 + bb;
        if (a >= b) sC[(relc[a] - ns - i0) * (TS + 1) + (relc[b] - ns - j0)] += Uc[(long long)b * nrc + a];
      }
    }
    __syncthreads();
  }
  // all small children of this tile at once
  apply_sorted_entries(sC, d.U, d.sc_tile_src, d.sc_tile_dst, d.sc_tile_ptr[blockIdx.x + tile_off],
                       d.sc_tile_ptr[blockIdx.x + tile_off + 1], 256);
  // 4x4 register tile per thread
  const int tx = tid & 15, ty = tid >> 4;
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.0;
  for (int k0 = 0; k0 < ns; k0 += KC) {
    const int kc = min(KC, ns - k0);
    __syncthreads();   // previous chunk fully consumed
    for (int idx = tid; idx < kc * TS; idx += 256) {
      const int k = idx / TS, r = idx - k * TS;
      const long long col = (long long)(k0 + k) * ld + ns;
      sAt[idx] = (r < ni) ? P[col + i0 + r] : 0.0;
      sBt[idx] = (r < nj) ? P[col + j0 + r] * d.D[f + k0 + k] : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < kc; k++) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; i++) { a[i] = sAt[k * TS + tx + 16 * i]; b[i] = sBt[k * TS + ty + 16 * i]; }
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] += a[i] * b[j];
    }
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int r = tx + 16 * i;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int c = ty + 16 * j;
      if (r < ni && c < nj && (i0 + r >= j0 + c))
        U[(long long)(j0 + c) * nr + (i0 + r)] = sC[r * (TS + 1) + c] - acc[i][j];
    }
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
// No floating-point atomics: results are bit-identical to the level-synchronous kernels.
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
// the update-matrix arena is recycled along the schedule).  Same arithmetic, same summation orders as the
// level-synchronous kernels: results are bit-identical.
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
  if (use_sm) for (long long i = tid; i < psz; i += DF_NT) P[i] = W[i];
}

// ---- task / child records built by the host (LDLObject::init) ----
// DFTask   (16 ints): kind, s, a, b, ns, nr, f, d0, d1, e0, e1, -, panel_off (2), upd_off (2)
// DFChild  (12 ints): U offset (2), rel offset (2), nrc, a0, a1, b0, b1, -, -, -
//   rows a0..a1 and columns b0..b1 (child-local indices) of the child's update matrix land in this task's
//   target (pivot block / row block / tile); only a >= b is stored.
struct DFChildRec { long long uoff, relp; int nrc, a0, a1, b0, b1, p0, p1, p2; };
#define DF_DCAP 32          /* child records staged per round */
#define DF_RB 128           /* rows per R task */

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
  if (ch.p0 == 3) {
    // rows and columns of the block are contiguous in the target (the previous panel of the same separator,
    // dense children): no index loads, warp-wide coalesced reads down the columns this warp owns
    const int r0 = ch.p1 - rowoff - ch.a0, c0 = ch.p2 - coloff - ch.b0;   // target row of a: r0 + a, column of b: c0 + b
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
    for (int i = threadIdx.x; i < cnt * 12; i += DF_NT) s_desc[i] = q.desc[(size_t)base * 12 + i];
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
__device__ void dff_diag(const LDLDev& d, const DFFactor& q, const int* tk, double* sm, int* s_desc, int* s_ed, double* s_ev) {
  double* sA = sm;                                     // [64][CB_PB_LD]
  double* sSign = sm + CB_PB_MAXNS * CB_PB_LD;         // [64]
  double* colbuf = sSign + CB_PB_MAXNS;                // [2][72]: column, then dj, 1/dj
  const int tid = threadIdx.x;
  const int s = tk[1], ns = tk[4], nr = tk[5], f = tk[6];
  const int ld = ns + nr;
  const long long poff = *reinterpret_cast<const long long*>(tk + 12);
  double* P = d.L + poff;
  DFEnt pe;
  df_ent_issue(d.U, d.sc_panel_src, d.sc_panel_dst, tk[9], tk[10], pe);
  for (int i = tid; i < CB_PB_MAXNS * CB_PB_LD; i += DF_NT) sA[i] = 0.0;
  if (tid < CB_PB_MAXNS) sSign[tid] = tid < ns ? (double)d.dsigns[f + tid] : 1.0;
  __syncthreads();
  df_scatter_asm(d, s, [&](long long dst, double v) {
    const int col = (int)(dst / ld), row = (int)(dst - (long long)col * ld);
    if (row < ns) sA[col * CB_PB_LD + row] = v;
  });
  __syncthreads();
  df_children(q, tk[7], tk[8], s_desc, [&](const DFChildRec& ch) { df_add_child<2>(d, ch, sA, 0, 1, 0, CB_PB_LD); });
  df_ent_apply(sA, d.U, d.sc_panel_src, d.sc_panel_dst, tk[9], tk[10], pe, s_ed, s_ev,
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
__device__ void dff_rows(const LDLDev& d, const DFFactor& q, const int* tk, double* sm, int* s_desc, int* s_ed, double* s_ev) {
  double* sA = sm;                                     // [64][CB_PB_LD]  L11 (unit lower, column major)
  double* sDval = sm + CB_PB_MAXNS * CB_PB_LD;
  double* sDinv = sDval + CB_PB_MAXNS;
  double* sR = sDinv + CB_PB_MAXNS;                    // [64][DF_RB]  the rows, column major
  const int tid = threadIdx.x;
  const int s = tk[1], blk = tk[2], ns = tk[4], nr = tk[5], f = tk[6];
  const int ld = ns + nr;
  double* P = d.L + *reinterpret_cast<const long long*>(tk + 12);
  const int r0 = blk * DF_RB, r1 = min(nr, r0 + DF_RB);
  const int g0 = ns + r0, g1 = ns + r1;
  DFEnt pe;
  df_ent_issue(d.U, d.sc_panel_src, d.sc_panel_dst, tk[9], tk[10], pe);
  for (int i = tid; i < CB_PB_MAXNS * DF_RB; i += DF_NT) sR[i] = 0.0;
  __syncthreads();
  df_scatter_asm(d, s, [&](long long dst, double v) {
    const int col = (int)(dst / ld), row = (int)(dst - (long long)col * ld);
    if (row >= g0 && row < g1) sR[col * DF_RB + row - g0] = v;
  });
  __syncthreads();
  df_children(q, tk[7], tk[8], s_desc, [&](const DFChildRec& ch) { df_add_child<4>(d, ch, sR, g0, 1, 0, DF_RB); });
  df_ent_apply(sR, d.U, d.sc_panel_src, d.sc_panel_dst, tk[9], tk[10], pe, s_ed, s_ev,
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

// ---- T: one 64x64 tile of the update matrix ----
__device__ void dff_tile(const LDLDev& d, const DFFactor& q, const int* tk, double* sm, int* s_desc, int* s_ed, double* s_ev) {
  double* sAt = sm;                      // [ns][TS]  L21 rows of tile-row I
  double* sBt = sm + TS * TS;            // [ns][TS]  L21 rows of tile-row J, scaled by D
  double* sC = sm + 2 * TS * TS;         // [TS][TS+1] children's contributions
  double* sD = sC + TS * (TS + 1);       // [ns]
  const int tid = threadIdx.x;
  const int ti = tk[2], tj = tk[3], ns = tk[4], nr = tk[5], f = tk[6];
  const int ld = ns + nr;
  const double* P = d.L + *reinterpret_cast<const long long*>(tk + 12);
  double* U = d.U + *reinterpret_cast<const long long*>(tk + 14);
  const int i0 = ti * TS, j0 = tj * TS;
  const int ni = min(TS, nr - i0), nj = min(TS, nr - j0);
  // every independent load of the task is issued up front (sorted entries, child records, the whole K range
  // of both panels) so that the task pays ~3 dependent memory round trips instead of one per stage
  DFEnt pe;
  df_ent_issue(d.U, d.sc_tile_src, d.sc_tile_dst, tk[9], tk[10], pe);
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
  const int ndense = tk[11];
  for (int kd = 0; kd < ndense; kd++) {
    const int* rec = q.desc + (size_t)(tk[7] + kd) * 12;
    const long long uoff = *reinterpret_cast<const long long*>(rec);
    const int nrc = rec[4], a0 = rec[5], a1 = rec[6], b0 = rec[7], b1 = rec[8];
    const int ra = a0 - (rec[10] - (ns + i0)), rb = b0 - (rec[11] - (ns + j0));   // child index = tile index + ra / rb
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
  const bool use_sc = (tk[8] - tk[7] > ndense) || (tk[10] > tk[9]);
  if (use_sc) {
    for (int idx = tid; idx < TS * (TS + 1); idx += DF_NT) sC[idx] = 0.0;
    __syncthreads();
    DF_STAMP(q, 7);
    df_children(q, tk[7] + ndense, tk[8], s_desc, [&](const DFChildRec& ch) { df_add_child<2>(d, ch, sC, ns + i0, TS + 1, ns + j0, 1); });
    DF_STAMP(q, 8);
    df_ent_apply(sC, d.U, d.sc_tile_src, d.sc_tile_dst, tk[9], tk[10], pe, s_ed, s_ev, [&](int dd) -> long long { return dd; });
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
  __shared__ __align__(16) int s_desc[DF_DCAP * 12];
  __shared__ __align__(16) int s_task[16];
  __shared__ int s_ed[DF_ENT_FAST];
  __shared__ double s_ev[DF_ENT_FAST];
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
    const int kind = s_task[0], s = s_task[1];
    if (kind == 0) {
      if (tid == 0) { df_wait_zero(q.pend + s); __threadfence(); if (q.trace) q.trace[10 * (size_t)qi + 1] = df_gtime(); }
      __syncthreads();
      dff_small(d, s, dfsm, nullptr);
      __syncthreads();
      if (tid == 0) { __threadfence(); df_front_complete(q, s); }
    } else if (kind == 1) {
      if (tid == 0) { df_wait_zero(q.pend + s); __threadfence(); if (q.trace) q.trace[10 * (size_t)qi + 1] = df_gtime(); }
      __syncthreads();
      dff_diag(d, q, s_task, dfsm, s_desc, s_ed, s_ev);
      __syncthreads();
      if (tid == 0) { __threadfence(); atomicExch(q.diag_done + s, 1); }
    } else if (kind == 2) {
      // the row task needs the children's data as well as the pivot block: it waits on the children counter
      // first, assembles, and only then waits for the D task of the front
      if (tid == 0) { df_wait_zero(q.pend + s); __threadfence(); if (q.trace) q.trace[10 * (size_t)qi + 1] = df_gtime(); }
      __syncthreads();
      dff_rows(d, q, s_task, dfsm, s_desc, s_ed, s_ev);
      __syncthreads();
      if (tid == 0) { __threadfence(); atomicSub(q.rows_left + s, 1); }
    } else {
      if (tid == 0) { df_wait_zero(q.rows_left + s); __threadfence(); if (q.trace) q.trace[10 * (size_t)qi + 1] = df_gtime(); }
      __syncthreads();
      dff_tile(d, q, s_task, dfsm, s_desc, s_ed, s_ev);
      __syncthreads();
      if (tid == 0) {
        __threadfence();
        if (atomicSub(q.tiles_left + s, 1) == 1) df_front_complete(q, s);
      }
    }
  }
}

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

template <class T>
static int upload(T** dptr, const std::vector<T>& v) {
  size_t bytes = (v.size() ? v.size() : 1) * sizeof(T);
  CK(cudaMalloc((void**)dptr, bytes));
  if (!v.empty()) CK(cudaMemcpy(*dptr, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}

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
  int rc = analyse(n, Ap, Ai, perm_in, so, S);
  cb_tmark("ldl: ordering + symbolic");
  if (rc == -2) return CLDL_E_EMPTY_COLUMN;
  if (rc == -3) return CLDL_E_NOT_TRIU;
  if (rc == -5) return CLDL_E_BAD_PERM;
  if (rc) return CLDL_E_ARG;
  shard_nranks = o.shard_nranks > 1 ? o.shard_nranks : 1;
  shard_rank = o.shard_rank;
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

  CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  if (std::getenv("CB_LEAF_STREAMS") == nullptr || std::atoi(std::getenv("CB_LEAF_STREAMS")) != 0) {
    CK(cudaStreamCreateWithFlags(&stream_a, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&stream_b, cudaStreamNonBlocking));
    for (auto& e : ev_leaf) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  CK(cudaEventCreate(&ev0));
  CK(cudaEventCreate(&ev1));
  CK(cudaMallocHost((void**)&h_status, ST_COUNT * sizeof(int)));

  int* tmp_i = nullptr;
  long long* tmp_l = nullptr;
  auto to_ll = [](const std::vector<int64_t>& v) { return std::vector<long long>(v.begin(), v.end()); };
  if ((rc = upload(&tmp_i, S.sn_first))) return rc; dev.sn_first = tmp_i;
  if ((rc = upload(&tmp_l, to_ll(S.sn_rowptr)))) return rc; dev.sn_rowptr = tmp_l;
  if ((rc = upload(&tmp_i, S.sn_rows))) return rc; dev.sn_rows = tmp_i;
  if ((rc = upload(&tmp_l, to_ll(S.child_ptr)))) return rc; dev.child_ptr = tmp_l;
  if ((rc = upload(&tmp_i, S.child_list))) return rc; dev.child_list = tmp_i;
  if ((rc = upload(&tmp_i, S.rel))) return rc; dev.rel = tmp_i;
  if ((rc = upload(&tmp_l, to_ll(S.panel_off)))) return rc; dev.panel_off = tmp_l;
  if ((rc = upload(&tmp_l, to_ll(S.upd_off)))) return rc; dev.upd_off = tmp_l;
  if ((rc = upload(&tmp_l, to_ll(S.asm_ptr)))) return rc; dev.asm_ptr = tmp_l;
  if ((rc = upload(&tmp_i, S.asm_src))) return rc; dev.asm_src = tmp_i;
  if ((rc = upload(&tmp_l, to_ll(S.asm_dst)))) return rc; dev.asm_dst = tmp_l;
  if ((rc = upload(&tmp_i, S.level_tasks))) return rc; dev.level_tasks = tmp_i;
  if ((rc = upload(&tmp_i, S.perm))) return rc; dev.perm = tmp_i;
  {
    std::vector<signed char> ds(n);
    for (int k = 0; k < n; k++) ds[k] = dsigns ? (signed char)dsigns[S.perm[k]] : (signed char)1;
    signed char* t = nullptr;
    if ((rc = upload(&t, ds))) return rc;
    dev.dsigns = t;
  }
  nnzA = Ap[n];
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
  // per-child constants for the big-front kernels and the per-destination gather lists for the solves
  std::vector<int> h_child_nb(S.nsup, 0);
  // (runs on a host thread next to the launch plan and the small-child lists below; it only reads the symbolic
  // structure and writes its own device arrays)
  auto build_child_consts = [&]() -> int {
    int rc = 0;
    if (cudaSetDevice(device) != cudaSuccess) return CLDL_E_CUDA;
    std::vector<int>& child_nb = h_child_nb;
    std::vector<int2> child_tr(S.nsup, make_int2(1, 0));
    std::vector<int> gptr((size_t)n + S.sn_rows.size() + 1, 0);
    for (int c = 0; c < S.nsup; c++) {
      const int p = S.sn_parent[c];
      if (p < 0) continue;
      const int pns = S.sn_first[p + 1] - S.sn_first[p];
      const int64_t pbase = (int64_t)S.sn_first[p] + S.sn_rowptr[p];
      const int64_t b0 = S.sn_rowptr[c], e0 = S.sn_rowptr[c + 1];
      int nb = 0;
      for (int64_t t = b0; t < e0; t++) { if (S.rel[t] < pns) nb++; gptr[pbase + S.rel[t] + 1]++; }
      child_nb[c] = nb;
      if (b0 + nb < e0) child_tr[c] = make_int2((S.rel[b0 + nb] - pns) / TS, (S.rel[e0 - 1] - pns) / TS);
    }
    for (size_t i = 0; i + 1 < gptr.size(); i++) gptr[i + 1] += gptr[i];
    std::vector<int> gsrc(S.sn_rows.size() ? S.sn_rows.size() : 1, 0), pos(gptr.begin(), gptr.end() - 1);
    // children in child_list order so that every destination sums in a fixed, reproducible order
    for (int p = 0; p < S.nsup; p++) {
      const int64_t pbase = (int64_t)S.sn_first[p] + S.sn_rowptr[p];
      for (int64_t ci = S.child_ptr[p]; ci < S.child_ptr[p + 1]; ci++) {
        const int c = S.child_list[ci];
        for (int64_t t = S.sn_rowptr[c]; t < S.sn_rowptr[c + 1]; t++) gsrc[pos[pbase + S.rel[t]]++] = (int)t;
      }
    }
    std::vector<int> tptr_off(S.nsup + 1, 0), tptr;
    for (int c = 0; c < S.nsup; c++) {
      tptr_off[c] = (int)tptr.size();
      const int p = S.sn_parent[c];
      if (p < 0 || child_tr[c].x > child_tr[c].y) continue;
      const int pns = S.sn_first[p + 1] - S.sn_first[p];
      const int64_t b0 = S.sn_rowptr[c], e0 = S.sn_rowptr[c + 1];
      int64_t t = b0 + child_nb[c];
      for (int tile = child_tr[c].x; tile <= child_tr[c].y + 1; tile++) {
        while (t < e0 && S.rel[t] < pns + tile * TS) t++;
        tptr.push_back((int)(t - b0));
      }
    }
    tptr_off[S.nsup] = (int)tptr.size();
    int* t1 = nullptr;
    if ((rc = upload(&t1, tptr_off))) return rc; dev.child_tptr_off = t1;
    if ((rc = upload(&t1, tptr))) return rc; dev.child_tptr = t1;
    if ((rc = upload(&t1, child_nb))) return rc; dev.child_nb = t1;
    if ((rc = upload(&t1, gptr))) return rc; dev.gat_ptr = t1;
    if ((rc = upload(&t1, gsrc))) return rc; dev.gat_src = t1;
    int2* t2 = nullptr;
    CK(cudaMalloc((void**)&t2, (size_t)(S.nsup ? S.nsup : 1) * sizeof(int2)));
    CK(cudaMemcpy(t2, child_tr.data(), (size_t)S.nsup * sizeof(int2), cudaMemcpyHostToDevice));
    dev.child_trange = t2;
      return rc;
  };
  int rc_child = 0;
  std::thread th_child([&]() { rc_child = build_child_consts(); });
  struct ThJoin { std::thread* t; ~ThJoin() { if (t->joinable()) t->join(); } } th_child_guard{&th_child};
  cb_tmark("ldl: child consts + gather lists");
  // per-level launch plan.  Small fronts: one fused CTA each, grouped by the shared-memory class of
  // their panel.  Big fronts (nr >= CB_BIG_NR): panel kernel + tiled update kernel.
  int max_optin = 0;
  CK(cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  const int cap_big = (max_optin - 2048) / 8;  // doubles
  CK(cudaFuncSetAttribute(k_factor_level<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap_big * 8));
  const size_t smem_panel = 0;   // static shared memory only
  const size_t smem_tiles = (size_t)(2 * KC * TS + TS * (TS + 1)) * 8;
  CK(cudaFuncSetAttribute(k_update_tiles, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tiles));
  const long long classes[3] = {1024, 5632, cap_big};  // 8 KB, 44 KB, ~225 KB panels
  plan.clear();
  const bool leaf1_kernel = std::getenv("CB_FACTOR_LEAF1") == nullptr || std::atoi(std::getenv("CB_FACTOR_LEAF1")) != 0;
  std::vector<int> big_tasks;
  std::vector<int4> tiles;
  for (int l = 0; l < S.nlevels; l++) {
    int b = S.level_ptr[l], e = S.level_ptr[l + 1];
    std::vector<int> order[4], order1;
    const size_t big0 = big_tasks.size(), tile0 = tiles.size();
    std::vector<int> not_mine;       // sharded: fronts of other ranks are parked at the end of the level's range
    for (int t = b; t < e; t++) {
      const int s = S.level_tasks[t];
      const long long ns = S.sn_first[s + 1] - S.sn_first[s];
      const long long nr = S.sn_rowptr[s + 1] - S.sn_rowptr[s];
      if (!mine(s) && !(nr >= CB_BIG_NR && ns <= CB_PB_MAXNS)) { not_mine.push_back(s); continue; }
      if (nr >= CB_BIG_NR && ns <= CB_PB_MAXNS) {
        big_tasks.push_back(s);
        const int nt = (int)((nr + TS - 1) / TS);
        for (int ti = 0; ti < nt; ti++)
          for (int tj = 0; tj <= ti; tj++) tiles.push_back(make_int4(s, ti, tj, 0));
        continue;
      }
      if (l == 0 && ns == 1 && leaf1_kernel) { order1.push_back(s); continue; }
      const long long p = (ns + nr) * ns;
      int c = p <= classes[0] ? 0 : p <= classes[1] ? 1 : p <= classes[2] ? 2 : 3;
      order[c].push_back(s);
    }
    int pos = b;
    if (!order1.empty()) {      // single-column leaves: one thread each (k_factor_leaf1)
      LaunchSeg seg;
      seg.kind = 3; seg.level = l; seg.base = pos; seg.count = (int)order1.size(); seg.smem_doubles = 0; seg.threads = 256;
      plan.push_back(seg);
      for (int s : order1) S.level_tasks[pos++] = s;
    }
    for (int c = 3; c >= 0; c--) {
      if (order[c].empty()) continue;
      LaunchSeg seg;
      seg.kind = 0;
      seg.level = l;
      seg.base = pos;
      seg.count = (int)order[c].size();
      seg.smem_doubles = c == 3 ? 0 : (int)classes[c];
      seg.threads = c == 0 ? 64 : 256;
      plan.push_back(seg);
      for (int s : order[c]) S.level_tasks[pos++] = s;
    }
    for (size_t k = big0; k < big_tasks.size(); k++) S.level_tasks[pos++] = big_tasks[k];
    for (int s : not_mine) S.level_tasks[pos++] = s;
    if (big_tasks.size() > big0) {
      LaunchSeg seg;
      seg.kind = 1; seg.level = l; seg.base = (int)big0; seg.count = (int)(big_tasks.size() - big0);
      seg.smem_doubles = (int)(smem_panel / 8); seg.threads = PB_NT;
      plan.push_back(seg);
      seg.kind = 2; seg.base = (int)tile0; seg.count = (int)(tiles.size() - tile0);
      seg.smem_doubles = (int)(smem_tiles / 8); seg.threads = 256;
      plan.push_back(seg);
    }
  }
  {
    int* t1 = nullptr;
    if ((rc = upload(&t1, big_tasks))) return rc;
    d_big_tasks = t1;
    int4* t4 = nullptr;
    CK(cudaMalloc((void**)&t4, (tiles.size() ? tiles.size() : 1) * sizeof(int4)));
    if (!tiles.empty()) CK(cudaMemcpy(t4, tiles.data(), tiles.size() * sizeof(int4), cudaMemcpyHostToDevice));
    d_tiles = t4;
    n_tiles = (int64_t)tiles.size();
  }
  cb_tmark("ldl: launch plan + tiles");
  // small children (nr <= CB_SMALL_CHILD) of big fronts: one dst-sorted (src,dst) list per panel and per tile
  std::vector<signed char> small_child;
  std::vector<int> h_sc_panel_ptr, h_sc_tile_ptr;
  {
    std::vector<int> big_pos(S.nsup, -1), tile_base(S.nsup, -1);
    for (size_t k = 0; k < big_tasks.size(); k++) big_pos[big_tasks[k]] = (int)k;
    for (size_t k = 0; k < tiles.size(); k++) if (tile_base[tiles[k].x] < 0) tile_base[tiles[k].x] = (int)k;
    std::vector<signed char>& small = small_child;
    small.assign(S.nsup, 0);
    struct Ent { int key; int dst; int src; };
    std::vector<Ent> pe, te;
    {
      // two passes over the children on host threads: count (pe / te entries per child), prefix sums, fill -- the
      // entry order (child, column b, row a) is the one of a single loop
      const unsigned hc2 = std::max(1u, std::min(16u, host_threads()));
      const unsigned nth2 = S.nsup < 20000 ? 1u : hc2;
      std::vector<int64_t> npe((size_t)S.nsup + 1, 0), nte((size_t)S.nsup + 1, 0);
      auto eligible = [&](int c) {
        const int p = S.sn_parent[c];
        if (p < 0 || big_pos[p] < 0) return false;
        const int nrc = (int)(S.sn_rowptr[c + 1] - S.sn_rowptr[c]);
        if (nrc > CB_SMALL_CHILD) return false;
        if (S.upd_off[c] + (int64_t)nrc * nrc > 0x7fffffffLL) return false;   // int32 source indices
        return true;
      };
      auto run = [&](auto&& fn) {
        if (nth2 == 1) { fn(0, S.nsup); return; }
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nth2; t++)
          th.emplace_back([&, t]() { fn((int)((int64_t)S.nsup * t / nth2), (int)((int64_t)S.nsup * (t + 1) / nth2)); });
        for (auto& x : th) x.join();
      };
      run([&](int c0, int c1) {
        for (int c = c0; c < c1; c++) {
          if (!eligible(c)) continue;
          small[c] = 1;
          const int p = S.sn_parent[c];
          const int64_t b0 = S.sn_rowptr[c];
          const int nrc = (int)(S.sn_rowptr[c + 1] - b0);
          const int pns = S.sn_first[p + 1] - S.sn_first[p];
          int64_t np_ = 0;
          for (int b = 0; b < nrc; b++) if (S.rel[b0 + b] < pns) np_ += nrc - b;
          npe[c + 1] = np_;
          nte[c + 1] = (int64_t)nrc * (nrc + 1) / 2 - np_;
        }
      });
      for (int c = 0; c < S.nsup; c++) { npe[c + 1] += npe[c]; nte[c + 1] += nte[c]; }
      pe.resize((size_t)npe[S.nsup]);
      te.resize((size_t)nte[S.nsup]);
      run([&](int c0, int c1) {
        for (int c = c0; c < c1; c++) {
          if (!small[c]) continue;
          const int p = S.sn_parent[c];
          const int64_t b0 = S.sn_rowptr[c];
          const int nrc = (int)(S.sn_rowptr[c + 1] - b0);
          const int pns = S.sn_first[p + 1] - S.sn_first[p];
          const int pld = pns + (int)(S.sn_rowptr[p + 1] - S.sn_rowptr[p]);
          Ent* wp = pe.data() + npe[c];
          Ent* wt = te.data() + nte[c];
          for (int b = 0; b < nrc; b++)
            for (int a = b; a < nrc; a++) {
              const int ra = S.rel[b0 + a], rb = S.rel[b0 + b];
              const int64_t src = S.upd_off[c] + (int64_t)b * nrc + a;
              if (rb < pns) *wp++ = Ent{big_pos[p], rb * pld + ra, (int)src};
              else {
                const int ti = (ra - pns) / TS, tj = (rb - pns) / TS;
                *wt++ = Ent{tile_base[p] + ti * (ti + 1) / 2 + tj,
                            (ra - pns - ti * TS) * (TS + 1) + (rb - pns - tj * TS), (int)src};
              }
            }
        }
      });
    }
    cb_tmark("ldl:   small-child: entries");
    // bucket by key (counting sort keeps the child order inside a key), then order every bucket by dst with a
    // stable sort; buckets are independent, so host threads share them
    auto build = [&](std::vector<Ent>& v, size_t nkeys, std::vector<int>& ptr, std::vector<int>& src, std::vector<int>& dst) {
      ptr.assign(nkeys + 1, 0);
      for (auto& e : v) ptr[e.key + 1]++;
      for (size_t i = 0; i < nkeys; i++) ptr[i + 1] += ptr[i];
      std::vector<Ent> w(v.size());
      {
        std::vector<int> pos(ptr.begin(), ptr.end() - 1);
        for (auto& e : v) w[pos[e.key]++] = e;
      }
      const unsigned hc = std::max(1u, std::min(16u, host_threads()));
      std::vector<std::thread> th;
      for (unsigned t = 0; t < hc; t++)
        th.emplace_back([&, t]() {
          for (size_t k = t; k < nkeys; k += hc)
            std::stable_sort(w.begin() + ptr[k], w.begin() + ptr[k + 1], [](const Ent& x, const Ent& y) { return x.dst < y.dst; });
        });
      for (auto& x : th) x.join();
      src.resize(w.size() ? w.size() : 1); dst.resize(w.size() ? w.size() : 1);
      for (size_t i = 0; i < w.size(); i++) { src[i] = w[i].src; dst[i] = w[i].dst; }
    };
    // the panel lists and the tile lists are independent: the tile lists are built on a second host thread
    std::vector<int> ptr, src, dst, tptr, tsrc, tdst;
    int* t1 = nullptr;
    {
      std::thread tb([&]() { build(te, tiles.size(), tptr, tsrc, tdst); });
      build(pe, big_tasks.size(), ptr, src, dst);
      tb.join();
    }
    cb_tmark("ldl:   small-child: panel + tile lists");
    h_sc_panel_ptr = ptr;
    if ((rc = upload(&t1, ptr))) return rc; dev.sc_panel_ptr = t1;
    if ((rc = upload(&t1, src))) return rc; dev.sc_panel_src = t1;
    if ((rc = upload(&t1, dst))) return rc; dev.sc_panel_dst = t1;
    h_sc_tile_ptr = tptr;
    if ((rc = upload(&t1, tptr))) return rc; dev.sc_tile_ptr = t1;
    if ((rc = upload(&t1, tsrc))) return rc; dev.sc_tile_src = t1;
    if ((rc = upload(&t1, tdst))) return rc; dev.sc_tile_dst = t1;
    signed char* t8 = nullptr;
    if ((rc = upload(&t8, small))) return rc; dev.child_small = t8;
  }
  th_child.join();
  if (rc_child) return rc_child;
  cb_tmark("ldl: small-child entry lists");
  // solve plan (ldl_solve.cuh): level-0 narrow fronts get plain kernels, everything else becomes queue tasks in level
  // order -- batches of narrow fronts, and for every wide front a head task (pivot block + first rows) followed by row
  // tasks when the panel exceeds the shared-memory slab.
  // level_tasks was re-ordered inside levels: re-upload
  CK(cudaMemcpy((void*)dev.level_tasks, S.level_tasks.data(), S.level_tasks.size() * sizeof(int),
                cudaMemcpyHostToDevice));
  {
    int nsm = 0;
    CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
    // resident CTAs per SM and the slab size that goes with it (227 KB of shared memory per SM, 1 KB reserved per CTA)
    solve_minb = 3;      // C4 on an H100 (700 W): 25.4 it/s against 25.0 with 2 and 25.1 with 4 resident CTAs
    if (const char* e = std::getenv("CB_SOLVE_MINB")) solve_minb = std::min(4, std::max(2, std::atoi(e)));
    const size_t extra2 = (size_t)2 * (2 * CB_PB_MAXNS + SV_MAXROWS + 4 * CB_PB_MAXNS) * sizeof(double);   // NR = 2 vectors
    {
      const size_t per_cta = ((size_t)227 * 1024) / solve_minb - 1024 - 64;
      sv_cap = (int)((per_cta - extra2) / sizeof(double)) - 2;
      sv_cap &= ~1;
      sv_cap = std::min(sv_cap, 16384);
      if (const char* e = std::getenv("CB_SOLVE_CAP")) sv_cap = std::max(CB_PB_MAXNS * (CB_PB_MAXNS + 9), std::atoi(e)) & ~1;
    }
    const int cap = sv_cap;
    auto wide = [&](int s) { return S.sn_first[s + 1] - S.sn_first[s] > CB_SOLVE_SMALL_NS; };
    auto has_kids = [&](int s) { return S.child_ptr[s + 1] > S.child_ptr[s]; };
    // head rows / rows per row task of a wide front
    auto split = [&](int ns, int nr, int& rh, int& nrt, int& chunk) {
      // a panel that fits goes to shared memory whole (one bulk copy, leading dimension ld); otherwise the head takes
      // the pivot block + as many rows as fit and row tasks take the rest: a slab of r staged rows needs
      // sv_lds(r, ld) * ns doubles + one for the alignment offset
      const int ld = ns + nr;
      if (nr <= SV_MAXROWS && (long long)ns * ld + 1 <= cap) { rh = nr; nrt = 0; chunk = 0; return; }
      auto fits = [&](int staged) { return (long long)sv_lds(staged, ld) * ns + 1 <= (long long)cap; };
      rh = std::min(nr, SV_MAXROWS);
      while (rh > 0 && !fits(ns + rh)) rh--;
      int rmax = SV_MAXROWS;
      while (rmax > 1 && !fits(rmax)) rmax--;
      const int rest = nr - rh;
      nrt = rest > 0 ? (rest + rmax - 1) / rmax : 0;
      chunk = nrt ? (rest + nrt - 1) / nrt : 0;
    };
    std::vector<int> leaf1, leafn, leafw, fronts, f2t(S.nsup, -1), nrt_of(S.nsup, 0), rh_of(S.nsup, 0), chunk_of(S.nsup, 0);
    std::vector<SVTask> tk;
    const int per = SV_NT / 32;
    for (int ph = 0; ph < (sharded() ? 2 : 1); ph++) {
      if (ph == 1) sv_ntask_owned = (int)tk.size();
      std::vector<std::vector<int>> lev_small(S.nlevels), lev_big(S.nlevels);
      for (int s = 0; s < S.nsup; s++) {
        if (sharded() && (ph == 0 ? !owned(s) : shard.owner[s] >= 0)) continue;
        if (!wide(s) && !has_kids(s)) { (S.sn_first[s + 1] - S.sn_first[s] == 1 ? leaf1 : leafn).push_back(s); continue; }
        if (wide(s) && !has_kids(s) && S.sn_rowptr[s + 1] - S.sn_rowptr[s] <= 1024) {
          leafw.push_back(s);
          sv_leafw_nrmax = std::max(sv_leafw_nrmax, (int)(S.sn_rowptr[s + 1] - S.sn_rowptr[s]));
          continue;
        }
        (wide(s) ? lev_big : lev_small)[S.sn_level[s]].push_back(s);
      }
      for (int l = 0; l < S.nlevels; l++) {
        for (size_t i = 0; i < lev_small[l].size(); i += per) {
          const int c = (int)std::min<size_t>(per, lev_small[l].size() - i);
          SVTask t{};
          t.kind = 0; t.s = (int)fronts.size(); t.cnt = c; t.dep1 = -1; t.dep2 = -1; t.bowner = -1; t.ptask = -1; t.cuoff = -1;
          for (int k = 0; k < c; k++) { f2t[lev_small[l][i + k]] = (int)tk.size(); fronts.push_back(lev_small[l][i + k]); }
          tk.push_back(t);
        }
        for (int s : lev_big[l]) {
          const int ns = S.sn_first[s + 1] - S.sn_first[s], nr = (int)(S.sn_rowptr[s + 1] - S.sn_rowptr[s]);
          int rh, nrt, chunk;
          split(ns, nr, rh, nrt, chunk);
          rh_of[s] = rh; nrt_of[s] = nrt; chunk_of[s] = chunk;
          f2t[s] = (int)tk.size();
          for (int b = -1; b < nrt; b++) {
            SVTask t{};
            t.kind = b < 0 ? 1 : 2; t.s = s; t.f = S.sn_first[s]; t.ns = ns; t.nr = nr;
            t.r0 = b < 0 ? 0 : rh + b * chunk;
            t.r1 = b < 0 ? rh : std::min(nr, rh + (b + 1) * chunk);
            t.poff = S.panel_off[s]; t.rp = S.sn_rowptr[s];
            t.dep0 = 0; t.dep1 = -1; t.dep2 = -1; t.nrt = nrt; t.bowner = -1; t.bslot = 0; t.pure = 0; t.ptask = -1; t.cuoff = -1;
            t.notify = 1;
            tk.push_back(t);
          }
        }
      }
    }
    const int nt = (int)tk.size();
    if (!sharded()) sv_ntask_owned = nt;
    // chain children of wide fronts: followed slab by slab instead of awaited as a whole
    std::vector<int> chain_child(S.nsup, -1), col2sn(n, 0);
    for (int s = 0; s < S.nsup; s++)
      for (int j = S.sn_first[s]; j < S.sn_first[s + 1]; j++) col2sn[j] = s;
    for (int c = 0; c < S.nsup; c++) {
      const int p = S.sn_parent[c];
      if (p < 0 || !wide(c) || !wide(p) || chain_child[p] >= 0) continue;
      const int64_t nrc = S.sn_rowptr[c + 1] - S.sn_rowptr[c];
      const int64_t nsp = S.sn_first[p + 1] - S.sn_first[p], nrp = S.sn_rowptr[p + 1] - S.sn_rowptr[p];
      if (nrc == nsp + nrp) chain_child[p] = c;       // rows(c) is a subset of cols(p)+rows(p): equal sizes = equal sets
    }
    // task of front c covering its row i (of its L21 part)
    auto task_of_row = [&](int c, int i) {
      if (i < rh_of[c]) return f2t[c];
      return f2t[c] + 1 + (i - rh_of[c]) / chunk_of[c];
    };
    int nslots = 0;
    std::vector<int> pend(nt, 0), fleft(S.nsup, 0), bleft(S.nsup, 0);
    for (int s = 0; s < S.nsup; s++) {
      if (f2t[s] < 0 || !wide(s)) continue;
      const int ns = S.sn_first[s + 1] - S.sn_first[s], nr = (int)(S.sn_rowptr[s + 1] - S.sn_rowptr[s]);
      const int h = f2t[s], nrt = nrt_of[s], p = S.sn_parent[s];
      fleft[s] = 1 + nrt; bleft[s] = nrt;
      const int c = chain_child[s];
      const bool follow = c >= 0 && f2t[c] >= 0;      // a chain child of another rank is complete before this phase starts
      const bool pure = c >= 0 && S.child_ptr[s + 1] - S.child_ptr[s] == 1;
      for (int b = -1; b < nrt; b++) {
        SVTask& t = tk[h + 1 + b];
        t.ptask = p >= 0 ? f2t[p] : -1;
        t.notify = (p >= 0 && chain_child[p] == s) ? 0 : 1;
        t.pure = pure ? 1 : 0;
        t.cuoff = pure ? (long long)S.sn_rowptr[c] : -1;
        t.bslot = b < 0 ? nslots : nslots + b;
        if (t.r1 > t.r0) t.bowner = col2sn[S.sn_rows[S.sn_rowptr[s] + t.r0]];
        if (follow) {
          if (b < 0) {
            t.dep0 = task_of_row(c, 0); t.dep1 = task_of_row(c, ns - 1);
            t.dep2 = t.r1 > 0 ? task_of_row(c, ns + t.r1 - 1) : t.dep1;
          } else {
            t.dep0 = task_of_row(c, ns + t.r0); t.dep1 = task_of_row(c, ns + t.r1 - 1);
          }
        }
      }
      nslots += nrt;
      (void)nr;
    }
    for (int s = 0; s < S.nsup; s++) {
      const int p = S.sn_parent[s];
      if (p >= 0 && f2t[s] >= 0 && chain_child[p] != s) pend[f2t[p]]++;   // leaves and other ranks' fronts are complete before the sweep starts
    }
    // wide fronts whose pivot block is inverted after every refactorisation (all that this rank factors)
    std::vector<int> wlist;
    for (int s = 0; s < S.nsup; s++) if (wide(s) && mine(s)) wlist.push_back(s);
    sv_nwide = (int)wlist.size();
    // sorted by pivot count, cut into at most 8 runs (each run is launched with the shared memory of its widest front)
    std::stable_sort(wlist.begin(), wlist.end(), [&](int a, int b) { return S.sn_first[a + 1] - S.sn_first[a] < S.sn_first[b + 1] - S.sn_first[b]; });
    sv_wide_runs.clear();
    {
      const int bounds[] = {16, 24, 32, 40, 48, 56, CB_PB_MAXNS};
      int pos = 0;
      for (int bd : bounds) {
        int e = pos;
        while (e < sv_nwide && S.sn_first[wlist[e] + 1] - S.sn_first[wlist[e]] <= bd) e++;
        if (e > pos) { sv_wide_runs.push_back(pos); sv_wide_runs.push_back(bd); pos = e; }
      }
      sv_wide_runs.push_back(sv_nwide); sv_wide_runs.push_back(0);
    }
    sv_nleaf1 = (int)leaf1.size(); sv_nleafn = (int)leafn.size(); sv_nleafw = (int)leafw.size();
    sv_leafw_grid = sv_nleafw;      // one CTA per front (a loop over fronts inside fewer CTAs was slower: 312 vs 189 us forward on C4)
    int* t1 = nullptr;
    if ((rc = upload(&t1, wlist))) return rc; d_sv_wide = t1;
    if ((rc = upload(&t1, leaf1))) return rc; d_sv_leaf1 = t1;
    if ((rc = upload(&t1, leafn))) return rc; d_sv_leafn = t1;
    if ((rc = upload(&t1, leafw))) return rc; d_sv_leafw = t1;
    if ((rc = upload(&t1, fronts))) return rc; sv.fronts = t1;
    if ((rc = upload(&t1, f2t))) return rc; sv.front2task = t1;
    if ((rc = upload(&t1, S.sn_parent))) return rc; sv.parent = t1;
    {
      static_assert(sizeof(SVTask) == 96, "SVTask is 6 x int4");
      int4* t4 = nullptr;
      CK(cudaMalloc((void**)&t4, (size_t)(nt ? nt : 1) * sizeof(SVTask)));
      if (nt) CK(cudaMemcpy(t4, tk.data(), (size_t)nt * sizeof(SVTask), cudaMemcpyHostToDevice));
      sv.tasks = t4;
    }
    // counters: [pend(nt) | fleft(nsup) | bleft(nsup)] are copied from their initial values before every solve,
    // [tdone(nt) | ydone(nsup) | done(nsup) | qhead(2)] are cleared
    sv_ninit = (size_t)nt + 2 * (size_t)S.nsup;
    sv_nzero = (size_t)nt + 2 * (size_t)S.nsup + 2;
    std::vector<int> init(sv_ninit ? sv_ninit : 1, 0);
    std::copy(pend.begin(), pend.end(), init.begin());
    std::copy(fleft.begin(), fleft.end(), init.begin() + nt);
    std::copy(bleft.begin(), bleft.end(), init.begin() + nt + S.nsup);
    if ((rc = upload(&t1, init))) return rc; d_sv_init = t1;
    CK(cudaMalloc((void**)&d_sv_cnt, (sv_ninit + sv_nzero) * sizeof(int)));
    sv.pend = d_sv_cnt; sv.fleft = d_sv_cnt + nt; sv.bleft = sv.fleft + S.nsup;
    sv.tdone = d_sv_cnt + sv_ninit; sv.ydone = sv.tdone + nt; sv.done = sv.ydone + S.nsup; sv.qhead = sv.done + S.nsup;
    sv.bpart_stride = (long long)(nslots ? nslots : 1) * CB_PB_MAXNS;
    CK(cudaMalloc((void**)&sv.bpart, (size_t)2 * sv.bpart_stride * sizeof(double)));
    sv.ntask = nt;
    // launch geometry: dynamic shared memory = slab + vectors for one or two right-hand sides
    for (int nr2 = 1; nr2 <= 2; nr2++)
      sv_smem[nr2 - 1] = ((size_t)cap + 2 + (size_t)nr2 * (2 * CB_PB_MAXNS + SV_MAXROWS + 4 * CB_PB_MAXNS)) * sizeof(double);
    if ((rc = sv_configure())) return rc;
    int occ = sv_occupancy();
    if (occ < 1) return CLDL_E_CUDA;
    df_grid = nsm * occ;
    if (const char* e = std::getenv("CB_DF_GRID")) df_grid = std::max(1, std::atoi(e));
    use_dataflow = true;
    if (std::getenv("CB_DF_TRACE_SOLVE") && nt > 0) {
      CK(cudaMalloc((void**)&sv.trace, (size_t)nt * 8 * sizeof(unsigned long long)));
      CK(cudaMemset(sv.trace, 0, (size_t)nt * 8 * sizeof(unsigned long long)));
      h_sv_tasks.assign((const int*)tk.data(), (const int*)tk.data() + (size_t)nt * 24);
    }
    if (std::getenv("CB_TIMING") != nullptr) std::fprintf(stderr, "[cb timing]     solve plan: %d tasks (%d leaf columns, %d narrow leaves, %d wide leaves, %d wide fronts, %d row slabs), slab %d doubles, %d CTAs\n",
                                     nt, sv_nleaf1, sv_nleafn, sv_nleafw, sv_nwide, nslots, cap, df_grid);
  }
  cb_tmark("ldl:   solve plan: dataflow solve tasks");
  // dataflow factorisation plan (k_factor_df): level 0's small fronts keep their level-synchronous launch
  // (no dependencies, ~10^5 tiny CTAs); everything else becomes queue tasks in level order.  Every task
  // record carries the front's constants and the range of its child records, so a task starts with two
  // dependent loads (record, child records) instead of walking the tree arrays.
  {
    std::vector<int> big_pos(S.nsup, -1), tile_base(S.nsup, -1);
    for (size_t k = 0; k < big_tasks.size(); k++) big_pos[big_tasks[k]] = (int)k;
    for (size_t k = 0; k < tiles.size(); k++) if (tile_base[tiles[k].x] < 0) tile_base[tiles[k].x] = (int)k;
    std::vector<int> tk;       // 16 ints per task
    std::vector<int> desc;     // 12 ints per child record
    std::vector<int> cnt_init(4 * (size_t)S.nsup, 0);   // [pend | diag_done | rows_left | tiles_left]
    int* pend = cnt_init.data();
    int* rows_left = cnt_init.data() + 2 * (size_t)S.nsup;
    int* tiles_left = cnt_init.data() + 3 * (size_t)S.nsup;
    auto is_big = [&](int s) { return big_pos[s] >= 0; };
    for (int s = 0; s < S.nsup; s++) {
      const int p = S.sn_parent[s];
      const bool presolved = (S.sn_level[s] == 0 && !is_big(s));
      if (p >= 0 && !presolved && mine(s)) pend[p]++;   // sharded: another rank's front is complete before the top phase starts
    }
    auto push_task = [&](int kind, int s, int a, int b, int d0, int d1, int e0, int e1) {
      const size_t o = tk.size();
      tk.resize(o + 16, 0);
      int* t = tk.data() + o;
      t[0] = kind; t[1] = s; t[2] = a; t[3] = b;
      t[4] = S.sn_first[s + 1] - S.sn_first[s];
      t[5] = (int)(S.sn_rowptr[s + 1] - S.sn_rowptr[s]);
      t[6] = S.sn_first[s];
      t[7] = d0; t[8] = d1; t[9] = e0; t[10] = e1;
      const long long po = S.panel_off[s], uo = S.upd_off[s];
      std::memcpy(t + 12, &po, 8);
      std::memcpy(t + 14, &uo, 8);
    };
    auto push_desc = [&](int c, int a0, int a1, int b0, int b1) {
      const size_t o = desc.size();
      desc.resize(o + 12, 0);
      int* t = desc.data() + o;
      const long long uo = S.upd_off[c], rp = S.sn_rowptr[c];
      std::memcpy(t, &uo, 8);
      std::memcpy(t + 2, &rp, 8);
      t[4] = (int)(S.sn_rowptr[c + 1] - S.sn_rowptr[c]);
      t[5] = a0; t[6] = a1; t[7] = b0; t[8] = b1;
      const int* rl = S.rel.data() + rp;
      const bool rc_ = rl[a1 - 1] - rl[a0] == a1 - 1 - a0, cc_ = rl[b1 - 1] - rl[b0] == b1 - 1 - b0;
      t[9] = (rc_ ? 1 : 0) | (cc_ ? 2 : 0);
      t[10] = rl[a0];
      t[11] = rl[b0];
    };
    // sharded: tasks of the owned subtrees first, then the tasks of the top part; nothing for other ranks' fronts
    std::vector<int> kidsbuf, tp;
    for (int ph = 0; ph < (sharded() ? 2 : 1); ph++) {
    if (ph == 1) dff_ntask_owned = (int)(tk.size() / 16);
    std::vector<std::vector<int>> lev(S.nlevels);
    for (int s = 0; s < S.nsup; s++) {
      if (sharded() && (ph == 0 ? !owned(s) : shard.owner[s] >= 0)) continue;
      lev[S.sn_level[s]].push_back(s);
    }
    for (int l = 0; l < S.nlevels; l++) {
      for (int s : lev[l]) if (!is_big(s) && l > 0) push_task(0, s, 0, 0, 0, 0, 0, 0);
      // the children of a big front that go through child records (the small ones use the sorted entry lists)
      auto heavy_kids = [&](int s) {
        kidsbuf.clear();
        for (int64_t ci = S.child_ptr[s]; ci < S.child_ptr[s + 1]; ci++) {
          const int c = S.child_list[ci];
          if (!small_child[c] && S.sn_rowptr[c + 1] > S.sn_rowptr[c]) kidsbuf.push_back(c);
        }
      };
      for (int s : lev[l]) if (is_big(s)) {
        heavy_kids(s);
        const int d0 = (int)(desc.size() / 12);
        for (int c : kidsbuf) if (h_child_nb[c] > 0) push_desc(c, 0, h_child_nb[c], 0, h_child_nb[c]);
        push_task(1, s, 0, 0, d0, (int)(desc.size() / 12), h_sc_panel_ptr[big_pos[s]], h_sc_panel_ptr[big_pos[s] + 1]);
      }
      for (int s : lev[l]) if (is_big(s)) {
        heavy_kids(s);
        const int ns = S.sn_first[s + 1] - S.sn_first[s];
        const int nr = (int)(S.sn_rowptr[s + 1] - S.sn_rowptr[s]);
        const int nb = (nr + DF_RB - 1) / DF_RB;
        rows_left[s] = nb;
        for (int b = 0; b < nb; b++) {
          const int g0 = ns + b * DF_RB, g1 = std::min(ns + nr, g0 + DF_RB);
          const int d0 = (int)(desc.size() / 12);
          for (int c : kidsbuf) {
            if (h_child_nb[c] == 0) continue;
            const int* rb = S.rel.data() + S.sn_rowptr[c];
            const int* re = S.rel.data() + S.sn_rowptr[c + 1];
            const int alo = (int)(std::lower_bound(rb, re, g0) - rb), ahi = (int)(std::lower_bound(rb, re, g1) - rb);
            if (ahi > alo) push_desc(c, alo, ahi, 0, h_child_nb[c]);
          }
          push_task(2, s, b, 0, d0, (int)(desc.size() / 12), h_sc_panel_ptr[big_pos[s]], h_sc_panel_ptr[big_pos[s] + 1]);
        }
      }
      for (int s : lev[l]) if (is_big(s)) {
        heavy_kids(s);
        const int ns = S.sn_first[s + 1] - S.sn_first[s];
        const int nr = (int)(S.sn_rowptr[s + 1] - S.sn_rowptr[s]);
        const int nt = (nr + TS - 1) / TS;
        tiles_left[s] = nt * (nt + 1) / 2;
        // per child: first child row of every tile row
        std::vector<std::vector<int>> ctp(kidsbuf.size());
        for (size_t k = 0; k < kidsbuf.size(); k++) {
          const int c = kidsbuf[k];
          const int* rb = S.rel.data() + S.sn_rowptr[c];
          const int* re = S.rel.data() + S.sn_rowptr[c + 1];
          ctp[k].resize(nt + 1);
          for (int t = 0; t <= nt; t++) ctp[k][t] = (int)(std::lower_bound(rb, re, ns + t * TS) - rb);
        }
        // the children that reach tile (ti, tj), in child order: bucketed per tile from each child's own tile rows
        // (a front under hundreds of children and with hundreds of tile rows -- the linking block of a
        // block-angular problem -- would otherwise test every child against every tile)
        const int ntile = nt * (nt + 1) / 2;
        std::vector<int> tile_ptr(ntile + 1, 0), tile_kid;
        {
          std::vector<std::vector<int>> trows(kidsbuf.size());
          for (size_t k = 0; k < kidsbuf.size(); k++)
            for (int t = 0; t < nt; t++) if (ctp[k][t + 1] > ctp[k][t]) trows[k].push_back(t);
          for (size_t k = 0; k < kidsbuf.size(); k++)
            for (size_t a = 0; a < trows[k].size(); a++)
              for (size_t b = 0; b <= a; b++) tile_ptr[trows[k][a] * (trows[k][a] + 1) / 2 + trows[k][b] + 1]++;
          for (int t = 0; t < ntile; t++) tile_ptr[t + 1] += tile_ptr[t];
          tile_kid.resize(tile_ptr[ntile]);
          std::vector<int> pos(tile_ptr.begin(), tile_ptr.end() - 1);
          for (size_t k = 0; k < kidsbuf.size(); k++)
            for (size_t a = 0; a < trows[k].size(); a++)
              for (size_t b = 0; b <= a; b++) tile_kid[pos[trows[k][a] * (trows[k][a] + 1) / 2 + trows[k][b]]++] = (int)k;
        }
        for (int ti = 0; ti < nt; ti++)
          for (int tj = 0; tj <= ti; tj++) {
            const int d0 = (int)(desc.size() / 12);
            // children whose block is contiguous in the tile go first: the tile task adds them in registers
            int ndense = 0;
            const int tix = ti * (ti + 1) / 2 + tj;
            for (int pass = 0; pass < 2; pass++)
              for (int q = tile_ptr[tix]; q < tile_ptr[tix + 1]; q++) {
                const size_t k = (size_t)tile_kid[q];
                const int a0 = ctp[k][ti], a1 = ctp[k][ti + 1], b0 = ctp[k][tj], b1 = ctp[k][tj + 1];
                if (!(a1 > a0 && b1 > b0)) continue;
                const int* rl = S.rel.data() + S.sn_rowptr[kidsbuf[k]];
                const bool dense = rl[a1 - 1] - rl[a0] == a1 - 1 - a0 && rl[b1 - 1] - rl[b0] == b1 - 1 - b0;
                if (dense != (pass == 0)) continue;
                push_desc(kidsbuf[k], a0, a1, b0, b1);
                if (dense) ndense++;
              }
            const int t = tile_base[s] + ti * (ti + 1) / 2 + tj;
            push_task(3, s, ti, tj, d0, (int)(desc.size() / 12), h_sc_tile_ptr[t], h_sc_tile_ptr[t + 1]);
            tk[tk.size() - 16 + 11] = ndense;
          }
      }
    }
    }
    cb_tmark("ldl:   solve plan: factor tasks built");
    if (std::getenv("CB_TIMING")) std::fprintf(stderr, "[cb timing]     factor plan: %zu tasks, %zu child records, %zu big fronts, %zu tiles\n",
                                                tk.size() / 16, desc.size() / 12, big_tasks.size(), tiles.size());
    dff.ntask = (int)(tk.size() / 16);
    if (!sharded()) dff_ntask_owned = dff.ntask;
    int4* t4 = nullptr;
    CK(cudaMalloc((void**)&t4, (tk.size() ? tk.size() : 16) * sizeof(int)));
    if (!tk.empty()) CK(cudaMemcpy(t4, tk.data(), tk.size() * sizeof(int), cudaMemcpyHostToDevice));
    dff.tasks = t4;
    int* t1 = nullptr;
    if ((rc = upload(&t1, desc))) return rc; dff.desc = t1;
    if ((rc = upload(&t1, cnt_init))) return rc; d_dff_init = t1;
    CK(cudaMalloc((void**)&d_dff_cnt, cnt_init.size() * sizeof(int) + 16));
    dff.pend = d_dff_cnt; dff.diag_done = d_dff_cnt + S.nsup; dff.rows_left = d_dff_cnt + 2 * (size_t)S.nsup;
    dff.tiles_left = d_dff_cnt + 3 * (size_t)S.nsup;
    CK(cudaMalloc((void**)&dff.qhead, sizeof(int)));
    if ((rc = upload(&t1, S.sn_parent))) return rc; dff.parent = t1;
    if ((rc = upload(&t1, big_pos))) return rc; dff.big_pos = t1;
    if ((rc = upload(&t1, tile_base))) return rc; dff.tile_base = t1;
    CK(cudaFuncSetAttribute(k_factor_df, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_SMEM_DOUBLES * 8));
    int nsm = 0, occ = 0;
    CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_factor_df, DF_NT, (size_t)DF_SMEM_DOUBLES * 8));
    dff_grid = nsm * std::max(1, occ);
    dff_nsup4 = 4 * (size_t)S.nsup;
    factor_dataflow = std::getenv("CB_FACTOR_LEVELSYNC") == nullptr;
    if (std::getenv("CB_DF_TRACE") && dff.ntask > 0) {
      h_dff_tasks = tk;
      CK(cudaMalloc((void**)&dff.trace, (size_t)dff.ntask * 10 * sizeof(unsigned long long)));
      CK(cudaMemset(dff.trace, 0, (size_t)dff.ntask * 10 * sizeof(unsigned long long)));
    }
  }
  cb_tmark("ldl: solve plan");
  if (sharded()) {
    d_shard_xidx.assign(shard_nranks, nullptr);
    for (int w = 0; w < 2; w++) { d_shard_segs[w].assign(shard_nranks, nullptr); shard_nsegs[w].assign(shard_nranks, 0); }
    for (int g = 0; g < shard_nranks; g++) { int* t1 = nullptr; if ((rc = upload(&t1, shard_xidx[g]))) return rc; d_shard_xidx[g] = t1; }
  }
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
  fr(d_tmp_idx); fr(d_tmp_val); fr(d_tmp_sgn); fr(d_big_tasks); fr(d_tiles); fr(sv.tasks); fr(sv.fronts); fr(sv.front2task); fr(sv.parent); fr(sv.bpart); fr(sv.trace); fr(d_sv_cnt); fr(d_sv_init); fr(d_sv_wide); fr(d_sv_leaf1); fr(d_sv_leafn); fr(d_sv_leafw); fr(d_xp2); fr(d_u2); fr(dff.tasks); fr(dff.desc); fr(d_dff_init); fr(d_dff_cnt); fr(dff.qhead); fr(dff.parent); fr(dff.big_pos); fr(dff.tile_base); fr(dff.trace); fr(dev.child_nb); fr(dev.child_trange); fr(dev.gat_ptr); fr(dev.gat_src); fr(dev.child_tptr); fr(dev.child_tptr_off); fr(dev.sc_panel_ptr); fr(dev.sc_panel_src); fr(dev.sc_panel_dst); fr(dev.sc_tile_ptr); fr(dev.sc_tile_src); fr(dev.sc_tile_dst); fr(dev.child_small);
  if (h_status) cudaFreeHost(h_status);
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  for (auto& e : ev_leaf) if (e) { cudaEventDestroy(e); e = nullptr; }
  if (stream_a) { cudaStreamDestroy(stream_a); stream_a = nullptr; }
  if (stream_b) { cudaStreamDestroy(stream_b); stream_b = nullptr; }
  if (stream) cudaStreamDestroy(stream);
}

int LDLObject::refactor_async() {
  if (sharded()) return has_transport() ? refactor_sharded() : CLDL_E_ARG;   // without a transport: the phase entry points
  CK(cudaSetDevice(device));
  CK(cudaMemsetAsync(dev.status, 0, ST_COUNT * sizeof(int), stream));
  if (factor_dataflow) {
    CK(cudaMemcpyAsync(d_dff_cnt, d_dff_init, dff_nsup4 * sizeof(int), cudaMemcpyDeviceToDevice, stream));
    CK(cudaMemsetAsync(dff.qhead, 0, sizeof(int), stream));
    for (const LaunchSeg& g : plan) {
      if (g.level != 0 || (g.kind != 0 && g.kind != 3)) continue;
      g_launches++;
      if (g.kind == 3) k_factor_leaf1<<<(g.count + 255) / 256, 256, 0, stream>>>(dev, g.base, g.count);
      else if (g.threads == 64)
        k_factor_level<64><<<g.count, 64, (size_t)g.smem_doubles * 8, stream>>>(dev, g.base, g.smem_doubles);
      else
        k_factor_level<256><<<g.count, 256, (size_t)g.smem_doubles * 8, stream>>>(dev, g.base, g.smem_doubles);
    }
    g_launches++;
    k_factor_df<<<dff_grid, DF_NT, (size_t)DF_SMEM_DOUBLES * 8, stream>>>(dev, dff);
    invert_pivots();
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(h_status, dev.status, ST_COUNT * sizeof(int), cudaMemcpyDeviceToHost, stream));
    factored = true;
    return CLDL_OK;
  }
  g_launches += plan.size();
  for (const LaunchSeg& g : plan) {
    if (g.kind == 3)
      k_factor_leaf1<<<(g.count + 255) / 256, 256, 0, stream>>>(dev, g.base, g.count);
    else if (g.kind == 1)
      k_panel_big<<<g.count, PB_NT, (size_t)g.smem_doubles * 8, stream>>>(dev, d_big_tasks + g.base, g.base);
    else if (g.kind == 2)
      k_update_tiles<<<g.count, 256, (size_t)g.smem_doubles * 8, stream>>>(dev, d_tiles + g.base, g.base);
    else if (g.threads == 64)
      k_factor_level<64><<<g.count, 64, (size_t)g.smem_doubles * 8, stream>>>(dev, g.base, g.smem_doubles);
    else
      k_factor_level<256><<<g.count, 256, (size_t)g.smem_doubles * 8, stream>>>(dev, g.base, g.smem_doubles);
  }
  invert_pivots();
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(h_status, dev.status, ST_COUNT * sizeof(int), cudaMemcpyDeviceToHost, stream));
  factored = true;
  return CLDL_OK;
}

// the solves multiply by the inverse of every wide pivot block (ldl_solve.cuh): strictly lower triangle replaced in place
void LDLObject::invert_pivots() {
  if (!sv_nwide) return;
  g_launches++;
  // the list is sorted by pivot count: launched in runs of equal width so that each run asks for just its own shared memory
  for (size_t g = 0; g + 2 < sv_wide_runs.size(); g += 2) {
    const int first = sv_wide_runs[g], cnt = sv_wide_runs[g + 2] - first, ns = sv_wide_runs[g + 1];
    k_invert_pivots<<<cnt, 64, (size_t)ns * (ns + 1) * sizeof(double), stream>>>(dev, d_sv_wide + first, cnt);
  }
}

int LDLObject::sync_status() {
  CK(cudaSetDevice(device));
  CK(cudaStreamSynchronize(stream));
  regularize_count = (uint64_t)h_status[ST_REGCOUNT];
  positive_inertia = (uint64_t)h_status[ST_POSINERTIA];
  if (dff.trace && factor_dataflow) {  // diagnostic: CB_DF_TRACE=<file> dumps the last refactor's task timeline
    std::vector<unsigned long long> tr((size_t)dff.ntask * 10);
    CK(cudaMemcpy(tr.data(), dff.trace, tr.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    if (FILE* fp = std::fopen(std::getenv("CB_DF_TRACE"), "wb")) {
      const long long nt = dff.ntask;
      std::fwrite(&nt, sizeof(nt), 1, fp);
      std::fwrite(h_dff_tasks.data(), sizeof(int), (size_t)nt * 16, fp);
      std::fwrite(tr.data(), sizeof(unsigned long long), tr.size(), fp);
      std::fclose(fp);
    }
  }
  if (h_status[ST_ZEROPIV] && !dev.reg_enable) return CLDL_E_ZERO_PIVOT;
  return h_status[ST_NONFINITE] ? 0 : 1;
}

// opt-in to the dynamic shared memory of the sweep kernels (every instantiation that can be launched)
template <bool FWD, int NR, int MINB>
static cudaError_t sv_attr(size_t bytes) {
  return cudaFuncSetAttribute(k_solve2<FWD, NR, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}
int LDLObject::sv_configure() {
  for (int nr = 1; nr <= 2; nr++) {
    const size_t b = sv_smem[nr - 1];
    cudaError_t e = cudaSuccess;
    if (solve_minb == 2) { e = nr == 1 ? sv_attr<true, 1, 2>(b) : sv_attr<true, 2, 2>(b); if (e == cudaSuccess) e = nr == 1 ? sv_attr<false, 1, 2>(b) : sv_attr<false, 2, 2>(b); }
    else if (solve_minb == 3) { e = nr == 1 ? sv_attr<true, 1, 3>(b) : sv_attr<true, 2, 3>(b); if (e == cudaSuccess) e = nr == 1 ? sv_attr<false, 1, 3>(b) : sv_attr<false, 2, 3>(b); }
    else { e = nr == 1 ? sv_attr<true, 1, 4>(b) : sv_attr<true, 2, 4>(b); if (e == cudaSuccess) e = nr == 1 ? sv_attr<false, 1, 4>(b) : sv_attr<false, 2, 4>(b); }
    CK(e);
  }
  return CLDL_OK;
}
int LDLObject::sv_occupancy() {
  int occ = 1 << 30;
  for (int fwd = 0; fwd < 2; fwd++) {
    int o = 0;
    cudaError_t e;
    // the two-right-hand-side instantiation needs the most shared memory: it decides how many CTAs are co-resident
    if (solve_minb == 2) e = fwd ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_solve2<true, 2, 2>, SV_NT, sv_smem[1]) : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_solve2<false, 2, 2>, SV_NT, sv_smem[1]);
    else if (solve_minb == 3) e = fwd ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_solve2<true, 2, 3>, SV_NT, sv_smem[1]) : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_solve2<false, 2, 3>, SV_NT, sv_smem[1]);
    else e = fwd ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_solve2<true, 2, 4>, SV_NT, sv_smem[1]) : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_solve2<false, 2, 4>, SV_NT, sv_smem[1]);
    if (e != cudaSuccess) return 0;
    occ = std::min(occ, o);
  }
  return occ;
}

template <bool FWD, int NR>
static void sv_launch(int minb, int grid, size_t smem, cudaStream_t st, const LDLDev& d, const SVPlan& q, const SVRhs& r, int cap) {
  if (minb == 2) k_solve2<FWD, NR, 2><<<grid, SV_NT, smem, st>>>(d, q, r, cap);
  else if (minb == 3) k_solve2<FWD, NR, 3><<<grid, SV_NT, smem, st>>>(d, q, r, cap);
  else k_solve2<FWD, NR, 4><<<grid, SV_NT, smem, st>>>(d, q, r, cap);
}

// one sweep kernel over the task queue as it stands (queue heads / counters are prepared by the caller)
void LDLObject::sv_sweep(bool fwd, int nrhs, const SVPlan& q, const SVRhs& r) {
  g_launches++;
  const size_t smem = sv_smem[nrhs - 1];
  if (fwd) { if (nrhs == 1) sv_launch<true, 1>(solve_minb, df_grid, smem, stream, dev, q, r, sv_cap); else sv_launch<true, 2>(solve_minb, df_grid, smem, stream, dev, q, r, sv_cap); }
  else { if (nrhs == 1) sv_launch<false, 1>(solve_minb, df_grid, smem, stream, dev, q, r, sv_cap); else sv_launch<false, 2>(solve_minb, df_grid, smem, stream, dev, q, r, sv_cap); }
}
// the level-0 fronts: before the forward sweep, after the backward sweep.  The three kernels touch disjoint fronts and
// none depends on another, so the two narrow-leaf kernels run on side streams next to the wide-leaf kernel
// (C4: 24 + 48 + 186 us one after the other -> ~190 us together)
void LDLObject::sv_leaves(bool fwd, int nrhs, const SVRhs& r) {
  const bool side = stream_a && stream_b && ((sv_nleaf1 ? 1 : 0) + (sv_nleafn ? 1 : 0) + (sv_nleafw ? 1 : 0)) > 1;
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
  if (!sharded() || !factor_dataflow) return CLDL_E_ARG;
  CK(cudaSetDevice(device));
  if (phase == 0) {
    CK(cudaMemsetAsync(dev.status, 0, ST_COUNT * sizeof(int), stream));
    CK(cudaMemcpyAsync(d_dff_cnt, d_dff_init, dff_nsup4 * sizeof(int), cudaMemcpyDeviceToDevice, stream));
    CK(cudaMemsetAsync(dff.qhead, 0, sizeof(int), stream));
    for (const LaunchSeg& g : plan) {
      if (g.level != 0 || (g.kind != 0 && g.kind != 3) || g.count == 0) continue;
      g_launches++;
      if (g.kind == 3) k_factor_leaf1<<<(g.count + 255) / 256, 256, 0, stream>>>(dev, g.base, g.count);
      else if (g.threads == 64)
        k_factor_level<64><<<g.count, 64, (size_t)g.smem_doubles * 8, stream>>>(dev, g.base, g.smem_doubles);
      else
        k_factor_level<256><<<g.count, 256, (size_t)g.smem_doubles * 8, stream>>>(dev, g.base, g.smem_doubles);
    }
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
  invert_pivots();
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
  if (nccl_comm) {      // stream-ordered: the unpack kernels below simply follow the collective on `stream`
    NcclApi* a = nccl_api(nullptr);
    const int r = a->AllGather(d_xsend, d_xrecv, (size_t)cnt, /* ncclFloat64 */ 8, (cb_ncclComm_t)nccl_comm, stream);
    if (r != 0) { std::fprintf(stderr, "[clarabel_b200] ncclAllGather: %s\n", a->GetErrorString ? a->GetErrorString(r) : "error"); return CLDL_E_CUDA; }
    n_collectives++;
  } else {
    CK(cudaStreamSynchronize(stream));
    if (transport(transport_ctx, d_xsend, d_xrecv, cnt) != 0) return CLDL_E_CUDA;
  }
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
      std::fwrite(o.h_sv_tasks.data(), sizeof(int), (size_t)nt * 24, fp);
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
