// Plans of the multifrontal LDL^T, built on the host from the symbolic analysis: the level-0 launch plan, the task
// queue of the dataflow factorisation (k_factor_df) and the task queue of the dataflow solves (k_solve2).  The task
// records and the constants the builders share with the kernels are defined here once.  Host-only code: no CUDA
// runtime, so a plan can be built and checked without a device.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

#include "symbolic.h"

#ifdef __CUDACC__
#define CB_HD __host__ __device__
#else
#define CB_HD
#endif

#define CB_PB_MAXNS 64      /* widest panel (columns) of a front */
#define CB_SOLVE_SMALL_NS 8 /* solves: fronts with at most this many pivots get one warp, wider ones one CTA */
#define CB_SMALL_CHILD 16   /* children of big fronts with at most this many rows go through sorted entry lists */
#define CB_BIG_NR 96        /* fronts with at least this many rows below the pivot block are factored by D, R and T tasks */
#define TS 64               /* rows and columns of an update-matrix tile (T tasks) */
#define DF_RB 128           /* rows per R task */
#define SV_NT 256
#define SV_MAXROWS 256      /* rows of L21 in one slab (bounds the staged x / the per-thread row count) */

namespace cb {

// leading dimension of a staged slab of `srows` rows cut out of a panel with leading dimension ld: the parity of ld (so
// that source and destination are 16-byte aligned at the same elements of every column) and, when even, not a multiple
// of 4 (the transposed reads of the backward sweep would pile up on a few shared-memory banks)
CB_HD inline int sv_lds(int srows, int ld) {
  int L = srows + ((srows ^ ld) & 1);
  if (!(L & 1) && !(L & 3)) L += 2;
  return L;
}

// One task of k_factor_df (64 bytes = 4 x int4).  kind 0: small front, fused (F); 1: pivot block of a big front (D);
// 2: row block a of DF_RB rows below the pivot block (R); 3: tile (a, b) of the update matrix (T).
struct DFTask {
  int kind, s, a, b;
  int ns, nr, f;            // pivots, rows below the pivot block, first column of front s
  int d0, d1;               // child records [d0, d1)
  int e0, e1;               // small-child entries [e0, e1) of the panel (D, R) or of the tile (T)
  int ndense;               // T: the first ndense child records are contiguous in the tile
  long long poff, uoff;     // panel_off[s], upd_off[s]
};
static_assert(sizeof(DFTask) == 64, "DFTask is 4 x int4");
static_assert(offsetof(DFTask, d0) == 28 && offsetof(DFTask, ndense) == 44, "DFTask layout");
static_assert(offsetof(DFTask, poff) == 48 && offsetof(DFTask, uoff) == 56, "DFTask layout");

// Rows a0..a1 and columns b0..b1 (child-local indices) of a child's update matrix that land in one factor task's
// target (pivot block / row block / tile); only a >= b is stored.
struct DFChildRec {
  long long uoff, relp;     // upd_off[c], sn_rowptr[c]
  int nrc, a0, a1, b0, b1;
  int contig;               // 1: rows a0..a1 contiguous in the parent, 2: columns b0..b1, 3: both
  int ra0, rb0;             // rel[a0], rel[b0]: parent-local index of the first row / column
};
static_assert(sizeof(DFChildRec) == 48, "DFChildRec is 12 ints");
static_assert(offsetof(DFChildRec, nrc) == 16 && offsetof(DFChildRec, contig) == 36 && offsetof(DFChildRec, rb0) == 44,
              "DFChildRec layout");

struct SVTask {             // 96 bytes = 6 x int4
  int kind, s, cnt, f;      // kind 0: narrow batch (s = first index into fronts[], cnt fronts); 1 head; 2 rows
  int ns, nr, r0, r1;       // slab = rows [r0, r1) of L21 (head: r0 = 0, r1 = rh, plus the pivot block)
  long long poff, rp;       // panel offset in d.L, sn_rowptr[s]
  int dep0, dep1, dep2, nrt;   // forward: chain-child tasks [dep0, dep1] before phase A (head) / before the product (rows); head: [.., dep2] before phase B; nrt = row tasks of the front
  int bowner, bslot, pure, ptask;   // backward: front owning the slab's first row (-1: none); slot in bpart; pure-chain gather; head task of the parent (-1: root)
  long long cuoff;          // pure chain: sn_rowptr[chain child] (row i of the child is local index i of this front)
  int notify, pad;          // notify = 1: the finished front decrements its parent's counter (0 for chain children)
};
static_assert(sizeof(SVTask) == 96, "SVTask is 6 x int4");
static_assert(offsetof(SVTask, poff) == 32 && offsetof(SVTask, dep0) == 48 && offsetof(SVTask, cuoff) == 80, "SVTask layout");

// The fronts one rank handles, in queue order: queue[phase][level] = fronts in ascending order.  Unsharded (owner
// empty) there is one phase with every front; sharded there are two, the rank's owned subtrees first and then the
// replicated top part (owner -1), and other ranks' fronts appear nowhere.
using QueueOrder = std::vector<std::vector<std::vector<int>>>;
QueueOrder queue_order(const Symbolic& S, const std::vector<int>& owner, int rank);

// one launch of the level-0 factorisation over level_tasks[base, base + count): k_factor_leaf1 (single-column fronts,
// one thread each) or k_factor_level<threads> with smem_doubles of dynamic shared memory
struct LaunchSeg {
  bool leaf1;
  int base, count, smem_doubles, threads;
};
struct Level0Plan {
  std::vector<LaunchSeg> segs;
  std::vector<int> level_tasks;   // S.level_tasks with level 0 reordered into the launches, then big and other ranks' fronts
};
// smem_cap: dynamic shared memory (doubles) of the largest k_factor_level class
Level0Plan build_level0_plan(const Symbolic& S, const std::vector<int>& owner, int rank, int smem_cap);

struct FactorPlan {
  std::vector<int> big_pos, tile_base;   // [nsup] position in the big-front list / first global tile id, or -1
  // small children of big fronts: (src, dst) entries sorted by dst per big front (panel) and per tile
  std::vector<int> sc_panel_ptr, sc_panel_src, sc_panel_dst, sc_tile_ptr, sc_tile_src, sc_tile_dst;
  std::vector<DFTask> tasks;
  std::vector<DFChildRec> recs;
  std::vector<int> cnt_init;             // [4 nsup]: pend | diag_done | rows_left | tiles_left
  int ntask_owned = 0;                   // tasks of the owned phase (they come first in the queue)
};
FactorPlan build_factor_plan(const Symbolic& S, const std::vector<int>& owner, int rank);

struct SolvePlan {
  std::vector<SVTask> tasks;
  std::vector<int> cnt_init;             // pend (ntask) | fleft (nsup) | bleft (nsup)
  std::vector<int> fronts, front2task;   // narrow batches' fronts; [nsup] head / batch task of a front or -1
  std::vector<int> leaf1, leafn, leafw;  // level-0 leaves solved by plain kernels: one column, narrow, wide
  std::vector<int> wide;                 // wide fronts this rank factors: their pivot blocks hold L11^-1
  std::vector<int> gat_ptr, gat_src;     // per front slot, CSR of contributing child update-vector entries
  int nslots = 0, leafw_nrmax = 0;
  int ntask_owned = 0;
};
// cap: doubles of the shared-memory slab of a sweep CTA
SolvePlan build_solve_plan(const Symbolic& S, const std::vector<int>& owner, int rank, int cap);

}  // namespace cb
