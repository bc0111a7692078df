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
#define SI_RB 64            /* selected inversion: rows of Z_RS per task (fronts with more rows get row tasks) */

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

// Pruned solves (cldl_solve_sparse, cldl_inverse_entries).  The nonzeros of L^-1 b lie in the fronts of b's indices
// and their ancestors, and the backward sweep needs only the fronts of the wanted entries and their ancestors: the
// upward closure of an index set in sn_parent.  A pruned plan is the full solve plan restricted to such a closure:
// a wide front keeps its full-plan tasks (same head / row split, same bslot), narrow fronts are regrouped into batches
// of the reached fronts, the leaf lists are filtered, task indices are remapped in the level order of the full queue,
// and waits on fronts outside the closure are dropped (pend counts reached non-chain children only; a chain child
// outside the closure is not followed).  Fronts outside the closure contribute exact zeros.
struct SolvePrune {                      // built once per handle from the full plan
  std::vector<int> col2sn;               // [n] permuted column -> front
  std::vector<signed char> cls;          // [nsup] 0 leaf1, 1 leafn, 2 leafw, 3 narrow batch, 4 wide tasks, -1 none
  std::vector<int> f2t;                  // [nsup] the full plan's front2task
  std::vector<unsigned> stamp;           // [nsup] closure marks: stamp[s] == epoch while the current closure holds s
  unsigned epoch = 0;
  std::vector<int> ntf2t;                // [nsup] scratch: the pruned plan's task of a reached front
};
SolvePrune build_solve_prune(const Symbolic& S, const SolvePlan& full);

struct PrunedPlan {
  std::vector<int> reached;              // the closure, in queue order (level, then front)
  std::vector<SVTask> tasks;
  std::vector<int> pend;                 // [tasks] forward: reached non-chain children with tasks
  std::vector<int> fronts;               // narrow batches' fronts
  std::vector<int> f2t;                  // (front, task) pairs of the reached fronts that have tasks
  std::vector<int> leaf1, leafn, leafw;
  long long entries = 0;                 // panel entries (ns + nr) ns of the reached fronts
  long long work = 0;                    // host steps: closure visits, sort comparisons, records written
};
// the upward closure of the fronts of permuted columns cols[0, k) (cols may repeat), then its plan.  O(r log r) in the
// r reached fronts plus O(k); nothing proportional to n or nsup.
void build_pruned_plan(const Symbolic& S, const SolvePlan& full, SolvePrune& X, const int* cols, size_t k,
                       PrunedPlan& P);

// Rank-k updates of the factor (cldl_updown, k_updown in ldl_updown.cuh).  A column w of W whose first eliminated row
// lies in front s0 changes only the fronts on the path from s0 to the root: its other rows are ancestors of that row
// in the elimination tree (the pattern condition), and each step of the update fills w only along L's column
// structure.  The columns go in passes of at most UD_PASS; a pass's plan is the upward closure of its columns' first
// fronts, in the level order of the full factor queue, with per front the mask of the pass's columns whose path passes
// through it.  A path is a chain, so sibling fronts never share a column: each column's alpha and work vector have one
// owner at a time.  Tasks: kind 0, a whole front with at most DF_RB rows below the pivot block (the pivot block's
// sequential recurrence, then its rows); kind 1, the pivot block of a front with more rows, which publishes (p, beta)
// per (pivot, column) in the front's slot; kind 2, rows [r0, r1) of such a front, DF_RB at most, which wait for their
// kind 1 task.  Kinds 0 and 1 wait for the reached children (pend); a front is complete when its kind 0 task or its
// last row task ends.  Every wait is on a task queued earlier.
#define UD_PASS 8           /* columns of W per pass of the factor update (bits of a front's mask) */
struct UDTask {             // 32 bytes = 2 x int4
  int kind, s, li, pli;     // li: the front's index in the plan (counters), pli: the parent's (-1: a root)
  int mask, r0, r1, slot;   // mask: the pass's columns whose path passes through s; kinds 1, 2: rows and (p, beta) slot
};
static_assert(sizeof(UDTask) == 32, "UDTask is 2 x int4");
struct UpdownPlan {
  std::vector<int> reached;              // the closure, in queue order (level, then front)
  std::vector<int> mask;                 // [reached]
  std::vector<UDTask> tasks;
  std::vector<int> cnt_init;             // [3 reached]: pend (reached children) | rows_left (row tasks) | done (0)
  int nslots = 0;                        // fronts with row tasks
  long long entries = 0;                 // panel entries (ns + nr) ns of the reached fronts
  long long work = 0;                    // host steps: path visits, sort comparisons, records written
};
// first[r] (r < k <= UD_PASS): the first eliminated (permuted) row of column r.  Uses X's col2sn, stamps and scratch;
// O(k r + r log r) in the r reached fronts, nothing proportional to n or nsup.
void build_updown_plan(const Symbolic& S, SolvePrune& X, const int* first, int k, UpdownPlan& P);
// an upper bound on the slots of any pass: UD_PASS times the most fronts with row tasks on one path to a root (O(nsup))
int updown_slot_bound(const Symbolic& S);

// One task of k_selinv (48 bytes = 3 x int4), queued root to leaves.  kind 0: a whole front with at most SI_RB rows
// (its rows, then its pivot block); 1: rows [r0, r1) of Z_RS of a front with more rows; 2: the pivot block Z_SS of
// such a front, after all of its row tasks.  Kinds 0 and 1 wait for the parent front's Z, kind 2 for its row tasks.
struct SITask {
  int kind, s, r0, r1;
  int ns, nr, f, parent;    // pivots, rows below the pivot block, first column, parent front (-1: root)
  long long poff, rp;       // panel_off[s], sn_rowptr[s]
};
static_assert(sizeof(SITask) == 48, "SITask is 3 x int4");
static_assert(offsetof(SITask, ns) == 16 && offsetof(SITask, poff) == 32 && offsetof(SITask, rp) == 40, "SITask layout");

// Selected inversion: Z = (K + E)^-1 in the layout of the factor's panels.  For the rows R of front s, entry
// (R[i], R[k]) with i >= k lies in the panel of the front a that owns column R[k], at
//     Z[col[rp + k] + segpos[seg[rp + k] + i]]
// col: offset of column R[k] in a's panel; segpos: positions (0 .. ns_a + nr_a) in a's front of the rows R[k0 ..] of
// the segment of R that a owns (rows k0 .. k1), the composition of `rel` along the path from s to a.
struct SelinvPlan {
  std::vector<SITask> tasks;
  std::vector<int> rows_left;            // [nsup] row tasks of a front (0 for kind 0 fronts)
  std::vector<long long> col, seg;       // indexed like sn_rows
  std::vector<int> segpos;
  std::vector<long long> caller_pos;     // [nnzA] offset in Z of the caller's entry p (triu, caller's CSC order)
};
SelinvPlan build_selinv_plan(const Symbolic& S);

// Schur complement handle (S.schur_first >= 0): the fronts of B are rank 0's owned subtrees and the fronts of S the
// top part, which is never factored.  The output is the k x k complement, column-major, in the caller's order of the
// Schur set; permuted S column j (column schur_first + j) is output column spos[j].
struct SchurRec {           // cut root whose local row b is the permuted S column of the list it is in
  long long uoff, rp;       // upd_off[c], sn_rowptr[c]
  int nr, b;
};
static_assert(sizeof(SchurRec) == 24, "SchurRec is 6 ints");
struct SchurPlan {
  int first = 0, k = 0;                  // schur_first, |S|
  std::vector<int> owner;                // [nsup] 0: front of B, -1: front of S
  std::vector<int> cut;                  // cut roots (fronts of B whose parent is in S), ascending
  std::vector<int> spos;                 // [k] output index of permuted S column j
  // original K_SS entries per permuted S column j (the lower one of the pair): caller CSC position and output position
  // (spos[j] * k + spos[i]), sorted by output position so that duplicates are adjacent
  std::vector<long long> kss_ptr, kss_dst;
  std::vector<int> kss_src;
  std::vector<int> rec_ptr;              // [k + 1] per permuted S column: the cut roots whose rows contain it, ascending
  std::vector<SchurRec> recs;
  // expansion: the backward sweep over B's tasks alone, waiting on no S front (x_S is preset in the work vector)
  std::vector<SVTask> bwd;
  std::vector<int> bparent;              // sn_parent with the cut roots' parents replaced by -1
};
// schur: the caller's Schur set, in output order; sp: the solve plan built with `owner`
SchurPlan build_schur_plan(const Symbolic& S, const std::vector<int>& schur, const SolvePlan& sp);
// the owner vector above, for the plan builders (first: S.schur_first)
std::vector<int> schur_owner(const Symbolic& S, int first);

// The factor's parts (cldl_mul_part, cldl_get_factor_csc; ldl_parts.cuh).  L's entries below the pivot blocks by row:
// for permuted row i, the positions e in sn_rows with sn_rows[e] == i, ascending (ptr: [n + 1], pos: [nnz of L21]);
// and the compressed-column pointers of L strictly lower on the stored pattern, column f + j of front s holding
// ns - 1 - j pivot-block entries and nr entries of L21 ([n + 1], ptr[n] = sum over the fronts of ns (ns - 1) / 2 + ns nr).
struct FactorParts {
  std::vector<long long> row_ptr, row_pos;
  std::vector<uint64_t> colptr;
};
FactorParts build_factor_parts(const Symbolic& S);

}  // namespace cb
