// Device-side view and host object of the multifrontal LDL^T (internal header).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <thread>
#include <vector>

#include "../../include/clarabel_b200.h"
#include "symbolic.h"
#include "ldl_plan.h"
#include "ldl_solve_plan.h"
#include "vec.cuh"

#define CB_MAX_PANEL 128
#define CB_PB_LD 66        /* padded leading dimension of the pivot block in shared memory */

namespace cb {

struct ncclComm;   // NCCL's communicator, opaque (ldl.cu loads NCCL with dlopen)

enum { ST_REGCOUNT = 0, ST_ZEROPIV = 1, ST_POSINERTIA = 2, ST_NONFINITE = 3, ST_NULLCOUNT = 4, ST_COUNT = 8 };

// Plain-pointer bundle passed by value to kernels.
struct LDLDev {
  const int* sn_first = nullptr;
  const long long* sn_rowptr = nullptr;
  const int* sn_rows = nullptr;
  const long long* child_ptr = nullptr;
  const int* child_list = nullptr;
  const int* rel = nullptr;  // indexed like sn_rows
  const long long* panel_off = nullptr;
  const long long* upd_off = nullptr;
  const long long* asm_ptr = nullptr;
  const int* asm_src = nullptr;
  const long long* asm_dst = nullptr;
  const int* level_tasks = nullptr;   // fronts of tree level 0 in the order of the launch plan (LaunchSeg)
  // small children of big fronts: (src,dst) entries sorted by dst, per big front (panel) and per update tile; a factor
  // task's range is in its record
  const int *sc_panel_src = nullptr, *sc_panel_dst = nullptr;
  const int *sc_tile_src = nullptr, *sc_tile_dst = nullptr;
  const int* gat_ptr = nullptr;       // solves: per front slot, CSR of contributing child update-vector entries
  const int* gat_src = nullptr;
  const int* perm = nullptr;
  const signed char* dsigns = nullptr;  // permuted order
  double* vals = nullptr;               // KKT values, caller's CSC order
  double* L = nullptr;                  // dense panels
  double* U = nullptr;                  // update-matrix arena
  double* D = nullptr;
  double* Dinv = nullptr;
  double* u = nullptr;                  // per-front update vectors for the solves
  int* status = nullptr;
  double reg_eps = 1e-13, reg_delta = 2e-7;
  int reg_enable = 1;
  // null pivots (cldl_set_null_pivot_tol): a pivot with |d| <= null_tol is stored as D = 1/D = 0 and marked; 0 = off.
  // Last in the struct, so that the kernels that never read them keep their parameter offsets.
  double null_tol = 0.0;
  unsigned char* nullmark = nullptr;    // [n] permuted order, 1 at the null pivots; cleared by every refactor with null_tol > 0
};

// dataflow factorisation plan (see k_factor_df in ldl.cu)
struct DFFactor {
  int ntask = 0;
  const int4* tasks = nullptr;      // 4 x int4 per task: DFTask
  const DFChildRec* recs = nullptr;
  int* pend = nullptr;              // [nsup] children still running
  int* diag_done = nullptr;         // [nsup]
  int* rows_left = nullptr;         // [nsup]
  int* tiles_left = nullptr;        // [nsup]
  int* qhead = nullptr;
  const int* parent = nullptr;
  const int* big_pos = nullptr;     // [nsup] position in the big-front list or -1
  const int* tile_base = nullptr;   // [nsup] first global tile id of the front or -1
  unsigned long long* trace = nullptr;  // optional [ntask][4]: grab, ready, end (globaltimer ns), smid
};

// selected-inversion plan on the device (see k_selinv in ldl_selinv.cuh, SelinvPlan in ldl_plan.h)
struct SIPlan {
  int ntask = 0;
  const int4* tasks = nullptr;      // 3 x int4 per task: SITask
  const long long* col = nullptr;   // indexed like sn_rows
  const long long* seg = nullptr;
  const int* segpos = nullptr;
  int* rows_left = nullptr;         // [nsup] row tasks still running
  int* done = nullptr;              // [nsup] 1 when the front's Z panel is complete
  int* qhead = nullptr;
  double* Z = nullptr;              // panels of (K + E)^-1, laid out like the factor's
};


// the level-0 fronts the plain leaf kernels solve: single-column, other narrow, wide
struct SVLeaves {
  const int *l1 = nullptr, *ln = nullptr, *lw = nullptr;
  int n1 = 0, nn = 0, nw = 0;
};

// one direction of a pruned solve on the device: the queue, its leaves and (forward) the closure with its task pairs
struct SparseSide {
  SVPlan q;
  SVLeaves lv;
  bool pruned = false;
  const int* reached = nullptr;
  const int* pairs = nullptr;
  int nreached = 0, npairs = 0;
};

class LDLObject {
 public:
  DevOwner own;                     // every stream, event and buffer below
  ~LDLObject() { release(); }
  // triangular solves (ldl_solve.cuh): task queue, counters, level-0 leaf lists
  SVPlan sv;
  int *d_sv_init = nullptr, *d_sv_cnt = nullptr, *d_sv_leaf1 = nullptr, *d_sv_leafn = nullptr, *d_sv_leafw = nullptr;
  size_t sv_ninit = 0, sv_nzero = 0, sv_smem[2] = {0, 0};
  int sv_cap = 0, sv_nwide = 0, sv_nleaf1 = 0, sv_nleafn = 0, sv_nleafw = 0, sv_leafw_nrmax = 0, sv_leafw_grid = 1, sv_ntask_owned = 0;
  std::vector<SVTask> h_sv_tasks;
  SolvePlan sv_host;                // the full solve plan on the host, gather lists dropped (pruned plans derive from it)
  int sv_configure();
  int sv_occupancy();
  int sv_reset();
  void sv_sweep(bool fwd, int nrhs, const SVPlan& q, const SVRhs& r);
  SVLeaves sv_leaf_lists() const { return SVLeaves{d_sv_leaf1, d_sv_leafn, d_sv_leafw, sv_nleaf1, sv_nleafn, sv_nleafw}; }
  void sv_leaves(bool fwd, int nrhs, const SVRhs& r, const SVLeaves& lv);
  // pruned solves (cldl_solve_sparse, cldl_inverse_entries; ldl_sparse.cuh): set up by the first call
  SolvePrune sp_prune;
  PrunedPlan sp_plan[2];            // forward, backward
  bool sp_ready = false;
  int* d_sp_cnt = nullptr;          // counters, laid out like d_sv_cnt
  int* d_sp_f2t = nullptr;          // [nsup] front2task of the pruned forward plan
  unsigned char* d_sp_mark = nullptr;   // [nsup] fronts of the pruned forward set
  double* d_sp_bpart = nullptr;     // like sv.bpart
  char* d_sp_stage = nullptr;       // the per-call payload (plans, index lists, values) on the device
  char* h_sp_stage[2] = {nullptr, nullptr};   // the same, pinned, used in turn; sp_ev[k] follows the copy out of [k]
  cudaEvent_t sp_ev[2] = {nullptr, nullptr};
  size_t sp_stage_cap = 0;
  int sp_turn = 0;
  double* d_sp_out = nullptr;       // host-pointer calls: the wanted entries
  size_t sp_out_cap = 0;
  std::vector<unsigned> sp_seen;    // [n] duplicate check of b's indices (stamps)
  unsigned sp_seen_epoch = 0;
  std::vector<char> sp_payload;
  double sp_plan_ms = 0.0;          // host time of the last call's plan building
  long long sp_work = 0, sp_reached[2] = {0, 0}, sp_entries[2] = {0, 0};   // the last call's counts (diagnostics)
  int sparse_setup();
  int sparse_stage(size_t need_out);
  int sparse_sweeps(int nrhs, const SparseSide& F, const SparseSide& B, const SVRhs& r);
  SparseSide sparse_full_side() const;
  int solve_sparse_async(uint64_t nb, const uint64_t* b_index, const double* b_values, bool b_dev, uint64_t nx,
                         const uint64_t* x_index, double* x_values, bool x_dev);
  int inverse_entries(uint64_t nnz, const uint64_t* rows, const uint64_t* cols, double* out);
  // rank-k updates (cldl_updown, ldl_updown.cuh): the payload goes through the pruned solves' stage; the rest is set
  // up by the first call
  bool ud_ready = false;
  std::vector<int> ud_cp, ud_row, ud_src;   // the caller's pattern per column, rows ascending, with CSC positions
  std::vector<unsigned> ud_seen;         // [n] duplicate check of a column's rows (stamps)
  unsigned ud_seen_epoch = 0;
  double* d_ud_w = nullptr;              // [UD_PASS n] permuted work vectors
  double* d_ud_pb = nullptr;             // [ud_slots][CB_PB_MAXNS][UD_PASS] (p, beta)
  int* d_ud_stat = nullptr;              // the last call's flags and sign-change count (UD_FAIL, ...)
  int* h_ud_stat = nullptr;              // the same, pinned
  int ud_slots = 0, ud_grid = 0;
  bool ud_last = false;                  // the last factor change enqueued was an update: sync_status reads h_ud_stat
  uint64_t ud_pos_base = 0;              // positive_inertia before it
  UpdownPlan ud_plan;
  double ud_plan_ms = 0.0;               // host time of the last call's checks and plans
  long long ud_passes = 0, ud_fronts = 0, ud_tasks = 0, ud_entries = 0, ud_work = 0;   // its counts (diagnostics)
  int updown_setup();
  int updown_async(uint64_t k, const uint64_t* w_colptr, const uint64_t* w_rowidx, const double* w_values, bool w_dev,
                   const double* sigma);
  int updown_verdict();
  // the factor's parts (cldl_solve_part, cldl_mul_part, cldl_get_factor_csc, cldl_sample; ldl_parts.cuh): work vectors
  // allocated by the first call, row lists and column pointers (FactorParts in ldl_plan.h) by the first that needs them
  double* d_pt_work = nullptr;           // [3 n]: the sweeps' caller-order store, two temporaries
  long long *d_pt_rptr = nullptr, *d_pt_rpos = nullptr;
  unsigned long long* d_pt_colptr = nullptr;
  uint64_t pt_nnz = 0;
  int parts_check();
  int parts_setup(bool lists);
  void pt_lmul(double* d_y, const double* d_x);    // y = L x (x and y distinct, permuted order)
  void pt_ltmul(double* d_y, const double* d_x);   // y = L^T x
  void pt_diag(int which, double* d_y, const double* d_x);   // y = s(a) x per entry (k_pt_diag): which 0 1/D, 1 D, 2 sqrt|1/D|, 3 sqrt|D|
  int solve_part_async(int sys, double* d_x, const double* d_b);
  int mul_part_async(int sys, double* d_y, const double* d_x);
  int factor_csc_async(unsigned long long* d_cp, unsigned long long* d_ri, double* d_Lx, double* d_D, double* d_Dinv);
  int sample_async(int form, uint64_t k, uint64_t seed, uint64_t offset, const double* d_mu, double* d_X, double* d_Z);
  DFFactor dff;
  int *d_dff_init = nullptr, *d_dff_cnt = nullptr;
  std::vector<DFTask> h_dff_tasks;
  int dff_grid = 0;
  size_t dff_nsup4 = 0;
  int sv_grid = 0;                  // CTAs of a sweep kernel (as many as can be co-resident)
  bool use_dataflow = true;
  int n = 0;
  int64_t nnzA = 0;
  int device = 0;
  cldl_opts opts{};
  Symbolic S;
  LDLDev dev;
  std::vector<LaunchSeg> plan;
  std::thread big_alloc;                 // init: allocates the factor storage beside the plan building
  int big_alloc_rc = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t stream_a = nullptr, stream_b = nullptr;   // side streams of the narrow-leaf solve kernels
  cudaEvent_t ev_leaf[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int* h_status = nullptr;
  double* d_xp = nullptr;  // permuted work vector
  double* d_bx = nullptr;  // staging for host-pointer solve: [b ; x]
  int* d_tmp_idx = nullptr;
  double* d_tmp_val = nullptr;
  signed char* d_tmp_sgn = nullptr;
  size_t tmp_cap = 0;
  std::vector<int> h_idx;
  bool factored = false;
  bool factor_ok = false;                // the last refactor's status was collected and it returned 1
  uint64_t regularize_count = 0, positive_inertia = 0;
  // null pivots (cldl_set_null_pivot_tol, cldl_null_pivots, cldl_null_space): dev.null_tol / dev.nullmark, the last
  // refactor's count, and the null-space sweeps' 1/D (ones) and scalars, allocated by their first call
  uint64_t null_count = 0;
  double* d_ns_ones = nullptr;           // [n]
  double* d_ns_stat = nullptr;           // [2 r + 1]: ||v_k||_inf, ||K v_k||_inf per column, then ||K||_inf
  size_t ns_stat_cap = 0;
  int set_null_tol(double tol);
  int null_positions(std::vector<int>& pos);   // the null pivots' permuted positions, ascending (synchronises)
  int null_space(uint64_t r, double* V, bool v_dev, double* resid);
  // selected inversion: plan, Z panels and counters, allocated by the first call
  SIPlan si;
  long long* d_si_pos = nullptr;         // [nnzA] caller entry -> offset in si.Z
  int *d_si_init = nullptr, *d_si_cnt = nullptr;
  double* d_si_out = nullptr;            // [nnzA] staging of the host-pointer call
  int si_grid = 0;
  int selinv_setup();
  int selected_inverse_async(double* d_out);
  // log-determinant and adjoint solves (cldl_logdet, cldl_adjoint_solve): buffers allocated by the first call of each
  std::vector<int> h_colptr, h_rowval;   // the caller's pattern, int32 CSC (kept by init for the pattern gradient)
  int *d_adj_cp = nullptr, *d_adj_rv = nullptr;   // the same on the device, uploaded by the first adjoint call
  double* d_adj_buf = nullptr;           // [3 n + nnzA] staging of the host-pointer adjoint: g, x, gb, gvals
  double* d_ld_ws = nullptr;             // [RED_BLOCKS + 1] partial sums of the log-determinant, then its value
  unsigned* d_ld_cnt = nullptr;          // the reduction's block counter
  int logdet(double* logabsdet, int32_t* sign);
  int adjoint_async(const double* d_g, const double* d_x, double* d_gb, double* d_gvals);
  // iterative refinement and error analysis (cldl_solve_refined, ldl_refine.cuh): allocated by the first call
  int *d_rf_rowptr = nullptr, *d_rf_col = nullptr, *d_rf_src = nullptr;   // K's mirrored pattern, CSR, src into vals
  double* d_rf_work = nullptr;           // [RF_NVEC n] work vectors
  double* d_rf_ws = nullptr;             // [8 RED_BLOCKS] reduction partials, then [RF_NS] scalars
  unsigned* d_rf_cnt = nullptr;          // the reductions' block counter
  double* h_rf = nullptr;                // [RF_NS] pinned copy of the scalars
  int refine_setup();
  int refine_analyse(const double* d_xv, const double* d_b, bool first);
  int condest(int which, const double* d_b, double* est, uint32_t* solves);
  int solve_refined(double* d_x, const double* d_b, const cldl_refine_opts& o, cldl_refine_info* info);
  // eigenvalues nearest a shift (cldl_eigsh; ldl_eig.cpp, ldl_eig.cuh): buffers allocated and freed by each call
  int eigsh(double sigma, const double* M, bool m_dev, uint64_t nev, const cldl_eig_opts& o, double* evals, double* X,
            bool x_dev, double* resid, cldl_eig_info* info);
  // FGMRES preconditioned by the factor (cldl_solve_gmres; ldl_krylov.cpp): basis buffers allocated and freed by each
  // call, the refined solves' mirrored pattern and work vectors shared
  int solve_gmres(double* d_x, const double* d_b, const cldl_gmres_opts& o, cldl_gmres_info* info);
  // Schur complement handle (cldl_create_schur; SchurPlan in ldl_plan.h): B's fronts are factored, S's never
  std::vector<int> schur_set;            // non-empty: a Schur complement handle
  bool schur = false;
  bool schur_fwd = false;                // a condensation since the last expansion / refactor left the forward state
  int schur_k = 0, schur_first = 0;
  SVPlan sv_bwd;                         // the B-only backward queue (counters shared with sv)
  int *d_sc_spos = nullptr, *d_sc_kss_src = nullptr, *d_sc_rec_ptr = nullptr;
  long long *d_sc_kss_ptr = nullptr, *d_sc_kss_dst = nullptr;
  SchurRec* d_sc_recs = nullptr;
  double* d_sc_out = nullptr;            // [k * k] the complement of the last refactor
  double* d_sc_vec = nullptr;            // [2 k] staging of the host-pointer partial solves
  int schur_setup(const SolvePlan& sp);
  int schur_reduce_async(double* d_wS, const double* d_b);
  int schur_expand_async(double* d_x, const double* d_xS);
  // ---- one factorisation on several GPUs: this object is one rank (see ShardPlan in symbolic.h) ----
  int shard_nranks = 1, shard_rank = 0;
  ShardPlan shard;                       // owner[front] = rank or -1 (replicated top)
  std::vector<std::vector<int>> shard_cut;   // per rank: its cut roots (fronts whose parent is in the top part)
  std::vector<std::vector<int>> shard_xidx;  // per rank: caller-order indices of the x entries it computes
  std::vector<int*> d_shard_xidx;            // the same lists on the device
  std::vector<long long*> d_shard_segs[2];   // per what (0 update matrices, 1 update vectors) and rank: (arena offset, buffer offset, length) of its cut roots
  std::vector<int> shard_nsegs[2];
  int shard_seglist(int what, int rank, const long long** d_out, int* nseg);
  int dff_ntask_owned = 0;               // tasks of the owned phase (they come first in the queue)
  int h_phase_start[2] = {0, 0};         // pinned-lifetime host copies of the queue heads the top phases start from
  uint64_t shard_count_owned[2] = {0, 0};    // regularize_count / positive_inertia of the owned phase
  bool sharded() const { return shard_nranks > 1; }
  int refactor_phase_async(int phase);   // 0: owned subtrees, 1: top part (after the cut roots' update matrices arrived)
  int solve_phase_async(double* d_x, const double* d_b, int phase);   // 0: permute + forward owned, 1: forward top + backward
  // what: 0 update matrices of the cut roots (per refactor), 1 their update vectors (per solve), 2 x entries
  uint64_t shard_count(int what, int rank) const;
  int shard_pack(int what, double* d_buf, const double* d_x);
  int shard_unpack(int what, int rank, const double* d_buf, double* d_x);
  // transport (all-gather between ranks) and the self-driven sharded refactor / solve built on it
  cldl_allgather_fn transport = nullptr;
  void* nccl_comm = nullptr;             // own NCCL communicator: exchanges are stream-ordered (set_nccl)
  unsigned long long n_collectives = 0;  // NCCL all-gathers issued by this handle
  bool has_transport() const { return transport != nullptr || nccl_comm != nullptr; }
  int set_nccl(const char* libpath, const unsigned char* id128, int nranks, int rank);
  void* transport_ctx = nullptr;
  double *d_xsend = nullptr, *d_xrecv = nullptr;
  size_t xbuf_cap = 0;
  int exchange(int what, double* d_x);
  // the communicator's ncclAllGather / ncclGetErrorString, taken by set_nccl from the NCCL library it loaded
  int (*nccl_allgather)(const void*, void*, size_t, int, ncclComm*, cudaStream_t) = nullptr;
  const char* (*nccl_error)(int) = nullptr;
  // one all-gather of `cnt` doubles per rank between device buffers through the installed transport; defined here
  // rather than in ldl.cu because the interior-point driver uses it too (the sharded termination-callback verdicts)
  int allgather(const double* d_send, double* d_recv, uint64_t cnt) {
    if (nccl_comm) {      // stream-ordered: whatever follows on `stream` simply follows the collective
      const int r = nccl_allgather(d_send, d_recv, (size_t)cnt, /* ncclFloat64 */ 8, (ncclComm*)nccl_comm, stream);
      if (r != 0) { std::fprintf(stderr, "[clarabel_b200] ncclAllGather: %s\n", nccl_error ? nccl_error(r) : "error"); return CLDL_E_CUDA; }
      n_collectives++;
      return CLDL_OK;
    }
    if (cudaStreamSynchronize(stream) != cudaSuccess) return CLDL_E_CUDA;
    return transport(transport_ctx, d_send, d_recv, cnt) != 0 ? CLDL_E_CUDA : CLDL_OK;
  }
  int refactor_sharded();
  int solve_sharded(double* d_x, const double* d_b);

  // a Schur complement handle sets schur_set (caller indices, in output order) before init
  int init(int n, const int64_t* Ap, const int32_t* Ai, const double* Ax, const int8_t* dsigns,
           const cldl_opts& o, const int* perm_in);
  void release();        // what is not the owner's: the NCCL communicator (the emulated build: its dense factor)
  int refactor_level0();   // the start of every refactor: counters reset, tree level 0 factored
  int refactor_async();
  int sync_status();
  // one right-hand side, or two swept together (d_x1 / d_b1 non-null): the panels are read once for both
  int solve_async(double* d_x, const double* d_b, double* d_x1 = nullptr, const double* d_b1 = nullptr);
  double *d_xp2 = nullptr, *d_u2 = nullptr;   // work vectors of the second right-hand side
  int ensure_tmp(size_t len);
  int stage_index(const uint64_t* index, uint64_t len);
};

}  // namespace cb
