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

#define CB_MAX_PANEL 128
#define CB_PB_LD 66        /* padded leading dimension of the pivot block in shared memory */

namespace cb {

struct ncclComm;   // NCCL's communicator, opaque (ldl.cu loads NCCL with dlopen)

enum { ST_REGCOUNT = 0, ST_ZEROPIV = 1, ST_POSINERTIA = 2, ST_NONFINITE = 3, ST_COUNT = 8 };

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


class LDLObject {
 public:
  // triangular solves (ldl_solve.cuh): task queue, counters, level-0 leaf lists
  SVPlan sv;
  int *d_sv_init = nullptr, *d_sv_cnt = nullptr, *d_sv_leaf1 = nullptr, *d_sv_leafn = nullptr, *d_sv_leafw = nullptr;
  size_t sv_ninit = 0, sv_nzero = 0, sv_smem[2] = {0, 0};
  int sv_cap = 0, sv_nwide = 0, sv_nleaf1 = 0, sv_nleafn = 0, sv_nleafw = 0, sv_leafw_nrmax = 0, sv_leafw_grid = 1, sv_ntask_owned = 0;
  std::vector<SVTask> h_sv_tasks;
  int sv_configure();
  int sv_occupancy();
  int sv_reset();
  void sv_sweep(bool fwd, int nrhs, const SVPlan& q, const SVRhs& r);
  void sv_leaves(bool fwd, int nrhs, const SVRhs& r);
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
  void release();
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
