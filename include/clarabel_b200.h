/*
 * clarabel_b200.h -- C-ABI of the GPU-native (H100, sm_90a) KKT backend for Clarabel-style
 * interior point solvers.  Plain pointers and sizes only; no C++/torch types.
 *
 * LEVEL 1  (cldl_*)  replaces the reference's `DirectLDLSolver` plugin trait
 *   /root/reference/src/solver/core/kktsolvers/direct/quasidef/mod.rs:14-26
 *   and its qdldl adapter .../ldlsolvers/qdldl.rs:19-107.  One handle = one
 *   factorisation object living on one GPU.
 *
 * Conventions (follow the reference's existing C-ABI, src/julia/interface.rs):
 *   - opaque handle + explicit destroy;
 *   - index type is uint64_t (Rust `usize`);
 *   - the two trait methods that return `bool` return 1 (true) / 0 (false);
 *     everything else returns 0 on success and a negative CLDL_E_* code on
 *     failure.  Nothing unwinds or aborts.
 *   - every entry point selects the handle's device itself (cudaSetDevice),
 *     so a handle may be used from a thread other than its creator
 *     (directldlkktsolver.rs:13-16: the trait object is Send + Sync);
 *   - `_dev` twins take DEVICE pointers (same meaning otherwise) and enqueue
 *     on the handle's stream without synchronising.
 */
#ifndef CLARABEL_B200_H
#define CLARABEL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cldl_handle cldl_t;

enum {
  CLDL_OK = 0,
  CLDL_E_DIM = -1,          /* QDLDLError::IncompatibleDimension */
  CLDL_E_EMPTY_COLUMN = -2, /* QDLDLError::EmptyColumn          */
  CLDL_E_NOT_TRIU = -3,     /* QDLDLError::NotUpperTriangular   */
  CLDL_E_ZERO_PIVOT = -4,   /* QDLDLError::ZeroPivot            */
  CLDL_E_BAD_PERM = -5,     /* QDLDLError::InvalidPermutation   */
  CLDL_E_CUDA = -20,        /* no device / CUDA runtime failure */
  CLDL_E_ARG = -21,
  CLDL_E_NOT_FACTORED = -22 /* solve() before refactor(): the reference panics (qdldl.rs:118) */
};

enum { CLDL_ORDER_AMD = 1, CLDL_ORDER_ND = 2, CLDL_ORDER_BEST = 3 };

/* Options read at construction.  Mirrors the fields of CoreSettings that the
 * qdldl adapter forwards (ldlsolvers/qdldl.rs:35-42) plus device selection. */
typedef struct {
  double regularize_eps;    /* settings.dynamic_regularization_eps   (default 1e-13) */
  double regularize_delta;  /* settings.dynamic_regularization_delta (default 2e-7)  */
  int32_t regularize_enable;/* adapter always passes true (qdldl.rs:38)               */
  double amd_dense_scale;   /* 1.5 in the reference adapter (qdldl.rs:41)             */
  int32_t ordering;         /* CLDL_ORDER_*; ignored when a permutation is supplied   */
  int32_t device;           /* CUDA device ordinal                                    */
  int32_t max_panel;        /* 0 = default                                            */
  int32_t nd_leaf;          /* 0 = default                                            */
  /* one factorisation on several GPUs (SURVEY 8e): this handle is rank `shard_rank` of `shard_nranks`; it factors
   * and solves the subtrees it owns plus the replicated top of the assembly tree.  0 / 1 ranks = whole tree. */
  int32_t shard_nranks, shard_rank;
} cldl_opts;

/* LinearSolverInfo (kktsolvers/mod.rs:24-38) + factorisation counters
 * (qdldl.rs:104-112). */
typedef struct {
  char name[16];            /* "cudaldl" */
  uint32_t threads;         /* resident device threads used per launch wave; 0 = n/a */
  int32_t direct;           /* 1 */
  uint64_t nnzA;
  uint64_t nnzL;            /* entries of L the reference would report (simplicial count) */
  uint64_t nnzL_stored;     /* entries actually stored in dense supernodal panels */
  uint64_t regularize_count;
  uint64_t positive_inertia;
  uint64_t n_supernodes;
  uint64_t n_levels;
  double flops;             /* dense flops per numeric factorisation */
  int32_t ordering_used;    /* 0 = caller's permutation */
} cldl_info_t;

void cldl_default_opts(cldl_opts *o);

/* Constructor: DirectLDLSolver ctor signature of ldlsolvers/config.rs:19-20,
 * `fn(&CscMatrix<T>, &[i8] Dsigns, &CoreSettings<T>, Option<Vec<usize>> perm)`.
 * (colptr,rowval,nzval) is the n x n upper-triangular KKT matrix in CSC with a
 * structural entry on every diagonal.  Performs ordering + symbolic analysis on
 * the host and uploads the static maps; like the reference adapter it does NOT
 * produce numeric factors ("logical" factorisation) -- call cldl_refactor. */
int cldl_create(cldl_t **out, uint64_t n, const uint64_t *colptr, const uint64_t *rowval,
                const double *nzval, const int8_t *dsigns, const cldl_opts *opts,
                const uint64_t *perm_or_null);
void cldl_destroy(cldl_t *h);

/* DirectLDLSolver::update_values / scale_values / offset_values
 * (mod.rs:15-17, qdldl.rs:142-183).  `index` addresses entries of the
 * caller's nzval array. */
int cldl_update_values(cldl_t *h, const uint64_t *index, const double *values, uint64_t len);
int cldl_scale_values(cldl_t *h, const uint64_t *index, uint64_t len, double scale);
int cldl_offset_values(cldl_t *h, const uint64_t *index, uint64_t len, double offset,
                       const int8_t *signs);

/* DirectLDLSolver::refactor (mod.rs:19) -> bool: all reciprocal pivots finite
 * (ldlsolvers/qdldl.rs:99-106).  Returns 1/0, or CLDL_E_ZERO_PIVOT when an
 * exact zero pivot is met with regularisation disabled (qdldl.rs:527,656). */
int cldl_refactor(cldl_t *h);

/* DirectLDLSolver::solve (mod.rs:18): x <- K^{-1} b; b is left untouched
 * (ldlsolvers/qdldl.rs:93-97).  Host buffers of length n. */
int cldl_solve(cldl_t *h, double *x, const double *b);

void cldl_info(const cldl_t *h, cldl_info_t *info);

/* The permutation actually used (new k <- old perm[k]); the parity tests hand
 * it to the CPU oracle so both sides eliminate in the same order. */
int cldl_get_perm(const cldl_t *h, uint64_t *perm_out);

/* The stored factor after the last refactor, for inspection and tests: the front panels as the solves read them
 * (info.nnzL_stored doubles, front after front in supernode order; pivot blocks wider than 8 columns hold L11^-1 in
 * their strictly lower triangle), the pivots D and their reciprocals (n doubles each, permuted order).  On a sharded
 * handle the fronts of other ranks are not this handle's and hold no values.  Synchronises the handle's stream. */
int cldl_get_factor(const cldl_t *h, double *L_out, double *D_out, double *Dinv_out);

/* Selected inversion: the entries of (K + E)^-1 at every stored entry of the upper triangle passed to cldl_create,
 * diagonal included, in the caller's CSC order (nnzA doubles).  K + E is the matrix the last refactor factored: E is
 * the dynamic regularisation it applied (cldl_info.regularize_count pivots), so with regularisation the result is the
 * inverse of the regularised matrix, not of K.  Computed on the device in one pass over the factor from the root of
 * the assembly tree to its leaves (about the work of one refactor).
 *   - Valid after a refactor that returned 1 (cldl_refactor, or cldl_refactor_dev followed by cldl_sync_status).
 *     Before any refactor, or after one that returned 0 or an error, the call returns CLDL_E_NOT_FACTORED.
 *   - On a sharded handle the call returns CLDL_E_ARG.
 *   - The first call builds the plan and allocates its device memory: panels of the inverse (info.nnzL_stored
 *     doubles, plus alignment), the gather maps and the task queue.  cldl_destroy frees them.
 *   - The factor, D, 1/D and every later solve are left bit for bit unchanged.
 * cldl_selected_inverse writes a host buffer and synchronises; the _dev form writes a device buffer and is only
 * enqueued on the handle's stream (cldl_stream). */
int cldl_selected_inverse(cldl_t *h, double *nzval_out);
int cldl_selected_inverse_dev(cldl_t *h, double *d_nzval_out);

/* Schur complement: a handle over the same matrix as cldl_create plus a Schur set S of nschur caller indices
 * (schur_idx, any order, 1 <= nschur < n: a set of all n indices is refused).  The rest, B, is eliminated and S never
 * is: B is ordered first (by opts->ordering on the subgraph B induces, or by perm_or_null, whose last nschur entries
 * must be exactly S, else CLDL_E_BAD_PERM), then S.  Every refactor factors B alone and assembles
 *     Sc = K_SS - K_SB K_BB^-1 K_BS
 * on the device: nschur x nschur doubles, column-major, both triangles, rows and columns in the order of schur_idx.
 * With dynamic regularisation, Sc is the complement of K + E_B: E_B the regularisation of B's pivots, the only pivots
 * factored (cldl_info.regularize_count / positive_inertia and the refactor's verdict cover B alone).  Value updates
 * reach Sc at the next refactor.  Every sum has a fixed order: repeated refactors give the same bits.
 *   - cldl_schur_reduce (condensation): w_S = b_S - K_SB K_BB^-1 b_B, nschur doubles in the order of schur_idx, from b
 *     (n doubles, caller's order).
 *   - cldl_schur_expand (expansion): given x_S (schur_idx order) solving Sc x_S = w_S, writes the whole x (n doubles,
 *     x_B = K_BB^-1 (b_B - K_BS x_S) and x_S) for the b of the last condensation, whose forward state it consumes:
 *     every expansion needs a condensation after the last refactor and after the previous expansion, else CLDL_E_ARG.
 *   - Refusals: an empty, duplicate or out-of-range Schur set, or opts->shard_nranks > 1, at create: CLDL_E_ARG; a set
 *     whose complement the device cannot allocate: CLDL_E_ARG.  The Schur calls before a refactor that returned 1:
 *     CLDL_E_NOT_FACTORED.  cldl_solve(_dev), cldl_selected_inverse(_dev) and the shard entry points on a Schur handle,
 *     and the Schur calls on any other handle: CLDL_E_ARG.
 * The host-pointer forms synchronise; the _dev forms are only enqueued on the handle's stream (cldl_stream). */
int cldl_create_schur(cldl_t **out, uint64_t n, const uint64_t *colptr, const uint64_t *rowval, const double *nzval,
                      const int8_t *dsigns, const cldl_opts *opts, const uint64_t *perm_or_null, uint64_t nschur,
                      const uint64_t *schur_idx);
int cldl_schur_complement(cldl_t *h, double *out);
int cldl_schur_complement_dev(cldl_t *h, double *d_out);
int cldl_schur_reduce(cldl_t *h, double *wS, const double *b);
int cldl_schur_reduce_dev(cldl_t *h, double *d_wS, const double *d_b);
int cldl_schur_expand(cldl_t *h, double *x, const double *xS);
int cldl_schur_expand_dev(cldl_t *h, double *d_x, const double *d_xS);

/* Log-determinant: log|det(K + E)| and its sign (-1)^(number of negative pivots), from the pivots D of the last refactor.
 * E is the dynamic regularisation that refactor applied (cldl_info.regularize_count pivots), so with regularisation
 * the result is the determinant of the regularised matrix, not of K.  One device sum of log|d_k| in a fixed order,
 * then an 8-byte read; the sign comes from the refactor's positive_inertia count.
 *   - Valid after a refactor that returned 1 (cldl_refactor, or cldl_refactor_dev followed by cldl_sync_status);
 *     otherwise CLDL_E_NOT_FACTORED.
 *   - On a Schur handle: log|det(K_BB + E_B)|, over B's pivots only (the first n - nschur in the permuted order),
 *     which are the pivots the verdict and the counters cover.
 *   - On a sharded handle: CLDL_E_ARG.
 *   - Synchronises the handle's stream.  The first call allocates a few kilobytes of reduction workspace. */
int cldl_logdet(cldl_t *h, double *logabsdet, int32_t *sign);

/* Adjoint solve: the adjoint of x = K^-1 b.  For an output gradient g (n doubles):
 *     gb = (K + E)^-1 g
 * and, when gvals is not NULL, the gradient of <g, x> with respect to the stored values of the upper triangle passed
 * to cldl_create (caller's CSC order, nnzA doubles):
 *     gvals = -(gb_i x_j + x_i gb_j) off the diagonal, -gb_i x_i on it,
 * where x is the solution being differentiated (cldl_solve(b) on the current factor).  NULL gvals computes gb only,
 * and x may then be NULL.  E is the refactor's dynamic regularisation, as for cldl_logdet: with
 * regularize_count > 0 these are the derivatives of the solve with K + E.  gb is the solve's launch sequence on g; the
 * gradient is one kernel with a warp per column.
 *   - Valid after a refactor that returned 1; otherwise CLDL_E_NOT_FACTORED.
 *   - On a Schur handle (no cldl_solve there) and on a sharded handle: CLDL_E_ARG.
 *   - The first call with gvals uploads the caller's pattern as int32 colptr / rowval ((n + 1 + nnzA) * 4 bytes); the
 *     first host-pointer call allocates (3 n + nnzA) doubles of staging.  cldl_destroy frees them.
 *   - No floating-point atomics: repeated calls give the same bits.
 * For both calls the factor, D, 1/D and every later solve are left bit for bit unchanged.  cldl_adjoint_solve reads
 * and writes host buffers and synchronises; the _dev form takes device buffers and is only enqueued on the handle's
 * stream (cldl_stream). */
int cldl_adjoint_solve(cldl_t *h, const double *g, const double *x, double *gb, double *gvals);
int cldl_adjoint_solve_dev(cldl_t *h, const double *d_g, const double *d_x, double *d_gb, double *d_gvals);

/* ---- device-pointer twins (asynchronous on the handle's stream) ---- */
int cldl_update_values_dev(cldl_t *h, const int32_t *d_index, const double *d_values, uint64_t len);
int cldl_set_values_dev(cldl_t *h, const double *d_nzval);   /* whole array, caller order */
int cldl_refactor_dev(cldl_t *h);                            /* enqueue only; status via cldl_sync_status */
int cldl_solve_dev(cldl_t *h, double *d_x, const double *d_b);
int cldl_sync_status(cldl_t *h);                             /* sync + refactor verdict (1/0/neg) */
void *cldl_stream(cldl_t *h);                                /* cudaStream_t */
double *cldl_values_dev(cldl_t *h);                          /* device copy of nzval, caller order */

/* ---- one factorisation on several GPUs (cldl_opts.shard_nranks > 1; SURVEY 8e) ----
 * Every rank creates its handle from the same matrix with its own shard_rank; the symbolic analysis and the
 * subtree-to-rank plan are deterministic, so all ranks agree on them.  A rank factors / solves the subtrees it owns
 * and the replicated top of the assembly tree; between the two phases the caller moves the packed contributions of
 * every rank to every other rank (NCCL all-gather / broadcast over NVLink, or plain copies when the handles share a
 * device) -- the library only packs and unpacks DEVICE buffers:
 *   what = 0  update matrices of the rank's cut roots   (between the refactor phases)
 *   what = 1  update vectors of the rank's cut roots    (between the solve phases)
 *   what = 2  the x entries the rank computed           (after solve phase 1: the all-gather of the solution)
 * cldl_shard_count(h, what, r) = doubles rank r contributes.  cldl_refactor / cldl_solve refuse on such a handle.
 *   refactor:  phase 0 on every rank -> pack(0) -> exchange -> unpack(0, r) for r != me -> phase 1 -> cldl_sync_status
 *   solve:     phase 0 -> pack(1) -> exchange -> unpack(1, r) -> phase 1 -> pack(2, x) -> exchange -> unpack(2, r, x)
 * cldl_shard_counts: {regularize_count, positive_inertia} of the owned phase, then of owned + top (after
 * cldl_sync_status); the global count is sum_r owned_r + (total_0 - owned_0). */
int cldl_shard_refactor_phase_dev(cldl_t *h, int phase);
int cldl_shard_solve_phase_dev(cldl_t *h, double *d_x, const double *d_b, int phase);
uint64_t cldl_shard_count(const cldl_t *h, int what, int rank);
int cldl_shard_pack_dev(cldl_t *h, int what, double *d_buf, const double *d_x);
int cldl_shard_unpack_dev(cldl_t *h, int what, int rank, const double *d_buf, double *d_x);
int cldl_shard_counts(const cldl_t *h, uint64_t *out4);
/* Transport for a sharded handle: an all-gather of `count` doubles per rank between DEVICE buffers (d_send: count
 * doubles of this rank; d_recv: nranks * count doubles, rank r's block at r * count).  It is called from the host
 * between the phases, after the send buffer is complete, and must return once d_recv is usable (0 = ok).  With a
 * transport installed, cldl_refactor(_dev) / cldl_solve(_dev) and the whole cipm_* driver run their phases and
 * exchanges themselves (contributions are padded to the largest one); every rank then executes the same interior
 * point iterations on identical data and only the factorisation / triangular solves are split. */
typedef int (*cldl_allgather_fn)(void *ctx, const double *d_send, double *d_recv, uint64_t count);
int cldl_set_transport(cldl_t *h, cldl_allgather_fn fn, void *ctx);
/* The same exchanges as stream-ordered NCCL all-gathers issued by the library itself on the handle's stream (no host
 * synchronisation between pack, collective and unpack).  The library is not linked against NCCL: `libpath` names the
 * libnccl.so.2 the calling process has loaded already (two NCCL builds in one process do not mix; NULL = the loader's
 * default).  Rank 0 draws the 128-byte unique id and the binding broadcasts it; cldl_set_nccl is collective (it
 * calls ncclCommInitRank).  Takes precedence over a callback transport. */
int cldl_nccl_unique_id(const char *libpath, unsigned char *id128);
int cldl_set_nccl(cldl_t *h, const char *libpath, const unsigned char *id128, int nranks, int rank);
int cldl_copy_dev(void *d_dst, const void *d_src, uint64_t bytes);   /* device-to-device copy, for transports in bindings */

/* timing helper for benches: runs `reps` refactors (or solves) back to back
 * on the device and returns the average milliseconds measured with CUDA
 * events on the handle's stream. */
double cldl_time_refactor_ms(cldl_t *h, int reps);
double cldl_time_solve_ms(cldl_t *h, int reps);


/* ======================================================================
 * LEVEL 2  (cipm_* / ckkt_* / ccone_*)  device-resident KKT system, cone
 * engine and interior-point driver.  Replaces, for the symmetric cones
 * (Zero / Nonnegative / SecondOrder):
 *   trait KKTSolver      src/solver/core/kktsolvers/mod.rs:7-19
 *     + DirectLDLKKTSolver .../direct/quasidef/directldlkktsolver.rs:18-405
 *   trait Cone / CompositeCone  src/solver/core/cones/mod.rs:42-154,
 *                               compositecone.rs:197-352
 *   DefaultSolver::new / IPSolver::solve
 *                        src/solver/implementations/default/solver.rs:57-126,
 *                        src/solver/core/solver.rs:224-465
 * One handle owns the equilibrated problem, the cone set, the KKT matrix and
 * its LDL^T on one GPU.  Vectors never leave the device during a solve.
 * ==================================================================== */
typedef struct cipm_handle cipm_t;

/* SupportedConeT tags (supportedcone.rs:17-52).  ExponentialConeT() and PowerConeT(alpha) occupy 3 rows each;
 * the exponent of a power cone travels in cone_params (cipm_create_ex); GenPowerConeT(alpha, dim2) has
 * cone_dims = len(alpha) and its dim2 / exponents in the two extra arrays of cipm_create_gp.
 * PSDTriangleConeT(n): cone_dims = n (matrix dimension, n (n + 1) / 2 rows); n <= 128, larger cones are refused. */
enum { CIPM_CONE_ZERO = 0, CIPM_CONE_NONNEG = 1, CIPM_CONE_SOC = 2, CIPM_CONE_PSD = 3, CIPM_CONE_EXP = 4,
       CIPM_CONE_POW = 5, CIPM_CONE_GENPOW = 6 };
/* ScalingStrategy (src/solver/core/cones/mod.rs) */
enum { CIPM_SCALING_PRIMAL_DUAL = 0, CIPM_SCALING_DUAL = 1 };

/* SolverStatus (src/solver/core/traits.rs / default/info.rs) */
enum { CIPM_UNSOLVED = 0, CIPM_SOLVED, CIPM_PRIMAL_INFEASIBLE, CIPM_DUAL_INFEASIBLE, CIPM_ALMOST_SOLVED,
       CIPM_ALMOST_PRIMAL_INFEASIBLE, CIPM_ALMOST_DUAL_INFEASIBLE, CIPM_MAX_ITERATIONS, CIPM_MAX_TIME,
       CIPM_NUMERICAL_ERROR, CIPM_INSUFFICIENT_PROGRESS,
       CIPM_CALLBACK_TERMINATED   /* the termination callback asked to stop (SolverStatus::CallbackTerminated) */ };

/* The fields of DefaultSettings the path reads (default/settings.rs:30-193),
 * same names, same defaults (cipm_default_settings). */
typedef struct {
  int32_t max_iter;
  double time_limit;
  double max_step_fraction;
  double tol_gap_abs, tol_gap_rel, tol_feas, tol_infeas_abs, tol_infeas_rel, tol_ktratio;
  double reduced_tol_gap_abs, reduced_tol_gap_rel, reduced_tol_feas, reduced_tol_infeas_abs,
      reduced_tol_infeas_rel, reduced_tol_ktratio;
  int32_t equilibrate_enable, equilibrate_max_iter;
  double equilibrate_min_scaling, equilibrate_max_scaling;
  double min_terminate_step_length;
  int32_t static_regularization_enable;
  double static_regularization_constant, static_regularization_proportional;
  int32_t dynamic_regularization_enable;
  double dynamic_regularization_eps, dynamic_regularization_delta;
  int32_t iterative_refinement_enable;
  double iterative_refinement_reltol, iterative_refinement_abstol;
  int32_t iterative_refinement_max_iter;
  double iterative_refinement_stop_ratio;
  /* nonsymmetric cones only (settings.rs:114-124) */
  double linesearch_backtrack_step, min_switch_step_length;
  int32_t presolve_enable;   /* drop nonnegative rows with an infinite bound (presolver.rs); default 1 */
  /* print a banner, the problem and settings, one row per iteration and a footer to the handle's print target
   * (cipm_set_print_target).  Default 0, where the reference defaults to true: this library sits below other code,
   * and a caller that did not ask for output gets none.  May change in cipm_update_settings. */
  int32_t verbose;
} cipm_settings;

/* DefaultInfo (default/info.rs:13-64) + timers of core/solver.rs:330-396 + counters */
typedef struct {
  int32_t status;
  uint32_t iterations;
  double cost_primal, cost_dual, res_primal, res_dual, res_primal_inf, res_dual_inf;
  double gap_abs, gap_rel, ktratio, mu, step_length, sigma;
  double solve_time;          /* host wall clock, seconds */
  double device_ms;           /* CUDA events around the whole solve on the handle's stream */
  double t_kkt_update, t_kkt_solve, t_scale_cones;   /* "kkt update" / "kkt solve" / "scale cones" */
  uint64_t n_refactor, n_ldl_solve, n_ir_steps, regularize_count;
  uint64_t nnzK, nnzL, kkt_dim;
} cipm_info;

void cipm_default_settings(cipm_settings *s);

/* DefaultSolver::new(P, q, A, b, cones, settings).  P: n x n upper triangle CSC;
 * A: m x n CSC; cones: parallel arrays (type tag, dimension).  Cones are
 * collapsed, data equilibrated (Ruiz), KKT assembled and analysed here.
 * kkt_perm_or_null: optional elimination order for the (n+m+p) KKT system. */
int cipm_create(cipm_t **out, uint64_t n, uint64_t m, const uint64_t *P_colptr, const uint64_t *P_rowval,
                const double *P_nzval, const double *q, const uint64_t *A_colptr, const uint64_t *A_rowval,
                const double *A_nzval, const double *b, uint64_t ncones, const int32_t *cone_types,
                const uint64_t *cone_dims, const cipm_settings *settings, const cldl_opts *ldl_opts,
                const uint64_t *kkt_perm_or_null);
/* Same, with one double per cone: the exponent alpha of a CIPM_CONE_POW entry (PowerConeT(alpha),
 * supportedcone.rs:36-38; the Julia interface carries it the same way, julia/types.rs:19-26), ignored for the other
 * cone types.  cone_params may be NULL when the problem has no power cones. */
int cipm_create_ex(cipm_t **out, uint64_t n, uint64_t m, const uint64_t *P_colptr, const uint64_t *P_rowval,
                   const double *P_nzval, const double *q, const uint64_t *A_colptr, const uint64_t *A_rowval,
                   const double *A_nzval, const double *b, uint64_t ncones, const int32_t *cone_types,
                   const uint64_t *cone_dims, const double *cone_params, const cipm_settings *settings,
                   const cldl_opts *ldl_opts, const uint64_t *kkt_perm_or_null);
/* Same, with generalised power cones (GenPowerConeT(alpha, dim2), supportedcone.rs:44): for a CIPM_CONE_GENPOW entry
 * cone_dims[k] = len(alpha), genpow_dim2[k] = dim2 (ignored for other cones) and genpow_alpha holds the exponents of
 * all such cones concatenated in cone order (each set positive, summing to one). */
int cipm_create_gp(cipm_t **out, uint64_t n, uint64_t m, const uint64_t *P_colptr, const uint64_t *P_rowval,
                   const double *P_nzval, const double *q, const uint64_t *A_colptr, const uint64_t *A_rowval,
                   const double *A_nzval, const double *b, uint64_t ncones, const int32_t *cone_types,
                   const uint64_t *cone_dims, const double *cone_params, const uint64_t *genpow_dim2,
                   const double *genpow_alpha, const cipm_settings *settings, const cldl_opts *ldl_opts,
                   const uint64_t *kkt_perm_or_null);
/* installs the all-gather of a sharded factorisation (cldl_opts.shard_nranks > 1 in ldl_opts) on the solver's LDL */
int cipm_set_transport(cipm_t *h, cldl_allgather_fn fn, void *ctx);
int cipm_set_nccl(cipm_t *h, const char *libpath, const unsigned char *id128, int nranks, int rank);
uint64_t cipm_collective_count(const cipm_t *h);      /* NCCL all-gathers the handle has issued so far */
/* Solver::update_settings (core/solver.rs:207-211): new settings for the next cipm_solve; CLDL_E_ARG when a field that
 * only acts at construction differs (equilibration parameters, presolve_enable: settings.rs:307-335). */
int cipm_update_settings(cipm_t *h, const cipm_settings *settings);
void cipm_destroy(cipm_t *h);
int cipm_solve(cipm_t *h);                                   /* IPSolver::solve */

/* Termination callback (set_termination_callback_c / unset_termination_callback, core/solver.rs; callbacks.rs).
 * cipm_solve calls `fn` once per pass of its iteration loop, iteration 0 included, after the iteration's info is
 * complete and its row printed and before the built-in termination checks; a pass that a strategy switch repeats calls
 * it again.  `info` is what cipm_get_info would return at that moment, valid for the duration of the call.  A nonzero
 * return ends the solve with CIPM_CALLBACK_TERMINATED on the current iterate (cipm_get_solution unscales it as usual).
 * On a sharded handle (a transport or NCCL installed) both calls are collective: every rank makes them, each with
 * its own function, before its next cipm_solve.  While a callback is set every pass all-gathers one value per rank
 * through the handle's transport, and the solve stops on every rank when the callback of any rank asked to.  With no
 * callback set no collective is added. */
typedef int (*cipm_callback_fn)(const cipm_info *info, void *user_data);
int cipm_set_termination_callback(cipm_t *h, cipm_callback_fn fn, void *user_data);
int cipm_unset_termination_callback(cipm_t *h);

/* Where verbose output goes (print_to_stdout / _file / _stream / _sink / _buffer, src/io/mod.rs).  STDOUT is the
 * default; FILE appends to `path`; STREAM hands every chunk of text to `fn(ctx, buf, len)`; BUFFER collects the text
 * in the handle (a new BUFFER target starts empty).  Arguments a kind does not use are ignored.  Every rank of a
 * sharded solver prints to its own target. */
enum { CIPM_PRINT_STDOUT = 0, CIPM_PRINT_SINK = 1, CIPM_PRINT_BUFFER = 2, CIPM_PRINT_FILE = 3, CIPM_PRINT_STREAM = 4 };
typedef int (*cipm_write_fn)(void *ctx, const char *buf, uint64_t len);
int cipm_set_print_target(cipm_t *h, int kind, const char *path, cipm_write_fn fn, void *ctx);
/* get_print_buffer: copies min(cap, length) bytes of the BUFFER target's text to `out` (no terminating zero) and returns
 * the full length; the buffer is not cleared.  CLDL_E_ARG when the target is not a buffer. */
int64_t cipm_get_print_buffer(cipm_t *h, char *out, uint64_t cap);
void cipm_get_info(const cipm_t *h, cipm_info *out);
int cipm_get_solution(cipm_t *h, double *x, double *z, double *s);   /* unscaled, host buffers */
uint64_t cipm_trace(const cipm_t *h, double *out, uint64_t cap_rows); /* rows of [mu,alpha,sigma,pres,dres,gap] */
/* device timestamps (ms since solve() start, CUDA events on the handle's stream) taken at the start of
 * every iteration; the last entry is the end of the solve. */
uint64_t cipm_iter_ms(const cipm_t *h, double *out, uint64_t cap);
uint64_t cipm_launch_count(void);
/* sizeof of {cldl_opts, cldl_info_t, cipm_settings, cipm_info} as compiled into the library: a binding checks its
 * own struct mirrors against them before the first call */
void cipm_abi_sizes(uint64_t *out4);
/* device-timed (CUDA events) average ms of: 0 numeric refactor, 1 one LDL solve, 2 one KKT solve incl. IR */
double cipm_time_ms(cipm_t *h, int which, int reps);                            /* kernels launched by this library so far */
/* Kernel-level test entry points: the sparse products and the reductions of the iteration body on caller data
 * (src/algebra/csc/matrix_math.rs:178-343, src/algebra/vecmath.rs:83-226), so that they can be compared with the
 * reference's own unit-test answers (src/algebra/tests/matrix.rs, vector.rs).
 * cipm_test_spmv: which = 0  y = a P x + b y (the handle's symmetric P), 1  y = a A x + b y, 2  y = a A' x + b y.
 * cipm_test_vec:  what = 0  ||x||_2, 1  ||x||_inf (NaN propagates), 2  ||x .* v||_2, 3  <x, v>. */
int cipm_test_spmv(cipm_t *h, int which, double *y, const double *x, double a, double b);
int cipm_test_vec(cipm_t *h, int what, const double *x, const double *v, uint64_t n, double *out);
/* get_infinity / set_infinity / default_infinity (src/src/utils/infbounds.rs; tests/presolve.rs:107-114): the
 * process-wide bound (default 1e20) beyond which a nonnegative-cone row counts as absent in the presolve; read when a
 * handle is created and when its solution is expanded. */
double cipm_get_infinity(void);
void cipm_set_infinity(double v);
void cipm_default_infinity(void);
uint64_t cipm_m_reduced(const cipm_t *h);   /* rows left after the inf-bound presolve (== m when nothing was dropped) */
/* DefaultProblemData::equilibration (problemdata.rs:229-312; pinned by tests/equilibration_bounds.rs): the Ruiz
 * scalings d [n], e [cipm_m_reduced] and the cost scaling c of the handle; any of the three pointers may be NULL. */
int cipm_get_equilibration(const cipm_t* h, double* d, double* e, double* c);
uint64_t cipm_kkt_dim(const cipm_t *h);
uint64_t cipm_kkt_nnz(const cipm_t *h);
int cipm_get_kkt(const cipm_t *h, uint64_t *colptr, uint64_t *rowval, double *nzval, int8_t *dsigns);
int cipm_get_kkt_perm(const cipm_t *h, uint64_t *perm);
void cipm_ldl_info(const cipm_t *h, cldl_info_t *info);

/* DefaultSolver::update_data (src/solver/implementations/default/data_updating.rs:68-163): overwrite the values of
 * P (triu, same pattern), q, A (same pattern), b in an existing solver; the stored equilibration is applied, symbolic
 * analysis and device plans are reused, the next cipm_solve starts from the default initial point.  NULL = unchanged. */
int cipm_update_data(cipm_t *h, const double *P_nzval, const double *q, const double *A_nzval, const double *b);

/* Derivatives of the solution map at the last solve.  With (x, z, s) the solution cipm_get_solution returns, the
 * optimality conditions linearised about it, with the complementarity of the final iterate held fixed, are
 *     K [dx; dz] = [-dq - dP x - dA' z;  db - dA x],   K = [P A'; A -H],   ds = db - dA x - A dx.
 * H is the cone scaling at the final iterate: on zero cones 0; on nonnegative, second-order and PSD cones the NT
 * scaling the interior-point method uses (s/z on a nonnegative row, the exact linearisation of s_i z_i = const); on
 * exponential, power and generalised power cones always the dual scaling mu * Hess f*(z) with mu = <s, z> / nu (the
 * linearisation of the central-path equation s = -mu grad f*(z)), whichever scaling strategy the solve ended in.
 * As mu -> 0 this tends to the derivative of the solution map wherever that map is differentiable, i.e. under strict
 * complementarity; at a finite mu it is the derivative of the point the solver returned.  On polyhedral cones the
 * limit is reached whatever the path; on second-order and PSD cones with s and z both on the boundary the NT scaling's
 * limit depends on how centred the final iterate is, so there the result approaches the solution map's derivative
 * only as the iterate approaches the central path.
 * Each call builds H, refactors K (static regularisation as in a solve) and solves once with iterative refinement
 * against the unregularised K; nothing is cached between calls.  It changes neither cipm_get_info, the trace, the
 * solution nor what the next cipm_solve computes.
 * Valid only after a cipm_solve that ended CIPM_SOLVED or CIPM_ALMOST_SOLVED, with no cipm_update_data, ckkt_update_P
 * or ckkt_update_A since, and only when the inf-bound presolve removed no rows (cipm_m_reduced == m); otherwise
 * CLDL_E_ARG.  CLDL_E_NOT_FACTORED when the cone scaling, the factorisation or the solve fails numerically.
 * On a sharded handle both calls are collective: every rank makes them, with the same inputs.
 *
 * Forward derivative: (dx, dz, ds) for a data perturbation (dP on P's triu pattern, dq, dA on A's pattern, db).
 * NULL input = zero; NULL output = not wanted. */
int cipm_derivative(cipm_t *h, const double *dP_nzval, const double *dq, const double *dA_nzval, const double *db,
                    double *dx, double *dz, double *ds);
/* Adjoint: gradients w.r.t. (P triu values, q, A values, b) of <gx,x> + <gz,z> + <gs,s>.  NULL input = zero; NULL
 * output = not wanted.  With K [u; v] = [gx - A' gs; gz] and w = v + gs: dq = -u, db = w, dA_ij = -(z_i u_j + w_i x_j)
 * on A's pattern, dP_ij = -(u_i x_j + x_i u_j) on P's stored upper triangle (i != j) and -u_i x_i on its diagonal. */
int cipm_adjoint_derivative(cipm_t *h, const double *gx, const double *gz, const double *gs,
                            double *gP_nzval, double *gq, double *gA_nzval, double *gb);

/* KKTSolver trait on the handle's KKT object (host buffers; x has length n, z length m).
 * ckkt_update / ckkt_solve return 1 (true) / 0 (false) like the trait's bools. */
int ckkt_update(cipm_t *h);                                  /* KKTSolver::update(cones, settings) */
int ckkt_setrhs(cipm_t *h, const double *rhsx, const double *rhsz);
int ckkt_solve(cipm_t *h, double *lhsx, double *lhsz);       /* LDL solve + iterative refinement */
int ckkt_update_P(cipm_t *h, const double *P_nzval_scaled);
int ckkt_update_A(cipm_t *h, const double *A_nzval_scaled);
int ckkt_get_values(cipm_t *h, double *nzval_out);           /* current (un-regularised) KKT values */

/* Cone trait on the handle's composite cone (host buffers of length m). */
int ccone_set_identity_scaling(cipm_t *h);
int ccone_update_scaling(cipm_t *h, const double *s, const double *z);   /* bool */
uint64_t ccone_Hs_len(const cipm_t *h);
int ccone_get_Hs(cipm_t *h, double *Hs);
int ccone_mul_Hs(cipm_t *h, double *y, const double *x);
int ccone_affine_ds(cipm_t *h, double *ds);
int ccone_combined_ds_shift(cipm_t *h, double *shift, const double *step_z, const double *step_s, double sigmamu);
int ccone_ds_from_dz_offset(cipm_t *h, double *out, const double *ds, const double *z);
int ccone_step_length(cipm_t *h, const double *dz, const double *ds, const double *z, const double *s,
                      double alpha_max, double *alpha_out);
int ccone_margins(cipm_t *h, const double *z, double *min_margin, double *pos_margin);
int ccone_scaled_unit_shift(cipm_t *h, double *z, double alpha, int primal);
/* the parts of the trait only nonsymmetric problems use (cones/mod.rs:61-66, 94-101, 148-153) */
int ccone_is_symmetric(const cipm_t *h);
int ccone_unit_initialization(cipm_t *h, double *z, double *s);
int ccone_update_scaling_ex(cipm_t *h, const double *s, const double *z, double mu, int strategy);   /* bool */
int ccone_affine_ds_ex(cipm_t *h, double *ds, const double *s);
int ccone_compute_barrier(cipm_t *h, const double *z, const double *s, const double *dz, const double *ds,
                          double alpha, double *barrier_out);

#ifdef __cplusplus
}
#endif
#endif
