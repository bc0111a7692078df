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

/* Sparse right-hand sides and selected solution entries: x = (K + E)^-1 b with b given by nb (index, value) pairs
 * (b_index NULL: b_values is dense, n doubles, and nb must be n) and x wanted at nx caller indices (x_index NULL: all
 * n, x_values n doubles, and nx must be n).  E is the refactor's dynamic regularisation, as for cldl_logdet.  The
 * solve is pruned to the assembly tree: the forward sweep visits only the fronts of b's indices and their ancestors
 * (the nonzeros of L^-1 b), the backward sweep only the fronts of the wanted indices and their ancestors.  Each front
 * it visits does the arithmetic cldl_solve does there, so the entries returned compare equal (==) to the same entries
 * of cldl_solve on the densified b.  Index lists stay on the host: the plan of a call is built there, in time
 * O(r log r) in the r fronts it reaches plus the lengths of the index lists.
 *   - Valid after a refactor that returned 1; otherwise CLDL_E_NOT_FACTORED.
 *   - CLDL_E_ARG on a Schur or sharded handle, for an index >= n, for a duplicate index in b_index, and for a NULL
 *     array that is needed.  Duplicates in x_index are allowed.  nb = 0 gives zeros.
 *   - The first call allocates counters and marks like the full solve's (about 4 (2 ntask + 6 nsup) bytes plus the
 *     backward partial sums) and keeps the host prune index (about 4 n + 13 nsup bytes); each call may grow a device
 *     buffer and two pinned buffers for its plan and index lists.  cldl_destroy frees them.
 *   - The factor, D, 1/D and every later cldl_solve are left bit for bit unchanged; cldl_solve keeps its launch
 *     sequence.  No floating-point atomics: repeated calls give the same bits.
 * cldl_solve_sparse reads and writes host buffers and synchronises.  The _dev form takes b_values / x_values in
 * device memory (the index lists on the host) and is only enqueued on the handle's stream; it waits on the host only
 * for the copy out of the pinned buffer it reuses (two calls back) and when a buffer grows. */
int cldl_solve_sparse(cldl_t *h, uint64_t nb, const uint64_t *b_index, const double *b_values,
                      uint64_t nx, const uint64_t *x_index, double *x_values);
int cldl_solve_sparse_dev(cldl_t *h, uint64_t nb, const uint64_t *b_index, const double *d_b_values,
                          uint64_t nx, const uint64_t *x_index, double *d_x_values);   /* indices on the host */

/* Entries of the inverse anywhere: out[k] = ((K + E)^-1)[rows[k], cols[k]] for nnz positions, not only K's pattern
 * (host arrays).  The positions are grouped by column; two columns at a time are solved in one pair of sweeps
 * (the two-right-hand-side sweeps) pruned to the union of their forward closures and of their wanted rows' closures,
 * and each column's rows are gathered.  out[k] compares equal to cldl_solve(e_cols[k])[rows[k]].  Validity, refusals
 * (an index >= n), regularisation and what stays unchanged as for cldl_solve_sparse.  Synchronises the handle's
 * stream. */
int cldl_inverse_entries(cldl_t *h, uint64_t nnz, const uint64_t *rows, const uint64_t *cols, double *out);

/* Null pivots: rank detection, inertia with zeros, solves of singular systems and a null-space basis (MUMPS ICNTL(24) /
 * CNTL(3), INFOG(28), ICNTL(25)).
 *   - cldl_set_null_pivot_tol: from the next refactor on, a pivot with |d| <= tol (absolute) is a null pivot.  It is
 *     taken as infinite: D = 1/D = 0 is stored, its column of L below the pivot is 0 and it updates no later pivot.
 *     It is tested before the sign test and the regularisation, counts neither in regularize_count nor in
 *     positive_inertia, and is not a zero pivot (no CLDL_E_ZERO_PIVOT): the refactor returns 1 when every other
 *     reciprocal pivot is finite.  tol = 0 turns the test off (the default; the factor is then bit for bit the one of a
 *     handle that never called this).  CLDL_E_ARG for tol < 0 or NaN, and on Schur and sharded handles.  The first
 *     tol > 0 allocates n bytes of marks.
 *   - cldl_null_pivots: the number of null pivots of the last refactor and, when index_out is not NULL, their caller
 *     indices in elimination order.  Synchronises.
 *   - cldl_inertia: (n+, n-, n0) of the last refactor: pivots > 0, < 0 and null (n0 = 0 with the test off).  On a Schur
 *     handle, of B's pivots.  CLDL_E_ARG on a sharded handle.
 *   - cldl_null_space: V (n x r, column-major, caller's order) with r the null count (else CLDL_E_ARG).  Column k is
 *     P^T L^-T e_{p_k} for the k-th null pivot p_k: it is exactly 1 at that pivot's caller index, and
 *     K v = P^T L D e_{p_k} = 0 for the factored matrix.  It is computed by the solve's backward sweeps with 1/D replaced
 *     by ones, two columns per pair of sweeps.  resid (r doubles, may be NULL) gets ||K v_k||_inf / (||K||_inf
 *     ||v_k||_inf) with K the handle's current values: this tells whether the pivots found span a null space of K.
 *     The first call with resid sets up what cldl_solve_refined sets up, and CLDL_E_ARG is returned when that set-up
 *     is refused.  Both forms synchronise; cldl_null_space_dev writes V to device memory, resid stays on the host.
 * All three need a refactor that returned 1, else CLDL_E_NOT_FACTORED.
 * With n0 > 0 every solve-type call (cldl_solve(_dev), cldl_solve_sparse(_dev), cldl_inverse_entries,
 * cldl_selected_inverse(_dev), cldl_adjoint_solve(_dev), cldl_solve_refined(_dev)) uses the generalised inverse
 *     K^- = P^T L^-T D^+ L^-1 P,   D^+ = 1/D with 0 at the null pivots,
 * which solves K x = b for a compatible b.  cldl_logdet returns sign 0 and logabsdet = -inf.
 * Scope: the test reads the pivot alone (static pivoting, no interchanges).  It finds the rank when each null pivot's
 * column of the Schur complement is as small as the pivot, which always holds for a semidefinite K
 * (|s_ik|^2 <= s_ii s_kk): the feature is meant for semidefinite matrices (graph Laplacians, floating finite-element
 * subdomains, duplicated variables).  On an indefinite (quasidefinite) matrix a zero pivot with a large column, such as
 * a constraint row eliminated first, is what regularisation is for; declaring it null drops that column, and resid
 * shows it. */
int cldl_set_null_pivot_tol(cldl_t *h, double tol);
int cldl_null_pivots(cldl_t *h, uint64_t *count, uint64_t *index_out /* NULL: count only */);
int cldl_inertia(const cldl_t *h, uint64_t out3[3]);
int cldl_null_space(cldl_t *h, uint64_t r, double *V, double *resid);
int cldl_null_space_dev(cldl_t *h, uint64_t r, double *d_V, double *resid);

/* Diagnostics of the last cldl_solve_sparse(_dev) / cldl_inverse_entries call: host milliseconds spent building its
 * plans, fronts reached forward and backward, panel entries ((ns + nr) ns per front) of those fronts forward and
 * backward, and the host steps the plan building took (summed over the column pairs of cldl_inverse_entries). */
int cldl_sparse_stats(const cldl_t *h, double *out6);

/* Rank-k updates and downdates (CHOLMOD's cholmod_updown): the handle's matrix K becomes K + sum_r sigma_r w_r w_r^T,
 * its stored values and its factor both, without a refactor.  W is n x k in CSC (w_colptr[k + 1], w_rowidx, w_values,
 * row indices in the caller's order), sigma k finite reals.
 *   - Pattern: every pair (a, b) of stored rows of one column of W must be a stored entry of the upper triangle passed
 *     to cldl_create (diagonal included): each column's pattern is a clique of K's graph.  Then every updated entry
 *     lies in L's structure (the column's rows are ancestors of its first eliminated row in the elimination tree, so
 *     only the fronts on the path from that row's front to the root change) and the supernodal storage stays as it is.
 *     Explicit zeros in K's pattern at create make room for more.
 *   - Values: per stored entry (i, j), i <= j, the contributions are added in ascending r, each operation rounded once:
 *     v += (sigma_r * w_i) * w_j.
 *   - Factor: Gill, Golub, Murray and Saunders' method C1 for L D L^T, per pivot column j on the paths in elimination
 *     order and per column r whose path contains j in ascending r (alpha_r starts at sigma_r):
 *         p = w[j];  dbar = d_j + alpha_r p^2;  beta = alpha_r p / dbar;  alpha_r <- alpha_r d_j / dbar;  d_j <- dbar
 *         rows i of the front below j:  w[i] -= p L_ij;  L_ij += beta w[i]
 *     then 1/D is rewritten, and wide pivot blocks (more than 8 pivots, which store L11^-1) are recovered, updated and
 *     inverted again.  Every solve-type call then works on the updated factor unchanged.  The dynamic regularisation E
 *     of the last refactor is kept: the result is the factor of (K + E) + W diag(sigma) W^T.  If values were changed
 *     since the last refactor (cldl_update_values and the like) the call is not refused, and the factor stays exactly
 *     as stale as it was.
 *   - Verdict, as cldl_refactor's: 1 on success; 0 when an updated pivot is not finite, or with regularisation on fails
 *     the refactor's sign test (dbar * dsign < regularize_eps), or with a null-pivot threshold set has |dbar| <= tol;
 *     CLDL_E_ZERO_PIVOT for an exact zero pivot with regularisation off.  After 0 or an error from the factor update the
 *     values are updated and the factor is invalid: solve-type calls return CLDL_E_NOT_FACTORED until cldl_refactor,
 *     which factors the updated matrix.  regularize_count is unchanged; with regularisation off, positive_inertia,
 *     cldl_inertia and the sign of cldl_logdet follow the pivots that change sign.
 *   - Refused before anything changes: CLDL_E_NOT_FACTORED without a refactor that returned 1 (or with an update whose
 *     verdict was not yet read by cldl_sync_status); CLDL_E_ARG on a Schur or sharded handle, after a refactor that
 *     found null pivots, for an index >= n, a duplicate row in a column, a non-finite sigma, a pair outside the pattern,
 *     and a NULL array that is needed.  k = 0, an empty column and sigma_r = 0 change nothing; the call returns 1.
 *   - Cost: the columns go in passes of 8; each pass is one dataflow kernel over the fronts on its columns' paths.
 *     Host work per call is O(r log r) in the r fronts reached plus the sum of the squared column counts (the pattern
 *     check).  The first call sorts a copy of the caller's pattern on the host (8 nnzA bytes) and allocates 8 n doubles
 *     of work vectors, the pruned solves' set-up and a few scalars per front; cldl_destroy frees them.
 *   - No floating-point atomics: repeated calls on equal handles give the same bits.
 * cldl_updown reads host arrays and synchronises.  cldl_updown_dev takes w_values in device memory (pattern and sigma
 * on the host) and is only enqueued on the handle's stream; its verdict comes from cldl_sync_status, as for
 * cldl_refactor_dev.  cldl_updown_stats gives the last call's host milliseconds, passes, fronts reached, tasks, panel
 * entries of the fronts reached ((ns + nr) ns per front, summed over the passes) and host steps. */
int cldl_updown(cldl_t *h, uint64_t k, const uint64_t *w_colptr, const uint64_t *w_rowidx, const double *w_values,
                const double *sigma);
int cldl_updown_dev(cldl_t *h, uint64_t k, const uint64_t *w_colptr, const uint64_t *w_rowidx,
                    const double *d_w_values, const double *sigma);   /* pattern and sigma on the host */
int cldl_updown_stats(const cldl_t *h, double *out6);

/* The factor's parts (CHOLMOD's cholmod_solve(sys, ...), PARDISO's phases 331 / 332 / 333).  With
 * P (K + E) P^T = L D L^T (L unit lower triangular, E the dynamic regularisation of the last refactor), (P b)[k] =
 * b[perm[k]] (cldl_get_perm) and D+ = D with 0 at null pivots (cldl_set_null_pivot_tol):
 *   cldl_solve_part     x = op^-1 b.  sys CLDL_SYS_A is x = (K + E)^-1 b in caller order: cldl_solve's launches, bit
 *                       for bit.  Every other sys works in permuted order: LDLT (L D L^T)^-1, LD (L D)^-1,
 *                       DLT (D L^T)^-1, L L^-1, LT L^-T, D D+ (1/D, 0 at null pivots), P x = P b, PT x = P^T b,
 *                       DHALF x = |D|^-1/2 b (0 at null pivots).  L^-1 is the forward sweep alone, (D L^T)^-1 the
 *                       backward sweep alone, L^-T the backward sweep with 1/D read as ones.
 *   cldl_mul_part       y = op x for op in A = P^T L D L^T P (caller order), LDLT, LD, DLT, L, LT, D, DHALF = |D|^1/2,
 *                       P, PT (permuted order).  L x and L^T x are one pass over the fronts each (ldl_parts.cuh).
 *   cldl_factor_csc_nnz / cldl_get_factor_csc
 *                       L strictly lower in compressed-column form, permuted order, rows ascending in every column, on
 *                       the stored supernodal pattern: nnz = sum over the fronts of ns (ns - 1) / 2 + ns nr.  Entries
 *                       below the pivot blocks and in pivot blocks of at most 8 columns are the factor's bits; wider
 *                       pivot blocks are recovered from their stored inverse and are within rounding of L11 (entries
 *                       outside the simplicial pattern come back at rounding level).  D and Dinv as stored, 0 at null
 *                       pivots.  colptr: n + 1, rowval and Lx: nnz, D and Dinv: n.  Any output may be NULL.
 *   cldl_sample         k draws, X n x k column-major in caller order: form CLDL_SAMPLE_PRECISION
 *                       x = mu + P^T L^-T |D|^-1/2 z (covariance (K + E)^-1; D+ at null pivots: draws in the range of
 *                       the generalised inverse), form CLDL_SAMPLE_COVARIANCE x = mu + P^T L |D|^1/2 z (covariance
 *                       K + E).  mu: n doubles or NULL (0).  Z: NULL or n x k, the standard normals used, in permuted
 *                       order.  z[r] of column c is normal 4 j + q (j = r / 4, q = r % 4) of Philox4x64-10 with key
 *                       (seed, 0) and counter (j, offset + c, 0, 0): four words w, u = (w >> 11) 2^-53, Box-Muller
 *                       on (1 - u0, u1) and (1 - u2, u3): sqrt(-2 ln(1 - u0)) cos(2 pi u1), ... sin(2 pi u1), then
 *                       the same on (u2, u3).  So draw c of a call equals draw 0 of a call at offset + c, bit for bit.
 *                       Precision draws go two per pair of backward sweeps; a draw has the same bits either way.
 *   - Valid after a refactor that returned 1 and after an update that returned 1; otherwise CLDL_E_NOT_FACTORED.
 *   - CLDL_E_ARG on Schur and sharded handles, for an unknown sys or form, a NULL array that is needed, and (sampling)
 *     when a pivot is negative: the matrix must be semidefinite.
 *   - The factor, D, 1/D and later solves are unchanged.  The host-pointer forms synchronise; the _dev forms take
 *     device pointers and are only enqueued on the handle's stream.  The first call allocates 3 n doubles of work
 *     vectors, the first product with L or export (n + 1) + nnz(L21) int64s of row lists and n + 1 of column
 *     pointers, the first L^-T solve n doubles of ones (shared with cldl_null_space); they stay until cldl_destroy.
 *     cldl_get_factor_csc stages rowval and Lx through nnz int64s and doubles, cldl_sample through at most 5 n
 *     doubles, allocated and freed by the call. */
enum {
  CLDL_SYS_A = 0, CLDL_SYS_LDLT = 1, CLDL_SYS_LD = 2, CLDL_SYS_DLT = 3, CLDL_SYS_L = 4, CLDL_SYS_LT = 5,
  CLDL_SYS_D = 6, CLDL_SYS_P = 7, CLDL_SYS_PT = 8, CLDL_SYS_DHALF = 9
};
enum { CLDL_SAMPLE_PRECISION = 0, CLDL_SAMPLE_COVARIANCE = 1 };
int cldl_solve_part(cldl_t *h, int sys, double *x, const double *b);
int cldl_solve_part_dev(cldl_t *h, int sys, double *d_x, const double *d_b);
int cldl_mul_part(cldl_t *h, int sys, double *y, const double *x);
int cldl_mul_part_dev(cldl_t *h, int sys, double *d_y, const double *d_x);
int cldl_factor_csc_nnz(const cldl_t *h, uint64_t *nnz);
int cldl_get_factor_csc(cldl_t *h, uint64_t *colptr, uint64_t *rowval, double *Lx, double *D, double *Dinv);
int cldl_get_factor_csc_dev(cldl_t *h, uint64_t *d_colptr, uint64_t *d_rowval, double *d_Lx, double *d_D,
                            double *d_Dinv);
int cldl_sample(cldl_t *h, int form, uint64_t k, uint64_t seed, uint64_t offset, const double *mu, double *X,
                double *Z);
int cldl_sample_dev(cldl_t *h, int form, uint64_t k, uint64_t seed, uint64_t offset, const double *d_mu, double *d_X,
                    double *d_Z);

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

/* Iterative refinement and error analysis (MUMPS ICNTL(10) / ICNTL(11), PARDISO iparm(8)).
 * K is the symmetric matrix of the handle's CURRENT values, cldl_values_dev: the caller's upper triangle mirrored,
 * including every cldl_update_values / scale / offset / set_values_dev since the last refactor.  The correction solves
 * use the factor of the last refactor; when the two differ the factor is only a preconditioner, and refinement
 * converges only when the change is small.  For an iterate x, with r = b - K x:
 *     den1_i = (|K||x|)_i + |b_i|
 *     den2_i = (|K||x|)_i + ||K_i||_inf ||x||_inf          (||K_i||_inf = max_j |K_ij|)
 *     tau_i  = 1000 n eps (||K_i||_inf ||x||_inf + |b_i|)
 *     I1 = {i : den1_i > tau_i}, I2 the rest
 *     omega1 = max over I1 of |r_i| / den1_i
 *     omega2 = max over I2 of |r_i| / den2_i, a row with den2_i = 0 and r_i = 0 counting 0
 * and an empty set gives 0: the componentwise backward errors of Arioli, Demmel and Duff (1989), as MUMPS reports them
 * in RINFOG(7..8).
 *   - Loop: x0 is the plain solve, bitwise cldl_solve(b).  Each step solves for dx with the factor and sets
 *     x <- x + dx.  It stops when omega1 + omega2 <= tol, when max_iter steps are done, when a step does not divide
 *     omega1 + omega2 by at least stop_ratio, or when omega1 + omega2 is not finite.  The iterate with the smallest
 *     omega1 + omega2 seen is returned (the earlier one on a tie), with its analysis in info.
 *   - Error analysis (error_analysis = 1), at the returned x:
 *         cond1 = || |K^-1| (den1 o 1_I1) ||_inf / ||x||_inf,   cond2 = || |K^-1| (den2 o 1_I2) ||_inf / ||x||_inf,
 *         ferr = omega1 cond1 + omega2 cond2,
 *     each from Higham's 1-norm estimator (Hager's method with Higham's safeguards, LAPACK dlacn2) applied to
 *     B = diag(g) K^-1, B^T y = K^-1 (g o y): at most 5 iterations plus the alternating-sign test vector, at most 11
 *     solves per estimate; an empty I1 or I2 costs no solves.  K^-1 here is the inverse of the factored matrix: with
 *     dynamic regularisation (cldl_info.regularize_count > 0) or values changed since the refactor, the estimates are
 *     of that matrix's inverse.  Without error analysis cond1, cond2 and ferr are 0; they are 0 also when x = 0.
 *   - Returns CLDL_OK or a negative code; convergence is info.converged (omega1 + omega2 <= tol for the returned x),
 *     not the return value.  CLDL_E_NOT_FACTORED without a refactor that returned 1.  CLDL_E_ARG on a Schur handle, a
 *     sharded handle, for max_iter < 0, tol < 0 or stop_ratio < 1 (or NaN), and when the mirrored pattern (2 nnzA - n
 *     entries) does not fit int32 indices.
 *   - No floating-point atomics: two calls give the same bits.  The factor, D, 1/D and every later plain solve are
 *     left bit for bit unchanged.
 *   - Synchronisation: the stopping test runs on the host, so BOTH forms synchronise the handle's stream: one read of a
 *     few scalars per refinement step, and one after every solve of the estimator.  cldl_solve_refined_dev takes
 *     device buffers (d_x and d_b must not overlap) and never copies a vector to the host.
 *   - The first call builds and uploads the mirrored pattern (int32 rowptr, column indices and a source map into the
 *     values: (n + 1 + 2 (2 nnzA - n)) * 4 bytes) and allocates 6 n doubles of work vectors, 8 * 296 + 16 doubles of
 *     reduction workspace and 16 doubles of pinned host memory.  cldl_destroy frees them.
 * opts == NULL means the defaults of cldl_default_refine_opts; info may be NULL. */
typedef struct {
  int32_t max_iter;        /* refinement steps at most; 0 = the plain solve, analysed only      (default 10) */
  double tol;              /* stop once omega1 + omega2 <= tol                                  (default DBL_EPSILON) */
  double stop_ratio;       /* stop when a step does not divide omega1 + omega2 by at least this (default 2) */
  int32_t error_analysis;  /* 1: also estimate cond1, cond2 and ferr (extra solves)             (default 0) */
} cldl_refine_opts;

typedef struct {
  uint32_t steps;          /* refinement steps taken */
  uint32_t solves;         /* LDL solves made by the call, estimator included */
  int32_t converged;       /* 1 when the returned x has omega1 + omega2 <= tol */
  double norm_K_inf, norm_x_inf, resid_inf;   /* ||K||_inf (current values), ||x||_inf, ||b - K x||_inf */
  double scaled_resid;     /* resid_inf / (norm_K_inf * norm_x_inf); 0 when resid_inf = 0 */
  double omega1, omega2;   /* componentwise backward errors of the returned x */
  double cond1, cond2, ferr;   /* error_analysis only, else 0 */
} cldl_refine_info;

void cldl_default_refine_opts(cldl_refine_opts *o);
int cldl_solve_refined(cldl_t *h, double *x, const double *b, const cldl_refine_opts *opts, cldl_refine_info *info);
int cldl_solve_refined_dev(cldl_t *h, double *d_x, const double *d_b, const cldl_refine_opts *opts,
                           cldl_refine_info *info);
void cldl_refine_abi_sizes(uint64_t *out2);   /* sizeof cldl_refine_opts, cldl_refine_info */

/* Eigenvalues nearest a shift (scipy.sparse.linalg.eigsh(sigma=), SLEPc's shift-and-invert).  The caller puts the
 * values F = A - sigma M in the handle (A its matrix, M positive definite, both on the handle's pattern) and refactors
 * with regularize_enable = 0.  cldl_eigsh returns the nev eigenpairs (lambda, x) of A x = lambda M x nearest sigma:
 *   - Method: thick-restart Lanczos (Wu and Simon 2000) on T = F^-1 M, self-adjoint in <x, y>_M = x^T M y.  Its
 *     eigenvalues theta give lambda = sigma + 1 / theta; the nev of largest |theta| are wanted.  Each step is one solve
 *     with the factor, one product with M (none when M_nzval is NULL: M = I), and classical Gram-Schmidt against the
 *     whole basis, twice, in the M-inner product.  An invariant subspace (the second pass removes more than 30% of what
 *     the first left, or leaves less than 2^-40 ||T v_j||_M) sets beta = 0 and continues with a fresh random vector
 *     orthogonalised against the basis.  A
 *     restart keeps the nev wanted Ritz vectors and up to (ncv - nev) / 2 more, as more have converged.
 *   - Converged: |beta_m y_{m,i}| <= tol |theta_i| (ARPACK's test, y_i the eigenvector of the projected matrix).
 *   - Single-vector Lanczos finds every eigenvalue but not necessarily every copy of a repeated one.  info.n_below is n-
 *     of the factor, which by Sylvester's law is the number of eigenvalues of (A, M) below sigma: the number of lambda
 *     in [a, b) is n_below at b minus n_below at a, the completeness check.
 *   - Output: evals ascending; X (n x nev column-major, or NULL) M-orthonormal, each column's entry of largest
 *     magnitude positive (the smallest index on a tie).  With status 0 the nconv converged pairs come first, then the
 *     other wanted Ritz pairs, each group ascending.
 *   - resid[i] (nev doubles, or NULL) = ||A x - lambda M x||_inf / ((||F||_inf + |sigma| ||M||_inf + |lambda| ||M||_inf)
 *     ||x||_inf), with A x - lambda M x = F x - (lambda - sigma) M x formed from the handle's values, not the factor:
 *     an inaccurate factor (it is taken without pivoting) shows in the residuals.  info.max_resid is their maximum.
 *   - The start vector is Philox draw 0 of `seed` (the normals of cldl_sample at offset 0), the k-th fresh vector draw k.
 *   - status: 1 all nev converged; 0 not within max_restarts (or a non-finite value met: evals, X and resid are then
 *     NaN when nconv = 0); -1 a zero or negative M-norm was met, M is not positive definite (evals, X and resid NaN).
 *     All return CLDL_OK.  The M-norms checked are those of the random draws and of T v_j, and that of a fresh vector
 *     after orthogonalisation: an indefinite M whose negative directions none of them meets is not detected, and the
 *     run then ends with status 0 or with pairs that are not eigenpairs of a definite pencil.  M must be positive
 *     definite; the check is a safeguard, not a test of definiteness.
 *   - CLDL_E_NOT_FACTORED without a refactor that returned 1.  CLDL_E_ARG on Schur and sharded handles, for nev = 0 or
 *     nev >= n, an ncv that is nonzero and outside (nev, min(n, 512)], ncv = 0 with nev >= min(n, 512) (the default
 *     basis would not exceed nev), max_restarts < 0, tol < 0 or NaN, NULL evals,
 *     when 2 nnzA - n does not fit int32 (the mirrored pattern of cldl_solve_refined), and for a factor with
 *     regularize_count > 0 (it would be the factor of F + E) or with null pivots (sigma is then numerically an
 *     eigenvalue: move it).  CLDL_E_CUDA when an allocation fails; the handle stays usable.
 *   - Synchronisation: BOTH forms synchronise the handle's stream once per Lanczos step (the iteration runs on the
 *     host), as cldl_solve_refined_dev does.  cldl_eigsh_dev reads M's values and writes X in device memory.
 *   - Memory: the call allocates (ncv + 1) n doubles of basis (twice that with M), ncv n of restart scratch, 2 n of
 *     work vectors and (ncv + 1) 296 of reduction partials (plus nnzA for a host M), and frees them before it returns;
 *     the first call also sets up cldl_solve_refined's mirrored pattern, which stays.
 *   - No floating-point atomics and fixed reduction orders: two calls give the same bits.  The call reads the factor and
 *     the values and writes only its own buffers: the factor and later solves are bit for bit unchanged.
 * opts == NULL means the defaults of cldl_default_eig_opts; resid and info may be NULL. */
typedef struct {
  int32_t ncv;             /* basis size; 0 = min(n, 512, max(2 nev + 1, 20))                   (default 0) */
  int32_t max_restarts;    /* thick restarts at most                                             (default 300) */
  double tol;              /* convergence tolerance; 0 = DBL_EPSILON                             (default 0) */
  uint64_t seed;           /* Philox key of the start vector and of fresh vectors                (default 0) */
} cldl_eig_opts;

typedef struct {
  int32_t status;          /* 1 converged, 0 not converged, -1 M not positive definite */
  int32_t nconv;           /* converged pairs among the nev returned (they come first) */
  int32_t restarts;        /* thick restarts made */
  uint32_t solves;         /* solves with the factor (one per Lanczos step) */
  uint32_t m_products;     /* products with M, residuals included (0 when M = I) */
  uint64_t n_below;        /* n- of the factor: eigenvalues of (A, M) below sigma */
  double max_resid;        /* max of resid */
} cldl_eig_info;

void cldl_default_eig_opts(cldl_eig_opts *o);
void cldl_eig_abi_sizes(uint64_t *out2);       /* sizeof cldl_eig_opts, cldl_eig_info */
int cldl_eigsh(cldl_t *h, double sigma, const double *M_nzval, uint64_t nev, const cldl_eig_opts *o, double *evals,
               double *X, double *resid, cldl_eig_info *info);
int cldl_eigsh_dev(cldl_t *h, double sigma, const double *d_M_nzval, uint64_t nev, const cldl_eig_opts *o,
                   double *evals, double *d_X, double *resid, cldl_eig_info *info);

/* Solves preconditioned by the factor: restarted right-preconditioned flexible GMRES (Saad 1993), the remedy for
 * static pivoting of Arioli, Duff, Gratton and Pralet (2007) and Arioli and Duff (2009); PARDISO's iparm(4) for a
 * factor reused on new values.  K is the matrix of the handle's CURRENT values, as in cldl_solve_refined; the
 * preconditioner K~ is the factor of the last refactor, which is K + E when pivots were regularised
 * (cldl_info.regularize_count) and that of older values when values changed since.  Where refinement stalls (a
 * regularised pivot, a large value change) FGMRES still converges: K~^-1 K is the identity plus a matrix of rank
 * regularize_count, or of rank at most 2 r for values changed in r columns, and GMRES needs about that many steps plus
 * one.
 *   - x0 is the plain solve, bitwise cldl_solve(b), analysed with omega1 / omega2 exactly as in cldl_solve_refined.
 *   - A cycle starts from r = b - K x of the last analysis, beta = ||r||_2, v_0 = r / beta.  Step j: z_j = K~^-1 v_j
 *     (kept as column j of Z), w = K z_j, classical Gram-Schmidt twice against v_0 .. v_j, giving h_{0..j,j} and
 *     h_{j+1,j} = ||w||_2, and v_{j+1} = w / h_{j+1,j}.  The Givens rotations and the least-squares solve run on the
 *     host in double precision, in a fixed order.
 *   - A cycle ends after `restart` steps, when the call has made max_iter steps, at a breakdown (h_{j+1,j} <=
 *     2^-40 ||K z_j||_2: the solution lies in the space), at a non-finite value (that step is not used), or when the
 *     estimated residual |g_{j+1}| <= (tol / omega_c) beta, omega_c = omega1 + omega2 at the cycle's start.  Then
 *     x = x + Z y (y the least-squares solution) is analysed.
 *   - The call stops at omega1 + omega2 <= tol, at max_iter steps, at a non-finite omega1 + omega2, or when a cycle
 *     did not lower omega1 + omega2 below omega_c.  The iterate with the smallest omega1 + omega2 is returned (the
 *     earlier one on a tie), with its analysis in info.  max_iter = 0 returns x0 and its analysis; tol = 0 runs until
 *     max_iter steps or stagnation.
 *   - Error analysis (error_analysis = 1): cond1, cond2 and ferr at the returned x, as in cldl_solve_refined (K^-1
 *     there is K~^-1, the inverse of the factored matrix).  The returned x is analysed once more first.
 *   - Returns CLDL_OK or a negative code; convergence is info.converged, not the return value.  CLDL_E_NOT_FACTORED
 *     without a refactor that returned 1.  CLDL_E_ARG on Schur and sharded handles, for restart outside
 *     [1, min(n, 512)], max_iter < 0, tol < 0 or NaN, when 2 nnzA - n does not fit int32 (the mirrored pattern), and
 *     for a factor with null pivots.  CLDL_E_CUDA when an allocation fails: the call's buffers are freed, the runtime's
 *     last error is cleared and the handle stays usable.
 *   - No floating-point atomics and fixed reduction orders: two calls give the same bits.  The factor, D, 1/D, the
 *     values and every later solve are left bit for bit unchanged.
 *   - Synchronisation: BOTH forms synchronise the handle's stream once per Arnoldi step and once per analysis (and
 *     after each solve of the estimator).  cldl_solve_gmres_dev takes device buffers (d_x and d_b must not overlap)
 *     and never copies a vector to the host.
 *   - Memory: the call allocates (restart + 1) n doubles for V, restart n for Z and (restart + 1) 296 of reduction
 *     partials plus a few scalars, and frees them before it returns.  The first call also sets up
 *     cldl_solve_refined's mirrored pattern and work vectors, which stay.
 * opts == NULL means the defaults of cldl_default_gmres_opts; info may be NULL. */
typedef struct {
  int32_t restart;         /* Arnoldi steps per cycle, 1 .. min(n, 512)                         (default 20) */
  int32_t max_iter;        /* Arnoldi steps in all; 0 = the plain solve, analysed only          (default 100) */
  double tol;              /* stop once omega1 + omega2 <= tol                                  (default DBL_EPSILON) */
  int32_t error_analysis;  /* 1: also estimate cond1, cond2 and ferr (extra solves)             (default 0) */
} cldl_gmres_opts;

typedef struct {
  uint32_t iterations;     /* Arnoldi steps taken */
  uint32_t cycles;         /* cycles begun */
  uint32_t solves;         /* LDL solves made by the call: x0, one per step, the estimator's */
  uint32_t products;       /* products with K: one per step and one per analysis */
  int32_t converged;       /* 1 when the returned x has omega1 + omega2 <= tol */
  double norm_K_inf, norm_x_inf, resid_inf;   /* ||K||_inf (current values), ||x||_inf, ||b - K x||_inf */
  double scaled_resid;     /* resid_inf / (norm_K_inf * norm_x_inf); 0 when resid_inf = 0 */
  double omega1, omega2;   /* componentwise backward errors of the returned x */
  double cond1, cond2, ferr;   /* error_analysis only, else 0 */
} cldl_gmres_info;

void cldl_default_gmres_opts(cldl_gmres_opts *o);
void cldl_gmres_abi_sizes(uint64_t *out2);     /* sizeof cldl_gmres_opts, cldl_gmres_info */
int cldl_solve_gmres(cldl_t *h, double *x, const double *b, const cldl_gmres_opts *opts, cldl_gmres_info *info);
int cldl_solve_gmres_dev(cldl_t *h, double *d_x, const double *d_b, const cldl_gmres_opts *opts,
                         cldl_gmres_info *info);

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
