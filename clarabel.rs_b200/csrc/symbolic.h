// Host-side symbolic analysis for the device multifrontal LDL^T.
//
// Plays the role of the reference's one-time `_qdldl_new` setup
// (/root/reference/src/qdldl/qdldl.rs:230-295: ordering, symmetric permute,
// etree, column counts, logical factorisation) but produces a *supernodal
// assembly tree scheduled by level* instead of a column-by-column up-looking
// schedule: that is the shape the GPU wants (independent fronts per level,
// dense panels, no per-entry row indices in the factor).
#pragma once
#include <cstdint>
#include <atomic>
#include <vector>

namespace cb {

// ---- orderings (ordering.cpp) ----
void amd_graph(int n, const std::vector<int64_t>& xadj, const std::vector<int>& adj,
               double dense_scale, std::vector<int>& order, const std::vector<char>* forced_first = nullptr,
               const std::vector<char>* halo = nullptr, const std::atomic<bool>* cancel = nullptr);
// cancel (optional): set by another thread to make the pass return early with an empty order
void amd_order(int n, const int64_t* Ap, const int32_t* Ai, double dense_scale,
               std::vector<int>& perm, const std::atomic<bool>* cancel = nullptr);
// sep_flop_cap > 0: give up (empty perm) as soon as one separator alone costs more than that many flops as a dense block
void nd_order(int n, const int64_t* Ap, const int32_t* Ai, double dense_scale,
              int leaf_size, std::vector<int>& perm, double sep_flop_cap = 0.0);

// host threads this process may use for the one-time analysis: the CPUs of its affinity mask (a launcher that pins
// every rank to its own cores -- taskset, sched_setaffinity -- thereby also sizes the thread pools), capped by
// CB_HOST_THREADS when set.  Ranks that share a box must not each assume all of its cores.
unsigned host_threads();

enum OrderingKind { ORDER_GIVEN = 0, ORDER_AMD = 1, ORDER_ND = 2, ORDER_BEST = 3 };

struct SymbolicOptions {
  int ordering = ORDER_BEST;
  double amd_dense_scale = 1.5;  // reference value, ldlsolvers/qdldl.rs:41
  int nd_leaf = 1600;     // regions below this size are ordered by AMD (C2 sweeps on the GPU: 200..12800, best 1600-3200)
  int max_panel = 64;     // widest supernode panel (columns) handled as one task
  int relax_subtree = 64; // merge every etree subtree with at most this many columns into one front (C2 sweep: 16/32/64 -> solve 1.76/1.66/1.58 ms)
  int relax_small = 8;    // always merge a child chain if the merged width stays <= this
  double relax_zeros = 0.25;  // otherwise merge when added explicit zeros / merged size <= this
  // Schur complement handles: the first permuted column of the Schur set S, whose columns are the last n -
  // schur_first of the given permutation.  B and S are post-ordered separately and no front holds columns of both.
  // -1: no Schur set.
  int schur_first = -1;
};

// One "task" = one supernode panel = one front of the multifrontal method.
struct Symbolic {
  int n = 0;
  int64_t nnzA = 0;
  std::vector<int> perm, iperm;  // final (postordered) permutation: new k <- old perm[k]
  std::vector<int> parent;       // etree in the final numbering (-1 root)
  std::vector<int> colcount;     // nnz of each column of L (strictly lower), simplicial
  int64_t nnzL_simplicial = 0;   // what the reference would report as nnzL
  double flops_simplicial = 0;   // sum_j Lnz_j (Lnz_j + 3)

  int nsup = 0;
  std::vector<int> sn_first;      // [nsup+1] first column of each task
  std::vector<int64_t> sn_rowptr; // [nsup+1]
  std::vector<int> sn_rows;       // row indices below the diagonal block, sorted
  std::vector<int> sn_parent;     // task tree
  std::vector<int> sn_level;
  std::vector<int> col2sn;        // [n]

  // children lists (CSR over tasks) and relative index maps child-row -> parent front index
  std::vector<int64_t> child_ptr;  // [nsup+1]
  std::vector<int> child_list;
  std::vector<int64_t> rel_ptr;    // [nsup+1] offsets into rel (length nr of each task)
  std::vector<int> rel;            // position of each task's rows inside its parent's front

  // storage
  std::vector<int64_t> panel_off;  // [nsup+1] doubles; panel is (ns+nr) x ns column major
  std::vector<int64_t> upd_off;    // [nsup] doubles; update matrix nr x nr column major
  int64_t upd_total = 0;           // doubles needed for the update-matrix arena
  int64_t nnzL_stored = 0;         // panel entries actually stored
  int64_t L_alloc = 0;             // doubles to allocate for the panels (32-byte aligned starts)

  // assembly of the original entries: per task CSR list of (src entry in caller
  // order, destination offset inside the task's panel)
  std::vector<int64_t> asm_ptr;    // [nsup+1]
  std::vector<int> asm_src;        // [nnzA]
  std::vector<int64_t> asm_dst;    // [nnzA] offset relative to panel_off[task]

  // level schedule
  int nlevels = 0;
  std::vector<int> level_ptr;   // [nlevels+1]
  std::vector<int> level_tasks; // tasks sorted by level

  double flops_stored = 0;      // dense flops actually executed
  int ordering_used = 0;
};

// see symbolic.cpp: ordering for matrices with dense diagonal blocks (group[v] = block id or -1)
int order_with_groups(int n, const int64_t* Ap, const int32_t* Ai, const int* group, int ngroups,
                      const SymbolicOptions& opt, std::vector<int>& perm_out, int* kind_out);

// Ap/Ai: triu CSC pattern of the KKT matrix (caller's order), n x n.
// perm_in: optional user permutation (length n) or nullptr.
// Returns 0 on success, negative on structural error.
int analyse(int n, const int64_t* Ap, const int32_t* Ai, const int* perm_in,
            const SymbolicOptions& opt, Symbolic& S);

// The analysis of a Schur complement handle: the columns outside `schur` (B) are ordered first, by opt.ordering on the
// subgraph B induces (or perm_in, whose last schur.size() entries must be the Schur set: -5 otherwise), then the Schur
// set S.  opt.schur_first is set to n - |S|.  -4: an empty, duplicate or out-of-range Schur set, or |S| = n.
int analyse_schur(int n, const int64_t* Ap, const int32_t* Ai, const int* perm_in, const std::vector<int>& schur,
                  const SymbolicOptions& opt, Symbolic& S);

// ---- multi-GPU: subtree-to-rank mapping of one factorisation (SURVEY section 8e) ----
// Independent subtrees of the assembly tree factor and solve independently; the fronts above the cut (the "top"
// part, ancestors of more than one rank's subtrees) are replicated on every rank.  What crosses ranks is the update
// matrix (refactor) and the update vector (solve) of every cut root, and the solution slices at the end.
struct ShardPlan {
  int nranks = 1;
  std::vector<int> owner;          // [nsup] rank that factors front s, -1 = replicated top part
  std::vector<int> cut_roots;      // fronts with an owner whose parent is in the top part
  std::vector<double> rank_flops;  // [nranks] dense flops of the owned subtrees
  double top_flops = 0, total_flops = 0;
  int64_t exchange_doubles = 0;    // sum nr^2 over the cut roots: all-gathered once per refactor
  int64_t exchange_vec = 0;        // sum nr over the cut roots: all-gathered once per solve sweep
  int top_levels = 0;              // tree levels inside the top part (its critical path)
  double model_speedup = 1.0;      // total_flops / (max rank_flops + top_flops)
};
// Greedy top-down splitting (largest subtree first) with longest-processing-time assignment of the subtrees to
// ranks; keeps the configuration with the best modelled makespan.  Only reads the front sizes and the tree.
int plan_shards(int nsup, const int* sn_first, const int64_t* sn_rowptr, const int* sn_parent, int nranks,
                ShardPlan& out);

}  // namespace cb
