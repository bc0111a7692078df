// Symbolic analysis: see symbolic.h.  All integer work, host only, one-time.
#include "symbolic.h"
#ifdef __linux__
#include <sched.h>
#endif

#include <algorithm>
#include <atomic>
#include <thread>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <map>
#include <memory_resource>
#include <numeric>
#include <chrono>

namespace cb {
unsigned host_threads() {
  unsigned n = std::thread::hardware_concurrency();
#ifdef __linux__
  cpu_set_t set;
  CPU_ZERO(&set);
  if (sched_getaffinity(0, sizeof(set), &set) == 0) { const int c = CPU_COUNT(&set); if (c > 0) n = (unsigned)c; }
#endif
  if (const char* e = std::getenv("CB_HOST_THREADS")) { const int v = std::atoi(e); if (v > 0 && (unsigned)v < n) n = (unsigned)v; }
  return n ? n : 1u;
}


static double tnow() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static bool timing_on() { static int v = -1; if (v < 0) v = std::getenv("CB_TIMING") ? 1 : 0; return v == 1; }
#define TMARK(label) do { if (timing_on()) { double t_ = tnow(); std::fprintf(stderr, "[cb timing] %-28s %.3f s\n", label, t_ - t_last); t_last = t_; } } while (0)

namespace {

// Upper-triangular CSC pattern of P A P^T (columns sorted) from the caller's
// triu CSC and iperm (old -> new).
void permuted_upper(int n, const int64_t* Ap, const int32_t* Ai, const std::vector<int>& iperm,
                    std::vector<int64_t>& Up, std::vector<int>& Ui, bool sorted = true) {
  Up.assign(n + 1, 0);
  for (int c = 0; c < n; c++)
    for (int64_t p = Ap[c]; p < Ap[c + 1]; p++) {
      int a = iperm[Ai[p]], b = iperm[c];
      Up[(a > b ? a : b) + 1]++;
    }
  for (int j = 0; j < n; j++) Up[j + 1] += Up[j];
  Ui.resize(Up[n]);
  std::vector<int64_t> pos(Up.begin(), Up.end() - 1);
  for (int c = 0; c < n; c++)
    for (int64_t p = Ap[c]; p < Ap[c + 1]; p++) {
      int a = iperm[Ai[p]], b = iperm[c];
      int col = a > b ? a : b, row = a > b ? b : a;
      Ui[pos[col]++] = row;
    }
  if (sorted)
    for (int j = 0; j < n; j++) std::sort(Ui.begin() + Up[j], Ui.begin() + Up[j + 1]);
}

// Liu's elimination tree with path compression, from upper-triangular columns.
void etree_upper(int n, const std::vector<int64_t>& Up, const std::vector<int>& Ui,
                 std::vector<int>& parent) {
  parent.assign(n, -1);
  std::vector<int> anc(n, -1);
  for (int k = 0; k < n; k++)
    for (int64_t p = Up[k]; p < Up[k + 1]; p++) {
      int i = Ui[p];
      while (i != -1 && i < k) {
        int nx = anc[i];
        anc[i] = k;
        if (nx == -1) parent[i] = k;
        i = nx;
      }
    }
}

// Post-order of a forest; children visited in ascending subtree size so the
// heaviest child ends up adjacent to its parent (longer supernode chains).
void postorder(int n, const std::vector<int>& parent, std::vector<int>& post) {
  std::vector<int> size(n, 1);
  for (int j = 0; j < n; j++)
    if (parent[j] >= 0) size[parent[j]] += size[j];  // valid: parent[j] > j
  std::vector<int> cptr(n + 2, 0), clist(n);
  for (int j = 0; j < n; j++) cptr[(parent[j] < 0 ? n : parent[j]) + 1]++;
  for (int j = 0; j <= n; j++) cptr[j + 1] += cptr[j];
  {
    std::vector<int> pos(cptr.begin(), cptr.end() - 1);
    for (int j = 0; j < n; j++) clist[pos[parent[j] < 0 ? n : parent[j]]++] = j;
  }
  for (int j = 0; j <= n; j++)
    std::stable_sort(clist.begin() + cptr[j], clist.begin() + cptr[j + 1],
                     [&](int a, int b) { return size[a] < size[b]; });
  post.clear();
  post.reserve(n);
  std::vector<int> stack, it(n + 1, 0);
  for (int r = cptr[n]; r < cptr[n + 1]; r++) {
    stack.push_back(clist[r]);
    while (!stack.empty()) {
      int v = stack.back();
      if (it[v] < cptr[v + 1] - cptr[v]) {
        stack.push_back(clist[cptr[v] + it[v]++]);
      } else {
        post.push_back(v);
        stack.pop_back();
      }
    }
  }
}

// Gilbert-Ng-Peyton column counts for a post-ordered matrix (post == identity).
// Lo_ptr/Lo_idx: for each column j the rows i > j with A_ij != 0.
void colcounts_postordered(int n, const std::vector<int>& parent, const std::vector<int64_t>& Lo_ptr,
                           const std::vector<int>& Lo_idx, std::vector<int>& cc) {
  std::vector<int> first(n, -1), maxfirst(n, -1), prevleaf(n, -1), anc(n);
  std::vector<int64_t> delta(n, 0);
  for (int k = 0; k < n; k++) {
    int j = k;
    delta[j] = (first[j] == -1) ? 1 : 0;
    for (; j != -1 && first[j] == -1; j = parent[j]) first[j] = k;
  }
  std::iota(anc.begin(), anc.end(), 0);
  for (int j = 0; j < n; j++) {
    if (parent[j] != -1) delta[parent[j]]--;
    for (int64_t p = Lo_ptr[j]; p < Lo_ptr[j + 1]; p++) {
      int i = Lo_idx[p];
      if (i <= j || first[j] <= maxfirst[i]) continue;
      maxfirst[i] = first[j];
      int jprev = prevleaf[i];
      prevleaf[i] = j;
      delta[j]++;
      if (jprev != -1) {
        int q = jprev;
        while (q != anc[q]) q = anc[q];
        for (int s = jprev; s != q;) { int sp = anc[s]; anc[s] = q; s = sp; }
        delta[q]--;
      }
    }
    if (parent[j] != -1) anc[j] = parent[j];
  }
  for (int j = 0; j < n; j++)
    if (parent[j] != -1) delta[parent[j]] += delta[j];
  cc.resize(n);
  for (int j = 0; j < n; j++) cc[j] = (int)(delta[j] - 1);  // strictly-lower count
}

struct Eval { double flops; int64_t nnzL; };

}  // namespace

// flop_cap > 0: give up (return 1) right after the column counts when the simplicial flop count exceeds it --
// used when comparing candidate orderings so that a hopeless candidate costs O(nnz), not O(nnz(L)).
// go_on (optional) is asked once the statistics (flops_stored, nnzL_stored, nlevels) are known: false -> return 2
// with the statistics only, true -> finish the analysis.
static int build(int n, const int64_t* Ap, const int32_t* Ai, const std::vector<int>& perm0,
                 const SymbolicOptions& opt, Symbolic& S, bool stats_only, double flop_cap = 0.0,
                 const std::function<bool(const Symbolic&)>* go_on = nullptr) {
  double t_last = tnow();
  S.n = n;
  S.nnzA = Ap[n];
  std::vector<int> iperm0(n);
  for (int k = 0; k < n; k++) iperm0[perm0[k]] = k;

  std::vector<int64_t> Up;
  std::vector<int> Ui, parent0, post;
  permuted_upper(n, Ap, Ai, iperm0, Up, Ui, false);   // the elimination tree does not need sorted columns
  TMARK("sym:   permuted upper");
  etree_upper(n, Up, Ui, parent0);
  TMARK("sym:   etree");
  postorder(n, parent0, post);
  const int sf = opt.schur_first;
  std::vector<int> post_cc;   // Schur set: the post-order of the whole tree, for the column counts
  if (sf >= 0) {
    // S columns are the last ones and their parents are S columns.  The subtrees of B that hang below S become roots
    // of their own, the forest is post-ordered and its B trees are moved ahead of its S trees: every B column stays
    // ahead of every S column and the numbering is still topological.
    std::vector<int> pB(parent0);
    for (int j = 0; j < sf; j++) if (pB[j] >= sf) pB[j] = -1;
    post_cc.swap(post);
    postorder(n, pB, post);
    std::stable_partition(post.begin(), post.end(), [&](int v) { return v < sf; });
  }
  S.perm.resize(n);
  S.iperm.resize(n);
  for (int k = 0; k < n; k++) S.perm[k] = perm0[post[k]];
  for (int k = 0; k < n; k++) S.iperm[S.perm[k]] = k;
  TMARK("sym:   postorder");

  {
    // the tree of the post-ordered matrix is the old tree relabelled
    std::vector<int> ipost(n);
    for (int k = 0; k < n; k++) ipost[post[k]] = k;
    S.parent.assign(n, -1);
    for (int j = 0; j < n; j++) if (parent0[j] >= 0) S.parent[ipost[j]] = ipost[parent0[j]];
  }
  const std::vector<int>& parent = S.parent;

  // strictly-lower pattern by columns of the post-ordered matrix, straight from the caller's entries (the column
  // counts and the row-structure unions below do not depend on the order inside a column)
  auto lower_pattern = [&](const std::vector<int>& ip, std::vector<int64_t>& Lo_ptr, std::vector<int>& Lo_idx) {
    Lo_ptr.assign(n + 1, 0);
    for (int c = 0; c < n; c++) {
      const int b = ip[c];
      for (int64_t p = Ap[c]; p < Ap[c + 1]; p++) {
        const int a = ip[Ai[p]];
        if (a != b) Lo_ptr[(a < b ? a : b) + 1]++;
      }
    }
    for (int j = 0; j < n; j++) Lo_ptr[j + 1] += Lo_ptr[j];
    Lo_idx.resize(Lo_ptr[n]);
    std::vector<int64_t> pos(Lo_ptr.begin(), Lo_ptr.end() - 1);
    for (int c = 0; c < n; c++) {
      const int b = ip[c];
      for (int64_t p = Ap[c]; p < Ap[c + 1]; p++) {
        const int a = ip[Ai[p]];
        if (a != b) Lo_idx[pos[a < b ? a : b]++] = a < b ? b : a;
      }
    }
  };
  std::vector<int64_t> Lo_ptr;
  std::vector<int> Lo_idx;
  lower_pattern(S.iperm, Lo_ptr, Lo_idx);
  std::vector<int64_t>().swap(Up);
  std::vector<int>().swap(Ui);
  TMARK("sym:   lower pattern");
  if (post_cc.empty()) {
    colcounts_postordered(n, parent, Lo_ptr, Lo_idx, S.colcount);
  } else {
    // every topological order of the tree has the same filled graph, so the counts are those of the post-order
    // (which the counting algorithm needs), relabelled
    std::vector<int> icc(n), pcc(n, -1), cc2;
    for (int k = 0; k < n; k++) icc[perm0[post_cc[k]]] = k;
    for (int j = 0; j < n; j++) if (parent0[j] >= 0) pcc[icc[perm0[j]]] = icc[perm0[parent0[j]]];
    std::vector<int64_t> Lp2;
    std::vector<int> Li2;
    lower_pattern(icc, Lp2, Li2);
    colcounts_postordered(n, pcc, Lp2, Li2, cc2);
    S.colcount.resize(n);
    for (int j = 0; j < n; j++) S.colcount[j] = cc2[icc[S.perm[j]]];
  }
  TMARK("sym:   column counts");
  S.nnzL_simplicial = 0;
  S.flops_simplicial = 0;
  for (int j = 0; j < n; j++) {
    S.nnzL_simplicial += S.colcount[j];
    S.flops_simplicial += (double)S.colcount[j] * ((double)S.colcount[j] + 3.0);
  }

  TMARK("sym: etree+postorder+colcount");
  if (flop_cap > 0.0 && S.flops_simplicial > flop_cap) return 1;
  // ---- supernode partition: fundamental -> relaxed -> split ----
  const std::vector<int>& cc = S.colcount;
  std::vector<int> sfirst;  // start column of every supernode
  {
    // (1) whole small subtrees become one dense front each: in a post-ordered tree the subtree of r is
    //     the contiguous column range [r - size(r) + 1, r] and every row it reaches beyond r is in
    //     struct(L(:,r)), so the merged front is size(r) pivots by colcount[r] rows.  This trades a few
    //     explicit zeros at the leaves for far fewer fronts / children / tree levels.
    //     With a Schur set, B's subtrees below S count as whole trees: a merged subtree is all B or all S.
    std::vector<int> pcut(parent);
    if (sf >= 0) for (int j = 0; j < sf; j++) if (pcut[j] >= sf) pcut[j] = -1;
    std::vector<int> sub(n, 1);
    for (int j = 0; j < n; j++) if (pcut[j] >= 0) sub[pcut[j]] += sub[j];
    std::vector<char> in_small(n, 0), small_root(n, 0);
    if (opt.relax_subtree > 1)
      for (int r = 0; r < n; r++) {
        const bool fits = sub[r] <= opt.relax_subtree;
        const bool top = pcut[r] < 0 || sub[pcut[r]] > opt.relax_subtree;
        if (fits && top && sub[r] > 1) {
          small_root[r] = 1;
          for (int j = r - sub[r] + 1; j <= r; j++) in_small[j] = 1;
        }
      }
    // (2) fundamental supernodes (structure-nested chains) for everything else
    std::vector<int> fs;   // first col
    for (int j = 0; j < n; j++) {
      bool join = j > 0 && parent[j - 1] == j && cc[j] == cc[j - 1] - 1;
      if (in_small[j]) join = !(j == 0 || !in_small[j - 1] || small_root[j - 1]);
      else if (j > 0 && in_small[j - 1]) join = false;
      if (j == sf) join = false;          // the first S column starts a supernode
      if (!join) fs.push_back(j);
    }
    int nf = (int)fs.size();
    fs.push_back(n);
    // relaxed amalgamation along "last child" links (contiguous columns)
    std::vector<int> start(fs.begin(), fs.end() - 1);  // may move left on merge
    std::vector<double> zeros(nf, 0.0);
    std::vector<char> dead(nf, 0);
    std::vector<int> col2f(n);
    for (int s = 0; s < nf; s++)
      for (int j = fs[s]; j < fs[s + 1]; j++) col2f[j] = s;
    for (int p = 0; p < nf; p++) {
      int lastcol = fs[p + 1] - 1;
      int nr_p = cc[lastcol];
      while (start[p] > 0 && start[p] != sf) {   // a B supernode never merges into an S one
        int c = col2f[start[p] - 1];        // supernode ending right before p
        int c_last = fs[c + 1] - 1;
        if (parent[c_last] < start[p] || parent[c_last] > lastcol) break;  // not a child of p
        int ns_c = fs[c + 1] - start[c];
        int ns_p = lastcol + 1 - start[p];
        int nr_c = cc[c_last];              // rows below c's block (into p and beyond)
        double newz = (double)ns_c * (double)(ns_p + nr_p - nr_c);
        double z = zeros[p] + zeros[c] + newz;
        int ns_m = ns_c + ns_p;
        double size_m = (double)ns_m * (double)(ns_m + 1) * 0.5 + (double)ns_m * nr_p;
        bool merge = (ns_m <= opt.relax_small) || (z <= opt.relax_zeros * size_m);
        if (!merge) break;
        zeros[p] = z;
        start[p] = start[c];
        dead[c] = 1;
        // columns of c now belong to p
        for (int j = start[c]; j < fs[c + 1]; j++) col2f[j] = p;
      }
    }
    for (int s = 0; s < nf; s++) {
      if (dead[s]) continue;
      int b = start[s], e = fs[s + 1];
      // split into panels of at most max_panel columns (balanced widths); a supernode lies in B or in S, so its
      // panels do too
      int w = e - b;
      int np = (w + opt.max_panel - 1) / opt.max_panel;
      for (int k = 0; k < np; k++) sfirst.push_back(b + (int)((int64_t)w * k / np));
    }
    std::sort(sfirst.begin(), sfirst.end());
  }
  int nsup = (int)sfirst.size();
  S.nsup = nsup;
  S.sn_first = sfirst;
  S.sn_first.push_back(n);
  S.col2sn.resize(n);
  for (int s = 0; s < nsup; s++)
    for (int j = S.sn_first[s]; j < S.sn_first[s + 1]; j++) S.col2sn[j] = s;

  TMARK("sym: supernode partition");
  // ---- row structures by bottom-up union, parents by min row ----
  // Independent subtrees of the supernode tree are independent here too: the tree is cut into chunks (maximal
  // subtrees below a work threshold; contiguous index ranges because supernodes are numbered in post-order) that
  // host threads take from a shared counter, each into its own buffer; the part above the cut runs afterwards in
  // index order exactly like the one-thread loop and the buffers are spliced in on the way, so the result is the
  // one-thread result.  The chunking uses the parent predicted by the column etree (first row below a supernode =
  // etree parent of its last column); should a computed parent ever leave its chunk, everything is redone on one
  // thread.
  S.sn_rowptr.assign(nsup + 1, 0);
  S.sn_rows.clear();
  S.sn_parent.assign(nsup, -1);
  std::vector<std::vector<int>> kids(nsup);
  // one supernode: rows >= l reached from its own columns and from its children (child rows through `child_rows`)
  auto union_rows = [&](int s, std::vector<int>& mark, std::vector<int>& tmp, auto&& child_rows) {
    const int f = S.sn_first[s], l = S.sn_first[s + 1];
    tmp.clear();
    for (int j = f; j < l; j++)
      for (int64_t p = Lo_ptr[j]; p < Lo_ptr[j + 1]; p++) {
        const int i = Lo_idx[p];
        if (i >= l && mark[i] != s) { mark[i] = s; tmp.push_back(i); }
      }
    for (int c : kids[s]) {
      const int *b = nullptr, *e = nullptr;
      child_rows(c, b, e);
      for (const int* q = b; q < e; q++) {
        const int i = *q;
        if (i >= l && mark[i] != s) { mark[i] = s; tmp.push_back(i); }
      }
    }
    std::sort(tmp.begin(), tmp.end());
  };
  auto sequential_rows = [&]() {
    S.sn_rows.clear();
    for (auto& k : kids) k.clear();
    std::fill(S.sn_parent.begin(), S.sn_parent.end(), -1);
    std::vector<int> mark(n, -1), tmp;
    for (int s = 0; s < nsup; s++) {
      union_rows(s, mark, tmp, [&](int c, const int*& b, const int*& e) {
        b = S.sn_rows.data() + S.sn_rowptr[c]; e = S.sn_rows.data() + S.sn_rowptr[c + 1];
      });
      S.sn_rows.insert(S.sn_rows.end(), tmp.begin(), tmp.end());
      S.sn_rowptr[s + 1] = (int64_t)S.sn_rows.size();
      if (!tmp.empty()) {
        const int ps = S.col2sn[tmp[0]];
        S.sn_parent[s] = ps;
        kids[ps].push_back(s);
      }
    }
  };
  const unsigned hw_rows = std::max(1u, std::min(16u, host_threads()));
  if (nsup < 20000 || hw_rows < 2) {
    sequential_rows();
  } else {
    // predicted tree, subtree work (entries of L below the diagonal blocks) and subtree sizes
    std::vector<int> gpar(nsup, -1), cntsub(nsup, 1);
    std::vector<double> wsub(nsup, 0.0);
    double wtot = 0.0;
    for (int s = 0; s < nsup; s++) {
      const int last = S.sn_first[s + 1] - 1;
      if (parent[last] >= 0 && !(last < sf && parent[last] >= sf)) gpar[s] = S.col2sn[parent[last]];   // B's trees are cut from S
      for (int j = S.sn_first[s]; j <= last; j++) wsub[s] += (double)cc[j] + 1.0;
      wtot += wsub[s];
    }
    for (int s = 0; s < nsup; s++) if (gpar[s] > s) { wsub[gpar[s]] += wsub[s]; cntsub[gpar[s]] += cntsub[s]; }
    const double thr = wtot / (8.0 * hw_rows);
    struct Chunk { int first, last; std::vector<int> rows; std::vector<int64_t> ptr; };   // ptr relative to rows
    std::vector<Chunk> chunks;
    std::vector<int> chunk_of(nsup, -1);
    for (int s = 0; s < nsup; s++) {
      const bool fits = wsub[s] <= thr;
      const bool top = gpar[s] < 0 || wsub[gpar[s]] > thr;
      if (fits && top && cntsub[s] > 1 && !(sf >= 0 && S.sn_first[s] >= sf)) {   // S fronts: after the chunks
        Chunk c; c.first = s - cntsub[s] + 1; c.last = s;
        for (int t = c.first; t <= c.last; t++) chunk_of[t] = (int)chunks.size();
        chunks.push_back(std::move(c));
      }
    }
    std::atomic<int> next{0};
    std::atomic<int> escaped{0};
    auto worker = [&]() {
      std::vector<int> mark(n, -1), tmp;
      for (;;) {
        const int ci = next.fetch_add(1);
        if (ci >= (int)chunks.size()) break;
        Chunk& C = chunks[ci];
        C.ptr.assign((size_t)(C.last - C.first + 2), 0);
        for (int s2 = C.first; s2 <= C.last; s2++) {
          union_rows(s2, mark, tmp, [&](int c, const int*& b, const int*& e) {
            b = C.rows.data() + C.ptr[c - C.first]; e = C.rows.data() + C.ptr[c - C.first + 1];
          });
          C.rows.insert(C.rows.end(), tmp.begin(), tmp.end());
          C.ptr[s2 - C.first + 1] = (int64_t)C.rows.size();
          if (!tmp.empty()) {
            const int ps = S.col2sn[tmp[0]];
            S.sn_parent[s2] = ps;
            if (ps <= C.last) { if (ps < C.first) escaped = 1; else kids[ps].push_back(s2); }
            else if (s2 != C.last) escaped = 1;       // only the chunk root may point above the chunk
          }
        }
      }
    };
    {
      std::vector<std::thread> th;
      for (unsigned t = 0; t < hw_rows; t++) th.emplace_back(worker);
      for (auto& x : th) x.join();
    }
    for (const Chunk& C : chunks)                    // a chunk root's parent must be above every chunk
      if (S.sn_parent[C.last] >= 0 && chunk_of[S.sn_parent[C.last]] >= 0) escaped = 1;
    if (escaped) {
      sequential_rows();
    } else {
      std::vector<int> mark(n, -1), tmp;
      for (int s = 0; s < nsup; s++) {
        const int ci = chunk_of[s];
        if (ci >= 0) {
          const Chunk& C = chunks[ci];
          const int64_t base = (int64_t)S.sn_rows.size();
          S.sn_rows.insert(S.sn_rows.end(), C.rows.begin(), C.rows.end());
          for (int t = C.first; t <= C.last; t++) S.sn_rowptr[t + 1] = base + C.ptr[t - C.first + 1];
          if (S.sn_parent[C.last] >= 0) kids[S.sn_parent[C.last]].push_back(C.last);
          s = C.last;
          continue;
        }
        union_rows(s, mark, tmp, [&](int c, const int*& b, const int*& e) {
          b = S.sn_rows.data() + S.sn_rowptr[c]; e = S.sn_rows.data() + S.sn_rowptr[c + 1];
        });
        S.sn_rows.insert(S.sn_rows.end(), tmp.begin(), tmp.end());
        S.sn_rowptr[s + 1] = (int64_t)S.sn_rows.size();
        if (!tmp.empty()) {
          const int ps = S.col2sn[tmp[0]];
          S.sn_parent[s] = ps;
          kids[ps].push_back(s);
        }
      }
    }
  }

  TMARK("sym: row structures");
  // ---- sizes, flops, levels ----
  S.panel_off.assign(nsup + 1, 0);
  S.flops_stored = 0;
  S.nnzL_stored = 0;
  for (int s = 0; s < nsup; s++) {
    int64_t ns = S.sn_first[s + 1] - S.sn_first[s];
    int64_t nr = S.sn_rowptr[s + 1] - S.sn_rowptr[s];
    // panels start on 32-byte boundaries: a memory sector never holds entries of two fronts (the dataflow
    // factorisation reads finished panels through L1 while other fronts are still being written)
    S.panel_off[s + 1] = (S.panel_off[s] + (ns + nr) * ns + 3) & ~(int64_t)3;
    S.nnzL_stored += (ns + nr) * ns;
    S.flops_stored += (double)ns * ns * ns / 3.0 + (double)ns * ns * nr + (double)ns * nr * nr;
  }
  S.L_alloc = S.panel_off[nsup];
  S.sn_level.assign(nsup, 0);
  int nlev = 0;
  for (int s = 0; s < nsup; s++) {
    int p = S.sn_parent[s];
    if (p >= 0 && S.sn_level[p] < S.sn_level[s] + 1) S.sn_level[p] = S.sn_level[s] + 1;
    if (S.sn_level[s] + 1 > nlev) nlev = S.sn_level[s] + 1;
  }
  S.nlevels = nlev;
  if (stats_only) return 0;
  if (go_on && !(*go_on)(S)) return 2;

  // The three remaining pieces -- (a) level schedule + children + relative index maps, (b) assembly map of the
  // original entries, (c) update-matrix arena -- only read the supernode structure built above and write disjoint
  // members of S: they run on three host threads.
  int rc_a = 0, rc_b = 0;
  auto part_a = [&]() {
  S.level_ptr.assign(nlev + 1, 0);
  for (int s = 0; s < nsup; s++) S.level_ptr[S.sn_level[s] + 1]++;
  for (int l = 0; l < nlev; l++) S.level_ptr[l + 1] += S.level_ptr[l];
  S.level_tasks.resize(nsup);
  {
    std::vector<int> pos(S.level_ptr.begin(), S.level_ptr.end() - 1);
    for (int s = 0; s < nsup; s++) S.level_tasks[pos[S.sn_level[s]]++] = s;
    auto work = [&](int s) {
      int64_t ns = S.sn_first[s + 1] - S.sn_first[s];
      int64_t nr = S.sn_rowptr[s + 1] - S.sn_rowptr[s];
      return (ns + nr) * (ns + nr);
    };
    for (int l = 0; l < nlev; l++)
      std::stable_sort(S.level_tasks.begin() + S.level_ptr[l], S.level_tasks.begin() + S.level_ptr[l + 1],
                       [&](int a, int b) { return work(a) > work(b); });
  }

  // ---- children CSR + relative index maps ----
  S.child_ptr.assign(nsup + 1, 0);
  for (int s = 0; s < nsup; s++) S.child_ptr[s + 1] = S.child_ptr[s] + (int64_t)kids[s].size();
  S.child_list.resize(S.child_ptr[nsup]);
  for (int s = 0; s < nsup; s++)
    std::copy(kids[s].begin(), kids[s].end(), S.child_list.begin() + S.child_ptr[s]);
  S.rel_ptr = S.sn_rowptr;
  S.rel.assign(S.sn_rows.size(), -1);
  for (int c = 0; c < nsup; c++) {
    int p = S.sn_parent[c];
    if (p < 0) continue;
    int pf = S.sn_first[p], pl = S.sn_first[p + 1], pns = pl - pf;
    int64_t q = S.sn_rowptr[p], qe = S.sn_rowptr[p + 1];
    for (int64_t t = S.sn_rowptr[c]; t < S.sn_rowptr[c + 1]; t++) {
      int r = S.sn_rows[t];
      if (r < pl) { S.rel[t] = r - pf; continue; }
      while (q < qe && S.sn_rows[q] < r) q++;
      if (q >= qe || S.sn_rows[q] != r) { std::fprintf(stderr, "symbolic: rel map failure\n"); rc_a = -10; return; }
      S.rel[t] = pns + (int)(q - S.sn_rowptr[p]);
    }
  }
  };

  // ---- assembly map of original entries ----
  auto part_b = [&]() {
  S.asm_ptr.assign(nsup + 1, 0);
  int64_t nnz = Ap[n];
  std::vector<int> ent_task(nnz);
  std::vector<int64_t> ent_dst(nnz);
  {
    // entries are independent: host threads take column ranges (one binary search per entry)
    const unsigned hc = std::max(1u, std::min(16u, host_threads()));
    const unsigned nth = nnz < 200000 ? 1u : hc;
    std::vector<int> bad(nth, 0);
    auto work = [&](unsigned t) {
      const int c0 = (int)((int64_t)n * t / nth), c1 = (int)((int64_t)n * (t + 1) / nth);
      for (int c = c0; c < c1; c++)
        for (int64_t p = Ap[c]; p < Ap[c + 1]; p++) {
          int a = S.iperm[Ai[p]], b = S.iperm[c];
          int col = a < b ? a : b, row = a < b ? b : a;  // lower-triangular position
          int s = S.col2sn[col];
          int f = S.sn_first[s], l = S.sn_first[s + 1];
          int64_t ns = l - f, nr = S.sn_rowptr[s + 1] - S.sn_rowptr[s];
          int64_t lrow;
          if (row < l) lrow = row - f;
          else {
            auto b0 = S.sn_rows.begin() + S.sn_rowptr[s], e0 = S.sn_rows.begin() + S.sn_rowptr[s + 1];
            auto it = std::lower_bound(b0, e0, row);
            if (it == e0 || *it != row) { bad[t] = 1; return; }
            lrow = ns + (it - b0);
          }
          ent_task[p] = s;
          ent_dst[p] = (int64_t)(col - f) * (ns + nr) + lrow;
        }
    };
    if (nth == 1) work(0);
    else {
      std::vector<std::thread> th;
      for (unsigned t = 0; t < nth; t++) th.emplace_back(work, t);
      for (auto& x : th) x.join();
    }
    for (unsigned t = 0; t < nth; t++)
      if (bad[t]) { std::fprintf(stderr, "symbolic: asm map failure\n"); rc_b = -11; return; }
    for (int64_t p = 0; p < nnz; p++) S.asm_ptr[ent_task[p] + 1]++;
  }
  for (int s = 0; s < nsup; s++) S.asm_ptr[s + 1] += S.asm_ptr[s];
  S.asm_src.resize(nnz);
  S.asm_dst.resize(nnz);
  {
    std::vector<int64_t> pos(S.asm_ptr.begin(), S.asm_ptr.end() - 1);
    for (int64_t p = 0; p < nnz; p++) {
      int64_t d = pos[ent_task[p]]++;
      S.asm_src[d] = (int)p;
      S.asm_dst[d] = ent_dst[p];
    }
  }
  };

  // ---- update-matrix arena ----
  // U_s is written by front s and read by parent(s).  The numeric phase runs as a dataflow graph (a front
  // starts as soon as its children are complete, with no level barrier), so a block may only be reused by a
  // front that is ordered AFTER its last reader by the dependency graph itself: U_c (c a child of s) is dead
  // once s completes, and exactly the proper ancestors of s start after that.  Every front therefore hands
  // the blocks of its subtree that are dead at its completion to its parent (free lists merged small into
  // large); a front allocates from the lists of its children before growing the arena.
  auto part_c = [&]() {
  S.upd_off.assign(nsup, 0);
  {
    // size -> offset; the nodes come from a pool (the lists are built and torn down ~nsup times)
    std::pmr::unsynchronized_pool_resource pool;
    typedef std::pmr::multimap<int64_t, int64_t> FreeList;
    std::vector<FreeList*> fl(nsup, nullptr);
    int64_t top = 0;
    for (int s = 0; s < nsup; s++) {  // supernodes are numbered in postorder: children first
      FreeList* mine = nullptr;
      for (int c : kids[s]) {
        FreeList* fc = fl[c];
        fl[c] = nullptr;
        if (!fc) continue;
        if (!mine) { mine = fc; continue; }
        if (fc->size() > mine->size()) std::swap(fc, mine);
        mine->insert(fc->begin(), fc->end());
        delete fc;
      }
      const int64_t nr = S.sn_rowptr[s + 1] - S.sn_rowptr[s];
      const int64_t sz = nr * nr;
      if (sz > 0) {
        bool got = false;
        if (mine) {
          auto it = mine->lower_bound(sz);
          if (it != mine->end() && it->first <= 2 * sz + 64) {
            const int64_t off = it->second, bs = it->first;
            mine->erase(it);
            if (bs - sz >= 64) mine->emplace(bs - sz, off + sz);
            S.upd_off[s] = off;
            got = true;
          }
        }
        if (!got) { S.upd_off[s] = top; top += sz; }
      }
      for (int c : kids[s]) {
        const int64_t nrc = S.sn_rowptr[c + 1] - S.sn_rowptr[c];
        if (nrc > 0) {
          if (!mine) mine = new FreeList(&pool);
          mine->emplace(nrc * nrc, S.upd_off[c]);
        }
      }
      fl[s] = mine;
    }
    for (FreeList* f : fl) delete f;
    S.upd_total = top;
  }
  };
  if (nsup < 2000) { part_a(); part_b(); part_c(); }
  else {
    std::thread tb(part_b), tc(part_c);
    part_a();
    tb.join(); tc.join();
  }
  TMARK("sym: schedule | assembly map | arena");
  if (rc_a) return rc_a;
  if (rc_b) return rc_b;
  return 0;
}

// Ordering for KKT matrices with dense diagonal blocks (PSD / dense SOC cones).  Minimum degree is myopic
// there: a dense block inflates the degree of its rows, so the coupling variables are eliminated first and
// the blocks smear into each other (measured on config C5: nnzL 4.9e9 instead of ~1e8).  Here every dense
// block is contracted to ONE vertex of the ordering graph; for AMD these vertices are forced to be
// eliminated first (each turns into an element = the clique it induces on the coupling variables, which is
// exactly what eliminating the block does), for ND they are ordinary vertices.  The contracted order is
// expanded back (a block vertex becomes its rows, in natural order) and both candidates are judged on the
// TRUE pattern with the device-time model.
int order_with_groups(int n, const int64_t* Ap, const int32_t* Ai, const int* group, int ngroups,
                      const SymbolicOptions& opt, std::vector<int>& perm_out, int* kind_out) {
  // contracted vertex ids: singletons first (in index order), then one per group
  std::vector<int> cid(n, -1);
  int nc = 0;
  for (int v = 0; v < n; v++) if (group[v] < 0) cid[v] = nc++;
  const int ns = nc;
  for (int v = 0; v < n; v++) if (group[v] >= 0) cid[v] = ns + group[v];
  nc = ns + ngroups;
  // contracted upper-triangular CSC (duplicates removed)
  std::vector<std::vector<int>> cols(nc);
  for (int j = 0; j < n; j++)
    for (int64_t p = Ap[j]; p < Ap[j + 1]; p++) {
      int a = cid[Ai[p]], b = cid[j];
      if (a == b) continue;
      if (a > b) std::swap(a, b);
      cols[b].push_back(a);
    }
  std::vector<int64_t> Cp(nc + 1, 0);
  std::vector<int32_t> Ci;
  for (int j = 0; j < nc; j++) {
    auto& c = cols[j];
    std::sort(c.begin(), c.end());
    c.erase(std::unique(c.begin(), c.end()), c.end());
    for (int a : c) Ci.push_back(a);
    Ci.push_back(j);   // structural diagonal (the orderings ignore it)
    Cp[j + 1] = (int64_t)Ci.size();
    std::vector<int>().swap(c);
  }
  // full adjacency for AMD with forced-first group vertices
  std::vector<int64_t> xadj(nc + 1, 0);
  for (int j = 0; j < nc; j++)
    for (int64_t p = Cp[j]; p < Cp[j + 1]; p++) if (Ci[p] != j) { xadj[Ci[p] + 1]++; xadj[j + 1]++; }
  for (int j = 0; j < nc; j++) xadj[j + 1] += xadj[j];
  std::vector<int> adj(xadj[nc]);
  {
    std::vector<int64_t> pos(xadj.begin(), xadj.end() - 1);
    for (int j = 0; j < nc; j++)
      for (int64_t p = Cp[j]; p < Cp[j + 1]; p++) if (Ci[p] != j) { adj[pos[Ci[p]]++] = j; adj[pos[j]++] = Ci[p]; }
  }
  std::vector<char> forced(nc, 0);
  for (int g = 0; g < ngroups; g++) forced[ns + g] = 1;
  std::vector<int> oa, on;
  amd_graph(nc, xadj, adj, opt.amd_dense_scale, oa, &forced);
  nd_order(nc, Cp.data(), Ci.data(), opt.amd_dense_scale, opt.nd_leaf, on);
  if ((int)oa.size() != nc || (int)on.size() != nc) return -6;
  // expand
  std::vector<std::vector<int>> members(ngroups);
  std::vector<int> single(ns);
  for (int v = 0; v < n; v++) { if (group[v] >= 0) members[group[v]].push_back(v); else single[cid[v]] = v; }
  auto expand = [&](const std::vector<int>& o, std::vector<int>& out) {
    out.clear(); out.reserve(n);
    for (int c : o) { if (c < ns) out.push_back(single[c]); else for (int v : members[c - ns]) out.push_back(v); }
  };
  std::vector<int> pa, pn;
  expand(oa, pa); expand(on, pn);
  if ((int)pa.size() != n || (int)pn.size() != n) return -6;
  Symbolic Sa, Sn;
  int ra = build(n, Ap, Ai, pa, opt, Sa, true);
  if (ra) return ra;
  int rn = build(n, Ap, Ai, pn, opt, Sn, true, 30.0 * Sa.flops_simplicial + 1e9);
  if (rn < 0) return rn;
  if (rn == 1) { Sn.flops_stored = 1e300; Sn.nnzL_stored = 0; Sn.nlevels = 0; }
  auto model = [](const Symbolic& s) {
    return s.flops_stored / 1.0e13 + (double)s.nnzL_stored * 8.0 / 2.0e12 + 10e-6 * s.nlevels;
  };
  if (timing_on()) std::fprintf(stderr, "[cb timing] grouped ordering: AMD nnzL %.3e flops %.3e levels %d | ND nnzL %.3e flops %.3e levels %d\n",
                                (double)Sa.nnzL_stored, Sa.flops_stored, Sa.nlevels, (double)Sn.nnzL_stored, Sn.flops_stored, Sn.nlevels);
  const bool use_nd = (opt.ordering == ORDER_ND) || (opt.ordering != ORDER_AMD && model(Sn) < model(Sa));
  perm_out = use_nd ? pn : pa;
  if (kind_out) *kind_out = use_nd ? ORDER_ND : ORDER_AMD;
  return 0;
}

int analyse(int n, const int64_t* Ap, const int32_t* Ai, const int* perm_in,
            const SymbolicOptions& opt_in, Symbolic& S) {
  if (n <= 0) return -1;
  SymbolicOptions opt = opt_in;
  if (const char* e = std::getenv("CB_RELAX_SUBTREE")) opt.relax_subtree = std::atoi(e);   // tuning knob
  if (const char* e = std::getenv("CB_ND_LEAF")) opt.nd_leaf = std::atoi(e);               // tuning knob (overrides the caller)
  for (int j = 0; j < n; j++) {
    if (!(Ap[j] < Ap[j + 1])) return -2;  // empty column (qdldl.rs:222-225)
    for (int64_t p = Ap[j]; p < Ap[j + 1]; p++)
      if (Ai[p] > j || Ai[p] < 0) return -3;  // not upper triangular
  }
  std::vector<int> perm0;
  int kind = opt.ordering;
  if (perm_in) {
    kind = ORDER_GIVEN;
    perm0.assign(perm_in, perm_in + n);
    std::vector<char> seen(n, 0);
    for (int k = 0; k < n; k++) {
      if (perm0[k] < 0 || perm0[k] >= n || seen[perm0[k]]) return -5;
      seen[perm0[k]] = 1;
    }
  } else if (kind == ORDER_AMD) {
    amd_order(n, Ap, Ai, opt.amd_dense_scale, perm0);
  } else if (kind == ORDER_ND) {
    double t_last = tnow();
    nd_order(n, Ap, Ai, opt.amd_dense_scale, opt.nd_leaf, perm0);
    TMARK("ordering: ND");
  } else {
    // ORDER_BEST: evaluate both, pick by a simple device-time model
    // model: dense flops at ~10 TF/s effective + memory at ~2 TB/s + 10 us per level
    auto model = [](const Symbolic& s) {
      return s.flops_stored / 1.0e13 + (double)s.nnzL_stored * 8.0 / 2.0e12 + 10e-6 * s.nlevels;
    };
    // Nested dissection goes first (it runs on all host threads; minimum degree is one sequential pass that costs
    // several times as much on a large graph) and the minimum-degree candidate is only produced when it could pay
    // for itself: the most it can save per refactorisation is taken as 70 % of the ND candidate's flop + memory
    // time plus half of its level latency (its fill is rarely below a third of ND's and its tree is never much
    // shallower than a balanced dissection tree), a solve is taken as 25 refactorisations, and one minimum-degree
    // pass as 1 us per vertex.  When that saving cannot cover the pass, the ND analysis is simply finished in
    // place.  The rule reads the candidate's statistics only, so the choice is the same on every run and host;
    // CB_ORDER_EXHAUSTIVE=1 always evaluates both.
    static const bool exhaustive = std::getenv("CB_ORDER_EXHAUSTIVE") != nullptr && std::atoi(std::getenv("CB_ORDER_EXHAUSTIVE")) != 0;
    std::vector<int> pa, pn;
    // The minimum-degree pass starts on a thread of its own right away and is told to stop if the rule below finds
    // that it cannot pay; when it is needed, its ordering and statistics are ready by the time the ND side is.
    std::atomic<bool> amd_cancel{false};
    Symbolic Sa;
    int ra = 0;
    std::thread amd_thread;
    // only where a spare core is certain: on a small host the extra thread takes time from the dissection's own
    // threads (8 cores, C2: 0.33 s -> 0.37 s when the pass is not needed, 1.30 s -> 0.97 s when it is)
    bool speculative = host_threads() >= 16;
    if (const char* e = std::getenv("CB_ORDER_SPECULATIVE")) speculative = std::atoi(e) != 0;
    if (speculative)
      amd_thread = std::thread([&]() {
        amd_order(n, Ap, Ai, opt.amd_dense_scale, pa, &amd_cancel);
        if ((int)pa.size() == n && !amd_cancel.load()) ra = build(n, Ap, Ai, pa, opt, Sa, true);
      });
    struct Joiner { std::thread& t; std::atomic<bool>& c; ~Joiner() { if (t.joinable()) { c.store(true); t.join(); } } } joiner{amd_thread, amd_cancel};
    // the dissection stops by itself when a single separator is already beyond the flop cap used below (C4: the first
    // cut of the 2.5e6-vertex graph has 3.3e5 vertices): minimum degree is then the only candidate
    nd_order(n, Ap, Ai, opt.amd_dense_scale, opt.nd_leaf, pn, exhaustive ? 0.0 : 1e12);
    if (pn.empty() && !exhaustive) {
      if (speculative) amd_thread.join();
      else {
        amd_order(n, Ap, Ai, opt.amd_dense_scale, pa);
      }
      if ((int)pa.size() != n) return -6;
      S.ordering_used = ORDER_AMD;
      return build(n, Ap, Ai, pa, opt, S, false);
    }
    if ((int)pn.size() != n) return -6;
    const std::function<bool(const Symbolic&)> amd_cannot_pay = [&](const Symbolic& sn) {
      if (exhaustive) return false;
      const double saving = 0.7 * (sn.flops_stored / 1.0e13 + (double)sn.nnzL_stored * 8.0 / 2.0e12) + 0.5 * 10e-6 * sn.nlevels;
      const bool no = 25.0 * saving < 1e-6 * (double)n;
      // tell the speculative pass to stop NOW: tearing down its quotient graph (millions of small vectors, 0.3 s on C4)
      // then overlaps with the rest of this analysis instead of being waited for at the join
      if (no) amd_cancel.store(true);
      return no;
    };
    Symbolic Sn;
    // a candidate beyond 1e12 simplicial flops is not analysed further before the other one is known
    int rn = build(n, Ap, Ai, pn, opt, Sn, false, 1e12, &amd_cannot_pay);
    if (rn < 0) return rn;
    if (rn == 0) { S = std::move(Sn); S.ordering_used = ORDER_ND; return 0; }      // (the joiner stops the AMD thread)
    if (speculative) amd_thread.join();
    else {
      amd_order(n, Ap, Ai, opt.amd_dense_scale, pa);
      if ((int)pa.size() == n) ra = build(n, Ap, Ai, pa, opt, Sa, true);
    }
    if ((int)pa.size() != n) return -6;
    if (ra) return ra;
    if (rn == 1) {      // ND statistics still missing: same early rejection relative to the AMD candidate as before
      rn = build(n, Ap, Ai, pn, opt, Sn, true, 30.0 * Sa.flops_simplicial + 1e9);
      if (rn < 0) return rn;
    } else if (Sn.flops_simplicial > 30.0 * Sa.flops_simplicial + 1e9) rn = 1;
    if (rn == 1) { Sn.flops_stored = 1e300; Sn.nnzL_stored = 0; Sn.nlevels = 0; }   // hopeless: rejected early
    if (model(Sn) < model(Sa)) { perm0.swap(pn); kind = ORDER_ND; }
    else { perm0.swap(pa); kind = ORDER_AMD; }
  }
  if ((int)perm0.size() != n) return -6;
  S.ordering_used = kind;
  return build(n, Ap, Ai, perm0, opt, S, false);
}

int analyse_schur(int n, const int64_t* Ap, const int32_t* Ai, const int* perm_in, const std::vector<int>& schur,
                  const SymbolicOptions& opt_in, Symbolic& S) {
  if (n <= 0) return -1;
  const int k = (int)schur.size();
  if (k < 1 || k >= n) return -4;
  std::vector<char> in_s(n, 0);
  for (int v : schur) {
    if (v < 0 || v >= n || in_s[v]) return -4;
    in_s[v] = 1;
  }
  for (int j = 0; j < n; j++) {
    if (!(Ap[j] < Ap[j + 1])) return -2;
    for (int64_t p = Ap[j]; p < Ap[j + 1]; p++)
      if (Ai[p] > j || Ai[p] < 0) return -3;
  }
  std::vector<int> perm0;
  int kind = ORDER_GIVEN;
  if (perm_in) {
    perm0.assign(perm_in, perm_in + n);
    std::vector<char> seen(n, 0);
    for (int q = 0; q < n; q++) {
      if (perm0[q] < 0 || perm0[q] >= n || seen[perm0[q]]) return -5;
      seen[perm0[q]] = 1;
      if ((q >= n - k) != (in_s[perm0[q]] != 0)) return -5;
    }
  } else {
    // B's own ordering on the subgraph it induces (diagonal added: a B column may hold entries in S rows only)
    std::vector<int> bidx, bpos(n, -1);
    for (int v = 0; v < n; v++) if (!in_s[v]) { bpos[v] = (int)bidx.size(); bidx.push_back(v); }
    const int nb = (int)bidx.size();
    std::vector<int64_t> Bp(nb + 1, 0);
    std::vector<int32_t> Bi;
    for (int c = 0; c < nb; c++) {
      const int v = bidx[c];
      for (int64_t p = Ap[v]; p < Ap[v + 1]; p++) if (bpos[Ai[p]] >= 0 && Ai[p] != v) Bi.push_back(bpos[Ai[p]]);
      Bi.push_back(c);
      Bp[c + 1] = (int64_t)Bi.size();
    }
    SymbolicOptions ob = opt_in;
    ob.schur_first = -1;
    Symbolic SB;
    if (int rc = analyse(nb, Bp.data(), Bi.data(), nullptr, ob, SB)) return rc;
    for (int q = 0; q < nb; q++) perm0.push_back(bidx[SB.perm[q]]);
    perm0.insert(perm0.end(), schur.begin(), schur.end());
    kind = SB.ordering_used;
  }
  SymbolicOptions opt = opt_in;
  if (const char* e = std::getenv("CB_RELAX_SUBTREE")) opt.relax_subtree = std::atoi(e);
  opt.schur_first = n - k;
  S.ordering_used = kind;
  return build(n, Ap, Ai, perm0, opt, S, false);
}

// ---------------------------------------------------------------------------------------------------------
// Subtree-to-rank mapping (see symbolic.h).  Fronts are numbered in post-order, so children precede parents.
int plan_shards(int nsup, const int* sn_first, const int64_t* sn_rowptr, const int* sn_parent, int nranks,
                ShardPlan& out) {
  if (nsup <= 0 || nranks < 1) return -1;
  out = ShardPlan();
  out.nranks = nranks;
  std::vector<double> fl(nsup), sub(nsup);
  std::vector<int> level(nsup, 0);
  for (int s = 0; s < nsup; s++) {
    const double ns = sn_first[s + 1] - sn_first[s], nr = (double)(sn_rowptr[s + 1] - sn_rowptr[s]);
    fl[s] = ns * ns * ns / 3.0 + ns * ns * nr + ns * nr * nr;
    sub[s] = fl[s];
  }
  for (int s = 0; s < nsup; s++) {
    const int p = sn_parent[s];
    if (p >= 0) { if (p <= s) return -2; sub[p] += sub[s]; }
  }
  std::vector<std::vector<int>> kids(nsup);
  std::vector<int> roots;
  for (int s = 0; s < nsup; s++) { if (sn_parent[s] >= 0) kids[sn_parent[s]].push_back(s); else roots.push_back(s); }
  double total = 0.0;
  for (int r : roots) total += sub[r];
  out.total_flops = total;

  // candidate set = subtree roots below the current top part, kept as a max-heap on subtree flops
  auto cmp = [&](int a, int b) { return sub[a] < sub[b] || (sub[a] == sub[b] && a > b); };
  std::vector<int> cand(roots);
  std::make_heap(cand.begin(), cand.end(), cmp);
  std::vector<char> in_top(nsup, 0);
  double top = 0.0;
  auto makespan = [&](const std::vector<int>& c) {
    std::vector<int> srt(c);
    std::sort(srt.begin(), srt.end(), [&](int a, int b) { return sub[a] > sub[b] || (sub[a] == sub[b] && a < b); });
    std::vector<double> load(nranks, 0.0);
    for (int s : srt) *std::min_element(load.begin(), load.end()) += sub[s];
    return *std::max_element(load.begin(), load.end());
  };
  double best = top + makespan(cand);
  std::vector<int> best_cand(cand);
  std::vector<char> best_top(in_top);
  double best_topfl = top;
  int since = 0;
  const int patience = 16 * nranks, max_cand = 4096;
  while (nranks > 1 && !cand.empty() && since < patience && (int)cand.size() < max_cand) {
    std::pop_heap(cand.begin(), cand.end(), cmp);
    const int s = cand.back();
    cand.pop_back();
    if (kids[s].empty()) { cand.push_back(s); std::push_heap(cand.begin(), cand.end(), cmp); break; }   // largest is a leaf
    in_top[s] = 1;
    top += fl[s];
    for (int c : kids[s]) { cand.push_back(c); std::push_heap(cand.begin(), cand.end(), cmp); }
    const double t = top + makespan(cand);
    if (t < best * (1.0 - 1e-9)) { best = t; best_cand = cand; best_top = in_top; best_topfl = top; since = 0; }
    else since++;
  }
  // assignment of the best configuration
  out.owner.assign(nsup, -1);
  out.rank_flops.assign(nranks, 0.0);
  std::sort(best_cand.begin(), best_cand.end(), [&](int a, int b) { return sub[a] > sub[b] || (sub[a] == sub[b] && a < b); });
  for (int s : best_cand) {
    const int g = (int)(std::min_element(out.rank_flops.begin(), out.rank_flops.end()) - out.rank_flops.begin());
    out.rank_flops[g] += sub[s];
    out.owner[s] = g;
    if (sn_parent[s] >= 0) out.cut_roots.push_back(s);
  }
  std::sort(out.cut_roots.begin(), out.cut_roots.end());
  // owners flow down the subtrees (parents have larger indices than children)
  for (int s = nsup - 1; s >= 0; s--) {
    const int p = sn_parent[s];
    if (best_top[s]) { out.owner[s] = -1; continue; }
    if (out.owner[s] < 0 && p >= 0) out.owner[s] = out.owner[p];
  }
  out.top_flops = best_topfl;
  for (int s : out.cut_roots) {
    const int64_t nr = sn_rowptr[s + 1] - sn_rowptr[s];
    out.exchange_doubles += nr * nr;
    out.exchange_vec += nr;
  }
  for (int s = 0; s < nsup; s++) {
    if (!best_top[s]) continue;
    int l = 0;
    for (int c : kids[s]) if (best_top[c] && level[c] + 1 > l) l = level[c] + 1;
    level[s] = l;
    if (l + 1 > out.top_levels) out.top_levels = l + 1;
  }
  const double mx = *std::max_element(out.rank_flops.begin(), out.rank_flops.end());
  out.model_speedup = total > 0.0 ? total / (mx + out.top_flops) : 1.0;
  return 0;
}

}  // namespace cb
