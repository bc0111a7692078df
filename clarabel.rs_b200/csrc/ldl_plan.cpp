// Host-side plan builders of the multifrontal LDL^T (see ldl_plan.h).  Pure functions of the symbolic analysis and
// the shard view; LDLObject::init (ldl.cu) uploads what they return.
#include "ldl_plan.h"

#include <algorithm>
#include <thread>

namespace cb {

namespace {

int ns_of(const Symbolic& S, int s) { return S.sn_first[s + 1] - S.sn_first[s]; }
int nr_of(const Symbolic& S, int s) { return (int)(S.sn_rowptr[s + 1] - S.sn_rowptr[s]); }

// fronts factored by k_factor_df's D, R and T tasks
bool is_big(const Symbolic& S, int s) { return nr_of(S, s) >= CB_BIG_NR && ns_of(S, s) <= CB_PB_MAXNS; }

// [nsup] 1 for the fronts that appear in the queue order
std::vector<char> queued(const QueueOrder& q, int nsup) {
  std::vector<char> m(nsup, 0);
  for (const auto& ph : q)
    for (const auto& lev : ph)
      for (int s : lev) m[s] = 1;
  return m;
}

}  // namespace

QueueOrder queue_order(const Symbolic& S, const std::vector<int>& owner, int rank) {
  const bool sharded = !owner.empty();
  QueueOrder q(sharded ? 2 : 1, std::vector<std::vector<int>>(S.nlevels));
  for (int s = 0; s < S.nsup; s++) {
    const int ph = !sharded ? 0 : owner[s] == rank ? 0 : owner[s] < 0 ? 1 : -1;
    if (ph >= 0) q[ph][S.sn_level[s]].push_back(s);
  }
  return q;
}

// Tree level 0 (leaves: no dependencies) is factored by plain launches before k_factor_df.  Single-column fronts take
// one thread each (k_factor_leaf1), the others one fused CTA each (k_factor_level), grouped by the shared-memory class
// of their panel.  Big fronts (k_factor_df's tasks) and fronts outside the first phase are parked at the end (a
// sharded top part has no leaves; a Schur handle's S fronts are never factored).
Level0Plan build_level0_plan(const Symbolic& S, const std::vector<int>& owner, int rank, int smem_cap) {
  Level0Plan P;
  P.level_tasks = S.level_tasks;
  if (S.nlevels == 0) return P;
  QueueOrder q = queue_order(S, owner, rank);
  q.resize(1);
  const std::vector<char> mine = queued(q, S.nsup);
  const long long classes[3] = {1024, 5632, smem_cap};  // 8 KB, 44 KB, ~225 KB panels
  const int b = S.level_ptr[0], e = S.level_ptr[1];
  std::vector<int> order[4], order1, big, not_mine;
  for (int t = b; t < e; t++) {
    const int s = S.level_tasks[t];
    const long long ns = ns_of(S, s), nr = nr_of(S, s);
    if (is_big(S, s)) { big.push_back(s); continue; }
    if (!mine[s]) { not_mine.push_back(s); continue; }
    if (ns == 1) { order1.push_back(s); continue; }
    const long long p = (ns + nr) * ns;
    int c = p <= classes[0] ? 0 : p <= classes[1] ? 1 : p <= classes[2] ? 2 : 3;
    order[c].push_back(s);
  }
  int pos = b;
  if (!order1.empty()) {
    P.segs.push_back(LaunchSeg{true, pos, (int)order1.size(), 0, 256});
    for (int s : order1) P.level_tasks[pos++] = s;
  }
  for (int c = 3; c >= 0; c--) {
    if (order[c].empty()) continue;
    P.segs.push_back(LaunchSeg{false, pos, (int)order[c].size(), c == 3 ? 0 : (int)classes[c], c == 0 ? 64 : 256});
    for (int s : order[c]) P.level_tasks[pos++] = s;
  }
  for (int s : big) P.level_tasks[pos++] = s;
  for (int s : not_mine) P.level_tasks[pos++] = s;
  return P;
}

// Everything above level 0 becomes queue tasks in level order: an F task per small front, and per big front a D task,
// R tasks and T tasks.  Every task record carries the front's constants and the range of its child records, so a
// task starts with two dependent loads (record, child records) instead of walking the tree arrays.
FactorPlan build_factor_plan(const Symbolic& S, const std::vector<int>& owner, int rank) {
  FactorPlan P;
  const int nsup = S.nsup;
  // big fronts in level order and the TS x TS tiles of their update matrices
  P.big_pos.assign(nsup, -1);
  P.tile_base.assign(nsup, -1);
  int nbig = 0, ntiles = 0;
  for (int s : S.level_tasks) {
    if (!is_big(S, s)) continue;
    const int nt = (nr_of(S, s) + TS - 1) / TS;
    P.big_pos[s] = nbig++;
    P.tile_base[s] = ntiles;
    ntiles += nt * (nt + 1) / 2;
  }
  const std::vector<int>& big_pos = P.big_pos;
  const std::vector<int>& tile_base = P.tile_base;

  // small children (nr <= CB_SMALL_CHILD) of big fronts: one dst-sorted (src,dst) list per panel and per tile
  std::vector<signed char> small(nsup, 0);
  {
    struct Ent { int key; int dst; int src; };
    std::vector<Ent> pe, te;
    {
      // two passes over the children on host threads: count (pe / te entries per child), prefix sums, fill -- the
      // entry order (child, column b, row a) is the one of a single loop
      const unsigned hc2 = std::max(1u, std::min(16u, host_threads()));
      const unsigned nth2 = nsup < 20000 ? 1u : hc2;
      std::vector<int64_t> npe((size_t)nsup + 1, 0), nte((size_t)nsup + 1, 0);
      auto eligible = [&](int c) {
        const int p = S.sn_parent[c];
        if (p < 0 || big_pos[p] < 0) return false;
        const int nrc = nr_of(S, c);
        if (nrc > CB_SMALL_CHILD) return false;
        if (S.upd_off[c] + (int64_t)nrc * nrc > 0x7fffffffLL) return false;   // int32 source indices
        return true;
      };
      auto run = [&](auto&& fn) {
        if (nth2 == 1) { fn(0, nsup); return; }
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nth2; t++)
          th.emplace_back([&, t]() { fn((int)((int64_t)nsup * t / nth2), (int)((int64_t)nsup * (t + 1) / nth2)); });
        for (auto& x : th) x.join();
      };
      run([&](int c0, int c1) {
        for (int c = c0; c < c1; c++) {
          if (!eligible(c)) continue;
          small[c] = 1;
          const int p = S.sn_parent[c];
          const int64_t b0 = S.sn_rowptr[c];
          const int nrc = nr_of(S, c);
          const int pns = ns_of(S, p);
          int64_t np_ = 0;
          for (int b = 0; b < nrc; b++) if (S.rel[b0 + b] < pns) np_ += nrc - b;
          npe[c + 1] = np_;
          nte[c + 1] = (int64_t)nrc * (nrc + 1) / 2 - np_;
        }
      });
      for (int c = 0; c < nsup; c++) { npe[c + 1] += npe[c]; nte[c + 1] += nte[c]; }
      pe.resize((size_t)npe[nsup]);
      te.resize((size_t)nte[nsup]);
      run([&](int c0, int c1) {
        for (int c = c0; c < c1; c++) {
          if (!small[c]) continue;
          const int p = S.sn_parent[c];
          const int64_t b0 = S.sn_rowptr[c];
          const int nrc = nr_of(S, c);
          const int pns = ns_of(S, p);
          const int pld = pns + nr_of(S, p);
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
    std::thread tb([&]() { build(te, ntiles, P.sc_tile_ptr, P.sc_tile_src, P.sc_tile_dst); });
    build(pe, nbig, P.sc_panel_ptr, P.sc_panel_src, P.sc_panel_dst);
    tb.join();
  }

  // rows of child c that land in its parent's pivot block (rel is ascending inside a child)
  auto child_nb = [&](int c) {
    const int* rb = S.rel.data() + S.sn_rowptr[c];
    const int* re = S.rel.data() + S.sn_rowptr[c + 1];
    return (int)(std::lower_bound(rb, re, ns_of(S, S.sn_parent[c])) - rb);
  };
  const QueueOrder queue = queue_order(S, owner, rank);
  const std::vector<char> mine = queued(queue, nsup);
  P.cnt_init.assign(4 * (size_t)nsup, 0);
  int* pend = P.cnt_init.data();
  int* rows_left = P.cnt_init.data() + 2 * (size_t)nsup;
  int* tiles_left = P.cnt_init.data() + 3 * (size_t)nsup;
  for (int s = 0; s < nsup; s++) {
    const int p = S.sn_parent[s];
    const bool presolved = (S.sn_level[s] == 0 && !is_big(S, s));
    if (p >= 0 && !presolved && mine[s]) pend[p]++;   // sharded: another rank's front is complete before the top phase starts
  }
  std::vector<DFTask>& tk = P.tasks;
  std::vector<DFChildRec>& recs = P.recs;
  auto push_task = [&](int kind, int s, int a, int b, int d0, int d1, int e0, int e1) {
    DFTask t{};
    t.kind = kind; t.s = s; t.a = a; t.b = b;
    t.ns = ns_of(S, s); t.nr = nr_of(S, s); t.f = S.sn_first[s];
    t.d0 = d0; t.d1 = d1; t.e0 = e0; t.e1 = e1;
    t.poff = S.panel_off[s]; t.uoff = S.upd_off[s];
    tk.push_back(t);
  };
  auto push_rec = [&](int c, int a0, int a1, int b0, int b1) {
    DFChildRec r{};
    r.uoff = S.upd_off[c]; r.relp = S.sn_rowptr[c];
    r.nrc = nr_of(S, c);
    r.a0 = a0; r.a1 = a1; r.b0 = b0; r.b1 = b1;
    const int* rl = S.rel.data() + r.relp;
    const bool rc_ = rl[a1 - 1] - rl[a0] == a1 - 1 - a0, cc_ = rl[b1 - 1] - rl[b0] == b1 - 1 - b0;
    r.contig = (rc_ ? 1 : 0) | (cc_ ? 2 : 0);
    r.ra0 = rl[a0];
    r.rb0 = rl[b0];
    recs.push_back(r);
  };
  std::vector<int> kidsbuf;
  // the children of a big front that go through child records (the small ones use the sorted entry lists)
  auto heavy_kids = [&](int s) {
    kidsbuf.clear();
    for (int64_t ci = S.child_ptr[s]; ci < S.child_ptr[s + 1]; ci++) {
      const int c = S.child_list[ci];
      if (!small[c] && S.sn_rowptr[c + 1] > S.sn_rowptr[c]) kidsbuf.push_back(c);
    }
  };
  for (size_t ph = 0; ph < queue.size(); ph++) {
    for (int l = 0; l < S.nlevels; l++) {
      const std::vector<int>& lev = queue[ph][l];
      for (int s : lev) if (!is_big(S, s) && l > 0) push_task(0, s, 0, 0, 0, 0, 0, 0);
      for (int s : lev) if (is_big(S, s)) {
        heavy_kids(s);
        const int d0 = (int)recs.size();
        for (int c : kidsbuf) if (const int nb = child_nb(c)) push_rec(c, 0, nb, 0, nb);
        push_task(1, s, 0, 0, d0, (int)recs.size(), P.sc_panel_ptr[big_pos[s]], P.sc_panel_ptr[big_pos[s] + 1]);
      }
      for (int s : lev) if (is_big(S, s)) {
        heavy_kids(s);
        const int ns = ns_of(S, s), nr = nr_of(S, s);
        const int nb = (nr + DF_RB - 1) / DF_RB;
        rows_left[s] = nb;
        for (int b = 0; b < nb; b++) {
          const int g0 = ns + b * DF_RB, g1 = std::min(ns + nr, g0 + DF_RB);
          const int d0 = (int)recs.size();
          for (int c : kidsbuf) {
            const int cnb = child_nb(c);
            if (cnb == 0) continue;
            const int* rb = S.rel.data() + S.sn_rowptr[c];
            const int* re = S.rel.data() + S.sn_rowptr[c + 1];
            const int alo = (int)(std::lower_bound(rb, re, g0) - rb), ahi = (int)(std::lower_bound(rb, re, g1) - rb);
            if (ahi > alo) push_rec(c, alo, ahi, 0, cnb);
          }
          push_task(2, s, b, 0, d0, (int)recs.size(), P.sc_panel_ptr[big_pos[s]], P.sc_panel_ptr[big_pos[s] + 1]);
        }
      }
      for (int s : lev) if (is_big(S, s)) {
        heavy_kids(s);
        const int ns = ns_of(S, s), nr = nr_of(S, s);
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
            const int d0 = (int)recs.size();
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
                push_rec(kidsbuf[k], a0, a1, b0, b1);
                if (dense) ndense++;
              }
            const int t = tile_base[s] + tix;
            push_task(3, s, ti, tj, d0, (int)recs.size(), P.sc_tile_ptr[t], P.sc_tile_ptr[t + 1]);
            tk.back().ndense = ndense;
          }
      }
    }
    if (ph == 0) P.ntask_owned = (int)tk.size();
  }
  return P;
}

// Level-0 narrow fronts get plain kernels, everything else becomes queue tasks in level order -- batches of narrow
// fronts, and for every wide front a head task (pivot block + first rows) followed by row tasks when the panel exceeds
// the shared-memory slab.
SolvePlan build_solve_plan(const Symbolic& S, const std::vector<int>& owner, int rank, int cap) {
  SolvePlan P;
  const int nsup = S.nsup, n = S.n;
  // per-destination gather lists of the children's update-vector entries, beside the task building
  std::thread th_gather([&]() {
    std::vector<int>& gptr = P.gat_ptr;
    gptr.assign((size_t)n + S.sn_rows.size() + 1, 0);
    for (int c = 0; c < nsup; c++) {
      const int p = S.sn_parent[c];
      if (p < 0) continue;
      const int64_t pbase = (int64_t)S.sn_first[p] + S.sn_rowptr[p];
      for (int64_t t = S.sn_rowptr[c]; t < S.sn_rowptr[c + 1]; t++) gptr[pbase + S.rel[t] + 1]++;
    }
    for (size_t i = 0; i + 1 < gptr.size(); i++) gptr[i + 1] += gptr[i];
    P.gat_src.assign(S.sn_rows.size() ? S.sn_rows.size() : 1, 0);
    std::vector<int> pos(gptr.begin(), gptr.end() - 1);
    // children in child_list order so that every destination sums in a fixed, reproducible order
    for (int p = 0; p < nsup; p++) {
      const int64_t pbase = (int64_t)S.sn_first[p] + S.sn_rowptr[p];
      for (int64_t ci = S.child_ptr[p]; ci < S.child_ptr[p + 1]; ci++) {
        const int c = S.child_list[ci];
        for (int64_t t = S.sn_rowptr[c]; t < S.sn_rowptr[c + 1]; t++) P.gat_src[pos[pbase + S.rel[t]]++] = (int)t;
      }
    }
  });
  struct Join { std::thread& t; ~Join() { t.join(); } } join_gather{th_gather};

  auto wide = [&](int s) { return ns_of(S, s) > CB_SOLVE_SMALL_NS; };
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
  const QueueOrder queue = queue_order(S, owner, rank);
  std::vector<int>& f2t = P.front2task;
  f2t.assign(nsup, -1);
  std::vector<int> nrt_of(nsup, 0), rh_of(nsup, 0), chunk_of(nsup, 0);
  std::vector<SVTask>& tk = P.tasks;
  const int per = SV_NT / 32;
  for (size_t ph = 0; ph < queue.size(); ph++) {
    std::vector<std::vector<int>> lev_small(S.nlevels), lev_big(S.nlevels);
    for (int l = 0; l < S.nlevels; l++)
      for (int s : queue[ph][l]) {
        // leaves of the first phase only (a sharded top part has none; a Schur handle's S fronts are never solved)
        if (ph == 0 && !wide(s) && !has_kids(s)) { (ns_of(S, s) == 1 ? P.leaf1 : P.leafn).push_back(s); continue; }
        if (ph == 0 && wide(s) && !has_kids(s) && nr_of(S, s) <= 1024) {
          P.leafw.push_back(s);
          P.leafw_nrmax = std::max(P.leafw_nrmax, nr_of(S, s));
          continue;
        }
        (wide(s) ? lev_big : lev_small)[l].push_back(s);
      }
    for (int l = 0; l < S.nlevels; l++) {
      for (size_t i = 0; i < lev_small[l].size(); i += per) {
        const int c = (int)std::min<size_t>(per, lev_small[l].size() - i);
        SVTask t{};
        t.kind = 0; t.s = (int)P.fronts.size(); t.cnt = c; t.dep1 = -1; t.dep2 = -1; t.bowner = -1; t.ptask = -1; t.cuoff = -1;
        for (int k = 0; k < c; k++) { f2t[lev_small[l][i + k]] = (int)tk.size(); P.fronts.push_back(lev_small[l][i + k]); }
        tk.push_back(t);
      }
      for (int s : lev_big[l]) {
        const int ns = ns_of(S, s), nr = nr_of(S, s);
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
    if (ph == 0) P.ntask_owned = (int)tk.size();
  }
  const int nt = (int)tk.size();
  // chain children of wide fronts: followed slab by slab instead of awaited as a whole
  std::vector<int> chain_child(nsup, -1), col2sn(n, 0);
  for (int s = 0; s < nsup; s++)
    for (int j = S.sn_first[s]; j < S.sn_first[s + 1]; j++) col2sn[j] = s;
  for (int c = 0; c < nsup; c++) {
    const int p = S.sn_parent[c];
    if (p < 0 || !wide(c) || !wide(p) || chain_child[p] >= 0) continue;
    if (nr_of(S, c) == ns_of(S, p) + nr_of(S, p)) chain_child[p] = c;   // rows(c) is a subset of cols(p)+rows(p): equal sizes = equal sets
  }
  // task of front c covering its row i (of its L21 part)
  auto task_of_row = [&](int c, int i) {
    if (i < rh_of[c]) return f2t[c];
    return f2t[c] + 1 + (i - rh_of[c]) / chunk_of[c];
  };
  P.cnt_init.assign(nt + 2 * (size_t)nsup, 0);
  int* pend = P.cnt_init.data();
  int* fleft = pend + nt;
  int* bleft = fleft + nsup;
  for (int s = 0; s < nsup; s++) {
    if (f2t[s] < 0 || !wide(s)) continue;
    const int ns = ns_of(S, s);
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
      t.bslot = b < 0 ? P.nslots : P.nslots + b;
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
    P.nslots += nrt;
  }
  for (int s = 0; s < nsup; s++) {
    const int p = S.sn_parent[s];
    if (p >= 0 && f2t[s] >= 0 && chain_child[p] != s) pend[f2t[p]]++;   // leaves and other ranks' fronts are complete before the sweep starts
  }
  // wide fronts whose pivot block the factorisation replaces by its inverse (all that this rank factors)
  const std::vector<char> mine = queued(queue, nsup);
  for (int s = 0; s < nsup; s++) if (wide(s) && mine[s]) P.wide.push_back(s);
  return P;
}

SolvePrune build_solve_prune(const Symbolic& S, const SolvePlan& full) {
  SolvePrune X;
  const int nsup = S.nsup;
  X.col2sn.assign(S.n, 0);
  for (int s = 0; s < nsup; s++)
    for (int j = S.sn_first[s]; j < S.sn_first[s + 1]; j++) X.col2sn[j] = s;
  X.cls.assign(nsup, -1);
  for (int s : full.leaf1) X.cls[s] = 0;
  for (int s : full.leafn) X.cls[s] = 1;
  for (int s : full.leafw) X.cls[s] = 2;
  for (int s = 0; s < nsup; s++)
    if (full.front2task[s] >= 0) X.cls[s] = full.tasks[full.front2task[s]].kind == 0 ? 3 : 4;
  X.f2t = full.front2task;
  X.stamp.assign(nsup, 0);
  X.ntf2t.assign(nsup, -1);
  return X;
}

void build_pruned_plan(const Symbolic& S, const SolvePlan& full, SolvePrune& X, const int* cols, size_t k,
                       PrunedPlan& P) {
  P.reached.clear(); P.tasks.clear(); P.pend.clear(); P.fronts.clear(); P.f2t.clear();
  P.leaf1.clear(); P.leafn.clear(); P.leafw.clear();
  P.entries = 0; P.work = 0;
  if (++X.epoch == 0) { std::fill(X.stamp.begin(), X.stamp.end(), 0u); X.epoch = 1; }   // once in 2^32 calls
  const unsigned ep = X.epoch;
  // upward closure: a walk stops at the first front already reached
  for (size_t i = 0; i < k; i++) {
    P.work++;
    for (int s = X.col2sn[cols[i]]; s >= 0 && X.stamp[s] != ep; s = S.sn_parent[s]) {
      X.stamp[s] = ep;
      P.reached.push_back(s);
      P.work++;
    }
  }
  // queue order of the full plan: levels ascending, fronts ascending inside a level
  std::sort(P.reached.begin(), P.reached.end(), [&](int a, int b) {
    P.work++;
    return S.sn_level[a] != S.sn_level[b] ? S.sn_level[a] < S.sn_level[b] : a < b;
  });
  const int per = SV_NT / 32;
  const size_t r = P.reached.size();
  // task indices, level by level: batches of the level's narrow fronts, then the wide fronts' task ranges
  for (size_t i0 = 0; i0 < r;) {
    size_t i1 = i0;
    while (i1 < r && S.sn_level[P.reached[i1]] == S.sn_level[P.reached[i0]]) i1++;
    int in_batch = 0;
    for (size_t i = i0; i < i1; i++) {
      const int s = P.reached[i];
      P.entries += (long long)(S.sn_first[s + 1] - S.sn_first[s]) *
                   (S.sn_first[s + 1] - S.sn_first[s] + S.sn_rowptr[s + 1] - S.sn_rowptr[s]);
      P.work++;
      switch (X.cls[s]) {
        case 0: P.leaf1.push_back(s); break;
        case 1: P.leafn.push_back(s); break;
        case 2: P.leafw.push_back(s); break;
        case 3:
          if (in_batch == 0) {
            SVTask t{};
            t.kind = 0; t.s = (int)P.fronts.size(); t.cnt = 0; t.dep1 = -1; t.dep2 = -1; t.bowner = -1; t.ptask = -1; t.cuoff = -1;
            P.tasks.push_back(t);
          }
          P.tasks.back().cnt++;
          X.ntf2t[s] = (int)P.tasks.size() - 1;
          P.fronts.push_back(s);
          in_batch = in_batch + 1 == per ? 0 : in_batch + 1;
          break;
        default: break;
      }
    }
    for (size_t i = i0; i < i1; i++) {
      const int s = P.reached[i];
      if (X.cls[s] != 4) continue;
      const int h = X.f2t[s], nrt = full.tasks[h].nrt;
      X.ntf2t[s] = (int)P.tasks.size();
      P.tasks.insert(P.tasks.end(), full.tasks.begin() + h, full.tasks.begin() + h + 1 + nrt);
      P.work += 1 + nrt;
    }
    i0 = i1;
  }
  // remapped index fields, counters and the (front, task) pairs
  P.pend.assign(P.tasks.size(), 0);
  for (size_t i = 0; i < r; i++) {
    const int s = P.reached[i];
    if (X.cls[s] < 3) continue;
    const int p = S.sn_parent[s], nt = X.ntf2t[s];
    P.f2t.push_back(s);
    P.f2t.push_back(nt);
    P.work++;
    if (X.cls[s] == 3) { if (p >= 0) P.pend[X.ntf2t[p]]++; continue; }
    const int h = X.f2t[s], nrt = full.tasks[h].nrt;
    if (p >= 0 && full.tasks[h].notify) P.pend[X.ntf2t[p]]++;
    for (int b = 0; b <= nrt; b++) {
      SVTask& t = P.tasks[nt + b];
      const SVTask& o = full.tasks[h + b];
      t.ptask = p >= 0 ? X.ntf2t[p] : -1;
      if (o.dep1 >= o.dep0) {                   // follows its chain child: remapped when reached, else dropped
        const int c = full.tasks[o.dep0].s;
        if (X.stamp[c] == ep) {
          const int d = X.ntf2t[c] - X.f2t[c];
          t.dep0 = o.dep0 + d; t.dep1 = o.dep1 + d; t.dep2 = o.dep2 >= 0 ? o.dep2 + d : o.dep2;
        } else {
          t.dep0 = 0; t.dep1 = -1; t.dep2 = -1;
        }
      }
      P.work++;
    }
  }
}

void build_updown_plan(const Symbolic& S, SolvePrune& X, const int* first, int k, UpdownPlan& P) {
  P.reached.clear(); P.mask.clear(); P.tasks.clear(); P.cnt_init.clear();
  P.nslots = 0; P.entries = 0; P.work = 0;
  if (++X.epoch == 0) { std::fill(X.stamp.begin(), X.stamp.end(), 0u); X.epoch = 1; }   // once in 2^32 calls
  const unsigned ep = X.epoch;
  // each column's whole path: its mask bit is needed on every front up to the root
  for (int r = 0; r < k; r++) {
    P.work++;
    for (int s = X.col2sn[first[r]]; s >= 0; s = S.sn_parent[s]) {
      if (X.stamp[s] != ep) {
        X.stamp[s] = ep;
        X.ntf2t[s] = (int)P.reached.size();
        P.reached.push_back(s);
        P.mask.push_back(0);
      }
      P.mask[X.ntf2t[s]] |= 1 << r;
      P.work++;
    }
  }
  std::vector<int> ord(P.reached.size());
  for (size_t i = 0; i < ord.size(); i++) ord[i] = (int)i;
  std::sort(ord.begin(), ord.end(), [&](int a, int b) {
    P.work++;
    const int sa = P.reached[a], sb = P.reached[b];
    return S.sn_level[sa] != S.sn_level[sb] ? S.sn_level[sa] < S.sn_level[sb] : sa < sb;
  });
  const size_t r = ord.size();
  std::vector<int> reached(r), mask(r);
  for (size_t i = 0; i < r; i++) {
    reached[i] = P.reached[ord[i]];
    mask[i] = P.mask[ord[i]];
    X.ntf2t[reached[i]] = (int)i;
  }
  P.reached.swap(reached);
  P.mask.swap(mask);
  P.cnt_init.assign(3 * r, 0);
  for (size_t i = 0; i < r; i++) {
    const int s = P.reached[i], p = S.sn_parent[s];
    const int ns = S.sn_first[s + 1] - S.sn_first[s], nr = (int)(S.sn_rowptr[s + 1] - S.sn_rowptr[s]);
    const int pli = p >= 0 ? X.ntf2t[p] : -1;
    if (pli >= 0) P.cnt_init[pli]++;
    P.entries += (long long)(ns + nr) * ns;
    UDTask t{};
    t.s = s; t.li = (int)i; t.pli = pli; t.mask = P.mask[i]; t.r0 = 0; t.r1 = nr; t.slot = -1;
    if (nr <= DF_RB) {
      t.kind = 0;
      P.tasks.push_back(t);
    } else {
      t.kind = 1; t.slot = P.nslots++;
      P.tasks.push_back(t);
      for (int a = 0; a < nr; a += DF_RB) {
        t.kind = 2; t.r0 = a; t.r1 = std::min(nr, a + DF_RB);
        P.tasks.push_back(t);
        P.cnt_init[r + i]++;
      }
    }
    P.work += 1 + P.cnt_init[r + i];
  }
}

int updown_slot_bound(const Symbolic& S) {
  const int nsup = S.nsup;
  std::vector<int> ord(nsup), cnt(nsup, 0);
  for (int s = 0; s < nsup; s++) ord[s] = s;
  std::sort(ord.begin(), ord.end(), [&](int a, int b) { return S.sn_level[a] > S.sn_level[b]; });   // parents first
  int most = 0;
  for (int s : ord) {
    const int p = S.sn_parent[s];
    cnt[s] = (S.sn_rowptr[s + 1] - S.sn_rowptr[s] > DF_RB ? 1 : 0) + (p >= 0 ? cnt[p] : 0);
    most = std::max(most, cnt[s]);
  }
  return UD_PASS * most;
}

// Selected inversion (k_selinv): the queue runs the levels from the root down, as the backward sweep does.  The
// gather maps follow every front's rows up the tree: `cur` holds their positions in the current ancestor's front; the
// rows that are pivots of that ancestor form the next segment (rows are ascending, so segments are contiguous and
// come in path order), the others move on to its parent through its `rel`.  Host threads take ranges of fronts.
SelinvPlan build_selinv_plan(const Symbolic& S) {
  SelinvPlan P;
  const int nsup = S.nsup;
  const size_t nrows = S.sn_rows.size();
  P.col.assign(nrows, 0);
  P.seg.assign(nrows, 0);
  {
    const unsigned nth = nsup < 20000 ? 1u : std::max(1u, std::min(16u, host_threads()));
    std::vector<std::vector<int>> part(nth);
    std::vector<std::thread> th;
    auto walk = [&](unsigned t, int s0, int s1) {
      std::vector<int>& sp = part[t];
      std::vector<int> cur;
      for (int s = s0; s < s1; s++) {
        const int nr = nr_of(S, s);
        const int64_t rp = S.sn_rowptr[s];
        if (nr == 0) continue;
        cur.assign(S.rel.begin() + rp, S.rel.begin() + rp + nr);
        int a = S.sn_parent[s], i0 = 0;
        while (i0 < nr) {
          const int nsa = ns_of(S, a);
          int k1 = i0;
          while (k1 < nr && cur[k1] < nsa) k1++;
          if (k1 > i0) {
            const long long base = (long long)sp.size();
            sp.insert(sp.end(), cur.begin() + i0, cur.end());
            for (int k = i0; k < k1; k++) {
              P.col[rp + k] = (long long)S.panel_off[a] + (long long)cur[k] * (nsa + nr_of(S, a));
              P.seg[rp + k] = base - i0;     // local to this thread's part until the parts are joined
            }
          }
          if (k1 < nr) {
            const int64_t pa = S.sn_rowptr[a];
            for (int i = k1; i < nr; i++) cur[i] = S.rel[pa + cur[i] - nsa];
            a = S.sn_parent[a];
          }
          i0 = k1;
        }
      }
    };
    for (unsigned t = 0; t < nth; t++)
      th.emplace_back(walk, t, (int)((int64_t)nsup * t / nth), (int)((int64_t)nsup * (t + 1) / nth));
    for (auto& x : th) x.join();
    size_t tot = 0;
    for (auto& v : part) tot += v.size();
    P.segpos.reserve(tot ? tot : 1);
    for (unsigned t = 0; t < nth; t++) {
      const long long off = (long long)P.segpos.size();
      const int s0 = (int)((int64_t)nsup * t / nth), s1 = (int)((int64_t)nsup * (t + 1) / nth);
      for (int64_t r = S.sn_rowptr[s0]; r < S.sn_rowptr[s1]; r++) P.seg[r] += off;
      P.segpos.insert(P.segpos.end(), part[t].begin(), part[t].end());
    }
    if (P.segpos.empty()) P.segpos.push_back(0);
  }
  P.caller_pos.assign((size_t)S.nnzA, -1);
  for (int s = 0; s < nsup; s++)
    for (int64_t e = S.asm_ptr[s]; e < S.asm_ptr[s + 1]; e++)
      P.caller_pos[S.asm_src[e]] = (long long)S.panel_off[s] + (long long)S.asm_dst[e];

  const QueueOrder q = queue_order(S, {}, 0);
  P.rows_left.assign(nsup, 0);
  auto push = [&](int kind, int s, int r0, int r1) {
    SITask t{};
    t.kind = kind; t.s = s; t.r0 = r0; t.r1 = r1;
    t.ns = ns_of(S, s); t.nr = nr_of(S, s); t.f = S.sn_first[s]; t.parent = S.sn_parent[s];
    t.poff = S.panel_off[s]; t.rp = S.sn_rowptr[s];
    P.tasks.push_back(t);
  };
  for (int l = S.nlevels - 1; l >= 0; l--) {
    const std::vector<int>& lev = q[0][l];
    for (int s : lev) {
      const int nr = nr_of(S, s);
      if (nr <= SI_RB) { push(0, s, 0, nr); continue; }
      for (int r0 = 0; r0 < nr; r0 += SI_RB) push(1, s, r0, std::min(nr, r0 + SI_RB));
      P.rows_left[s] = (nr + SI_RB - 1) / SI_RB;
    }
    for (int s : lev) if (nr_of(S, s) > SI_RB) push(2, s, 0, 0);
  }
  return P;
}

std::vector<int> schur_owner(const Symbolic& S, int first) {
  std::vector<int> owner(S.nsup, 0);
  for (int s = 0; s < S.nsup; s++) if (S.sn_first[s] >= first) owner[s] = -1;
  return owner;
}

SchurPlan build_schur_plan(const Symbolic& S, const std::vector<int>& schur, const SolvePlan& sp) {
  SchurPlan P;
  const int nsup = S.nsup, n = S.n, k = (int)schur.size();
  P.k = k;
  P.first = n - k;
  const int sf = P.first;
  P.owner = schur_owner(S, sf);
  for (int s = 0; s < nsup; s++)
    if (P.owner[s] == 0 && S.sn_parent[s] >= 0 && P.owner[S.sn_parent[s]] < 0) P.cut.push_back(s);
  std::vector<int> out_of(n, -1);        // caller index -> output index
  for (int i = 0; i < k; i++) out_of[schur[i]] = i;
  P.spos.resize(k);
  for (int j = 0; j < k; j++) P.spos[j] = out_of[S.perm[sf + j]];

  // K_SS: bucket by the lower permuted column, then sort each bucket by output position (stable: caller order
  // among duplicates)
  P.kss_ptr.assign(k + 1, 0);
  struct E { long long dst; int src; int col; };
  std::vector<E> ents;
  {
    // the K_SS entries are the original entries assembled into S fronts (the analysis keeps no copy of the caller's
    // pattern; the assembly map gives each entry's front and panel position)
    for (int s = 0; s < nsup; s++) {
      if (P.owner[s] == 0) continue;
      const int f = S.sn_first[s], ns = ns_of(S, s), nr = nr_of(S, s), ld = ns + nr;
      for (int64_t e = S.asm_ptr[s]; e < S.asm_ptr[s + 1]; e++) {
        const int64_t d = S.asm_dst[e];
        const int lc = (int)(d / ld), lr = (int)(d % ld);
        const int jc = f + lc - sf;
        const int jr = (lr < ns ? f + lr : S.sn_rows[S.sn_rowptr[s] + lr - ns]) - sf;
        ents.push_back(E{(long long)P.spos[jc] * k + P.spos[jr], S.asm_src[e], jc});
      }
    }
    for (const E& x : ents) P.kss_ptr[x.col + 1]++;
    for (int j = 0; j < k; j++) P.kss_ptr[j + 1] += P.kss_ptr[j];
    std::vector<E> w(ents.size());
    std::vector<long long> pos(P.kss_ptr.begin(), P.kss_ptr.end() - 1);
    for (const E& x : ents) w[pos[x.col]++] = x;
    for (int j = 0; j < k; j++)
      std::stable_sort(w.begin() + P.kss_ptr[j], w.begin() + P.kss_ptr[j + 1], [](const E& a, const E& b) { return a.dst < b.dst; });
    P.kss_dst.resize(w.size() ? w.size() : 1, 0);
    P.kss_src.resize(w.size() ? w.size() : 1, 0);
    for (size_t i = 0; i < w.size(); i++) { P.kss_dst[i] = w[i].dst; P.kss_src[i] = w[i].src; }
  }

  // cut roots per permuted S column, ascending
  P.rec_ptr.assign(k + 1, 0);
  for (int c : P.cut)
    for (int64_t t = S.sn_rowptr[c]; t < S.sn_rowptr[c + 1]; t++) P.rec_ptr[S.sn_rows[t] - sf + 1]++;
  for (int j = 0; j < k; j++) P.rec_ptr[j + 1] += P.rec_ptr[j];
  P.recs.resize(P.rec_ptr[k] ? P.rec_ptr[k] : 1);
  {
    std::vector<int> pos(P.rec_ptr.begin(), P.rec_ptr.end() - 1);
    for (int c : P.cut)
      for (int64_t t = S.sn_rowptr[c]; t < S.sn_rowptr[c + 1]; t++)
        P.recs[pos[S.sn_rows[t] - sf]++] = SchurRec{(long long)S.upd_off[c], (long long)S.sn_rowptr[c], nr_of(S, c),
                                                     (int)(t - S.sn_rowptr[c])};
  }

  // B-only backward queue: the owned tasks, with the waits on S fronts dropped
  P.bwd.assign(sp.tasks.begin(), sp.tasks.begin() + sp.ntask_owned);
  for (SVTask& t : P.bwd) if (t.kind != 0 && t.bowner >= 0 && P.owner[t.bowner] < 0) t.bowner = -1;
  P.bparent = S.sn_parent;
  for (int c : P.cut) P.bparent[c] = -1;
  return P;
}

FactorParts build_factor_parts(const Symbolic& S) {
  FactorParts F;
  const int n = S.n;
  const int64_t nnz21 = S.sn_rowptr[S.nsup];
  F.row_ptr.assign((size_t)n + 1, 0);
  for (int64_t e = 0; e < nnz21; e++) F.row_ptr[S.sn_rows[e] + 1]++;
  for (int i = 0; i < n; i++) F.row_ptr[i + 1] += F.row_ptr[i];
  F.row_pos.resize(nnz21 ? (size_t)nnz21 : 1, 0);
  std::vector<long long> next(F.row_ptr.begin(), F.row_ptr.end() - 1);
  for (int64_t e = 0; e < nnz21; e++) F.row_pos[next[S.sn_rows[e]]++] = e;
  F.colptr.assign((size_t)n + 1, 0);
  for (int s = 0; s < S.nsup; s++) {
    const int f = S.sn_first[s], ns = S.sn_first[s + 1] - f;
    const int64_t nr = S.sn_rowptr[s + 1] - S.sn_rowptr[s];
    for (int j = 0; j < ns; j++) F.colptr[f + j + 1] = F.colptr[f + j] + (uint64_t)(ns - 1 - j) + (uint64_t)nr;
  }
  return F;
}

}  // namespace cb
