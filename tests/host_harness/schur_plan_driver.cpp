// TEST INFRASTRUCTURE ONLY -- runs the host analysis of one KKT matrix (csrc/{symbolic,ordering,ldl_plan}.cpp, no CUDA
// runtime) and writes it out for tests/test_schur_plan_cpu.py: with a Schur set, the Schur analysis and every plan a
// Schur handle builds; without one, the ordinary analysis and plans, field for field.
//
// usage: schur_plan_driver <in> <out>
//   in : int64 n, nnz, has_perm, nschur; int64 Ap[n+1]; int32 Ai[nnz]; int32 perm[n] when has_perm; int32 schur[nschur]
//   out: records (int32 name length, name, int64 count, int64 values[count])
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "ldl_plan.h"

using namespace cb;

static FILE* g_out;

template <class T>
static void put(const std::string& name, const std::vector<T>& v) {
  const int len = (int)name.size();
  const long long cnt = (long long)v.size();
  std::fwrite(&len, sizeof(len), 1, g_out);
  std::fwrite(name.data(), 1, name.size(), g_out);
  std::fwrite(&cnt, sizeof(cnt), 1, g_out);
  for (const T& x : v) { const long long y = (long long)x; std::fwrite(&y, sizeof(y), 1, g_out); }
}
// a vector of task records as their 32-bit words
template <class R>
static void put_raw(const std::string& name, const std::vector<R>& v) {
  std::vector<int> w(v.size() * sizeof(R) / 4);
  if (!v.empty()) std::memcpy(w.data(), v.data(), w.size() * 4);
  put(name, w);
}

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s <in> <out>\n", argv[0]); return 2; }
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  long long hdr[4];
  if (std::fread(hdr, sizeof(long long), 4, in) != 4) return 2;
  const int n = (int)hdr[0];
  std::vector<int64_t> Ap(n + 1);
  std::vector<int32_t> Ai(hdr[1]), perm(hdr[2] ? n : 0), schur(hdr[3]);
  if (std::fread(Ap.data(), sizeof(int64_t), Ap.size(), in) != Ap.size() ||
      std::fread(Ai.data(), sizeof(int32_t), Ai.size(), in) != Ai.size() ||
      std::fread(perm.data(), sizeof(int32_t), perm.size(), in) != perm.size() ||
      std::fread(schur.data(), sizeof(int32_t), schur.size(), in) != schur.size()) return 2;
  std::fclose(in);

  Symbolic S;
  SymbolicOptions so;
  std::vector<int> owner;
  const int* pp = perm.empty() ? nullptr : perm.data();
#ifndef PLAIN_ONLY
  if (!schur.empty()) {
    const std::vector<int> sv(schur.begin(), schur.end());
    if (int rc = analyse_schur(n, Ap.data(), Ai.data(), pp, sv, so, S)) { std::fprintf(stderr, "analyse_schur: %d\n", rc); return 3; }
    owner = schur_owner(S, n - (int)sv.size());
  } else
#endif
  if (int rc = analyse(n, Ap.data(), Ai.data(), pp, so, S)) { std::fprintf(stderr, "analyse: %d\n", rc); return 1; }
  const Level0Plan l0 = build_level0_plan(S, owner, 0, 28000);
  const FactorPlan fp = build_factor_plan(S, owner, 0);
  const SolvePlan sp = build_solve_plan(S, owner, 0, 14000);
  g_out = std::fopen(argv[2], "wb");
  if (!g_out) return 2;
  put("sym.scalars", std::vector<long long>{S.n, S.nnzA, S.nnzL_simplicial, S.nsup, S.upd_total, S.nnzL_stored, S.L_alloc,
                                            S.nlevels, S.ordering_used, (long long)S.flops_simplicial, (long long)S.flops_stored});
  put("sym.perm", S.perm); put("sym.iperm", S.iperm); put("sym.parent", S.parent); put("sym.colcount", S.colcount);
  put("sym.sn_first", S.sn_first); put("sym.sn_rowptr", S.sn_rowptr); put("sym.sn_rows", S.sn_rows);
  put("sym.sn_parent", S.sn_parent); put("sym.sn_level", S.sn_level); put("sym.col2sn", S.col2sn);
  put("sym.child_ptr", S.child_ptr); put("sym.child_list", S.child_list); put("sym.rel_ptr", S.rel_ptr); put("sym.rel", S.rel);
  put("sym.panel_off", S.panel_off); put("sym.upd_off", S.upd_off); put("sym.asm_ptr", S.asm_ptr);
  put("sym.asm_src", S.asm_src); put("sym.asm_dst", S.asm_dst); put("sym.level_ptr", S.level_ptr);
  put("sym.level_tasks", S.level_tasks);
  std::vector<int> segs;
  for (const LaunchSeg& g : l0.segs) { segs.push_back(g.leaf1); segs.push_back(g.base); segs.push_back(g.count); segs.push_back(g.smem_doubles); segs.push_back(g.threads); }
  put("l0.segs", segs); put("l0.level_tasks", l0.level_tasks);
  put_raw("fp.tasks", fp.tasks); put_raw("fp.recs", fp.recs); put("fp.cnt_init", fp.cnt_init);
  put("fp.big_pos", fp.big_pos); put("fp.tile_base", fp.tile_base); put("fp.sc_panel_ptr", fp.sc_panel_ptr);
  put("fp.sc_panel_src", fp.sc_panel_src); put("fp.sc_panel_dst", fp.sc_panel_dst); put("fp.sc_tile_ptr", fp.sc_tile_ptr);
  put("fp.sc_tile_src", fp.sc_tile_src); put("fp.sc_tile_dst", fp.sc_tile_dst);
  put("fp.ntask_owned", std::vector<int>{fp.ntask_owned});
  put_raw("sp.tasks", sp.tasks); put("sp.cnt_init", sp.cnt_init); put("sp.fronts", sp.fronts); put("sp.front2task", sp.front2task);
  put("sp.leaf1", sp.leaf1); put("sp.leafn", sp.leafn); put("sp.leafw", sp.leafw); put("sp.wide", sp.wide);
  put("sp.gat_ptr", sp.gat_ptr); put("sp.gat_src", sp.gat_src);
  put("sp.scalars", std::vector<int>{sp.nslots, sp.leafw_nrmax, sp.ntask_owned});
#ifndef PLAIN_ONLY
  if (!schur.empty()) {
    const SchurPlan P = build_schur_plan(S, std::vector<int>(schur.begin(), schur.end()), sp);
    put("sc.scalars", std::vector<int>{P.first, P.k});
    put("sc.owner", P.owner); put("sc.cut", P.cut); put("sc.spos", P.spos);
    put("sc.kss_ptr", P.kss_ptr); put("sc.kss_dst", P.kss_dst); put("sc.kss_src", P.kss_src);
    put("sc.rec_ptr", P.rec_ptr);
    std::vector<long long> ru, rr, rn, rb;
    for (const SchurRec& r : P.recs) { ru.push_back(r.uoff); rr.push_back(r.rp); rn.push_back(r.nr); rb.push_back(r.b); }
    put("sc.rec_uoff", ru); put("sc.rec_rp", rr); put("sc.rec_nr", rn); put("sc.rec_b", rb);
    put_raw("sc.bwd", P.bwd); put("sc.bparent", P.bparent);
  }
#endif
  std::fclose(g_out);
  return 0;
}
