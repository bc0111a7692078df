// TEST INFRASTRUCTURE ONLY -- builds the LDL factorisation and solve plans of one KKT matrix on the host
// (csrc/ldl_plan.cpp, no CUDA runtime) and writes them out for tests/test_ldl_plan_cpu.py and
// tests/test_ldl_shapes_cpu.py to check.
//
// usage: ldl_plan_driver <in> <out>
//   in : int64 n, nnz, nranks, has_perm; int64 Ap[n+1]; int32 Ai[nnz]; int32 perm[n] when has_perm
//   out: records (int32 name length, name, int64 count, int64 values[count]): the tree ("sym.*"), the shard owner
//        ("owner"), then the plans of the unsharded view ("u.") and, when nranks > 1, of every rank ("r<k>.")
#include <cstdio>
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
template <class R, class F>
static std::vector<long long> col(const std::vector<R>& v, F R::*m) {
  std::vector<long long> out;
  for (const R& r : v) out.push_back((long long)(r.*m));
  return out;
}
#define PUT_FIELD(pfx, vec, Rec, field) put(pfx + #field, col(vec, &Rec::field))

static void put_plans(const std::string& p, const Symbolic& S, const std::vector<int>& owner, int rank) {
  const Level0Plan l0 = build_level0_plan(S, owner, rank, 28800);   // the shared-memory caps on an H100
  std::vector<long long> segs;
  for (const LaunchSeg& g : l0.segs) { segs.push_back(g.leaf1); segs.push_back(g.base); segs.push_back(g.count); }
  put(p + "l0.segs", segs);
  put(p + "l0.level_tasks", l0.level_tasks);

  const FactorPlan fp = build_factor_plan(S, owner, rank);
  const std::string f = p + "f.";
  PUT_FIELD(f, fp.tasks, DFTask, kind); PUT_FIELD(f, fp.tasks, DFTask, s); PUT_FIELD(f, fp.tasks, DFTask, a);
  PUT_FIELD(f, fp.tasks, DFTask, b); PUT_FIELD(f, fp.tasks, DFTask, d0); PUT_FIELD(f, fp.tasks, DFTask, d1);
  PUT_FIELD(f, fp.tasks, DFTask, e0); PUT_FIELD(f, fp.tasks, DFTask, e1);
  PUT_FIELD(f, fp.tasks, DFTask, ns); PUT_FIELD(f, fp.tasks, DFTask, nr); PUT_FIELD(f, fp.tasks, DFTask, ndense);
  put(f + "rec.contig", col(fp.recs, &DFChildRec::contig));
  put(f + "cnt_init", fp.cnt_init);
  put(f + "ntask_owned", std::vector<int>{fp.ntask_owned});
  put(f + "big_pos", fp.big_pos);
  put(f + "tile_base", fp.tile_base);
  put(f + "sc_panel_ptr", fp.sc_panel_ptr); put(f + "sc_panel_src", fp.sc_panel_src); put(f + "sc_panel_dst", fp.sc_panel_dst);
  put(f + "sc_tile_ptr", fp.sc_tile_ptr); put(f + "sc_tile_src", fp.sc_tile_src); put(f + "sc_tile_dst", fp.sc_tile_dst);

  const SolvePlan sp = build_solve_plan(S, owner, rank, 8266);
  const std::string s = p + "s.";
  PUT_FIELD(s, sp.tasks, SVTask, kind); PUT_FIELD(s, sp.tasks, SVTask, s); PUT_FIELD(s, sp.tasks, SVTask, cnt);
  PUT_FIELD(s, sp.tasks, SVTask, dep0); PUT_FIELD(s, sp.tasks, SVTask, dep1); PUT_FIELD(s, sp.tasks, SVTask, dep2);
  PUT_FIELD(s, sp.tasks, SVTask, bslot); PUT_FIELD(s, sp.tasks, SVTask, ptask); PUT_FIELD(s, sp.tasks, SVTask, nrt);
  PUT_FIELD(s, sp.tasks, SVTask, ns); PUT_FIELD(s, sp.tasks, SVTask, nr); PUT_FIELD(s, sp.tasks, SVTask, r0);
  PUT_FIELD(s, sp.tasks, SVTask, r1);
  put(s + "cnt_init", sp.cnt_init);
  put(s + "ntask_owned", std::vector<int>{sp.ntask_owned});
  put(s + "fronts", sp.fronts); put(s + "front2task", sp.front2task);
  put(s + "leaf1", sp.leaf1); put(s + "leafn", sp.leafn); put(s + "leafw", sp.leafw);
  put(s + "wide", sp.wide);
  put(s + "gat_ptr", sp.gat_ptr); put(s + "gat_src", sp.gat_src);
}

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s <in> <out>\n", argv[0]); return 2; }
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  long long hdr[4];
  if (std::fread(hdr, sizeof(long long), 4, in) != 4) return 2;
  const int n = (int)hdr[0], nranks = (int)hdr[2];
  std::vector<int64_t> Ap(n + 1);
  std::vector<int32_t> Ai(hdr[1]), perm(hdr[3] ? n : 0);
  if (std::fread(Ap.data(), sizeof(int64_t), Ap.size(), in) != Ap.size() ||
      std::fread(Ai.data(), sizeof(int32_t), Ai.size(), in) != Ai.size() ||
      std::fread(perm.data(), sizeof(int32_t), perm.size(), in) != perm.size()) return 2;
  std::fclose(in);

  Symbolic S;
  SymbolicOptions so;
  if (int rc = analyse(n, Ap.data(), Ai.data(), perm.empty() ? nullptr : perm.data(), so, S)) {
    std::fprintf(stderr, "analyse failed: %d\n", rc);
    return 1;
  }
  g_out = std::fopen(argv[2], "wb");
  if (!g_out) return 2;
  put("sym.sn_first", S.sn_first); put("sym.sn_rowptr", S.sn_rowptr); put("sym.sn_parent", S.sn_parent);
  put("sym.sn_level", S.sn_level); put("sym.child_ptr", S.child_ptr); put("sym.child_list", S.child_list);
  put("sym.upd_off", S.upd_off); put("sym.level_ptr", S.level_ptr);
  put_plans("u.", S, {}, 0);
  if (nranks > 1) {
    ShardPlan shard;
    if (plan_shards(S.nsup, S.sn_first.data(), S.sn_rowptr.data(), S.sn_parent.data(), nranks, shard)) return 1;
    put("owner", shard.owner);
    for (int r = 0; r < nranks; r++) put_plans("r" + std::to_string(r) + ".", S, shard.owner, r);
  }
  std::fclose(g_out);
  return 0;
}
