// TEST INFRASTRUCTURE ONLY -- builds the solve plan of one KKT matrix and the pruned plans of a list of index sets on
// the host (build_solve_plan / build_pruned_plan in csrc/ldl_plan.cpp, no CUDA runtime) and writes them out, with the
// symbolic analysis they index, for tests/test_sparse_plan_cpu.py to check.
//
// usage: sparse_plan_driver <in> <out>
//   in : int64 n, nnz, has_perm, cap, nq; int64 Ap[n+1]; int32 Ai[nnz]; int32 perm[n] when has_perm;
//        then per index set: int64 k, int32 permuted columns[k]
//   out: records (int32 name length, name, int64 count, int64 values[count]); a task is 20 values (SVTask's fields)
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
static std::vector<long long> flat(const std::vector<SVTask>& v) {
  std::vector<long long> o;
  for (const SVTask& t : v) {
    const long long f[20] = {t.kind, t.s, t.cnt, t.f, t.ns, t.nr, t.r0, t.r1, t.poff, t.rp, t.dep0, t.dep1, t.dep2, t.nrt,
                             t.bowner, t.bslot, t.pure, t.ptask, t.cuoff, t.notify};
    o.insert(o.end(), f, f + 20);
  }
  return o;
}

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s <in> <out>\n", argv[0]); return 2; }
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  long long hdr[5];
  if (std::fread(hdr, sizeof(long long), 5, in) != 5) return 2;
  const int n = (int)hdr[0];
  std::vector<int64_t> Ap(n + 1);
  std::vector<int32_t> Ai(hdr[1]), perm(hdr[2] ? n : 0);
  if (std::fread(Ap.data(), sizeof(int64_t), Ap.size(), in) != Ap.size() ||
      std::fread(Ai.data(), sizeof(int32_t), Ai.size(), in) != Ai.size() ||
      std::fread(perm.data(), sizeof(int32_t), perm.size(), in) != perm.size()) return 2;
  std::vector<std::vector<int>> sets(hdr[4]);
  for (auto& q : sets) {
    long long k = 0;
    if (std::fread(&k, sizeof(k), 1, in) != 1) return 2;
    q.resize(k);
    if (std::fread(q.data(), sizeof(int), q.size(), in) != q.size()) return 2;
  }
  std::fclose(in);

  Symbolic S;
  SymbolicOptions so;
  if (int rc = analyse(n, Ap.data(), Ai.data(), perm.empty() ? nullptr : perm.data(), so, S)) {
    std::fprintf(stderr, "analyse failed: %d\n", rc);
    return 1;
  }
  const SolvePlan F = build_solve_plan(S, {}, 0, (int)hdr[3]);
  SolvePrune X = build_solve_prune(S, F);
  g_out = std::fopen(argv[2], "wb");
  if (!g_out) return 2;
  put("sym.sn_first", S.sn_first); put("sym.sn_rowptr", S.sn_rowptr); put("sym.sn_parent", S.sn_parent);
  put("sym.sn_level", S.sn_level); put("sym.child_ptr", S.child_ptr); put("sym.child_list", S.child_list);
  put("full.tasks", flat(F.tasks)); put("full.cnt_init", F.cnt_init); put("full.fronts", F.fronts);
  put("full.front2task", F.front2task); put("full.leaf1", F.leaf1); put("full.leafn", F.leafn); put("full.leafw", F.leafw);
  PrunedPlan P;
  for (size_t i = 0; i < sets.size(); i++) {
    build_pruned_plan(S, F, X, sets[i].data(), sets[i].size(), P);
    const std::string q = "q" + std::to_string(i) + ".";
    put(q + "reached", P.reached); put(q + "tasks", flat(P.tasks)); put(q + "pend", P.pend); put(q + "fronts", P.fronts);
    put(q + "f2t", P.f2t); put(q + "leaf1", P.leaf1); put(q + "leafn", P.leafn); put(q + "leafw", P.leafw);
    put(q + "stats", std::vector<long long>{P.entries, P.work});
  }
  std::fclose(g_out);
  return 0;
}
