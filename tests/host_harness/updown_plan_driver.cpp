// TEST INFRASTRUCTURE ONLY -- builds the update plans (build_updown_plan in csrc/ldl_plan.cpp, no CUDA runtime) of a
// list of column sets of one matrix on the host and writes them out, with the symbolic analysis they index, for
// tests/test_updown_plan_cpu.py to check.
//
// usage: updown_plan_driver <in> <out>
//   in : int64 n, nnz, has_perm, nq; int64 Ap[n+1]; int32 Ai[nnz]; int32 perm[n] when has_perm;
//        then per set: int64 k (<= UD_PASS), int32 first permuted row of each column[k]
//   out: records (int32 name length, name, int64 count, int64 values[count]); a task is 8 values (UDTask's fields)
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

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s <in> <out>\n", argv[0]); return 2; }
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  long long hdr[4];
  if (std::fread(hdr, sizeof(long long), 4, in) != 4) return 2;
  const int n = (int)hdr[0];
  std::vector<int64_t> Ap(n + 1);
  std::vector<int32_t> Ai(hdr[1]), perm(hdr[2] ? n : 0);
  if (std::fread(Ap.data(), sizeof(int64_t), Ap.size(), in) != Ap.size() ||
      std::fread(Ai.data(), sizeof(int32_t), Ai.size(), in) != Ai.size() ||
      std::fread(perm.data(), sizeof(int32_t), perm.size(), in) != perm.size()) return 2;
  std::vector<std::vector<int>> sets(hdr[3]);
  for (auto& q : sets) {
    long long k = 0;
    if (std::fread(&k, sizeof(k), 1, in) != 1 || k > UD_PASS) return 2;
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
  const SolvePlan F = build_solve_plan(S, {}, 0, 8266);
  SolvePrune X = build_solve_prune(S, F);
  g_out = std::fopen(argv[2], "wb");
  if (!g_out) return 2;
  put("sym.sn_first", S.sn_first); put("sym.sn_rowptr", S.sn_rowptr); put("sym.sn_parent", S.sn_parent);
  put("sym.sn_level", S.sn_level);
  put("const", std::vector<long long>{UD_PASS, DF_RB, (long long)sizeof(UDTask), updown_slot_bound(S)});
  UpdownPlan P;
  for (size_t i = 0; i < sets.size(); i++) {
    build_updown_plan(S, X, sets[i].data(), (int)sets[i].size(), P);
    const std::string q = "q" + std::to_string(i) + ".";
    std::vector<long long> t;
    for (const UDTask& a : P.tasks) {
      const long long f[8] = {a.kind, a.s, a.li, a.pli, a.mask, a.r0, a.r1, a.slot};
      t.insert(t.end(), f, f + 8);
    }
    put(q + "reached", P.reached); put(q + "mask", P.mask); put(q + "tasks", t); put(q + "cnt", P.cnt_init);
    put(q + "stats", std::vector<long long>{P.nslots, P.entries, P.work});
  }
  std::fclose(g_out);
  return 0;
}
