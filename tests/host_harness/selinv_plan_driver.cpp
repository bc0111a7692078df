// TEST INFRASTRUCTURE ONLY -- builds the selected-inversion plan of one KKT matrix on the host (build_selinv_plan in
// csrc/ldl_plan.cpp, no CUDA runtime) and writes it out, with the symbolic analysis it indexes, for
// tests/test_selinv_plan_cpu.py to check.
//
// usage: selinv_plan_driver <in> <out>
//   in : int64 n, nnz, has_perm; int64 Ap[n+1]; int32 Ai[nnz]; int32 perm[n] when has_perm
//   out: records (int32 name length, name, int64 count, int64 values[count])
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
template <class F>
static std::vector<long long> field(const std::vector<SITask>& v, F SITask::*m) {
  std::vector<long long> out;
  for (const SITask& r : v) out.push_back((long long)(r.*m));
  return out;
}

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s <in> <out>\n", argv[0]); return 2; }
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  long long hdr[3];
  if (std::fread(hdr, sizeof(long long), 3, in) != 3) return 2;
  const int n = (int)hdr[0];
  std::vector<int64_t> Ap(n + 1);
  std::vector<int32_t> Ai(hdr[1]), perm(hdr[2] ? n : 0);
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
  const SelinvPlan P = build_selinv_plan(S);
  g_out = std::fopen(argv[2], "wb");
  if (!g_out) return 2;
  put("sym.perm", S.perm); put("sym.sn_first", S.sn_first); put("sym.sn_rowptr", S.sn_rowptr);
  put("sym.sn_rows", S.sn_rows); put("sym.sn_parent", S.sn_parent); put("sym.panel_off", S.panel_off);
  put("t.kind", field(P.tasks, &SITask::kind)); put("t.s", field(P.tasks, &SITask::s));
  put("t.r0", field(P.tasks, &SITask::r0)); put("t.r1", field(P.tasks, &SITask::r1));
  put("t.ns", field(P.tasks, &SITask::ns)); put("t.nr", field(P.tasks, &SITask::nr));
  put("t.parent", field(P.tasks, &SITask::parent)); put("t.poff", field(P.tasks, &SITask::poff));
  put("t.rp", field(P.tasks, &SITask::rp));
  put("rows_left", P.rows_left); put("col", P.col); put("seg", P.seg); put("segpos", P.segpos);
  put("caller_pos", P.caller_pos);
  std::fclose(g_out);
  return 0;
}
