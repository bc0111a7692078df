// TEST INFRASTRUCTURE ONLY -- runs the interior-point solver's host set-up (csrc/problem_setup.cpp, no CUDA runtime)
// on one problem and writes what it built for tests/test_problem_setup_cpu.py to check.
//
// usage: problem_setup_driver <in> <out>
//   in : int64 n, m, nnzP, nnzA, ncones, nalpha, presolve_enable, equilibrate_enable, equilibrate_max_iter, nperm;
//        float64 infbound, equilibrate_min_scaling, equilibrate_max_scaling;
//        uint64 Pp[n+1], Pi[nnzP]; float64 Px[nnzP], q[n]; uint64 Ap[n+1], Ai[nnzA]; float64 Ax[nnzA], b[m];
//        int64 cone_types[ncones]; uint64 cone_dims[ncones]; float64 cone_params[ncones]; uint64 genpow_dim2[ncones];
//        float64 genpow_alpha[nalpha]; uint64 kkt_perm[nperm]
//   out: records (int32 name length, name, char type 'i' / 'f', int64 count, int64 or float64 values[count]); "rc" is
//        the first nonzero return code, or 0 after the last stage
#include <cstdio>
#include <string>
#include <type_traits>
#include <vector>

#include "problem_setup.h"

using namespace cb;

static FILE* g_out;

template <class T>
static void put(const std::string& name, const std::vector<T>& v) {
  const int len = (int)name.size();
  const long long cnt = (long long)v.size();
  const char type = std::is_floating_point<T>::value ? 'f' : 'i';
  std::fwrite(&len, sizeof(len), 1, g_out);
  std::fwrite(name.data(), 1, name.size(), g_out);
  std::fwrite(&type, 1, 1, g_out);
  std::fwrite(&cnt, sizeof(cnt), 1, g_out);
  for (const T& x : v) {
    if (type == 'f') { const double y = (double)x; std::fwrite(&y, sizeof(y), 1, g_out); }
    else { const long long y = (long long)x; std::fwrite(&y, sizeof(y), 1, g_out); }
  }
}
static void put_csr(const std::string& p, const CsrMap& M) {
  put(p + ".rowptr", M.rowptr); put(p + ".col", M.col); put(p + ".src", M.src);
}
static void put_csc(const std::string& p, const HostCsc& M) {
  put(p + ".colptr", M.colptr); put(p + ".rowval", M.rowval); put(p + ".nzval", M.nzval);
}

template <class T>
static bool get(FILE* f, std::vector<T>& v, long long n) {
  v.resize((size_t)n);
  return std::fread(v.data(), sizeof(T), v.size(), f) == v.size();
}

static int finish(int rc) {
  put("rc", std::vector<int>{rc});
  std::fclose(g_out);
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s <in> <out>\n", argv[0]); return 2; }
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  std::vector<long long> h;
  std::vector<double> hf;
  if (!get(in, h, 10) || !get(in, hf, 3)) return 2;
  const int n = (int)h[0], m = (int)h[1];
  const long long nnzP = h[2], nnzA = h[3], nc = h[4], nalpha = h[5];
  cipm_settings set{};
  set.presolve_enable = (int)h[6];
  set.equilibrate_enable = (int)h[7];
  set.equilibrate_max_iter = (int)h[8];
  set.equilibrate_min_scaling = hf[1];
  set.equilibrate_max_scaling = hf[2];
  const double infbound = hf[0];
  std::vector<uint64_t> Pp, Pi, Ap, Ai, cdim, gdim2, perm;
  std::vector<double> Px, q, Ax, b, cparam, galpha;
  std::vector<long long> ctype64;
  if (!get(in, Pp, n + 1) || !get(in, Pi, nnzP) || !get(in, Px, nnzP) || !get(in, q, n) || !get(in, Ap, n + 1) ||
      !get(in, Ai, nnzA) || !get(in, Ax, nnzA) || !get(in, b, m) || !get(in, ctype64, nc) || !get(in, cdim, nc) ||
      !get(in, cparam, nc) || !get(in, gdim2, nc) || !get(in, galpha, nalpha) || !get(in, perm, h[9]))
    return 2;
  std::fclose(in);
  const std::vector<int32_t> ctype(ctype64.begin(), ctype64.end());
  g_out = std::fopen(argv[2], "wb");
  if (!g_out) return 2;

  int rc = check_csc(Pp.data(), Pi.data(), (uint64_t)n, n, true);
  if (rc || (rc = check_csc(Ap.data(), Ai.data(), (uint64_t)m, n, false))) return finish(rc);
  HostCsc P = host_csc(n, n, Pp.data(), Pi.data(), Px.data()), A = host_csc(m, n, Ap.data(), Ai.data(), Ax.data());
  std::vector<ConeSpec> cs;
  if ((rc = collapse_cones(ctype.data(), cdim.data(), (uint64_t)nc, cs, cparam.data(), gdim2.data(), galpha.data())))
    return finish(rc);
  std::vector<char> keep;
  if ((rc = presolve(cs, A, b, infbound, set.presolve_enable != 0, keep))) return finish(rc);
  put("keep", keep);
  put("m_reduced", std::vector<int>{A.m});
  ConeLayout L;
  if ((rc = cone_layout(cs, L))) return finish(rc);
  put("layout.p", std::vector<int>{L.p});
  KKTAssembly K;
  if ((rc = assemble_kkt(P, A, L, K))) return finish(rc);
  put("K.N", std::vector<int>{K.N});
  put("K.Kp", K.Kp); put("K.Ki", K.Ki); put("K.dsigns", K.dsigns);
  if (!perm.empty()) put("kkt_perm", kkt_perm(perm.data(), n, A.m, L));
  // the transposes, on the presolved data before equilibration
  put_csc("P", P); put_csc("A", A);
  put_csr("Psym", triu_to_sym_csr(n, P.colptr.data(), P.rowval.data()));
  put_csr("Acsr", csc_to_csr(A));
  put_csr("Ksym", triu_to_sym_csr(K.N, K.Kp.data(), K.Ki.data()));
  const Equilibration eq = equilibrate(P, A, q, b, L, set);
  put("eq.d", eq.d); put("eq.e", eq.e); put("eq.c", std::vector<double>{eq.c});
  // the solution of an iterate of ones with t = 1, in the caller's rows
  const std::vector<double> ones((size_t)(n > A.m ? n : A.m), 1.0);
  std::vector<double> x(n), z(m), s(m);
  unscale_solution(eq, keep, infbound, 1.0, n, m, ones.data(), ones.data(), ones.data(), x.data(), z.data(), s.data());
  put("sol.x", x); put("sol.z", z); put("sol.s", s);
  return finish(0);
}
