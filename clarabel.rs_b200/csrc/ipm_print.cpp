// Verbose output of the interior-point driver: see ipm_print.h.  The number formats are those of the reference's
// table (info_print.rs): `expformat` numbers always carry an exponent sign and at least two exponent digits (C's %e),
// the settings block prints Rust's plain LowerExp (no '+', no leading exponent zeros).
#include "ipm_print.h"

#include <cmath>
#include <cstdlib>
#include <cstring>

namespace cb {

int PrintTarget::set(int k, const char* path, cipm_write_fn f, void* c) {
  std::FILE* nf = nullptr;
  if (k == CIPM_PRINT_FILE) {
    if (!path || !(nf = std::fopen(path, "a"))) return CLDL_E_ARG;
  } else if (k == CIPM_PRINT_STREAM) {
    if (!f) return CLDL_E_ARG;
  } else if (k != CIPM_PRINT_STDOUT && k != CIPM_PRINT_SINK && k != CIPM_PRINT_BUFFER) {
    return CLDL_E_ARG;
  }
  close();
  kind = k; file = nf;
  fn = k == CIPM_PRINT_STREAM ? f : nullptr;
  ctx = k == CIPM_PRINT_STREAM ? c : nullptr;
  return 0;
}

void PrintTarget::close() {
  if (file) std::fclose(file);
  file = nullptr; fn = nullptr; ctx = nullptr;
  buffer.clear();
}

void PrintTarget::write(const std::string& text) {
  if (text.empty()) return;
  switch (kind) {
    case CIPM_PRINT_STDOUT: std::fwrite(text.data(), 1, text.size(), stdout); std::fflush(stdout); break;
    case CIPM_PRINT_FILE: std::fwrite(text.data(), 1, text.size(), file); std::fflush(file); break;
    case CIPM_PRINT_BUFFER: buffer += text; break;
    case CIPM_PRINT_STREAM: fn(ctx, text.data(), (uint64_t)text.size()); break;   // a failed write does not stop the solve
    default: break;                                                                 // sink
  }
}

// ------------------------------------------------------------------------------------------------- number formats
template <class... A>
static std::string fmt(const char* f, A... a) {
  char buf[256];
  std::snprintf(buf, sizeof(buf), f, a...);
  return buf;
}

static std::string pad_left(std::string s, size_t width) {
  return s.size() < width ? std::string(width - s.size(), ' ') + s : s;
}

// a table entry: C's %e for finite values; "inf" / "NaN" spelled and padded as Rust's LowerExp does
static std::string exp_table(double v, int prec, bool plus, size_t width) {
  if (std::isfinite(v)) return plus ? fmt("%+.*e", prec, v) : fmt("%.*e", prec, v);
  std::string s = std::isnan(v) ? "NaN" : (v < 0 ? "-inf" : (plus ? "+inf" : "inf"));
  return pad_left(s, width);
}

// Rust's `{:.Ne}`: 1.0e-8, 1.0e4
static std::string exp_plain(double v, int prec) {
  if (!std::isfinite(v)) return std::isnan(v) ? "NaN" : (v < 0 ? "-inf" : "inf");
  std::string s = fmt("%.*e", prec, v);
  const size_t e = s.find('e');
  std::string mant = s.substr(0, e + 1), ex = s.substr(e + 1);
  const bool neg = ex[0] == '-';
  ex = ex.substr(1);
  while (ex.size() > 1 && ex[0] == '0') ex.erase(0, 1);
  return mant + (neg ? "-" : "") + ex;
}

// Rust's `{:?}` of an f64: shortest text that reads back to the same value, ".0" on integral values
static std::string float_debug(double v) {
  if (std::isinf(v)) return v < 0 ? "-inf" : "inf";
  if (std::isnan(v)) return "NaN";
  const double a = std::fabs(v);
  if (a != 0.0 && (a < 1e-5 || a >= 1e16)) {
    for (int p = 0; p < 17; p++) {
      std::string s = exp_plain(v, p);
      if (std::strtod(s.c_str(), nullptr) == v) return s;
    }
    return exp_plain(v, 16);
  }
  for (int p = 0; p < 17; p++) {
    std::string s = fmt("%.*f", p, v);
    if (std::strtod(s.c_str(), nullptr) == v) return p == 0 ? s + ".0" : s;
  }
  return fmt("%.17g", v);
}

// Rust's `{:?}` of a Duration: 3.2s, 41.253ms, 812.5µs, 950ns
static std::string duration_debug(double seconds) {
  if (!(seconds > 0.0)) return "0ns";
  const uint64_t ns = (uint64_t)std::llround(seconds * 1e9);
  auto with_frac = [](uint64_t whole, uint64_t frac, int digits, const char* unit) {
    std::string s = std::to_string(whole);
    if (frac) {
      std::string f = fmt("%0*llu", digits, (unsigned long long)frac);
      while (!f.empty() && f.back() == '0') f.pop_back();
      s += "." + f;
    }
    return s + unit;
  };
  if (ns >= 1000000000ull) return with_frac(ns / 1000000000ull, ns % 1000000000ull, 9, "s");
  if (ns >= 1000000ull) return with_frac(ns / 1000000ull, ns % 1000000ull, 6, "ms");
  if (ns >= 1000ull) return with_frac(ns / 1000ull, ns % 1000ull, 3, "µs");
  return std::to_string(ns) + "ns";
}

static const char* on_off(int v) { return v ? "on" : "off"; }

static const std::string RULE(93, '-');

// ---------------------------------------------------------------------------------------------------------- blocks
const char* status_name(int status) {
  static const char* const names[] = {"Unsolved", "Solved", "PrimalInfeasible", "DualInfeasible", "AlmostSolved",
                                      "AlmostPrimalInfeasible", "AlmostDualInfeasible", "MaxIterations", "MaxTime",
                                      "NumericalError", "InsufficientProgress", "CallbackTerminated"};
  return status >= 0 && status < (int)(sizeof(names) / sizeof(names[0])) ? names[status] : "Unknown";
}

std::string print_banner() {
  const std::string rule(61, '=');
  return rule + "\n"
         "  clarabel.rs_b200: an interior point solver whose iterates,\n"
         "  KKT factorisation and cones stay on one CUDA device.\n"
         "  Its algorithm and settings follow Clarabel.rs v0.11.\n" +
         rule + "\n";
}

std::string print_configuration(const PrintSetup& ps, const cipm_settings& s) {
  std::string o;
  if (ps.presolve_removed > 0) o += fmt("\npresolve: removed %lld constraints\n", (long long)ps.presolve_removed);
  o += "\nproblem:\n";
  o += fmt("  variables     = %lld\n", (long long)ps.n);
  o += fmt("  constraints   = %lld\n", (long long)ps.m);
  o += fmt("  nnz(P)        = %lld\n", (long long)ps.nnzP);
  o += fmt("  nnz(A)        = %lld\n", (long long)ps.nnzA);
  o += fmt("  cones (total) = %zu\n", ps.cones.size());
  // one line per cone type present, in the reference's type order; the sizes of at most five cones are listed
  static const std::pair<int, const char*> kinds[] = {
      {CIPM_CONE_ZERO, "Zero"}, {CIPM_CONE_NONNEG, "Nonnegative"}, {CIPM_CONE_SOC, "SecondOrder"},
      {CIPM_CONE_EXP, "Exponential"}, {CIPM_CONE_POW, "Power"}, {CIPM_CONE_GENPOW, "GenPower"},
      {CIPM_CONE_PSD, "PSDTriangle"}};
  for (const auto& kd : kinds) {
    std::vector<int64_t> numel;
    for (const auto& c : ps.cones) if (c.first == kd.first) numel.push_back(c.second);
    if (numel.empty()) continue;
    o += fmt("    : %11s = %zu, ", kd.second, numel.size());
    if (numel.size() == 1) {
      o += fmt(" numel = %lld", (long long)numel[0]);
    } else {
      o += " numel = (";
      const size_t shown = numel.size() <= 5 ? numel.size() - 1 : 4;
      for (size_t i = 0; i < shown; i++) o += fmt("%lld,", (long long)numel[i]);
      if (numel.size() > 5) o += "...,";
      o += fmt("%lld)", (long long)numel.back());
    }
    o += "\n";
  }
  o += "\nsettings:\n";
  o += "  linear algebra: direct / " + ps.linsolver + ", precision: 64 bit\n";
  o += "  device: " + (ps.device.empty() ? std::string("unknown") : ps.device) + "\n";
  o += "  max iter = " + std::to_string(s.max_iter) + ", time limit = " +
       (std::isinf(s.time_limit) ? std::string("Inf") : float_debug(s.time_limit)) +
       fmt(",  max step = %.3f\n", s.max_step_fraction);
  o += "  tol_feas = " + exp_plain(s.tol_feas, 1) + ", tol_gap_abs = " + exp_plain(s.tol_gap_abs, 1) +
       ", tol_gap_rel = " + exp_plain(s.tol_gap_rel, 1) + ",\n";
  o += std::string("  static reg : ") + on_off(s.static_regularization_enable) + ", ϵ1 = " +
       exp_plain(s.static_regularization_constant, 1) + ", ϵ2 = " +
       exp_plain(s.static_regularization_proportional, 1) + "\n";
  o += std::string("  dynamic reg: ") + on_off(s.dynamic_regularization_enable) + ", ϵ = " +
       exp_plain(s.dynamic_regularization_eps, 1) + ", δ = " + exp_plain(s.dynamic_regularization_delta, 1) + "\n";
  o += std::string("  iter refine: ") + on_off(s.iterative_refinement_enable) + ", reltol = " +
       exp_plain(s.iterative_refinement_reltol, 1) + ", abstol = " + exp_plain(s.iterative_refinement_abstol, 1) + ",\n";
  o += fmt("               max iter = %d, stop ratio = %.1f\n", s.iterative_refinement_max_iter,
           s.iterative_refinement_stop_ratio);
  o += std::string("  equilibrate: ") + on_off(s.equilibrate_enable) + ", min_scale = " +
       exp_plain(s.equilibrate_min_scaling, 1) + ", max_scale = " + exp_plain(s.equilibrate_max_scaling, 1) + "\n";
  o += fmt("               max iter = %d\n\n", s.equilibrate_max_iter);
  return o;
}

std::string print_header() {
  static const char* const cols[] = {"iter", "pcost", "dcost", "gap", "pres", "dres", "k/t", " μ", "step"};
  static const int width[] = {8, 13, 12, 10, 10, 10, 10, 9, 10};   // in characters; "μ" is one
  std::string o;
  for (int i = 0; i < 9; i++) {
    int len = 0;
    for (const char* p = cols[i]; *p; p++) len += ((unsigned char)*p & 0xC0) != 0x80;   // count UTF-8 characters
    o += cols[i] + std::string(width[i] - len, ' ');
  }
  return o + "\n" + RULE + "\n";
}

std::string print_row(const cipm_info& in) {
  std::string o = fmt("%3u  ", in.iterations);
  o += exp_table(in.cost_primal, 4, true, 8) + "  ";
  o += exp_table(in.cost_dual, 4, true, 8) + "  ";
  o += exp_table(std::fmin(in.gap_abs, in.gap_rel), 2, false, 6) + "  ";
  o += exp_table(in.res_primal, 2, false, 6) + "  ";
  o += exp_table(in.res_dual, 2, false, 6) + "  ";
  o += exp_table(in.ktratio, 2, false, 6) + "  ";
  o += exp_table(in.mu, 2, false, 6) + "  ";
  o += in.iterations > 0 ? exp_table(in.step_length, 2, false, 0) + "  " : std::string(" ------   ");
  return o + "\n";
}

std::string print_footer(const cipm_info& in) {
  return RULE + "\nTerminated with status = " + status_name(in.status) + "\nsolve time = " +
         duration_debug(in.solve_time) + "\n";
}

}  // namespace cb
