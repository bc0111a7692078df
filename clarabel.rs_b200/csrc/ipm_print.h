// Verbose output of the interior-point driver (default/info_print.rs, src/io/mod.rs): the text of the banner, the
// problem / settings block, the iteration table and the footer, and the print target it goes to.  Host-only C++:
// nothing here touches the device, so printing adds no launch, copy or synchronisation to a solve.
#pragma once

#include <cstdint>
#include <cstdio>
#include <string>
#include <utility>
#include <vector>

#include "../../include/clarabel_b200.h"

namespace cb {

// PrintTarget (io/mod.rs:99-130): stdout, sink, in-memory buffer, file (appended to) or a caller's write function
struct PrintTarget {
  int kind = CIPM_PRINT_STDOUT;
  std::FILE* file = nullptr;
  cipm_write_fn fn = nullptr;
  void* ctx = nullptr;
  std::string buffer;

  PrintTarget() = default;
  PrintTarget(const PrintTarget&) = delete;
  PrintTarget& operator=(const PrintTarget&) = delete;
  ~PrintTarget() { close(); }
  int set(int kind, const char* path, cipm_write_fn fn, void* ctx);   // 0 or CLDL_E_ARG
  void write(const std::string& text);
  void close();
};

// what the problem / settings block reports; collected once when the handle is created
struct PrintSetup {
  int64_t n = 0, m = 0, nnzP = 0, nnzA = 0;
  int64_t presolve_removed = 0;                  // rows the inf-bound presolve dropped
  std::vector<std::pair<int, int64_t>> cones;    // (CIPM_CONE_* tag, numel) in cone order
  std::string linsolver = "cudaldl";
  std::string device;                            // CUDA device name
};

const char* status_name(int status);             // SolverStatus names, "Solved", "CallbackTerminated", ...
std::string print_banner();
std::string print_configuration(const PrintSetup& ps, const cipm_settings& s);
std::string print_header();
std::string print_row(const cipm_info& info);
std::string print_footer(const cipm_info& info);

}  // namespace cb
