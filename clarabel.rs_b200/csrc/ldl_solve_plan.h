// Device view of the dataflow triangular solves' plan (task records: SVTask in ldl_plan.h) and their counters.
#pragma once
#include <cuda_runtime.h>

#include "ldl_plan.h"

namespace cb {

#define SV_MINB 3           /* resident sweep CTAs per SM, sets the slab size; C4 on an H100 (700 W): 25.4 it/s against 25.0 with 2 and 25.1 with 4 */

struct SVPlan {
  int ntask = 0;
  const int4* tasks = nullptr;
  const int* fronts = nullptr;       // narrow batches
  const int* front2task = nullptr;   // [nsup] head / batch task of a front (-1: leaf or not mine)
  const int* parent = nullptr;       // sn_parent
  int* pend = nullptr;               // [ntask] forward: non-chain children (with tasks) still unfinished
  int* fleft = nullptr;              // [nsup] forward: tasks of the front still running
  int* bleft = nullptr;              // [nsup] backward: row tasks still running
  int* tdone = nullptr;              // [ntask] forward: task finished
  int* ydone = nullptr;              // [nsup] forward: pivot solution of a wide front published
  int* done = nullptr;               // [nsup] backward: front finished
  int* qhead = nullptr;              // [2]
  double* bpart = nullptr;           // backward: partial column sums of row tasks, 64 per slot and right-hand side
  long long bpart_stride = 0;        // doubles between the two right-hand sides
  unsigned long long* trace = nullptr;   // optional [2][ntask][4]: grab, ready, end (globaltimer ns)
};

struct SVRhs { double* xp[2]; double* u[2]; double* out[2]; };


}  // namespace cb
