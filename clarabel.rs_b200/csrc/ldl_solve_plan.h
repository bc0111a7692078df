// Task records and counters of the dataflow triangular solves (shared by the host plan builder in ldl.cu and the
// kernels in ldl_solve.cuh).
#pragma once
#include <cuda_runtime.h>

namespace cb {

#define SV_NT 256
#define SV_MINB 3           /* resident sweep CTAs per SM, sets the slab size; C4 on an H100 (700 W): 25.4 it/s against 25.0 with 2 and 25.1 with 4 */
#define SV_MAXROWS 256      /* rows of L21 in one slab (bounds the staged x / the per-thread row count) */

// leading dimension of a staged slab of `srows` rows cut out of a panel with leading dimension ld: the parity of ld (so
// that source and destination are 16-byte aligned at the same elements of every column) and, when even, not a multiple
// of 4 (the transposed reads of the backward sweep would pile up on a few shared-memory banks)
__host__ __device__ inline int sv_lds(int srows, int ld) {
  int L = srows + ((srows ^ ld) & 1);
  if (!(L & 1) && !(L & 3)) L += 2;
  return L;
}

struct SVTask {             // 96 bytes = 6 x int4, built on the host (LDLObject::init)
  int kind, s, cnt, f;      // kind 0: narrow batch (s = first index into fronts[], cnt fronts); 1 head; 2 rows
  int ns, nr, r0, r1;       // slab = rows [r0, r1) of L21 (head: r0 = 0, r1 = rh, plus the pivot block)
  long long poff, rp;       // panel offset in d.L, sn_rowptr[s]
  int dep0, dep1, dep2, nrt;   // forward: chain-child tasks [dep0, dep1] before phase A (head) / before the product (rows); head: [.., dep2] before phase B; nrt = row tasks of the front
  int bowner, bslot, pure, ptask;   // backward: front owning the slab's first row (-1: none); slot in bpart; pure-chain gather; head task of the parent (-1: root)
  long long cuoff;          // pure chain: sn_rowptr[chain child] (row i of the child is local index i of this front)
  int notify, pad;          // notify = 1: the finished front decrements its parent's counter (0 for chain children)
};

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
