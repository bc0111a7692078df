// Pruned solves (cldl_solve_sparse, cldl_inverse_entries; device code, included by ldl.cu).  The sweeps are the
// unchanged kernels of ldl_solve.cuh run over a pruned plan (PrunedPlan in ldl_plan.h); these kernels put the
// right-hand side in, give the sweeps exact zeros where the pruned forward set ends, and take the wanted entries out.
#pragma once

// xp[pos[k]] = v[k] (v null: 1), into a work vector cleared beforehand
__global__ void k_sparse_scatter(int cnt, const int* __restrict__ pos, const double* __restrict__ v, double* __restrict__ xp) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < cnt) xp[pos[k]] = v ? v[k] : 1.0;
}

// mark[] = 1 at the fronts of the forward set (cleared beforehand), and front2task[] at the (front, task) pairs of its
// plan
__global__ void k_sparse_setup(int nmark, const int* __restrict__ fronts, unsigned char* __restrict__ mark, int npair,
                               const int* __restrict__ pairs, int* __restrict__ front2task) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < nmark) mark[fronts[k]] = 1;
  if (k < npair) front2task[pairs[2 * k]] = pairs[2 * k + 1];
}

// The fringe of the forward set: children outside it whose parent is inside.  The gather lists of a reached front
// read the update vectors of all its children, so the fringe's are set to zero (the values a full sweep computes
// there for a right-hand side that is zero in their subtrees, up to the sign of zero).  One warp per reached front.
__global__ void __launch_bounds__(256) k_sparse_fringe(LDLDev d, const int* __restrict__ fronts, int count,
                                                       const unsigned char* __restrict__ mark, double* __restrict__ u0,
                                                       double* __restrict__ u1) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= count) return;
  const int p = fronts[w];
  for (long long ci = d.child_ptr[p]; ci < d.child_ptr[p + 1]; ci++) {
    const int c = d.child_list[ci];
    if (mark[c]) continue;
    for (long long t = d.sn_rowptr[c] + lane; t < d.sn_rowptr[c + 1]; t += 32) {
      u0[t] = 0.0;
      if (u1) u1[t] = 0.0;
    }
  }
}

// out[dst[k]] = x[pos[k]] (dst null: out[k]), x = x0 for k < cnt0, else x1
__global__ void k_sparse_gather(int cnt, int cnt0, const int* __restrict__ pos, const int* __restrict__ dst,
                                const double* __restrict__ x0, const double* __restrict__ x1, double* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < cnt) out[dst ? dst[k] : k] = __ldcg((k < cnt0 ? x0 : x1) + pos[k]);
}
