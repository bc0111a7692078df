// Schur complement handles (included by ldl.cu): the dense complement Sc = K_SS - K_SB K_BB^-1 K_BS and the two partial
// solves, from a factorisation of B's fronts alone (SchurPlan in ldl_plan.h).  Every B front whose parent is in S (a
// cut root) leaves its update matrix in the arena and its update vector in `u`: no S front runs, so nothing reuses
// them.  Sc is K_SS plus the cut roots' update matrices, the condensed right-hand side b_S plus their update vectors.
// Each output column (and each entry of the condensed vector) is summed by one CTA (thread) in a fixed order -- K_SS,
// then the cut roots in ascending order -- with no atomics, so repeated refactors give the same bits.
#define SC_NT 128

// One CTA per permuted S column j: the entries of the permuted lower triangle (rows i >= j) in the output's column
// spos[j], then their mirror images in the rows spos[j] of the later columns.  Both triangles of an entry are written
// by the CTA of its lower permuted column only.
__global__ void __launch_bounds__(SC_NT) k_schur_assemble(const double* __restrict__ vals, const double* __restrict__ U,
                                                          const int* __restrict__ sn_rows, int first, int k,
                                                          const int* __restrict__ spos,
                                                          const long long* __restrict__ kss_ptr,
                                                          const long long* __restrict__ kss_dst,
                                                          const int* __restrict__ kss_src,
                                                          const int* __restrict__ rec_ptr,
                                                          const SchurRec* __restrict__ recs, double* out) {
  const int j = blockIdx.x, tid = threadIdx.x;
  const long long kk = k;
  double* col = out + (long long)spos[j] * kk;
  for (int i = j + tid; i < k; i += SC_NT) col[spos[i]] = 0.0;
  __syncthreads();
  // original entries: one thread per output position, its caller entries (duplicates) in caller order
  const long long e0 = kss_ptr[j], e1 = kss_ptr[j + 1];
  for (long long e = e0 + tid; e < e1; e += SC_NT) {
    const long long dst = kss_dst[e];
    if (e > e0 && kss_dst[e - 1] == dst) continue;
    double acc = 0.0;
    for (long long q = e; q < e1 && kss_dst[q] == dst; q++) acc += vals[kss_src[q]];
    out[dst] += acc;
  }
  __syncthreads();
  // cut roots in ascending order: column b of the update matrix (its lower triangle, rows b..nr-1)
  for (int r = rec_ptr[j]; r < rec_ptr[j + 1]; r++) {
    const SchurRec R = recs[r];
    const double* __restrict__ uc = U + R.uoff + (long long)R.b * R.nr;
    const int* __restrict__ rows = sn_rows + R.rp;
    for (int a = R.b + tid; a < R.nr; a += SC_NT) col[spos[rows[a] - first]] += uc[a];
    __syncthreads();
  }
  for (int i = j + 1 + tid; i < k; i += SC_NT) out[(long long)spos[i] * kk + spos[j]] = col[spos[i]];
}

// condensation, after the forward sweep over B: w_S[spos[j]] = b_S + the cut roots' update-vector entries at row j
__global__ void k_schur_reduce(int first, int k, const int* __restrict__ spos, const int* __restrict__ rec_ptr,
                               const SchurRec* __restrict__ recs, const double* __restrict__ xp,
                               const double* __restrict__ u, double* __restrict__ wS) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= k) return;
  double acc = xp[first + j];
  for (int r = rec_ptr[j]; r < rec_ptr[j + 1]; r++) acc += u[recs[r].rp + recs[r].b];
  wS[spos[j]] = acc;
}

// expansion, before the backward sweep over B: x_S into the permuted work vector and into the solution
__global__ void k_schur_expand_in(int first, int k, const int* __restrict__ spos, const int* __restrict__ perm,
                                  const double* __restrict__ xS, double* __restrict__ xp, double* __restrict__ x) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= k) return;
  const double v = xS[spos[j]];
  xp[first + j] = v;
  x[perm[first + j]] = v;
}
