// Micro-benchmark: aggregate load bandwidth of 8-byte loads by flavour (plain / ld.global.cg / volatile),
// L2-resident (32 MB) and HBM-resident (1 GB) buffers, 296 CTAs x 256 threads (2-3 per SM), 32 loads in flight per thread.
#include <cstdio>
#include <cuda_runtime.h>
template <int MODE>
__global__ void __launch_bounds__(256, 2) k_read(const double* __restrict__ p, size_t n, int reps, double* out, int misalign) {
  double acc = 0.0;
  const size_t stride = (size_t)gridDim.x * 256 * 32;
  for (int r = 0; r < reps; r++) {
    for (size_t base = (size_t)blockIdx.x * 256 * 32; base + 256 * 32 <= n; base += stride) {
      double v[32];
#pragma unroll
      for (int u = 0; u < 32; u++) {
        const double* q = p + misalign + base + u * 256 + threadIdx.x;
        if (MODE == 0) v[u] = *q;
        else if (MODE == 1) v[u] = __ldcg(q);
        else if (MODE == 2) v[u] = *(const volatile double*)q;
        else v[u] = __ldcs(q);
      }
#pragma unroll
      for (int u = 0; u < 32; u++) acc += v[u];
    }
  }
  if (acc == 1.2345) out[0] = acc;
}
template <int MODE>
void run(const char* name, const double* p, size_t n, int reps, double* out, int mis) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k_read<MODE><<<296, 256>>>(p, n, 1, out, mis);
  cudaEventRecord(a);
  k_read<MODE><<<296, 256>>>(p, n, reps, out, mis);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  printf("%-10s n=%6.0f MB mis=%d  %8.1f GB/s\n", name, n * 8 / 1e6, mis, (double)n * 8 * reps / ms / 1e6);
}
int main() {
  double *p, *out; size_t big = (size_t)1 << 27;  // 1 GB
  cudaMalloc(&p, (big + 64) * 8); cudaMalloc(&out, 8); cudaMemset(p, 0, (big + 64) * 8);
  for (int mis = 0; mis < 2; mis++) {
    size_t small = (size_t)4 << 20;  // 32 MB
    run<0>("plain", p, small, 40, out, mis); run<1>("ldcg", p, small, 40, out, mis); run<2>("volatile", p, small, 40, out, mis); run<3>("ldcs", p, small, 40, out, mis);
    run<0>("plain", p, big, 2, out, mis); run<1>("ldcg", p, big, 2, out, mis); run<2>("volatile", p, big, 2, out, mis); run<3>("ldcs", p, big, 2, out, mis);
  }
  return 0;
}
