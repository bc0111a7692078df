// Micro-benchmark: FP64 dependent-chain latency, shuffle+DFMA step latency, barrier cost, on one CTA.
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k_lat(double* out, long long* cyc, int iters) {
  double x = out[threadIdx.x], a = 1.0000001, b = 1e-9;
  long long t0, t1;
  // 1. dependent DFMA chain
  __syncthreads();
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < iters; i++) x = fma(x, a, b);
  t1 = clock64();
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
  // 2. dependent FFMA chain
  float xf = (float)x, af = 1.0000001f, bf = 1e-9f;
  __syncthreads();
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < iters; i++) xf = fmaf(xf, af, bf);
  t1 = clock64();
  if (threadIdx.x == 0) cyc[1] = t1 - t0;
  x += xf;
  // 3. shuffle(double) + DFMA dependent step (like a warp trsv)
  __syncthreads();
  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < iters; i++) { double xj = __shfl_sync(0xffffffffu, x, i & 31); x = fma(-xj, b, x); }
  t1 = clock64();
  if (threadIdx.x == 0) cyc[2] = t1 - t0;
  // 4. __syncthreads in a loop
  __syncthreads();
  t0 = clock64();
  for (int i = 0; i < iters; i++) { __syncthreads(); }
  t1 = clock64();
  if (threadIdx.x == 0) cyc[3] = t1 - t0;
  // 5. smem store -> barrier -> smem load -> DFMA (pivot-loop skeleton)
  __shared__ double sb[64];
  __syncthreads();
  t0 = clock64();
  for (int i = 0; i < iters; i++) {
    if (threadIdx.x == (i & 63)) sb[i & 63] = x;
    __syncthreads();
    x = fma(sb[i & 63], b, x);
  }
  t1 = clock64();
  if (threadIdx.x == 0) cyc[4] = t1 - t0;
  // 6. 1.0 / x (IEEE division) dependent chain and __drcp_rn chain
  __syncthreads();
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < iters; i++) x = 1.0 / (x + 1.5);
  t1 = clock64();
  if (threadIdx.x == 0) cyc[5] = t1 - t0;
  __syncthreads();
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < iters; i++) x = __drcp_rn(x + 1.5);
  t1 = clock64();
  if (threadIdx.x == 0) cyc[6] = t1 - t0;
  out[threadIdx.x] = x;
}
// FP64 throughput: all warps of many CTAs doing independent DFMAs
__global__ void __launch_bounds__(256) k_tput(double* out, int iters) {
  double acc[8];
  for (int u = 0; u < 8; u++) acc[u] = out[threadIdx.x] + u;
  double a = 1.0000001, b = 1e-9;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int u = 0; u < 8; u++) acc[u] = fma(acc[u], a, b);
  }
  double s = 0;
  for (int u = 0; u < 8; u++) s += acc[u];
  if (s == 1.2345) out[0] = s;
}
int main() {
  double* out; long long* cyc;
  cudaMalloc(&out, 1024 * 8); cudaMemset(out, 0, 1024 * 8);
  cudaMallocManaged(&cyc, 64);
  const int iters = 4096;
  for (int nt : {32, 256}) {
    k_lat<<<1, nt>>>(out, cyc, iters); cudaDeviceSynchronize();
    k_lat<<<1, nt>>>(out, cyc, iters); cudaDeviceSynchronize();
    printf("threads=%3d  cycles/iter: DFMA chain %.1f  FFMA chain %.1f  shfl64+DFMA %.1f  syncthreads %.1f  sts+bar+lds+dfma %.1f  div %.1f  drcp %.1f\n", nt,
           (double)cyc[0] / iters, (double)cyc[1] / iters, (double)cyc[2] / iters, (double)cyc[3] / iters, (double)cyc[4] / iters, (double)cyc[5] / iters, (double)cyc[6] / iters);
  }
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  int nsm = 0;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);
  for (int per : {1, 2, 4}) {
    k_tput<<<nsm * per, 256>>>(out, 1000);
    cudaEventRecord(a);
    k_tput<<<nsm * per, 256>>>(out, 20000);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    double fma_total = (double)nsm * per * 256 * 8 * 20000;
    printf("FP64 throughput, %d CTAs/SM x 256 thr: %.1f GFMA/s = %.2f TFLOP/s\n", per, fma_total / ms / 1e6, 2 * fma_total / ms / 1e9);
  }
  return 0;
}
