// TC row of the north star ("tensor cores only for the dense Schur blocks arising from SDP cones"): is the FP64 tensor
// path (mma.sync.aligned.m8n8k4.f64, SASS DMMA -- FP64 MMA on sm_90a is mma.sync only; wgmma has no FP64 kind) worth building for
// the 64 x 64 x 64 tile products of the refactorisation (k_factor_df T tasks) and the skron blocks of the PSD cone?
// Both variants compute C(64x64) -= A(64x64) * B(64x64)^T per CTA from shared memory, `iters` times, 256 threads:
//   fma  : 4 x 4 register tile per thread (what k_factor_df does)
//   dmma : 8 warps, each owns a 32 x 16 piece of C as 4 x 2 mma tiles of 8 x 8, k in steps of 4
// Prints GFLOP/s over the whole chip (grid = 2 CTAs per SM).   nvcc -O3 -gencode arch=compute_90a,code=sm_90a
#include <cstdio>
#include <cuda_runtime.h>
#define TS 64
#define LD 65
__global__ void __launch_bounds__(256, 2) k_fma(double* out, int iters) {
  extern __shared__ double sm_[]; double *sA = sm_, *sB = sm_ + TS * LD;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  for (int i = tid; i < TS * LD; i += 256) { sA[i] = 1e-3 * (i % 17); sB[i] = 1e-3 * (i % 13); }
  __syncthreads();
  double c[4][4] = {};
  for (int it = 0; it < iters; it++) {
#pragma unroll 4
    for (int k = 0; k < TS; k++) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; i++) { a[i] = sA[k * LD + ty * 4 + i]; b[i] = sB[k * LD + tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) c[i][j] -= a[i] * b[j];
    }
  }
  double s = 0;
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) s += c[i][j];
  out[blockIdx.x * 256 + tid] = s;
}
__global__ void __launch_bounds__(256, 2) k_dmma(double* out, int iters) {
  extern __shared__ double sm_[]; double *sA = sm_, *sB = sm_ + TS * LD;     // sA[k][row], sB[k][col]
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  for (int i = tid; i < TS * LD; i += 256) { sA[i] = 1e-3 * (i % 17); sB[i] = 1e-3 * (i % 13); }
  __syncthreads();
  const int r0 = (w & 1) * 32, c0 = (w >> 1) * 16;   // 2 x 4 warps: 32 rows x 16 columns each
  double c[4][2][2] = {};
  for (int it = 0; it < iters; it++) {
#pragma unroll 4
    for (int k = 0; k < TS; k += 4) {
      double a[4], b[2];
#pragma unroll
      for (int i = 0; i < 4; i++) a[i] = sA[(k + (lane & 3)) * LD + r0 + 8 * i + (lane >> 2)];
#pragma unroll
      for (int j = 0; j < 2; j++) b[j] = -sB[(k + (lane & 3)) * LD + c0 + 8 * j + (lane >> 2)];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 2; j++)
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                       : "+d"(c[i][j][0]), "+d"(c[i][j][1]) : "d"(a[i]), "d"(b[j]));
    }
  }
  double s = 0;
  for (int i = 0; i < 4; i++) for (int j = 0; j < 2; j++) s += c[i][j][0] + c[i][j][1];
  out[blockIdx.x * 256 + tid] = s;
}
int main() {
  int nsm = 0;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);
  const int grid = 2 * nsm, iters = 4000;
  double* out;
  cudaMalloc(&out, (size_t)grid * 256 * 8);
  const size_t SM = 2 * TS * LD * sizeof(double);
  cudaFuncSetAttribute(k_fma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SM);
  cudaFuncSetAttribute(k_dmma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SM);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int v = 0; v < 2; v++) {
    float best = 1e30f;
    for (int rep = 0; rep < 4; rep++) {
      cudaEventRecord(e0);
      if (v == 0) k_fma<<<grid, 256, SM>>>(out, iters); else k_dmma<<<grid, 256, SM>>>(out, iters);
      cudaEventRecord(e1); cudaEventSynchronize(e1);
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      if (rep && ms < best) best = ms;
    }
    const double flops = 2.0 * TS * TS * TS * (double)iters * grid;
    printf("%s: %.3f ms  %.1f GFLOP/s FP64 (grid %d x 256 threads, 64x64x64 tile from shared memory)\n", v == 0 ? "fma 4x4 register tile" : "mma.sync m8n8k4 f64  ", best, flops / best / 1e6, grid);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
