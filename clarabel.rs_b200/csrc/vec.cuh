// Device vector kernels and deterministic reductions (internal header).
//
// Counterpart of the reference's VectorMath trait
// (/root/reference/src/algebra/vecmath.rs:83-226) for device-resident vectors.
// Sums use a fixed two-level tree (per-block partials, then the last block to
// finish folds them in index order) so results are bit-reproducible run to run;
// max/min reductions use atomics on the IEEE bit pattern of non-negative
// doubles, which are order independent (and propagate NaN like
// vecmath.rs:132-141 does, because |NaN| orders above +inf).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <vector>

namespace cb {

// setup-phase timing to stderr when CB_TIMING is set
inline void cb_tmark(const char* label) {
  static std::atomic<double> last{-1.0};      // marks come from several host threads (per-rank drivers, helper threads)
  static const bool on = std::getenv("CB_TIMING") != nullptr;
  if (!on) return;
  const double t = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
  const double prev = last.exchange(t);
  if (label && prev >= 0.0) std::fprintf(stderr, "[cb timing] %-34s %.3f s\n", label, t - prev);
}

// number of kernels launched by this library (bench.py reports it as gpu_launches)
extern std::atomic<unsigned long long> g_launches;   // bumped from several host threads (per-rank threads, helper threads)

// Fixed, not derived from the SM count: the reduction order, and with it every result bit, is then the same on any
// GPU.  On the 132 SMs of an H100 all 296 blocks of 256 threads are resident at once (up to 8 per SM).
constexpr int RED_BLOCKS = 296;
constexpr int RED_THREADS = 256;

struct ReduceWS {
  double* partials = nullptr;    // [RED_BLOCKS * 4]
  unsigned int* counter = nullptr;
};

__device__ __forceinline__ double warp_sum(double v) {
  __syncwarp();   // a diverged warp takes the slow shuffle path
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
  __syncwarp();   // a diverged warp takes the slow shuffle path
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
  __syncwarp();   // a diverged warp takes the slow shuffle path
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// block-wide sum; result valid in every thread. sh must hold >= 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  double r = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.0;
  if (w == 0) { r = warp_sum(r); if (lane == 0) sh[0] = r; }
  __syncthreads();
  r = sh[0];
  return r;
}

__device__ __forceinline__ void atomic_max_nonneg(double* addr, double v) {
  // NaN-propagating max for |.| values: compare bit patterns as unsigned.
  atomicMax((unsigned long long*)addr, (unsigned long long)__double_as_longlong(v));
}
__device__ __forceinline__ void atomic_min_nonneg(double* addr, double v) {
  atomicMin((unsigned long long*)addr, (unsigned long long)__double_as_longlong(v));
}

// out[0] = sum_i f(i), deterministic.  F is a device lambda/functor int -> double.
template <class F>
__global__ void __launch_bounds__(RED_THREADS) k_sum(int n, F f, ReduceWS ws, double* out) {
  __shared__ double sh[32];
  __shared__ bool last;
  double acc = 0.0;
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += gridDim.x * RED_THREADS) acc += f(i);
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) {
    ws.partials[blockIdx.x] = acc;
    __threadfence();
    unsigned t = atomicInc(ws.counter, gridDim.x - 1);
    last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {
    __threadfence();
    double a = 0.0;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += RED_THREADS) a += ((volatile double*)ws.partials)[i];
    a = block_sum(a, sh);
    if (threadIdx.x == 0) out[0] = a;
  }
}

// ---- overflow-safe 2-norm (the reference's stable_norm, vecmath.rs:206-226) ----
// The reference threads a running (scale, sumsq) pair through the vector; a parallel reduction cannot, so the same
// guarantee comes from Blue's three accumulators (the scheme of LAPACK's dnrm2): squares of large entries are summed
// after scaling by 2^-538, squares of tiny ones after scaling by 2^537, the rest unscaled.  No intermediate overflows
// or underflows for any finite input, the result is sqrt(sum x_i^2) to a few ulps, NaN propagates, and the three
// sums are deterministic like every other sum here.
struct Blue3 { double big, med, sml; };
__device__ __forceinline__ void blue_add(Blue3& a, double x) {
  const double tsml = 1.4916681462400413e-154, tbig = 1.9979190722022350e+146;   // 2^-511, 2^486
  const double ssml = 4.4989137945431964e+161, sbig = 1.1113793747425387e-162;   // 2^537, 2^-538
  const double ax = fabs(x);
  if (ax > tbig) { const double t = ax * sbig; a.big += t * t; }
  else if (ax < tsml) { const double t = ax * ssml; a.sml += t * t; }
  else a.med += ax * ax;                                                          // NaN lands here and propagates
}
__device__ __forceinline__ double blue_norm(const Blue3& a) {
  const double ssml = 4.4989137945431964e+161, sbig = 1.1113793747425387e-162;
  if (a.big > 0.0) {
    double s = a.big;
    if (a.med > 0.0 || a.med != a.med) s += (a.med * sbig) * sbig;
    return sqrt(s) / sbig;
  }
  if (a.sml > 0.0) {
    if (a.med > 0.0 || a.med != a.med) {
      const double m = sqrt(a.med), l = sqrt(a.sml) / ssml;
      const double ymin = fmin(m, l), ymax = fmax(m, l);
      return ymax * sqrt(1.0 + (ymin / ymax) * (ymin / ymax));
    }
    return sqrt(a.sml) / ssml;
  }
  return sqrt(a.med);
}

// out[0] = || f(i) ||_2 over i < n, overflow-safe and deterministic
template <class F>
__global__ void __launch_bounds__(RED_THREADS) k_norm2(int n, F f, ReduceWS ws, double* out) {
  __shared__ double sh[32];
  __shared__ bool last;
  Blue3 a{0.0, 0.0, 0.0};
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += gridDim.x * RED_THREADS) blue_add(a, f(i));
  a.big = block_sum(a.big, sh);
  a.med = block_sum(a.med, sh);
  a.sml = block_sum(a.sml, sh);
  if (threadIdx.x == 0) {
    ws.partials[blockIdx.x] = a.big;
    ws.partials[RED_BLOCKS + blockIdx.x] = a.med;
    ws.partials[2 * RED_BLOCKS + blockIdx.x] = a.sml;
    __threadfence();
    unsigned t = atomicInc(ws.counter, gridDim.x - 1);
    last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {
    __threadfence();
    Blue3 b{0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < (int)gridDim.x; i += RED_THREADS) {
      b.big += ((volatile double*)ws.partials)[i];
      b.med += ((volatile double*)ws.partials)[RED_BLOCKS + i];
      b.sml += ((volatile double*)ws.partials)[2 * RED_BLOCKS + i];
    }
    b.big = block_sum(b.big, sh);
    b.med = block_sum(b.med, sh);
    b.sml = block_sum(b.sml, sh);
    if (threadIdx.x == 0) out[0] = blue_norm(b);
  }
}

template <class F>
__global__ void __launch_bounds__(RED_THREADS) k_max_nonneg(int n, F f, double* out) {
  double m = 0.0;
  bool nan = false;
  for (int i = blockIdx.x * RED_THREADS + threadIdx.x; i < n; i += gridDim.x * RED_THREADS) {
    double v = fabs(f(i));
    if (v != v) nan = true;
    m = fmax(m, v);
  }
  m = warp_max(m);
  nan = __any_sync(0xffffffffu, nan);
  if ((threadIdx.x & 31) == 0) {
    if (nan) atomic_max_nonneg(out, __longlong_as_double(0x7ff8000000000000LL));
    else atomic_max_nonneg(out, m);
  }
}

template <class F>
__global__ void k_map(int n, F f) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) f(i);
}

// gradient of <g, x> with respect to the stored upper triangle of a symmetric matrix K (CSC, the caller's order), with
// x = K^-1 b and u = K^-1 g: -(u_i x_j + x_i u_j) off the diagonal, -u_i x_i on it; one warp per column.  Used by the
// interior-point adjoint (P's gradient, solver.cu) and by cldl_adjoint_solve (ldl.cu); static, so that each translation
// unit has its own copy of the one definition.
static __global__ void k_grad_P(int n, const int* __restrict__ colptr, const int* __restrict__ rowval,
                                const double* __restrict__ x, const double* __restrict__ u, double* __restrict__ g) {
  const int j = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (j >= n) return;
  const double xj = x[j], uj = u[j];
  for (int p = colptr[j] + lane; p < colptr[j + 1]; p += 32) {
    const int i = rowval[p];
    g[p] = i == j ? -(u[i] * xj) : -(u[i] * xj + x[i] * uj);
  }
}

inline int red_grid(int n) {
  int g = (n + RED_THREADS - 1) / RED_THREADS;
  return g < 1 ? 1 : (g > RED_BLOCKS ? RED_BLOCKS : g);
}

// a device copy of v in *dst, at least one element long so that an empty vector still gets a pointer the kernels may
// be passed; *dst is set as soon as the allocation succeeds, so that a failed copy leaves nothing unowned
template <class D, class T>
inline cudaError_t upload(D** dst, const std::vector<T>& v) {
  T* p = nullptr;
  cudaError_t e = cudaMalloc((void**)&p, (v.size() ? v.size() : 1) * sizeof(T));
  if (e != cudaSuccess) return e;
  *dst = reinterpret_cast<D*>(p);
  return v.empty() ? cudaSuccess : cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
}

}  // namespace cb
