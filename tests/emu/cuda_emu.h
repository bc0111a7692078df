// TEST INFRASTRUCTURE ONLY -- never part of the product library.
//
// CUDA-on-CPU emulation layer, just large enough to compile clarabel.rs_b200/csrc/{cones,cones_psd,cones_nonsym,
// solver}.cu (after tests/emu/transform.py has rewritten the <<<...>>> launches) with g++ and to RUN their kernels
// on the host: every CUDA thread of a block is a fiber (own stack, cooperative switching); __syncthreads, __syncwarp
// and the warp shuffles / votes are rendezvous points between fibers; blocks of a grid run one after the other;
// atomics are plain operations (one OS thread executes everything); streams and events are synchronous.
//
// What this is for: the IPM driver, the KKT layer and every cone kernel -- including the code written while no GPU
// was available -- can be executed end to end on a CPU and compared with the oracle (tests/test_emu_cpu.py).  What it
// is not: a model of the hardware.  Memory ordering, warp divergence and co-residency are not reproduced, the
// multifrontal LDL^T kernels of ldl.cu are not part of the emulated build (tests/emu/ldl_emu.cpp supplies a dense
// host factorisation with the same pivot rule behind the same LDLObject interface), and nothing measured here says
// anything about the GPU.  The GPU tests (-m gpu) remain the parity proof.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <type_traits>

#define CB_EMU 1

// ------------------------------------------------------------------------------------------------ vector types
struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct alignas(8) int2 { int x, y; };       // same alignment as the CUDA vector types: -fsanitize=alignment
struct alignas(8) float2 { float x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(16) double2 { double x, y; };
inline double2 make_double2(double x, double y) { return double2{x, y}; }
inline int2 make_int2(int x, int y) { return int2{x, y}; }
inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }

// ------------------------------------------------------------------------------------------------ qualifiers
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
/* __shared__ declarations are rewritten by tests/emu/transform.py into per-block storage (emu::shared_slot) */

// ------------------------------------------------------------------------------------------------ runtime
namespace emu {
struct Fiber;
struct ThreadView { uint3 tid; };
uint3& cur_tid();
uint3& cur_bid();
extern uint3 g_blockDim, g_gridDim;
void* dyn_smem();
void* shared_slot(int site, size_t bytes);   // per-block storage of one static __shared__ declaration, zeroed on first use
void spin_yield();                           // a spin-wait lets every other resident fiber run
void sync_block();
void sync_warp();
uint64_t warp_exchange(uint64_t bits, int src_lane);   // every live lane of the warp calls; returns src lane's bits
int lane_id();
unsigned warp_vote(bool pred);                         // ballot over the live lanes
void run_grid(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body);

struct Cfg {
  dim3 grid, block;
  size_t smem;
  Cfg(dim3 g, dim3 b, size_t s = 0, void* = nullptr) : grid(g), block(b), smem(s) {}
};
// a launch after tests/emu/transform.py: the kernel call sits in `body` and runs once per emulated thread
void note_smem_optin(const void* fn, int bytes);     // cudaFuncSetAttribute(MaxDynamicSharedMemorySize)
void check_smem_optin(const void* fn, size_t smem);   // aborts when a launch exceeds 48 KB without (enough) opt-in
template <class F> inline const void* fn_key(F f) { return (const void*)f; }
inline void run_grid_cfg(const Cfg& c, const std::function<void()>& body, const void* fn = nullptr) {
  if (fn) check_smem_optin(fn, c.smem);
  run_grid(c.grid, c.block, c.smem, body);
}
}  // namespace emu

#define threadIdx (emu::cur_tid())
#define blockIdx (emu::cur_bid())
#define blockDim (emu::g_blockDim)
#define gridDim (emu::g_gridDim)
#define warpSize 32

inline void __syncthreads() { emu::sync_block(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::sync_warp(); }
inline void __nanosleep(unsigned) { emu::spin_yield(); }
inline void __threadfence() {}
inline void __threadfence_block() {}

template <class T>
inline T emu_shfl_from(T v, int src) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  uint64_t b = 0;
  std::memcpy(&b, &v, sizeof(T));
  b = emu::warp_exchange(b, src & 31);
  T r;
  std::memcpy(&r, &b, sizeof(T));
  return r;
}
template <class T> inline T __shfl_xor_sync(unsigned, T v, int o) { return emu_shfl_from(v, emu::lane_id() ^ o); }
template <class T> inline T __shfl_sync(unsigned, T v, int src) { return emu_shfl_from(v, src); }
template <class T> inline T __shfl_down_sync(unsigned, T v, unsigned d) { const int l = emu::lane_id(); return emu_shfl_from(v, l + (int)d < 32 ? l + (int)d : l); }
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned d) { const int l = emu::lane_id(); return emu_shfl_from(v, l - (int)d >= 0 ? l - (int)d : l); }
inline int __any_sync(unsigned, int p) { return emu::warp_vote(p != 0) != 0; }
inline int __all_sync(unsigned, int p) { return emu::warp_vote(p == 0) == 0; }
inline unsigned __ballot_sync(unsigned, int p) { return emu::warp_vote(p != 0); }

// atomics: one OS thread runs every fiber, so read-modify-write is already indivisible
template <class T> inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <class T> inline T atomicSub(T* p, T v) { T o = *p; *p = o - v; return o; }
template <class T> inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <class T> inline T atomicAnd(T* p, T v) { T o = *p; *p = o & v; return o; }
template <class T> inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <class T> inline T atomicCAS(T* p, T c, T v) { T o = *p; if (o == c) *p = v; return o; }
inline unsigned atomicInc(unsigned* p, unsigned lim) { unsigned o = *p; *p = (o >= lim) ? 0u : o + 1u; return o; }

inline long long __double_as_longlong(double x) { long long r; std::memcpy(&r, &x, 8); return r; }
inline double __longlong_as_double(long long x) { double r; std::memcpy(&r, &x, 8); return r; }
template <class T> inline T __ldg(const T* p) { return *p; }
template <class T> inline T __ldcg(const T* p) { return *p; }
inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)p; }
inline double __drcp_rn(double x) { return 1.0 / x; }
inline double __dsqrt_rn(double x) { return std::sqrt(x); }
inline double __fma_rn(double a, double b, double c) { return std::fma(a, b, c); }
inline double rsqrt(double x) { return 1.0 / std::sqrt(x); }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __ffs(int x) { return __builtin_ffs(x); }
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
using std::isfinite; using std::isnan; using std::isinf;
using std::fabs; using std::fmax; using std::fmin; using std::sqrt; using std::exp; using std::log; using std::pow;
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
inline double min(double a, double b) { return a < b ? a : b; }
inline double max(double a, double b) { return a > b ? a : b; }

// ------------------------------------------------------------------------------------------------ runtime API
typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16, cudaDevAttrMaxSharedMemoryPerBlockOptin = 97 };

inline cudaError_t cudaGetDeviceCount(int* c) { *c = 1; return 0; }
inline cudaError_t cudaSetDevice(int) { return 0; }
// EMU_GUARD=1: device memory comes from an arena the host may only touch inside copies, memsets and kernel launches
// (cuda_emu.cpp); a host-side dereference of a device pointer -- invisible otherwise, device memory being host memory
// here -- ends the process with SIGSEGV.
// Every resource is counted by kind (emu_live_resources), and any creation can be made to fail (emu_fail_alloc_at).
namespace emu {
enum { RES_DEV = 0, RES_HOST, RES_STREAM, RES_EVENT };
void* dev_alloc(size_t n);
void dev_free(void* p);
void* res_create(int kind, size_t n);     // pinned host memory, a stream or an event
void res_destroy(int kind, void* p);
void dev_open();
void dev_close();
struct DevScope { DevScope() { dev_open(); } ~DevScope() { dev_close(); } };
}
inline cudaError_t cudaMalloc(void** p, size_t n) { *p = emu::dev_alloc(n); return *p ? 0 : 2; }
inline cudaError_t cudaFree(void* p) { emu::dev_free(p); return 0; }
inline cudaError_t cudaMallocHost(void** p, size_t n) { *p = emu::res_create(emu::RES_HOST, n); return *p ? 0 : 2; }
inline cudaError_t cudaFreeHost(void* p) { emu::res_destroy(emu::RES_HOST, p); return 0; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, int) { emu::DevScope o; if (n) std::memmove(d, s, n); return 0; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t = nullptr) { emu::DevScope o; if (n) std::memmove(d, s, n); return 0; }
inline cudaError_t cudaMemset(void* d, int v, size_t n) { emu::DevScope o; if (n) std::memset(d, v, n); return 0; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { emu::DevScope o; if (n) std::memset(d, v, n); return 0; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = emu::res_create(emu::RES_STREAM, 1); return *s ? 0 : 2; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { emu::res_destroy(emu::RES_STREAM, s); return 0; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
inline cudaError_t cudaDeviceSynchronize() { return 0; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return 0; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = emu::res_create(emu::RES_EVENT, 1); return *e ? 0 : 2; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { emu::res_destroy(emu::RES_EVENT, e); return 0; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return 0; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return 0; }
inline cudaError_t cudaGetLastError() { return 0; }
inline const char* cudaGetErrorString(cudaError_t) { return "emulated CUDA runtime (tests/emu)"; }
template <class F> inline cudaError_t cudaFuncSetAttribute(F f, int attr, int v) {
  if (attr == 8) emu::note_smem_optin((const void*)f, v);      // cudaFuncAttributeMaxDynamicSharedMemorySize
  return 0;
}
inline cudaError_t cudaDeviceGetAttribute(int* v, int attr, int) { *v = attr == 97 ? 232448 : attr == 16 ? 2 : 0; return 0; }
template <class F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 2; return 0; }
