/* TEST INFRASTRUCTURE ONLY -- never shipped, never linked into the product library.
 *
 * A stand-in for the handful of CUDA runtime entry points libclarabel_b200.so imports, for LD_PRELOAD in a
 * SUBPROCESS of the CPU test-suite (tests/test_host_setup_cpu.py): device memory is host memory, copies are
 * memcpy, streams / events are tokens and KERNEL LAUNCHES ARE DROPPED.  Nothing numeric can be checked this way
 * (no kernel runs); what it makes checkable without a GPU is the HOST side of cipm_create / cldl_create: cone
 * collapsing, the inf-bound presolve, KKT assembly (pattern, signs, expansion columns), ordering, symbolic analysis
 * and plan construction run to completion, do not crash, and produce the same KKT structure as the oracle.
 * The product keeps failing loudly without a real device (tests/test_abi.py::test_no_cpu_fallback runs without
 * this shim). */
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef int cudaError_t;
struct dim3_ { unsigned x, y, z; };

cudaError_t cudaGetDeviceCount(int *c) { *c = 1; return 0; }
cudaError_t cudaSetDevice(int d) { (void)d; return 0; }
/* FAKE_CUDART_GUARD=1: "device" memory comes from one arena that the host may not touch (PROT_NONE) except inside the
   copy / memset entry points below.  Kernel launches are dropped, so nothing legitimate ever dereferences a device
   pointer on the host: a host-side read or write of device memory -- which the plain shim and the emulator cannot see,
   device memory being ordinary host memory there -- ends the process with SIGSEGV. */
#include <pthread.h>
#include <sys/mman.h>
static int guard_mode = -1;
static char *arena; static size_t arena_cap, arena_top;
static pthread_mutex_t arena_mu = PTHREAD_MUTEX_INITIALIZER;
static int arena_open_count;
static int guard_on(void)
{
    if (guard_mode < 0) { const char *e = getenv("FAKE_CUDART_GUARD"); guard_mode = (e && atoi(e)) ? 1 : 0; }
    return guard_mode;
}
static void arena_open(void)
{
    if (!guard_on() || !arena) return;
    pthread_mutex_lock(&arena_mu);
    if (arena_open_count++ == 0) mprotect(arena, arena_top ? arena_top : 4096, PROT_READ | PROT_WRITE);
    pthread_mutex_unlock(&arena_mu);
}
static void arena_close(void)
{
    if (!guard_on() || !arena) return;
    pthread_mutex_lock(&arena_mu);
    if (--arena_open_count == 0) mprotect(arena, arena_top ? arena_top : 4096, PROT_NONE);
    pthread_mutex_unlock(&arena_mu);
}
cudaError_t cudaMalloc(void **p, size_t n)
{
    if (!guard_on()) { *p = calloc(1, n ? n : 1); return *p ? 0 : 2; }
    pthread_mutex_lock(&arena_mu);
    if (!arena) {
        arena_cap = (size_t)64 << 30;
        arena = mmap(NULL, arena_cap, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (arena == MAP_FAILED) { arena = NULL; pthread_mutex_unlock(&arena_mu); return 2; }
    }
    const size_t need = ((n ? n : 1) + 4095) & ~(size_t)4095;      /* page granular: neighbours never share a page */
    if (arena_top + need + 4096 > arena_cap) { pthread_mutex_unlock(&arena_mu); return 2; }
    *p = arena + arena_top;
    arena_top += need + 4096;                                       /* one guard page between allocations */
    if (arena_open_count > 0) mprotect(arena, arena_top, PROT_READ | PROT_WRITE);
    {   /* FAKE_CUDART_FILL=<byte>: what an unlaunched kernel "left" in device memory; 0x3f makes every double 4.8e-4
           and every int32 about 1e9, so that the host drivers see non-converged, non-zero numbers and keep iterating */
        const char *f = getenv("FAKE_CUDART_FILL");
        if (f) {
            mprotect(*p, need, PROT_READ | PROT_WRITE);
            memset(*p, (int)strtol(f, NULL, 0), n);
            if (arena_open_count == 0) mprotect(*p, need, PROT_NONE);
        }
    }
    pthread_mutex_unlock(&arena_mu);
    return 0;
}
cudaError_t cudaFree(void *p)
{
    if (guard_on() && arena && (char *)p >= arena && (char *)p < arena + arena_cap) return 0;   /* never reused */
    free(p);
    return 0;
}
cudaError_t cudaMallocHost(void **p, size_t n) { *p = calloc(1, n ? n : 1); return *p ? 0 : 2; }
cudaError_t cudaFreeHost(void *p) { free(p); return 0; }
/* FAKE_CUDART_LOG=<file>: one line "bytes fnv1a64" per host-to-device copy, so that a change of the host-side plan
   builders can be checked to upload exactly the same arrays (compare the sorted logs) */
static void log_h2d(const void *s, size_t n, int kind)
{
    static const char *path = (const char *)-1;
    if (path == (const char *)-1) path = getenv("FAKE_CUDART_LOG");
    if (!path || kind != 1 || n == 0) return;
    uint64_t h = 1469598103934665603ull;
    const unsigned char *b = (const unsigned char *)s;
    for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 1099511628211ull; }
    FILE *f = fopen(path, "a");
    if (f) { fprintf(f, "%zu %016llx\n", n, (unsigned long long)h); fclose(f); }
}
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, int kind) { log_h2d(s, n, kind); arena_open(); if (n) memmove(d, s, n); arena_close(); return 0; }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, int kind, void *st) { (void)st; log_h2d(s, n, kind); arena_open(); if (n) memmove(d, s, n); arena_close(); return 0; }
cudaError_t cudaMemset(void *d, int v, size_t n) { arena_open(); if (n) memset(d, v, n); arena_close(); return 0; }
cudaError_t cudaMemsetAsync(void *d, int v, size_t n, void *st) { (void)st; arena_open(); if (n) memset(d, v, n); arena_close(); return 0; }
cudaError_t cudaStreamCreateWithFlags(void **s, unsigned f) { (void)f; *s = malloc(1); return 0; }
cudaError_t cudaStreamDestroy(void *s) { free(s); return 0; }
cudaError_t cudaStreamSynchronize(void *s) { (void)s; return 0; }
cudaError_t cudaDeviceSynchronize(void) { return 0; }
cudaError_t cudaStreamWaitEvent(void *s, void *e, unsigned f) { (void)s; (void)e; (void)f; return 0; }
cudaError_t cudaEventCreate(void **e) { *e = malloc(1); return 0; }
cudaError_t cudaEventCreateWithFlags(void **e, unsigned f) { (void)f; *e = malloc(1); return 0; }
cudaError_t cudaEventDestroy(void *e) { free(e); return 0; }
cudaError_t cudaEventRecord(void *e, void *s) { (void)e; (void)s; return 0; }
cudaError_t cudaEventSynchronize(void *e) { (void)e; return 0; }
cudaError_t cudaEventElapsedTime(float *ms, void *a, void *b) { (void)a; (void)b; *ms = 0.0f; return 0; }
cudaError_t cudaFuncSetAttribute(const void *f, int a, int v) { (void)f; (void)a; (void)v; return 0; }
cudaError_t cudaDeviceGetAttribute(int *v, int attr, int dev)
{
    (void)dev;
    *v = attr == 97 ? 232448 /* max opt-in shared memory per block (H100) */ : attr == 16 ? 132 /* SMs */ : 0;
    return 0;
}
cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(int *n, const void *f, int bs, size_t sm, unsigned fl)
{ (void)f; (void)bs; (void)sm; (void)fl; *n = 2; return 0; }
cudaError_t cudaGetLastError(void) { return 0; }
const char *cudaGetErrorString(cudaError_t e) { (void)e; return "fake cudart (tests/host_harness)"; }
cudaError_t cudaLaunchKernel(const void *f, struct dim3_ g, struct dim3_ b, void **args, size_t sm, void *st)
{ (void)f; (void)g; (void)b; (void)args; (void)sm; (void)st; return 0; }
/* launch stubs: "if (__cudaPushCallConfiguration(...) == 0) stub(args)": a non-zero return drops the launch */
unsigned __cudaPushCallConfiguration(struct dim3_ g, struct dim3_ b, size_t sm, void *st) { (void)g; (void)b; (void)sm; (void)st; return 1; }
cudaError_t __cudaPopCallConfiguration(struct dim3_ *g, struct dim3_ *b, size_t *sm, void *st) { (void)g; (void)b; (void)sm; (void)st; return 0; }
static void *fat_handle[4];
void **__cudaRegisterFatBinary(void *f) { (void)f; return fat_handle; }
void __cudaRegisterFatBinaryEnd(void **h) { (void)h; }
void __cudaUnregisterFatBinary(void **h) { (void)h; }
void __cudaRegisterFunction(void **h, const char *hf, char *df, const char *dn, int tl, void *tid, void *bid, void *bd, void *gd, int *ws)
{ (void)h; (void)hf; (void)df; (void)dn; (void)tl; (void)tid; (void)bid; (void)bd; (void)gd; (void)ws; }
void __cudaRegisterVar(void **h, char *hv, char *da, const char *dn, int ext, size_t sz, int cst, int glb)
{ (void)h; (void)hv; (void)da; (void)dn; (void)ext; (void)sz; (void)cst; (void)glb; }
