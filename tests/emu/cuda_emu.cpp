// TEST INFRASTRUCTURE ONLY.  Fiber scheduler behind tests/emu/cuda_emu.h.
//
// One fiber per CUDA thread.  Blocks of a launch run one after the other, unless the whole grid is small enough to
// be resident at once (EMU_MAX_RESIDENT threads): then all its blocks run concurrently, which is what the persistent
// dataflow kernels of ldl.cu need (their blocks wait on each other through counters in global memory and call
// __nanosleep while they spin -- a yield point here).  __syncthreads / __syncwarp / shuffles / votes park a fiber
// until its block / warp has arrived.  EMU_ORDER=reverse walks the fibers in descending order.
#include "cuda_emu.h"

#include <sys/mman.h>
#include <atomic>
#include <cstring>
#include <mutex>
#include <utility>

#include <map>
#include <vector>

extern "C" void emu_switch(void** from_sp, void* to_sp);
asm(R"(
.text
.globl emu_switch
.type emu_switch,@function
emu_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size emu_switch,.-emu_switch
)");

namespace emu {

enum { READY = 0, DONE = 1, WAIT_BLOCK = 2, WAIT_WARP = 3 };
constexpr size_t STACK_BYTES = 512 * 1024;
constexpr int EMU_MAX_RESIDENT = 4096;

struct Block {
  uint3 idx{0, 0, 0};
  int first = 0, nthreads = 0;               // fibers[first .. first+nthreads)
  std::vector<char> dyn;                     // dynamic shared memory
  std::vector<uint64_t> warp_slot;           // [nwarps][32]
  std::map<int, void*> shared;               // static __shared__ variables by declaration site
  ~Block() { for (auto& kv : shared) std::free(kv.second); }
};
struct Fiber {
  void* sp = nullptr;
  char* stack = nullptr;
  int state = DONE;
  uint3 tid{0, 0, 0};
  int lin = 0;                               // linear thread index inside its block
  Block* blk = nullptr;
};

uint3 g_blockDim{1, 1, 1}, g_gridDim{1, 1, 1};
static uint3 zero3{0, 0, 0};
static std::vector<Fiber> fibers;            // stacks are kept across launches
static Fiber* cur = nullptr;
static void* sched_sp = nullptr;
static const std::function<void()>* body_fn = nullptr;
static bool spun = false;                    // the running fiber yielded from a spin-wait
// EMU_ORDER: "reverse" = descending thread order; "random[:seed]" = a fresh random permutation of the resident fibers in
// every scheduling pass (the most adversarial schedule: lanes of a warp and blocks of a grid interleave arbitrarily
// between their synchronisation points)
static const bool reverse_order = [] { const char* e = std::getenv("EMU_ORDER"); return e && e[0] == 'r' && e[1] == 'e'; }();
static const bool random_order = [] { const char* e = std::getenv("EMU_ORDER"); return e && e[0] == 'r' && e[1] == 'a'; }();
static uint64_t rng_state = [] {
  const char* e = std::getenv("EMU_ORDER");
  const char* c = e ? std::strchr(e, ':') : nullptr;
  return (uint64_t)(c ? std::atoll(c + 1) : 1) * 0x9E3779B97F4A7C15ull + 0x1234567ull;
}();
static inline uint64_t rng_next() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }

uint3& cur_tid() { return cur ? cur->tid : zero3; }
uint3& cur_bid() { return cur ? cur->blk->idx : zero3; }
void* dyn_smem() { return cur->blk->dyn.data(); }
int lane_id() { return cur->lin & 31; }
// shared memory is not cleared at block start on the device: 0xCB here as well (EMU_POISON=0: zeros)
static int shared_fill() {
  static int v = -1;
  if (v < 0) { const char* e = std::getenv("EMU_POISON"); v = (e && !std::atoi(e)) ? 0 : 0xCB; }
  return v;
}
void* shared_slot(int id, size_t bytes) {
  void*& p = cur->blk->shared[id];
  if (!p) { if (posix_memalign(&p, 64, bytes ? bytes : 8)) std::abort(); std::memset(p, shared_fill(), bytes ? bytes : 8); }
  return p;
}

static void yield_to_scheduler() { emu_switch(&cur->sp, sched_sp); }
void spin_yield() { spun = true; yield_to_scheduler(); }

static void fiber_main() {
  (*body_fn)();
  cur->state = DONE;
  yield_to_scheduler();
  std::fprintf(stderr, "[emu] finished fiber resumed\n");
  std::abort();
}

static void prepare(Fiber& f) {
  if (!f.stack) {
    void* p = mmap(nullptr, STACK_BYTES, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) { std::perror("[emu] mmap"); std::abort(); }
    f.stack = (char*)p;
  }
  uintptr_t top = ((uintptr_t)f.stack + STACK_BYTES) & ~(uintptr_t)15;
  void** base = (void**)(top - 64);          // 6 callee-saved registers, return address, 8 bytes of padding
  for (int i = 0; i < 6; i++) base[i] = nullptr;
  base[6] = (void*)&fiber_main;
  f.sp = base;
  f.state = READY;
}

void sync_block() { cur->state = WAIT_BLOCK; yield_to_scheduler(); }
void sync_warp() { cur->state = WAIT_WARP; yield_to_scheduler(); }

uint64_t warp_exchange(uint64_t bits, int src_lane) {
  Block* b = cur->blk;
  const int w = cur->lin >> 5;
  b->warp_slot[(size_t)w * 32 + (cur->lin & 31)] = bits;
  sync_warp();
  const uint64_t r = b->warp_slot[(size_t)w * 32 + src_lane];
  sync_warp();
  return r;
}
unsigned warp_vote(bool pred) {
  Block* b = cur->blk;
  const int w = cur->lin >> 5;
  b->warp_slot[(size_t)w * 32 + (cur->lin & 31)] = pred ? 1u : 0u;
  sync_warp();
  unsigned m = 0;
  const int lo = w * 32, hi = lo + 32 < b->nthreads ? lo + 32 : b->nthreads;
  for (int t = lo; t < hi; t++) if (fibers[b->first + t].state != DONE && b->warp_slot[(size_t)w * 32 + (t & 31)]) m |= 1u << (t & 31);
  sync_warp();
  return m;
}

// run the fibers [0, total) (one or several blocks) to completion
static std::vector<int> order;
static void run_resident(std::vector<Block>& blocks, int total) {
  for (int t = 0; t < total; t++) prepare(fibers[t]);
  long long idle_passes = 0;
  for (;;) {
    bool progressed = false, any_live = false;
    if (random_order) {
      if ((int)order.size() != total) { order.resize(total); for (int i = 0; i < total; i++) order[i] = i; }
      for (int i = total - 1; i > 0; i--) { const int j = (int)(rng_next() % (uint64_t)(i + 1)); std::swap(order[i], order[j]); }
    }
    for (int t0 = 0; t0 < total; t0++) {
      const int t = random_order ? order[t0] : (reverse_order ? total - 1 - t0 : t0);
      Fiber& f = fibers[t];
      if (f.state != READY) { if (f.state != DONE) any_live = true; continue; }
      any_live = true;
      cur = &f;
      spun = false;
      emu_switch(&sched_sp, f.sp);
      cur = nullptr;
      if (!spun) progressed = true;            // a fiber that only spun has not changed anything
    }
    if (!any_live) break;
    for (Block& b : blocks) {
      const int nw = (b.nthreads + 31) / 32;
      for (int w = 0; w < nw; w++) {           // complete warp rendezvous
        const int lo = b.first + w * 32, hi = lo + 32 < b.first + b.nthreads ? lo + 32 : b.first + b.nthreads;
        bool all = true, some = false;
        for (int t = lo; t < hi; t++) {
          if (fibers[t].state == WAIT_WARP) some = true;
          else if (fibers[t].state != DONE) all = false;
        }
        if (some && all) { for (int t = lo; t < hi; t++) if (fibers[t].state == WAIT_WARP) fibers[t].state = READY; progressed = true; }
      }
      bool all = true, some = false;           // complete block barrier
      for (int t = b.first; t < b.first + b.nthreads; t++) {
        if (fibers[t].state == WAIT_BLOCK) some = true;
        else if (fibers[t].state != DONE) all = false;
      }
      if (some && all) { for (int t = b.first; t < b.first + b.nthreads; t++) if (fibers[t].state == WAIT_BLOCK) fibers[t].state = READY; progressed = true; }
    }
    if (progressed) idle_passes = 0;
    else if (++idle_passes > 200000) {
      std::fprintf(stderr, "[emu] no progress: deadlock or a spin-wait nobody will satisfy (%zu resident blocks)\n", blocks.size());
      for (Block& b : blocks) {
        std::fprintf(stderr, "  block (%u,%u,%u):", b.idx.x, b.idx.y, b.idx.z);
        for (int t = 0; t < b.nthreads && t < 40; t++) std::fprintf(stderr, " %d", fibers[b.first + t].state);
        std::fprintf(stderr, "\n");
      }
      std::abort();
    }
  }
}

// ---- guarded device memory (EMU_GUARD=1) ----
extern std::vector<std::pair<size_t, size_t>> g_blocks;      // (offset, bytes) of every allocation
namespace {
std::mutex g_mu;
char* g_arena = nullptr;
size_t g_cap = 0, g_top = 0;
int g_open = 0;
int guard_mode() {
  static int v = -1;
  if (v < 0) { const char* e = std::getenv("EMU_GUARD"); v = (e && std::atoi(e)) ? 1 : 0; }
  return v;
}
}  // namespace

// cudaMalloc does not clear memory: new allocations are filled with 0xCB bytes (a double of about -6e57, an int of about
// -875 million), so that code which silently relies on zeroed device memory shows here.  EMU_POISON=0 turns it off.
static int poison_mode() {
  static int v = -1;
  if (v < 0) { const char* e = std::getenv("EMU_POISON"); v = (e && !std::atoi(e)) ? 0 : 1; }
  return v;
}
// live resources by kind, and the countdown to the creation that is made to fail (0: none)
static std::atomic<int64_t> g_live[4];
static std::atomic<int> g_fail_in{0};
static bool fail_now() {
  int k = g_fail_in.load();
  while (k > 0 && !g_fail_in.compare_exchange_weak(k, k - 1)) {}
  return k == 1;
}
void* res_create(int kind, size_t n) {
  if (fail_now()) return nullptr;
  void* p = std::calloc(1, n ? n : 1);
  if (p) g_live[kind]++;
  return p;
}
void res_destroy(int kind, void* p) {
  if (!p) return;
  g_live[kind]--;
  std::free(p);
}

static void* dev_alloc_raw(size_t n);
void* dev_alloc(size_t n) {
  if (fail_now()) return nullptr;
  void* p = dev_alloc_raw(n);
  if (p) g_live[RES_DEV]++;
  return p;
}
static void* dev_alloc_raw(size_t n) {
  if (!guard_mode()) {
    void* p = std::malloc(n ? n : 1);
    if (p) std::memset(p, poison_mode() ? 0xCB : 0, n ? n : 1);
    return p;
  }
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_arena) {
    g_cap = (size_t)64 << 30;
    void* a = mmap(nullptr, g_cap, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (a == MAP_FAILED) return nullptr;
    g_arena = (char*)a;
  }
  const size_t need = ((n ? n : 1) + 4095) & ~(size_t)4095;
  if (g_top + need > g_cap) return nullptr;
  void* p = g_arena + g_top;
  g_blocks.emplace_back(g_top, need);
  g_top += need;
  mprotect(p, need, PROT_READ | PROT_WRITE);
  if (poison_mode()) std::memset(p, 0xCB, need);
  if (g_open == 0) mprotect(p, need, PROT_NONE);
  return p;
}
void dev_free(void* p) {
  if (!p) return;
  g_live[RES_DEV]--;
  if (guard_mode() && g_arena && (char*)p >= g_arena && (char*)p < g_arena + g_cap) return;   // never reused
  std::free(p);
}
// open / close: one mprotect over the used part of the arena (a launch-heavy test makes ~1e5 of these calls)
static void protect_all(int prot) { if (g_top) mprotect(g_arena, g_top, prot); }
std::vector<std::pair<size_t, size_t>> g_blocks;
void dev_open() {
  if (!guard_mode()) return;
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_open++ == 0 && g_arena) protect_all(PROT_READ | PROT_WRITE);
}
void dev_close() {
  if (!guard_mode()) return;
  std::lock_guard<std::mutex> lk(g_mu);
  if (--g_open == 0 && g_arena) protect_all(PROT_NONE);
}

static std::map<const void*, int> g_smem_optin;
static std::mutex g_smem_mu;
void note_smem_optin(const void* fn, int bytes) { std::lock_guard<std::mutex> lk(g_smem_mu); g_smem_optin[fn] = bytes; }
void check_smem_optin(const void* fn, size_t smem) {
  if (smem <= 48 * 1024) return;
  std::lock_guard<std::mutex> lk(g_smem_mu);
  auto it = g_smem_optin.find(fn);
  if (it == g_smem_optin.end() || (size_t)it->second < smem) {
    std::fprintf(stderr, "[emu] launch with %zu bytes of dynamic shared memory, opt-in %d: the device refuses this launch\n", smem,
                 it == g_smem_optin.end() ? 0 : it->second);
    std::abort();
  }
}

void run_grid(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body) {
  if (cur) { std::fprintf(stderr, "[emu] nested launch\n"); std::abort(); }
  DevScope dev_scope;
  const int bt = (int)(block.x * block.y * block.z);
  const long long nblocks = (long long)grid.x * grid.y * grid.z;
  // what the hardware refuses with "invalid configuration argument" must not pass silently here
  if (bt <= 0 || bt > 1024 || nblocks == 0 || grid.y > 65535u || grid.z > 65535u || grid.x > 2147483647u || block.z > 64u ||
      smem > 232448) {
    std::fprintf(stderr, "[emu] invalid launch configuration: grid (%u,%u,%u) block (%u,%u,%u) smem %zu\n", grid.x, grid.y, grid.z,
                 block.x, block.y, block.z, smem);
    std::abort();
  }
  body_fn = &body;
  g_blockDim = uint3{block.x, block.y, block.z};
  g_gridDim = uint3{grid.x, grid.y, grid.z};
  const bool all_resident = nblocks * bt <= EMU_MAX_RESIDENT;
  const int batch = all_resident ? (int)nblocks : 1;
  if ((int)fibers.size() < batch * bt) fibers.resize((size_t)batch * bt);
  std::vector<Block> blocks;
  auto flush = [&]() {
    if (blocks.empty()) return;
    run_resident(blocks, (int)blocks.size() * bt);
    blocks.clear();
  };
  blocks.reserve(batch);
  for (unsigned bz = 0; bz < grid.z; bz++)
    for (unsigned by = 0; by < grid.y; by++)
      for (unsigned bx = 0; bx < grid.x; bx++) {
        blocks.emplace_back();
        Block& b = blocks.back();
        b.idx = uint3{bx, by, bz};
        b.first = ((int)blocks.size() - 1) * bt;
        b.nthreads = bt;
        b.dyn.assign(smem + 64, (char)shared_fill());
        b.warp_slot.assign((size_t)((bt + 31) / 32) * 32, 0);
        int lin = 0;
        for (unsigned tz = 0; tz < block.z; tz++)
          for (unsigned ty = 0; ty < block.y; ty++)
            for (unsigned tx = 0; tx < block.x; tx++, lin++) {
              Fiber& f = fibers[b.first + lin];
              f.tid = uint3{tx, ty, tz}; f.lin = lin; f.blk = &b;
            }
        if ((int)blocks.size() == batch) flush();
      }
  flush();
  body_fn = nullptr;
}

}  // namespace emu

extern "C" void emu_live_resources(int64_t out[4]) {
  for (int k = 0; k < 4; k++) out[k] = emu::g_live[k].load();
}
// the k-th creation of a resource from now (device or pinned memory, stream, event) fails; 0 disarms
extern "C" void emu_fail_alloc_at(int k) { emu::g_fail_in.store(k > 0 ? k : 0); }
