// Host-side SIMT emulator for the flpr CUDA-core kernels (tests only; no GPU, no CUDA runtime call).
//
// A kernel source is compiled as plain C++ (tests/emu/build_emu.py rewrites `k<<<grid, block, smem, stream>>>(args)` into
// flpr_emu::launch(...), turns `__shared__` declarations into block-local storage, drops the inline-PTX helpers and
// includes this header instead of csrc/ptx.cuh). Every CUDA thread is a ucontext fiber on ONE OS thread:
//   * __syncthreads / __syncthreads_or : cooperative block barrier (threads that returned from the kernel stop counting,
//                                        as on the hardware);
//   * __shfl_xor_sync / __shfl_sync / __shfl_down_sync : exchange through a per-warp buffer between two warp barriers -
//                                        the lanes really read each other's registers, so a wrong lane mask or a shuffle
//                                        under divergent control flow shows up as a wrong result or a reported deadlock;
//   * __shared__                       : storage owned by the running block.
// Two execution modes:
//   * immediate (default): `launch` runs the grid block by block and returns when the kernel is done (layer_ops.cu);
//   * deferred (flpr_emu_defer(1)): launches are queued per stream key; flpr_emu_run(seed, ...) then executes ALL queues
//     concurrently - kernels of one queue in order, every block of a running kernel resident, fibers picked in a seeded
//     random order with random stalls. This is how the peer-memory collectives of fedcomm.cu run here: R "ranks" are R
//     queues whose kernels spin on each other's flags (`ld_acquire_sys` yields), under many different interleavings, with
//     a virtual `%globaltimer` so that the watchdog path is testable, and an emulated NVSwitch multicast window for the
//     `multimem` instructions.
// What this checks: index mathematics, reductions, barrier placement, the flag / epoch protocol under sequentially
// consistent interleavings, argument marshalling of the extern "C" entry points. What it cannot check: alignment
// faults, weak-memory-model effects (missing fences), performance.
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <deque>
#include <functional>
#include <map>
#include <vector>

#undef __global__
#define __global__
#undef __device__
#define __device__
#undef __launch_bounds__
#define __launch_bounds__(...)
#undef __forceinline__
#define __forceinline__ inline

namespace flpr_emu {

struct Dim3 {
  unsigned x = 0, y = 0, z = 0;
};

static inline Dim3 dims(const dim3& d) {
  Dim3 o;
  o.x = d.x; o.y = d.y; o.z = d.z;
  return o;
}
template <class T>
static inline Dim3 dims(T v) {
  Dim3 o;
  o.x = (unsigned)v; o.y = 1; o.z = 1;
  return o;
}
static inline unsigned volume(const Dim3& d) { return d.x * d.y * d.z; }

constexpr int MAX_THREADS = 1024;
constexpr size_t STACK_BYTES = 32 * 1024;

struct Block;
struct KernelRun;

struct Fiber {
  ucontext_t ctx;
  Block* blk = nullptr;
  Dim3 tid;
  unsigned lin = 0;              // linear thread id (warp = lin / 32, lane = lin % 32)
  bool done = false;
};

struct WarpState {
  int alive = 0, count = 0;
  unsigned gen = 0;
  uint64_t buf[32];
};

struct Block {
  KernelRun* k = nullptr;
  Dim3 bid;
  int n = 0, alive = 0;
  int sync_count = 0, sync_or = 0, sync_or_result = 0;
  unsigned sync_gen = 0;
  std::vector<WarpState> warps;
  std::vector<Fiber> fibers;
  std::map<int, void*> shared;
  void* dyn_shared = nullptr;    // `extern __shared__` storage (size from the launch configuration)
  char* stacks = nullptr;
};

struct KernelRun {
  Dim3 gdim, bdim;
  size_t smem = 0;               // dynamic shared memory per block
  std::function<void()> body;
  std::vector<Block*> blocks;
  unsigned slow = 0;             // deferred runs: this kernel's threads only run in one of `slow` passes (a slow rank)
};

struct Pending {
  Dim3 grid, block;
  size_t smem;
  std::function<void()> body;
};

struct Multicast {
  char* base;
  size_t bytes;
  std::vector<char*> members;
};

// (internal linkage: one emulator state per emulated library)
static Fiber* g_cur = nullptr;
static ucontext_t g_main;
static unsigned long long g_progress = 0;   // bumped whenever a barrier releases or a thread exits
static unsigned long long g_clock_ns = 0;   // virtual %globaltimer
static int g_deadlocks = 0;
static bool g_defer = false;
static unsigned g_stall_one_in = 0;         // deferred runs: a memory-op yield point stalls with probability 1 / this
static uint64_t g_rng = 0x9e3779b97f4a7c15ull;
static std::map<const void*, std::deque<Pending>> g_queues;
static std::map<const void*, int> g_start_delay;
static std::map<const void*, unsigned> g_lane_slow;
static std::vector<Multicast> g_mc;

static inline uint64_t rnd() {
  g_rng ^= g_rng << 13;
  g_rng ^= g_rng >> 7;
  g_rng ^= g_rng << 17;
  return g_rng;
}

static inline void yield() {
  Fiber* me = g_cur;
  swapcontext(&me->ctx, &g_main);
}
static inline void maybe_yield() {
  if (g_stall_one_in && rnd() % g_stall_one_in == 0) yield();
}

static inline void release_block_barrier(Block& b) {
  b.sync_or_result = b.sync_or;
  b.sync_or = 0;
  b.sync_count = 0;
  b.sync_gen++;
  g_progress++;
}

static inline int sync_impl(int pred) {
  Block& b = *g_cur->blk;
  const unsigned g = b.sync_gen;
  b.sync_or |= (pred != 0);
  if (++b.sync_count == b.alive)
    release_block_barrier(b);
  else
    while (b.sync_gen == g) yield();
  return b.sync_or_result;
}

static inline void warp_barrier() {
  WarpState& w = g_cur->blk->warps[g_cur->lin >> 5];
  const unsigned g = w.gen;
  if (++w.count == w.alive) {
    w.count = 0;
    w.gen++;
    g_progress++;
  } else {
    while (w.gen == g) yield();
  }
}

static inline uint64_t exchange(uint64_t v, int src_lane) {
  WarpState& w = g_cur->blk->warps[g_cur->lin >> 5];
  w.buf[g_cur->lin & 31] = v;
  warp_barrier();
  const uint64_t r = w.buf[src_lane & 31];
  warp_barrier();
  return r;
}

template <class T>
static inline T shfl_from(T v, int src_lane) {
  static_assert(sizeof(T) <= 8, "shuffle payload");
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  bits = exchange(bits, src_lane);
  T out;
  memcpy(&out, &bits, sizeof(T));
  return out;
}

// block-local storage behind a `__shared__` declaration (id = position of the declaration in the source)
template <class T>
static inline T* shared(int id) {
  Block& b = *g_cur->blk;
  auto it = b.shared.find(id);
  if (it == b.shared.end()) it = b.shared.emplace(id, calloc(1, sizeof(T))).first;
  return reinterpret_cast<T*>(it->second);
}

// storage behind `extern __shared__ T name[]`
static inline void* dyn_shared() {
  Block& b = *g_cur->blk;
  if (b.dyn_shared == nullptr) b.dyn_shared = calloc(1, b.k->smem + 1024);
  return b.dyn_shared;
}

[[noreturn]] static inline void unsupported(const char* what) {
  fprintf(stderr, "[flpr_emu] %s is a tensor-core / TMA instruction: this kernel cannot run under the emulator\n", what);
  abort();
}

static void fiber_entry() {
  Fiber* me = g_cur;
  me->blk->k->body();
  Block& b = *me->blk;
  WarpState& w = b.warps[me->lin >> 5];
  me->done = true;
  b.alive--;
  w.alive--;
  g_progress++;
  // threads that exited no longer take part in barriers: release the ones that were only waiting for this thread
  if (b.sync_count > 0 && b.sync_count == b.alive) release_block_barrier(b);
  if (w.count > 0 && w.count == w.alive) {
    w.count = 0;
    w.gen++;
  }
  // uc_link returns to g_main
}

static Block* make_block(KernelRun* k, unsigned bid) {
  const unsigned n = volume(k->bdim);
  Block* b = new Block();
  b->k = k;
  b->bid.x = bid % k->gdim.x;
  b->bid.y = (bid / k->gdim.x) % k->gdim.y;
  b->bid.z = bid / (k->gdim.x * k->gdim.y);
  b->n = b->alive = (int)n;
  b->warps.resize((n + 31) / 32);
  for (unsigned w = 0; w < b->warps.size(); ++w) b->warps[w].alive = (int)((n - w * 32 >= 32) ? 32 : n - w * 32);
  b->fibers.resize(n);
  b->stacks = (char*)malloc(STACK_BYTES * n);
  for (unsigned t = 0; t < n; ++t) {
    Fiber& f = b->fibers[t];
    f.blk = b;
    f.lin = t;
    f.tid.x = t % k->bdim.x;
    f.tid.y = (t / k->bdim.x) % k->bdim.y;
    f.tid.z = t / (k->bdim.x * k->bdim.y);
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = b->stacks + STACK_BYTES * t;
    f.ctx.uc_stack.ss_size = STACK_BYTES;
    f.ctx.uc_link = &g_main;
    makecontext(&f.ctx, (void (*)())fiber_entry, 0);
  }
  return b;
}

static void free_block(Block* b) {
  for (auto& kv : b->shared) free(kv.second);
  free(b->dyn_shared);
  free(b->stacks);
  delete b;
}

static inline void resume(Fiber* f) {
  g_cur = f;
  swapcontext(&g_main, &f->ctx);
  g_cur = nullptr;
}

static void check_block_size(const Dim3& block) {
  if (volume(block) == 0 || volume(block) > (unsigned)MAX_THREADS) {
    fprintf(stderr, "[flpr_emu] unsupported block size %u\n", volume(block));
    abort();
  }
}

// immediate mode: one block at a time
static void run_now(const Dim3& grid, const Dim3& block, size_t smem, const std::function<void()>& body) {
  check_block_size(block);
  KernelRun k;
  k.smem = smem;
  k.gdim = grid;
  k.bdim = block;
  k.body = body;
  const unsigned nthreads = volume(block);
  for (unsigned bid = 0; bid < volume(grid); ++bid) {
    Block* b = make_block(&k, bid);
    unsigned long long last = ~0ull;
    int idle_rounds = 0;
    while (b->alive > 0) {
      for (unsigned t = 0; t < nthreads; ++t)
        if (!b->fibers[t].done) resume(&b->fibers[t]);
      if (g_progress == last) {
        if (++idle_rounds > 4) {   // every live thread is parked at a barrier that can never release
          fprintf(stderr, "[flpr_emu] deadlock in block %u: %d threads wait at a barrier not every live thread reaches\n",
                  bid, b->alive);
          g_deadlocks++;
          break;
        }
      } else {
        idle_rounds = 0;
        last = g_progress;
      }
    }
    free_block(b);
  }
}

static inline void launch(const Dim3& grid, const Dim3& block, size_t smem, const void* stream_key,
                          const std::function<void()>& body) {
  if (!g_defer) {
    run_now(grid, block, smem, body);
    return;
  }
  check_block_size(block);
  g_queues[stream_key].push_back(Pending{grid, block, smem, body});
}

// deferred mode: every queue concurrently, kernels of a queue in order, all blocks of a running kernel resident
static int run_queues(unsigned seed, long max_passes, unsigned stall_one_in) {
  struct Lane {
    const void* key;
    std::deque<Pending>* q;
    KernelRun* cur = nullptr;
    int delay = 0;
  };
  std::vector<Lane> lanes;
  for (auto& kv : g_queues) {
    Lane l;
    l.key = kv.first;
    l.q = &kv.second;
    auto d = g_start_delay.find(kv.first);
    l.delay = d == g_start_delay.end() ? 0 : d->second;
    lanes.push_back(l);
  }
  g_rng = 0x9e3779b97f4a7c15ull ^ ((uint64_t)seed * 0xbf58476d1ce4e5b9ull);
  g_stall_one_in = seed ? stall_one_in : 0;
  std::vector<Fiber*> live;
  int rc = 0;
  long pass = 0;
  for (;; ++pass) {
    bool changed = false, any = false;
    for (Lane& l : lanes) {
      if (l.cur != nullptr) {
        bool done = true;
        for (Block* b : l.cur->blocks) done = done && b->alive == 0;
        if (done) {
          for (Block* b : l.cur->blocks) free_block(b);
          delete l.cur;
          l.cur = nullptr;
          l.q->pop_front();
          changed = true;
        }
      }
      if (l.cur == nullptr && !l.q->empty()) {
        if (l.delay > 0) {
          l.delay--;
        } else {
          const Pending& p = l.q->front();
          KernelRun* k = new KernelRun();
          k->gdim = p.grid;
          k->bdim = p.block;
          k->body = p.body;
          k->smem = p.smem;
          auto sl = g_lane_slow.find(l.key);
          k->slow = (seed && sl != g_lane_slow.end()) ? sl->second : 0;
          for (unsigned bid = 0; bid < volume(p.grid); ++bid) k->blocks.push_back(make_block(k, bid));
          l.cur = k;
          changed = true;
          if (seed) l.delay = (int)(rnd() % 3);      // host-side gap before this lane's NEXT launch
        }
      }
      any = any || l.cur != nullptr || !l.q->empty();
    }
    if (!any) break;
    if (pass >= max_passes) {
      fprintf(stderr, "[flpr_emu] %ld scheduler passes without completion: deadlock (or a livelock)\n", pass);
      g_deadlocks++;
      rc = 1;
      break;
    }
    if (changed || live.empty()) {
      live.clear();
      for (Lane& l : lanes)
        if (l.cur != nullptr)
          for (Block* b : l.cur->blocks)
            for (Fiber& f : b->fibers)
              if (!f.done) live.push_back(&f);
    }
    if (seed) {
      for (size_t i = live.size(); i > 1; --i) {
        const size_t j = rnd() % i;
        Fiber* t = live[i - 1];
        live[i - 1] = live[j];
        live[j] = t;
      }
    }
    size_t kept = 0;
    for (size_t i = 0; i < live.size(); ++i) {
      Fiber* f = live[i];
      const unsigned slow = f->blk->k->slow;
      const bool stalled = seed && (rnd() % 5 == 0 || (slow > 1 && rnd() % slow != 0));   // this fiber skips the pass
      if (!f->done && !stalled) resume(f);
      if (!f->done) live[kept++] = f;
    }
    live.resize(kept);
    g_clock_ns += 1000;
  }
  // abandoned work (deadlock): release it
  for (Lane& l : lanes) {
    if (l.cur != nullptr) {
      for (Block* b : l.cur->blocks) free_block(b);
      delete l.cur;
    }
  }
  g_queues.clear();
  g_start_delay.clear();
  g_lane_slow.clear();
  g_stall_one_in = 0;
  return rc;
}

static inline const Multicast* find_mc(const void* p) {
  const char* c = reinterpret_cast<const char*>(p);
  for (const Multicast& m : g_mc)
    if (c >= m.base && c < m.base + m.bytes) return &m;
  fprintf(stderr, "[flpr_emu] multimem access outside every registered multicast window\n");
  abort();
}

}  // namespace flpr_emu

#define threadIdx (flpr_emu::g_cur->tid)
#define blockIdx (flpr_emu::g_cur->blk->bid)
#define blockDim (flpr_emu::g_cur->blk->k->bdim)
#define gridDim (flpr_emu::g_cur->blk->k->gdim)

static inline void __syncthreads() { flpr_emu::sync_impl(0); }
static inline int __syncthreads_or(int pred) { return flpr_emu::sync_impl(pred); }
static inline void __syncwarp(unsigned = 0xffffffffu) { flpr_emu::warp_barrier(); }
static inline void __threadfence_system() {}
static inline void __threadfence() {}

template <class T>
static inline T __shfl_xor_sync(unsigned, T v, int lane_mask) {
  return flpr_emu::shfl_from(v, (int)(flpr_emu::g_cur->lin & 31) ^ lane_mask);
}
template <class T>
static inline T __shfl_sync(unsigned, T v, int src_lane) {
  return flpr_emu::shfl_from(v, src_lane);
}
template <class T>
static inline T __shfl_down_sync(unsigned, T v, unsigned delta) {
  const int l = (int)(flpr_emu::g_cur->lin & 31);
  const T r = flpr_emu::shfl_from(v, l + (int)delta);
  return (l + (int)delta < 32) ? r : v;
}

static inline unsigned atomicExch(unsigned* p, unsigned v) {
  const unsigned o = *p;
  *p = v;
  return o;
}
static inline float atomicAdd(float* p, float v) {
  const float o = *p;
  *p = o + v;
  return o;
}
static inline int atomicAdd(int* p, int v) {
  const int o = *p;
  *p = o + v;
  return o;
}
static inline int atomicMin(int* p, int v) {
  const int o = *p;
  if (v < o) *p = v;
  return o;
}
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
#define __expf(x) expf(x)
template <class T>
static inline T min(T a, T b) { return b < a ? b : a; }
template <class T>
static inline T max(T a, T b) { return a < b ? b : a; }
static inline float __uint_as_float(unsigned u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}
#undef __align__
#define __align__(n) alignas(n)

// ---- the pieces of csrc/ptx.cuh (and the inline-PTX helpers of the kernel sources) the CUDA-core kernels use ------------------
namespace flpr {
static inline void bind_device_of(const void*) {}
static inline float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
static inline float warp_max(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// wgmma / shared-space helpers of ptx.cuh: declared so that a source which ALSO contains a tensor-core kernel compiles
static inline uint32_t smem_u32(const void*) { flpr_emu::unsupported("cvta.shared"); }
static inline void fence_proxy_async() { flpr_emu::unsupported("fence.proxy.async"); }
static inline uint64_t make_smem_desc_sw128(uint32_t, uint32_t, uint32_t) { flpr_emu::unsupported("smem descriptor"); }
static inline void sts_128(uint32_t, const uint4&) { flpr_emu::unsupported("st.shared.v4"); }
static inline void reg_fence(float&) { flpr_emu::unsupported("wgmma register fence"); }
static inline void wgmma_fence() { flpr_emu::unsupported("wgmma.fence"); }
static inline void wgmma_commit() { flpr_emu::unsupported("wgmma.commit_group"); }
template <int N>
static inline void wgmma_wait() { flpr_emu::unsupported("wgmma.wait_group"); }
template <int TA, int TB>
static inline void wgmma_m64n64k16(float (&)[32], uint64_t, uint64_t, uint32_t) { flpr_emu::unsupported("wgmma"); }
template <int TA, int TB>
static inline void wgmma_m64n32k16(float (&)[16], uint64_t, uint64_t, uint32_t) { flpr_emu::unsupported("wgmma"); }
// system-scope flag accesses: the spin loops of the peer-memory protocol are cooperative here
static inline void st_release_sys(uint32_t* p, uint32_t v) {
  flpr_emu::maybe_yield();
  *reinterpret_cast<volatile uint32_t*>(p) = v;
}
static inline uint32_t ld_acquire_sys(const uint32_t* p) {
  flpr_emu::yield();
  return *reinterpret_cast<const volatile uint32_t*>(p);
}
static inline float4 ld_stream_f4(const float4* p) {
  flpr_emu::maybe_yield();
  return *p;
}
static inline void st_stream_f4(float4* p, const float4& v) {
  flpr_emu::maybe_yield();
  *p = v;
}
static inline unsigned long long gtimer() {
  flpr_emu::g_clock_ns += 50;
  return flpr_emu::g_clock_ns;
}
// NVSwitch multicast window: ld_reduce adds the word of every member, st writes it to every member
static inline float4 multimem_ld_reduce_add_f4(const float* mc) {
  flpr_emu::maybe_yield();
  const flpr_emu::Multicast* m = flpr_emu::find_mc(mc);
  const size_t off = reinterpret_cast<const char*>(mc) - m->base;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (char* b : m->members) {
    const float4 v = *reinterpret_cast<const float4*>(b + off);
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  return s;
}
static inline void multimem_st_f4(float* mc, const float4& v) {
  flpr_emu::maybe_yield();
  const flpr_emu::Multicast* m = flpr_emu::find_mc(mc);
  const size_t off = reinterpret_cast<const char*>(mc) - m->base;
  for (char* b : m->members) *reinterpret_cast<float4*>(b + off) = v;
}
}  // namespace flpr
using flpr::bind_device_of;

#define cudaGetLastError() (cudaSuccess)
#define cudaFuncSetAttribute(...) (cudaSuccess)

extern "C" {
int flpr_emu_deadlocks() { return flpr_emu::g_deadlocks; }
void flpr_emu_defer(int on) { flpr_emu::g_defer = on != 0; }
// Execute everything queued since flpr_emu_defer(1). seed 0: round-robin, no stalls; otherwise a seeded random schedule.
// Returns 0, or 1 when `max_passes` scheduler passes did not finish the work (deadlock).
int flpr_emu_run(unsigned seed, long max_passes, unsigned stall_one_in) {
  return flpr_emu::run_queues(seed, max_passes, stall_one_in ? stall_one_in : 4);
}
void flpr_emu_set_start_delay(const void* stream_key, int passes) { flpr_emu::g_start_delay[stream_key] = passes; }
// Threads of the kernels on this stream only run in one of `one_in` scheduler passes (seeded runs): a slow rank.
void flpr_emu_set_lane_slowdown(const void* stream_key, unsigned one_in) { flpr_emu::g_lane_slow[stream_key] = one_in; }
int flpr_emu_mc_register(void* mc_base, size_t bytes, int world, void* const* members) {
  flpr_emu::Multicast m;
  m.base = reinterpret_cast<char*>(mc_base);
  m.bytes = bytes;
  for (int r = 0; r < world; ++r) m.members.push_back(reinterpret_cast<char*>(members[r]));
  flpr_emu::g_mc.push_back(m);
  return (int)flpr_emu::g_mc.size() - 1;
}
void flpr_emu_mc_clear() { flpr_emu::g_mc.clear(); }
unsigned long long flpr_emu_clock_ns() { return flpr_emu::g_clock_ns; }
}
