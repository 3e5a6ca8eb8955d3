// simt.h -- TEST ONLY: a SIMT runtime on the host, so that a .cuh holding __global__ kernels compiles under g++ unchanged
// and runs as a grid.  Never linked into the product.
//
//   * Every thread of a block is a fiber with a stack of its own.  The blocks of a grid run on SIMT_WORKERS OS threads
//     at once, so blocks really overlap in time (the page kernel's word cache is shared by all blocks of a grid).
//     __shared__ becomes `static thread_local`: a worker runs one block at a time, so every block has its own shared
//     memory.
//   * A fiber runs until it reaches a sync point: a warp intrinsic, __syncthreads / __syncthreads_or, or its end.  Which
//     runnable fiber of the block goes next is drawn from the launch's seed (or taken in thread order when the seed is 0),
//     so code that relies on lanes running in lockstep between sync points sees its lanes in a different order.
//   * __syncwarp, __shfl_sync, __shfl_up_sync, __shfl_down_sync, __shfl_xor_sync, __ballot_sync, __any_sync, __all_sync
//     and __reduce_add_sync complete once every lane named in the mask has arrived; then the values are exchanged as the
//     PTX ISA defines (shfl: a source lane outside [0, width) of the lane's segment returns the lane's own value).
//     __syncthreads completes once every thread of the block that has not exited has arrived.
//   * Checks.  The launch stops and reports the kernel, block, warp, lanes and intrinsic when
//       - lanes named in one mask arrive at different intrinsics or with different masks,
//       - a lane executes an intrinsic whose mask does not name it, or names a lane that has exited or that waits at
//         __syncthreads, or a shuffle reads a lane outside the mask,
//       - the block can make no progress (a __syncthreads that only some threads reach, a mask that is never completed), or
//         passes MAX_SWITCHES sync points (a loop that never exits).
//   * Atomics are the __atomic builtins (seq_cst), __threadfence is a seq_cst fence, __ldg a plain load, the bit
//     intrinsics are compiler builtins.
//
// What it cannot find.  The host's memory model (x86: total store order) is stronger than the GPU's, so a missing fence
// or a missing acquire that the GPU's weaker ordering would expose does not show here.  Fibers switch only at sync
// points, so two lanes never interleave inside one statement: a race between lanes of a block that needs the exact
// timing of the hardware (not just another order of whole sync-free stretches) is not reproduced.  Timing, occupancy,
// register and shared-memory limits and out-of-bounds accesses that stay inside host memory are not checked.
//
// Include order: <cuda_runtime.h> first (vector types, the attribute macros), then this file, then the kernels.
#pragma once
#include <stdint.h>
#include <string.h>
#include <sys/mman.h>
#include <algorithm>
#include <atomic>
#include <deque>
#include <functional>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <vector>
#include <cuda_runtime.h>

// ------------------------------------------------------------------------------------------------ keywords
#undef __shared__
#define __shared__ static thread_local
#define __launch_bounds__(...)
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))
#endif

namespace simt {

constexpr int SIMT_WORKERS = 4;
constexpr size_t STACK_BYTES = 128 << 10;
constexpr uint64_t MAX_SWITCHES = 1ull << 28;   // per block: more and the block counts as stuck (a merge loop that never ends)

enum Op { OP_NONE = 0, OP_SYNCWARP, OP_SHFL, OP_SHFL_UP, OP_SHFL_DOWN, OP_SHFL_XOR, OP_BALLOT, OP_ANY, OP_ALL, OP_REDUCE_ADD,
          OP_BAR, OP_BAR_OR };
inline const char* op_name(int op) {
  static const char* n[] = {"-", "__syncwarp", "__shfl_sync", "__shfl_up_sync", "__shfl_down_sync", "__shfl_xor_sync", "__ballot_sync",
                            "__any_sync", "__all_sync", "__reduce_add_sync", "__syncthreads", "__syncthreads_or"};
  return n[op];
}
enum State { RUNNABLE = 0, WAIT_WARP, WAIT_BAR, DONE };

struct Fiber {
  void* sp = nullptr;
  void* stack = nullptr;
  uint3 tid{0, 0, 0};
  int state = RUNNABLE;
  int op = OP_NONE, arg = 0, width = 32;
  unsigned mask = 0;
  uint64_t val = 0, result = 0;
};

struct Worker;
struct Grid {
  const char* name;
  dim3 grid, block;
  std::function<void()> body;
  uint64_t seed;
  std::atomic<uint64_t> next{0};
  std::atomic<bool> failed{false};
  std::mutex mu;
  std::string error;
  void fail(const std::string& m) {
    std::lock_guard<std::mutex> g(mu);
    if (!failed.load()) { error = m; failed = true; }
  }
};

struct Worker {
  Grid* g = nullptr;
  std::vector<Fiber> f;
  void* sched_sp = nullptr;
  Fiber* cur = nullptr;
  uint3 bid{0, 0, 0};
  std::mt19937_64 rng;
  std::deque<int> runnable;
  int live = 0, at_bar = 0, bar_kind = OP_NONE;
  uint64_t bar_any = 0;
  bool abort_block = false;
};

inline thread_local Worker* tw = nullptr;

// ------------------------------------------------------------------------------------------------ context switch
// x86-64: callee-saved registers, MXCSR and the x87 control word (glibc's swapcontext costs a system call per switch, and
// a page of the page kernel switches a few hundred thousand times)
#if defined(__x86_64__)
extern "C" void simt_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.globl simt_switch
.type simt_switch,@function
simt_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  subq $8, %rsp
  stmxcsr (%rsp)
  fnstcw 4(%rsp)
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  ldmxcsr (%rsp)
  fldcw 4(%rsp)
  addq $8, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size simt_switch,.-simt_switch
)");
#else
#error "tests/native/simt.h: the fiber switch is written for x86-64"
#endif

[[noreturn]] inline void fiber_entry() {
  Worker* w = tw;
  w->g->body();
  w = tw;
  w->cur->state = DONE;
  simt_switch(&w->cur->sp, w->sched_sp);
  __builtin_unreachable();
}

inline void fiber_init(Fiber& fb) {
  if (!fb.stack) {
    void* m = mmap(nullptr, STACK_BYTES + 4096, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (m == MAP_FAILED) abort();
    mprotect(m, 4096, PROT_NONE);   // guard page below the stack
    fb.stack = m;
  }
  uintptr_t top = ((uintptr_t)fb.stack + 4096 + STACK_BYTES) & ~(uintptr_t)15;
  uint64_t* a = reinterpret_cast<uint64_t*>(top - 16);   // the "return address" simt_switch pops: 16-byte aligned slot
  a[0] = (uint64_t)(uintptr_t)&fiber_entry;
  for (int k = 1; k <= 6; ++k) a[-k] = 0;                  // rbp rbx r12..r15
  uint32_t* csr = reinterpret_cast<uint32_t*>(a - 7);
  csr[0] = 0x1F80u; csr[1] = 0x037Fu;                      // default MXCSR / x87 control word
  fb.sp = a - 7;
}

// ------------------------------------------------------------------------------------------------ diagnostics
inline std::string lanes_str(unsigned m) {
  std::string s;
  for (int l = 0; l < 32; ++l)
    if ((m >> l) & 1u) { if (!s.empty()) s += ","; s += std::to_string(l); }
  return "{" + s + "}";
}
inline std::string where(const Worker& w, int warp) {
  char b[200];
  snprintf(b, sizeof(b), "kernel %s, block (%u,%u,%u), warp %d", w.g->name, w.bid.x, w.bid.y, w.bid.z, warp);
  return b;
}
inline void block_fail(Worker& w, const std::string& m) {
  w.g->fail(m);
  w.abort_block = true;
}

// ------------------------------------------------------------------------------------------------ collectives
inline int n_threads(const Worker& w) { return (int)w.f.size(); }

// The fiber at index i just arrived at a warp intrinsic: complete the collective if every named lane is there.
inline void try_warp(Worker& w, int i) {
  Fiber& me = w.f[i];
  const int warp = i / 32, base = warp * 32, lane = i % 32;
  const int nt = n_threads(w);
  if (!((me.mask >> lane) & 1u)) {
    char mb[64];
    snprintf(mb, sizeof(mb), " with mask 0x%08x", me.mask);
    block_fail(w, where(w, warp) + ": lane " + std::to_string(lane) + " executes " + op_name(me.op) + mb + ", which does not name it");
    return;
  }
  unsigned waiting_other = 0;
  for (int l = 0; l < 32; ++l) {
    if (!((me.mask >> l) & 1u)) continue;
    if (base + l >= nt) {
      block_fail(w, where(w, warp) + ": " + op_name(me.op) + " names lane " + std::to_string(l) + ", which the block does not have");
      return;
    }
    const Fiber& o = w.f[base + l];
    if (o.state == DONE) {
      block_fail(w, where(w, warp) + ": lane " + std::to_string(lane) + " at " + op_name(me.op) + " names lane " + std::to_string(l) +
                        ", which has exited");
      return;
    }
    if (o.state == WAIT_BAR) {
      block_fail(w, where(w, warp) + ": lane " + std::to_string(lane) + " at " + op_name(me.op) + " names lane " + std::to_string(l) +
                        ", which waits at " + op_name(o.op) + " (divergent warp)");
      return;
    }
    if (o.state == RUNNABLE) return;   // not there yet
    if (o.op != me.op || o.mask != me.mask) waiting_other |= 1u << l;
  }
  if (waiting_other) {
    unsigned same = 0;
    for (int l = 0; l < 32; ++l)
      if (((me.mask >> l) & 1u) && !((waiting_other >> l) & 1u)) same |= 1u << l;
    const Fiber& o = w.f[base + __builtin_ctz(waiting_other)];
    char mb[64];
    snprintf(mb, sizeof(mb), " (mask 0x%08x) and lanes ", me.mask);
    char ob[64];
    snprintf(ob, sizeof(ob), " (mask 0x%08x)", o.mask);
    block_fail(w, where(w, warp) + ": divergent warp sync: lanes " + lanes_str(same) + " at " + op_name(me.op) + mb + lanes_str(waiting_other) +
                      " at " + op_name(o.op) + ob);
    return;
  }
  // every named lane is here: exchange
  const unsigned m = me.mask;
  uint64_t ballot = 0, sum = 0;
  for (int l = 0; l < 32; ++l)
    if ((m >> l) & 1u) {
      const Fiber& o = w.f[base + l];
      if (o.val) ballot |= 1ull << l;
      sum += (uint32_t)o.val;
    }
  for (int l = 0; l < 32; ++l) {
    if (!((m >> l) & 1u)) continue;
    Fiber& o = w.f[base + l];
    const int wd = o.width, seg = l & ~(wd - 1);
    int src = -1;
    switch (o.op) {
      case OP_SHFL: src = seg + (o.arg & (wd - 1)); break;
      case OP_SHFL_UP: src = (l - seg) - o.arg >= 0 ? l - o.arg : l; break;
      case OP_SHFL_DOWN: src = (l - seg) + o.arg < wd ? l + o.arg : l; break;
      case OP_SHFL_XOR: src = ((l - seg) ^ o.arg) < wd ? seg + ((l - seg) ^ o.arg) : l; break;
      default: break;
    }
    if (src >= 0) {
      if (!((m >> src) & 1u)) {
        block_fail(w, where(w, warp) + ": lane " + std::to_string(l) + " at " + op_name(o.op) + " reads lane " + std::to_string(src) +
                          ", which the mask does not name");
        return;
      }
      o.result = w.f[base + src].val;
    } else if (o.op == OP_BALLOT) o.result = ballot;
    else if (o.op == OP_ANY) o.result = ballot != 0;
    else if (o.op == OP_ALL) o.result = ballot == (uint64_t)m;
    else if (o.op == OP_REDUCE_ADD) o.result = (uint32_t)sum;
    else o.result = 0;
  }
  for (int l = 0; l < 32; ++l)
    if ((m >> l) & 1u) { w.f[base + l].state = RUNNABLE; w.f[base + l].op = OP_NONE; w.runnable.push_back(base + l); }
}

// a fiber arrived at __syncthreads or exited: the other lanes of its warp must not wait for it at a warp intrinsic;
// complete the barrier if every live thread is there
inline void try_bar(Worker& w, int i) {
  const Fiber& me = w.f[i];
  const int warp = i / 32, base = warp * 32, lane = i % 32, nt = n_threads(w);
  for (int l = 0; l < 32 && base + l < nt; ++l) {
    const Fiber& o = w.f[base + l];
    if (o.state == WAIT_WARP && ((o.mask >> lane) & 1u)) {
      block_fail(w, where(w, warp) + ": lane " + std::to_string(l) + " waits at " + op_name(o.op) + " for lane " + std::to_string(lane) +
                        (me.state == DONE ? std::string(", which has exited") : std::string(", which is at ") + op_name(me.op)) + " (divergent warp)");
      return;
    }
  }
  if (me.state == DONE) --w.live;
  else {
    if (w.at_bar && me.op != w.bar_kind) {
      block_fail(w, where(w, warp) + ": threads meet at __syncthreads and __syncthreads_or at once");
      return;
    }
    w.bar_kind = me.op;
    ++w.at_bar;
    if (me.val) w.bar_any = 1;
  }
  if (!w.at_bar || w.at_bar != w.live) return;
  for (int k = 0; k < nt; ++k)
    if (w.f[k].state == WAIT_BAR) { w.f[k].state = RUNNABLE; w.f[k].result = w.bar_any; w.f[k].op = OP_NONE; w.runnable.push_back(k); }
  w.at_bar = 0; w.bar_any = 0;
}

inline std::string stuck_report(const Worker& w) {
  std::string s = std::string("kernel ") + w.g->name + ", block (" + std::to_string(w.bid.x) + "," + std::to_string(w.bid.y) + "," +
                  std::to_string(w.bid.z) + "): no progress;";
  const int nt = (int)w.f.size();
  for (int warp = 0; warp * 32 < nt; ++warp) {
    unsigned bar = 0, done = 0;
    std::string ops;
    for (int l = 0; l < 32 && warp * 32 + l < nt; ++l) {
      const Fiber& o = w.f[warp * 32 + l];
      if (o.state == DONE) done |= 1u << l;
      else if (o.state == WAIT_BAR) bar |= 1u << l;
      else if (o.state == WAIT_WARP) {
        char b[96];
        snprintf(b, sizeof(b), " lane %d at %s (mask 0x%08x);", l, op_name(o.op), o.mask);
        ops += b;
      }
    }
    if (bar == (done ^ (nt - warp * 32 >= 32 ? 0xFFFFFFFFu : ((1u << (nt - warp * 32)) - 1u))) && ops.empty()) continue;
    s += " warp " + std::to_string(warp) + ":";
    if (bar) s += " lanes " + lanes_str(bar) + " at __syncthreads;";
    if (done) s += " lanes " + lanes_str(done) + " exited;";
    s += ops;
  }
  return s;
}

// ------------------------------------------------------------------------------------------------ block / grid
inline void run_block(Worker& w, uint64_t b) {
  Grid& g = *w.g;
  const unsigned gx = g.grid.x, gy = g.grid.y;
  w.bid = make_uint3((unsigned)(b % gx), (unsigned)((b / gx) % gy), (unsigned)(b / ((uint64_t)gx * gy)));
  const int nt = (int)(g.block.x * g.block.y * g.block.z);
  if ((int)w.f.size() != nt) w.f.resize(nt);
  w.runnable.clear();
  for (int k = 0; k < nt; ++k) {
    Fiber& fb = w.f[k];
    fiber_init(fb);
    fb.tid = make_uint3(k % g.block.x, (k / g.block.x) % g.block.y, k / (g.block.x * g.block.y));
    fb.state = RUNNABLE; fb.op = OP_NONE; fb.mask = 0; fb.val = fb.result = 0;
    w.runnable.push_back(k);
  }
  w.rng.seed(g.seed * 0x9E3779B97F4A7C15ull + b);
  w.abort_block = false;
  w.live = nt; w.at_bar = 0; w.bar_any = 0; w.bar_kind = OP_NONE;
  int done = 0;
  uint64_t switches = 0;
  while (!w.abort_block) {
    if (++switches > MAX_SWITCHES) {
      block_fail(w, std::string("kernel ") + w.g->name + ", block (" + std::to_string(w.bid.x) + "," + std::to_string(w.bid.y) + "," +
                        std::to_string(w.bid.z) + "): no end after " + std::to_string(MAX_SWITCHES) + " sync points (a loop that never exits?)");
      break;
    }
    if (w.runnable.empty()) {
      if (done < nt) block_fail(w, stuck_report(w));
      break;
    }
    if (g.seed) std::swap(w.runnable.front(), w.runnable[(size_t)(w.rng() % w.runnable.size())]);
    const int i = w.runnable.front();   // (seed 0: first come, first served -- thread order to begin with)
    w.runnable.pop_front();
    w.cur = &w.f[i];
    simt_switch(&w.sched_sp, w.f[i].sp);
    w.cur = nullptr;
    const Fiber& fb = w.f[i];
    if (fb.state == WAIT_WARP) try_warp(w, i);
    else if (fb.state == WAIT_BAR) try_bar(w, i);
    else if (fb.state == DONE) {
      ++done;
      try_bar(w, i);
    }
    if (g.failed.load()) break;
  }
}

inline void worker_main(Grid* g) {
  Worker w;
  w.g = g;
  tw = &w;
  const uint64_t nb = (uint64_t)g->grid.x * g->grid.y * g->grid.z;
  while (!g->failed.load()) {
    const uint64_t b = g->next.fetch_add(1);
    if (b >= nb) break;
    run_block(w, b);
  }
  for (Fiber& fb : w.f) if (fb.stack) munmap(fb.stack, STACK_BYTES + 4096);
  tw = nullptr;
}

// Runs body() as every thread of grid x block; "" or the first check that failed.  seed 0: lanes in thread order.
inline std::string launch(const char* name, dim3 grid, dim3 block, uint64_t seed, std::function<void()> body) {
  Grid g;
  g.name = name; g.grid = grid; g.block = block; g.body = std::move(body); g.seed = seed;
  const uint64_t nb = (uint64_t)grid.x * grid.y * grid.z;
  if (!nb) return "";
  const int nw = (int)std::min<uint64_t>(SIMT_WORKERS, nb);
  std::vector<std::thread> th;
  for (int k = 0; k < nw; ++k) th.emplace_back(worker_main, &g);
  for (auto& t : th) t.join();
  return g.failed.load() ? g.error : std::string();
}

// ------------------------------------------------------------------------------------------------ from a fiber
inline uint64_t warp_op(int op, unsigned mask, uint64_t v, int arg = 0, int width = 32) {
  Worker* w = tw;
  Fiber* f = w->cur;
  f->op = op; f->mask = mask; f->val = v; f->arg = arg; f->width = width; f->state = WAIT_WARP;
  simt_switch(&f->sp, w->sched_sp);
  return f->result;
}
inline uint64_t bar_op(int op, uint64_t v) {
  Worker* w = tw;
  Fiber* f = w->cur;
  f->op = op; f->val = v; f->state = WAIT_BAR;
  simt_switch(&f->sp, w->sched_sp);
  return f->result;
}

template <class T> inline uint64_t to_u64(T v) { static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes"); uint64_t r = 0; memcpy(&r, &v, sizeof(T)); return r; }
template <class T> inline T from_u64(uint64_t r) { T v; memcpy(&v, &r, sizeof(T)); return v; }

}  // namespace simt

// ------------------------------------------------------------------------------------------------ built-in variables
#define threadIdx (::simt::tw->cur->tid)
#define blockIdx (::simt::tw->bid)
#define blockDim (::simt::tw->g->block)
#define gridDim (::simt::tw->g->grid)

// ------------------------------------------------------------------------------------------------ intrinsics
inline void __syncthreads() { simt::bar_op(simt::OP_BAR, 0); }
inline int __syncthreads_or(int p) { return (int)simt::bar_op(simt::OP_BAR_OR, p != 0); }
inline void __syncwarp(unsigned mask = 0xFFFFFFFFu) { simt::warp_op(simt::OP_SYNCWARP, mask, 0); }
template <class T> inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
  return simt::from_u64<T>(simt::warp_op(simt::OP_SHFL, mask, simt::to_u64(v), src, width));
}
template <class T> inline T __shfl_up_sync(unsigned mask, T v, unsigned d, int width = 32) {
  return simt::from_u64<T>(simt::warp_op(simt::OP_SHFL_UP, mask, simt::to_u64(v), (int)d, width));
}
template <class T> inline T __shfl_down_sync(unsigned mask, T v, unsigned d, int width = 32) {
  return simt::from_u64<T>(simt::warp_op(simt::OP_SHFL_DOWN, mask, simt::to_u64(v), (int)d, width));
}
template <class T> inline T __shfl_xor_sync(unsigned mask, T v, int lm, int width = 32) {
  return simt::from_u64<T>(simt::warp_op(simt::OP_SHFL_XOR, mask, simt::to_u64(v), lm, width));
}
inline unsigned __ballot_sync(unsigned mask, int p) { return (unsigned)simt::warp_op(simt::OP_BALLOT, mask, p != 0); }
inline int __any_sync(unsigned mask, int p) { return (int)simt::warp_op(simt::OP_ANY, mask, p != 0); }
inline int __all_sync(unsigned mask, int p) { return (int)simt::warp_op(simt::OP_ALL, mask, p != 0); }
inline unsigned __reduce_add_sync(unsigned mask, unsigned v) { return (unsigned)simt::warp_op(simt::OP_REDUCE_ADD, mask, v); }

template <class T> inline T __ldg(const T* p) { return *p; }
inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }

inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicOr(unsigned* p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicMax(unsigned* p, unsigned v) {
  unsigned o = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (o < v && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return o;
}
inline unsigned atomicExch(unsigned* p, unsigned v) { return __atomic_exchange_n(p, v, __ATOMIC_SEQ_CST); }
inline unsigned long long atomicExch(unsigned long long* p, unsigned long long v) { return __atomic_exchange_n(p, v, __ATOMIC_SEQ_CST); }
inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
  __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return cmp;
}

inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }

inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
inline int __ffs(int x) { return __builtin_ffs(x); }
inline int __ffsll(long long x) { return __builtin_ffsll(x); }
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { return (unsigned)((((uint64_t)hi << 32) | lo) >> (s & 31u)); }
inline unsigned __funnelshift_rc(unsigned lo, unsigned hi, unsigned s) { return (unsigned)((((uint64_t)hi << 32) | lo) >> (s > 32u ? 32u : s)); }
inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned s) { return (unsigned)(((((uint64_t)hi << 32) | lo) << (s & 31u)) >> 32); }
inline unsigned __byte_perm(unsigned x, unsigned y, unsigned s) {
  const uint64_t v = ((uint64_t)y << 32) | x;
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) r |= (unsigned)((v >> (8 * ((s >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
  return r;
}
