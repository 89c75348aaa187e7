// Thin runtime layer: devices, device memory, streams, copies, kernel launches and stage timers.
//
// Product build (nvcc, sm_90a): every `launch<Tag>(n, fn)` is a real kernel on the engine's CUDA
// stream; failures surface as zkb::Error (never a silent CPU path).
// Test build (-DZKB_EMU, plain g++): the same orchestration code runs the kernel bodies in a host
// loop so tests/host_emu can check indexing logic without a GPU.  libzkb200.so is never built with
// ZKB_EMU.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>
#include "hd.cuh"
#include "zkb.h"  // status codes (include/zkb.h)

#if !defined(ZKB_EMU)
#include <atomic>
#include <cuda_runtime.h>
#else
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#endif

namespace zkb {

struct Error : public std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};


#if !defined(ZKB_EMU)

#define ZKB_CUDA(expr)                                                                                   \
  do {                                                                                                    \
    cudaError_t _e = (expr);                                                                              \
    if (_e != cudaSuccess)                                                                                \
      throw ::zkb::Error(_e == cudaErrorMemoryAllocation ? ZKB_E_OOM : ZKB_E_CUDA,          \
                         std::string(#expr) + ": " + cudaGetErrorString(_e));                             \
  } while (0)

struct Stream {
  cudaStream_t s = nullptr;
};

template <class Tag, int BLOCK, int MINB, class Fn>
__global__ void __launch_bounds__(BLOCK, MINB) zkb_kernel(size_t n, Fn fn) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid < n) fn(tid);
}

#define ZKB_LAMBDA [=] __device__

inline uint64_t& launch_counter() {
  static uint64_t c = 0;
  return c;
}

template <class Tag, int BLOCK = 128, int MINB = 1, class Fn>
inline void launch(Stream st, size_t n, Fn fn) {
  if (n == 0) return;
  launch_counter()++;
  size_t blocks = (n + BLOCK - 1) / BLOCK;
  if (blocks > 0x7fffffffull) throw Error(ZKB_E_ARG, "grid too large");
  zkb_kernel<Tag, BLOCK, MINB, Fn><<<(unsigned)blocks, BLOCK, 0, st.s>>>(n, fn);
  ZKB_CUDA(cudaGetLastError());
}

// Block kernels with static shared memory: `nphases` steps separated by __syncthreads(); fn(block, thread, phase, smem).
// Registers do not live across phases (the body is re-entered per phase); the host emulation gives every block a
// heap buffer and runs phase by phase.
template <class Tag, int BLOCK, int SMEM_BYTES, class Fn>
__global__ void __launch_bounds__(BLOCK) zkb_block_kernel(uint32_t nphases, Fn fn) {
  __shared__ __align__(16) uint8_t smem[SMEM_BYTES];
  for (uint32_t ph = 0; ph < nphases; ph++) {
    fn((uint32_t)blockIdx.x, (uint32_t)threadIdx.x, ph, (void*)smem);
    __syncthreads();
  }
}
template <class Tag, int BLOCK, int SMEM_BYTES, class Fn>
inline void launch_block(Stream st, size_t nblocks, uint32_t nphases, Fn fn) {
  if (nblocks == 0) return;
  launch_counter()++;
  if (nblocks > 0x7fffffffull) throw Error(ZKB_E_ARG, "grid too large");
  zkb_block_kernel<Tag, BLOCK, SMEM_BYTES, Fn><<<(unsigned)nblocks, BLOCK, 0, st.s>>>(nphases, fn);
  ZKB_CUDA(cudaGetLastError());
}

inline void* dev_alloc(size_t bytes) {
  void* p = nullptr;
  if (bytes == 0) bytes = 16;
  ZKB_CUDA(cudaMalloc(&p, bytes));
  return p;
}
inline void dev_free(void* p) {
  if (p) cudaFree(p);
}
inline void h2d(Stream st, void* dst, const void* src, size_t bytes) {
  if (bytes) ZKB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st.s));
}
inline void d2h(Stream st, void* dst, const void* src, size_t bytes) {
  if (bytes) ZKB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st.s));
}
inline void d2d(Stream st, void* dst, const void* src, size_t bytes) {
  if (bytes) ZKB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st.s));
}
inline void dev_zero(Stream st, void* p, size_t bytes) {
  if (bytes) ZKB_CUDA(cudaMemsetAsync(p, 0, bytes, st.s));
}
inline void dev_fill_ff(Stream st, void* p, size_t bytes) {
  if (bytes) ZKB_CUDA(cudaMemsetAsync(p, 0xff, bytes, st.s));
}
inline void stream_sync(Stream st) { ZKB_CUDA(cudaStreamSynchronize(st.s)); }
// side streams (high priority: their small latency-bound kernels are scheduled ahead of the pending blocks of
// a big kernel on the main stream) and cross-stream ordering
inline Stream stream_create_high_priority() {
  int lo = 0, hi = 0;
  ZKB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  Stream s;
  ZKB_CUDA(cudaStreamCreateWithPriority(&s.s, cudaStreamNonBlocking, hi));
  return s;
}
inline Stream stream_create() {
  Stream s;
  ZKB_CUDA(cudaStreamCreateWithFlags(&s.s, cudaStreamNonBlocking));
  return s;
}
inline void stream_destroy(Stream s) { if (s.s) cudaStreamDestroy(s.s); }
struct Event {
  cudaEvent_t e = nullptr;
  void ensure() { if (!e) ZKB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); }
  void record(Stream s) { ensure(); ZKB_CUDA(cudaEventRecord(e, s.s)); }
  void wait(Stream s) { if (e) ZKB_CUDA(cudaStreamWaitEvent(s.s, e, 0)); }
  void sync() { if (e) ZKB_CUDA(cudaEventSynchronize(e)); }     // host waits
  void destroy() { if (e) { cudaEventDestroy(e); e = nullptr; } }
};
// stage timer: named spans between CUDA events on a stream (no-op in the host emulation)
struct StageTimer {
  struct Ev { const char* name; cudaEvent_t a, b; };
  std::vector<Ev> evs;
  std::vector<size_t> open;  // stack of stages begun but not ended (stages may nest)
  Stream st;
  explicit StageTimer(Stream s) : st(s) {}
  void begin(const char* name) {
    Ev e{name, nullptr, nullptr};
    ZKB_CUDA(cudaEventCreate(&e.a));
    ZKB_CUDA(cudaEventCreate(&e.b));
    ZKB_CUDA(cudaEventRecord(e.a, st.s));
    open.push_back(evs.size());
    evs.push_back(e);
  }
  void end() {
    size_t i = open.back();
    open.pop_back();
    ZKB_CUDA(cudaEventRecord(evs[i].b, st.s));
  }
  // spans on other streams (tails): begin_on returns a handle for end_on
  size_t begin_on(Stream s, const char* name) {
    Ev e{name, nullptr, nullptr};
    ZKB_CUDA(cudaEventCreate(&e.a));
    ZKB_CUDA(cudaEventCreate(&e.b));
    ZKB_CUDA(cudaEventRecord(e.a, s.s));
    evs.push_back(e);
    return evs.size() - 1;
  }
  void end_on(Stream s, size_t i) { ZKB_CUDA(cudaEventRecord(evs[i].b, s.s)); }
  void collect(std::vector<std::pair<const char*, double>>& out) {
    out.clear();
    for (auto& e : evs) {
      ZKB_CUDA(cudaEventSynchronize(e.b));
      float ms = 0;
      ZKB_CUDA(cudaEventElapsedTime(&ms, e.a, e.b));
      out.push_back({e.name, (double)ms});
      cudaEventDestroy(e.a);
      cudaEventDestroy(e.b);
    }
    evs.clear();
  }
  ~StageTimer() { for (auto& e : evs) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); } }
};
// page-locked host memory (asynchronous device -> host copies land here while the next proof's kernels run)
inline void* host_alloc_pinned(size_t bytes) {
  void* p = nullptr;
  ZKB_CUDA(cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocDefault));
  return p;
}
inline void host_free_pinned(void* p) { if (p) cudaFreeHost(p); }

// ---- devices -------------------------------------------------------------------------------------------------------------
inline size_t dev_mem_free() {
  size_t free_b = 0, total_b = 0;
  ZKB_CUDA(cudaMemGetInfo(&free_b, &total_b));
  return free_b;
}
// multiprocessor count of the current device, queried once per device
inline int device_sm_count() {
  static std::atomic<int> cached[64];
  int dev = 0, n = 0;
  ZKB_CUDA(cudaGetDevice(&dev));
  if (dev < 64) n = cached[dev].load(std::memory_order_relaxed);
  if (!n) {
    ZKB_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    if (dev < 64) cached[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}
// visible devices, or -1 with *why set to the reason (the failed query is not left as the thread's last error)
inline int device_count(const char** why) {
  int n = 0;
  const cudaError_t e = cudaGetDeviceCount(&n);
  if (e == cudaSuccess) return n;
  cudaGetLastError();
  *why = cudaGetErrorString(e);
  return -1;
}
inline void device_select(int dev) { ZKB_CUDA(cudaSetDevice(dev)); }
// a failed launch configuration sticks as the thread's last error; clear it before the next call checks its own launches
inline void clear_device_error() { cudaGetLastError(); }
// before a context's engine is destroyed: wait for the context's main stream on its device; never throws (zkb_ctx_destroy)
inline void device_drain(int dev, Stream st) {
  cudaSetDevice(dev);
  if (st.s) cudaStreamSynchronize(st.s);
}
// a caller's stream passed through the C ABI as void* (cudaStream_t)
inline Stream stream_from_handle(void* h) {
  Stream s;
  s.s = (cudaStream_t)h;
  return s;
}

#else  // ------------------------------------------------------------------ host emulation (tests)

struct Stream {
  int s = 0;   // emulated stream id (stream_create); 0 is a stream like any other
};
#define ZKB_LAMBDA [=]
inline uint64_t& launch_counter() {
  static uint64_t c = 0;
  return c;
}
// The order in which the emulation runs a launch's threads, and a block kernel's blocks and the threads of each
// phase.  The device promises no order, so a kernel whose result depends on it is wrong even when ascending order
// (the default) hides the race.  The other orders make such a race reproducible on a CPU: descending, or a
// bijection of [0, n) keyed by the seed and the launch number.  Set through zkb_emu_launch_order (api.cu).
enum { EMU_ORDER_ASCENDING = 0, EMU_ORDER_DESCENDING = 1, EMU_ORDER_SEEDED = 2 };
struct EmuOrder {
  uint32_t mode = EMU_ORDER_ASCENDING;
  uint64_t seed = 0;
};
inline EmuOrder& emu_order() {
  static EmuOrder o;
  return o;
}
inline uint64_t emu_mix(uint64_t x) {  // splitmix64 finaliser
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
// Visiting order of one loop of n steps: perm(i) is the index run at step i.  The seeded order is a bijection of
// [0, 2^k) (2^k >= n) made of odd multiplies, additions and xor-shifts mod 2^k, cycle-walked down to [0, n).
struct EmuPerm {
  size_t n, mask = 0;
  uint32_t mode, shift = 0;
  uint64_t key[3] = {0, 0, 0};
  // `o`: the order in force when the launch was enqueued (a deferred launch runs later, possibly under another order)
  EmuPerm(size_t n_, uint64_t salt, const EmuOrder& o = emu_order()) : n(n_), mode(o.mode) {
    if (mode != EMU_ORDER_SEEDED) return;
    uint32_t k = 0;
    while (k < 63 && ((size_t)1 << k) < n) k++;
    mask = ((size_t)1 << k) - 1;
    shift = (k + 1) / 2;
    uint64_t h = emu_mix(o.seed ^ emu_mix(salt + 0x9e3779b97f4a7c15ull));
    for (auto& v : key) v = h = emu_mix(h + 0x9e3779b97f4a7c15ull);
  }
  size_t step(size_t x) const {
    for (uint64_t v : key) {
      x = (size_t)(x * (v | 1) + (v >> 32)) & mask;
      if (shift) x ^= x >> shift;
    }
    return x;
  }
  size_t operator()(size_t i) const {
    if (mode == EMU_ORDER_ASCENDING) return i;
    if (mode == EMU_ORDER_DESCENDING) return n - 1 - i;
    size_t x = step(i);
    while (x >= n) x = step(x);
    return x;
  }
};
// ---- emulated streams ---------------------------------------------------------------------------------------------------
// The device runs a stream's work in order and the streams of a context concurrently, ordered only by events; the host reads
// a result once a sync says it is there.  Under the default policy (EAGER) every operation runs when it is issued, so a
// missing Event::wait or sync can never show.  The other policies queue every launch, copy, fill and event per stream
// (process-wide: all contexts share one device) and run an operation only when the host needs its result:
//   LAZY    nothing runs until a sync, a copy to pageable memory, a free or a drain; then only the dependency closure of that
//           point runs (earlier operations of the same stream and, through each event wait, the recording stream up to the
//           record), the newest ready queue head first.  A reader whose writer nobody waited for runs before it; a writer
//           that overtakes a reader still queued on another stream runs first.
//   SEEDED  after every enqueue and in every drain, a seeded random number of ready queue heads runs, picked at random across
//           streams; a drain finishes its closure in a random interleaving.
// The calls follow the CUDA semantics the engine relies on: Event::wait binds to the event's last record at call time (a
// never-recorded event is a no-op); h2d reads a pageable source at call time (CUDA stages it) and a pinned one
// (host_alloc_pinned) when it runs; d2h to pageable memory returns after the copy, d2h to pinned memory is deferred;
// dev_free and host_free_pinned drain everything (cudaFree / cudaFreeHost synchronise); dev_alloc is no barrier and, under
// EMU_STREAM_POISON, returns memory filled with a nonzero pattern (cudaMalloc memory is not zero; a large malloc is).
// Set through zkb_emu_stream_order (api.cu).
enum { EMU_STREAMS_EAGER = 0, EMU_STREAMS_LAZY = 1, EMU_STREAMS_SEEDED = 2 };
enum { EMU_STREAM_POISON = 1u };
struct EmuOp {
  uint64_t seq;                 // enqueue number (process-wide)
  std::function<void()> fn;     // empty: an event record or an event wait
  int dep_stream = -1;          // an event wait: runs once stream dep_stream has run everything up to dep_seq
  uint64_t dep_seq = 0;
};
struct EmuStreams {
  std::recursive_mutex mu;
  uint32_t mode = EMU_STREAMS_EAGER, flags = 0;
  uint64_t rng = 0, seq = 0;
  uint64_t max_run = 0;                   // highest enqueue number run so far
  uint64_t reordered = 0, queued = 0, peak = 0;
  int next_id = 1;
  std::map<int, std::deque<EmuOp>> q;
  std::set<int> dead;                     // destroyed streams whose queue still holds work
  std::map<uintptr_t, size_t> pinned;     // host_alloc_pinned ranges: base -> bytes
};
inline EmuStreams& emu_streams() {
  static EmuStreams e;
  return e;
}
inline bool emu_eager() { return emu_streams().mode == EMU_STREAMS_EAGER; }
inline uint64_t emu_rand(EmuStreams& E) { return emu_mix(E.rng += 0x9e3779b97f4a7c15ull); }
// stream `sid` has run everything up to enqueue number `seq`
inline bool emu_done(EmuStreams& E, int sid, uint64_t seq) {
  auto it = E.q.find(sid);
  return it == E.q.end() || it->second.empty() || it->second.front().seq > seq;
}
inline bool emu_ready(EmuStreams& E, const EmuOp& op) { return op.dep_stream < 0 || emu_done(E, op.dep_stream, op.dep_seq); }
inline void emu_run_head(EmuStreams& E, int sid) {
  auto it = E.q.find(sid);
  EmuOp op = std::move(it->second.front());
  it->second.pop_front();
  if (it->second.empty() && E.dead.count(sid)) { E.q.erase(it); E.dead.erase(sid); }
  E.queued--;
  if (op.seq < E.max_run) E.reordered++;
  else E.max_run = op.seq;
  if (op.fn) op.fn();
}
// one of the ready heads among `cand`: the newest (LAZY: the order furthest from the issue order), or a random one (SEEDED)
inline int emu_pick(EmuStreams& E, const std::vector<int>& cand) {
  if (E.mode == EMU_STREAMS_SEEDED) return cand[emu_rand(E) % cand.size()];
  int best = cand[0];
  for (int s : cand) if (E.q[s].front().seq > E.q[best].front().seq) best = s;
  return best;
}
inline void emu_run_random(EmuStreams& E, uint64_t count) {
  for (uint64_t k = 0; k < count; k++) {
    std::vector<int> cand;
    for (auto& kv : E.q) if (!kv.second.empty() && emu_ready(E, kv.second.front())) cand.push_back(kv.first);
    if (cand.empty()) return;
    emu_run_head(E, emu_pick(E, cand));
  }
}
// run the dependency closure of (stream sid, enqueue number seq)
inline void emu_drain(int sid, uint64_t seq) {
  EmuStreams& E = emu_streams();
  std::lock_guard<std::recursive_mutex> lock(E.mu);
  // need[s]: stream s must run everything up to need[s]; grown through every wait in range until nothing changes
  std::map<int, uint64_t> need{{sid, seq}};
  for (bool grew = true; grew;) {
    grew = false;
    for (auto kv : std::map<int, uint64_t>(need)) {
      auto q = E.q.find(kv.first);
      if (q == E.q.end()) continue;
      for (const EmuOp& op : q->second) {
        if (op.seq > kv.second) break;
        if (op.dep_stream < 0) continue;
        auto it = need.find(op.dep_stream);
        if (it == need.end() || it->second < op.dep_seq) { need[op.dep_stream] = op.dep_seq; grew = true; }
      }
    }
  }
  while (!emu_done(E, sid, seq)) {
    std::vector<int> cand;
    for (auto& kv : need)
      if (!emu_done(E, kv.first, kv.second) && emu_ready(E, E.q[kv.first].front())) cand.push_back(kv.first);
    if (cand.empty()) throw Error(ZKB_E_INTERNAL, "emulated streams: a wait that can never be satisfied");
    emu_run_head(E, emu_pick(E, cand));
  }
}
inline void emu_drain_all() {
  EmuStreams& E = emu_streams();
  std::lock_guard<std::recursive_mutex> lock(E.mu);
  while (E.queued) {
    std::vector<int> cand;
    for (auto& kv : E.q) if (!kv.second.empty() && emu_ready(E, kv.second.front())) cand.push_back(kv.first);
    if (cand.empty()) throw Error(ZKB_E_INTERNAL, "emulated streams: a wait that can never be satisfied");
    emu_run_head(E, emu_pick(E, cand));
  }
}
// queue one operation on stream sid (EAGER: run it now); returns its enqueue number (0 when it ran)
inline uint64_t emu_push(int sid, std::function<void()> fn, int dep_stream = -1, uint64_t dep_seq = 0) {
  EmuStreams& E = emu_streams();
  std::lock_guard<std::recursive_mutex> lock(E.mu);
  EmuOp op;
  op.seq = ++E.seq;
  op.fn = std::move(fn);
  op.dep_stream = dep_stream;
  op.dep_seq = dep_seq;
  const uint64_t s = op.seq;
  E.q[sid].push_back(std::move(op));
  if (++E.queued > E.peak) E.peak = E.queued;
  if (E.mode == EMU_STREAMS_SEEDED) emu_run_random(E, emu_rand(E) % 4);
  return s;
}
template <class Fn>
inline uint64_t emu_enqueue(Stream st, Fn fn) {
  if (emu_eager()) { fn(); return 0; }
  return emu_push(st.s, std::function<void()>(std::move(fn)));
}
inline bool emu_is_pinned(const void* p, size_t bytes) {
  EmuStreams& E = emu_streams();
  std::lock_guard<std::recursive_mutex> lock(E.mu);
  auto it = E.pinned.upper_bound((uintptr_t)p);
  if (it == E.pinned.begin()) return false;
  --it;
  return (uintptr_t)p + bytes <= it->first + it->second;
}
// the stream policy (EMU_STREAMS_*), its seed and EMU_STREAM_POISON; drains what the previous policy left queued
inline void emu_set_streams(uint32_t mode, uint64_t seed, uint32_t flags) {
  emu_drain_all();
  EmuStreams& E = emu_streams();
  std::lock_guard<std::recursive_mutex> lock(E.mu);
  E.mode = mode;
  E.flags = flags;
  E.rng = emu_mix(seed ^ 0x5eedull);
  E.reordered = 0;
  E.peak = 0;
}

template <class Tag, int BLOCK = 128, int MINB = 1, class Fn>
inline void launch(Stream st, size_t n, Fn fn) {
  if (!n) return;
  const uint64_t id = ++launch_counter();
  const EmuOrder o = emu_order();   // the launch order in force at enqueue time
  emu_enqueue(st, [=] {
    EmuPerm perm(n, id, o);
    for (size_t i = 0; i < n; i++) fn(perm(i));
  });
}
// Phases stay in sequence (each stands for a __syncthreads()); blocks, and threads within a phase, are permuted.
template <class Tag, int BLOCK, int SMEM_BYTES, class Fn>
inline void launch_block(Stream st, size_t nblocks, uint32_t nphases, Fn fn) {
  if (!nblocks) return;
  const uint64_t id = ++launch_counter();
  const EmuOrder o = emu_order();
  emu_enqueue(st, [=] {
    void* smem = malloc(SMEM_BYTES);
    if (!smem) throw Error(ZKB_E_OOM, "malloc");
    EmuPerm bperm(nblocks, id, o);
    for (size_t i = 0; i < nblocks; i++) {
      uint32_t b = (uint32_t)bperm(i);
      for (uint32_t ph = 0; ph < nphases; ph++) {
        EmuPerm tperm(BLOCK, emu_mix(id) ^ ((uint64_t)b << 20) ^ ph, o);
        for (uint32_t t = 0; t < (uint32_t)BLOCK; t++) fn(b, (uint32_t)tperm(t), ph, smem);
      }
    }
    free(smem);
  });
}
inline void* dev_alloc(size_t bytes) {
  if (bytes == 0) bytes = 16;
  void* p = malloc(bytes);
  if (!p) throw Error(ZKB_E_OOM, "malloc");
  if (emu_streams().flags & EMU_STREAM_POISON) memset(p, 0x5a, bytes);
  return p;
}
inline void dev_free(void* p) {
  if (!p) return;
  if (!emu_eager()) emu_drain_all();
  free(p);
}
inline void h2d(Stream st, void* dst, const void* src, size_t bytes) {
  if (!bytes) return;
  if (emu_eager()) { memcpy(dst, src, bytes); return; }
  if (emu_is_pinned(src, bytes)) { emu_push(st.s, [=] { memcpy(dst, src, bytes); }); return; }
  std::shared_ptr<std::vector<uint8_t>> staged(new std::vector<uint8_t>((const uint8_t*)src, (const uint8_t*)src + bytes));
  emu_push(st.s, [=] { memcpy(dst, staged->data(), bytes); });
}
inline void d2h(Stream st, void* dst, const void* src, size_t bytes) {
  if (!bytes) return;
  if (emu_eager()) { memcpy(dst, src, bytes); return; }
  const uint64_t seq = emu_push(st.s, [=] { memcpy(dst, src, bytes); });
  if (!emu_is_pinned(dst, bytes)) emu_drain(st.s, seq);
}
inline void d2d(Stream st, void* dst, const void* src, size_t bytes) {
  if (bytes) emu_enqueue(st, [=] { memmove(dst, src, bytes); });
}
inline void dev_zero(Stream st, void* p, size_t bytes) {
  if (bytes) emu_enqueue(st, [=] { memset(p, 0, bytes); });
}
inline void dev_fill_ff(Stream st, void* p, size_t bytes) {
  if (bytes) emu_enqueue(st, [=] { memset(p, 0xff, bytes); });
}
inline void stream_sync(Stream st) {
  if (!emu_eager()) emu_drain(st.s, emu_streams().seq);
}
inline Stream stream_create() {
  EmuStreams& E = emu_streams();
  std::lock_guard<std::recursive_mutex> lock(E.mu);
  Stream s;
  s.s = E.next_id++;
  return s;
}
inline Stream stream_create_high_priority() { return stream_create(); }
// work still queued on a destroyed stream runs later, as on the device
inline void stream_destroy(Stream s) {
  EmuStreams& E = emu_streams();
  std::lock_guard<std::recursive_mutex> lock(E.mu);
  auto it = E.q.find(s.s);
  if (it == E.q.end()) return;
  if (it->second.empty()) E.q.erase(it);
  else E.dead.insert(s.s);
}
struct Event {
  int sid = -1;        // the stream and enqueue number of the last record
  uint64_t seq = 0;
  void record(Stream s) {
    if (emu_eager()) return;
    sid = s.s;
    seq = emu_push(s.s, std::function<void()>());
  }
  void wait(Stream s) {
    if (!emu_eager() && sid >= 0) emu_push(s.s, std::function<void()>(), sid, seq);
  }
  void sync() {
    if (!emu_eager() && sid >= 0) emu_drain(sid, seq);
  }
  void destroy() { sid = -1; }
};
struct StageTimer {
  explicit StageTimer(Stream) {}
  void begin(const char*) {}
  void end() {}
  size_t begin_on(Stream, const char*) { return 0; }
  void end_on(Stream, size_t) {}
  void collect(std::vector<std::pair<const char*, double>>& out) { out.clear(); }
};
inline void* host_alloc_pinned(size_t bytes) {
  if (bytes == 0) bytes = 16;
  void* p = malloc(bytes);
  if (!p) throw Error(ZKB_E_OOM, "malloc");
  if (emu_streams().flags & EMU_STREAM_POISON) memset(p, 0x5a, bytes);
  EmuStreams& E = emu_streams();
  std::lock_guard<std::recursive_mutex> lock(E.mu);
  E.pinned[(uintptr_t)p] = bytes;
  return p;
}
inline void host_free_pinned(void* p) {
  if (!p) return;
  if (!emu_eager()) emu_drain_all();
  {
    EmuStreams& E = emu_streams();
    std::lock_guard<std::recursive_mutex> lock(E.mu);
    E.pinned.erase((uintptr_t)p);
  }
  free(p);
}

// ---- one emulated device ------------------------------------------------------------------------------------------------
// Half the address space, so every memory clamp runs and none binds: a pass size derived from it is far above any batch,
// and adding the device bytes a caller already holds cannot overflow.  Pass sizes come from the other limits alone.
inline size_t dev_mem_free() { return ~(size_t)0 >> 1; }
inline int device_sm_count() { return 1; }   // read only by device-only launches (the tile2 NTT)
inline int device_count(const char**) { return 1; }
inline void device_select(int) {}
inline void clear_device_error() {}
// runs the work queued on every stream, not only the context's, as the engine's first dev_free would
inline void device_drain(int, Stream) { emu_drain_all(); }
inline Stream stream_from_handle(void* h) {   // an emulated stream id (zkb_emu_stream_create)
  Stream s;
  s.s = (int)(intptr_t)h;
  return s;
}

#endif

// free device memory every pass-size and window-table budget leaves unused
static constexpr size_t DEV_MEM_RESERVE = (size_t)1 << 30;

// RAII device buffer
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t count = 0;
  DevBuf() {}
  explicit DevBuf(size_t n) { alloc(n); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), count(o.count) { o.p = nullptr; o.count = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; count = o.count; o.p = nullptr; o.count = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  void alloc(size_t n) {
    release();
    p = (T*)dev_alloc(n * sizeof(T));
    count = n;
  }
  void ensure(size_t n) {
    if (n > count) alloc(n);
  }
  void release() {
    dev_free(p);
    p = nullptr;
    count = 0;
  }
  size_t bytes() const { return count * sizeof(T); }
};

// RAII pinned host buffer
struct HostBuf {
  uint8_t* p = nullptr;
  size_t count = 0;
  HostBuf() {}
  HostBuf(const HostBuf&) = delete;
  HostBuf& operator=(const HostBuf&) = delete;
  ~HostBuf() { host_free_pinned(p); }
  void ensure(size_t n) {
    if (n <= count) return;
    host_free_pinned(p);
    p = nullptr; count = 0;
    p = (uint8_t*)host_alloc_pinned(n);
    count = n;
  }
};

}  // namespace zkb
