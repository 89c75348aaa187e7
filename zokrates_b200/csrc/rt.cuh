// Thin runtime layer: device memory, copies and kernel launches.
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
#include "hd.cuh"
#include "zkb.h"  // status codes (include/zkb.h)

#if !defined(ZKB_EMU)
#include <cuda_runtime.h>
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

// Block-cooperative kernels: `nphases` steps separated by __syncthreads(); threads of a block exchange data
// through (L1-coherent) global scratch.  fn(block, thread, phase).  The host emulation runs phase by phase.
template <class Tag, int BLOCK, class Fn>
__global__ void __launch_bounds__(BLOCK) zkb_phased_kernel(uint32_t nphases, Fn fn) {
  for (uint32_t ph = 0; ph < nphases; ph++) {
    fn((uint32_t)blockIdx.x, (uint32_t)threadIdx.x, ph);
    __syncthreads();
  }
}
template <class Tag, int BLOCK, class Fn>
inline void launch_phased(Stream st, size_t nblocks, uint32_t nphases, Fn fn) {
  if (nblocks == 0) return;
  launch_counter()++;
  if (nblocks > 0x7fffffffull) throw Error(ZKB_E_ARG, "grid too large");
  zkb_phased_kernel<Tag, BLOCK, Fn><<<(unsigned)nblocks, BLOCK, 0, st.s>>>(nphases, fn);
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
// page-locked host memory (asynchronous device -> host copies land here while the next proof's kernels run)
inline void* host_alloc_pinned(size_t bytes) {
  void* p = nullptr;
  ZKB_CUDA(cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocDefault));
  return p;
}
inline void host_free_pinned(void* p) { if (p) cudaFreeHost(p); }

#else  // ------------------------------------------------------------------ host emulation (tests)

struct Stream {
  int s = 0;
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
  EmuPerm(size_t n_, uint64_t salt) : n(n_), mode(emu_order().mode) {
    if (mode != EMU_ORDER_SEEDED) return;
    uint32_t k = 0;
    while (k < 63 && ((size_t)1 << k) < n) k++;
    mask = ((size_t)1 << k) - 1;
    shift = (k + 1) / 2;
    uint64_t h = emu_mix(emu_order().seed ^ emu_mix(salt + 0x9e3779b97f4a7c15ull));
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
template <class Tag, int BLOCK = 128, int MINB = 1, class Fn>
inline void launch(Stream, size_t n, Fn fn) {
  if (!n) return;
  uint64_t id = ++launch_counter();
  EmuPerm perm(n, id);
  for (size_t i = 0; i < n; i++) fn(perm(i));
}
// Phases stay in sequence (each stands for a __syncthreads()); blocks, and threads within a phase, are permuted.
template <class Tag, int BLOCK, class Fn>
inline void launch_phased(Stream, size_t nblocks, uint32_t nphases, Fn fn) {
  if (!nblocks) return;
  uint64_t id = ++launch_counter();
  EmuPerm bperm(nblocks, id);
  for (size_t i = 0; i < nblocks; i++) {
    uint32_t b = (uint32_t)bperm(i);
    for (uint32_t ph = 0; ph < nphases; ph++) {
      EmuPerm tperm(BLOCK, emu_mix(id) ^ ((uint64_t)b << 20) ^ ph);
      for (uint32_t t = 0; t < (uint32_t)BLOCK; t++) fn(b, (uint32_t)tperm(t), ph);
    }
  }
}
template <class Tag, int BLOCK, int SMEM_BYTES, class Fn>
inline void launch_block(Stream, size_t nblocks, uint32_t nphases, Fn fn) {
  if (!nblocks) return;
  uint64_t id = ++launch_counter();
  void* smem = malloc(SMEM_BYTES);
  if (!smem) throw Error(ZKB_E_OOM, "malloc");
  EmuPerm bperm(nblocks, id);
  for (size_t i = 0; i < nblocks; i++) {
    uint32_t b = (uint32_t)bperm(i);
    for (uint32_t ph = 0; ph < nphases; ph++) {
      EmuPerm tperm(BLOCK, emu_mix(id) ^ ((uint64_t)b << 20) ^ ph);
      for (uint32_t t = 0; t < (uint32_t)BLOCK; t++) fn(b, (uint32_t)tperm(t), ph, smem);
    }
  }
  free(smem);
}
inline void* dev_alloc(size_t bytes) {
  void* p = malloc(bytes ? bytes : 16);
  if (!p) throw Error(ZKB_E_OOM, "malloc");
  return p;
}
inline void dev_free(void* p) { free(p); }
inline void h2d(Stream, void* dst, const void* src, size_t bytes) { memcpy(dst, src, bytes); }
inline void d2h(Stream, void* dst, const void* src, size_t bytes) { memcpy(dst, src, bytes); }
inline void d2d(Stream, void* dst, const void* src, size_t bytes) { memmove(dst, src, bytes); }
inline void dev_zero(Stream, void* p, size_t bytes) { memset(p, 0, bytes); }
inline void dev_fill_ff(Stream, void* p, size_t bytes) { memset(p, 0xff, bytes); }
inline void stream_sync(Stream) {}
inline Stream stream_create_high_priority() { return Stream(); }
inline Stream stream_create() { return Stream(); }
inline void stream_destroy(Stream) {}
struct Event {
  void record(Stream) {}
  void wait(Stream) {}
  void sync() {}
  void destroy() {}
};
inline void* host_alloc_pinned(size_t bytes) {
  void* p = malloc(bytes ? bytes : 16);
  if (!p) throw Error(ZKB_E_OOM, "malloc");
  return p;
}
inline void host_free_pinned(void* p) { free(p); }

#endif

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
