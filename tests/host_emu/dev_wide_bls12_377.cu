// Device harness (TEST ONLY) for BLS12-377: the op wrappers of wide_ops.cuh over Bls377Fr / Bls377Fq, its
// Fq2 = Fq[u]/(u^2 + 5) and G1 / G2, compiled for sm_90a (inline-PTX carries).  One kernel launch per call, one thread per
// case; the entry points take emu_wide_bls12_377.cpp's arguments and return 0 or the CUDA error code.
#include <cuda_runtime.h>

#include "wide_ops.cuh"
using namespace zkb;
using namespace zkb::wide;

static constexpr int BLOCK = 128;

template <class P>
static __global__ void __launch_bounds__(BLOCK) k_fp(int op, size_t count, const uint32_t* a, const uint32_t* b,
                                                     const uint32_t* c, const uint32_t* d, uint32_t* o) {
  const size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (i < count) fp_case<P>(op, i, a, b, c, d, o);
}
static __global__ void __launch_bounds__(BLOCK) k_fp2(int op, size_t count, const uint32_t* a, const uint32_t* b,
                                                      const uint32_t* c, const uint32_t* d, uint32_t* o) {
  const size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (i >= count) return;
  if (op == 3) st2<Bls377Fq>(Fp2<Bls377Fq>::inv(ld2<Bls377Fq>(a + 24 * i)), o + 24 * i);   // inv: the norm c0^2 + 5 c1^2
  else fp2_case<Bls377Fq>(op, i, a, b, c, d, o);
}
template <class F, int K>
static __global__ void __launch_bounds__(BLOCK) k_ec(int op, size_t count, const uint32_t* a, const uint32_t* b, uint32_t* o) {
  const size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (i < count) ec_case<F, K, Bls377Fq>(op, i, a, b, o);
}

// Device copies of the operand buffers; the result travels back into `out`.
struct Batch {
  uint32_t* d[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  size_t bytes[5] = {0, 0, 0, 0, 0};
  cudaError_t err = cudaSuccess;
  Batch(const uint32_t* const* host, const size_t* words, int k) {
    for (int j = 0; j < k && err == cudaSuccess; j++) {
      bytes[j] = words[j] * sizeof(uint32_t);
      err = cudaMalloc(&d[j], bytes[j] ? bytes[j] : 4);
      if (err == cudaSuccess && host[j] && bytes[j]) err = cudaMemcpy(d[j], host[j], bytes[j], cudaMemcpyHostToDevice);
    }
  }
  int finish(int j_out, uint32_t* out) {
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    if (err == cudaSuccess && bytes[j_out]) err = cudaMemcpy(out, d[j_out], bytes[j_out], cudaMemcpyDeviceToHost);
    for (auto p : d) if (p) cudaFree(p);
    return (int)err;
  }
};

static unsigned blocks(size_t count) { return (unsigned)((count + BLOCK - 1) / BLOCK); }

// field 0: Fr (8 limbs), 1: Fq (12 limbs)
extern "C" int dev_wide_fp(int field, int op, size_t count, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                           const uint32_t* d, uint32_t* o) {
  const size_t n = field == 0 ? 8 : 12;
  const uint32_t* host[5] = {a, b, c, d, nullptr};
  const size_t words[5] = {2 * n * count, n * count, n * count, n * count, 2 * n * count};
  Batch bt(host, words, 5);
  if (bt.err == cudaSuccess && count) {
    uint32_t* const* p = bt.d;
    if (field == 0) k_fp<Bls377Fr><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2], p[3], p[4]);
    else k_fp<Bls377Fq><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2], p[3], p[4]);
  }
  return bt.finish(4, o);
}
extern "C" int dev_wide_fp2(int, int op, size_t count, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                            const uint32_t* d, uint32_t* o) {
  const size_t s = 2 * 12 * count;
  const uint32_t* host[5] = {a, b, c, d, nullptr};
  const size_t words[5] = {s, s, s, s, s};
  Batch bt(host, words, 5);
  if (bt.err == cudaSuccess && count) {
    uint32_t* const* p = bt.d;
    k_fp2<<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2], p[3], p[4]);
  }
  return bt.finish(4, o);
}
// group 1: G1, 2: G2
extern "C" int dev_wide_ec(int, int group, int op, size_t count, const uint32_t* a, const uint32_t* b, uint32_t* o) {
  const size_t s = 4 * (size_t)group * 12 * count;
  const uint32_t* host[3] = {a, b, nullptr};
  const size_t words[3] = {s, s, s};
  Batch bt(host, words, 3);
  if (bt.err == cudaSuccess && count) {
    uint32_t* const* p = bt.d;
    if (group == 1) k_ec<Fp<Bls377Fq>, 1><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2]);
    else k_ec<Fp2<Bls377Fq>, 2><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2]);
  }
  return bt.finish(2, o);
}
