// Device harness (TEST ONLY) for the separated Montgomery arithmetic of fp.cuh / fp2.cuh and the point additions of
// ec.cuh: the op wrappers of wide_ops.cuh (shared with the g++ harness emu_wide.cpp) compiled for sm_90a, where every
// carry primitive is the inline PTX of hd.cuh.  Each entry point copies a batch of cases to the device, runs ONE kernel
// launch for the (field, op) with one thread per case, and copies the results back; the entry points take the same
// arguments as emu_wide.cpp's.  Returns 0, or the CUDA error code.
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
template <class P>
static __global__ void __launch_bounds__(BLOCK) k_fp2(int op, size_t count, const uint32_t* a, const uint32_t* b,
                                                      const uint32_t* c, const uint32_t* d, uint32_t* o) {
  const size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (i < count) fp2_case<P>(op, i, a, b, c, d, o);
}
template <class F, int K, class P>
static __global__ void __launch_bounds__(BLOCK) k_ec(int op, size_t count, const uint32_t* a, const uint32_t* b, uint32_t* o) {
  const size_t i = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (i < count) ec_case<F, K, P>(op, i, a, b, o);
}

// Device copies of the operand buffers; results travel back into `out`.
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

// field 0: BN254 Fr, 1: BN254 Fq, 2: BLS12-381 Fr, 3: BLS12-381 Fq
extern "C" int dev_wide_fp(int field, int op, size_t count, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                           const uint32_t* d, uint32_t* o) {
  const size_t n = field == 3 ? 12 : 8;
  const uint32_t* host[5] = {a, b, c, d, nullptr};
  const size_t words[5] = {2 * n * count, n * count, n * count, n * count, 2 * n * count};
  Batch bt(host, words, 5);
  if (bt.err == cudaSuccess && count) {
    uint32_t* const* p = bt.d;
    switch (field) {
      case 0: k_fp<Bn254Fr><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2], p[3], p[4]); break;
      case 1: k_fp<Bn254Fq><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2], p[3], p[4]); break;
      case 2: k_fp<Bls381Fr><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2], p[3], p[4]); break;
      case 3: k_fp<Bls381Fq><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2], p[3], p[4]); break;
    }
  }
  return bt.finish(4, o);
}
// curve 0: BN254 Fq2, 1: BLS12-381 Fq2
extern "C" int dev_wide_fp2(int curve, int op, size_t count, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                            const uint32_t* d, uint32_t* o) {
  const size_t s = 2 * (curve == 0 ? 8 : 12) * count;
  const uint32_t* host[5] = {a, b, c, d, nullptr};
  const size_t words[5] = {s, s, s, s, s};
  Batch bt(host, words, 5);
  if (bt.err == cudaSuccess && count) {
    uint32_t* const* p = bt.d;
    if (curve == 0) k_fp2<Bn254Fq><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2], p[3], p[4]);
    else k_fp2<Bls381Fq><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2], p[3], p[4]);
  }
  return bt.finish(4, o);
}
// curve 0: BN254, 1: BLS12-381; group 1: G1, 2: G2
extern "C" int dev_wide_ec(int curve, int group, int op, size_t count, const uint32_t* a, const uint32_t* b, uint32_t* o) {
  const size_t s = 4 * (size_t)group * (curve == 0 ? 8 : 12) * count;
  const uint32_t* host[3] = {a, b, nullptr};
  const size_t words[3] = {s, s, s};
  Batch bt(host, words, 3);
  if (bt.err == cudaSuccess && count) {
    uint32_t* const* p = bt.d;
    if (curve == 0) {
      if (group == 1) k_ec<Fp<Bn254Fq>, 1, Bn254Fq><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2]);
      else k_ec<Fp2<Bn254Fq>, 2, Bn254Fq><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2]);
    } else {
      if (group == 1) k_ec<Fp<Bls381Fq>, 1, Bls381Fq><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2]);
      else k_ec<Fp2<Bls381Fq>, 2, Bls381Fq><<<blocks(count), BLOCK>>>(op, count, p[0], p[1], p[2]);
    }
  }
  return bt.finish(2, o);
}
