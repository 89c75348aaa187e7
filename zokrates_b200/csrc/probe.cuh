// Integer-pipe peak probes: the denominators of the modular-multiplication roofline (SURVEY.md §8d
// asks for a measured IMAD peak, not the datasheet estimate).
#pragma once
#include "fp.cuh"
#include "rt.cuh"

namespace zkb {

#if !defined(ZKB_EMU)
// kind 0: 8 independent 32x32+64 multiply-add chains per thread, no memory traffic
static __global__ void zkb_probe_imad(uint32_t iters, uint32_t seed, uint64_t* sink) {
  uint32_t a = seed + threadIdx.x, b = seed * 2654435761u + blockIdx.x;
  uint64_t acc[8];
#pragma unroll
  for (int k = 0; k < 8; k++) acc[k] = a + k;
  for (uint32_t i = 0; i < iters; i++) {
#pragma unroll
    for (int k = 0; k < 8; k++)
      asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[k]) : "r"(a), "r"(b));
    a += (uint32_t)acc[0];
  }
  uint64_t s = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) s ^= acc[k];
  if (s == 0x1234567) sink[0] = s;
}
// kind 2: the same count of wide multiply-adds, but CARRY-CHAINED as a multi-limb multiplier needs them: rows of 8
// (mad.lo.cc/madc.hi.cc, 6 x madc.lo.cc/madc.hi.cc, madc.lo.cc/madc.hi) = IMAD.WIDE.U32 followed by 7 IMAD.WIDE.U32.X with
// predicate carries, 4 independent rows per thread.  The .X form costs more multiply-pipe cycles than the carry-free
// one: this is the multiply-add rate a carry-propagating multiplication can reach.
static __global__ void zkb_probe_imad_carry(uint32_t iters, uint32_t seed, uint64_t* sink) {
  uint32_t a = seed + threadIdx.x, b = seed * 2654435761u + blockIdx.x;
  uint32_t lo[4][8], hi[4][8];
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int k = 0; k < 8; k++) { lo[r][k] = a + k; hi[r][k] = b + r; }
  for (uint32_t i = 0; i < iters; i++) {
#pragma unroll
    for (int r = 0; r < 4; r++) {
      ptx::mad_wide_cc(lo[r][0], hi[r][0], a, b, lo[r][0], hi[r][0]);
#pragma unroll
      for (int k = 1; k < 7; k++) ptx::madc_wide_cc(lo[r][k], hi[r][k], a, b, lo[r][k], hi[r][k]);
      ptx::madc_wide(lo[r][7], hi[r][7], a, b, lo[r][7], hi[r][7]);
    }
    a += lo[0][0];
  }
  uint64_t s = 0;
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= ((uint64_t)hi[r][k] << 32) | lo[r][k];
  if (s == 0x1234567) sink[0] = s;
}
// kind 1: register-resident Montgomery multiplications, 2 independent chains per thread
template <class F>
static __global__ void zkb_probe_modmul(uint32_t iters, uint32_t seed, F* sink) {
  F x = F::one(), y = F::r2();
  x.v[0] += threadIdx.x + seed;
  y.v[1] += blockIdx.x;
  F u = y, w = x;
  for (uint32_t i = 0; i < iters; i++) {
    x = F::mul(x, y);
    u = F::mul(u, w);
  }
  F r = F::add(x, u);
  if (r.v[0] == 0x1234567 && r.v[1] == 0x89abcdef) sink[0] = r;
}
#endif

inline double peak_probe(Stream st, int kind, uint32_t iters) {
#if !defined(ZKB_EMU)
  typedef Fp<Bn254Fq> F;
  const int block = 256, blocks = device_sm_count() * 8;
  DevBuf<uint64_t> sink(16);
  cudaEvent_t a, b;
  ZKB_CUDA(cudaEventCreate(&a));
  ZKB_CUDA(cudaEventCreate(&b));
  for (int rep = 0; rep < 2; rep++) {  // first repetition is the warm-up
    ZKB_CUDA(cudaEventRecord(a, st.s));
    if (kind == 0) zkb_probe_imad<<<blocks, block, 0, st.s>>>(iters, 12345u, sink.p);
    else if (kind == 2) zkb_probe_imad_carry<<<blocks, block, 0, st.s>>>(iters, 12345u, sink.p);
    else zkb_probe_modmul<F><<<blocks, block, 0, st.s>>>(iters, 12345u, (F*)sink.p);
    ZKB_CUDA(cudaGetLastError());
    ZKB_CUDA(cudaEventRecord(b, st.s));
    ZKB_CUDA(cudaEventSynchronize(b));
  }
  float ms = 0;
  ZKB_CUDA(cudaEventElapsedTime(&ms, a, b));
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  double per_thread = kind == 0 ? 8.0 * iters : kind == 2 ? 32.0 * iters : 2.0 * iters;
  return per_thread * block * blocks / (ms * 1e-3);
#else
  (void)st; (void)kind; (void)iters;
  throw Error(ZKB_E_CUDA, "peak probe needs a GPU");
#endif
}

}  // namespace zkb
