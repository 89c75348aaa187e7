// Shared-memory NTT tile pass, second generation (device build only; the host emulation keeps ntt_block_body).
//
// Same transform as ntt.cuh::ntt_block_body — S <= 10 consecutive radix-2 stages of a size-n transform on a tile of 1024
// elements held in shared memory, bit-identical results — with three changes against the first tile pass (which stalled on
// per-butterfly twiddle gathers out of a 16 MB table, shared-memory bank conflicts and a synchronous tile load):
//
//   * FOUR-STEP twiddles.  The stages of a pass act on index bits [lo_bit, lo_bit + S).  Their twiddles factor as
//       w_n^(((j << lo_bit) | low) << sh) = W_1024^(j << (9 - lg_h)) * w_n^(low << sh):
//     the first factor depends on the position inside the tile only (512 roots of unity W_1024^k, kept in shared memory), and
//     the second factors accumulate, over the S stages of the pass, to ONE per-element factor w_{n'}^(low * k1), n' = 2^(lo_bit+S),
//     k1 = bitrev_S(local position) — applied after the last stage of a DIF pass / before the first stage of a DIT pass
//     (Cooley-Tukey: a size-n1*n2 DFT is n2 column DFTs, a twiddle multiplication, n1 row DFTs).  One gathered load and one
//     extra multiplication per element and pass replace S/2 gathered loads per element.  Exact field arithmetic: same bits.
//   * ASYNCHRONOUS tile load: global -> shared with cp.async (LDGSTS), no register staging.
//   * CONFLICT-FREE shared memory: an element is split into two 16-byte halves stored in two planes (a quarter-warp of
//     LDS.128 then covers all 32 banks), slots XOR-swizzled inside rows of 8 (strided register steps hit distinct banks).
//   The last compute phase writes its registers straight to global memory (no store phase).
#pragma once
#include "ntt.cuh"
#include "rt.cuh"

#if !defined(ZKB_EMU)
namespace zkb {

static constexpr uint32_t NTT2_PLANE = NTT_TILE;                     // slots per plane (swizzled inside rows of 8, no padding)
static constexpr uint32_t NTT2_SMEM = (2 * NTT2_PLANE + 2 * 512) * 16;  // data planes + twiddle planes: 49 152 bytes

// A quarter-warp of LDS.128 / STS.128 is conflict-free when its 8 slots differ modulo 8 (8 x 16 B = all 32 banks).  The register
// steps address 8 slots whose indices differ in three bits: {0,1,2} (half-span >= 8), {0,1,4}, {0,1,5}, {0,3,4}, {0,4,5},
// {2,3,4} or {3,4,5} depending on the step.  XOR-ing the low three bits with a GF(2)-linear image of bits 3, 4, 5
// (010, 101, 110) makes every one of these triples independent, so every step is conflict-free; the map is a bijection
// inside each row of 8 slots.
__device__ __forceinline__ uint32_t ntt2_slot(uint32_t pos) {
  const uint32_t x = ((pos >> 3) & 1u) * 2u ^ ((pos >> 4) & 1u) * 5u ^ ((pos >> 5) & 1u) * 6u;
  return pos ^ x;
}
// The twiddle index of a butterfly is imod << sh: 8 lanes read entries whose indices differ in bits {sh, sh+1, sh+2}.  Images
// 011, 110, 111, 101, 001, 010 for bits 3..8 keep any three consecutive bits independent.
__device__ __forceinline__ uint32_t ntt2_wslot(uint32_t wi) {
  const uint32_t x = ((wi >> 3) & 1u) * 3u ^ ((wi >> 4) & 1u) * 6u ^ ((wi >> 5) & 1u) * 7u ^ ((wi >> 6) & 1u) * 5u ^ ((wi >> 7) & 1u) * 1u ^
                     ((wi >> 8) & 1u) * 2u;
  return wi ^ x;
}

template <class Fr>
__device__ __forceinline__ Fr ntt2_ld(const uint4* lo, const uint4* hi, uint32_t slot) {
  static_assert(sizeof(Fr) == 32, "two 16-byte halves");
  Fr r;
  uint4 a = lo[slot], b = hi[slot];
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
template <class Fr>
__device__ __forceinline__ void ntt2_st(uint4* lo, uint4* hi, uint32_t slot, const Fr& r) {
  lo[slot] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
  hi[slot] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}
template <class Fr>
__device__ __forceinline__ Fr ntt2_ldg(const Fr* p) {   // two 128-bit read-only loads
  const uint4 a = __ldg((const uint4*)p), b = __ldg((const uint4*)p + 1);
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
__device__ __forceinline__ void ntt2_cp_async16(void* smem_dst, const void* gmem_src) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void ntt2_cp_async_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// the per-element factor of the four-step split: w_{n'}^(low * k1) = tw[(low * k1) << (log_n - lo_bit - S)], tw holding w_n^k for
// k < n/2 (the upper half of the circle is the negated lower half)
template <class Fr>
__device__ __forceinline__ Fr ntt2_factor(const Fr* tw, const NttPass& ps, uint32_t low, uint32_t j_local) {
  const uint32_t k1 = __brev(j_local) >> (32 - ps.S);
  const uint32_t e = (low * k1) << (ps.log_n - ps.lo_bit - ps.S);     // < n
  const uint32_t half = 1u << (ps.log_n - 1);
  Fr f = ntt2_ldg<Fr>(tw + (e & (half - 1)));
  return (e & half) ? Fr::neg(f) : f;
}

// One compute phase: K stages on 8 (4, 2) register-resident elements, exactly the butterflies of ntt_block_stages with the
// twiddles taken from the shared 1024th roots.  FIRST / LAST select the fused factor multiplication and the direct store.
template <class Fr, bool DIT, int K>
__device__ __forceinline__ void ntt2_stages(Fr* __restrict__ x, const Fr* __restrict__ tw, const Fr* __restrict__ scale, const NttPass& ps, uint4* dlo, uint4* dhi, const uint4* wlo,
                                            const uint4* whi, uint32_t tile, uint32_t done, bool first, bool last) {
  constexpr uint32_t R = 1u << K;
  const uint32_t G = NTT_TILE >> ps.S;
  const uint32_t lg_hmin = DIT ? done : ps.S - done - K;
  const uint32_t hmin = 1u << lg_hmin;
  const uint32_t per_group = (1u << ps.S) >> K;
  uint32_t low_base = 0;
  if (ps.lo_bit) low_base = (tile % ((1u << ps.lo_bit) / G)) * G;
  for (uint32_t tt = threadIdx.x; tt < (NTT_TILE >> K); tt += NTT_BLOCK) {
    uint32_t g, jj;
    if (ps.lo_bit) { g = tt % G; jj = tt / G; } else { jj = tt % per_group; g = tt / per_group; }
    const uint32_t off = jj & (hmin - 1), blk = jj >> lg_hmin;
    const uint32_t j0 = (blk << (lg_hmin + K)) | off;
    const uint32_t low = ps.lo_bit ? low_base + g : 0;
    Fr e[R];
#pragma unroll
    for (uint32_t m = 0; m < R; m++) {
      const uint32_t j = j0 + m * hmin;
      e[m] = ntt2_ld<Fr>(dlo, dhi, ntt2_slot(ps.lo_bit ? j * G + g : (g << ps.S) + j));
    }
    if (DIT && first) {
      if (ps.lo_bit) {                     // four-step factor before the first stage
#pragma unroll
        for (uint32_t m = 0; m < R; m++) if (low) e[m] = Fr::mul(e[m], ntt2_factor<Fr>(tw, ps, low, j0 + m * hmin));
      } else if (scale) {                  // coset shift fused into the first pass of the forward transform
#pragma unroll
        for (uint32_t m = 0; m < R; m++) {
          uint32_t jd, lw;
          const uint32_t gi = ntt_tile_global(ps, tile, (g << ps.S) + j0 + m * hmin, &jd, &lw);
          e[m] = Fr::mul(e[m], ntt2_ldg<Fr>(scale + bitrev32(gi, ps.log_n)));
        }
      }
    }
    const bool dif_factor = !DIT && last && ps.lo_bit && low;
#pragma unroll
    for (int q = 0; q < K; q++) {
      const uint32_t hm = DIT ? (1u << q) : (1u << (K - 1 - q));
      const uint32_t lg_hl = lg_hmin + (DIT ? q : K - 1 - q);     // log2 of the LOCAL half-span
#pragma unroll
      for (uint32_t m = 0; m < R; m++) {
        if (m & hm) continue;
        const uint32_t imod = off + (m & (hm - 1)) * hmin;         // position inside the half-span
        const uint32_t wi = imod << (9 - lg_hl);                   // index into the 512 roots W_1024^k
        Fr u = e[m];
        if (DIT) {
          Fr v = wi ? Fr::mul(e[m + hm], ntt2_ld<Fr>(wlo, whi, ntt2_wslot(wi))) : e[m + hm];
          e[m] = Fr::add(u, v);
          e[m + hm] = Fr::sub(u, v);
        } else {
          Fr v = e[m + hm];
          e[m] = Fr::add(u, v);
          Fr d = Fr::sub(u, v);
          e[m + hm] = wi ? Fr::mul(d, ntt2_ld<Fr>(wlo, whi, ntt2_wslot(wi))) : d;
        }
      }
    }
    if (dif_factor) {                      // four-step factor after the last stage (R independent gathers, then R multiplications)
#pragma unroll
      for (uint32_t m = 0; m < R; m++) e[m] = Fr::mul(e[m], ntt2_factor<Fr>(tw, ps, low, j0 + m * hmin));
    }
#pragma unroll
    for (uint32_t m = 0; m < R; m++) {
      const uint32_t j = j0 + m * hmin;
      const uint32_t pos = ps.lo_bit ? j * G + g : (g << ps.S) + j;
      if (last) {
        uint32_t jd, lw;
        x[ntt_tile_global(ps, tile, pos, &jd, &lw)] = e[m];
      } else {
        ntt2_st<Fr>(dlo, dhi, ntt2_slot(pos), e[m]);
      }
    }
  }
}

// `tiles` counts the tiles of all vectors: a batch of vectors of 2^log_n elements back to back shares the twiddles
template <class Fr, bool DIT>
__global__ void __launch_bounds__(NTT_BLOCK, 4) zkb_ntt_tile2(Fr* x_all, const Fr* tw, const Fr* scale, NttPass ps, uint32_t tiles) {
  extern __shared__ uint4 ntt2_smem[];
  uint4* dlo = ntt2_smem;
  uint4* dhi = dlo + NTT2_PLANE;
  uint4* wlo = dhi + NTT2_PLANE;
  uint4* whi = wlo + 512;
  // the 512 roots W_1024^k = w_n^(k * n / 1024): a strided read of the domain table, once per block
  {
    const uint32_t stride = 1u << (ps.log_n - NTT_TILE_LOG);
    for (uint32_t k = threadIdx.x; k < 512; k += NTT_BLOCK) {
      const uint4* src = (const uint4*)(tw + (size_t)k * stride);
      wlo[ntt2_wslot(k)] = src[0];
      whi[ntt2_wslot(k)] = src[1];
    }
  }
  const uint32_t lg_tpv = ps.log_n - NTT_TILE_LOG;                    // tiles per vector: 2^lg_tpv
  for (uint32_t bt = blockIdx.x; bt < tiles; bt += gridDim.x) {
    Fr* x = x_all + ((size_t)(bt >> lg_tpv) << ps.log_n);
    const uint32_t tile = bt & ((1u << lg_tpv) - 1u);
    __syncthreads();                       // the previous tile's last phase has read its shared data
    for (uint32_t k = 0; k < NTT_TILE / NTT_BLOCK; k++) {
      const uint32_t e = threadIdx.x + k * NTT_BLOCK;
      uint32_t j, low;
      const uint4* src = (const uint4*)(x + ntt_tile_global(ps, tile, e, &j, &low));
      const uint32_t slot = ntt2_slot(e);
      ntt2_cp_async16(dlo + slot, src);
      ntt2_cp_async16(dhi + slot, src + 1);
    }
    ntt2_cp_async_wait();
    __syncthreads();
    uint32_t done = 0;
    for (uint32_t p = 0; p < ps.nk; p++) {
      const bool first = p == 0, last = p + 1 == ps.nk;
      switch (ps.K[p]) {
        case 3: ntt2_stages<Fr, DIT, 3>(x, tw, scale, ps, dlo, dhi, wlo, whi, tile, done, first, last); break;
        case 2: ntt2_stages<Fr, DIT, 2>(x, tw, scale, ps, dlo, dhi, wlo, whi, tile, done, first, last); break;
        default: ntt2_stages<Fr, DIT, 1>(x, tw, scale, ps, dlo, dhi, wlo, whi, tile, done, first, last); break;
      }
      done += ps.K[p];
      if (!last) __syncthreads();
    }
  }
}

template <class Fr, bool DIT>
inline void launch_ntt_tile2(Stream st, Fr* x, const Fr* tw, const Fr* scale, const NttPass& ps, size_t tiles, int sm_count) {
  static bool configured = false;          // per instantiation: opt in to > 48 KB of dynamic shared memory once
  if (!configured) {
    ZKB_CUDA(cudaFuncSetAttribute(zkb_ntt_tile2<Fr, DIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)NTT2_SMEM));
    configured = true;
  }
  launch_counter()++;
  const size_t resident = (size_t)sm_count * 4;
  const unsigned grid = (unsigned)(tiles < resident ? tiles : resident);
  zkb_ntt_tile2<Fr, DIT><<<grid, NTT_BLOCK, NTT2_SMEM, st.s>>>(x, tw, scale, ps, (uint32_t)tiles);
  ZKB_CUDA(cudaGetLastError());
}

}  // namespace zkb
#endif
