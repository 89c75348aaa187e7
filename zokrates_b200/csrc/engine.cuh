// Per-curve proving engine: owns the resident proving key shards, R1CS matrices, NTT domain tables
// and MSM workspaces of ONE GPU and sequences the kernels of the Groth16 prover.
//
// Follows ark-groth16 0.3.0 `create_proof_with_reduction` (external crate; call site
// /root/reference/zokrates_ark/src/groth16.rs:44; restated in SURVEY.md App. B.1):
//   h = witness_map(A z, B z, C z);  H = <h_query, h>;  L = <l_query, aux>;
//   A = r d1 + a_0 + <a_query[1..], z[1..]> + alpha1;   B likewise in G1 and G2;
//   C = s A + r B1 - r s d1 + L + H.
// Everything from "z on the host" to "three affine points on the host" runs on the device.
#pragma once
#include <map>
#include <memory>
#include <vector>
#include <chrono>
#include <cmath>
#include <future>
#include <thread>
#include "fp64.cuh"
#include "msm.cuh"
#include "msm_affine.cuh"
#include "ntt.cuh"
#include "ntt_tile.cuh"
#include "solvers.cuh"
#include "rt.cuh"
#include "engine_base.cuh"

#ifndef ZKB_G2_MINB
#define ZKB_G2_MINB 2
#endif

namespace zkb {

// kernel name tags (show up in ncu / nsys kernel names)
struct k_fr_convert; struct k_spmv; struct k_ntt_dif; struct k_ntt_dit; struct k_ntt_scale; struct k_ntt_brev;
struct k_ntt_table; struct k_qap_pointwise; struct k_msm_digits; struct k_msm_scatter; struct k_msm_accum1;
struct k_msm_accum2; struct k_msm_bitsum; struct k_pk_convert; struct k_final_a; struct k_final_b;
struct k_final_c; struct k_final_d; struct k_point_out; struct k_field_op; struct k_setup_scalars; struct k_fixed_base;
struct k_to_affine; struct k_copy; struct k_msm_view; struct k_solver_level; struct k_ba_halve; struct k_ba_round; struct k_msm_table; struct k_ntt_dif_tile; struct k_ntt_dit_tile; struct k_witness_level;

// ---------------------------------------------------------------------------------------------
// stage timer: CUDA events on the engine stream (no-op in the host emulation)
struct StageTimer {
#if !defined(ZKB_EMU)
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
#else
  explicit StageTimer(Stream) {}
  void begin(const char*) {}
  void end() {}
  size_t begin_on(Stream, const char*) { return 0; }
  void end_on(Stream, size_t) {}
  void collect(std::vector<std::pair<const char*, double>>& out) { out.clear(); }
#endif
};

// exclusive scan of NB counters -> offsets[NB+1]
#if !defined(ZKB_EMU)
static __global__ void zkb_scan_kernel(const uint32_t* counts, uint32_t* offsets, uint32_t n) {
  __shared__ uint32_t sums[1024];
  const uint32_t tid = threadIdx.x;
  const uint32_t per = (n + 1023u) / 1024u;
  const uint32_t lo = tid * per < n ? tid * per : n;
  const uint32_t hi = lo + per < n ? lo + per : n;
  uint32_t s = 0;
  for (uint32_t i = lo; i < hi; i++) s += counts[i];
  sums[tid] = s;
  __syncthreads();
  for (uint32_t off = 1; off < 1024; off <<= 1) {
    uint32_t v = tid >= off ? sums[tid - off] : 0;
    __syncthreads();
    sums[tid] += v;
    __syncthreads();
  }
  uint32_t base = tid ? sums[tid - 1] : 0;
  for (uint32_t i = lo; i < hi; i++) {
    offsets[i] = base;
    base += counts[i];
  }
  if (tid == 1023) offsets[n] = sums[1023];
}
#endif
#if !defined(ZKB_EMU)
// three-phase scan for large n: per-tile sums, scan of the tile sums (single block), per-tile rescan
static constexpr int SCAN_BLOCK = 256, SCAN_PER = 8, SCAN_TILE = SCAN_BLOCK * SCAN_PER;
static __global__ void zkb_scan_tile_sums(const uint32_t* in, uint32_t* tile_sums, uint32_t n) {
  __shared__ uint32_t red[SCAN_BLOCK / 32];
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER;
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_PER; k++) s += (base + k < n) ? in[base + k] : 0;
  for (int off = 16; off; off >>= 1) s += __shfl_down_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int k = 0; k < SCAN_BLOCK / 32; k++) t += red[k];
    tile_sums[blockIdx.x] = t;
  }
}
static __global__ void zkb_scan_tile_apply(const uint32_t* in, const uint32_t* tile_offsets, uint32_t* out, uint32_t n,
                                           uint32_t ntiles) {
  __shared__ uint32_t wsum[SCAN_BLOCK / 32];
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER;
  uint32_t v[SCAN_PER], s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_PER; k++) { v[k] = (base + k < n) ? in[base + k] : 0; s += v[k]; }
  // exclusive scan of the per-thread sums across the block
  uint32_t incl = s;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int off = 1; off < 32; off <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= (uint32_t)off) incl += y; }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  uint32_t wbase = 0;
  for (uint32_t k = 0; k < warp; k++) wbase += wsum[k];
  uint32_t run = tile_offsets[blockIdx.x] + wbase + incl - s;
#pragma unroll
  for (int k = 0; k < SCAN_PER; k++) { if (base + k < n) out[base + k] = run; run += v[k]; }
  if (blockIdx.x == ntiles - 1 && threadIdx.x == SCAN_BLOCK - 1) out[n] = tile_offsets[ntiles];
}
#endif
inline void exclusive_scan(Stream st, const uint32_t* counts, uint32_t* offsets, uint32_t n, uint32_t* tile_tmp = nullptr) {
#if !defined(ZKB_EMU)
  if (tile_tmp && n > 4096) {
    const uint32_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    launch_counter() += 3;
    zkb_scan_tile_sums<<<ntiles, SCAN_BLOCK, 0, st.s>>>(counts, tile_tmp, n);
    zkb_scan_kernel<<<1, 1024, 0, st.s>>>(tile_tmp, tile_tmp + ntiles + 1, ntiles);   // offsets of the tiles (+ total)
    zkb_scan_tile_apply<<<ntiles, SCAN_BLOCK, 0, st.s>>>(counts, tile_tmp + ntiles + 1, offsets, n, ntiles);
    ZKB_CUDA(cudaGetLastError());
    return;
  }
  launch_counter()++;
  zkb_scan_kernel<<<1, 1024, 0, st.s>>>(counts, offsets, n);
  ZKB_CUDA(cudaGetLastError());
#else
  (void)tile_tmp;
  uint32_t base = 0;
  for (uint32_t i = 0; i < n; i++) { offsets[i] = base; base += counts[i]; }
  offsets[n] = base;
#endif
}

// ---- MSM views by stable compaction of the sorted list (msm.cuh: "views") -----------------------------------------
static constexpr int VIEW_BLOCK = 256, VIEW_ITERS = 8, VIEW_TILE = VIEW_BLOCK * VIEW_ITERS, VIEW_GROUPS = VIEW_TILE / 32;
#if !defined(ZKB_EMU)
// phase 1: kept entries of view 1 and view 2 per tile of 2048 sorted positions
static __global__ void __launch_bounds__(VIEW_BLOCK) zkb_view_count(MsmShape sh, const uint8_t* skip, const uint32_t* sorted0,
                                                                    const uint32_t* offsets0, uint32_t NB, uint32_t* tile_cnt,
                                                                    uint32_t ntiles) {
  __shared__ uint32_t cnt[2];
  if (threadIdx.x < 2) cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t M = offsets0[NB];
  uint32_t c1 = 0, c2 = 0;
#pragma unroll
  for (int it = 0; it < VIEW_ITERS; it++) {
    const uint32_t p = blockIdx.x * VIEW_TILE + it * VIEW_BLOCK + threadIdx.x;
    if (p < M) {
      const uint32_t e = sorted0[p];
      c1 += msm_view_keep(sh, skip, e, 1);
      c2 += msm_view_keep(sh, skip, e, 2);
    }
  }
  for (int off = 16; off; off >>= 1) { c1 += __shfl_down_sync(0xffffffffu, c1, off); c2 += __shfl_down_sync(0xffffffffu, c2, off); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(&cnt[0], c1); atomicAdd(&cnt[1], c2); }
  __syncthreads();
  if (threadIdx.x < 2) tile_cnt[threadIdx.x * ntiles + blockIdx.x] = cnt[threadIdx.x];
}
// phase 3: write the kept entries at tile offset + rank inside the tile; keep (exclusive count, keep-mask) per 32 positions
static __global__ void __launch_bounds__(VIEW_BLOCK) zkb_view_apply(MsmShape sh, const uint8_t* skip, const uint32_t* sorted0,
                                                                    const uint32_t* offsets0, uint32_t NB, uint32_t nv,
                                                                    const uint32_t* tile_off, uint32_t ntiles, uint32_t* sorted_v,
                                                                    size_t total, uint32_t* pre32, uint32_t* mask32, uint32_t ngroups) {
  __shared__ uint32_t gcnt[2][VIEW_GROUPS];
  const uint32_t M = offsets0[NB];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t e[VIEW_ITERS], m[2][VIEW_ITERS];
#pragma unroll
  for (int it = 0; it < VIEW_ITERS; it++) {
    const uint32_t p = blockIdx.x * VIEW_TILE + it * VIEW_BLOCK + threadIdx.x;
    const bool valid = p < M;
    e[it] = valid ? sorted0[p] : 0;
    const bool f1 = valid && msm_view_keep(sh, skip, e[it], 1), f2 = valid && msm_view_keep(sh, skip, e[it], 2);
    m[0][it] = __ballot_sync(0xffffffffu, f1);
    m[1][it] = __ballot_sync(0xffffffffu, f2);
    if (lane == 0) { gcnt[0][it * 8 + warp] = __popc(m[0][it]); gcnt[1][it * 8 + warp] = __popc(m[1][it]); }
  }
  __syncthreads();
  if (warp < 2) {  // exclusive scan of the 64 group counts of view `warp`: two groups per lane
    const uint32_t a = gcnt[warp][2 * lane], b = gcnt[warp][2 * lane + 1];
    uint32_t incl = a + b;
    for (int off = 1; off < 32; off <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= (uint32_t)off) incl += y; }
    const uint32_t excl = incl - (a + b);
    gcnt[warp][2 * lane] = excl;
    gcnt[warp][2 * lane + 1] = excl + a;
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < VIEW_ITERS; it++) {
    const uint32_t p = blockIdx.x * VIEW_TILE + it * VIEW_BLOCK + threadIdx.x;
    for (uint32_t v = 0; v < nv; v++) {
      const uint32_t base = tile_off[(size_t)v * (ntiles + 1) + blockIdx.x] + gcnt[v][it * 8 + warp];
      const uint32_t mk = m[v][it];
      if (lane == 0 && p < M) { pre32[(size_t)v * ngroups + (p >> 5)] = base; mask32[(size_t)v * ngroups + (p >> 5)] = mk; }
      if ((mk >> lane) & 1u) sorted_v[(size_t)v * total + base + __popc(mk & ((1u << lane) - 1u))] = e[it];
    }
  }
}
#endif

// ---------------------------------------------------------------------------------------------
struct MsmPlan {
  MsmShape sh{0, 0, 0, 0, 0, 1};
  uint32_t nbuckets = 0;
  uint32_t T1 = 32, T2 = 32;
  uint32_t nt1 = 0;  // level-1 chunks
  uint32_t nviews = 1;
  DevBuf<uint32_t> digits, ranks, counts, offsets, sorted, scan_tmp;
  DevBuf<uint32_t> view_tile_cnt, view_tile_off, view_pre32, view_mask32;   // views by compaction (build_views)
};

inline uint32_t msm_pick_c(uint64_t n, int fr_bits) {
  uint32_t best = 4;
  double best_cost = 1e300;
  for (uint32_t c = 4; c <= 16; c++) {
    double W = (double)((fr_bits + 1 + c - 1) / c);
    double cost = W * (10.0 * (double)n + 40.0 * (double)(1u << (c - 1)));
    if (cost < best_cost) { best_cost = cost; best = c; }
  }
  return best;
}

// with precomputed window multiples all windows share one bucket set, so larger windows pay off
inline uint32_t msm_pick_c_pre(uint64_t n, int fr_bits, uint64_t max_w = 16 /* msm_table_body keeps W multiples per thread */) {
  uint32_t best = 0;
  double best_cost = 1e300;
  for (uint32_t c = 4; c <= 22; c++) {
    uint64_t W = (fr_bits + 1 + c - 1) / c;
    if (W > max_w || n * W >= (1ull << 31)) continue;
    // relative costs in Fq multiplications: 10 per mixed addition, ~70 per bucket in the reductions (segmented partial
    // levels + bit sums, full additions).  The dedicated square and the once-reduced Y3 (DESIGN.md §4) made both sides
    // cheaper by similar fractions (G1 mixed addition 1360 -> 1232 wide MADs, -9.4 %; full addition 1904 -> 1776, -6.7 %),
    // so the 10 : 70 ratio, and with it the window picked at every size, stays as measured on H100 (DESIGN.md §7)
    double cost = (double)W * 10.0 * (double)n + 70.0 * (double)(1u << (c - 1));
    if (cost < best_cost) { best_cost = cost; best = c; }
  }
  return best;
}

// fixed-base window table: table[j * 256 + d] = d * 2^(8 j) * G, j < 32 (setup.cuh)
template <class F>
struct FixedBase {
  DevBuf<Affine<F>> table;
  DevBuf<XYZZ<F>> bases;
};

template <class FrP, class FqP>
struct CurveT {
  typedef Fp<FrP> Fr;
  typedef Fp<FqP> Fq;
  typedef Fp2<FqP> Fq2;
  typedef Affine<Fq> G1A;
  typedef Affine<Fq2> G2A;
  typedef XYZZ<Fq> G1X;
  typedef XYZZ<Fq2> G2X;
  // host mirrors (64-bit limbs, identical memory layout) for the serial tail of the prover
  typedef Fp64<FrP> HFr;
  typedef Fp64<FqP> HFq;
  typedef Fp2T<HFq> HFq2;
  static constexpr int FR_BITS = FrP::BITS;
  static constexpr int FQ_BYTES = FqP::N * 4;
};

template <class C>
class Engine : public EngineBase {
 public:
  typedef typename C::Fr Fr;
  typedef typename C::Fq Fq;
  typedef typename C::Fq2 Fq2;
  typedef typename C::G1A G1A;
  typedef typename C::G2A G2A;
  typedef typename C::G1X G1X;
  typedef typename C::G2X G2X;
  typedef typename C::HFr HFr;
  typedef typename C::HFq HFq;
  typedef typename C::HFq2 HFq2;
  typedef Affine<HFq> HG1A;
  typedef Affine<HFq2> HG2A;
  typedef XYZZ<HFq> HG1X;
  typedef XYZZ<HFq2> HG2X;
  static_assert(sizeof(HG1X) == sizeof(G1X) && sizeof(HG2X) == sizeof(G2X) && sizeof(HG1A) == sizeof(G1A), "host/device layout");
  static constexpr size_t FRB = 32, FQB = C::FQ_BYTES, G1B = 2 * FQB, G2B = 4 * FQB;
  static_assert(sizeof(Fr) == 32 && sizeof(G1A) == G1B && sizeof(G2A) == G2B, "layout");

  struct Partial {  // per-rank partial sums, in this order
    G1X h, l, a, b1;
    G2X b2;
  };

  explicit Engine(Stream st) : st_(st) {}

  void sizes(uint64_t out[4]) override {
    out[0] = FRB; out[1] = FQB; out[2] = 8 * FQB; out[3] = sizeof(Partial);
  }

  // ------------------------------------------------------------------------------ domains
  struct DomainT {
    uint32_t log_n = 0;
    DevBuf<Fr> tw_fwd, tw_inv, cos_fwd, cos_inv;  // w^k, w^-k (k < n/2);  g^k / n, g^-k / n (k < n)
    Fr zinv;                                      // 1 / (g^n - 1)
    Fr ninv;
  };
  std::map<uint32_t, std::unique_ptr<DomainT>> domains_;

  static Fr fr_gen() { Fr g; for (int i = 0; i < Fr::N; i++) g.v[i] = Fr::Params::gen(i); return g; }
  static Fr fr_root() { Fr g; for (int i = 0; i < Fr::N; i++) g.v[i] = Fr::Params::root(i); return g; }
  static Fr fr_omega(uint32_t log_n) {
    Fr w = fr_root();
    for (uint32_t i = log_n; i < (uint32_t)Fr::Params::TWO_ADICITY; i++) w = Fr::sqr(w);
    return w;
  }

  DomainT& domain(uint32_t log_n) {
    auto it = domains_.find(log_n);
    if (it != domains_.end()) return *it->second;
    if (log_n > (uint32_t)Fr::Params::TWO_ADICITY || log_n > 28) throw Error(ZKB_E_ARG, "domain too large");
    std::unique_ptr<DomainT> d(new DomainT());
    d->log_n = log_n;
    const uint32_t n = 1u << log_n;
    Fr w = fr_omega(log_n), wi = Fr::inv(w), g = fr_gen(), gi = Fr::inv(g);
    Fr nf = Fr::to_mont(fr_from_u64(n));
    d->ninv = Fr::inv(nf);
    d->zinv = Fr::inv(Fr::sub(Fr::pow_u64(g, n), Fr::one()));
    d->tw_fwd.alloc(n / 2 + 1); d->tw_inv.alloc(n / 2 + 1); d->cos_fwd.alloc(n); d->cos_inv.alloc(n);
    Fr one = Fr::one(), ninv = d->ninv;
    Fr* p0 = d->tw_fwd.p; Fr* p1 = d->tw_inv.p; Fr* p2 = d->cos_fwd.p; Fr* p3 = d->cos_inv.p;
    launch<k_ntt_table>(st_, n / 2, ZKB_LAMBDA(size_t t) { ntt_powers_body<Fr>(w, one, p0, n / 2, (uint32_t)t); });
    launch<k_ntt_table>(st_, n / 2, ZKB_LAMBDA(size_t t) { ntt_powers_body<Fr>(wi, one, p1, n / 2, (uint32_t)t); });
    launch<k_ntt_table>(st_, n, ZKB_LAMBDA(size_t t) { ntt_powers_body<Fr>(g, ninv, p2, n, (uint32_t)t); });
    launch<k_ntt_table>(st_, n, ZKB_LAMBDA(size_t t) { ntt_powers_body<Fr>(gi, ninv, p3, n, (uint32_t)t); });
    DomainT& ref = *d;
    domains_[log_n] = std::move(d);
    return ref;
  }

  static Fr fr_from_u64(uint64_t v) {
    Fr r = Fr::zero();
    r.v[0] = (uint32_t)v;
    r.v[1] = (uint32_t)(v >> 32);
    return r;
  }

  // Transforms of 2^10 and more points run as shared-memory tile passes (ntt_block_body: 10 stages per HBM round
  // trip); smaller ones as register passes (3 stages per round trip).  ZKB_OPT_NTT_TILE_MIN / ZKB_OPT_NTT_MAX_S: test knobs.
  uint32_t ntt_tile_min() const { return opts.ntt_tile_min < (int64_t)NTT_TILE_LOG ? NTT_TILE_LOG : (uint32_t)opts.ntt_tile_min; }
  uint32_t ntt_max_s() const { return opts.ntt_max_s < 5 ? 5u : (uint32_t)opts.ntt_max_s; }
  bool ntt_tiled(uint32_t log_n) const { return log_n >= ntt_tile_min(); }
  int sm_count_ = 0;
  int sm_count() {
#if !defined(ZKB_EMU)
    if (!sm_count_) {
      int dev = 0;
      ZKB_CUDA(cudaGetDevice(&dev));
      ZKB_CUDA(cudaDeviceGetAttribute(&sm_count_, cudaDevAttrMultiProcessorCount, dev));
    }
#endif
    return sm_count_ ? sm_count_ : 1;
  }

  // natural -> bit-reversed.  `count` vectors of 2^log_n elements back to back (a batch of proofs): every launch transforms
  // all of them with the same twiddles, a thread or tile finds its vector from its index.
  void ntt_dif(Fr* x, const Fr* tw, uint32_t log_n, uint32_t count = 1) {
    NttPass ps[8];
    const uint32_t np = ntt_tiled(log_n) ? ntt_plan_passes(log_n, ntt_max_s(), ps) : 0;
    if (np) {
      const uint32_t lg_tpv = log_n - NTT_TILE_LOG;
      const size_t tiles = (size_t)count << lg_tpv;
      const Fr* nul = nullptr;
#if !defined(ZKB_EMU)
      if (opts.ntt_kernel == 2) {           // four-step twiddles, cp.async tile load, padded planes (ntt_tile.cuh)
        for (uint32_t i = 0; i < np; i++) launch_ntt_tile2<Fr, false>(st_, x, tw, nul, ps[i], tiles, sm_count());
        return;
      }
#endif
      for (uint32_t i = 0; i < np; i++) {   // top stage bits first
        NttPass p = ps[i];
        launch_block<k_ntt_dif_tile, NTT_BLOCK, NTT_TILE * sizeof(Fr)>(st_, tiles, p.nk + 2, ZKB_LAMBDA(uint32_t b, uint32_t t, uint32_t ph, void* sm) {
          ntt_block_body<Fr, false>(x + ((size_t)(b >> lg_tpv) << log_n), tw, nul, p, (Fr*)sm, b & ((1u << lg_tpv) - 1u), t, ph);
        });
      }
      return;
    }
    uint32_t h = (1u << log_n) >> 1, rem = log_n;
    const size_t cn = (size_t)count << log_n;
    while (rem > 0) {
      uint32_t K = rem >= 3 ? 3 : rem;
      uint32_t h0 = h;
      // thread t of the launch: vector t >> (log_n - K), butterfly group t mod 2^(log_n - K)
      const uint32_t lg = log_n - K;
      if (K == 3) launch<k_ntt_dif>(st_, cn >> 3, ZKB_LAMBDA(size_t t) { ntt_dif_body<Fr, 3>(x + ((t >> lg) << log_n), tw, log_n, h0, (uint32_t)(t & ((1u << lg) - 1u))); });
      else if (K == 2) launch<k_ntt_dif>(st_, cn >> 2, ZKB_LAMBDA(size_t t) { ntt_dif_body<Fr, 2>(x + ((t >> lg) << log_n), tw, log_n, h0, (uint32_t)(t & ((1u << lg) - 1u))); });
      else launch<k_ntt_dif>(st_, cn >> 1, ZKB_LAMBDA(size_t t) { ntt_dif_body<Fr, 1>(x + ((t >> lg) << log_n), tw, log_n, h0, (uint32_t)(t & ((1u << lg) - 1u))); });
      h >>= K;
      rem -= K;
    }
  }
  // bit-reversed -> natural; `scale` (optional): x[i] *= scale[bitrev(i)] first (the coset shift between ifft and coset fft)
  void ntt_dit(Fr* x, const Fr* tw, uint32_t log_n, const Fr* scale = nullptr, uint32_t count = 1) {
    NttPass ps[8];
    const uint32_t np = ntt_tiled(log_n) ? ntt_plan_passes(log_n, ntt_max_s(), ps) : 0;
    if (np) {
      const uint32_t lg_tpv = log_n - NTT_TILE_LOG;
      const size_t tiles = (size_t)count << lg_tpv;
#if !defined(ZKB_EMU)
      if (opts.ntt_kernel == 2) {
        for (uint32_t i = np; i-- > 0;) launch_ntt_tile2<Fr, true>(st_, x, tw, (i == np - 1) ? scale : nullptr, ps[i], tiles, sm_count());
        return;
      }
#endif
      for (uint32_t i = np; i-- > 0;) {     // low stage bits first
        NttPass p = ps[i];
        const Fr* sc = (i == np - 1) ? scale : nullptr;
        launch_block<k_ntt_dit_tile, NTT_BLOCK, NTT_TILE * sizeof(Fr)>(st_, tiles, p.nk + 2, ZKB_LAMBDA(uint32_t b, uint32_t t, uint32_t ph, void* sm) {
          ntt_block_body<Fr, true>(x + ((size_t)(b >> lg_tpv) << log_n), tw, sc, p, (Fr*)sm, b & ((1u << lg_tpv) - 1u), t, ph);
        });
      }
      return;
    }
    const size_t cn = (size_t)count << log_n;
    const uint32_t nmask = (1u << log_n) - 1u;
    if (scale) launch<k_ntt_scale>(st_, cn, ZKB_LAMBDA(size_t t) { ntt_scale_brev_body<Fr>(x + ((t >> log_n) << log_n), scale, log_n, (uint32_t)(t & nmask)); });
    uint32_t h = 1, rem = log_n;
    while (rem > 0) {
      uint32_t K = rem >= 3 ? 3 : rem;
      uint32_t h0 = h;
      const uint32_t lg = log_n - K;
      if (K == 3) launch<k_ntt_dit>(st_, cn >> 3, ZKB_LAMBDA(size_t t) { ntt_dit_body<Fr, 3>(x + ((t >> lg) << log_n), tw, log_n, h0, (uint32_t)(t & ((1u << lg) - 1u))); });
      else if (K == 2) launch<k_ntt_dit>(st_, cn >> 2, ZKB_LAMBDA(size_t t) { ntt_dit_body<Fr, 2>(x + ((t >> lg) << log_n), tw, log_n, h0, (uint32_t)(t & ((1u << lg) - 1u))); });
      else launch<k_ntt_dit>(st_, cn >> 1, ZKB_LAMBDA(size_t t) { ntt_dit_body<Fr, 1>(x + ((t >> lg) << log_n), tw, log_n, h0, (uint32_t)(t & ((1u << lg) - 1u))); });
      h <<= K;
      rem -= K;
    }
  }

  void convert(const Fr* in, Fr* out, int dir, size_t n) {
    launch<k_fr_convert>(st_, n, ZKB_LAMBDA(size_t t) { fr_convert_body<Fr>(in, out, dir, n, t); });
  }

  // zkb_ntt: natural order in/out, canonical LE on the host
  void ntt(uint64_t* data, uint32_t log_n, int inverse, int coset) override {
    StageTimer tm(st_);
    DomainT& d = domain(log_n);
    const size_t n = (size_t)1 << log_n;
    scratch_a_.ensure(n);
    scratch_b_.ensure(n);
    Fr* x = scratch_a_.p;
    Fr* y = scratch_b_.p;
    h2d(st_, x, data, n * FRB);
    convert(x, x, 0, n);
    tm.begin("ntt");
    if (!inverse) {
      if (coset) {  // x[k] *= g^k  (table holds g^k / n: undo the 1/n)
        const Fr* tab = d.cos_fwd.p;
        Fr nf = Fr::to_mont(fr_from_u64(n));
        launch<k_ntt_scale>(st_, n, ZKB_LAMBDA(size_t t) { x[t] = Fr::mul(Fr::mul(x[t], tab[t]), nf); });
      }
      ntt_dif(x, d.tw_fwd.p, log_n);
      const Fr* nul = nullptr;
      launch<k_ntt_brev>(st_, n, ZKB_LAMBDA(size_t t) { ntt_brev_copy_body<Fr>(x, y, nul, log_n, 1, (uint32_t)t); });
    } else {
      ntt_dif(x, d.tw_inv.p, log_n);
      if (coset) {
        const Fr* tab = d.cos_inv.p;
        launch<k_ntt_brev>(st_, n, ZKB_LAMBDA(size_t t) { ntt_brev_copy_body<Fr>(x, y, tab, log_n, 1, (uint32_t)t); });
      } else {
        Fr ninv = d.ninv;
        launch<k_ntt_brev>(st_, n, ZKB_LAMBDA(size_t t) {
          uint32_t j = bitrev32((uint32_t)t, log_n);
          y[j] = Fr::from_mont(Fr::mul(x[t], ninv));
        });
      }
    }
    tm.end();
    d2h(st_, data, y, n * FRB);
    stream_sync(st_);
    tm.collect(timings);
  }

  // ------------------------------------------------------------------------------ R1CS
  struct R1cs {
    uint64_t N = 0, ni = 0, nw = 0, m = 0;
    uint32_t log_n = 0;
    DevBuf<uint32_t> rowptr[3], col[3];
    DevBuf<Fr> val[3];
    DevBuf<Fr> z_canon, z_mont;     // resident assignment (zkb_r1cs_set_assignment / zkb_witness_eval); per-proof vectors live in ProofSlot
    bool has_z = false;
    bool sparse_z = false;  // most assignment values are tiny (bits): the z MSMs are cheap, prefer the per-window bucket sets (shallower reductions)
    // host copies kept for setup (CSC transposition) — small relative to the device data
    std::vector<uint32_t> h_rowptr[3], h_col[3];
  };
  std::map<uint64_t, std::unique_ptr<R1cs>> r1cs_;
  uint64_t next_handle_ = 1;

  R1cs& get_r1cs(uint64_t h) {
    auto it = r1cs_.find(h);
    if (it == r1cs_.end()) throw Error(ZKB_E_ARG, "unknown r1cs handle");
    return *it->second;
  }

  uint64_t r1cs_load(uint64_t N, uint64_t ni, uint64_t nw, const uint64_t* const rowptr[3], const uint32_t* const col[3],
                     const uint64_t* const val[3]) override {
    if (ni < 1) throw Error(ZKB_E_ARG, "n_instance must count the constant one");
    std::unique_ptr<R1cs> r(new R1cs());
    r->N = N; r->ni = ni; r->nw = nw; r->m = ni + nw;
    uint64_t dom = N + ni, n = 1;
    uint32_t lg = 0;
    while (n < dom) { n <<= 1; lg++; }
    if (lg > 28 || r->m >= (1ull << 31)) throw Error(ZKB_E_ARG, "circuit too large");
    r->log_n = lg;
    for (int k = 0; k < 3; k++) {
      uint64_t nnz = rowptr[k][N];
      if (nnz >= (1ull << 32)) throw Error(ZKB_E_ARG, "too many non-zeros");
      std::vector<uint32_t>& rp = r->h_rowptr[k];
      rp.resize(N + 1);
      for (uint64_t i = 0; i <= N; i++) {
        if (rowptr[k][i] > nnz || (i && rowptr[k][i] < rowptr[k][i - 1])) throw Error(ZKB_E_ARG, "bad rowptr");
        rp[i] = (uint32_t)rowptr[k][i];
      }
      r->h_col[k].assign(col[k], col[k] + nnz);
      for (uint64_t i = 0; i < nnz; i++)
        if (col[k][i] >= r->m) throw Error(ZKB_E_ARG, "column index out of range");
      r->rowptr[k].alloc(N + 1);
      r->col[k].alloc(nnz);
      r->val[k].alloc(nnz);
      h2d(st_, r->rowptr[k].p, rp.data(), (N + 1) * 4);
      h2d(st_, r->col[k].p, col[k], nnz * 4);
      h2d(st_, r->val[k].p, val[k], nnz * FRB);
      convert(r->val[k].p, r->val[k].p, 0, nnz);
    }
    r->z_canon.alloc(r->m); r->z_mont.alloc(r->m);
    (void)n;
    domain(lg);
    stream_sync(st_);
    uint64_t h = next_handle_++;
    r1cs_[h] = std::move(r);
    return h;
  }
  void r1cs_free(uint64_t h) override {
    for (auto& sl : slots_)
      if (sl.state != 0 && sl.r1cs == h) throw Error(ZKB_E_ARG, "a proof that uses this R1CS is in flight (collect it first)");
    r1cs_.erase(h);
  }

  void set_assignment(uint64_t h, const uint64_t* z) override {
    R1cs& r = get_r1cs(h);
    h2d(st_, r.z_canon.p, z, r.m * FRB);
    stream_sync(st_);
    r.has_z = true;
    r.sparse_z = assignment_is_sparse(z, r.m);
  }

  // ------------------------------------------------------------------------------ per-proof state
  // Everything one proof writes on the device lives in a ProofSlot, and there are two of them: while the host finishes
  // proof i (the last few hundred point additions of every MSM, the final combination, the multi-GPU gather) the GPU
  // already runs proof i + 1 — its digit plans and accumulate kernels overlap the latency-bound reduction tails of
  // proof i.  Read-only state (key shards, matrices, domain tables) is shared.
  // the four scalar multiplications that only need (pk, r, s): computed on host threads while the GPU works
  struct FixedMults {
    HG1X rd, sd, rsd;
    HG2X sd2;
  };
  struct MsmWs {
    DevBuf<uint8_t> buckets, val[2], tree[4];
    DevBuf<uint32_t> key[2];
    Stream tail;          // high-priority side stream for accum2 / bit sums
    Event acc_done, tail_done;
    bool has_stream = false;
    // filled by msm_tail: the bit-sum reduction consumed `tree_bits` index bits and left `tree_cnt` block totals per window
    uint32_t nt1 = 0;         // chunks of the last accumulation into this workspace (the partial lists hold 2 nt1 entries)
    uint32_t tree_cnt = 1, tree_bits = 0;
    size_t out_entries = 0;   // XYZZ entries of the result slot the host has to read: (1 + tree_bits) * W * tree_cnt
    void destroy() { if (has_stream) { stream_destroy(tail); has_stream = false; } acc_done.destroy(); tail_done.destroy(); }
  };
  struct ProofSlot {
    DevBuf<Fr> z_canon, z_mont, a, b, c, h;   // assignment (when it came from the host), its Montgomery image, witness-map vectors
    const Fr* z_src = nullptr;                // canonical assignment this proof reads (own upload or the resident one)
    bool sparse_z = false;
    MsmPlan plan_z, plan_h;
    MsmWs ws[5];                              // h, l, a, b1, b2
    DevBuf<uint8_t> d_win;                    // result slots of the five MSMs
    HostBuf hw;                               // pinned landing zone of the same
    std::unique_ptr<StageTimer> tm, tm2;
    Event ev_z_ready, ev_h_ready, ev_chains_done, ev_exchange, ev_plan_z, done;
    Stream fin; bool has_fin = false;         // waits for the five tails and copies the results out, off the main stream
    uint64_t pk = 0, r1cs = 0, ticket = 0;
    int state = 0;                            // 0 free, 1 begun (assignment MSMs enqueued), 2 fully enqueued (collectable)
    bool has_rs = false;
    uint32_t r[8], s[8];
    std::future<FixedMults> fm;
    void destroy() {
      for (auto& w : ws) w.destroy();
      ev_z_ready.destroy(); ev_h_ready.destroy(); ev_chains_done.destroy(); ev_exchange.destroy(); ev_plan_z.destroy(); done.destroy();
      if (has_fin) { stream_destroy(fin); has_fin = false; }
    }
  };
  static constexpr int NUM_SLOTS = 2;
  ProofSlot slots_[NUM_SLOTS];
  uint64_t next_ticket_ = 1;
  void slot_vectors(ProofSlot& sl, const R1cs& r) {
    const size_t n = (size_t)1 << r.log_n;
    sl.z_canon.ensure(r.m); sl.z_mont.ensure(r.m);
    sl.a.ensure(n); sl.b.ensure(n); sl.c.ensure(n); sl.h.ensure(n);
  }

  // h (canonical, natural order) = witness_map(z)   [device-resident]
  // The witness map in two halves so that several GPUs can share it (zkb_groth16_prove_begin / _end):
  //   chains: for every k in `mask`: v_k = coset_fft(ifft(M_k z)) — three independent SpMV + 2 transforms (a, b, c)
  //   finish: h = coset_ifft((a∘b − c) / Z)  — needs all three chains
  void wm_chains(R1cs& r, ProofSlot& sl, uint32_t mask, StageTimer& tm) {
    DomainT& d = domain(r.log_n);
    const uint32_t lg = r.log_n;
    const size_t n = (size_t)1 << lg;
    tm.begin("witness_map_chains");
    convert(sl.z_src, sl.z_mont.p, 0, r.m);
    Fr* vec[3] = {sl.a.p, sl.b.p, sl.c.p};
    const Fr* zm = sl.z_mont.p;
    const Fr* t1 = d.cos_fwd.p;
    for (int k = 0; k < 3; k++) {
      if (!((mask >> k) & 1u)) continue;
      Fr* out = vec[k];
      const uint32_t* rp = r.rowptr[k].p;
      const uint32_t* cl = r.col[k].p;
      const Fr* vl = r.val[k].p;
      const uint32_t N = (uint32_t)r.N;
      dev_zero(st_, out + r.N, (n - r.N) * FRB);
      launch<k_spmv>(st_, r.N, ZKB_LAMBDA(size_t t) { spmv_body<Fr>(rp, cl, vl, zm, out, N, (uint32_t)t); });
      if (k == 0) d2d(st_, sl.a.p + r.N, sl.z_mont.p, r.ni * FRB);  // a[N + j] = z[j] for the instance variables
      ntt_dif(out, d.tw_inv.p, lg);
      ntt_dit(out, d.tw_fwd.p, lg, t1);   // coset shift (g^k / n at the bit-reversed position) fused into the first pass
    }
    tm.end();
  }
  // `count` proofs: vector k of a, b, c and h at offset k n (the chains of a batch are back to back)
  void wm_finish(R1cs& r, Fr* pa, const Fr* pb, const Fr* pc, Fr* ph, uint32_t count, StageTimer& tm, const char* name) {
    DomainT& d = domain(r.log_n);
    const uint32_t lg = r.log_n;
    const size_t cn = (size_t)count << lg;
    tm.begin(name);
    Fr zinv = d.zinv;
    launch<k_qap_pointwise>(st_, cn, ZKB_LAMBDA(size_t t) { qap_pointwise_body<Fr>(pa, pb, pc, zinv, (uint32_t)cn, (uint32_t)t); });
    ntt_dif(pa, d.tw_inv.p, lg, count);
    const Fr* t2 = d.cos_inv.p;
    const uint32_t nmask = (1u << lg) - 1u;
    launch<k_ntt_brev>(st_, cn, ZKB_LAMBDA(size_t t) {
      const size_t base = (t >> lg) << lg;
      ntt_brev_copy_body<Fr>(pa + base, ph + base, t2, lg, 1, (uint32_t)(t & nmask));
    });
    tm.end();
  }

  void witness_map(uint64_t h, const uint64_t* z, uint64_t* h_out, uint64_t cap) override {
    R1cs& r = get_r1cs(h);
    const size_t n = (size_t)1 << r.log_n;
    if (cap < n) throw Error(ZKB_E_ARG, "h_out too small");
    ProofSlot& sl = slots_[0];
    if (sl.state != 0) throw Error(ZKB_E_ARG, "a proof is in flight on this context");
    slot_vectors(sl, r);
    StageTimer tm(st_);
    h2d(st_, sl.z_canon.p, z, r.m * FRB);
    sl.z_src = sl.z_canon.p;
    tm.begin("witness_map");
    wm_chains(r, sl, 7, tm);
    wm_finish(r, sl.a.p, sl.b.p, sl.c.p, sl.h.p, 1, tm, "witness_map_finish");
    tm.end();
    d2h(st_, h_out, sl.h.p, n * FRB);
    stream_sync(st_);
    tm.collect(timings);
  }

  // Witness evaluation by dependency levels and the R1CS satisfaction check (ntt.cuh::witness_level_body).
  // z_io: canonical assignment, inputs filled in, m x 32 bytes (nullptr: check the resident assignment);
  // level_ptr[n_levels + 1] indexes rows / out_var (column assigned by that row or WIT_CHECK).  n_levels == 0: check all rows.
  // The finished assignment stays resident (zkb_groth16_prove_resident can follow).  Returns the first unsatisfied row or ~0.
  uint64_t witness_eval(uint64_t rh, uint64_t* z_io, uint32_t n_levels, const uint32_t* level_ptr, const uint32_t* rows,
                        const uint32_t* out_var) override {
    R1cs& r = get_r1cs(rh);
    StageTimer tm(st_);
    if (z_io) h2d(st_, r.z_canon.p, z_io, r.m * FRB);
    else if (!r.has_z) throw Error(ZKB_E_ARG, "no resident assignment");
    DevBuf<uint32_t> d_rows, d_out, d_flag(1);
    dev_fill_ff(st_, d_flag.p, 4);
    tm.begin("witness_eval");
    convert(r.z_canon.p, r.z_mont.p, 0, r.m);
    const uint32_t* rpA = r.rowptr[0].p; const uint32_t* clA = r.col[0].p; const Fr* vlA = r.val[0].p;
    const uint32_t* rpB = r.rowptr[1].p; const uint32_t* clB = r.col[1].p; const Fr* vlB = r.val[1].p;
    const uint32_t* rpC = r.rowptr[2].p; const uint32_t* clC = r.col[2].p; const Fr* vlC = r.val[2].p;
    Fr* zm = r.z_mont.p;
    uint32_t* flag = d_flag.p;
    if (n_levels == 0) {
      const uint32_t* nul = nullptr;
      const uint32_t N = (uint32_t)r.N;
      launch<k_witness_level>(st_, r.N, ZKB_LAMBDA(size_t t) {
        witness_level_body<Fr>(rpA, clA, vlA, rpB, clB, vlB, rpC, clC, vlC, zm, nul, nul, 0, N, 1u, flag, (uint32_t)t);
      });
    } else {
      if (!level_ptr || !rows || !out_var) throw Error(ZKB_E_ARG, "null level description");
      const uint32_t total = level_ptr[n_levels];
      for (uint32_t l = 0; l < n_levels; l++)
        if (level_ptr[l] > level_ptr[l + 1] || level_ptr[l + 1] > total) throw Error(ZKB_E_ARG, "bad level_ptr");
      for (uint32_t i = 0; i < total; i++)
        if (rows[i] >= r.N || (out_var[i] != WIT_CHECK && out_var[i] >= r.m)) throw Error(ZKB_E_ARG, "row / variable index out of range");
      d_rows.alloc(total ? total : 1); d_out.alloc(total ? total : 1);
      h2d(st_, d_rows.p, rows, (size_t)total * 4);
      h2d(st_, d_out.p, out_var, (size_t)total * 4);
      const uint32_t* pr = d_rows.p; const uint32_t* po = d_out.p;
      for (uint32_t l = 0; l < n_levels; l++) {
        const uint32_t lo = level_ptr[l], hi = level_ptr[l + 1];
        launch<k_witness_level>(st_, hi - lo, ZKB_LAMBDA(size_t t) {
          witness_level_body<Fr>(rpA, clA, vlA, rpB, clB, vlB, rpC, clC, vlC, zm, pr, po, lo, hi, 1u, flag, (uint32_t)t);
        });
      }
      convert(r.z_mont.p, r.z_canon.p, 1, r.m);
    }
    tm.end();
    uint32_t first = 0;
    d2h(st_, &first, d_flag.p, 4);
    if (z_io && n_levels) d2h(st_, z_io, r.z_canon.p, r.m * FRB);
    stream_sync(st_);
    tm.collect(timings);
    if (z_io || n_levels) { r.has_z = true; }
    if (z_io && n_levels) r.sparse_z = assignment_is_sparse(z_io, r.m);
    else if (z_io) r.sparse_z = assignment_is_sparse(z_io, r.m);
    return first == 0xFFFFFFFFu ? ~0ull : (uint64_t)first;
  }

  // ------------------------------------------------------------------------------ compiled programs (`out` files)
  // zkb_prog_load: parse the program file, synthesise the R1CS in ark order and keep it resident (an ordinary R1CS handle),
  // keep the directive tables and the level schedule on the device.  zkb_prog_compute_witness then runs the statements
  // level by level: constraints through witness_level_body (assign or check), directives through solver_body.
  struct ProgDev {
    ProgData d;
    DevBuf<uint32_t> kind, arg, in_ptr, out_ptr, out_cols, lc_ptr, lc_col, rows, out_var, dirs, arg_cols;
    DevBuf<Fr> lc_val;
    std::vector<uint64_t> z_host;   // the assignment of the last compute_witness / set_witness (m x 4 words), for public_inputs
    uint64_t fp[2] = {0, 0};        // content fingerprint of the program file
  };
  // programs are shared by content like proving keys (ZKB_OPT_PK_CACHE): the static trait method receives the program on every
  // call, a second load of the same bytes returns a handle onto the resident program, the last one released stays resident
  std::map<uint64_t, std::shared_ptr<ProgDev>> progs_;
  std::shared_ptr<ProgDev> idle_prog_;
  ProgDev& get_prog(uint64_t h) {
    auto it = progs_.find(h);
    if (it == progs_.end()) throw Error(ZKB_E_ARG, "unknown program handle");
    return *it->second;
  }
  static void fr_modulus(uint32_t mod[8]) { for (int i = 0; i < 8; i++) mod[i] = Fr::Params::mod(i); }
  template <class T>
  void upload(DevBuf<T>& buf, const std::vector<T>& v) {
    buf.alloc(v.size() ? v.size() : 1);
    h2d(st_, buf.p, v.data(), v.size() * sizeof(T));
  }

  uint64_t prog_load(const uint8_t* data, size_t len, int curve) override {
    uint64_t fp[2] = {0, 0};
    if (opts.pk_cache) {
      fingerprint_par(data, len, 0x70726f67ull /* "prog" */, fp);
      std::shared_ptr<ProgDev> hit;
      if (idle_prog_ && idle_prog_->fp[0] == fp[0] && idle_prog_->fp[1] == fp[1]) { hit = idle_prog_; idle_prog_.reset(); }
      else for (auto& kv : progs_) if (kv.second->fp[0] == fp[0] && kv.second->fp[1] == fp[1]) { hit = kv.second; break; }
      if (hit) {
        timings.clear();
        timings.push_back({"prog_cache_hit", 1.0});
        uint64_t h = next_handle_++;
        progs_[h] = hit;
        return h;
      }
    }
    if (idle_prog_) { r1cs_free(idle_prog_->d.r1cs); idle_prog_.reset(); }
    std::shared_ptr<ProgDev> p(new ProgDev());
    p->fp[0] = fp[0]; p->fp[1] = fp[1];
    uint32_t mod[8];
    fr_modulus(mod);
    prog_parse(data, len, curve, mod, p->d);
    prog_schedule(p->d);
    ProgData& d = p->d;
    const uint64_t* rp[3] = {d.rowptr[0].data(), d.rowptr[1].data(), d.rowptr[2].data()};
    const uint32_t* cl[3] = {d.col[0].data(), d.col[1].data(), d.col[2].data()};
    const uint64_t* vl[3] = {d.val[0].data(), d.val[1].data(), d.val[2].data()};
    d.r1cs = r1cs_load(d.N, d.ni, d.nw, rp, cl, vl);
    try {
      upload(p->kind, d.d_kind); upload(p->arg, d.d_arg); upload(p->in_ptr, d.d_in_ptr); upload(p->out_ptr, d.d_out_ptr);
      upload(p->out_cols, d.d_out_cols); upload(p->lc_ptr, d.lc_ptr); upload(p->lc_col, d.lc_col);
      upload(p->rows, d.rows); upload(p->out_var, d.out_var); upload(p->dirs, d.dirs); upload(p->arg_cols, d.arg_cols);
      const size_t nt = d.lc_col.size();
      p->lc_val.alloc(nt ? nt : 1);
      h2d(st_, p->lc_val.p, d.lc_val.data(), nt * FRB);
      convert(p->lc_val.p, p->lc_val.p, 0, nt);
      stream_sync(st_);
    } catch (...) {
      r1cs_free(d.r1cs);
      throw;
    }
    // the matrices now live on the device (and, for setup, in the R1cs host copy): drop the parser's copies of the values
    for (int k = 0; k < 3; k++) { std::vector<uint64_t>().swap(d.val[k]); }
    std::vector<uint64_t>().swap(d.lc_val);
    uint64_t h = next_handle_++;
    progs_[h] = std::move(p);
    return h;
  }
  // out: constraints, instance count (incl. one), witness count, arguments, return values, directives, levels, R1CS handle,
  //      extra (directive-only) variables, directives without a device solver, public argument count, schedulable (0/1)
  void prog_info(uint64_t h, uint64_t out[12]) override {
    const ProgData& d = get_prog(h).d;
    uint64_t pub = 0;
    for (uint8_t pr : d.arg_private) pub += pr ? 0 : 1;
    out[0] = d.N; out[1] = d.ni; out[2] = d.nw; out[3] = d.arg_ids.size(); out[4] = d.n_ret; out[5] = d.d_kind.size();
    out[6] = d.n_levels; out[7] = d.r1cs; out[8] = d.m_ext - d.m; out[9] = d.n_unsupported; out[10] = pub;
    out[11] = d.schedule_error.empty() ? 1 : 0;
  }
  void prog_free(uint64_t h) override {
    auto it = progs_.find(h);
    if (it == progs_.end()) throw Error(ZKB_E_ARG, "unknown program handle");
    std::shared_ptr<ProgDev> last = it->second;
    if (last.use_count() == 2) {   // this map entry + `last`: the last handle
      for (auto& sl : slots_)
        if (sl.state != 0 && sl.r1cs == last->d.r1cs) throw Error(ZKB_E_ARG, "a proof that uses this program is in flight (collect it first)");
    }
    progs_.erase(it);
    if (last.use_count() > 1) return;                     // other handles share it
    if (opts.pk_cache && (last->fp[0] | last->fp[1])) {
      if (idle_prog_) r1cs_free(idle_prog_->d.r1cs);
      idle_prog_ = last;                                  // stays resident until another program is loaded
    } else {
      r1cs_free(last->d.r1cs);
    }
  }

  // the refusals of a witness call, before any launch: input count, canonical inputs (K sets of n_inputs), schedulable
  // program, no solver without a device path
  void prog_check_inputs(const ProgData& d, const uint64_t* inputs, uint64_t n_inputs, uint64_t K) {
    if (n_inputs != d.arg_ids.size())
      throw Error(ZKB_E_ARG, "WrongInputCount: expected " + std::to_string(d.arg_ids.size()) + ", received " + std::to_string(n_inputs));
    if (!d.schedule_error.empty()) throw Error(ZKB_E_FORMAT, "program cannot be executed: " + d.schedule_error);
    if (d.n_unsupported) throw Error(ZKB_E_ARG, "the program calls a solver that has no device path (Zir function / embed gadget)");
    uint32_t mod[8];
    fr_modulus(mod);
    for (uint64_t i = 0; i < K * n_inputs; i++)
      if (!prog_detail::canonical((const uint8_t*)(inputs + 4 * i), mod))
        throw Error(ZKB_E_ARG, "input is not a canonical field element" + (K > 1 ? " (input set " + std::to_string(i / n_inputs) + ")" : std::string()));
  }
  static size_t witness_file_len(const ProgData& d) {   // all witness files of one program have this length
    return 8 + 40 * (size_t)std::count(d.defined.begin(), d.defined.end(), (uint8_t)1);
  }

  // The level sweep of K input sets: constraints through witness_level_body, directives through solver_body, one launch each
  // per level whatever K is.  zp: interleaved Montgomery assignments z[col * K + k] (m_ext columns), inputs in place;
  // flag[k] (0xFFFFFFFF on entry) receives set k's first violated row.
  void prog_levels(const ProgDev& p, R1cs& r, uint32_t K, Fr* zp, uint32_t* flag, uint32_t flags) {
    const ProgData& d = p.d;
    const uint32_t* rpA = r.rowptr[0].p; const uint32_t* clA = r.col[0].p; const Fr* vlA = r.val[0].p;
    const uint32_t* rpB = r.rowptr[1].p; const uint32_t* clB = r.col[1].p; const Fr* vlB = r.val[1].p;
    const uint32_t* rpC = r.rowptr[2].p; const uint32_t* clC = r.col[2].p; const Fr* vlC = r.val[2].p;
    const uint32_t* pr = p.rows.p; const uint32_t* po = p.out_var.p; const uint32_t* pd = p.dirs.p;
    const uint32_t* kd = p.kind.p; const uint32_t* ar = p.arg.p; const uint32_t* ip = p.in_ptr.p; const uint32_t* op = p.out_ptr.p;
    const uint32_t* oc = p.out_cols.p; const uint32_t* lp = p.lc_ptr.p; const uint32_t* lc = p.lc_col.p; const Fr* lv = p.lc_val.p;
    for (uint32_t l = 1; l <= d.n_levels; l++) {
      const uint32_t rlo = d.row_level_ptr[l - 1], rhi = d.row_level_ptr[l], dlo = d.dir_level_ptr[l - 1], dhi = d.dir_level_ptr[l];
      if (rhi > rlo)
        launch<k_witness_level>(st_, (size_t)(rhi - rlo) * K, ZKB_LAMBDA(size_t t) {
          witness_level_body<Fr>(rpA, clA, vlA, rpB, clB, vlB, rpC, clC, vlC, zp, pr, po, rlo, rhi, K, flag, (uint32_t)t);
        });
      if (dhi > dlo)
        launch<k_solver_level, 64>(st_, (size_t)(dhi - dlo) * K, ZKB_LAMBDA(size_t t) {
          solver_body<Fr>(kd, ar, ip, op, oc, lp, lc, lv, zp, pd, dlo, dhi, K, flags, (uint32_t)t);
        });
    }
  }

  // inputs: one canonical field element per program argument.  Returns the first unsatisfied constraint or ~0; on success
  // the assignment stays resident in the program's R1CS (zkb_groth16_prove_resident can follow) and `wit_out` receives the
  // witness FILE bytes (ir/witness.rs:44-53) when it is non-null.
  uint64_t prog_compute_witness(uint64_t h, const uint64_t* inputs, uint64_t n_inputs, uint32_t flags, uint8_t* wit_out, size_t cap,
                                size_t* wit_len) override {
    ProgDev& p = get_prog(h);
    const ProgData& d = p.d;
    prog_check_inputs(d, inputs, n_inputs, 1);
    R1cs& r = get_r1cs(d.r1cs);
    std::vector<uint64_t> z((size_t)d.m_ext * 4, 0);
    z[0] = 1;
    for (uint64_t i = 0; i < n_inputs; i++) memcpy(&z[4 * (size_t)d.arg_cols[i]], inputs + 4 * i, 32);
    DevBuf<Fr> zc(d.m_ext), zm(d.m_ext);
    DevBuf<uint32_t> d_flag(1);
    StageTimer tm(st_);
    h2d(st_, zc.p, z.data(), d.m_ext * FRB);
    dev_fill_ff(st_, d_flag.p, 4);
    tm.begin("witness_eval");
    convert(zc.p, zm.p, 0, d.m_ext);
    prog_levels(p, r, 1, zm.p, d_flag.p, flags);
    convert(zm.p, zc.p, 1, d.m_ext);
    tm.end();
    uint32_t first = 0;
    d2h(st_, &first, d_flag.p, 4);
    d2h(st_, z.data(), zc.p, d.m_ext * FRB);
    d2d(st_, r.z_canon.p, zc.p, d.m * FRB);
    stream_sync(st_);
    tm.collect(timings);
    if (first != 0xFFFFFFFFu) return (uint64_t)first;
    r.has_z = true;
    r.sparse_z = assignment_is_sparse(z.data(), d.m);
    p.z_host.assign(z.begin(), z.begin() + (size_t)d.m * 4);
    if (wit_len) *wit_len = witness_file_len(d);
    if (wit_out) {
      std::vector<uint8_t> bytes;
      witness_write(d, z.data(), bytes);
      if (bytes.size() > cap) throw Error(ZKB_E_ARG, "witness buffer too small");
      memcpy(wit_out, bytes.data(), bytes.size());
    }
    return ~0ull;
  }

  // ---- batches of input sets (zkb_prog_compute_witness_batch / zkb_prog_prove_batch)
  // The level schedule, the matrices and the directive tables do not depend on the inputs, so one sweep serves K input sets
  // with every launch K times wider; the assignments come out in the interleaved Montgomery layout the batched SpMV reads.
  // Neither batch call touches the program's resident assignment (z_host, the R1CS's z_canon).

  // most input sets one sweep holds: the 32-bit thread index of its launches (statements x K, columns x K)
  static uint64_t prog_sweep_max(const ProgData& d) {
    const uint64_t widest = std::max<uint64_t>({(uint64_t)d.m_ext, (uint64_t)d.rows.size(), (uint64_t)d.dirs.size(), (uint64_t)d.arg_ids.size() + 1});
    return ((1ull << 32) - 1) / widest;
  }
  // upload K input sets and scatter them into zm = interleaved Montgomery z (m_ext x K, `one` in column 0, every other column
  // zero), then sweep the levels; flag[k] receives set k's first violated row
  void prog_sweep_batch(const ProgDev& p, uint32_t K, const uint64_t* inputs, uint32_t flags, Fr* zm, uint32_t* flag) {
    const ProgData& d = p.d;
    R1cs& r = get_r1cs(d.r1cs);
    const uint32_t n_in = (uint32_t)d.arg_ids.size();
    DevBuf<Fr> din((size_t)K * n_in);
    h2d(st_, din.p, inputs, (size_t)K * n_in * FRB);
    dev_zero(st_, zm, (size_t)K * d.m_ext * FRB);
    dev_fill_ff(st_, flag, (size_t)K * 4);
    const Fr* in = din.p;
    const uint32_t* ac = p.arg_cols.p;
    launch<k_fr_convert>(st_, (size_t)K * (n_in + 1), ZKB_LAMBDA(size_t t) {
      const uint32_t k = (uint32_t)(t % K), i = (uint32_t)(t / K);
      if (i == 0) zm[k] = Fr::one();
      else zm[(size_t)ac[i - 1] * K + k] = Fr::to_mont(in[(size_t)k * n_in + i - 1]);
    });
    prog_levels(p, r, K, zm, flag, flags);
  }
  // one pass of K input sets to the host: z_out gets K canonical assignments of m_ext columns back to back, first[k] set k's
  // first violated row or ~0
  void prog_witness_pass(const ProgDev& p, uint32_t K, const uint64_t* inputs, uint32_t flags, uint64_t* z_out, uint64_t* first) {
    const size_t me = p.d.m_ext;
    DevBuf<Fr> zm(K * me), zc(K * me);
    DevBuf<uint32_t> d_flag(K);
    prog_sweep_batch(p, K, inputs, flags, zm.p, d_flag.p);
    const Fr* zi = zm.p; Fr* zo = zc.p;
    launch<k_fr_convert>(st_, K * me, ZKB_LAMBDA(size_t t) { zo[t] = Fr::from_mont(zi[(t % me) * K + t / me]); });
    std::vector<uint32_t> f(K);
    d2h(st_, f.data(), d_flag.p, (size_t)K * 4);
    d2h(st_, z_out, zc.p, K * me * FRB);
    stream_sync(st_);
    for (uint32_t k = 0; k < K; k++) first[k] = f[k] == 0xFFFFFFFFu ? ~0ull : (uint64_t)f[k];
  }
  // input sets per witness pass: the sweep's thread index, ZKB_OPT_BATCH_PASS_MAX, and free HBM (two m_ext x K vectors)
  uint32_t prog_witness_pass_size(const ProgData& d, uint32_t K) {
    uint64_t kmax = std::min<uint64_t>(K, prog_sweep_max(d));
    if (opts.batch_pass_max > 0) kmax = std::min<uint64_t>(kmax, (uint64_t)opts.batch_pass_max);
#if !defined(ZKB_EMU)
    size_t free_b = 0, total_b = 0;
    ZKB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t reserve = (size_t)1 << 30, per = (2 * (size_t)d.m_ext + d.arg_ids.size()) * FRB + 4;
    const uint64_t fit = free_b > reserve ? (free_b - reserve) / per : 0;
    kmax = std::min<uint64_t>(kmax, fit);
#endif
    if (kmax == 0) throw Error(ZKB_E_OOM, "not even one input set fits in device memory");
    return (uint32_t)kmax;
  }
  // K input sets (K x n_inputs canonical elements) -> K witness files of one length back to back in wit_out; first[k] set k's
  // first violated row (its file zero-filled) or ~0.  Returns whether every set was satisfied.
  bool prog_compute_witness_batch(uint64_t h, uint32_t K, const uint64_t* inputs, uint64_t n_inputs, uint32_t flags, uint8_t* wit_out,
                                  size_t cap, size_t* wit_len, uint64_t* first) override {
    if (K == 0) throw Error(ZKB_E_ARG, "empty batch");
    ProgDev& p = get_prog(h);
    const ProgData& d = p.d;
    prog_check_inputs(d, inputs, n_inputs, K);
    const size_t len = witness_file_len(d);
    if (wit_out && cap < K * len) throw Error(ZKB_E_ARG, "witness buffer too small");
    if (wit_len) *wit_len = len;
    const uint32_t kp = prog_witness_pass_size(d, K);
    std::vector<uint64_t> z((size_t)kp * d.m_ext * 4);
    bool all = true;
    for (uint32_t k0 = 0; k0 < K; k0 += kp) {
      const uint32_t cnt = std::min(kp, K - k0);
      prog_witness_pass(p, cnt, inputs + (size_t)k0 * n_inputs * 4, flags, z.data(), first + k0);
      for (uint32_t k = 0; k < cnt; k++) all &= first[k0 + k] == ~0ull;
      if (!wit_out) continue;
      host_parallel(cnt, [&](uint32_t k) {
        uint8_t* dst = wit_out + (size_t)(k0 + k) * len;
        if (first[k0 + k] != ~0ull) { memset(dst, 0, len); return; }
        std::vector<uint8_t> bytes;
        witness_write(d, z.data() + (size_t)k * d.m_ext * 4, bytes);
        memcpy(dst, bytes.data(), len);
      });
    }
    return all;
  }

  // witness file -> resident assignment of the program's R1CS (what `generate-proof -w witness` reads, generate_proof.rs:161-166)
  void prog_set_witness(uint64_t h, const uint8_t* wit, size_t len) override {
    ProgDev& p = get_prog(h);
    uint32_t mod[8];
    fr_modulus(mod);
    witness_parse(p.d, wit, len, mod, p.z_host);
    set_assignment(p.d.r1cs, p.z_host.data());
  }
  // the current assignment of the program (ark column order), as the last compute_witness / set_witness left it
  void prog_assignment(uint64_t h, uint64_t* z_out, uint64_t cap_elems) override {
    ProgDev& p = get_prog(h);
    if (p.z_host.size() != (size_t)p.d.m * 4) throw Error(ZKB_E_ARG, "the program has no assignment yet");
    if (cap_elems < p.d.m) throw Error(ZKB_E_ARG, "assignment buffer too small");
    memcpy(z_out, p.z_host.data(), p.z_host.size() * 8);
  }
  // the columns of the public inputs: public arguments in declaration order, then the return values ~out_0.. (ir/mod.rs:278-288)
  static std::vector<uint32_t> public_cols(const ProgData& d) {
    std::vector<uint32_t> cols;
    for (size_t i = 0; i < d.arg_ids.size(); i++) if (!d.arg_private[i]) cols.push_back(d.arg_cols[i]);
    for (uint32_t k = 0; k < d.n_ret; k++) {
      const int64_t id = -(int64_t)k - 1;
      uint32_t c = 0;
      for (; c < d.ni; c++) if (d.var_of_col[c] == id) break;
      if (c == d.ni) throw Error(ZKB_E_FORMAT, "return value ~out_" + std::to_string(k) + " does not occur in the constraints");
      cols.push_back(c);
    }
    return cols;
  }
  // public arguments in declaration order, then the return values ~out_0.. (ir/mod.rs:278-288), from the current assignment
  uint64_t prog_public_inputs(uint64_t h, uint64_t* out, uint64_t cap) override {
    ProgDev& p = get_prog(h);
    if (p.z_host.size() != (size_t)p.d.m * 4) throw Error(ZKB_E_ARG, "the program has no assignment yet");
    const std::vector<uint32_t> cols = public_cols(p.d);
    if (out) {
      if (cols.size() > cap) throw Error(ZKB_E_ARG, "public input buffer too small");
      for (size_t i = 0; i < cols.size(); i++) memcpy(out + 4 * i, &p.z_host[4 * (size_t)cols[i]], 32);
    }
    return cols.size();
  }

  // ------------------------------------------------------------------------------ MSM

  // window width of an MSM of n pairs: the table's c, or the cost model's
  static uint32_t plan_c(uint64_t n, uint32_t pre_c) { return pre_c ? pre_c : msm_pick_c(n, C::FR_BITS); }
  static uint32_t plan_w(uint32_t c) { return (C::FR_BITS + 1 + c - 1) / c; }
  // The sorted lists index (pair, window) entries of all proofs and views with uint32 offsets: the largest batch one plan holds
  static uint64_t plan_max_batch(uint64_t n, uint32_t nviews, uint32_t pre_c) {
    const uint64_t per = n * plan_w(plan_c(n, pre_c)) * nviews;
    return per ? ((1ull << 32) - 1) / per : ~0ull;
  }

  // K > 1: a batch of K scalar vectors, vector k at scalars + k * stride (MsmShape)
  void plan_build(MsmPlan& pl, const Fr* scalars, uint64_t n, uint32_t nviews = 1, const uint8_t* skip = nullptr,
                  uint32_t pre_c = 0 /* != 0: precomputed window tables with this c */, uint32_t K = 1, size_t stride = 0) {
    pl.sh.n = (uint32_t)n;
    pl.sh.K = K;
    pl.nviews = nviews;
    pl.sh.pre = pre_c ? 1 : 0;
    if (n == 0) return;
    uint32_t c = plan_c(n, pre_c);
    pl.sh.c = c;
    pl.sh.W = plan_w(c);
    pl.sh.B = 1u << (c - 1);
    pl.nbuckets = msm_nbuckets(pl.sh);
    uint64_t total = (uint64_t)K * n * pl.sh.W;
    if (K == 0 || total * nviews >= (1ull << 32)) throw Error(ZKB_E_ARG, "msm too large");
    // chunk size: aim for several waves of resident threads, at least 8 entries per chunk
    uint64_t target = (uint64_t)opts.chunk_target;
    uint64_t T = (total + target - 1) / target;
    if (T < 8) T = 8;
    if (T > 64) T = 64;
    T = (T + 1) & ~1ull;
    pl.T1 = (uint32_t)T;
    pl.T2 = 8;   // short chunks at the partial levels: fewer dependent additions per level
    pl.nt1 = (uint32_t)((total + pl.T1 - 1) / pl.T1);
    const uint32_t NB = pl.nbuckets;
    if (nviews > 3) throw Error(ZKB_E_INTERNAL, "at most two filtered views");
    pl.digits.ensure(total); pl.ranks.ensure(total); pl.sorted.ensure(total * nviews);
    pl.counts.ensure(NB); pl.offsets.ensure((size_t)(NB + 1) * nviews);
    dev_zero(st_, pl.counts.p, (size_t)NB * 4);
    MsmShape sh = pl.sh;
    const uint32_t* sc = (const uint32_t*)scalars;
    uint32_t* dg = pl.digits.p; uint32_t* rk = pl.ranks.p; uint32_t* cn = pl.counts.p; uint32_t* of = pl.offsets.p;
    uint32_t* so = pl.sorted.p;
    launch<k_msm_digits>(st_, (size_t)K * n, ZKB_LAMBDA(size_t t) { msm_digits_body(sh, sc, stride, dg, rk, cn, (uint32_t)t); });
    const uint32_t ntiles = (uint32_t)((total + VIEW_TILE - 1) / VIEW_TILE);
    pl.scan_tmp.ensure(2 * ((size_t)(NB > ntiles ? NB : ntiles) / 2048 + 4));
    exclusive_scan(st_, cn, of, NB, pl.scan_tmp.p);
    launch<k_msm_scatter>(st_, total, ZKB_LAMBDA(size_t t) { msm_scatter_body(sh, dg, rk, of, so, (uint32_t)t); });
    if (nviews > 1) build_views(pl, skip, total, ntiles);
  }

  // views 1.. = stable compaction of the sorted list of view 0 (kernels above; host loop in the emulation)
  void build_views(MsmPlan& pl, const uint8_t* skip, uint64_t total, uint32_t ntiles) {
    const uint32_t NB = pl.nbuckets, nv = pl.nviews - 1;
    const MsmShape sh = pl.sh;
    const uint32_t* of0 = pl.offsets.p;
    const uint32_t* so0 = pl.sorted.p;
    uint32_t* sov = pl.sorted.p + total;
#if !defined(ZKB_EMU)
    const uint32_t ngroups = (uint32_t)((total + 31) / 32);
    pl.view_tile_cnt.ensure((size_t)2 * ntiles); pl.view_tile_off.ensure((size_t)2 * (ntiles + 1));
    pl.view_pre32.ensure((size_t)2 * ngroups); pl.view_mask32.ensure((size_t)2 * ngroups);
    launch_counter() += 2;
    zkb_view_count<<<ntiles, VIEW_BLOCK, 0, st_.s>>>(sh, skip, so0, of0, NB, pl.view_tile_cnt.p, ntiles);
    ZKB_CUDA(cudaGetLastError());
    for (uint32_t v = 0; v < nv; v++)
      exclusive_scan(st_, pl.view_tile_cnt.p + (size_t)v * ntiles, pl.view_tile_off.p + (size_t)v * (ntiles + 1), ntiles, pl.scan_tmp.p);
    zkb_view_apply<<<ntiles, VIEW_BLOCK, 0, st_.s>>>(sh, skip, so0, of0, NB, nv, pl.view_tile_off.p, ntiles, sov, (size_t)total,
                                                     pl.view_pre32.p, pl.view_mask32.p, ngroups);
    ZKB_CUDA(cudaGetLastError());
    for (uint32_t v = 0; v < nv; v++) {
      const uint32_t* pre = pl.view_pre32.p + (size_t)v * ngroups; const uint32_t* msk = pl.view_mask32.p + (size_t)v * ngroups;
      const uint32_t* tot = pl.view_tile_off.p + (size_t)v * (ntiles + 1) + ntiles;
      uint32_t* ofv = pl.offsets.p + (size_t)(v + 1) * (NB + 1);
      launch<k_msm_view>(st_, (size_t)NB + 1, ZKB_LAMBDA(size_t t) { msm_view_offsets_body(NB, of0, pre, msk, tot, ofv, (uint32_t)t); });
    }
#else
    (void)ntiles;
    const uint32_t M = of0[NB];
    for (uint32_t v = 0; v < nv; v++) {
      uint32_t* ofv = pl.offsets.p + (size_t)(v + 1) * (NB + 1);
      uint32_t* out = sov + (size_t)v * total;
      uint32_t kept = 0, b = 0;
      for (uint32_t p = 0; p <= M; p++) {
        while (b <= NB && of0[b] == p) ofv[b++] = kept;
        if (p < M && msm_view_keep(sh, skip, so0[p], v + 1)) out[kept++] = so0[p];
      }
    }
#endif
  }

  MsmWs ws_misc_;       // standalone zkb_msm_g1 / g2
  // witness map + h-plan run on their own stream underneath the z-dependent MSMs
  Stream wm_stream_, plan_stream_;
  bool has_wm_stream_ = false, has_plan_stream_ = false;
  struct StreamScope {  // temporarily redirect every helper that launches on st_
    Stream& ref; Stream saved;
    StreamScope(Stream& r, Stream s) : ref(r), saved(r) { ref = s; }
    ~StreamScope() { ref = saved; }
  };
  Stream tail_stream(MsmWs& ws) {
    if (!ws.has_stream) { ws.tail = stream_create_high_priority(); ws.has_stream = true; }
    return ws.tail;
  }
  ~Engine() override {
    if (prepared_.fut.valid()) prepared_.fut.wait();
    for (auto& sl : slots_) { if (sl.fm.valid()) sl.fm.wait(); sl.destroy(); }
    ws_misc_.destroy();
    batch_.destroy();
    if (has_wm_stream_) stream_destroy(wm_stream_);
    if (has_plan_stream_) stream_destroy(plan_stream_);
  }

  // scratch of the batch-affine rounds: shared by all MSMs (the accumulations run one after the other on the main stream)
  DevBuf<uint8_t> ba_pts_[2];
  DevBuf<uint32_t> ba_off_[2], ba_cnt_, ba_scan_tmp_;

  // phase 1 (main stream): bucket accumulation of one MSM.  Throughput-bound (INT32 multiply pipe).
  //   optional batch-affine rounds (msm_affine.cuh): every round halves each bucket with affine additions that share one
  //   inversion per block, then the XYZZ chunk accumulation runs on the shortened list.
  template <class F>
  void msm_accumulate(const MsmPlan& pl, const Affine<F>* pts, MsmWs& ws, StageTimer* tm, const char* accum_name, uint32_t view) {
    typedef XYZZ<F> X;
    if (pl.sh.n == 0) return;
    const uint32_t NB = pl.nbuckets;
    ws.buckets.ensure((size_t)NB * sizeof(X));
    X* buckets = (X*)ws.buckets.p;
    const uint32_t* of = pl.offsets.p + (size_t)view * (NB + 1);
    uint64_t bound = (uint64_t)pl.sh.K * pl.sh.n * pl.sh.W;   // upper bound of the list length (the exact length is offsets[NB], on the device)
    const uint32_t* so = pl.sorted.p + (size_t)view * bound;
    uint32_t rounds = 0;
    if (opts.batch_affine > 0 && bound >= ((uint64_t)1 << opts.batch_affine_min_log) && bound < (1ull << 31)) rounds = (uint32_t)opts.batch_affine;
    ws.tail_done.wait(st_);  // the previous proof's tail may still be reading these buffers
    if (tm && accum_name) tm->begin(accum_name);
    const Affine<F>* cur_pts = pts;
    for (uint32_t r = 0; r < rounds; r++) {
      const uint64_t out_bound = (bound + NB) / 2 + 1;     // sum of ceil(L / 2) over at most NB non-empty buckets
      ba_cnt_.ensure(NB); ba_off_[r & 1].ensure((size_t)NB + 1); ba_scan_tmp_.ensure(2 * ((size_t)NB / 2048 + 4));
      ba_pts_[r & 1].ensure(out_bound * sizeof(Affine<F>));
      const uint32_t* off_in = of;
      uint32_t* cnt = ba_cnt_.p; uint32_t* off_out = ba_off_[r & 1].p;
      launch<k_ba_halve>(st_, NB, ZKB_LAMBDA(size_t t) { ba_halve_counts_body(NB, off_in, cnt, (uint32_t)t); });
      exclusive_scan(st_, cnt, off_out, NB, ba_scan_tmp_.p);
      Affine<F>* out = (Affine<F>*)ba_pts_[r & 1].p;
      const uint32_t* srt = so;
      const Affine<F>* pin = cur_pts;
#if !defined(ZKB_EMU)
      {
        constexpr int MINB = sizeof(F) > sizeof(Fq) ? 2 : 3;
        static bool configured = false;                    // per instantiation: opt in to the dynamic shared memory size once
        if (!configured) {
          ZKB_CUDA(cudaFuncSetAttribute(zkb_batch_affine<F, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba_smem_bytes<F>()));
          configured = true;
        }
        const size_t blocks = (size_t)((out_bound + BA_TILE - 1) / BA_TILE);
        launch_counter()++;
        zkb_batch_affine<F, MINB><<<(unsigned)blocks, BA_BLOCK, ba_smem_bytes<F>(), st_.s>>>(NB, off_in, off_out, srt, pin, out);
        ZKB_CUDA(cudaGetLastError());
      }
#else
      {  // the same passes as the device kernel, block after block
        const size_t blocks = (size_t)((out_bound + BA_TILE - 1) / BA_TILE);
        launch_counter()++;
        for (size_t blk = 0; blk < blocks; blk++) ba_block_emulate<F>(NB, off_in, off_out, srt, pin, out, (uint32_t)blk);
      }
#endif
      of = off_out; so = nullptr; cur_pts = out; bound = out_bound;
    }
    // chunk size of the XYZZ stage: several waves of resident threads, 8 .. 64 entries per chunk
    uint32_t T1 = pl.T1, nt1 = pl.nt1;
    if (rounds) {
      uint64_t T = (bound + 600000 - 1) / 600000;
      if (T < 8) T = 8;
      if (T > 64) T = 64;
      T1 = (uint32_t)((T + 1) & ~1ull);
      nt1 = (uint32_t)((bound + T1 - 1) / T1);
    }
    ws.nt1 = nt1;
    for (int k = 0; k < 2; k++) { ws.key[k].ensure(2 * (size_t)nt1 + 2); ws.val[k].ensure((2 * (size_t)nt1 + 2) * sizeof(X)); }
    dev_zero(st_, buckets, (size_t)NB * sizeof(X));
    uint32_t* k0 = ws.key[0].p; X* v0 = (X*)ws.val[0].p;
    const Affine<F>* fin_pts = cur_pts;
    // G2 (Fq2 coordinates) wants > 200 registers: two blocks per SM (more blocks force spills)
    if (sizeof(F) > sizeof(Fq)) {
      launch<k_msm_accum1, 128, ZKB_G2_MINB>(st_, nt1, ZKB_LAMBDA(size_t t) { msm_accum1_body<F>(NB, T1, of, so, fin_pts, buckets, k0, v0, nt1, (uint32_t)t); });
    } else {
      launch<k_msm_accum1>(st_, nt1, ZKB_LAMBDA(size_t t) { msm_accum1_body<F>(NB, T1, of, so, fin_pts, buckets, k0, v0, nt1, (uint32_t)t); });
    }
    if (tm && accum_name) tm->end();
    ws.acc_done.record(st_);
  }

  // Levels of the device bucket reduction: it stops when a proof's windows hold at most host_nodes block totals, so the host
  // share of every proof is the same whatever the batch size.  Returns the XYZZ entries of the result slot (all K proofs).
  template <class F>
  size_t tail_levels(const MsmPlan& pl, uint32_t& cnt, uint32_t& nbits) const {
    const uint32_t Wp = pl.sh.pre ? 1 : pl.sh.W;
    const uint32_t rbits = opts.bitsum_radix == 8 ? 3u : 1u;
    // a G2 addition costs 1.3 us on a host core against 0.45 us in G1, and the G2 tail is never the last to finish:
    // run it further down on the GPU
    const size_t host_nodes = sizeof(F) > sizeof(Fq) ? HOST_TREE_NODES / 8 : HOST_TREE_NODES;
    cnt = pl.sh.B; nbits = 0;
    while (cnt >= (1u << rbits) && (size_t)Wp * cnt > host_nodes) { cnt >>= rbits; nbits += rbits; }
    return (size_t)pl.sh.K * Wp * cnt * (1 + (size_t)nbits);
  }

  // phase 2 (side stream): reduce chunk-boundary partials, then the bucket reduction by bit sums.  Latency-bound
  // (7 dependent point additions per level), so it runs on a high-priority stream underneath the next MSM's accumulation.
  template <class F>
  void msm_tail(const MsmPlan& pl, MsmWs& ws, XYZZ<F>* win_out /* K * MAXW entries */, StageTimer* tm = nullptr, const char* tail_name = nullptr) {
    typedef XYZZ<F> X;
    if (pl.sh.n == 0) return;
    Stream ts = tail_stream(ws);
    ws.acc_done.wait(ts);
    size_t span = (tm && tail_name) ? tm->begin_on(ts, tail_name) : 0;
    // the K bucket sets of a batch are K * W windows to the reduction kernels
    const uint32_t W = (pl.sh.pre ? 1 : pl.sh.W) * pl.sh.K, B = pl.sh.B, T2 = pl.T2, nt1 = ws.nt1;   // chunks of THIS accumulation
    X* buckets = (X*)ws.buckets.p;
    uint32_t L = 2 * nt1;
    int cur = 0;
    while (true) {
      uint32_t nt = L / T2 + 1;
      const uint32_t* ik = ws.key[cur].p; const X* iv = (const X*)ws.val[cur].p;
      uint32_t* ok = ws.key[cur ^ 1].p; X* ov = (X*)ws.val[cur ^ 1].p;
      uint32_t Lc = L;
      launch<k_msm_accum2>(ts, nt, ZKB_LAMBDA(size_t t) { msm_accum2_body<F>(Lc, T2, ik, iv, buckets, ok, ov, nt, (uint32_t)t); });
      if (nt == 1) break;
      L = 2 * nt;
      cur ^= 1;
    }
    // bucket reduction by bit sums (msm.cuh::msm_bitsum2_body / msm_bitsum_body): one launch per level, 1 (radix 2, default)
    // or 7 (radix 8) dependent additions each
    const uint32_t rbits = opts.bitsum_radix == 8 ? 3u : 1u;
    const size_t half = ((size_t)W * B) >> 1;   // largest level output: A' <= W B / 2 entries, pending <= W B / 2 entries
    if (rbits == 3) {
      const size_t first = (size_t)W * (B >> 3);
      ws.tree[0].ensure((first + 1) * sizeof(X)); ws.tree[1].ensure((first / 8 + 1) * sizeof(X));
      ws.tree[2].ensure((3 * first + 1) * sizeof(X)); ws.tree[3].ensure((3 * first + 1) * sizeof(X));
    } else {
      ws.tree[0].ensure((half + 1) * sizeof(X)); ws.tree[1].ensure((half / 2 + 1) * sizeof(X));
      ws.tree[2].ensure((half + 1) * sizeof(X)); ws.tree[3].ensure((half + 1) * sizeof(X));
    }
    const X* inA = buckets; const X* inP = nullptr;
    uint32_t cnt = B, lvl = 0, nbits = 0, end_cnt = 0, end_bits = 0;
    const size_t out_entries = tail_levels<F>(pl, end_cnt, end_bits);
    while (nbits < end_bits) {
      X* oA = (X*)ws.tree[lvl & 1].p; X* oP = (X*)ws.tree[2 + (lvl & 1)].p;
      const X* iA = inA; const X* iP = inP;
      const uint32_t ci = cnt, np = nbits;
      if (rbits == 3) {
        const size_t threads = (size_t)(4 + np) * W * (cnt >> 3);
        launch<k_msm_bitsum>(ts, threads, ZKB_LAMBDA(size_t t) { msm_bitsum_body<F>(W, ci, np, iA, iP, oA, oP, (uint32_t)t); });
      } else {
        const size_t threads = (size_t)(2 + np) * W * (cnt >> 1);
        launch<k_msm_bitsum, 64>(ts, threads, ZKB_LAMBDA(size_t t) { msm_bitsum2_body<F>(W, ci, np, iA, iP, oA, oP, (uint32_t)t); });
      }
      inA = oA; inP = oP; cnt >>= rbits; lvl++; nbits += rbits;
    }
    // result slot: [A : W*cnt][pending 0 : W*cnt] ... [pending nbits-1 : W*cnt]; the host finishes (host_finish)
    ws.tree_cnt = cnt; ws.tree_bits = nbits;
    const size_t nodes = (size_t)W * cnt;
    ws.out_entries = out_entries;
    if (ws.out_entries > (size_t)MAXW * pl.sh.K) throw Error(ZKB_E_INTERNAL, "msm result slot overflow");
    d2d(ts, win_out, inA, nodes * sizeof(X));
    if (nbits) d2d(ts, win_out + nodes, inP, nodes * nbits * sizeof(X));
    if (tm && tail_name) tm->end_on(ts, span);
    ws.tail_done.record(ts);
  }

  template <class F>
  void msm_exec(const MsmPlan& pl, const Affine<F>* pts, XYZZ<F>* win_out, MsmWs& ws, StageTimer* tm = nullptr,
                const char* accum_name = nullptr, uint32_t view = 0, const char* tail_name = nullptr) {
    msm_accumulate<F>(pl, pts, ws, tm, accum_name, view);
    msm_tail<F>(pl, ws, win_out, tm, tail_name);
  }

  // Host finish of one MSM.  Per window: total = sum_k A_k, hi = sum_k k A_k (running sums), S_bit = sum_k P_bit[k];
  //   sum_j (j + 1) B_j = total + sum_bit 2^bit S_bit + 2^nbits hi    (Horner from the top bit),
  // then result = sum_w 2^(c w) (window sum).  A few hundred point additions on a host core.
  static constexpr size_t HOST_TREE_NODES = 32;
  // `proof`: which of the plan's K proofs (its windows are proof * W .. proof * W + W - 1 of every array of the slot)
  template <class HX>
  static HX host_finish(const HX* slot, const MsmPlan& pl, const MsmWs& ws, uint32_t proof = 0) {
    const uint32_t W = pl.sh.pre ? 1 : pl.sh.W, cnt = ws.tree_cnt, nbits = ws.tree_bits, c = pl.sh.c;
    const size_t nodes = (size_t)W * pl.sh.K * cnt, first = (size_t)proof * W * cnt;
    const HX* A = slot + first;
    auto window_sum = [&](uint32_t w) {
      HX run = HX::identity(), hi = HX::identity();
      for (uint32_t k = cnt; k-- > 0;) {
        run = HX::add(run, A[(size_t)w * cnt + k]);
        if (k > 0) hi = HX::add(hi, run);
      }
      for (uint32_t bit = nbits; bit-- > 0;) {
        const HX* P = slot + nodes * (1 + (size_t)bit) + first + (size_t)w * cnt;
        HX sb = HX::identity();
        for (uint32_t k = 0; k < cnt; k++) sb = HX::add(sb, P[k]);
        hi = HX::add(HX::dbl(hi), sb);
      }
      return HX::add(hi, run);   // bucket j holds weight j + 1
    };
    std::vector<HX> S(W);
    if (W >= 8) {   // window mode (sparse witnesses, small MSMs): the per-window sums are independent, four host threads
      auto part = [&](uint32_t q) { for (uint32_t w = q; w < W; w += 4) S[w] = window_sum(w); };
      std::future<void> f1 = std::async(std::launch::async, part, 1u), f2 = std::async(std::launch::async, part, 2u),
                        f3 = std::async(std::launch::async, part, 3u);
      part(0);
      f1.get(); f2.get(); f3.get();
    } else {
      for (uint32_t w = 0; w < W; w++) S[w] = window_sum(w);
    }
    HX acc = HX::identity();
    for (uint32_t w = W; w-- > 0;) {
      if (w + 1 < W) for (uint32_t d = 0; d < c; d++) acc = HX::dbl(acc);
      acc = HX::add(acc, S[w]);
    }
    return acc;
  }

  // ------------------------------------------------------------------------------ proving key
  struct Pk {
    uint64_t ni = 0, m = 0, hl = 0, ll = 0;
    uint32_t rank = 0, world = 1;
    uint64_t lo = 0, hi = 0, hlo = 0, hhi = 0;  // assignment / h index slices of this rank
    DevBuf<G1A> a, b1, l, h;                    // a_query[1+lo..1+hi), b_g1 likewise, l_ext[lo..hi), h_query[hlo..hhi)
    DevBuf<G2A> b2;
    DevBuf<G1A> fixed1;                          // alpha1, beta1, delta1, a_query[0], b_g1_query[0]
    DevBuf<G2A> fixed2;                          // beta2, delta2, b_g2_query[0]
    uint32_t pre_cz = 0, pre_ch = 0;             // != 0: a/b1/b2/l (resp. h) hold W window tables 2^(c w) P (HBM-resident precomputation)
    int z_status = 0, h_status = 0;              // why the tables were (not) built: TAB_* codes, reported by zkb_pk_table_info
    size_t table_bytes = 0;
    DevBuf<uint8_t> skip;                        // per assignment index: bit0 = a_query point is infinity, bit1 = b_query point is infinity
    HG1A h_fixed1[5];                            // host copies (Montgomery form) for the serial tail
    HG2A h_fixed2[3];
    uint64_t fp[2] = {0, 0};                     // content fingerprint (key bytes, shard, table options): the cache key
  };
  // Handles share keys by CONTENT: the reference's `Backend::generate_proof` is static and receives the key bytes on every
  // call (zokrates_ark/src/groth16.rs:40-42), so the trait-shaped use is pk_load / prove / pk_free per proof.  A second load of
  // the same bytes (same shard, same table options) returns a new handle onto the resident key, and the last key released
  // stays resident (`idle_pk_`) until a different key needs the memory — the 0.9 s / 5.6 GB of window tables are built once.
  std::map<uint64_t, std::shared_ptr<Pk>> pks_;
  std::shared_ptr<Pk> idle_pk_;
  // 128-bit fingerprint of the key bytes: four multiply-rotate lanes over 8-byte words (not cryptographic: a cache key for
  // bytes the caller already trusts as its proving key)
  static void fingerprint(const uint8_t* data, size_t len, uint64_t salt, uint64_t out[2]) {
    uint64_t h[4] = {0x9E3779B97F4A7C15ull ^ salt, 0xC2B2AE3D27D4EB4Full + len, 0x165667B19E3779F9ull, 0x27D4EB2F165667C5ull ^ (salt << 17)};
    const uint64_t k1 = 0xff51afd7ed558ccdull, k2 = 0xc4ceb9fe1a85ec53ull;
    size_t i = 0;
    for (; i + 32 <= len; i += 32) {
      uint64_t w[4];
      memcpy(w, data + i, 32);
      for (int l = 0; l < 4; l++) { uint64_t x = (h[l] ^ w[l]) * k1; h[l] = ((x << 29) | (x >> 35)) + k2; }
    }
    uint8_t tail[32] = {0};
    memcpy(tail, data + i, len - i);
    uint64_t w[4];
    memcpy(w, tail, 32);
    for (int l = 0; l < 4; l++) { uint64_t x = (h[l] ^ w[l]) * k2; h[l] = ((x << 31) | (x >> 33)) * k1; }
    auto mix = [&](uint64_t x) { x ^= x >> 33; x *= k1; x ^= x >> 29; x *= k2; x ^= x >> 32; return x; };
    out[0] = mix(h[0] + mix(h[1])) ^ mix(h[2] ^ (h[3] << 1));
    out[1] = mix(h[2] + mix(h[3] ^ k1)) + mix(h[0] ^ (h[1] >> 3));
  }
  // fingerprint of a large buffer on 8 host threads (the pieces are salted with their index, the piece results hashed again):
  // 403 MB in ~8 ms instead of 55 ms, so that the trait-shaped call (load by content, prove, free) stays close to the proof time
  static void fingerprint_par(const uint8_t* data, size_t len, uint64_t salt, uint64_t out[2]) {
    constexpr int PARTS = 8;
    if (len < ((size_t)8 << 20)) { fingerprint(data, len, salt, out); return; }
    uint64_t part[PARTS][2];
    std::vector<std::future<void>> fs;
    const size_t step = ((len / PARTS) + 31) & ~(size_t)31;
    for (int k = 0; k < PARTS; k++) {
      const size_t lo = std::min(len, step * k), hi = k == PARTS - 1 ? len : std::min(len, step * (k + 1));
      fs.push_back(std::async(std::launch::async, [=, &part] { fingerprint(data + lo, hi - lo, salt ^ (0x9E37ull * (k + 1)), part[k]); }));
    }
    for (auto& f : fs) f.get();
    fingerprint((const uint8_t*)part, sizeof part, salt ^ len, out);
  }
  Pk& get_pk(uint64_t h) {
    auto it = pks_.find(h);
    if (it == pks_.end()) throw Error(ZKB_E_ARG, "unknown pk handle");
    return *it->second;
  }

  template <class F>
  void pk_convert(Affine<F>* pts, size_t count) {
    launch<k_pk_convert>(st_, count, ZKB_LAMBDA(size_t t) {
      Affine<F> p = pts[t];
      uint32_t* raw = (uint32_t*)&p;
      const int last = sizeof(Affine<F>) / 4 - 1;
      bool inf = (raw[last] >> 30) & 1u;  // flag bit 6 of the last byte (ark SWFlags::infinity)
      raw[last] &= 0x3FFFFFFFu;
      if (inf) {
        p = Affine<F>::inf();
      } else {
        p.x = F::to_mont(p.x);
        p.y = F::to_mont(p.y);
      }
      pts[t] = p;
    });
  }

  // The query vectors are fixed per key and HBM is large (80 GB on an H100), so keep 2^(c w) P_i for every window w
  // resident when they fit (precompute_tables checks the free memory).  All windows of an MSM then share one bucket set: larger windows (fewer mixed additions per
  // scalar), half as many buckets in total, and no 2^(c w) Horner at the end.
  template <class F>
  void build_table(DevBuf<Affine<F>>& buf, size_t n, uint32_t c, uint32_t W) {
    DevBuf<Affine<F>> tab(n * W);
    const Affine<F>* src = buf.p;
    Affine<F>* dst = tab.p;
    launch<k_msm_table>(st_, n, ZKB_LAMBDA(size_t t) { msm_table_body<F, 16>(src, dst, (uint32_t)n, c, W, (uint32_t)t); });
    stream_sync(st_);
    buf = std::move(tab);
  }
  // Table status codes reported by zkb_pk_table_info (out[6] for the z tables, out[7] for the h table).
  enum { TAB_BUILT = 1, TAB_TOO_SMALL = 2, TAB_NO_MEMORY = 3, TAB_DISABLED = 4, TAB_NO_WINDOW = 5 };
  void precompute_tables(Pk& p) {
    const uint64_t cnt = p.hi - p.lo, hcnt = p.hhi - p.hlo;
    p.z_status = p.h_status = TAB_DISABLED;
    if (opts.tables == 0) return;
    auto plan = [&](uint64_t n, uint32_t& c, uint32_t& W, int& status) {
      c = 0; W = 0;
      if (n < (1ull << opts.table_min_log)) { status = TAB_TOO_SMALL; return; }   // small MSMs are latency-bound; tables buy nothing
      // the search is restricted to W <= 16 (an 8-way shard of 2^20 would otherwise pick c = 15, W = 17 and lose the tables)
      uint32_t cc = opts.table_c ? (uint32_t)opts.table_c : msm_pick_c_pre(n, C::FR_BITS);
      uint32_t ww = cc ? (C::FR_BITS + 1 + cc - 1) / cc : 0;
      if (cc == 0 || ww > 16) { status = TAB_NO_WINDOW; return; }
      c = cc; W = ww; status = TAB_BUILT;
    };
    uint32_t cz, Wz, ch, Wh;
    plan(cnt, cz, Wz, p.z_status);
    plan(hcnt, ch, Wh, p.h_status);
    // HBM budget: the tables must leave room for the sort plans (digits + 3 sorted views: 16 B per (pair, window)), the bucket
    // sets and the witness-map vectors of the circuit this key belongs to, plus 1 GiB of slack.
    const size_t need_z = (size_t)Wz * cnt * (3 * G1B + G2B), need_h = (size_t)Wh * hcnt * G1B;
    const size_t reserve = (size_t)16 * (cnt * (Wz ? Wz : 17) + hcnt * (Wh ? Wh : 17)) + 6 * (p.hl + 1) * FRB + ((size_t)1 << 30);
#if !defined(ZKB_EMU)
    size_t free_b = 0, total_b = 0;
    ZKB_CUDA(cudaMemGetInfo(&free_b, &total_b));
#else
    size_t free_b = ~(size_t)0 >> 1;
#endif
    size_t avail = free_b > reserve ? free_b - reserve : 0;
    auto fits = [&](size_t need, int& status, const char* what) {
      if (status != TAB_BUILT) return false;
      if (need <= avail) { avail -= need; return true; }
      if (opts.tables == 2)
        throw Error(ZKB_E_OOM, std::string("window tables for ") + what + " need " + std::to_string(need >> 20) + " MiB, " +
                                   std::to_string(avail >> 20) + " MiB available (ZKB_OPT_TABLES = 2)");
      status = TAB_NO_MEMORY;
      return false;
    };
    // the z tables serve four MSMs (one of them G2) and come first
    if (fits(need_z, p.z_status, "a/b1/b2/l")) {
      build_table<Fq>(p.a, cnt, cz, Wz); build_table<Fq>(p.b1, cnt, cz, Wz); build_table<Fq>(p.l, cnt, cz, Wz);
      build_table<Fq2>(p.b2, cnt, cz, Wz);
      p.pre_cz = cz;
      p.table_bytes += need_z;
    }
    if (fits(need_h, p.h_status, "h")) { build_table<Fq>(p.h, hcnt, ch, Wh); p.pre_ch = ch; p.table_bytes += need_h; }
  }
  // out: c_z, W_z, c_h, W_h, table bytes, resident key bytes (tables included), z status, h status
  void pk_table_info(uint64_t h, uint64_t out[8]) override {
    Pk& p = get_pk(h);
    auto Wof = [](uint32_t c) -> uint64_t { return c ? (uint64_t)((C::FR_BITS + 1 + c - 1) / c) : 0; };
    out[0] = p.pre_cz; out[1] = Wof(p.pre_cz); out[2] = p.pre_ch; out[3] = Wof(p.pre_ch);
    out[4] = p.table_bytes;
    out[5] = p.a.bytes() + p.b1.bytes() + p.l.bytes() + p.b2.bytes() + p.h.bytes();
    out[6] = (uint64_t)p.z_status; out[7] = (uint64_t)p.h_status;
  }

  uint64_t pk_load(const uint8_t* pk, size_t len, uint32_t rank, uint32_t world) override {
    if (world == 0 || rank >= world) throw Error(ZKB_E_ARG, "bad rank/world");
    uint64_t fp[2] = {0, 0};
    if (opts.pk_cache) {
      const uint64_t salt = ((uint64_t)rank << 48) ^ ((uint64_t)world << 32) ^ ((uint64_t)opts.tables << 24) ^ ((uint64_t)opts.table_c << 16) ^
                            ((uint64_t)opts.table_min_log << 8);
      fingerprint_par(pk, len, salt, fp);
      std::shared_ptr<Pk> hit;
      if (idle_pk_ && idle_pk_->fp[0] == fp[0] && idle_pk_->fp[1] == fp[1]) { hit = idle_pk_; idle_pk_.reset(); }
      else for (auto& kv : pks_) if (kv.second->fp[0] == fp[0] && kv.second->fp[1] == fp[1]) { hit = kv.second; break; }
      if (hit) {
        timings.clear();
        timings.push_back({"pk_cache_hit", 1.0});
        uint64_t h = next_handle_++;
        pks_[h] = hit;
        return h;
      }
    }
    if (idle_pk_) {   // a different key: release the cached one first (its fixed points may still feed host threads)
      for (auto& sl : slots_) if (sl.fm.valid()) sl.fm.wait();
      if (prepared_.fut.valid()) prepared_.fut.wait();
      idle_pk_.reset();
    }
    size_t off = 0;
    auto need = [&](size_t k) { if (off + k > len) throw Error(ZKB_E_FORMAT, "proving key truncated"); };
    auto take = [&](size_t k) { need(k); const uint8_t* p = pk + off; off += k; return p; };
    auto take_len = [&]() { need(8); uint64_t v; memcpy(&v, pk + off, 8); off += 8; return v; };
    const uint8_t* alpha1 = take(G1B);
    const uint8_t* beta2 = take(G2B);
    take(G2B);  // gamma_g2 (verifier only)
    const uint8_t* delta2 = take(G2B);
    uint64_t ni = take_len();
    if (ni > (len - off) / G1B) throw Error(ZKB_E_FORMAT, "gamma_abc length");
    take(ni * G1B);
    const uint8_t* beta1 = take(G1B);
    const uint8_t* delta1 = take(G1B);
    uint64_t m = take_len();
    if (m > (len - off) / G1B) throw Error(ZKB_E_FORMAT, "a_query length");
    const uint8_t* aq = take(m * G1B);
    uint64_t m1 = take_len();
    if (m1 != m) throw Error(ZKB_E_FORMAT, "b_g1_query length differs from a_query");
    const uint8_t* b1q = take(m * G1B);
    uint64_t m2 = take_len();
    if (m2 != m) throw Error(ZKB_E_FORMAT, "b_g2_query length differs from a_query");
    const uint8_t* b2q = take(m * G2B);
    uint64_t hl = take_len();
    if (hl > (len - off) / G1B) throw Error(ZKB_E_FORMAT, "h_query length");
    const uint8_t* hq = take(hl * G1B);
    uint64_t ll = take_len();
    if (ll > (len - off) / G1B) throw Error(ZKB_E_FORMAT, "l_query length");
    const uint8_t* lq = take(ll * G1B);
    if (off != len) throw Error(ZKB_E_FORMAT, "trailing bytes after proving key");
    if (ni < 1 || m < ni || ll != m - ni) throw Error(ZKB_E_FORMAT, "inconsistent query lengths");

    std::shared_ptr<Pk> p(new Pk());
    p->fp[0] = fp[0]; p->fp[1] = fp[1];
    p->ni = ni; p->m = m; p->hl = hl; p->ll = ll; p->rank = rank; p->world = world;
    const uint64_t na = m - 1;  // pairs with assignment = z[1..]
    p->lo = na * rank / world; p->hi = na * (rank + 1) / world;
    p->hlo = hl * rank / world; p->hhi = hl * (rank + 1) / world;
    if (world > 1 && na > 0) {
      // The four z-MSMs share one index range per rank, but a_query / b_query are sparse (variables that never occur in
      // A resp. B are the point at infinity and are skipped) and the sparsity is rarely uniform over the index — in the
      // benchmark circuit 95 % of the non-infinity b points sit in the first half.  Cut the range where the WORK is
      // equal: weight 1 (l) + 1.1 (a != inf) + 4.5 (b != inf: G1 and G2; a G2 addition is 28 / 10 of a G1 addition and runs less efficiently).
      // Every rank derives the same cuts from the same key bytes.
      auto is_inf = [](const uint8_t* pt, size_t bytes) { return (pt[bytes - 1] & 0x40) != 0; };
      std::vector<float> w(na);
      double total = 0;
      for (uint64_t i = 0; i < na; i++) {
        float wi = 1.0f;
        if (!is_inf(aq + (1 + i) * G1B, G1B)) wi += 1.1f;    // measured per-point times relative to l (single GPU, 2^20)
        if (!is_inf(b2q + (1 + i) * G2B, G2B)) wi += 4.5f;
        w[i] = wi;
        total += wi;
      }
      // With three or more ranks the witness-map chains are computed once each by ranks 0, 1, 2 at the head of their main
      // stream (DESIGN.md §6): those ranks get a smaller share of the MSM work so that all ranks reach the h-MSM together.
      // f = one chain's cost as a fraction of the whole MSM work, from a cost model fitted at 2^20 (a chain = 0.19 n
      // log2(n)/20 weight units in BN254, 0.086 in BLS12-381, a weight unit = one G1 point through all windows; BLS12-377 has
      // BLS12-381's limb counts and takes its figure, not re-fitted);
      // ZKB_OPT_CHAIN_SHARE: -1 model (default), 0 equal shares, > 0 f in 1/1000.
      std::vector<double> cum(world + 1, 0.0);
      {
        double f = 0;
        if (world >= 3 && opts.chain_share != 0) {
          const double n_dom = (double)hl + 1, lg = std::log2(n_dom > 2 ? n_dom : 2);
          const double chain_units = (Fq::N > 8 ? 0.086 : 0.19) * n_dom * lg / 20.0;
          f = opts.chain_share > 0 ? opts.chain_share / 1000.0 : chain_units / (total + (double)hl);
          const double fmax = 0.6 / world;                // an owner keeps at least ~40 % of an equal share
          if (f > fmax) f = fmax;
        }
        for (uint32_t k = 0; k < world; k++) cum[k + 1] = cum[k] + (1.0 + 3.0 * f) / world - (k < 3 ? f : 0.0);
        cum[world] = 1.0;
      }
      auto cut = [&](uint32_t k) -> uint64_t {   // first index whose prefix weight reaches this rank's cumulative share
        if (k == 0) return 0;
        if (k >= world) return na;
        const double target = total * cum[k];
        double acc = 0;
        for (uint64_t i = 0; i < na; i++) { if (acc >= target) return i; acc += w[i]; }
        return na;
      };
      p->lo = cut(rank); p->hi = cut(rank + 1);
      p->hlo = (uint64_t)((double)hl * cum[rank]); p->hhi = rank + 1 == world ? hl : (uint64_t)((double)hl * cum[rank + 1]);
    }
    const uint64_t cnt = p->hi - p->lo, hcnt = p->hhi - p->hlo;
    p->a.alloc(cnt); p->b1.alloc(cnt); p->l.alloc(cnt); p->b2.alloc(cnt); p->h.alloc(hcnt);
    h2d(st_, p->a.p, aq + (1 + p->lo) * G1B, cnt * G1B);
    h2d(st_, p->b1.p, b1q + (1 + p->lo) * G1B, cnt * G1B);
    h2d(st_, p->b2.p, b2q + (1 + p->lo) * G2B, cnt * G2B);
    h2d(st_, p->h.p, hq + p->hlo * G1B, hcnt * G1B);
    // l_ext[j] = infinity for j < ni - 1, else l_query[j - (ni - 1)]   (aux = assignment[ni-1..])
    {
      const uint64_t shift = ni - 1;
      dev_zero(st_, p->l.p, cnt * G1B);
      uint64_t j0 = p->lo > shift ? p->lo : shift;  // first assignment index with a real l point
      if (j0 < p->hi) h2d(st_, p->l.p + (j0 - p->lo), lq + (j0 - shift) * G1B, (p->hi - j0) * G1B);
    }
    p->fixed1.alloc(5); p->fixed2.alloc(3);
    std::vector<uint8_t> inf1(G1B, 0), inf2(G2B, 0);
    inf1[G1B - 1] = 0x40; inf2[G2B - 1] = 0x40;
    h2d(st_, p->fixed1.p + 0, alpha1, G1B);
    h2d(st_, p->fixed1.p + 1, beta1, G1B);
    h2d(st_, p->fixed1.p + 2, delta1, G1B);
    h2d(st_, p->fixed1.p + 3, m ? aq : inf1.data(), G1B);
    h2d(st_, p->fixed1.p + 4, m ? b1q : inf1.data(), G1B);
    h2d(st_, p->fixed2.p + 0, beta2, G2B);
    h2d(st_, p->fixed2.p + 1, delta2, G2B);
    h2d(st_, p->fixed2.p + 2, m ? b2q : inf2.data(), G2B);
    pk_convert<Fq>(p->a.p, cnt); pk_convert<Fq>(p->b1.p, cnt); pk_convert<Fq>(p->h.p, hcnt);
    pk_convert<Fq2>(p->b2.p, cnt); pk_convert<Fq>(p->fixed1.p, 5); pk_convert<Fq2>(p->fixed2.p, 3);
    {  // l_ext: only the uploaded part carries raw bytes; zero-filled prefix is already "infinity"
      const uint64_t shift = ni - 1;
      uint64_t j0 = p->lo > shift ? p->lo : shift;
      if (j0 < p->hi) pk_convert<Fq>(p->l.p + (j0 - p->lo), p->hi - j0);
    }
    {  // infinity flags of the a / b query slices -> filtered MSM views (ark's mixed add skips infinity bases too)
      p->skip.alloc(cnt ? cnt : 1);
      uint8_t* fl = p->skip.p;
      const G1A* pa = p->a.p; const G1A* pb = p->b1.p;
      launch<k_pk_convert>(st_, cnt, ZKB_LAMBDA(size_t t) { fl[t] = (uint8_t)((pa[t].is_inf() ? 1 : 0) | (pb[t].is_inf() ? 2 : 0)); });
    }
    precompute_tables(*p);
    d2h(st_, p->h_fixed1, p->fixed1.p, 5 * G1B);
    d2h(st_, p->h_fixed2, p->fixed2.p, 3 * G2B);
    stream_sync(st_);
    uint64_t h = next_handle_++;
    pks_[h] = std::move(p);
    return h;
  }
  void pk_info(uint64_t h, uint64_t out[4]) override {
    Pk& p = get_pk(h);
    out[0] = p.ni; out[1] = p.m; out[2] = p.hl; out[3] = p.ll;
  }
  void pk_free(uint64_t h) override {
    for (auto& sl : slots_) {
      if (sl.state != 0 && sl.pk == h) throw Error(ZKB_E_ARG, "a proof that uses this key is in flight (collect it first)");
      if (sl.fm.valid()) sl.fm.wait();     // a finished proof's host multiplications may still read the key's fixed points
    }
    if (prepared_.pk == h) { if (prepared_.fut.valid()) prepared_.fut.wait(); prepared_.pk = 0; }
    auto it = pks_.find(h);
    if (it == pks_.end()) throw Error(ZKB_E_ARG, "unknown pk handle");
    std::shared_ptr<Pk> last = it->second;
    pks_.erase(it);
    if (opts.pk_cache && last.use_count() == 1 && (last->fp[0] | last->fp[1])) idle_pk_ = last;   // the last handle: stay resident

  }

  // ------------------------------------------------------------------------------ prove
  DevBuf<Fr> scratch_a_, scratch_b_;
  static constexpr uint32_t MAXW = 1024;  // result slot entries per MSM: (1 + 3 levels) * W * tree_cnt <= 19 * 32

  struct HostPartial {  // same layout as Partial
    HG1X h, l, a, b1;
    HG2X b2;
  };
  static_assert(sizeof(HostPartial) == sizeof(Partial), "partial layout");

  // sample the assignment: a witness dominated by 0/1 values (hash circuits) makes the z MSMs nearly free, and the
  // proof time is then set by the reduction tails — the windows mode (16 x 2^15 buckets) has the shallower reduction.
  static bool assignment_is_sparse(const uint64_t* z, uint64_t m) {
    const uint64_t step = m > 4096 ? m / 4096 : 1;
    uint64_t small = 0, cnt = 0;
    for (uint64_t i = 0; i < m; i += step, cnt++) small += (z[4 * i + 1] | z[4 * i + 2] | z[4 * i + 3]) == 0;
    return cnt && small * 2 > cnt;
  }

  bool z_window_mode(bool sparse) const { return opts.z_mode == 2 || (opts.z_mode == 0 && sparse); }

  // One proof's device work is ENQUEUED in two steps and COLLECTED in a third, so that (a) the host can exchange witness-map
  // chains between the ranks in the middle and (b) two proofs can be in flight (ProofSlot):
  //   begin  : upload z, start the chains of `chain_mask` on the witness-map stream, the z plan and the four z-MSMs on the
  //            main stream; if some chains are left to other ranks, wait until this rank's chains are complete
  //   finish : (all three chain buffers hold coset evaluations) rest of the witness map, h plan, h-MSM; a side stream waits
  //            for the five reduction tails and copies their results to pinned host memory.  Returns without synchronising.
  //   collect: waits for that copy, runs the host part of the reductions, returns the five partial sums.
  // zkb_groth16_prove_partial = begin(all chains) + finish + collect;  zkb_groth16_prove_submit = begin + finish.
  uint64_t open_ticket_ = 0;     // the proof opened by the legacy zkb_groth16_prove_begin

  ProofSlot& slot_of(uint64_t ticket) {
    for (auto& sl : slots_)
      if (sl.state != 0 && sl.ticket == ticket) return sl;
    throw Error(ZKB_E_ARG, "unknown proof ticket");
  }
  Stream fin_stream(ProofSlot& sl) {
    if (!sl.has_fin) { sl.fin = stream_create_high_priority(); sl.has_fin = true; }
    return sl.fin;
  }

  static constexpr uint32_t CHAIN_NO_HOST_SYNC = 0x80000000u;   // chain_mask flag: the caller orders the exchange with stream events
  uint64_t slot_begin(uint64_t pkh, uint64_t rh, const uint64_t* z, uint32_t chain_mask_in) {
    const bool no_host_sync = (chain_mask_in & CHAIN_NO_HOST_SYNC) != 0;
    const uint32_t chain_mask = chain_mask_in & ~CHAIN_NO_HOST_SYNC;
    Pk& pk = get_pk(pkh);
    R1cs& r = get_r1cs(rh);
    const size_t n = (size_t)1 << r.log_n;
    if (pk.m != r.m || pk.ni != r.ni) throw Error(ZKB_E_ARG, "proving key does not match the R1CS (variable counts)");
    if (pk.hl + 1 != n) throw Error(ZKB_E_ARG, "proving key does not match the R1CS (domain size)");
    if (chain_mask > 7) throw Error(ZKB_E_ARG, "chain_mask");
    ProofSlot* free_slot = nullptr;
    for (auto& c : slots_) if (c.state == 0) { free_slot = &c; break; }
    if (!free_slot) throw Error(ZKB_E_ARG, "two proofs are already in flight on this context (collect one first)");
    ProofSlot& sl = *free_slot;
    if (!z && !r.has_z) throw Error(ZKB_E_ARG, "no resident assignment");
    slot_vectors(sl, r);
    sl.tm.reset(new StageTimer(st_));
    StageTimer& tm = *sl.tm;
    if (z) {
      tm.begin("h2d_z");
      h2d(st_, sl.z_canon.p, z, r.m * FRB);
      tm.end();
      sl.z_src = sl.z_canon.p;
      sl.sparse_z = assignment_is_sparse(z, r.m);
    } else {
      sl.z_src = r.z_canon.p;
      sl.sparse_z = r.sparse_z;
    }
    const size_t slot1 = MAXW * sizeof(G1X), slot2 = MAXW * sizeof(G2X);
    sl.d_win.ensure(4 * slot1 + slot2);
    sl.hw.ensure(4 * slot1 + slot2);
    G1X* w_l = (G1X*)(sl.d_win.p + slot1);
    G1X* w_a = (G1X*)(sl.d_win.p + 2 * slot1);
    G1X* w_b1 = (G1X*)(sl.d_win.p + 3 * slot1);
    G2X* w_b2 = (G2X*)(sl.d_win.p + 4 * slot1);
    // The witness map (3 SpMV, 7 NTT, latency/bandwidth-bound at this size) and the h digit plan go to a second
    // (high-priority) stream and fill the multiply-pipe bubbles of the z-dependent MSMs running on the main stream.
    if (!has_wm_stream_) { wm_stream_ = stream_create_high_priority(); has_wm_stream_ = true; }
    sl.tm2.reset(new StageTimer(wm_stream_));
    sl.ev_z_ready.record(st_);                       // the assignment is in place (uploaded on the main stream, or resident)
    // The digit / sort plan of the z-dependent MSMs needs nothing but z: it runs on its own stream, so that with two proofs in
    // flight it overlaps the PREVIOUS proof's accumulate kernels (memory- and atomic-bound work under multiply-bound work)
    // instead of heading the main stream.  Measured: no gain (17.47 vs 17.46 ms per proof) — the GPU is work-bound and the
    // overlapped plan slows the accumulate kernels by what it saves; kept as an option, off by default.
    const uint32_t pre_c_z = z_window_mode(sl.sparse_z) ? 0 : pk.pre_cz;
    if (opts.plan_stream) {
      if (!has_plan_stream_) { plan_stream_ = stream_create_high_priority(); has_plan_stream_ = true; }
      const size_t span = tm.begin_on(plan_stream_, "msm_plan_z");
      StreamScope sc(st_, plan_stream_);
      sl.ev_z_ready.wait(st_);
      plan_build(sl.plan_z, sl.z_src + 1 + pk.lo, pk.hi - pk.lo, 3, pk.skip.p, pre_c_z);
      tm.end_on(plan_stream_, span);
      sl.ev_plan_z.record(st_);
    }
    if (chain_mask == 7) {   // replicated witness map: underneath the z-dependent MSMs
      StreamScope sc(st_, wm_stream_);
      sl.ev_z_ready.wait(st_);
      wm_chains(r, sl, chain_mask, *sl.tm2);
      sl.ev_chains_done.record(st_);
    } else {
      // shared witness map: the other ranks wait for this rank's chains, so they run FIRST and alone on the main stream
      // (0.5 ms with the GPU to themselves; underneath the accumulate kernels they took twice as long and h arrived
      // late: wait_h 1.1 ms at 8 GPUs).  The exchange and the finish step then hide under this rank's z-dependent MSMs.
      wm_chains(r, sl, chain_mask, tm);
      sl.ev_chains_done.record(st_);
    }
    if (opts.plan_stream) {
      tm.begin("wait_plan_z");
      sl.ev_plan_z.wait(st_);
      tm.end();
    } else {
      tm.begin("msm_plan_z");
      plan_build(sl.plan_z, sl.z_src + 1 + pk.lo, pk.hi - pk.lo, 3, pk.skip.p, pre_c_z);
      tm.end();
    }
    msm_exec<Fq2>(sl.plan_z, pk.b2.p, w_b2, sl.ws[4], &tm, "accum1_g2_b2", 2, "tail_g2_b2");
    msm_exec<Fq>(sl.plan_z, pk.l.p, w_l, sl.ws[1], &tm, "accum1_g1_l", 0, "tail_g1_l");
    msm_exec<Fq>(sl.plan_z, pk.a.p, w_a, sl.ws[2], &tm, "accum1_g1_a", 1, "tail_g1_a");
    msm_exec<Fq>(sl.plan_z, pk.b1.p, w_b1, sl.ws[3], &tm, "accum1_g1_b1", 2, "tail_g1_b1");
    sl.pk = pkh; sl.r1cs = rh; sl.ticket = next_ticket_++; sl.state = 1; sl.has_rs = false;
    // chains left to other ranks: the caller exchanges buffers next, so this rank's chains must be complete in memory
    if (chain_mask != 7 && !no_host_sync) sl.ev_chains_done.sync();   // the host exchanges the buffers next: wait for the chains only
    return sl.ticket;
  }

  void slot_finish(ProofSlot& sl) {
    if (sl.state != 1) throw Error(ZKB_E_ARG, "proof is not open");
    Pk& pk = get_pk(sl.pk);
    R1cs& r = get_r1cs(sl.r1cs);
    StageTimer& tm = *sl.tm;
    StageTimer& tm2 = *sl.tm2;
    const size_t slot1 = MAXW * sizeof(G1X);
    G1X* w_h = (G1X*)sl.d_win.p;
    {
      StreamScope sc(st_, wm_stream_);
      wm_finish(r, sl.a.p, sl.b.p, sl.c.p, sl.h.p, 1, tm2, "witness_map_finish");
      tm2.begin("msm_plan_h");
      plan_build(sl.plan_h, sl.h.p + pk.hlo, pk.hhi - pk.hlo, 1, nullptr, pk.pre_ch);
      tm2.end();
      sl.ev_h_ready.record(st_);
    }
    tm.begin("wait_h");
    sl.ev_h_ready.wait(st_);
    tm.end();
    msm_exec<Fq>(sl.plan_h, pk.h.p, w_h, sl.ws[0], &tm, "accum1_g1_h", 0, "tail_g1_h");
    // the rest happens OFF the main stream, so the next proof's plan and accumulate kernels follow at once
    Stream fs = fin_stream(sl);
    sl.ws[0].acc_done.wait(fs);
    size_t span = tm.begin_on(fs, "tails_wait");
    for (int k = 0; k < 5; k++) sl.ws[k].tail_done.wait(fs);
    tm.end_on(fs, span);
    span = tm.begin_on(fs, "d2h_windows");
    {  // only the entries each tail produced (tree_cnt block totals + the pending bit-sum arrays)
      const size_t offs[5] = {0, slot1, 2 * slot1, 3 * slot1, 4 * slot1};
      const size_t esz[5] = {sizeof(G1X), sizeof(G1X), sizeof(G1X), sizeof(G1X), sizeof(G2X)};
      const MsmPlan* pls[5] = {&sl.plan_h, &sl.plan_z, &sl.plan_z, &sl.plan_z, &sl.plan_z};
      for (int k = 0; k < 5; k++)
        if (pls[k]->sh.n) d2h(fs, sl.hw.p + offs[k], sl.d_win.p + offs[k], sl.ws[k].out_entries * esz[k]);
    }
    tm.end_on(fs, span);
    sl.done.record(fs);
    sl.state = 2;
  }

  void slot_collect(ProofSlot& sl, uint8_t* partial_out) {
    if (sl.state != 2) throw Error(ZKB_E_ARG, "proof is not fully enqueued (zkb_groth16_prove_end first)");
    const size_t slot1 = MAXW * sizeof(G1X);
    try {
      sl.done.sync();             // everything this proof enqueued on any stream precedes `done`
      sl.tm->collect(timings);
      std::vector<std::pair<const char*, double>> t2;
      sl.tm2->collect(t2);
      for (auto& e : t2) timings.push_back(e);
    } catch (...) {
      sl.state = 0;
      throw;
    }
    HostPartial hp;
    const uint8_t* hw = sl.hw.p;
    const auto t_host0 = std::chrono::steady_clock::now();
    // five independent host reductions (a few hundred point additions each): one thread per MSM
    auto hor1 = [&](size_t k, const MsmPlan& pl) {
      return pl.sh.n ? host_finish<HG1X>((const HG1X*)(hw + k * slot1), pl, sl.ws[k]) : HG1X::identity();
    };
    auto f_b2 = std::async(std::launch::async, [&] {
      return sl.plan_z.sh.n ? host_finish<HG2X>((const HG2X*)(hw + 4 * slot1), sl.plan_z, sl.ws[4]) : HG2X::identity();
    });
    auto f_h = std::async(std::launch::async, [&] { return hor1(0, sl.plan_h); });
    auto f_l = std::async(std::launch::async, [&] { return hor1(1, sl.plan_z); });
    auto f_a = std::async(std::launch::async, [&] { return hor1(2, sl.plan_z); });
    hp.b1 = hor1(3, sl.plan_z);
    hp.h = f_h.get(); hp.l = f_l.get(); hp.a = f_a.get(); hp.b2 = f_b2.get();
    timings.push_back({"host_tree_finish", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host0).count()});
    memcpy(partial_out, &hp, sizeof hp);
    sl.state = 0;
  }

  // ---- legacy two-call form (one open proof), used by the multi-GPU chain exchange
  void prove_begin(uint64_t pkh, uint64_t rh, const uint64_t* z, uint32_t chain_mask, void* chain_ptrs[3],
                   uint64_t* chain_bytes) override {
    if (open_ticket_) throw Error(ZKB_E_ARG, "a proof is already open on this context (call zkb_groth16_prove_end)");
    const uint64_t t = slot_begin(pkh, rh, z, chain_mask);
    open_ticket_ = t;
    ProofSlot& sl = slot_of(t);
    if (chain_ptrs) { chain_ptrs[0] = sl.a.p; chain_ptrs[1] = sl.b.p; chain_ptrs[2] = sl.c.p; }
    if (chain_bytes) *chain_bytes = ((size_t)1 << get_r1cs(rh).log_n) * FRB;
  }
  void prove_end(uint64_t pkh, uint64_t rh, uint8_t* partial_out) override {
    if (!open_ticket_) throw Error(ZKB_E_ARG, "zkb_groth16_prove_end without a matching prove_begin");
    ProofSlot& sl = slot_of(open_ticket_);
    if (sl.pk != pkh || sl.r1cs != rh) throw Error(ZKB_E_ARG, "zkb_groth16_prove_end without a matching prove_begin");
    open_ticket_ = 0;
    try {
      slot_finish(sl);
    } catch (...) {
      sl.state = 0;
      throw;
    }
    slot_collect(sl, partial_out);
  }
  // ---- pipelined form: enqueue now, collect later (two proofs may be in flight)
  uint64_t prove_begin_async(uint64_t pkh, uint64_t rh, const uint64_t* z, uint32_t chain_mask, void* chain_ptrs[3],
                             uint64_t* chain_bytes) override {
    const uint64_t t = slot_begin(pkh, rh, z, chain_mask);
    ProofSlot& sl = slot_of(t);
    if (chain_ptrs) { chain_ptrs[0] = sl.a.p; chain_ptrs[1] = sl.b.p; chain_ptrs[2] = sl.c.p; }
    if (chain_bytes) *chain_bytes = ((size_t)1 << get_r1cs(rh).log_n) * FRB;
    return t;
  }
  // Stream-ordered chain exchange (no host synchronisation): the caller's stream (NCCL / torch) waits for this rank's chains,
  // runs its broadcasts, and the finish step waits for whatever that stream has enqueued by then.
  void prove_chains_to_stream(uint64_t ticket, void* ext_stream) override {
#if !defined(ZKB_EMU)
    ProofSlot& sl = slot_of(ticket);
    Stream ext; ext.s = (cudaStream_t)ext_stream;
    sl.ev_chains_done.wait(ext);
#else
    (void)ticket; (void)ext_stream;
#endif
  }
  void prove_stream_to_finish(uint64_t ticket, void* ext_stream) override {
#if !defined(ZKB_EMU)
    ProofSlot& sl = slot_of(ticket);
    Stream ext; ext.s = (cudaStream_t)ext_stream;
    if (!has_wm_stream_) throw Error(ZKB_E_INTERNAL, "no witness-map stream");
    sl.ev_exchange.record(ext);
    sl.ev_exchange.wait(wm_stream_);
#else
    (void)ticket; (void)ext_stream;
#endif
  }
  void prove_end_async(uint64_t ticket) override {
    ProofSlot& sl = slot_of(ticket);
    try {
      slot_finish(sl);
    } catch (...) {
      sl.state = 0;
      throw;
    }
  }
  uint64_t prove_submit(uint64_t pkh, uint64_t rh, const uint64_t* z, const uint64_t* r, const uint64_t* s) override {
    const uint64_t t = slot_begin(pkh, rh, z, 7);
    ProofSlot& sl = slot_of(t);
    try {
      slot_finish(sl);
    } catch (...) {
      sl.state = 0;
      throw;
    }
    if (r && s) {
      // r*d1, s*d1, rs*d1, s*d2 need nothing from the GPU: host threads compute them underneath the kernels
      memcpy(sl.r, r, 32); memcpy(sl.s, s, 32);
      sl.has_rs = true;
      const Pk* pkp = &get_pk(pkh);
      const uint32_t* rr = sl.r; const uint32_t* ss = sl.s;
      sl.fm = std::async(std::launch::async, [pkp, rr, ss] { return fixed_mults(*pkp, rr, ss); });
    }
    return t;
  }
  void prove_collect_partial(uint64_t ticket, uint8_t* partial_out) override {
    ProofSlot& sl = slot_of(ticket);
    if (sl.fm.valid()) sl.fm.wait();
    slot_collect(sl, partial_out);
  }
  void prove_collect(uint64_t ticket, uint8_t* proof_out) override {
    ProofSlot& sl = slot_of(ticket);
    if (!sl.has_rs) throw Error(ZKB_E_ARG, "zkb_groth16_prove_collect needs r and s at submit time");
    const Pk& pk = get_pk(sl.pk);
    std::vector<uint8_t> partial(sizeof(HostPartial));
    try {
      slot_collect(sl, partial.data());
    } catch (...) {
      if (sl.fm.valid()) sl.fm.wait();
      throw;
    }
    const auto t0 = std::chrono::steady_clock::now();
    FixedMults fm = sl.fm.get();
    finalize_with(pk, fm, partial.data(), 1, sl.r, sl.s, proof_out);
    timings.push_back({"host_final_combine", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count()});
  }

  void prove_partial(uint64_t pkh, uint64_t rh, const uint64_t* z, uint8_t* partial_out) override {
    const uint64_t t = prove_submit(pkh, rh, z, nullptr, nullptr);
    slot_collect(slot_of(t), partial_out);
  }

  static FixedMults fixed_mults(const Pk& pk, const uint32_t* r, const uint32_t* s) {
    FixedMults f;
    HFr a, b;
    memcpy(a.v, r, 32); memcpy(b.v, s, 32);
    HFr rs = HFr::mul(HFr::to_mont(a), b);  // canonical r * s
    // four independent scalar multiplications (0.12 ms each in G1, 0.35 ms in G2): one host thread each
    auto f_sd2 = std::async(std::launch::async, [&] { return HG2X::mul_affine(pk.h_fixed2[1], s, 8); });
    auto f_rd = std::async(std::launch::async, [&] { return HG1X::mul_affine(pk.h_fixed1[2], r, 8); });
    auto f_sd = std::async(std::launch::async, [&] { return HG1X::mul_affine(pk.h_fixed1[2], s, 8); });
    f.rsd = HG1X::mul_affine(pk.h_fixed1[2], (const uint32_t*)rs.v, 8);
    f.rd = f_rd.get(); f.sd = f_sd.get(); f.sd2 = f_sd2.get();
    return f;
  }

  void finalize_with(const Pk& pk, const FixedMults& fm, const uint8_t* partials, uint32_t world, const uint32_t* r,
                     const uint32_t* s, uint8_t* proof_out) {
    HostPartial sum;
    sum.h = HG1X::identity(); sum.l = HG1X::identity(); sum.a = HG1X::identity(); sum.b1 = HG1X::identity();
    sum.b2 = HG2X::identity();
    for (uint32_t k = 0; k < world; k++) {
      HostPartial p;
      memcpy(&p, partials + (size_t)k * sizeof(HostPartial), sizeof p);
      sum.h = HG1X::add(sum.h, p.h); sum.l = HG1X::add(sum.l, p.l); sum.a = HG1X::add(sum.a, p.a);
      sum.b1 = HG1X::add(sum.b1, p.b1); sum.b2 = HG2X::add(sum.b2, p.b2);
    }
    // A = r d1 + a_0 + <a, z> + alpha1 ; B1, B2 likewise (fixed1: alpha1, beta1, delta1, a_0, b1_0; fixed2: beta2, delta2, b2_0)
    HG1X ga = HG1X::madd(HG1X::madd(HG1X::add(fm.rd, sum.a), pk.h_fixed1[3]), pk.h_fixed1[0]);
    HG1X gb1 = HG1X::madd(HG1X::madd(HG1X::add(fm.sd, sum.b1), pk.h_fixed1[4]), pk.h_fixed1[1]);
    HG2X gb2 = HG2X::madd(HG2X::madd(HG2X::add(fm.sd2, sum.b2), pk.h_fixed2[2]), pk.h_fixed2[0]);
    // C = s A + r B1 - r s d1 + L + H.  The two variable-base multiplications and the G2 normalisation are
    // independent: three host threads.
    auto fut_u2 = std::async(std::launch::async, [&gb1, r] { return HG1X::mul_xyzz(gb1, r, 8); });
    auto fut_pb = std::async(std::launch::async, [&gb2] { return HG2X::to_affine(gb2); });
    HG1X gc = HG1X::mul_xyzz(ga, s, 8);
    HG1A pa = HG1X::to_affine(ga);
    gc = HG1X::add(gc, fut_u2.get());
    gc = HG1X::add(gc, HG1X::neg(fm.rsd));
    gc = HG1X::add(gc, sum.l);
    gc = HG1X::add(gc, sum.h);
    HG1A pc = HG1X::to_affine(gc);
    HG2A pb = fut_pb.get();
    write_proof(proof_out, pa, pb, pc);
  }
  // A | B | C in ark's uncompressed encoding: canonical affine coordinates, and the point at infinity as zero coordinates with
  // the infinity flag (bit 6 of the point's last byte)
  static void write_proof(uint8_t* out, const HG1A& pa, const HG2A& pb, const HG1A& pc) {
    auto put = [&](size_t slot, const HFq& v) { HFq c = HFq::from_mont(v); memcpy(out + slot * FQB, c.v, FQB); };
    put(0, pa.x); put(1, pa.y); put(2, pb.x.c0); put(3, pb.x.c1); put(4, pb.y.c0); put(5, pb.y.c1); put(6, pc.x); put(7, pc.y);
    if (pa.is_inf()) out[G1B - 1] |= 0x40;
    if (pb.is_inf()) out[G1B + G2B - 1] |= 0x40;
    if (pc.is_inf()) out[2 * G1B + G2B - 1] |= 0x40;
  }

  // Multi-GPU: the rank that will finalize may announce (pk, r, s) before it starts its own share of the proof; the four
  // scalar multiplications that depend on nothing else then run on host threads underneath the GPU work.
  struct Prepared {
    uint64_t pk = 0;
    uint32_t r[8], s[8];
    std::future<FixedMults> fut;
  } prepared_;
  void finalize_prepare(uint64_t pkh, const uint64_t* r, const uint64_t* s) override {
    Pk& pk = get_pk(pkh);
    if (prepared_.pk && prepared_.fut.valid()) prepared_.fut.wait();
    prepared_.pk = pkh;
    memcpy(prepared_.r, r, 32); memcpy(prepared_.s, s, 32);
    const Pk* pkp = &pk;
    const uint32_t* rr = prepared_.r; const uint32_t* ss = prepared_.s;
    prepared_.fut = std::async(std::launch::async, [pkp, rr, ss] { return fixed_mults(*pkp, rr, ss); });
  }

  void finalize(uint64_t pkh, const uint8_t* partials, uint32_t world, const uint64_t* r, const uint64_t* s,
                uint8_t* proof_out) override {
    Pk& pk = get_pk(pkh);
    if (world == 0) throw Error(ZKB_E_ARG, "world");
    FixedMults fm;
    if (prepared_.pk == pkh && prepared_.fut.valid() && !memcmp(prepared_.r, r, 32) && !memcmp(prepared_.s, s, 32)) {
      fm = prepared_.fut.get();
      prepared_.pk = 0;
    } else {
      fm = fixed_mults(pk, (const uint32_t*)r, (const uint32_t*)s);
    }
    finalize_with(pk, fm, partials, world, (const uint32_t*)r, (const uint32_t*)s, proof_out);
  }

  void prove_full(uint64_t pkh, uint64_t rh, const uint64_t* z, const uint64_t* r, const uint64_t* s,
                  uint8_t* proof_out) override {
    const uint64_t t = prove_submit(pkh, rh, z, r, s);
    prove_collect(t, proof_out);
  }

  // ------------------------------------------------------------------------------ batch of proofs (zkb_groth16_prove_batch)
  // K proofs of one circuit under one key share the key, its window tables, the matrices and the domain; only the
  // assignments differ.  So a PASS of K proofs is one set of launches: one SpMV over all K assignments, transforms of all 3K
  // chain vectors at once, and MSM plans with a batch dimension (K bucket sets keyed k * NB + bucket over the shared points,
  // MsmShape).  The host tails of the K proofs (the last additions of each MSM, r / s multiples, final combination) run in
  // parallel on host threads.
  struct BatchState {
    DevBuf<Fr> zc, zm, v, h;    // assignments (canonical, back to back; Montgomery, interleaved), 3K chains, K h vectors
    MsmPlan plan_z, plan_h;
    MsmWs ws[5];                // h, l, a, b1, b2
    DevBuf<uint8_t> d_win;      // the K x 5 result slots, packed
    HostBuf hw;
    void destroy() { for (auto& w : ws) w.destroy(); }
    size_t device_bytes() const {
      size_t b = zc.bytes() + zm.bytes() + v.bytes() + h.bytes() + d_win.bytes();
      for (const MsmPlan* p : {&plan_z, &plan_h})
        b += p->digits.bytes() + p->ranks.bytes() + p->counts.bytes() + p->offsets.bytes() + p->sorted.bytes() + p->scan_tmp.bytes() +
             p->view_tile_cnt.bytes() + p->view_tile_off.bytes() + p->view_pre32.bytes() + p->view_mask32.bytes();
      for (const MsmWs& w : ws) {
        b += w.buckets.bytes();
        for (int k = 0; k < 2; k++) b += w.val[k].bytes() + w.key[k].bytes();
        for (int k = 0; k < 4; k++) b += w.tree[k].bytes();
      }
      return b;
    }
  } batch_;
  // From this domain size on a batch gains nothing over the two-slot pipeline (which overlaps the witness map with the MSMs
  // and each proof's host tail with the next proof's kernels), so prove_batch drives the slots instead; so it does for a
  // single proof.  Measured on H100: batches gain up to 2^17, break even at 2^18 and lose at 2^20 (DESIGN.md §7).
  static constexpr uint32_t BATCH_SLOTS_MIN_LOG = 18;
  static constexpr int SPMV_GROUP = 4;   // assignments per thread of the batched SpMV

  // device bytes of one pass of K proofs (the buffers BatchState grows to, plus `extra` per proof), an upper estimate
  size_t batch_bytes(const Pk& pk, const R1cs& rc, uint64_t K, uint32_t pre_c_z, size_t extra) const {
    const uint64_t n = 1ull << rc.log_n;
    size_t bytes = (size_t)K * ((2 * rc.m + 4 * n) * FRB + extra);
    auto plan = [&](uint64_t cnt, uint32_t nviews, uint32_t pre_c, std::initializer_list<size_t> xs) -> size_t {
      if (!cnt) return 0;
      const uint32_t c = plan_c(cnt, pre_c), W = plan_w(c);
      const uint64_t NB = K * (pre_c ? 1ull : W) << (c - 1), tot = K * cnt * W;
      uint64_t T = (tot + opts.chunk_target - 1) / opts.chunk_target;
      T = T < 8 ? 8 : T > 64 ? 64 : T;
      const uint64_t nt1 = (tot + T - 1) / T;
      size_t b = (size_t)tot * 4 * (2 + nviews) + (size_t)NB * 4 * (1 + nviews);
      for (size_t x : xs) b += (size_t)NB * x * 11 / 4 + 2 * (2 * nt1 + 2) * (4 + x);   // buckets + reduction levels, partials
      return b;
    };
    bytes += plan(pk.hi - pk.lo, 3, pre_c_z, {sizeof(G1X), sizeof(G1X), sizeof(G1X), sizeof(G2X)});
    bytes += plan(pk.hhi - pk.hlo, 1, pk.pre_ch, {sizeof(G1X)});
    return bytes;
  }
  // proofs per pass: the uint32 bound of the sorted lists, ZKB_OPT_BATCH_PASS_MAX, and what fits in free HBM
  uint32_t batch_pass_size(const Pk& pk, const R1cs& rc, uint32_t K, uint32_t pre_c_z, size_t extra = 0) {
    uint64_t kmax = std::min<uint64_t>(plan_max_batch(pk.hi - pk.lo, 3, pre_c_z), plan_max_batch(pk.hhi - pk.hlo, 1, pk.pre_ch));
    if (opts.batch_pass_max > 0) kmax = std::min<uint64_t>(kmax, (uint64_t)opts.batch_pass_max);
    kmax = std::min<uint64_t>(kmax, K);
    if (kmax == 0) throw Error(ZKB_E_ARG, "msm too large");
#if !defined(ZKB_EMU)
    size_t free_b = 0, total_b = 0;
    ZKB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t reserve = (size_t)1 << 30, have = free_b + batch_.device_bytes();
    const size_t avail = have > reserve ? have - reserve : 0;
    for (size_t need = batch_bytes(pk, rc, kmax, pre_c_z, extra); kmax > 1 && need > avail; need = batch_bytes(pk, rc, kmax, pre_c_z, extra))
      kmax = std::max<uint64_t>(1, std::min<uint64_t>(kmax - 1, (uint64_t)((double)kmax * avail / need)));
#endif
    return (uint32_t)kmax;
  }

  template <class Fn>
  static void host_parallel(uint32_t count, Fn fn) {   // fn(k) for k < count on up to one host thread per core
    uint32_t P = std::thread::hardware_concurrency();
    P = std::max(1u, std::min(P ? P : 4u, count));
    std::vector<std::future<void>> fs;
    for (uint32_t q = 1; q < P; q++) fs.push_back(std::async(std::launch::async, [&fn, q, P, count] { for (uint32_t k = q; k < count; k += P) fn(k); }));
    for (uint32_t k = 0; k < count; k += P) fn(k);
    for (auto& f : fs) f.get();
  }

  // the refusals of a batch of proofs, before any launch
  void batch_check(uint32_t K, const Pk& pk, const R1cs& rc) {
    if (K == 0) throw Error(ZKB_E_ARG, "empty batch");
    if (pk.m != rc.m || pk.ni != rc.ni) throw Error(ZKB_E_ARG, "proving key does not match the R1CS (variable counts)");
    if (pk.hl + 1 != ((uint64_t)1 << rc.log_n)) throw Error(ZKB_E_ARG, "proving key does not match the R1CS (domain size)");
    if (pk.world != 1) throw Error(ZKB_E_ARG, "a batch needs a key loaded whole (world = 1)");
    for (auto& sl : slots_)
      if (sl.state != 0) throw Error(ZKB_E_ARG, "a proof is in flight on this context (collect it first)");
  }

  void prove_batch(uint64_t pkh, uint64_t rh, uint32_t K, const uint64_t* z, const uint64_t* r, const uint64_t* s,
                   uint8_t* proofs_out) override {
    if (K == 0) throw Error(ZKB_E_ARG, "empty batch");
    Pk& pk = get_pk(pkh);
    R1cs& rc = get_r1cs(rh);
    batch_check(K, pk, rc);
    const size_t zw = (size_t)rc.m * 4, pb = 8 * FQB;    // words per assignment, bytes per proof
    if (rc.log_n >= BATCH_SLOTS_MIN_LOG || K == 1) {     // large circuits and single proofs: the two-slot pipeline
      uint64_t prev = 0;
      try {
        for (uint32_t k = 0; k < K; k++) {
          const uint64_t t = prove_submit(pkh, rh, z + k * zw, r + 4 * (size_t)k, s + 4 * (size_t)k);
          if (k) prove_collect(prev, proofs_out + (k - 1) * pb);
          prev = t;
        }
        prove_collect(prev, proofs_out + (K - 1) * pb);
      } catch (...) {
        std::vector<uint8_t> sink(pb);
        for (auto& sl : slots_)
          if (sl.state == 2) { try { prove_collect(sl.ticket, sink.data()); } catch (...) { sl.state = 0; } }
        throw;
      }
      return;
    }
    // one z-MSM mode for the whole batch, from a sample of its assignments
    uint32_t sampled = 0, sparse = 0;
    for (uint32_t i = 0; i < std::min(K, 8u); i++, sampled++) sparse += assignment_is_sparse(z + (size_t)i * K / std::min(K, 8u) * zw, rc.m);
    const uint32_t pre_c_z = z_window_mode(2 * sparse > sampled) ? 0 : pk.pre_cz;
    const uint32_t kp = batch_pass_size(pk, rc, K, pre_c_z);
    std::vector<std::pair<const char*, double>> all, part;
    for (uint32_t k0 = 0; k0 < K; k0 += kp) {
      const uint32_t cnt = std::min(kp, K - k0);
      batch_pass(pk, rc, cnt, z + k0 * zw, r + 4 * (size_t)k0, s + 4 * (size_t)k0, pre_c_z, proofs_out + k0 * pb, part);
      all.insert(all.end(), part.begin(), part.end());
    }
    timings = all;
  }

  // z == nullptr: the pass's assignments are already in batch_.zc (canonical, back to back) and batch_.zm (Montgomery,
  // interleaved with stride K), written by prog_prove_batch's witness sweep
  void batch_pass(const Pk& pk, R1cs& rc, uint32_t K, const uint64_t* z, const uint64_t* r, const uint64_t* s, uint32_t pre_c_z,
                  uint8_t* proofs_out, std::vector<std::pair<const char*, double>>& times) {
    BatchState& b = batch_;
    DomainT& d = domain(rc.log_n);
    const uint32_t lg = rc.log_n;
    const size_t n = (size_t)1 << lg, m = rc.m;
    // r * d1, s * d1, rs * d1 and s * d2 need nothing from the GPU: host threads compute them underneath the kernels
    std::vector<FixedMults> fms(K);
    std::future<void> fm_all = std::async(std::launch::async, [&] {
      host_parallel(K, [&](uint32_t k) { fms[k] = fixed_mults(pk, (const uint32_t*)(r + 4 * (size_t)k), (const uint32_t*)(s + 4 * (size_t)k)); });
    });
    b.zc.ensure(K * m); b.zm.ensure(K * m); b.v.ensure(3 * K * n); b.h.ensure(K * n);
    StageTimer tm(st_);
    if (z) {
      tm.begin("h2d_z_batch");
      h2d(st_, b.zc.p, z, K * m * FRB);
      tm.end();
    }
    tm.begin("witness_map_batch");
    {
      const Fr* zc = b.zc.p; Fr* zm = b.zm.p;
      if (z) launch<k_fr_convert>(st_, K * m, ZKB_LAMBDA(size_t t) { zm[(t % m) * K + t / m] = Fr::to_mont(zc[t]); });
      const uint32_t* rpA = rc.rowptr[0].p; const uint32_t* clA = rc.col[0].p; const Fr* vlA = rc.val[0].p;
      const uint32_t* rpB = rc.rowptr[1].p; const uint32_t* clB = rc.col[1].p; const Fr* vlB = rc.val[1].p;
      const uint32_t* rpC = rc.rowptr[2].p; const uint32_t* clC = rc.col[2].p; const Fr* vlC = rc.val[2].p;
      Fr* v = b.v.p;
      const uint32_t N = (uint32_t)rc.N, ni = (uint32_t)rc.ni, ngroups = (K + SPMV_GROUP - 1) / SPMV_GROUP;
      // thread (matrix, group of assignments, row): the row index runs fastest, so the output stores are coalesced
      launch<k_spmv>(st_, 3 * (size_t)ngroups * n, ZKB_LAMBDA(size_t t) {
        const uint32_t row = (uint32_t)(t & (n - 1)), q = (uint32_t)(t >> lg), kind = q / ngroups, g = q % ngroups;
        const uint32_t* rp = kind == 0 ? rpA : kind == 1 ? rpB : rpC;
        const uint32_t* cl = kind == 0 ? clA : kind == 1 ? clB : clC;
        const Fr* vl = kind == 0 ? vlA : kind == 1 ? vlB : vlC;
        spmv_batch_body<Fr, SPMV_GROUP>(rp, cl, vl, zm, K, g * SPMV_GROUP, v + (size_t)kind * K * n, n, N, kind == 0 ? ni : 0, row);
      });
      ntt_dif(v, d.tw_inv.p, lg, 3 * K);
      ntt_dit(v, d.tw_fwd.p, lg, d.cos_fwd.p, 3 * K);   // coset shift fused into the first pass, as in wm_chains
      wm_finish(rc, v, v + K * n, v + 2 * K * n, b.h.p, K, tm, "witness_map_finish_batch");
    }
    tm.end();
    tm.begin("msm_plan_z_batch");
    plan_build(b.plan_z, b.zc.p + 1 + pk.lo, pk.hi - pk.lo, 3, pk.skip.p, pre_c_z, K, m);
    tm.end();
    tm.begin("msm_plan_h_batch");
    plan_build(b.plan_h, b.h.p + pk.hlo, pk.hhi - pk.hlo, 1, nullptr, pk.pre_ch, K, n);
    tm.end();
    // result slots of the five MSMs (h, l, a, b1: G1; b2: G2), packed so that one copy brings all of them to the host
    uint32_t tc, tb;
    const size_t ez = b.plan_z.sh.n ? tail_levels<Fq>(b.plan_z, tc, tb) : 0, ez2 = b.plan_z.sh.n ? tail_levels<Fq2>(b.plan_z, tc, tb) : 0;
    const size_t eh = b.plan_h.sh.n ? tail_levels<Fq>(b.plan_h, tc, tb) : 0;
    const size_t off[6] = {0, eh * sizeof(G1X), (eh + ez) * sizeof(G1X), (eh + 2 * ez) * sizeof(G1X), (eh + 3 * ez) * sizeof(G1X),
                           (eh + 3 * ez) * sizeof(G1X) + ez2 * sizeof(G2X)};
    b.d_win.ensure(off[5]);
    b.hw.ensure(off[5]);
    uint8_t* dw = b.d_win.p;
    msm_exec<Fq2>(b.plan_z, pk.b2.p, (G2X*)(dw + off[4]), b.ws[4], &tm, "accum1_g2_b2_batch", 2, "tail_g2_b2_batch");
    msm_exec<Fq>(b.plan_z, pk.l.p, (G1X*)(dw + off[1]), b.ws[1], &tm, "accum1_g1_l_batch", 0, "tail_g1_l_batch");
    msm_exec<Fq>(b.plan_z, pk.a.p, (G1X*)(dw + off[2]), b.ws[2], &tm, "accum1_g1_a_batch", 1, "tail_g1_a_batch");
    msm_exec<Fq>(b.plan_z, pk.b1.p, (G1X*)(dw + off[3]), b.ws[3], &tm, "accum1_g1_b1_batch", 2, "tail_g1_b1_batch");
    msm_exec<Fq>(b.plan_h, pk.h.p, (G1X*)(dw + off[0]), b.ws[0], &tm, "accum1_g1_h_batch", 0, "tail_g1_h_batch");
    for (auto& w : b.ws) w.tail_done.wait(st_);
    tm.begin("d2h_windows_batch");
    d2h(st_, b.hw.p, dw, off[5]);
    tm.end();
    stream_sync(st_);
    tm.collect(times);
    fm_all.get();
    const auto t0 = std::chrono::steady_clock::now();
    const uint8_t* hw = b.hw.p;
    host_parallel(K, [&](uint32_t k) {
      HostPartial hp;
      auto g1 = [&](int slot, const MsmPlan& pl) { return pl.sh.n ? host_finish<HG1X>((const HG1X*)(hw + off[slot]), pl, b.ws[slot], k) : HG1X::identity(); };
      hp.h = g1(0, b.plan_h); hp.l = g1(1, b.plan_z); hp.a = g1(2, b.plan_z); hp.b1 = g1(3, b.plan_z);
      hp.b2 = b.plan_z.sh.n ? host_finish<HG2X>((const HG2X*)(hw + off[4]), b.plan_z, b.ws[4], k) : HG2X::identity();
      finalize_with(pk, fms[k], (const uint8_t*)&hp, 1, (const uint32_t*)(r + 4 * (size_t)k), (const uint32_t*)(s + 4 * (size_t)k),
                    proofs_out + (size_t)k * 8 * FQB);
    });
    times.push_back({"host_tails_batch", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count()});
  }

  // Inputs -> K proofs of one program under one key, the assignments resident on the device between witness generation
  // and proving.  Below BATCH_SLOTS_MIN_LOG (K > 1) the witness sweep of a pass writes straight into the batch buffers:
  // columns [0, m) of its interleaved z are batch_.zm's layout (directive-only columns sit at m .. m_ext), one kernel fills
  // the canonical batch_.zc and the public columns, and batch_pass proves from there.  Otherwise the witnesses go to the host
  // and prove_batch drives the two-slot pipeline.  public_out: K x (public inputs) elements; a set whose witness fails gets
  // first[k] = its first violated row and zero-filled proof and public slots.  Returns whether every set was satisfied.
  bool prog_prove_batch(uint64_t ph, uint64_t pkh, uint32_t K, const uint64_t* inputs, uint64_t n_inputs, uint32_t flags,
                        const uint64_t* r, const uint64_t* s, uint8_t* proofs_out, uint64_t* public_out, uint64_t public_cap,
                        uint64_t* first) override {
    if (K == 0) throw Error(ZKB_E_ARG, "empty batch");
    ProgDev& p = get_prog(ph);
    const ProgData& d = p.d;
    Pk& pk = get_pk(pkh);
    R1cs& rc = get_r1cs(d.r1cs);
    batch_check(K, pk, rc);
    prog_check_inputs(d, inputs, n_inputs, K);
    const std::vector<uint32_t> pub = public_cols(d);
    const size_t np = pub.size(), pb = 8 * FQB, me = d.m_ext, m = d.m, ni = d.ni;
    if (public_out && public_cap < K * np) throw Error(ZKB_E_ARG, "public input buffer too small");
    auto finish = [&](uint32_t k, const uint64_t* zk) {   // set k's public inputs from its assignment, or zeroed slots
      if (first[k] != ~0ull) {
        memset(proofs_out + (size_t)k * pb, 0, pb);
        if (public_out) memset(public_out + (size_t)k * np * 4, 0, np * FRB);
      } else if (public_out) {
        for (size_t i = 0; i < np; i++) memcpy(public_out + ((size_t)k * np + i) * 4, zk + 4 * (size_t)pub[i], 32);
      }
    };
    if (rc.log_n >= BATCH_SLOTS_MIN_LOG || K == 1) {
      std::vector<uint64_t> zall((size_t)K * m * 4);
      const uint32_t kw = prog_witness_pass_size(d, K);
      std::vector<uint64_t> z((size_t)kw * me * 4);
      for (uint32_t k0 = 0; k0 < K; k0 += kw) {
        const uint32_t cnt = std::min(kw, K - k0);
        prog_witness_pass(p, cnt, inputs + (size_t)k0 * n_inputs * 4, flags, z.data(), first + k0);
        for (uint32_t k = 0; k < cnt; k++) memcpy(&zall[(size_t)(k0 + k) * m * 4], &z[(size_t)k * me * 4], m * FRB);
      }
      prove_batch(pkh, d.r1cs, K, zall.data(), r, s, proofs_out);
      bool all = true;
      for (uint32_t k = 0; k < K; k++) { finish(k, &zall[(size_t)k * m * 4]); all &= first[k] == ~0ull; }
      return all;
    }
    // pass size: what fits in either z-MSM mode, with the wider interleaved z, the inputs and the public columns per proof
    const size_t extra = (me - m + n_inputs + ni) * FRB + 4;
    uint32_t kp = std::min(batch_pass_size(pk, rc, K, pk.pre_cz, extra), batch_pass_size(pk, rc, K, 0, extra));
    kp = (uint32_t)std::min<uint64_t>(kp, prog_sweep_max(d));
    // one z-MSM mode for the whole batch, from the assignments prove_batch would sample.  Several passes: the sampled sets
    // are swept first; one pass: they are read back from its sweep.
    const uint32_t ns = std::min(K, 8u);
    std::vector<uint32_t> sample(ns);
    for (uint32_t i = 0; i < ns; i++) sample[i] = (uint32_t)((size_t)i * K / ns);
    int pre_c_z = -1;
    if (kp < K) {
      std::vector<uint64_t> sin((size_t)ns * n_inputs * 4), sz((size_t)ns * me * 4), sf(ns);
      for (uint32_t i = 0; i < ns; i++) memcpy(&sin[(size_t)i * n_inputs * 4], inputs + (size_t)sample[i] * n_inputs * 4, n_inputs * FRB);
      prog_witness_pass(p, ns, sin.data(), flags, sz.data(), sf.data());
      uint32_t sparse = 0;
      for (uint32_t i = 0; i < ns; i++) sparse += assignment_is_sparse(&sz[(size_t)i * me * 4], m);
      pre_c_z = z_window_mode(2 * sparse > ns) ? 0 : (int)pk.pre_cz;
      kp = batch_pass_size(pk, rc, K, (uint32_t)pre_c_z, extra);
      kp = (uint32_t)std::min<uint64_t>(kp, prog_sweep_max(d));
    }
    BatchState& b = batch_;
    std::vector<std::pair<const char*, double>> all_t, part;
    std::vector<uint64_t> hpub, zs(m * 4);
    std::vector<uint32_t> f;
    bool all = true;
    for (uint32_t k0 = 0; k0 < K; k0 += kp) {
      const uint32_t cnt = std::min(kp, K - k0);
      b.zc.ensure((size_t)cnt * m); b.zm.ensure((size_t)cnt * me);
      DevBuf<uint32_t> d_flag(cnt);
      DevBuf<Fr> d_pub((size_t)cnt * ni);
      prog_sweep_batch(p, cnt, inputs + (size_t)k0 * n_inputs * 4, flags, b.zm.p, d_flag.p);
      const Fr* zi = b.zm.p; Fr* zo = b.zc.p; Fr* po = d_pub.p;
      launch<k_fr_convert>(st_, (size_t)cnt * m, ZKB_LAMBDA(size_t t) {
        const size_t k = t / m, col = t % m;
        const Fr v = Fr::from_mont(zi[col * cnt + k]);
        zo[t] = v;
        if (col < ni) po[k * ni + col] = v;
      });
      f.resize(cnt); hpub.resize((size_t)cnt * ni * 4);
      d2h(st_, f.data(), d_flag.p, (size_t)cnt * 4);
      d2h(st_, hpub.data(), d_pub.p, (size_t)cnt * ni * FRB);
      stream_sync(st_);
      for (uint32_t k = 0; k < cnt; k++) first[k0 + k] = f[k] == 0xFFFFFFFFu ? ~0ull : (uint64_t)f[k];
      if (pre_c_z < 0) {   // the whole batch is this pass
        uint32_t sparse = 0;
        for (uint32_t i = 0; i < ns; i++) {
          d2h(st_, zs.data(), b.zc.p + (size_t)sample[i] * m, m * FRB);
          stream_sync(st_);
          sparse += assignment_is_sparse(zs.data(), m);
        }
        pre_c_z = z_window_mode(2 * sparse > ns) ? 0 : (int)pk.pre_cz;
      }
      batch_pass(pk, rc, cnt, nullptr, r + 4 * (size_t)k0, s + 4 * (size_t)k0, (uint32_t)pre_c_z, proofs_out + k0 * pb, part);
      all_t.insert(all_t.end(), part.begin(), part.end());
      for (uint32_t k = 0; k < cnt; k++) { finish(k0 + k, &hpub[(size_t)k * ni * 4]); all &= first[k0 + k] == ~0ull; }
    }
    timings = all_t;
    return all;
  }

  // ------------------------------------------------------------------------------ standalone MSM (tests / microbench)
  DevBuf<uint8_t> msm_pts_, d_win_;
  DevBuf<Fr> msm_scalars_;
  MsmPlan plan_misc_;

  template <class F, class HF>
  void msm_t(const uint8_t* points, const uint64_t* scalars, uint64_t n, uint8_t* out) {
    typedef Affine<F> A;
    typedef XYZZ<F> X;
    typedef XYZZ<HF> HX;
    typedef Affine<HF> HA;
    StageTimer tm(st_);
    msm_pts_.ensure(n * sizeof(A) + 16);
    msm_scalars_.ensure(n + 1);
    d_win_.ensure(MAXW * sizeof(X));
    A* pts = (A*)msm_pts_.p;
    h2d(st_, pts, points, n * sizeof(A));
    h2d(st_, msm_scalars_.p, scalars, n * FRB);
    pk_convert<F>(pts, n);
    tm.begin("msm_plan");
    plan_build(plan_misc_, msm_scalars_.p, n);
    tm.end();
    tm.begin("msm_exec");
    msm_exec<F>(plan_misc_, pts, (X*)d_win_.p, ws_misc_, &tm, "accum1");
    ws_misc_.tail_done.wait(st_);
    tm.end();
    std::vector<uint8_t> hw(MAXW * sizeof(X));
    d2h(st_, hw.data(), d_win_.p, ws_misc_.out_entries * sizeof(X));
    stream_sync(st_);
    tm.collect(timings);
    HX res = n ? host_finish<HX>((const HX*)hw.data(), plan_misc_, ws_misc_) : HX::identity();
    HA a = HX::to_affine(res);
    const size_t words = sizeof(A) / 4;
    uint32_t* o = (uint32_t*)out;
    if (a.is_inf()) {
      memset(out, 0, sizeof(A));
      o[words - 1] = 0x40000000u;
    } else {
      HA c{HF::from_mont(a.x), HF::from_mont(a.y)};
      memcpy(out, &c, sizeof(A));
    }
  }
  void msm(int group, const uint8_t* points, const uint64_t* scalars, uint64_t n, uint8_t* out) override {
    if (group == 1) msm_t<Fq, HFq>(points, scalars, n, out);
    else if (group == 2) msm_t<Fq2, HFq2>(points, scalars, n, out);
    else throw Error(ZKB_E_ARG, "group");
  }

  // ------------------------------------------------------------------------------ field ops
  template <class F>
  void field_op_t(int op, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n) {
    DevBuf<F> da(n), db(n), dc(n);
    h2d(st_, da.p, a, n * sizeof(F));
    if (b) h2d(st_, db.p, b, n * sizeof(F)); else dev_zero(st_, db.p, n * sizeof(F));
    F* pa = da.p; F* pb = db.p; F* pc = dc.p;
    launch<k_field_op>(st_, n, ZKB_LAMBDA(size_t t) {
      F x = F::to_mont(pa[t]), y = F::to_mont(pb[t]), r;
      switch (op) {
        case 0: r = F::mul(x, y); break;
        case 1: r = F::add(x, y); break;
        case 2: r = F::sub(x, y); break;
        default: r = F::inv(x); break;
      }
      pc[t] = F::from_mont(r);
    });
    d2h(st_, out, pc, n * sizeof(F));
    stream_sync(st_);
  }
  void field_op(int field, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n) override {
    if (op < 0 || op > 3) throw Error(ZKB_E_ARG, "op");
    if (field == 0) field_op_t<Fr>(op, a, b, out, n);
    else if (field == 1) field_op_t<Fq>(op, a, b, out, n);
    else throw Error(ZKB_E_ARG, "field");
  }

  // ------------------------------------------------------------------------------ GM17 (see gm17.cuh)
  struct Gm17Pk {
    uint64_t ni = 0, nv = 0, nh = 0;            // instance count (incl. one), SAP variables (incl. one), |g_gamma2_z_t|
    DevBuf<G1A> a, c1, c2, gz;                  // a_query[1..], c_query_1, c_query_2[1..], g_gamma2_z_t
    DevBuf<G2A> b;                              // b_query[1..]
    HG1A h1[6];                                 // a_query[0], c_query_2[0], g_gamma_z, g_ab_gamma_z, g_gamma2_z2, g_gamma2_z_t[0]
    HG2A h2[2];                                 // b_query[0], h_gamma_z
  };
  std::map<uint64_t, std::unique_ptr<Gm17Pk>> gm17_pks_;
  uint64_t gm17_pk_load(const uint8_t* pk, size_t len) override;
  void gm17_pk_free(uint64_t h) override { if (!gm17_pks_.erase(h)) throw Error(ZKB_E_ARG, "unknown gm17 pk handle"); }
  template <class F, class HX> HX gm17_msm(const Fr* scalars, const Affine<F>* pts, uint64_t n, bool replan);
  void gm17_prove(uint64_t pk, uint64_t r1cs, const uint64_t* z, const uint64_t* d1, const uint64_t* d2, const uint64_t* r,
                  uint8_t* proof_out) override;
  size_t gm17_setup_size(uint64_t rh) override;
  void gm17_setup(uint64_t rh, const uint64_t* trapdoor6, uint8_t* pk_out, size_t cap, size_t* len) override;

  // ------------------------------------------------------------------------------ setup (see setup.cuh)
  template <class F> void fb_build(FixedBase<F>& fb, Affine<F> stdgen, const uint32_t* gk);
  template <class F> void fb_emit(const FixedBase<F>& fb, const Fr* scalars, size_t count, uint32_t* dst);
  size_t setup_size(uint64_t rh) override;
  void setup(uint64_t rh, const uint64_t* trapdoor7, uint8_t* pk_out, size_t cap, size_t* len) override;

 protected:
  Stream st_;
};

}  // namespace zkb
