// Radix-2 NTT over the scalar field and the pointwise steps of the QAP witness map.
//
// Replaces ark-poly 0.3.0 `Radix2EvaluationDomain::{fft,ifft,coset_fft,coset_ifft}_in_place` and
// `divide_by_vanishing_poly_on_coset_in_place` as used by ark-groth16's
// `LibsnarkReduction::witness_map` (external, Cargo.lock:282,221; reached from
// /root/reference/zokrates_ark/src/groth16.rs:44; SURVEY.md §8 row a4, App. B.2).  The domain
// generator is ark's: omega = TWO_ADIC_ROOT^(2^(S - log n)), coset shift g = multiplicative generator.
//
// Schedule: decimation-in-frequency passes (natural -> bit-reversed) for the inverse transforms and
// decimation-in-time passes (bit-reversed -> natural) for the forward coset transforms, so no
// bit-reversal pass is needed between ifft and coset_fft.  Each pass does up to 3 butterfly stages
// on 8 elements held in registers (one read + one write of the vector per pass); twiddles come from
// a per-domain table of omega^k, k < n/2, built once on the device.
#pragma once
#include "fp.cuh"

namespace zkb {

ZKB_HD uint32_t bitrev32(uint32_t x, uint32_t bits) {
#if defined(__CUDA_ARCH__)
  return bits ? (__brev(x) >> (32 - bits)) : 0;
#else
  uint32_t r = 0;
  for (uint32_t i = 0; i < bits; i++) r |= ((x >> i) & 1u) << (bits - 1 - i);
  return r;
#endif
}

// tw[k] = w^k for k < count (w given in Montgomery form); each thread exponentiates independently.
template <class Fr>
ZKB_HDN inline void ntt_powers_body(Fr w, Fr scale, Fr* out, uint32_t count, uint32_t t) {
  if (t >= count) return;
  out[t] = Fr::mul(scale, Fr::pow_u64(w, t));
}

// One DIF pass: K stages with half-spans h0, h0/2, ..., h0 >> (K-1).   (natural -> bit-reversed)
template <class Fr, int K>
ZKB_HDN inline void ntt_dif_body(Fr* x, const Fr* tw, uint32_t log_n, uint32_t h0, uint32_t t) {
  constexpr uint32_t R = 1u << K;
  const uint32_t n = 1u << log_n;
  if (t >= (n >> K)) return;
  const uint32_t hmin = h0 >> (K - 1);
  const uint32_t off = t & (hmin - 1), blk = t / hmin;
  const size_t i0 = (size_t)blk * (2 * (size_t)h0) + off;
  Fr e[R];
#pragma unroll
  for (uint32_t m = 0; m < R; m++) e[m] = x[i0 + (size_t)m * hmin];
#pragma unroll
  for (int q = 0; q < K; q++) {
    const uint32_t hm = 1u << (K - 1 - q);
    const uint32_t h = hm * hmin;
    const uint32_t step = n / (2 * h);
#pragma unroll
    for (uint32_t m = 0; m < R; m++) {
      if (m & hm) continue;
      Fr u = e[m], v = e[m + hm];
      e[m] = Fr::add(u, v);
      Fr d = Fr::sub(u, v);
      uint32_t ex = (off + (m & (hm - 1)) * hmin) * step;
      e[m + hm] = ex ? Fr::mul(d, tw[ex]) : d;
    }
  }
#pragma unroll
  for (uint32_t m = 0; m < R; m++) x[i0 + (size_t)m * hmin] = e[m];
}

// One DIT pass: K stages with half-spans h0, 2 h0, ..., h0 << (K-1).   (bit-reversed -> natural)
template <class Fr, int K>
ZKB_HDN inline void ntt_dit_body(Fr* x, const Fr* tw, uint32_t log_n, uint32_t h0, uint32_t t) {
  constexpr uint32_t R = 1u << K;
  const uint32_t n = 1u << log_n;
  if (t >= (n >> K)) return;
  const uint32_t off = t & (h0 - 1), blk = t / h0;
  const size_t i0 = (size_t)blk * ((size_t)R * h0) + off;
  Fr e[R];
#pragma unroll
  for (uint32_t m = 0; m < R; m++) e[m] = x[i0 + (size_t)m * h0];
#pragma unroll
  for (int q = 0; q < K; q++) {
    const uint32_t hm = 1u << q;
    const uint32_t h = hm * h0;
    const uint32_t step = n / (2 * h);
#pragma unroll
    for (uint32_t m = 0; m < R; m++) {
      if (m & hm) continue;
      uint32_t ex = (off + (m & (hm - 1)) * h0) * step;
      Fr u = e[m];
      Fr v = ex ? Fr::mul(e[m + hm], tw[ex]) : e[m + hm];
      e[m] = Fr::add(u, v);
      e[m + hm] = Fr::sub(u, v);
    }
  }
#pragma unroll
  for (uint32_t m = 0; m < R; m++) x[i0 + (size_t)m * h0] = e[m];
}


// ---- shared-memory pass: S consecutive radix-2 stages on 1024-element tiles --------------------------------
// The register passes above move the whole vector through HBM once per 3 stages (7 round trips for n = 2^20).
// Here a block keeps a tile of 1024 elements (32 KB) in shared memory and runs S <= 10 stages on it, so a
// transform is ceil(log n / 10) round trips.  The stages of a pass act on index bits [lo_bit, lo_bit + S); a tile
// is G = 1024 >> S independent groups of 2^S elements.  For lo_bit > 0 the G groups are neighbours in the low
// index bits (runs of G contiguous elements in HBM, local position j * G + g); for lo_bit == 0 a tile is 1024
// contiguous elements (local position g * 2^S + j).  Phase 0 loads (optionally scaling by table[bitrev(i)], the
// coset shift between ifft and coset fft), phases 1..nk run K[p] <= 3 stages on 8 register-resident elements per
// step exactly like ntt_dif_body / ntt_dit_body, the last phase stores.  In place: tiles are disjoint.
struct NttPass {
  uint32_t log_n, lo_bit, S, nk;
  uint32_t K[4];
};
static constexpr uint32_t NTT_TILE_LOG = 10, NTT_TILE = 1u << NTT_TILE_LOG, NTT_BLOCK = 128;

ZKB_HD uint32_t ntt_tile_global(const NttPass& ps, uint32_t block, uint32_t e, uint32_t* j_out, uint32_t* low_out) {
  const uint32_t G = NTT_TILE >> ps.S;
  if (ps.lo_bit == 0) {
    *j_out = e & ((1u << ps.S) - 1u);
    *low_out = 0;
    return (block << NTT_TILE_LOG) | e;
  }
  const uint32_t per_hi = (1u << ps.lo_bit) / G;  // tiles per value of the high index bits
  const uint32_t hi = block / per_hi, lb = block % per_hi;
  const uint32_t j = e / G, g = e % G;
  *j_out = j;
  *low_out = lb * G + g;
  return (hi << (ps.lo_bit + ps.S)) | (j << ps.lo_bit) | (lb * G + g);
}

// one compute phase: K stages (compile-time, so the 2^K elements stay in registers) starting after `done` local stages
template <class Fr, bool DIT, int K>
ZKB_HDN inline void ntt_block_stages(const Fr* tw, const NttPass& ps, Fr* sm, uint32_t block, uint32_t thread, uint32_t done) {
  constexpr uint32_t R = 1u << K;
  const uint32_t G = NTT_TILE >> ps.S;
  const uint32_t lg_hmin = DIT ? done : ps.S - done - K;   // smallest local half-span of this phase
  const uint32_t hmin = 1u << lg_hmin;
  const uint32_t per_group = (1u << ps.S) >> K;             // work items per group
  uint32_t low_base = 0;
  if (ps.lo_bit) low_base = (block % ((1u << ps.lo_bit) / G)) * G;
  for (uint32_t tt = thread; tt < (NTT_TILE >> K); tt += NTT_BLOCK) {
    uint32_t g, jj;
    if (ps.lo_bit) { g = tt % G; jj = tt / G; } else { jj = tt % per_group; g = tt / per_group; }
    const uint32_t off = jj & (hmin - 1), blk = jj >> lg_hmin;
    const uint32_t j0 = (blk << (lg_hmin + K)) | off;
    const uint32_t low = ps.lo_bit ? low_base + g : 0;
    Fr e[R];
#pragma unroll
    for (uint32_t m = 0; m < R; m++) {
      const uint32_t j = j0 + m * hmin;
      e[m] = sm[ps.lo_bit ? j * G + g : (g << ps.S) + j];
    }
#pragma unroll
    for (int q = 0; q < K; q++) {
      const uint32_t hm = DIT ? (1u << q) : (1u << (K - 1 - q));
      const uint32_t lg_h = lg_hmin + (DIT ? q : K - 1 - q) + ps.lo_bit;   // log2 of the global half-span
      const uint32_t sh = ps.log_n - 1 - lg_h;                              // exponent step n / 2h
#pragma unroll
      for (uint32_t m = 0; m < R; m++) {
        if (m & hm) continue;
        const uint32_t imod = ((off + (m & (hm - 1)) * hmin) << ps.lo_bit) | low;
        const uint32_t ex = imod << sh;
        Fr u = e[m];
        if (DIT) {
          Fr v = ex ? Fr::mul(e[m + hm], tw[ex]) : e[m + hm];
          e[m] = Fr::add(u, v);
          e[m + hm] = Fr::sub(u, v);
        } else {
          Fr v = e[m + hm];
          e[m] = Fr::add(u, v);
          Fr d = Fr::sub(u, v);
          e[m + hm] = ex ? Fr::mul(d, tw[ex]) : d;
        }
      }
    }
#pragma unroll
    for (uint32_t m = 0; m < R; m++) {
      const uint32_t j = j0 + m * hmin;
      sm[ps.lo_bit ? j * G + g : (g << ps.S) + j] = e[m];
    }
  }
}

template <class Fr, bool DIT>
ZKB_HDN inline void ntt_block_body(Fr* x, const Fr* tw, const Fr* scale, NttPass ps, Fr* sm, uint32_t block, uint32_t thread,
                                   uint32_t phase) {
  if (phase == 0 || phase == ps.nk + 1) {
    for (uint32_t k = 0; k < NTT_TILE / NTT_BLOCK; k++) {
      const uint32_t e = thread + k * NTT_BLOCK;
      uint32_t j, low;
      const uint32_t gi = ntt_tile_global(ps, block, e, &j, &low);
      if (phase == 0) {
        Fr v = x[gi];
        if (scale) v = Fr::mul(v, scale[bitrev32(gi, ps.log_n)]);
        sm[e] = v;
      } else {
        x[gi] = sm[e];
      }
    }
    return;
  }
  uint32_t done = 0;
  for (uint32_t p = 1; p < phase; p++) done += ps.K[p - 1];
  switch (ps.K[phase - 1]) {
    case 3: ntt_block_stages<Fr, DIT, 3>(tw, ps, sm, block, thread, done); break;
    case 2: ntt_block_stages<Fr, DIT, 2>(tw, ps, sm, block, thread, done); break;
    default: ntt_block_stages<Fr, DIT, 1>(tw, ps, sm, block, thread, done); break;
  }
}

// split log_n stage bits into passes of at most max_s bits (balanced), top pass first; returns the pass count
// (0: this split cannot be tiled — the caller uses the register passes)
inline uint32_t ntt_plan_passes(uint32_t log_n, uint32_t max_s, NttPass out[8]) {
  if (max_s > NTT_TILE_LOG) max_s = NTT_TILE_LOG;
  const uint32_t np = (log_n + max_s - 1) / max_s;
  uint32_t hi = log_n;
  for (uint32_t i = 0; i < np; i++) {
    uint32_t S = log_n / np + (i < log_n % np ? 1 : 0);
    NttPass& p = out[i];
    p.log_n = log_n; p.S = S; p.lo_bit = hi - S;
    p.nk = (S + 2) / 3;
    for (uint32_t k = 0; k < 4; k++) p.K[k] = 0;
    for (uint32_t k = 0; k < p.nk; k++) p.K[k] = S / p.nk + (k < S % p.nk ? 1 : 0);
    hi -= S;
    // interleaved groups need runs of G = 1024 >> S elements inside the low index bits
    if (p.lo_bit && p.lo_bit + S < NTT_TILE_LOG) return 0;
  }
  return np;
}

// x[i] *= table[bitrev(i)]  (coset shift / 1/n scaling applied to a bit-reversed coefficient vector)
template <class Fr>
ZKB_HDN inline void ntt_scale_brev_body(Fr* x, const Fr* table, uint32_t log_n, uint32_t t) {
  if (t >= (1u << log_n)) return;
  x[t] = Fr::mul(x[t], table[bitrev32(t, log_n)]);
}

// out[bitrev(i)] = in[i] * table[bitrev(i)] (table may be null), optionally leaving Montgomery form
template <class Fr>
ZKB_HDN inline void ntt_brev_copy_body(const Fr* in, Fr* out, const Fr* table, uint32_t log_n, int to_canonical, uint32_t t) {
  if (t >= (1u << log_n)) return;
  uint32_t j = bitrev32(t, log_n);
  Fr v = in[t];
  if (table) v = Fr::mul(v, table[j]);
  if (to_canonical) v = Fr::from_mont(v);
  out[j] = v;
}

// ab[i] = (a[i]*b[i] - c[i]) * zinv      (witness_map: a∘b - c, divided by the vanishing polynomial)
template <class Fr>
ZKB_HDN inline void qap_pointwise_body(Fr* a, const Fr* b, const Fr* c, Fr zinv, uint32_t n, uint32_t t) {
  if (t >= n) return;
  a[t] = Fr::mul(Fr::sub(Fr::mul(a[t], b[t]), c[t]), zinv);
}

// Montgomery conversion of a vector: dir = 0 canonical -> Montgomery, 1 Montgomery -> canonical
template <class Fr>
ZKB_HDN inline void fr_convert_body(const Fr* in, Fr* out, int dir, size_t n, size_t t) {
  if (t >= n) return;
  out[t] = dir ? Fr::from_mont(in[t]) : Fr::to_mont(in[t]);
}

// CSR sparse matrix-vector product in Montgomery form for a batch of K assignments, G of them per thread: one thread reads a
// CSR row (columns and coefficients) once and accumulates G dot products (G = 1 for a single assignment).  z is INTERLEAVED,
// z[col * K + k]: the G values a term needs sit in G * 32 consecutive bytes (one or two cache lines) instead of G lines
// K * m * 32 bytes apart.  Vector k of the output starts at out + k * n (rows 0 .. n - 1 of the domain): rows below n_rows
// hold the products, the next n_copy rows z[row - n_rows] (the instance variables of the A chain, n_copy = 0 for B and C),
// the rest zero.
template <class Fr, int G>
ZKB_HDN inline void spmv_batch_body(const uint32_t* rowptr, const uint32_t* col, const Fr* val, const Fr* z, uint32_t K, uint32_t k0,
                                    Fr* out, size_t n, uint32_t n_rows, uint32_t n_copy, uint32_t row) {
  const uint32_t kn = K - k0 < (uint32_t)G ? K - k0 : (uint32_t)G;
  Fr acc[G];
#pragma unroll
  for (int g = 0; g < G; g++) acc[g] = Fr::zero();
  if (row < n_rows) {
    for (uint32_t e = rowptr[row]; e < rowptr[row + 1]; e++) {
      const Fr v = val[e];
      const Fr* zr = z + (size_t)col[e] * K + k0;
#pragma unroll
      for (int g = 0; g < G; g++)
        if ((uint32_t)g < kn) acc[g] = Fr::add(acc[g], Fr::mul(v, zr[g]));
    }
  } else if (row - n_rows < n_copy) {
#pragma unroll
    for (int g = 0; g < G; g++)
      if ((uint32_t)g < kn) acc[g] = z[(size_t)(row - n_rows) * K + k0 + g];
  }
#pragma unroll
  for (int g = 0; g < G; g++)
    if ((uint32_t)g < kn) out[(size_t)(k0 + g) * n + row] = acc[g];
}


// ---- levelised witness evaluation / R1CS satisfaction check ------------------------------------------------
// Restates the per-statement rule of zokrates_interpreter/src/lib.rs:61-138 on the R1CS rows: a constraint whose linear side
// is one fresh variable with coefficient one ASSIGNS it the value of the quadratic side, every other constraint is CHECKED
// (`Error::UnsatisfiedConstraint`).  The statements of one dependency level are independent: one thread each per input set.
// A batch of K input sets shares the schedule: z is INTERLEAVED, z[col * K + k] (the layout of spmv_batch_body), thread t
// runs statement lo + t / K for set t % K, so the K threads of a statement read one CSR row and adjacent values; set k's
// first violated row goes to first_unsat[k].  K = 1 is the single assignment.
// rows == nullptr: row = index (check of the whole system); out_var == nullptr: every row is a check.
static constexpr uint32_t WIT_CHECK = 0xFFFFFFFFu;
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ void zkb_atomic_min(uint32_t* p, uint32_t v) { atomicMin(p, v); }
#else
inline void zkb_atomic_min(uint32_t* p, uint32_t v) { if (v < *p) *p = v; }
#endif
template <class Fr>
ZKB_HDN inline Fr csr_row_dot(const uint32_t* rowptr, const uint32_t* col, const Fr* val, const Fr* z, uint32_t K, uint32_t k,
                              uint32_t row) {
  Fr acc = Fr::zero();
  for (uint32_t e = rowptr[row]; e < rowptr[row + 1]; e++) acc = Fr::add(acc, Fr::mul(val[e], z[(size_t)col[e] * K + k]));
  return acc;
}
template <class Fr>
ZKB_HDN inline void witness_level_body(const uint32_t* rpA, const uint32_t* clA, const Fr* vlA, const uint32_t* rpB,
                                       const uint32_t* clB, const Fr* vlB, const uint32_t* rpC, const uint32_t* clC,
                                       const Fr* vlC, Fr* z, const uint32_t* rows, const uint32_t* out_var, uint32_t lo,
                                       uint32_t hi, uint32_t K, uint32_t* first_unsat, uint32_t t) {
  const uint32_t i = lo + t / K, k = t % K;
  if (i >= hi) return;
  const uint32_t row = rows ? rows[i] : i;
  const Fr q = Fr::mul(csr_row_dot<Fr>(rpA, clA, vlA, z, K, k, row), csr_row_dot<Fr>(rpB, clB, vlB, z, K, k, row));
  const uint32_t ov = out_var ? out_var[i] : WIT_CHECK;
  if (ov != WIT_CHECK) {
    z[(size_t)ov * K + k] = q;
  } else if (!(q == csr_row_dot<Fr>(rpC, clC, vlC, z, K, k, row))) {
    zkb_atomic_min(first_unsat + k, row);
  }
}

}  // namespace zkb
