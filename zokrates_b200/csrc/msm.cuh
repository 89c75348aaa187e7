// Multi-scalar multiplication sum_i s_i * P_i (Pippenger bucket method) for G1 and G2.
//
// Replaces ark-ec 0.3.0 `VariableBaseMSM::multi_scalar_mul` (external, Cargo.lock:146) as called
// five times per proof by ark-groth16's prover (reached from
// /root/reference/zokrates_ark/src/groth16.rs:44; SURVEY.md §8 rows a5/a6, App. B.4).  The result
// is a group element, so any window size / digit encoding gives the same affine point as ark's
// (unsigned windows, c = ln-rule) — only the schedule is redesigned for the GPU:
//
//   digits   : signed c-bit digits per scalar (halves the bucket count), histogram per bucket
//   scan     : exclusive prefix sum -> bucket offsets
//   scatter  : counting sort of (point index, sign) by (window, bucket)
//   accumulate: the sorted list is cut into FIXED-SIZE chunks, one thread per chunk, so the load is
//              balanced for any scalar distribution (real witnesses are mostly 0/1, SURVEY.md §7).
//              A bucket wholly inside a chunk is written directly; a bucket cut by a chunk border
//              is deferred as a partial sum to the next (much smaller) level, which runs the same
//              segmented reduction on XYZZ partials.
//   bucket reduction: sum_j (j+1) * B_j by bit sums (msm_bitsum_body); the last few hundred additions run on the host.
//
// One "plan" (digits/sort) is reused for every point vector that shares the scalars: a_query,
// b_g1_query, b_g2_query and l_query all pair with the same assignment vector.
#pragma once
#include "ec.cuh"

namespace zkb {

static constexpr uint32_t MSM_NONE = 0xFFFFFFFFu;   // zero digit / empty slot
static constexpr uint32_t MSM_NEG = 0x80000000u;

#if defined(__CUDA_ARCH__)
__device__ __forceinline__ uint32_t zkb_atomic_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
#else
inline uint32_t zkb_atomic_add(uint32_t* p, uint32_t v) { uint32_t o = *p; *p = o + v; return o; }
#endif

// A plan may carry a BATCH of K scalar vectors over the same n points (K proofs of one circuit): every proof has its own
// bucket set, bucket key k * NB + bucket with NB = msm_set_buckets, while the sorted entries still name the shared point
// (or its table entry w * n + i).  The accumulate and reduction kernels only see K * NB buckets and K * W windows.
struct MsmShape {
  uint32_t n;        // number of (scalar, point) pairs of one proof
  uint32_t c;        // window bits
  uint32_t W;        // windows
  uint32_t B;        // buckets per window = 2^(c-1)
  uint32_t pre;      // 1: the point table holds 2^(c w) P_i at index w*n + i, so all windows share ONE bucket set
  uint32_t K;        // scalar vectors (proofs) in the batch, >= 1
};
ZKB_HD uint32_t msm_set_buckets(const MsmShape& sh) { return sh.pre ? sh.B : sh.W * sh.B; }
ZKB_HD uint32_t msm_nbuckets(const MsmShape& sh) { return sh.K * msm_set_buckets(sh); }

ZKB_HD uint32_t scalar_bits(const uint32_t* s, uint32_t lo, uint32_t cnt) {
  // bits [lo, lo+cnt) of a 256-bit little-endian scalar, cnt <= 31
  uint32_t limb = lo >> 5, sh = lo & 31;
  uint64_t v = limb < 8 ? s[limb] : 0;
  if (limb + 1 < 8) v |= (uint64_t)s[limb + 1] << 32;
  return (uint32_t)(v >> sh) & ((1u << cnt) - 1u);
}

// ---- digits + histogram: one thread per (proof, scalar) ---------------------------------------
// Scalar vector k starts at scalars + k * stride elements.  digits[(k W + w) n + i] = (|d| - 1) | sign, or MSM_NONE when
// d == 0;  ranks[.] = arrival order of the entry inside its bucket (the value the histogram atomic returned), so the scatter
// needs no second atomic.  The plan keeps K n W < 2^32 (engine.cuh::plan_build), so thread indices divide in 32 bits.
ZKB_HDN inline void msm_digits_body(MsmShape sh, const uint32_t* scalars /* canonical, 8 words each */, size_t stride, uint32_t* digits,
                                    uint32_t* ranks, uint32_t* counts /* K * msm_set_buckets */, uint32_t t) {
  if (t >= sh.K * sh.n) return;
  const uint32_t k = t / sh.n, i = t % sh.n;
  const uint32_t* src = scalars + ((size_t)k * stride + i) * 8;
  uint32_t s[8];
#pragma unroll
  for (int q = 0; q < 8; q++) s[q] = src[q];
  uint32_t carry = 0;
  const uint32_t full = 1u << sh.c, half = sh.B;
  const uint32_t kbase = k * msm_set_buckets(sh);
  const size_t row0 = (size_t)k * sh.W;
  for (uint32_t w = 0; w < sh.W; w++) {
    uint32_t d = scalar_bits(s, w * sh.c, sh.c) + carry;
    uint32_t code;
    if (d == 0) {
      code = MSM_NONE;
      carry = 0;
    } else if (d > half) {
      code = (full - d - 1) | MSM_NEG;  // digit d - 2^c < 0, magnitude 2^c - d in [1, 2^(c-1) - 1]
      carry = 1;
      if (full - d == 0) {              // d == 2^c: digit 0, carry 1
        code = MSM_NONE;
      }
    } else {
      code = d - 1;
      carry = 0;
    }
    const size_t slot = (row0 + w) * sh.n + i;
    digits[slot] = code;
    if (code != MSM_NONE) {
      const uint32_t key = kbase + (sh.pre ? 0u : w * sh.B) + (code & ~MSM_NEG);
      ranks[slot] = zkb_atomic_add(&counts[key], 1);
    }
  }
}

// ---- scatter: one thread per (proof, window, scalar) ----------------------------------------------
// sorted[offsets[key] + rank] = point index | sign      (counting sort; the order inside a bucket is irrelevant: sums)
ZKB_HDN inline void msm_scatter_body(MsmShape sh, const uint32_t* digits, const uint32_t* ranks, const uint32_t* offsets,
                                     uint32_t* sorted, uint32_t t) {
  if (t >= sh.K * sh.n * sh.W) return;
  uint32_t code = digits[t];
  if (code == MSM_NONE) return;
  const uint32_t kw = t / sh.n, i = t % sh.n, w = kw % sh.W, k = kw / sh.W;
  uint32_t key = k * msm_set_buckets(sh) + (sh.pre ? 0u : w * sh.B) + (code & ~MSM_NEG);
  const uint32_t val = (sh.pre ? w * sh.n + i : i) | (code & MSM_NEG);
  sorted[offsets[key] + ranks[t]] = val;
}

// ---- views: filtered copies of the sorted list ----------------------------------------------------
// View v > 0 drops the pairs whose point is the point at infinity in that query vector (bit v-1 of skip[i]; ark's
// add_assign_mixed treats them as a no-op too).  A view is a STABLE COMPACTION of the sorted list of view 0 — a streaming
// pass with ballots and a tile scan instead of a second and third round of histogram / cursor atomics (round 1: the
// three-view plan cost 2.6 ms per proof, most of it atomics).  Per group of 32 consecutive sorted positions the pass keeps
// the keep-mask and the exclusive count before the group, from which the bucket offsets of the view follow:
//   offsets_v[b] = pre32[g] + popc(mask32[g] & lanes below p),  p = offsets_0[b], g = p / 32.
ZKB_HD uint32_t msm_view_keep(const MsmShape& sh, const uint8_t* skip, uint32_t entry, uint32_t v) {
  const uint32_t idx = entry & ~MSM_NEG;
  const uint32_t i = sh.pre ? idx % sh.n : idx;
  return !((skip[i] >> (v - 1)) & 1u);
}
ZKB_HDN inline void msm_view_offsets_body(uint32_t NB, const uint32_t* offsets0, const uint32_t* pre32, const uint32_t* mask32,
                                          const uint32_t* total_v, uint32_t* offsets_v, uint32_t b) {
  if (b > NB) return;
  const uint32_t M = offsets0[NB], p = offsets0[b];
  if (p >= M) { offsets_v[b] = *total_v; return; }
  const uint32_t g = p >> 5, lane = p & 31u;
  const uint32_t below = mask32[g] & ((1u << lane) - 1u);
#if defined(__CUDA_ARCH__)
  offsets_v[b] = pre32[g] + __popc(below);
#else
  offsets_v[b] = pre32[g] + (uint32_t)__builtin_popcount(below);
#endif
}

// ---- level-1 accumulate: affine points, keys implied by the offsets array -----------------------
// Thread t owns sorted positions [t*T, (t+1)*T).  Deferred partials go to slots 2t (first segment)
// and 2t+1 (last segment) of (pkey, pval); unused slots get MSM_NONE.
template <class F>
ZKB_HDN inline void msm_accum1_body(uint32_t nbuckets, uint32_t T, const uint32_t* offsets, const uint32_t* sorted,
                                    const Affine<F>* points, XYZZ<F>* buckets, uint32_t* pkey, XYZZ<F>* pval,
                                    uint32_t nthreads, uint32_t t) {
  if (t >= nthreads) return;
  const uint32_t M = offsets[nbuckets];
  uint32_t k0 = MSM_NONE, k1 = MSM_NONE;
  uint64_t start64 = (uint64_t)t * T;
  if (start64 < M) {
    uint32_t pos = (uint32_t)start64;
    uint32_t end = (M - pos > T) ? pos + T : M;
    // bucket containing pos: largest b with offsets[b] <= pos  (offsets is non-decreasing)
    uint32_t lo = 0, hi = nbuckets;  // invariant offsets[lo] <= pos < offsets[hi]
    while (hi - lo > 1) {
      uint32_t mid = (lo + hi) >> 1;
      if (offsets[mid] <= pos) lo = mid; else hi = mid;
    }
    uint32_t b = lo;
    const uint32_t cstart = pos;
    while (offsets[b + 1] <= pos) b++;  // (lo may be an empty bucket sharing the offset)
    uint32_t bstart = offsets[b], bend = offsets[b + 1];
    XYZZ<F> acc = XYZZ<F>::identity();
    // ONE flat loop over the chunk: the bucket change is a short predicated block, so every lane of the
    // warp meets at the same mixed addition each iteration (no nested-loop divergence).
    // software pipeline: the index (and, when registers allow, the point) of entry p+1 is fetched before the
    // mixed addition of entry p, so the dependent gather sorted[p] -> points[.] hides behind ~2500 instructions
    constexpr bool PREFETCH_POINT = sizeof(Affine<F>) <= 64;
    // sorted == nullptr: the points ARE the list (output of the batch-affine rounds, msm_affine.cuh), entry p = point p
    uint32_t e = sorted ? sorted[pos] : pos;
    Affine<F> q;
    if (PREFETCH_POINT) q = points[e & ~MSM_NEG];
    for (uint32_t p = pos; p < end; p++) {
      uint32_t e_next = 0;
      Affine<F> q_next;
      if (p + 1 < end) {
        e_next = sorted ? sorted[p + 1] : p + 1;
        if (PREFETCH_POINT) q_next = points[e_next & ~MSM_NEG];
      }
      if (p == bend) {
        if (bstart >= cstart) buckets[b] = acc;            // complete (it also ends inside the chunk)
        else { k0 = b; pval[2 * (size_t)t] = acc; }        // began in the previous chunk
        b++;
        while (offsets[b + 1] <= p) b++;
        bstart = p;
        bend = offsets[b + 1];
        acc = XYZZ<F>::identity();
      }
      if (!PREFETCH_POINT) q = points[e & ~MSM_NEG];
      if (e & MSM_NEG) q.y = F::neg(q.y);
      acc = XYZZ<F>::madd(acc, q);
      e = e_next;
      if (PREFETCH_POINT) q = q_next;
    }
    if (bstart >= cstart && bend <= end) buckets[b] = acc;
    else if (bstart < cstart) { k0 = b; pval[2 * (size_t)t] = acc; }
    else { k1 = b; pval[2 * (size_t)t + 1] = acc; }
  }
  pkey[2 * (size_t)t] = k0;
  pkey[2 * (size_t)t + 1] = k1;
}

// ---- level >= 2: segmented reduction over (key, XYZZ) entries with holes ------------------------
// Chunk t owns entries [t*T - 1, (t+1)*T - 1) (shifted by one so that the pair "last of chunk u /
// first of chunk u+1" emitted by the level below is never cut again).  Same-key entries are
// separated by at most one MSM_NONE hole (see DESIGN.md), so two-entry look-behind/ahead decides
// whether a run is complete.
template <class F>
ZKB_HDN inline void msm_accum2_body(uint32_t L, uint32_t T, const uint32_t* key, const XYZZ<F>* val, XYZZ<F>* buckets,
                                    uint32_t* okey, XYZZ<F>* oval, uint32_t nthreads, uint32_t t) {
  if (t >= nthreads) return;
  uint64_t s64 = (uint64_t)t * T;
  uint32_t s = s64 == 0 ? 0 : (uint32_t)(s64 - 1);
  uint64_t e64 = s64 + T - 1;
  uint32_t e = e64 < L ? (uint32_t)e64 : L;
  uint32_t k0 = MSM_NONE, k1 = MSM_NONE;
  // key just left of the chunk (skipping one hole)
  uint32_t left = MSM_NONE;
  if (s >= 1) {
    left = key[s - 1];
    if (left == MSM_NONE && s >= 2) left = key[s - 2];
  }
  uint32_t right = MSM_NONE;
  if (e < L) {
    right = key[e];
    if (right == MSM_NONE && e + 1 < L) right = key[e + 1];
  }
  uint32_t cur = MSM_NONE;
  XYZZ<F> acc = XYZZ<F>::identity();
  bool first = true;  // cur is the first run of this chunk
  for (uint32_t p = s; p <= e; p++) {
    uint32_t k = (p < e) ? key[p] : MSM_NONE - 1;  // sentinel flushes the last run
    if (p < e && k == MSM_NONE) continue;
    if (k != cur) {
      if (cur != MSM_NONE) {
        bool last = (p == e);
        bool open_left = first && left == cur;
        bool open_right = last && right == cur;
        if (!open_left && !open_right) {
          buckets[cur] = acc;
        } else if (open_left) {
          k0 = cur;
          oval[2 * (size_t)t] = acc;
        } else {
          k1 = cur;
          oval[2 * (size_t)t + 1] = acc;
        }
        first = false;
      }
      cur = k;
      acc = XYZZ<F>::identity();
    }
    if (p < e) acc = XYZZ<F>::add(acc, val[p]);
  }
  okey[2 * (size_t)t] = k0;
  okey[2 * (size_t)t + 1] = k1;
}

// ---- window table: table[w * n + i] = 2^(c w) * P_i (affine), one thread per point ------------------
// The W-1 multiples are normalised with one shared inversion (Montgomery's trick) per point.
template <class F, int MAXW>
ZKB_HDN inline void msm_table_body(const Affine<F>* pts, Affine<F>* table, uint32_t n, uint32_t c, uint32_t W, uint32_t i) {
  if (i >= n) return;
  Affine<F> p = pts[i];
  table[i] = p;
  if (p.is_inf()) {
    for (uint32_t w = 1; w < W; w++) table[(size_t)w * n + i] = Affine<F>::inf();
    return;
  }
  XYZZ<F> cur = XYZZ<F>::from_affine(p);
  XYZZ<F> mult[MAXW];
  F pref[MAXW];
  F run = F::one();
  for (uint32_t w = 1; w < W; w++) {
    for (uint32_t d = 0; d < c; d++) cur = XYZZ<F>::dbl_ni(cur);
    mult[w] = cur;
    pref[w] = run;                                   // product of the denominators before w
    run = F::mul_ni(run, F::mul_ni(cur.zz, cur.zzz));  // a prime-order point never doubles to infinity
  }
  F inv = F::inv(run);
  for (uint32_t w = W; w-- > 1;) {
    F dinv = F::mul_ni(inv, pref[w]);                // 1 / (zz zzz)
    inv = F::mul_ni(inv, F::mul_ni(mult[w].zz, mult[w].zzz));
    F zzi = F::mul_ni(dinv, mult[w].zzz), zzzi = F::mul_ni(dinv, mult[w].zz);
    table[(size_t)w * n + i] = Affine<F>{F::mul_ni(mult[w].x, zzi), F::mul_ni(mult[w].y, zzzi)};
  }
}

// ---- bucket reduction: per window sum_j (j+1) * bucket[j] by BIT SUMS ---------------------------------
// sum_j j B_j = sum_bit 2^bit * S_bit with S_bit = sum of the buckets whose index has that bit set, so the weighted sum
// needs no weighted arithmetic on the device at all — only plain sums over subsets, which reduce in parallel with a
// dependent chain of 7 additions per level (the previous (sum, weighted-sum) tree ran 23 per level plus 3*lvl doublings).
// One level groups 8 consecutive entries (3 index bits) and is ONE launch of uniform "masked 8-sums":
//   role 0      : A'[k]      = sum of all 8 entries of A[8k..8k+8)            (block totals, feed the next level)
//   role 1+b    : P_new_b[k] = sum of the entries i of that block with bit b of i set   (b = 0, 1, 2)
//   role 4+r    : P_r'[k]    = sum of all 8 entries of the pending array P_r  (plain reduction of older bit sums)
// so every array has the same length at every level.  After L levels the host holds A (cnt entries) and 3L pending
// arrays per window and finishes with a few hundred additions:  S_(3l+b) = sum_k P_(3l+b)[k],
//   sum_j (j+1) B_j = total + Horner_bits(S) + 2^(3L) * sum_k k A[k]   (engine.cuh::host_finish).
// Pending array r of the input holds bit 3*(r/3) + r%3; the three new arrays are appended after the npend old ones.
template <class F>
ZKB_HDN inline void msm_bitsum_body(uint32_t W, uint32_t cnt_in, uint32_t npend, const XYZZ<F>* inA, const XYZZ<F>* inP,
                                    XYZZ<F>* outA, XYZZ<F>* outP, uint32_t t) {
  const uint32_t cnt_out = cnt_in >> 3;
  const uint32_t per_role = W * cnt_out;
  const uint32_t role = t / per_role, node = t % per_role;
  if (role >= 4 + npend) return;
  const uint32_t w = node / cnt_out, k = node % cnt_out;
  const XYZZ<F>* src = (role < 4 ? inA : inP + (size_t)(role - 4) * W * cnt_in) + (size_t)w * cnt_in + ((size_t)k << 3);
  uint32_t mask = 0xFFu;
  if (role == 1) mask = 0xAAu; else if (role == 2) mask = 0xCCu; else if (role == 3) mask = 0xF0u;
  XYZZ<F> sum = XYZZ<F>::identity();
#pragma unroll 1
  for (uint32_t i = 0; i < 8; i++)
    if ((mask >> i) & 1u) sum = XYZZ<F>::add(sum, src[i]);
  XYZZ<F>* dst;
  if (role == 0) dst = outA;
  else if (role < 4) dst = outP + (size_t)(npend + role - 1) * per_role;
  else dst = outP + (size_t)(role - 4) * per_role;
  dst[node] = sum;
}

// ---- radix-2 level of the same scheme: cnt_in -> cnt_in / 2, ONE dependent addition per level ------------------------
// role 0        : A'[k]   = A[2k] + A[2k+1]
// role 1+r      : P_r'[k] = P_r[2k] + P_r[2k+1]        (r < npend: plain halving of the older bit-sum arrays)
// role 1+npend  : P_new[k] = A[2k+1]                   (the entries whose index bit `level` is set: a copy, no arithmetic)
// Pending array r holds index bit r.  Against the radix-8 level this is less work (4 instead of 9 additions per 8 entries
// for the new bits) and, above all, a dependent chain of 1 instead of 7 additions per launch: the upper levels are pure
// latency (a G2 addition is ~28 us on one thread), so the tail of an MSM shrinks by the ratio of the chain lengths.
template <class F>
ZKB_HDN inline void msm_bitsum2_body(uint32_t W, uint32_t cnt_in, uint32_t npend, const XYZZ<F>* inA, const XYZZ<F>* inP,
                                     XYZZ<F>* outA, XYZZ<F>* outP, uint32_t t) {
  const uint32_t cnt_out = cnt_in >> 1;
  const uint32_t per_role = W * cnt_out;
  const uint32_t role = t / per_role, node = t % per_role;
  if (role >= 2 + npend) return;
  const uint32_t w = node / cnt_out, k = node % cnt_out;
  const bool from_a = role == 0 || role == 1 + npend;
  const XYZZ<F>* src = (from_a ? inA : inP + (size_t)(role - 1) * W * cnt_in) + (size_t)w * cnt_in + ((size_t)k << 1);
  if (role == 0) outA[node] = XYZZ<F>::add(src[0], src[1]);
  else if (role == 1 + npend) outP[(size_t)npend * per_role + node] = src[1];
  else outP[(size_t)(role - 1) * per_role + node] = XYZZ<F>::add(src[0], src[1]);
}

}  // namespace zkb
