// Montgomery-form prime-field arithmetic on 32-bit limbs (8 limbs: BN254 Fr/Fq, BLS12-381 Fr, BLS12-377 Fr;
// 12 limbs: BLS12-381 Fq, BLS12-377 Fq).
//
// Replaces, on the device, what the reference reaches through `zokrates_field::FieldPrime`
// (/root/reference/zokrates_field/src/lib.rs:407-503 -> ark_ff::Fp256/Fp384 Montgomery ops, ark-ff
// 0.3.0, Cargo.lock:161).  Values are the same residues; the limb width (32 vs ark's 64) and the
// Montgomery radix R = 2^(32 N) = 2^256 / 2^384 coincide with ark's, so Montgomery images are
// bit-identical to ark's in-memory representation.
//
// mul(): CIOS Montgomery multiplication with the product columns split into an "even" and an
// "odd" accumulator so that every 32x32->64 product is ONE multiply-add (IMAD.WIDE.U32 with a
// predicate carry) and each row is two independent carry chains: N*(2N+1) wide MADs per
// multiplication (136 for N = 8, 300 for N = 12) — the unit SURVEY.md §8(d) counts.
// redc(mul_wide(a, b)) needs the same wide MADs but keeps a 2N-limb product live between the two halves.
// Compiled for sm_90a with mul() defined that way, the BN254 G1 accumulate needed 150 registers instead of
// 144 (IMAD.WIDE 1833 vs 1843 per kernel), accum2 168 instead of 150, the bit sums 164 instead of 136, and the
// 128-register NTT tile spilled 52 / 96 bytes instead of 40 / 16 (DIT / DIF).  So the fused CIOS body stays
// the plain multiplication; the separated form is used where it saves work: squarings (sqr_wide) and sums of
// products reduced once.
//
// mul() also accepts one unreduced operand: with a < 2p and b < p its running value stays < a + p < 3p < R
// (N limbs) and the result (ab + mp)/R < ab/R + p < 2p, so the one conditional subtraction reduces it fully.
// That needs 3p < R and 2p^2 < p*R, both implied by LAZY_HEADROOM below.
#pragma once
#include "hd.cuh"
#include "field_params.cuh"

namespace zkb {

// beta of Fq2 = Fq[u]/(u^2 - beta): P::FP2_NONRESIDUE where the parameters define it (BLS12-377 Fq: -5), else -1
template <class P, class = void>
struct Fp2NonResidue {
  static constexpr int value = -1;
};
template <class P>
struct Fp2NonResidue<P, decltype((void)P::FP2_NONRESIDUE)> {
  static constexpr int value = P::FP2_NONRESIDUE;
};

template <class P>
struct alignas(16) Fp {
  static constexpr int N = P::N;
  static constexpr int FP2_NONRESIDUE = Fp2NonResidue<P>::value;
  typedef P Params;
  uint32_t v[N];

  ZKB_HD static Fp zero() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = 0;
    return r;
  }
  ZKB_HD static Fp one() {  // Montgomery image of 1
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = P::r1(i);
    return r;
  }
  ZKB_HD static Fp r2() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = P::r2(i);
    return r;
  }
  ZKB_HD static Fp modulus() {
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = P::mod(i);
    return r;
  }
  ZKB_HD bool is_zero() const {
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < N; i++) acc |= v[i];
    return acc == 0;
  }
  ZKB_HD bool operator==(const Fp& o) const {
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < N; i++) acc |= v[i] ^ o.v[i];
    return acc == 0;
  }
  ZKB_HD bool operator!=(const Fp& o) const { return !(*this == o); }

  // r = a - p if a >= p else a   (a < 2p)
  ZKB_HD static Fp reduce_once(const Fp& a) {
    Fp t;
    t.v[0] = ptx::sub_cc(a.v[0], P::mod(0));
#pragma unroll
    for (int i = 1; i < N; i++) t.v[i] = ptx::subc_cc(a.v[i], P::mod(i));
    uint32_t borrow = ptx::subc(0, 0);  // 0 - 0 - CF  -> 0xffffffff when a < p
    Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.v[i] = borrow ? a.v[i] : t.v[i];
    return r;
  }

  ZKB_HD static Fp add(const Fp& a, const Fp& b) {
    Fp t;  // 2p < 2^(32N) for every field here, so the raw sum does not overflow
    t.v[0] = ptx::add_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) t.v[i] = ptx::addc_cc(a.v[i], b.v[i]);
    t.v[N - 1] = ptx::addc(a.v[N - 1], b.v[N - 1]);
    return reduce_once(t);
  }

  ZKB_HD static Fp sub(const Fp& a, const Fp& b) {
    Fp t;
    t.v[0] = ptx::sub_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < N; i++) t.v[i] = ptx::subc_cc(a.v[i], b.v[i]);
    uint32_t borrow = ptx::subc(0, 0);  // all-ones when a < b
    Fp r;
    r.v[0] = ptx::add_cc(t.v[0], P::mod(0) & borrow);
#pragma unroll
    for (int i = 1; i < N - 1; i++) r.v[i] = ptx::addc_cc(t.v[i], P::mod(i) & borrow);
    r.v[N - 1] = ptx::addc(t.v[N - 1], P::mod(N - 1) & borrow);
    return r;
  }

  ZKB_HD static Fp neg(const Fp& a) {
    if (a.is_zero()) return a;
    Fp r;
    r.v[0] = ptx::sub_cc(P::mod(0), a.v[0]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) r.v[i] = ptx::subc_cc(P::mod(i), a.v[i]);
    r.v[N - 1] = ptx::subc(P::mod(N - 1), a.v[N - 1]);
    return r;
  }

  ZKB_HD static Fp dbl(const Fp& a) { return add(a, a); }

  // Montgomery product a*b*R^-1 mod p, fully reduced.
  ZKB_HD static Fp mul(const Fp& a, const Fp& b) {
    static_assert(N % 2 == 0, "even limb count");
    // T = sum E[k] W^k + sum O[k] W^(k+1)
    uint32_t E[N], O[N];
    {
      const uint32_t y = b.v[0];
#pragma unroll
      for (int j = 0; j < N; j += 2) {
        uint64_t w = (uint64_t)a.v[j] * y;
        E[j] = (uint32_t)w;
        E[j + 1] = (uint32_t)(w >> 32);
        uint64_t u = (uint64_t)a.v[j + 1] * y;
        O[j] = (uint32_t)u;
        O[j + 1] = (uint32_t)(u >> 32);
      }
    }
#pragma unroll
    for (int i = 0; i < N; i++) {
      if (i > 0) {
        // shift one word down (E[0] == 0 after the previous reduction) and add a * b[i]
        const uint32_t y = b.v[i];
        uint32_t nE[N], nO[N];
        nE[0] = ptx::add_cc(O[0], E[1]);
#pragma unroll
        for (int j = 1; j < N - 1; j += 2) ptx::madc_wide_cc(nO[j - 1], nO[j], a.v[j], y, E[j + 1], E[j + 2]);
        ptx::madc_wide(nO[N - 2], nO[N - 1], a.v[N - 1], y, 0, 0);
        ptx::mad_wide_cc(nE[0], nE[1], a.v[0], y, nE[0], O[1]);
#pragma unroll
        for (int j = 2; j < N; j += 2) ptx::madc_wide_cc(nE[j], nE[j + 1], a.v[j], y, O[j], O[j + 1]);
        nO[N - 1] = ptx::addc(nO[N - 1], 0);
#pragma unroll
        for (int j = 0; j < N; j++) {
          E[j] = nE[j];
          O[j] = nO[j];
        }
      }
      // T += m * p with m chosen so that word 0 cancels
      const uint32_t m = E[0] * P::INV;
      ptx::mad_wide_cc(O[0], O[1], P::mod(1), m, O[0], O[1]);
#pragma unroll
      for (int j = 3; j < N; j += 2) ptx::madc_wide_cc(O[j - 1], O[j], P::mod(j), m, O[j - 1], O[j]);
      ptx::mad_wide_cc(E[0], E[1], P::mod(0), m, E[0], E[1]);
#pragma unroll
      for (int j = 2; j < N; j += 2) ptx::madc_wide_cc(E[j], E[j + 1], P::mod(j), m, E[j], E[j + 1]);
      O[N - 1] = ptx::addc(O[N - 1], 0);
    }
    // result = T / W = O + (E >> 32)
    Fp t;
    t.v[0] = ptx::add_cc(O[0], E[1]);
#pragma unroll
    for (int k = 1; k < N - 1; k++) t.v[k] = ptx::addc_cc(O[k], E[k + 1]);
    t.v[N - 1] = ptx::addc(O[N - 1], 0);
    return reduce_once(t);
  }

  // ---- separated Montgomery multiplication: wide products, wide sums, one reduction ----
  //
  // A Wide holds a 2N-limb integer.  mul_wide/sqr_wide produce a*b exactly; redc(T) returns T*R^-1 mod p
  // fully reduced for any T < p*R.  Formulas that sum several products (ec.cuh's fused Y3, fp2.cuh's lazy
  // Karatsuba) add Wides and reduce once.  Unreduced values exist only inside those formulas; every Fp that
  // leaves them is fully reduced.
  //
  // Headroom: redc needs T < p*R, which a single product of reduced values (< p^2) always meets.  The lazy
  // formulas need more: an unreduced N-limb sum of two reduced values is < 2p, a product of two such sums
  // is < 4p^2, and callers sum up to four products of reduced values (< 4p^2).  All of that needs 4p < R,
  // which holds for both base fields (BN254 Fq: R/p ~ 5.3, BLS12-381 Fq: R/p ~ 9.7) and BN254 Fr, but not
  // BLS12-381 Fr (R/p ~ 2.2); the functions that build such operands assert it.
  // p < 2^(32N-2), i.e. 4p < R.  Covers: two-product sums and four-product sums of reduced values < 4p^2 < p*R
  // (redc's bound); products of unreduced sums < 2p, (2p)^2 = 4p^2 < p*R; and mul() with one operand < 2p, whose
  // running value < a + p < 3p must fit in N limbs (3p < R) and whose product < 2p^2 < p*R.
  static constexpr bool LAZY_HEADROOM = (P::mod(N - 1) >> 30) == 0;
  // K p < R, evaluated on the modulus limbs (BN254 Fq: K <= 5, BLS12-381 Fq: K <= 9, BLS12-377 Fq: K <= 152)
  template <int K>
  ZKB_HD static constexpr bool fits_kp() {
    uint64_t c = 0;
    for (int i = 0; i < N; i++) c = ((uint64_t)P::mod(i) * K + c) >> 32;
    return c == 0;
  }
  struct Wide {
    uint32_t v[2 * N];
  };

  // M p^2 as a Wide: a multiple of p that keeps a difference of products non-negative and below p*R
  template <int M>
  struct PSq {
    uint32_t v[2 * N];
    ZKB_HD constexpr PSq() : v() {
      for (int i = 0; i < N; i++) {
        uint64_t c = 0;
        for (int j = 0; j < N; j++) {
          uint64_t t = (uint64_t)P::mod(i) * P::mod(j) + v[i + j] + c;
          v[i + j] = (uint32_t)t;
          c = t >> 32;
        }
        v[i + N] = (uint32_t)c;
      }
      uint64_t c = 0;
      for (int k = 0; k < 2 * N; k++) {
        uint64_t t = (uint64_t)v[k] * M + c;
        v[k] = (uint32_t)t;
        c = t >> 32;
      }
    }
  };

  // acc[s .. s + 2*cnt) += sum_t x[j0 + 2t] * y * W^(2t), then the carry into acc[s + 2 cnt] (dropped past
  // `size`, where the bound of the caller's value makes it zero).  Every product is one IMAD.WIDE.U32(.X).
  // A carry word only ever receives carries before later rows chain over it, so it never overflows
  // as long as the callers issue rows in order of non-decreasing end word (they do).
  template <int SIZE>
  ZKB_HD static void mad_row(uint32_t (&acc)[SIZE], int s, const uint32_t* x, int j0, int cnt, uint32_t y) {
#pragma unroll
    for (int t = 0; t < cnt; t++) {
      const int k = s + 2 * t;
      if (t == 0)
        ptx::mad_wide_cc(acc[k], acc[k + 1], x[j0], y, acc[k], acc[k + 1]);
      else
        ptx::madc_wide_cc(acc[k], acc[k + 1], x[j0 + 2 * t], y, acc[k], acc[k + 1]);
    }
    if (cnt > 0 && s + 2 * cnt < SIZE) acc[s + 2 * cnt] = ptx::addc(acc[s + 2 * cnt], 0);
  }

  // T = E + O * W  ->  Wide
  ZKB_HD static Wide merge_eo(const uint32_t (&E)[2 * N], const uint32_t (&O)[2 * N]) {
    Wide r;
    r.v[0] = E[0];
    r.v[1] = ptx::add_cc(E[1], O[0]);
#pragma unroll
    for (int k = 2; k < 2 * N - 1; k++) r.v[k] = ptx::addc_cc(E[k], O[k - 1]);
    r.v[2 * N - 1] = ptx::addc(E[2 * N - 1], O[2 * N - 2]);
    return r;
  }

  // a*b, N^2 wide MADs.  Products with i + j even go to E (word i+j), odd ones to O (word i+j-1), so each
  // row of the schoolbook is two independent carry chains.
  ZKB_HD static Wide mul_wide(const Fp& a, const Fp& b) {
    static_assert(N % 2 == 0, "even limb count");
    uint32_t E[2 * N], O[2 * N];
#pragma unroll
    for (int k = 0; k < 2 * N; k++) E[k] = O[k] = 0;
#pragma unroll
    for (int i = 0; i < N; i++) {
      if (i % 2 == 0) {
        mad_row(E, i, a.v, 0, N / 2, b.v[i]);      // even j
        mad_row(O, i, a.v, 1, N / 2, b.v[i]);      // odd j
      } else {
        mad_row(O, i - 1, a.v, 0, N / 2, b.v[i]);  // even j
        mad_row(E, i + 1, a.v, 1, N / 2, b.v[i]);  // odd j
      }
    }
    return merge_eo(E, O);
  }

  // a^2: the N(N-1)/2 off-diagonal products once, doubled, plus the N diagonal squares
  ZKB_HD static Wide sqr_wide(const Fp& a) {
    uint32_t E[2 * N], O[2 * N];
#pragma unroll
    for (int k = 0; k < 2 * N; k++) E[k] = O[k] = 0;
#pragma unroll
    for (int i = 0; i < N - 1; i++) {
      // a_i * a_j, j > i: j - i odd -> O word 2i + (j-i) - 1, j - i even -> E word 2i + (j-i)
      mad_row(O, 2 * i, a.v, i + 1, (N - i) / 2, a.v[i]);
      mad_row(E, 2 * i + 2, a.v, i + 2, (N - 1 - i) / 2, a.v[i]);
    }
    Wide t = merge_eo(E, O);  // off-diagonal sum < a^2 / 2, so the doubling below loses no bit
    Wide r;
    r.v[0] = 0;
#pragma unroll
    for (int k = 2 * N - 1; k >= 1; k--) r.v[k] = (t.v[k] << 1) | (t.v[k - 1] >> 31);
    ptx::mad_wide_cc(r.v[0], r.v[1], a.v[0], a.v[0], r.v[0], r.v[1]);
#pragma unroll
    for (int i = 1; i < N; i++) ptx::madc_wide_cc(r.v[2 * i], r.v[2 * i + 1], a.v[i], a.v[i], r.v[2 * i], r.v[2 * i + 1]);
    return r;
  }

  // T * R^-1 mod p for T < p*R, fully reduced: N^2 wide MADs + N m-multiplications.  The low half is reduced
  // with the split-accumulator rows of mul() (the shift folded into the next row's addends), giving
  // (T_lo + M p) / R <= p; adding T_hi < p leaves a value < 2p for the one final conditional subtraction.
  ZKB_HD static Fp redc(const Wide& T) {
    uint32_t E[N], O[N];
#pragma unroll
    for (int j = 0; j < N; j++) {
      E[j] = T.v[j];
      O[j] = 0;
    }
    {
      const uint32_t m = E[0] * P::INV;
      ptx::mad_wide_cc(O[0], O[1], P::mod(1), m, O[0], O[1]);
#pragma unroll
      for (int j = 3; j < N; j += 2) ptx::madc_wide_cc(O[j - 1], O[j], P::mod(j), m, O[j - 1], O[j]);
      ptx::mad_wide_cc(E[0], E[1], P::mod(0), m, E[0], E[1]);
#pragma unroll
      for (int j = 2; j < N; j += 2) ptx::madc_wide_cc(E[j], E[j + 1], P::mod(j), m, E[j], E[j + 1]);
      O[N - 1] = ptx::addc(O[N - 1], 0);
    }
#pragma unroll
    for (int i = 1; i < N; i++) {
      // value = O + (E >> 32); add m*p with m chosen from its low word, re-pairing E and O as mul() does
      uint32_t nE[N], nO[N];
      nE[0] = ptx::add_cc(O[0], E[1]);
      const uint32_t m = nE[0] * P::INV;
#pragma unroll
      for (int j = 1; j < N - 1; j += 2) ptx::madc_wide_cc(nO[j - 1], nO[j], P::mod(j), m, E[j + 1], E[j + 2]);
      ptx::madc_wide(nO[N - 2], nO[N - 1], P::mod(N - 1), m, 0, 0);
      ptx::mad_wide_cc(nE[0], nE[1], P::mod(0), m, nE[0], O[1]);
#pragma unroll
      for (int j = 2; j < N; j += 2) ptx::madc_wide_cc(nE[j], nE[j + 1], P::mod(j), m, O[j], O[j + 1]);
      nO[N - 1] = ptx::addc(nO[N - 1], 0);
#pragma unroll
      for (int j = 0; j < N; j++) {
        E[j] = nE[j];
        O[j] = nO[j];
      }
    }
    // (T_lo + M p) / R = O + (E >> 32); then + T_hi
    Fp t;
    t.v[0] = ptx::add_cc(O[0], E[1]);
#pragma unroll
    for (int k = 1; k < N - 1; k++) t.v[k] = ptx::addc_cc(O[k], E[k + 1]);
    t.v[N - 1] = ptx::addc(O[N - 1], 0);
    t.v[0] = ptx::add_cc(t.v[0], T.v[N]);
#pragma unroll
    for (int k = 1; k < N - 1; k++) t.v[k] = ptx::addc_cc(t.v[k], T.v[N + k]);
    t.v[N - 1] = ptx::addc(t.v[N - 1], T.v[2 * N - 1]);
    return reduce_once(t);
  }

  ZKB_HD static Wide add_wide(const Wide& a, const Wide& b) {  // caller guarantees no overflow
    Wide r;
    r.v[0] = ptx::add_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int k = 1; k < 2 * N - 1; k++) r.v[k] = ptx::addc_cc(a.v[k], b.v[k]);
    r.v[2 * N - 1] = ptx::addc(a.v[2 * N - 1], b.v[2 * N - 1]);
    return r;
  }
  ZKB_HD static Wide sub_wide(const Wide& a, const Wide& b) {  // caller guarantees a >= b
    Wide r;
    r.v[0] = ptx::sub_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int k = 1; k < 2 * N - 1; k++) r.v[k] = ptx::subc_cc(a.v[k], b.v[k]);
    r.v[2 * N - 1] = ptx::subc(a.v[2 * N - 1], b.v[2 * N - 1]);
    return r;
  }
  // a + M p^2.  Callers add it to a sum of at most two products of reduced values (< 2p^2) before subtracting
  // at most M p^2, so the operand of the following redc is < (M + 2) p^2, and (M + 2) p < R keeps it < p*R.
  template <int M>
  ZKB_HD static Wide add_psq(const Wide& a) {
    static_assert(fits_kp<M + 2>(), "M p^2 plus the operand must stay < p*R");
    constexpr PSq<M> K{};
    Wide r;
    r.v[0] = ptx::add_cc(a.v[0], K.v[0]);
#pragma unroll
    for (int i = 1; i < 2 * N - 1; i++) r.v[i] = ptx::addc_cc(a.v[i], K.v[i]);
    r.v[2 * N - 1] = ptx::addc(a.v[2 * N - 1], K.v[2 * N - 1]);
    return r;
  }
  // 5a as (a << 2) + a, for fp2.cuh's beta = -5 products; caller guarantees 5a < 2^(64N)
  ZKB_HD static Wide mul5_wide(const Wide& a) {
    Wide s;
#pragma unroll
    for (int k = 2 * N - 1; k >= 1; k--) s.v[k] = (a.v[k] << 2) | (a.v[k - 1] >> 30);
    s.v[0] = a.v[0] << 2;
    return add_wide(s, a);
  }
  // a + b without the conditional subtraction: < 2p for reduced inputs; only for mul_wide/mul operands
  ZKB_HD static Fp add_nr(const Fp& a, const Fp& b) {
    static_assert(LAZY_HEADROOM, "a product of two unreduced sums (< 4p^2) must stay < p*R");
    Fp t;
    t.v[0] = ptx::add_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) t.v[i] = ptx::addc_cc(a.v[i], b.v[i]);
    t.v[N - 1] = ptx::addc(a.v[N - 1], b.v[N - 1]);
    return t;
  }

  // a*b - c*d with one reduction: a*b + c*(p - d), operand < 2p^2 < p*R
  ZKB_HD static Fp mul_sub(const Fp& a, const Fp& b, const Fp& c, const Fp& d) {
    static_assert(LAZY_HEADROOM, "a sum of two products (< 2p^2) must stay < p*R");
    return redc(add_wide(mul_wide(a, b), mul_wide(c, neg(d))));
  }

  ZKB_HD static Fp sqr(const Fp& a) { return redc(sqr_wide(a)); }
  // out-of-line copies for cold code (scalar multiplications, inversions, final combination): keeps
  // code size and compile time down; hot kernels use the inlined mul().
  ZKB_NI static Fp mul_ni(const Fp& a, const Fp& b) { return mul(a, b); }

  ZKB_HD static Fp to_mont(const Fp& a) { return mul(a, r2()); }
  ZKB_HD static Fp from_mont(const Fp& a) {
    Fp o = zero();
    o.v[0] = 1;
    return mul(a, o);
  }

  // a^e for a little-endian 32-bit-limb exponent with N limbs (square-and-multiply, MSB first)
  ZKB_NI static Fp pow_limbs(const Fp& a, const uint32_t* e, int nlimbs) {
    Fp r = one();
    bool started = false;
    for (int i = nlimbs - 1; i >= 0; i--) {
      for (int b = 31; b >= 0; b--) {
        if (started) r = mul_ni(r, r);
        if ((e[i] >> b) & 1) {
          r = started ? mul_ni(r, a) : a;
          started = true;
        }
      }
    }
    return r;
  }

  // Fermat inverse a^(p-2); inv(0) = 0
  ZKB_NI static Fp inv(const Fp& a) {
    uint32_t e[N];
#pragma unroll
    for (int i = 0; i < N; i++) e[i] = P::pm2(i);
    return pow_limbs(a, e, N);
  }

  ZKB_NI static Fp pow_u64(const Fp& a, uint64_t k) {
    uint32_t e[2] = {(uint32_t)k, (uint32_t)(k >> 32)};
    return pow_limbs(a, e, 2);
  }
};

}  // namespace zkb
