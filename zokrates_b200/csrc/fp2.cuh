// Quadratic extension Fq2 = Fq[u]/(u^2 - beta) used by G2: beta = -1 for BN254 and BLS12-381, beta = -5 for BLS12-377
// (ark-bn254 / ark-bls12-381 / ark-bls12-377 0.3.0 Fq2Parameters::NONRESIDUE; SURVEY.md App. C).  beta is B::FP2_NONRESIDUE,
// a compile-time property of the base field; the beta = -1 code is the same as before beta became a parameter.
// Same static interface as Fp<P> so the curve code is generic over the coordinate field.
#pragma once
#include "fp.cuh"

namespace zkb {

template <class Bt>
struct Fp2T {
  typedef Bt B;
  typedef Fp2T Fp2;
  static constexpr int NR = B::FP2_NONRESIDUE;
  static_assert(NR == -1 || NR == -5, "Fq2 formulas exist for u^2 = -1 and u^2 = -5");
  B c0, c1;

  ZKB_HD static Fp2 zero() { return Fp2{B::zero(), B::zero()}; }
  ZKB_HD static Fp2 one() { return Fp2{B::one(), B::zero()}; }
  ZKB_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  ZKB_HD bool operator==(const Fp2& o) const { return c0 == o.c0 && c1 == o.c1; }
  ZKB_HD bool operator!=(const Fp2& o) const { return !(*this == o); }
  ZKB_HD static Fp2 add(const Fp2& a, const Fp2& b) { return Fp2{B::add(a.c0, b.c0), B::add(a.c1, b.c1)}; }
  ZKB_HD static Fp2 sub(const Fp2& a, const Fp2& b) { return Fp2{B::sub(a.c0, b.c0), B::sub(a.c1, b.c1)}; }
  ZKB_HD static Fp2 neg(const Fp2& a) { return Fp2{B::neg(a.c0), B::neg(a.c1)}; }
  ZKB_HD static Fp2 dbl(const Fp2& a) { return Fp2{B::dbl(a.c0), B::dbl(a.c1)}; }
  // Karatsuba: 3 base-field multiplications (M2 = 3 in SURVEY.md §8d's accounting); complex squaring: 2 (S2 = 2).
  // Both are OUT OF LINE with by-value arguments: ptxas passes the operands in registers (no local-memory traffic), and
  // the G2 mixed addition shrinks from ~6 560 SASS instructions (105 KB, `no_instruction` the top stall of the round-1
  // G2 accumulate kernel — the instruction cache is 32 KB) to ~2 000: ten calls into one ~600-instruction body.
  //
  // Lazy reduction (fp.cuh's Wide): the three Karatsuba products stay 2N limbs wide and each coordinate is
  // reduced once, so a multiplication is 3 wide products + 2 redc instead of 3 full multiplications.  The
  // bounds below are for reduced inputs (< p); fp.cuh asserts 4p < R, i.e. p*R > 4p^2.
  //
  // beta = -5: c0 = a0 b0 - 5 a1 b1.  5 p^2 keeps it non-negative: redc(v0 + 5p^2 - 5 v1) < 6p^2 (add_psq<5> asserts
  // 7p < R; BLS12-377 Fq has R/p ~ 152).  5 v1 < 5p^2 is a shift and an add (mul5_wide).
  ZKB_HD static B mul5(const B& x) { return B::add(B::dbl(B::dbl(x)), x); }
  // c0 = t + beta v1 reduced once, for v1 < M p^2: beta = -1: redc(t + M p^2 - v1), beta = -5: redc(t + 5M p^2 - 5 v1)
  template <int M, class Wd>
  ZKB_HD static B redc_c0(const Wd& t, const Wd& v1) {
    if constexpr (NR == -1) return B::redc(B::sub_wide(B::template add_psq<M>(t), v1));
    else return B::redc(B::sub_wide(B::template add_psq<5 * M>(t), B::mul5_wide(v1)));
  }
  ZKB_NI static Fp2 mul_v(Fp2 a, Fp2 b) {
    if constexpr (!B::LAZY_HEADROOM) {  // fp64.cuh's host tail: every product reduced
      B v0 = B::mul(a.c0, b.c0), v1 = B::mul(a.c1, b.c1);
      B s = B::mul(B::add(a.c0, a.c1), B::add(b.c0, b.c1));
      if constexpr (NR == -1) return Fp2{B::sub(v0, v1), B::sub(B::sub(s, v0), v1)};
      else return Fp2{B::sub(v0, mul5(v1)), B::sub(B::sub(s, v0), v1)};
    } else {
      typedef typename B::Wide Wd;
      Wd v0 = B::mul_wide(a.c0, b.c0);                                       // < p^2
      Wd v1 = B::mul_wide(a.c1, b.c1);                                       // < p^2
      Wd s = B::mul_wide(B::add_nr(a.c0, a.c1), B::add_nr(b.c0, b.c1));      // sums < 2p: s < 4p^2
      B c1 = B::redc(B::sub_wide(B::sub_wide(s, v0), v1));                   // a0 b1 + a1 b0 < 2p^2
      B c0 = redc_c0<1>(v0, v1);                                             // 0 < v0 + p^2 - v1 < 2p^2 (beta = -5: < 6p^2)
      return Fp2{c0, c1};
    }
  }
  // complex squaring: (a0 + a1)(a0 - a1) and 2 a0 a1 with the sums left unreduced (< 2p).  The CIOS mul() reduces
  // fully with one operand < 2p and the other < p: its running value stays < 3p < R and the product < 2p^2 < p*R
  // (fp.cuh, next to LAZY_HEADROOM; add_nr asserts it)
  //
  // beta = -5: t = a0 a1, c0 = (a0 + a1)(a0 - 5 a1) + 4t, c1 = 2t: two CIOS multiplications, the sum unreduced (< 2p).  Chosen
  // by SASS count on sm_90a (one out-of-line sqr_v per kernel): 1328 instructions, 289 IMAD.WIDE, against 1352 and 298 for
  // redc(a0^2 + 5p^2 - 5 a1^2) from two wide squares plus c1 = mul(2 a0, a1).
  ZKB_NI static Fp2 sqr_v(Fp2 a) {
    if constexpr (NR == -1) {
      B r0 = B::mul(B::add_nr(a.c0, a.c1), B::sub(a.c0, a.c1));
      B r1 = B::mul(B::add_nr(a.c0, a.c0), a.c1);
      return Fp2{r0, r1};
    } else {
      B t = B::mul(a.c0, a.c1);
      B r0 = B::add(B::mul(B::add_nr(a.c0, a.c1), B::sub(a.c0, mul5(a.c1))), B::dbl(B::dbl(t)));
      return Fp2{r0, B::dbl(t)};
    }
  }
  // a*b - c*d with two reductions: a*b + c*(-d) as six wide products
  // beta = -5: c0 = v0 + w0 - 5 v1 with v1 < 2p^2, so redc(v0 + w0 + 10p^2 - 5 v1) < 12p^2 (add_psq<10>: 12p < R).
  ZKB_NI static Fp2 mul_sub_v(Fp2 a, Fp2 b, Fp2 c, Fp2 d) {
    if constexpr (!B::LAZY_HEADROOM) {
      return sub(mul_v(a, b), mul_v(c, d));
    } else {
      typedef typename B::Wide Wd;
      Fp2 e = neg(d);
      Wd v0 = B::mul_wide(a.c0, b.c0);                                       // < p^2
      Wd w0 = B::mul_wide(c.c0, e.c0);                                       // < p^2
      Wd v1 = B::add_wide(B::mul_wide(a.c1, b.c1), B::mul_wide(c.c1, e.c1));  // < 2p^2
      Wd s = B::add_wide(B::mul_wide(B::add_nr(a.c0, a.c1), B::add_nr(b.c0, b.c1)),
                         B::mul_wide(B::add_nr(c.c0, c.c1), B::add_nr(e.c0, e.c1)));  // < 8p^2 < 2^(64N)
      B c1 = B::redc(B::sub_wide(B::sub_wide(B::sub_wide(s, v0), w0), v1));  // a0b1 + a1b0 + c0e1 + c1e0 < 4p^2
      B c0 = redc_c0<2>(B::add_wide(v0, w0), v1);                            // 0 < v0 + w0 + 2p^2 - v1 < 4p^2 (beta = -5: < 12p^2)
      return Fp2{c0, c1};
    }
  }
  ZKB_HD static Fp2 mul_sub(const Fp2& a, const Fp2& b, const Fp2& c, const Fp2& d) { return mul_sub_v(a, b, c, d); }
  ZKB_HD static Fp2 mul(const Fp2& a, const Fp2& b) { return mul_v(a, b); }
  ZKB_HD static Fp2 sqr(const Fp2& a) { return sqr_v(a); }
  ZKB_HD static Fp2 mul_ni(const Fp2& a, const Fp2& b) { return mul_v(a, b); }
  ZKB_HD static B norm(const Fp2& a) {  // c0^2 - beta c1^2
    if constexpr (NR == -1) return B::add(B::sqr(a.c0), B::sqr(a.c1));
    else return B::add(B::sqr(a.c0), mul5(B::sqr(a.c1)));
  }
  ZKB_NI static Fp2 inv(const Fp2& a) {
    B d = B::inv(norm(a));
    return Fp2{B::mul(a.c0, d), B::neg(B::mul(a.c1, d))};
  }
  ZKB_HD static Fp2 to_mont(const Fp2& a) { return Fp2{B::to_mont(a.c0), B::to_mont(a.c1)}; }
  ZKB_HD static Fp2 from_mont(const Fp2& a) { return Fp2{B::from_mont(a.c0), B::from_mont(a.c1)}; }
};

template <class P>
using Fp2 = Fp2T<Fp<P>>;

}  // namespace zkb
