// Quadratic extension Fq2 = Fq[u]/(u^2 + 1) used by G2 of BN254 and BLS12-381
// (ark-bn254 / ark-bls12-381 0.3.0 Fq2Parameters::NONRESIDUE = -1; SURVEY.md App. C).
// Same static interface as Fp<P> so the curve code is generic over the coordinate field.
#pragma once
#include "fp.cuh"

namespace zkb {

template <class Bt>
struct Fp2T {
  typedef Bt B;
  typedef Fp2T Fp2;
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
  ZKB_NI static Fp2 mul_v(Fp2 a, Fp2 b) {
    if constexpr (!B::LAZY_HEADROOM) {  // fp64.cuh's host tail: every product reduced
      B v0 = B::mul(a.c0, b.c0), v1 = B::mul(a.c1, b.c1);
      B s = B::mul(B::add(a.c0, a.c1), B::add(b.c0, b.c1));
      return Fp2{B::sub(v0, v1), B::sub(B::sub(s, v0), v1)};
    } else {
      typedef typename B::Wide Wd;
      Wd v0 = B::mul_wide(a.c0, b.c0);                                       // < p^2
      Wd v1 = B::mul_wide(a.c1, b.c1);                                       // < p^2
      Wd s = B::mul_wide(B::add_nr(a.c0, a.c1), B::add_nr(b.c0, b.c1));      // sums < 2p: s < 4p^2
      B c1 = B::redc(B::sub_wide(B::sub_wide(s, v0), v1));                   // a0 b1 + a1 b0 < 2p^2
      B c0 = B::redc(B::sub_wide(B::template add_psq<1>(v0), v1));           // 0 < v0 + p^2 - v1 < 2p^2
      return Fp2{c0, c1};
    }
  }
  // complex squaring: (a0 + a1)(a0 - a1) and 2 a0 a1 with the sums left unreduced (< 2p).  The CIOS mul() reduces
  // fully with one operand < 2p and the other < p: its running value stays < 3p < R and the product < 2p^2 < p*R
  // (fp.cuh, next to LAZY_HEADROOM; add_nr asserts it)
  ZKB_NI static Fp2 sqr_v(Fp2 a) {
    B r0 = B::mul(B::add_nr(a.c0, a.c1), B::sub(a.c0, a.c1));
    B r1 = B::mul(B::add_nr(a.c0, a.c0), a.c1);
    return Fp2{r0, r1};
  }
  // a*b - c*d with two reductions: a*b + c*(-d) as six wide products
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
      B c0 = B::redc(B::sub_wide(B::template add_psq<2>(B::add_wide(v0, w0)), v1));  // 0 < v0 + w0 + 2p^2 - v1 < 4p^2
      return Fp2{c0, c1};
    }
  }
  ZKB_HD static Fp2 mul_sub(const Fp2& a, const Fp2& b, const Fp2& c, const Fp2& d) { return mul_sub_v(a, b, c, d); }
  ZKB_HD static Fp2 mul(const Fp2& a, const Fp2& b) { return mul_v(a, b); }
  ZKB_HD static Fp2 sqr(const Fp2& a) { return sqr_v(a); }
  ZKB_HD static Fp2 mul_ni(const Fp2& a, const Fp2& b) { return mul_v(a, b); }
  ZKB_NI static Fp2 inv(const Fp2& a) {
    B d = B::inv(B::add(B::sqr(a.c0), B::sqr(a.c1)));
    return Fp2{B::mul(a.c0, d), B::neg(B::mul(a.c1, d))};
  }
  ZKB_HD static Fp2 to_mont(const Fp2& a) { return Fp2{B::to_mont(a.c0), B::to_mont(a.c1)}; }
  ZKB_HD static Fp2 from_mont(const Fp2& a) { return Fp2{B::from_mont(a.c0), B::from_mont(a.c1)}; }
};

template <class P>
using Fp2 = Fp2T<Fp<P>>;

}  // namespace zkb
