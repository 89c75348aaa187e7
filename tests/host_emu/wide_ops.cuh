// Op wrappers (TEST ONLY) over the separated Montgomery arithmetic of fp.cuh / fp2.cuh and the point additions of
// ec.cuh, shared by the g++ harness (emu_wide.cpp) and the device harness (dev_wide.cu), so that both run the same
// code on the same cases: the host build steps the carry emulation of hd.cuh, the device build its inline PTX.
// Limbs are little-endian uint32.
#pragma once
#include "ec.cuh"

namespace zkb {
namespace wide {

template <class P>
ZKB_HD Fp<P> ld(const uint32_t* a) {
  Fp<P> x;
  for (int i = 0; i < P::N; i++) x.v[i] = a[i];
  return x;
}
template <class P>
ZKB_HD void st(const Fp<P>& x, uint32_t* o) {
  for (int i = 0; i < P::N; i++) o[i] = x.v[i];
}
template <class P>
ZKB_HD Fp2<P> ld2(const uint32_t* a) {
  return Fp2<P>{ld<P>(a), ld<P>(a + P::N)};
}
template <class P>
ZKB_HD void st2(const Fp2<P>& x, uint32_t* o) {
  st<P>(x.c0, o);
  st<P>(x.c1, o + P::N);
}

// op 0: mul_wide(a, b) -> 2N limbs   1: sqr_wide(a) -> 2N   2: redc(a as 2N limbs) -> N
//    3: sqr(a) -> N                  4: mul_sub(a, b, c, d) -> N
template <class P>
ZKB_HD void fp_op(int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* o) {
  typedef Fp<P> F;
  typename F::Wide w;
  switch (op) {
    case 0:
      w = F::mul_wide(ld<P>(a), ld<P>(b));
      for (int i = 0; i < 2 * P::N; i++) o[i] = w.v[i];
      break;
    case 1:
      w = F::sqr_wide(ld<P>(a));
      for (int i = 0; i < 2 * P::N; i++) o[i] = w.v[i];
      break;
    case 2:
      for (int i = 0; i < 2 * P::N; i++) w.v[i] = a[i];
      st<P>(F::redc(w), o);
      break;
    case 3: st<P>(F::sqr(ld<P>(a)), o); break;
    case 4:  // lazy sums need 4p < R (not BLS12-381 Fr)
      if constexpr (F::LAZY_HEADROOM) st<P>(F::mul_sub(ld<P>(a), ld<P>(b), ld<P>(c), ld<P>(d)), o);
      break;
  }
}

// op 0: mul_v(a, b)   1: sqr_v(a)   2: mul_sub_v(a, b, c, d)     (each operand 2N limbs: c0 then c1)
template <class P>
ZKB_HD void fp2_op(int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* o) {
  typedef Fp2<P> F;
  switch (op) {
    case 0: st2<P>(F::mul_v(ld2<P>(a), ld2<P>(b)), o); break;
    case 1: st2<P>(F::sqr_v(ld2<P>(a)), o); break;
    case 2: st2<P>(F::mul_sub_v(ld2<P>(a), ld2<P>(b), ld2<P>(c), ld2<P>(d)), o); break;
  }
}

// op 0: madd(acc, q)   1: add(acc, b).  Points are XYZZ (x, y, zz, zzz) / affine (x, y), coordinates of
// `K` base-field elements each (K = 1 for G1, 2 for G2); the result is XYZZ.
template <class F, int K, class P>
ZKB_HD F ldf(const uint32_t* a) {
  if constexpr (K == 1) return ld<P>(a); else return ld2<P>(a);
}
template <class F, int K, class P>
ZKB_HD void stf(const F& x, uint32_t* o) {
  if constexpr (K == 1) st<P>(x, o); else st2<P>(x, o);
}
template <class F, int K, class P>
ZKB_HD void ec_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* o) {
  const int S = K * P::N;
  XYZZ<F> acc{ldf<F, K, P>(a), ldf<F, K, P>(a + S), ldf<F, K, P>(a + 2 * S), ldf<F, K, P>(a + 3 * S)}, r;
  if (op == 0) {
    r = XYZZ<F>::madd(acc, Affine<F>{ldf<F, K, P>(b), ldf<F, K, P>(b + S)});
  } else {
    XYZZ<F> q{ldf<F, K, P>(b), ldf<F, K, P>(b + S), ldf<F, K, P>(b + 2 * S), ldf<F, K, P>(b + 3 * S)};
    r = XYZZ<F>::add(acc, q);
  }
  stf<F, K, P>(r.x, o);
  stf<F, K, P>(r.y, o + S);
  stf<F, K, P>(r.zz, o + 2 * S);
  stf<F, K, P>(r.zzz, o + 3 * S);
}

// Case i of a batch: every operand and result sits at a fixed stride per case (uint32 limbs).
//   fp : a 2N (a redc input is 2N limbs), b / c / d N, result 2N
//   fp2: every operand and the result 2N
//   ec : every operand and the result 4 K N
template <class P>
ZKB_HD void fp_case(int op, size_t i, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* o) {
  const size_t n = P::N;
  fp_op<P>(op, a + 2 * n * i, b + n * i, c + n * i, d + n * i, o + 2 * n * i);
}
template <class P>
ZKB_HD void fp2_case(int op, size_t i, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* o) {
  const size_t s = 2 * P::N;
  fp2_op<P>(op, a + s * i, b + s * i, c + s * i, d + s * i, o + s * i);
}
template <class F, int K, class P>
ZKB_HD void ec_case(int op, size_t i, const uint32_t* a, const uint32_t* b, uint32_t* o) {
  const size_t s = 4 * K * P::N;
  ec_op<F, K, P>(op, a + s * i, b + s * i, o + s * i);
}

}  // namespace wide
}  // namespace zkb
