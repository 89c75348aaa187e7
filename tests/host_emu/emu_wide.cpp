// Host emulation harness (TEST ONLY) for the separated Montgomery arithmetic of fp.cuh / fp2.cuh and the
// point additions of ec.cuh: the device headers compiled as plain C++.  Limbs are little-endian uint32.
#include "ec.cuh"
using namespace zkb;

template <class P>
static Fp<P> ld(const uint32_t* a) {
  Fp<P> x;
  for (int i = 0; i < P::N; i++) x.v[i] = a[i];
  return x;
}
template <class P>
static void st(const Fp<P>& x, uint32_t* o) {
  for (int i = 0; i < P::N; i++) o[i] = x.v[i];
}
template <class P>
static Fp2<P> ld2(const uint32_t* a) {
  return Fp2<P>{ld<P>(a), ld<P>(a + P::N)};
}
template <class P>
static void st2(const Fp2<P>& x, uint32_t* o) {
  st<P>(x.c0, o);
  st<P>(x.c1, o + P::N);
}

// op 0: mul_wide(a, b) -> 2N limbs   1: sqr_wide(a) -> 2N   2: redc(a as 2N limbs) -> N
//    3: sqr(a) -> N                  4: mul_sub(a, b, c, d) -> N
template <class P>
static void fp_op(int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* o) {
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
static void fp2_op(int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* o) {
  typedef Fp2<P> F;
  switch (op) {
    case 0: st2<P>(F::mul_v(ld2<P>(a), ld2<P>(b)), o); break;
    case 1: st2<P>(F::sqr_v(ld2<P>(a)), o); break;
    case 2: st2<P>(F::mul_sub_v(ld2<P>(a), ld2<P>(b), ld2<P>(c), ld2<P>(d)), o); break;
  }
}

// op 0: madd(acc, q)   1: add(acc, b).  Points are XYZZ (x, y, zz, zzz) / affine (x, y), coordinates of
// `k` base-field elements each (k = 1 for G1, 2 for G2); the result is XYZZ.
template <class F, int K, class P>
static F ldf(const uint32_t* a) {
  if constexpr (K == 1) return ld<P>(a); else return ld2<P>(a);
}
template <class F, int K, class P>
static void stf(const F& x, uint32_t* o) {
  if constexpr (K == 1) st<P>(x, o); else st2<P>(x, o);
}
template <class F, int K, class P>
static void ec_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* o) {
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

extern "C" void emu_wide_fp(int field, int op, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                            const uint32_t* d, uint32_t* o) {
  switch (field) {
    case 0: fp_op<Bn254Fr>(op, a, b, c, d, o); break;
    case 1: fp_op<Bn254Fq>(op, a, b, c, d, o); break;
    case 2: fp_op<Bls381Fr>(op, a, b, c, d, o); break;
    case 3: fp_op<Bls381Fq>(op, a, b, c, d, o); break;
  }
}
// curve 0: BN254 Fq2, 1: BLS12-381 Fq2
extern "C" void emu_wide_fp2(int curve, int op, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                             const uint32_t* d, uint32_t* o) {
  if (curve == 0) fp2_op<Bn254Fq>(op, a, b, c, d, o);
  else fp2_op<Bls381Fq>(op, a, b, c, d, o);
}
// curve 0: BN254, 1: BLS12-381; group 1: G1, 2: G2
extern "C" void emu_wide_ec(int curve, int group, int op, const uint32_t* a, const uint32_t* b, uint32_t* o) {
  if (curve == 0) {
    if (group == 1) ec_op<Fp<Bn254Fq>, 1, Bn254Fq>(op, a, b, o);
    else ec_op<Fp2<Bn254Fq>, 2, Bn254Fq>(op, a, b, o);
  } else {
    if (group == 1) ec_op<Fp<Bls381Fq>, 1, Bls381Fq>(op, a, b, o);
    else ec_op<Fp2<Bls381Fq>, 2, Bls381Fq>(op, a, b, o);
  }
}
