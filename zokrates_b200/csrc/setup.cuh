// Circuit-specific Groth16 setup on the device from an explicit trapdoor.
//
// Follows ark-groth16 0.3.0 `generate_parameters` (external crate; reached from
// `Groth16::circuit_specific_setup`, /root/reference/zokrates_ark/src/groth16.rs:95; restated in
// SURVEY.md App. B.6) and writes the key in ark's `serialize_unchecked` layout (groth16.rs:97-98,
// App. A.3).  Trapdoor sampling (ark draws alpha..delta, two random generators and tau from the
// rng) stays with the caller — this entry point is deterministic in the trapdoor, which is what the
// benchmarks and the trapdoor parity check need (SURVEY.md §8c).
//
//   u_j   = L_j(tau)                          = ifft(tau^0 .. tau^(n-1))_j
//   a_i   = (A^T u)_i (+ u_{N+i} for instance i),  b_i = (B^T u)_i,  c_i = (C^T u)_i
//   gamma_abc_i = (beta a_i + alpha b_i + c_i) / gamma   (i < ni),   l_i = (...) / delta   (i >= ni)
//   h_k   = tau^k (tau^n - 1) / delta          (k < n - 1)
// and every point is a fixed-base multiple of the (scaled) generator, done with an 8-bit window table.
#pragma once
#include <algorithm>
#include "engine.cuh"

namespace zkb {

template <class Gen, class Fq>
ZKB_HD Affine<Fq> std_g1() {
  Affine<Fq> g;
  for (int i = 0; i < Fq::N; i++) { g.x.v[i] = Gen::g1x(i); g.y.v[i] = Gen::g1y(i); }
  return g;
}
template <class Gen, class Fq2>
ZKB_HD Affine<Fq2> std_g2() {
  Affine<Fq2> g;
  for (int i = 0; i < Fq2::B::N; i++) {
    g.x.c0.v[i] = Gen::g2x0(i); g.x.c1.v[i] = Gen::g2x1(i);
    g.y.c0.v[i] = Gen::g2y0(i); g.y.c1.v[i] = Gen::g2y1(i);
  }
  return g;
}

template <class C> struct GenOf;
template <> struct GenOf<CurveT<Bn254Fr, Bn254Fq>> { typedef Bn254Gen T; };
template <> struct GenOf<CurveT<Bls381Fr, Bls381Fq>> { typedef Bls381Gen T; };
template <> struct GenOf<CurveT<Bls377Fr, Bls377Fq>> { typedef Bls377Gen T; };

// write one affine point in ark's uncompressed encoding (canonical LE, infinity flag 0x40 on the last byte)
template <class F>
ZKB_HD void write_ark_point(uint32_t* out, const Affine<F>& a) {
  const int words = sizeof(Affine<F>) / 4;
  if (a.is_inf()) {
    for (int i = 0; i < words; i++) out[i] = 0;
    out[words - 1] = 0x40000000u;
  } else {
    Affine<F> c{F::from_mont(a.x), F::from_mont(a.y)};
    const uint32_t* raw = (const uint32_t*)&c;
    for (int i = 0; i < words; i++) out[i] = raw[i];
  }
}

template <class C>
template <class F>
void Engine<C>::fb_build(FixedBase<F>& fb, Affine<F> stdgen, const uint32_t* gk) {
  typedef XYZZ<F> X;
  typedef Affine<F> A;
  fb.table.alloc(32 * 256);
  fb.bases.alloc(32);
  X* bases = fb.bases.p;
  A* table = fb.table.p;
  launch<k_fixed_base, 1>(st_, 1, ZKB_LAMBDA(size_t) {
    X g = X::mul_affine(stdgen, gk, 8);
    for (int j = 0; j < 32; j++) {
      bases[j] = g;
      for (int b = 0; b < 8; b++) g = X::dbl_ni(g);
    }
  });
  launch<k_fixed_base>(st_, 32 * 256, ZKB_LAMBDA(size_t t) {
    uint32_t dgt = (uint32_t)(t & 255);
    X acc = X::mul_xyzz(bases[t >> 8], &dgt, 1);
    table[t] = X::to_affine(acc);
  });
}

template <class C>
template <class F>
void Engine<C>::fb_emit(const FixedBase<F>& fb, const Fr* scalars, size_t count, uint32_t* dst) {
  typedef XYZZ<F> X;
  typedef Affine<F> A;
  const A* table = fb.table.p;
  launch<k_fixed_base>(st_, count, ZKB_LAMBDA(size_t t) {
    Fr s = Fr::from_mont(scalars[t]);
    X acc = X::identity();
    for (int j = 0; j < 32; j++) {
      uint32_t dgt = (s.v[j >> 2] >> ((j & 3) * 8)) & 255u;
      if (dgt) acc = X::madd_ni(acc, table[j * 256 + dgt]);
    }
    write_ark_point<F>(dst + t * (sizeof(A) / 4), X::to_affine(acc));
  });
}

template <class C>
size_t Engine<C>::setup_size(uint64_t rh) {
  R1cs& r = get_r1cs(rh);
  const size_t n = (size_t)1 << r.log_n;
  return G1B + 3 * G2B + 8 + r.ni * G1B + 2 * G1B + (8 + r.m * G1B) * 2 + 8 + r.m * G2B + 8 + (n - 1) * G1B + 8 +
         (r.m - r.ni) * G1B;
}

template <class C>
void Engine<C>::setup(uint64_t rh, const uint64_t* trapdoor7, uint8_t* pk_out, size_t cap, size_t* len) {
  typedef typename GenOf<C>::T Gen;
  R1cs& r = get_r1cs(rh);
  const uint32_t lg = r.log_n;
  const size_t n = (size_t)1 << lg;
  const size_t total = setup_size(rh);
  if (cap < total) throw Error(ZKB_E_ARG, "pk_out too small");
  StageTimer tm(st_);
  DomainT& d = domain(lg);
  const uint32_t N = (uint32_t)r.N, ni = (uint32_t)r.ni, m = (uint32_t)r.m;

  // trapdoor scalars (host-side constants; a handful of field operations)
  Fr td[7];
  for (int k = 0; k < 7; k++) {
    Fr c;
    for (int i = 0; i < 8; i++) c.v[i] = ((const uint32_t*)trapdoor7)[k * 8 + i];
    td[k] = Fr::to_mont(c);
  }
  const Fr alpha = td[0], beta = td[1], gamma = td[2], delta = td[3], tau = td[4];
  const Fr ginv = Fr::inv(gamma), dinv = Fr::inv(delta);
  Fr tn = tau;
  for (uint32_t i = 0; i < lg; i++) tn = Fr::sqr(tn);
  const Fr zt = Fr::sub(tn, Fr::one());
  const Fr hscale = Fr::mul(zt, dinv);

  tm.begin("setup_scalars");
  // u = ifft(powers of tau), natural order, Montgomery
  DevBuf<Fr> pw(n), u(n);
  {
    Fr one = Fr::one();
    Fr* pp = pw.p;
    launch<k_ntt_table>(st_, n, ZKB_LAMBDA(size_t t) { ntt_powers_body<Fr>(tau, one, pp, (uint32_t)n, (uint32_t)t); });
    d2d(st_, u.p, pw.p, n * FRB);
    ntt_dif(u.p, d.tw_inv.p, lg);
    scratch_a_.ensure(n);
    Fr* src = u.p; Fr* dst = scratch_a_.p;
    Fr ninv = d.ninv;
    launch<k_ntt_brev>(st_, n, ZKB_LAMBDA(size_t t) { dst[bitrev32((uint32_t)t, lg)] = Fr::mul(src[t], ninv); });
    d2d(st_, u.p, scratch_a_.p, n * FRB);
  }
  // transposed products via CSC built on the host (integer work only)
  DevBuf<Fr> abc[3];
  for (int k = 0; k < 3; k++) {
    const std::vector<uint32_t>& rp = r.h_rowptr[k];
    const std::vector<uint32_t>& cl = r.h_col[k];
    const size_t nnz = cl.size();
    std::vector<uint32_t> colptr(m + 1, 0), rowidx(nnz), perm(nnz);
    for (size_t i = 0; i < nnz; i++) colptr[cl[i] + 1]++;
    for (uint32_t i = 0; i < m; i++) colptr[i + 1] += colptr[i];
    std::vector<uint32_t> cur(colptr.begin(), colptr.end() - 1);
    for (uint32_t row = 0; row < N; row++)
      for (uint32_t e = rp[row]; e < rp[row + 1]; e++) {
        uint32_t pos = cur[cl[e]]++;
        rowidx[pos] = row;
        perm[pos] = e;
      }
    DevBuf<uint32_t> d_colptr(m + 1), d_rowidx(nnz), d_perm(nnz);
    h2d(st_, d_colptr.p, colptr.data(), (m + 1) * 4);
    h2d(st_, d_rowidx.p, rowidx.data(), nnz * 4);
    h2d(st_, d_perm.p, perm.data(), nnz * 4);
    abc[k].alloc(m);
    Fr* out = abc[k].p;
    const uint32_t* cp = d_colptr.p; const uint32_t* ri = d_rowidx.p; const uint32_t* pm = d_perm.p;
    const Fr* vl = r.val[k].p; const Fr* uu = u.p;
    const int add_inst = (k == 0);
    launch<k_setup_scalars>(st_, m, ZKB_LAMBDA(size_t t) {
      Fr acc = Fr::zero();
      for (uint32_t e = cp[t]; e < cp[t + 1]; e++) acc = Fr::add(acc, Fr::mul(vl[pm[e]], uu[ri[e]]));
      if (add_inst && t < ni) acc = Fr::add(acc, uu[N + t]);
      out[t] = acc;
    });
    stream_sync(st_);  // host vectors and the temporary index buffers go out of scope
  }
  // combined scalars: gamma_abc / l, and h
  DevBuf<Fr> lq(m), hq(n);
  {
    const Fr* pa = abc[0].p; const Fr* pb = abc[1].p; const Fr* pc = abc[2].p;
    Fr* pl = lq.p;
    launch<k_setup_scalars>(st_, m, ZKB_LAMBDA(size_t t) {
      Fr v = Fr::add(Fr::add(Fr::mul(beta, pa[t]), Fr::mul(alpha, pb[t])), pc[t]);
      pl[t] = Fr::mul(v, t < ni ? ginv : dinv);
    });
    Fr* ph = hq.p; const Fr* pp = pw.p;
    launch<k_setup_scalars>(st_, n, ZKB_LAMBDA(size_t t) { ph[t] = Fr::mul(pp[t], hscale); });
  }
  // the six key scalars alpha, beta, gamma, delta (G1 and G2 as needed)
  DevBuf<Fr> ks(4);
  {
    Fr hostk[4] = {alpha, beta, gamma, delta};
    h2d(st_, ks.p, hostk, sizeof(hostk));
  }
  tm.end();

  // fixed-base tables for g1 = g1_k * G1std and g2 = g2_k * G2std
  tm.begin("setup_fixed_base");
  FixedBase<Fq> fb1;
  FixedBase<Fq2> fb2;
  DevBuf<uint32_t> gk(16);
  h2d(st_, gk.p, trapdoor7 + 5 * 4, 64);
  const uint32_t* gkp = gk.p;
  fb_build<Fq>(fb1, std_g1<Gen, Fq>(), gkp);
  fb_build<Fq2>(fb2, std_g2<Gen, Fq2>(), gkp + 8);

  DevBuf<uint8_t> out(total);
  uint8_t* ob = out.p;
  auto emit = [&](auto& fb, const Fr* scalars, size_t count, size_t byte_off) {
    fb_emit(fb, scalars, count, (uint32_t*)(ob + byte_off));
  };
  auto put_len = [&](uint64_t v, size_t byte_off) { h2d(st_, ob + byte_off, &v, 8); stream_sync(st_); };
  size_t off = 0;
  emit(fb1, ks.p + 0, 1, off); off += G1B;            // alpha_g1
  emit(fb2, ks.p + 1, 1, off); off += G2B;            // beta_g2
  emit(fb2, ks.p + 2, 1, off); off += G2B;            // gamma_g2
  emit(fb2, ks.p + 3, 1, off); off += G2B;            // delta_g2
  put_len(ni, off); off += 8;
  emit(fb1, lq.p, ni, off); off += (size_t)ni * G1B;  // gamma_abc_g1
  emit(fb1, ks.p + 1, 1, off); off += G1B;            // beta_g1
  emit(fb1, ks.p + 3, 1, off); off += G1B;            // delta_g1
  put_len(m, off); off += 8;
  emit(fb1, abc[0].p, m, off); off += (size_t)m * G1B;  // a_query
  put_len(m, off); off += 8;
  emit(fb1, abc[1].p, m, off); off += (size_t)m * G1B;  // b_g1_query
  put_len(m, off); off += 8;
  emit(fb2, abc[1].p, m, off); off += (size_t)m * G2B;  // b_g2_query
  put_len(n - 1, off); off += 8;
  emit(fb1, hq.p, n - 1, off); off += (n - 1) * G1B;    // h_query
  put_len(m - ni, off); off += 8;
  emit(fb1, lq.p + ni, m - ni, off); off += (size_t)(m - ni) * G1B;  // l_query
  if (off != total) throw Error(ZKB_E_INTERNAL, "setup size mismatch");
  tm.end();
  d2h(st_, pk_out, ob, total);
  stream_sync(st_);
  *len = total;
  tm.collect(timings);
}

}  // namespace zkb
