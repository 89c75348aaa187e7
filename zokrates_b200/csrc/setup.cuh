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
size_t Engine<C>::key_size(const std::vector<KeySection>& key) {
  size_t bytes = 0;
  for (const KeySection& s : key) bytes += (s.vec ? 8 : 0) + s.count * (s.group == 1 ? G1B : G2B);
  return bytes;
}

// Every point is a fixed-base multiple of g1 = g1_k * G1std or g2 = g2_k * G2std (gk: g1_k, g2_k, 4 limbs each).  The
// points go to one device buffer and back in one copy; the length prefixes are written into pk_out on the host.
template <class C>
void Engine<C>::write_key(const std::vector<KeySection>& key, const uint64_t* gk, uint8_t* pk_out) {
  typedef typename GenOf<C>::T Gen;
  DevBuf<uint32_t> dgk(16);
  h2d(st_, dgk.p, gk, 64);
  FixedBase<Fq> fb1;
  FixedBase<Fq2> fb2;
  fb_build<Fq>(fb1, std_g1<Gen, Fq>(), dgk.p);
  fb_build<Fq2>(fb2, std_g2<Gen, Fq2>(), dgk.p + 8);
  std::vector<Fr> single;
  for (const KeySection& s : key) if (!s.vec) single.push_back(s.scalar);
  DevBuf<Fr> ds(single.size());
  h2d(st_, ds.p, single.data(), single.size() * FRB);
  const size_t total = key_size(key);
  DevBuf<uint8_t> out(total);
  size_t off = 0, j = 0;
  for (const KeySection& s : key) {
    if (s.vec) off += 8;
    uint32_t* dst = (uint32_t*)(out.p + off);
    const Fr* sc = s.vec ? s.scalars : ds.p + j++;
    if (s.group == 1) fb_emit(fb1, sc, s.count, dst);
    else fb_emit(fb2, sc, s.count, dst);
    off += s.count * (s.group == 1 ? G1B : G2B);
  }
  d2h(st_, pk_out, out.p, total);
  stream_sync(st_);
  off = 0;
  for (const KeySection& s : key) {
    if (s.vec) { memcpy(pk_out + off, &s.count, 8); off += 8; }
    off += s.count * (s.group == 1 ? G1B : G2B);
  }
}

// u_j = L_j(tau) over the domain of size n = 2^lg: ifft(tau^0 .. tau^(n-1)), in natural order, Montgomery.  The powers
// tau^0 .. tau^(n-1) are left in pw.
template <class C>
auto Engine<C>::lagrange_at(uint32_t lg, Fr tau, DevBuf<Fr>& pw) -> DevBuf<Fr> {
  const size_t n = (size_t)1 << lg;
  DomainT& d = domain(lg);
  pw.alloc(n);
  DevBuf<Fr> u(n);
  Fr* pp = pw.p; Fr* pu = u.p;
  const Fr one = Fr::one(), ninv = d.ninv;
  launch<k_ntt_table>(st_, n, ZKB_LAMBDA(size_t t) { ntt_powers_body<Fr>(tau, one, pp, (uint32_t)n, (uint32_t)t); });
  d2d(st_, pu, pp, n * FRB);
  ntt_dif(pu, d.tw_inv.p, lg);
  // bit-reversal permutation in place, scaled by 1/n: the thread of the lower index of each pair swaps it
  launch<k_ntt_brev>(st_, n, ZKB_LAMBDA(size_t t) {
    const uint32_t i = (uint32_t)t, j = bitrev32(i, lg);
    if (j < i) return;
    const Fr a = pu[i], b = pu[j];
    pu[i] = Fr::mul(b, ninv);
    pu[j] = Fr::mul(a, ninv);
  });
  return u;
}

// out = M_k^T w for matrix k (A, B, C) of the R1CS and a weight per row:  out_i = sum_row M_k[row][i] w_row.  The CSC of M_k
// is built on the host (integer work only).
template <class C>
auto Engine<C>::mul_transposed(const R1cs& r, int k, const Fr* w) -> DevBuf<Fr> {
  const std::vector<uint32_t>& rp = r.h_rowptr[k];
  const std::vector<uint32_t>& cl = r.h_col[k];
  const uint32_t N = (uint32_t)r.N, m = (uint32_t)r.m;
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
  DevBuf<uint32_t> d_colptr(m + 1), d_rowidx(nnz ? nnz : 1), d_perm(nnz ? nnz : 1);
  h2d(st_, d_colptr.p, colptr.data(), (m + 1) * 4);
  h2d(st_, d_rowidx.p, rowidx.data(), nnz * 4);
  h2d(st_, d_perm.p, perm.data(), nnz * 4);
  DevBuf<Fr> out(m);
  Fr* po = out.p;
  const uint32_t* cp = d_colptr.p; const uint32_t* ri = d_rowidx.p; const uint32_t* pm = d_perm.p;
  const Fr* vl = r.val[k].p;
  launch<k_setup_scalars>(st_, m, ZKB_LAMBDA(size_t t) {
    Fr acc = Fr::zero();
    for (uint32_t e = cp[t]; e < cp[t + 1]; e++) acc = Fr::add(acc, Fr::mul(vl[pm[e]], w[ri[e]]));
    po[t] = acc;
  });
  stream_sync(st_);  // host vectors and the temporary index buffers go out of scope
  return out;
}

template <class C>
auto Engine<C>::groth16_key(const R1cs& r, const Groth16Scalars& s) -> std::vector<KeySection> {
  const uint64_t n = (uint64_t)1 << r.log_n;
  return {point(1, s.alpha), point(2, s.beta), point(2, s.gamma), point(2, s.delta),   // alpha_g1, beta_g2, gamma_g2, delta_g2
          points(1, s.gamma_abc, r.ni),                                               // gamma_abc_g1
          point(1, s.beta), point(1, s.delta),                                        // beta_g1, delta_g1
          points(1, s.a, r.m), points(1, s.b, r.m), points(2, s.b, r.m),              // a_query, b_g1_query, b_g2_query
          points(1, s.h, n - 1), points(1, s.l, r.m - r.ni)};                         // h_query, l_query
}

template <class C>
size_t Engine<C>::setup_size(uint64_t rh) {
  return key_size(groth16_key(get_r1cs(rh), {}));
}

template <class C>
void Engine<C>::setup(uint64_t rh, const uint64_t* trapdoor7, uint8_t* pk_out, size_t cap, size_t* len) {
  R1cs& r = get_r1cs(rh);
  const uint32_t lg = r.log_n;
  const size_t n = (size_t)1 << lg;
  const size_t total = setup_size(rh);
  if (cap < total) throw Error(ZKB_E_ARG, "pk_out too small");
  StageTimer tm(st_);
  const uint32_t N = (uint32_t)r.N, ni = (uint32_t)r.ni, m = (uint32_t)r.m;

  // trapdoor scalars (host-side constants; a handful of field operations)
  const Fr alpha = trapdoor_fr(trapdoor7, 0), beta = trapdoor_fr(trapdoor7, 1), gamma = trapdoor_fr(trapdoor7, 2),
           delta = trapdoor_fr(trapdoor7, 3), tau = trapdoor_fr(trapdoor7, 4);
  const Fr ginv = Fr::inv(gamma), dinv = Fr::inv(delta);
  const Fr hscale = Fr::mul(vanishing_at(tau, lg), dinv);

  tm.begin("setup_scalars");
  DevBuf<Fr> pw;
  DevBuf<Fr> u = lagrange_at(lg, tau, pw);
  DevBuf<Fr> abc[3];
  for (int k = 0; k < 3; k++) abc[k] = mul_transposed(r, k, u.p);
  DevBuf<Fr> lq(m), hq(n);
  {
    Fr* pa = abc[0].p; const Fr* pb = abc[1].p; const Fr* pc = abc[2].p; const Fr* uu = u.p;
    // the instance rows x_i * 1 = x_i that ark appends after the constraints
    launch<k_setup_scalars>(st_, ni, ZKB_LAMBDA(size_t t) { pa[t] = Fr::add(pa[t], uu[N + t]); });
    // combined scalars: gamma_abc / l, and h
    Fr* pl = lq.p;
    launch<k_setup_scalars>(st_, m, ZKB_LAMBDA(size_t t) {
      Fr v = Fr::add(Fr::add(Fr::mul(beta, pa[t]), Fr::mul(alpha, pb[t])), pc[t]);
      pl[t] = Fr::mul(v, t < ni ? ginv : dinv);
    });
    Fr* ph = hq.p; const Fr* pp = pw.p;
    launch<k_setup_scalars>(st_, n, ZKB_LAMBDA(size_t t) { ph[t] = Fr::mul(pp[t], hscale); });
  }
  tm.end();

  tm.begin("setup_fixed_base");
  write_key(groth16_key(r, {alpha, beta, gamma, delta, lq.p, abc[0].p, abc[1].p, hq.p, lq.p + ni}), trapdoor7 + 5 * 4, pk_out);
  tm.end();
  *len = total;
  tm.collect(timings);
}

}  // namespace zkb
