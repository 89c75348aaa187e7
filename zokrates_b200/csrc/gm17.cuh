// GM17 prover on the same kernels (SURVEY.md §8 row f3).
//
// Replaces `<Ark as Backend<T, GM17>>::generate_proof` (/root/reference/zokrates_ark/src/gm17.rs:43-75): ark-gm17 0.3.0
// `ProvingKey::deserialize_unchecked` + `create_proof` — the R1CS -> SAP witness map (two square constraints per R1CS row and per
// public input; 5 transforms on a domain of 2N + 2(l-1) + 1 rows), five MSMs (a_query, c_query_2, c_query_1, g_gamma2_z_t in G1,
// b_query in G2) and the final combination with the masks d1, d2, r.  ark-gm17 is an external crate whose sources are not in
// /root/reference: the algorithm is restated from Groth-Maller 2017 and the crate's structure in oracle/gm17.py (PARITY
// UNPINNED against real ark-gm17 output; the GPU result is checked against that restatement, the two pairing equations and
// the trapdoor prediction).  SpMV, NTT, digit plans, bucket accumulation and reduction are the Groth16 kernels unchanged; the
// MSMs run one after the other without window tables (this path is about coverage, not the headline).
#pragma once
#include "engine.cuh"
#include "setup.cuh"

namespace zkb {

struct k_gm17_build; struct k_gm17_extra; struct k_gm17_h;

template <class C>
uint64_t Engine<C>::gm17_pk_load(const uint8_t* pk, size_t len) {
  size_t off = 0;
  auto need = [&](size_t k) { if (k > len - off) throw Error(ZKB_E_FORMAT, "gm17 proving key truncated"); };
  auto take = [&](size_t k) { need(k); const uint8_t* p = pk + off; off += k; return p; };
  auto take_vec = [&](size_t elem, uint64_t& count) {
    need(8); memcpy(&count, pk + off, 8); off += 8;
    if (count > (len - off) / elem) throw Error(ZKB_E_FORMAT, "gm17 proving key: vector length");
    return take(count * elem);
  };
  take(G2B);                     // vk.h_g2            (verifier only)
  take(G1B);                     // vk.g_alpha_g1
  take(G2B);                     // vk.h_beta_g2
  take(G1B);                     // vk.g_gamma_g1
  take(G2B);                     // vk.h_gamma_g2
  uint64_t ni, na, nb, nc1, nc2, nh;
  take_vec(G1B, ni);             // vk.query
  const uint8_t* aq = take_vec(G1B, na);
  const uint8_t* bq = take_vec(G2B, nb);
  const uint8_t* c1q = take_vec(G1B, nc1);
  const uint8_t* c2q = take_vec(G1B, nc2);
  const uint8_t* g_gamma_z = take(G1B);
  const uint8_t* h_gamma_z = take(G2B);
  const uint8_t* g_ab_gamma_z = take(G1B);
  const uint8_t* g_gamma2_z2 = take(G1B);
  const uint8_t* gzq = take_vec(G1B, nh);
  if (off != len) throw Error(ZKB_E_FORMAT, "trailing bytes after gm17 proving key");
  if (ni < 1 || na < ni || nb != na || nc2 != na || nc1 != na - ni || nh < 2) throw Error(ZKB_E_FORMAT, "gm17 proving key: inconsistent query lengths");
  std::unique_ptr<Gm17Pk> p(new Gm17Pk());
  p->ni = ni; p->nv = na; p->nh = nh;
  const uint64_t rest = na - 1;
  p->a.alloc(rest ? rest : 1); p->c2.alloc(rest ? rest : 1); p->b.alloc(rest ? rest : 1); p->c1.alloc(nc1 ? nc1 : 1); p->gz.alloc(nh);
  h2d(st_, p->a.p, aq + G1B, rest * G1B);
  h2d(st_, p->c2.p, c2q + G1B, rest * G1B);
  h2d(st_, p->b.p, bq + G2B, rest * G2B);
  h2d(st_, p->c1.p, c1q, nc1 * G1B);
  h2d(st_, p->gz.p, gzq, nh * G1B);
  DevBuf<G1A> f1(6);
  DevBuf<G2A> f2(2);
  h2d(st_, f1.p + 0, aq, G1B); h2d(st_, f1.p + 1, c2q, G1B); h2d(st_, f1.p + 2, g_gamma_z, G1B);
  h2d(st_, f1.p + 3, g_ab_gamma_z, G1B); h2d(st_, f1.p + 4, g_gamma2_z2, G1B); h2d(st_, f1.p + 5, gzq, G1B);
  h2d(st_, f2.p + 0, bq, G2B); h2d(st_, f2.p + 1, h_gamma_z, G2B);
  pk_convert<Fq>(p->a.p, rest); pk_convert<Fq>(p->c2.p, rest); pk_convert<Fq2>(p->b.p, rest); pk_convert<Fq>(p->c1.p, nc1);
  pk_convert<Fq>(p->gz.p, nh); pk_convert<Fq>(f1.p, 6); pk_convert<Fq2>(f2.p, 2);
  d2h(st_, p->h1, f1.p, 6 * G1B);
  d2h(st_, p->h2, f2.p, 2 * G2B);
  stream_sync(st_);
  uint64_t h = next_handle_++;
  gm17_pks_[h] = std::move(p);
  return h;
}

// one MSM on the shared scratch plan: digits/sort (or the plan built by the previous call when `replan` is false), accumulate,
// reduce, host finish
template <class C>
template <class F, class HX>
HX Engine<C>::gm17_msm(const Fr* scalars, const Affine<F>* pts, uint64_t n, bool replan) {
  typedef XYZZ<F> X;
  if (n == 0) return HX::identity();
  d_win_.ensure(MAXW * sizeof(X));
  if (replan) plan_build(plan_misc_, scalars, n);
  msm_exec<F>(plan_misc_, pts, (X*)d_win_.p, ws_misc_);
  ws_misc_.tail_done.wait(st_);
  std::vector<uint8_t> hw(MAXW * sizeof(X));
  d2h(st_, hw.data(), d_win_.p, ws_misc_.out_entries * sizeof(X));
  stream_sync(st_);
  return host_finish<HX>((const HX*)hw.data(), plan_misc_, ws_misc_);
}

template <class C>
void Engine<C>::gm17_prove(uint64_t pkh, uint64_t rh, const uint64_t* z, const uint64_t* d1p, const uint64_t* d2p, const uint64_t* rp,
                           uint8_t* proof_out) {
  auto it = gm17_pks_.find(pkh);
  if (it == gm17_pks_.end()) throw Error(ZKB_E_ARG, "unknown gm17 pk handle");
  Gm17Pk& pk = *it->second;
  R1cs& r = get_r1cs(rh);
  for (auto& sl : slots_) if (sl.state != 0) throw Error(ZKB_E_ARG, "a Groth16 proof is in flight on this context");
  const uint64_t N = r.N, ni = r.ni, m = r.m;
  const uint64_t rows = 2 * N + 2 * (ni - 1) + 1, nv = m + N + (ni - 1);
  if (pk.ni != ni || pk.nv != nv) throw Error(ZKB_E_ARG, "gm17 proving key does not match the R1CS (variable counts)");
  uint32_t lg = 0;
  while (((uint64_t)1 << lg) < rows) lg++;
  const size_t n = (size_t)1 << lg;
  if (pk.nh != n + 1) throw Error(ZKB_E_ARG, "gm17 proving key does not match the R1CS (domain size)");
  if (!z && !r.has_z) throw Error(ZKB_E_ARG, "no resident assignment");
  DomainT& d = domain(lg);
  StageTimer tm(st_);
  tm.begin("gm17_witness_map");
  DevBuf<Fr> full_m(nv), full_c(nv), va(n), vc(n), vq(n), a2(n), hc(n + 1), t0(N ? N : 1), t1(N ? N : 1), t2(N ? N : 1);
  if (z) h2d(st_, full_c.p, z, m * FRB); else d2d(st_, full_c.p, r.z_canon.p, m * FRB);
  convert(full_c.p, full_m.p, 0, m);
  {  // A z, B z, C z
    Fr* outs[3] = {t0.p, t1.p, t2.p};
    const Fr* zm = full_m.p;
    for (int k = 0; k < 3; k++) {
      Fr* out = outs[k];
      const uint32_t* rpk = r.rowptr[k].p; const uint32_t* cl = r.col[k].p; const Fr* vl = r.val[k].p;
      const uint32_t Nn = (uint32_t)N;
      launch<k_spmv>(st_, N, ZKB_LAMBDA(size_t t) { spmv_body<Fr>(rpk, cl, vl, zm, out, Nn, (uint32_t)t); });
    }
  }
  dev_zero(st_, va.p, n * FRB);
  dev_zero(st_, vc.p, n * FRB);
  {
    const Fr* az = t0.p; const Fr* bz = t1.p; const Fr* cz = t2.p;
    Fr* pa = va.p; Fr* pc = vc.p; Fr* fm = full_m.p;
    const size_t mm = m, NN = N;
    // rows 2i, 2i+1:  (A + B)^2 = 4 C + x_i,  (A - B)^2 = x_i   with the extra variable x_i = (A - B)^2 at column m + i
    launch<k_gm17_build>(st_, N, ZKB_LAMBDA(size_t i) {
      const Fr s = Fr::add(az[i], bz[i]), df = Fr::sub(az[i], bz[i]);
      const Fr x = Fr::sqr(df);
      const Fr c4 = Fr::dbl(Fr::dbl(cz[i]));
      pa[2 * i] = s; pa[2 * i + 1] = df;
      pc[2 * i] = Fr::add(c4, x); pc[2 * i + 1] = x;
      fm[mm + i] = x;
    });
    // the constant row 1^2 = 1 and, per public input j >= 1, (z_j + 1)^2 = 4 z_j + y_j, (z_j - 1)^2 = y_j, y_j at column m + N - 1 + j
    const size_t nin = ni;
    launch<k_gm17_extra>(st_, ni, ZKB_LAMBDA(size_t j) {
      const Fr one = Fr::one();
      if (j == 0) { pa[2 * NN] = one; pc[2 * NN] = one; return; }
      const Fr zj = fm[j];
      const Fr dm = Fr::sub(zj, one);
      const Fr y = Fr::sqr(dm);
      pa[2 * NN + 2 * j - 1] = Fr::add(zj, one); pa[2 * NN + 2 * j] = dm;
      pc[2 * NN + 2 * j - 1] = Fr::add(Fr::dbl(Fr::dbl(zj)), y); pc[2 * NN + 2 * j] = y;
      fm[mm + NN - 1 + j] = y;
      (void)nin;
    });
  }
  convert(full_m.p, full_c.p, 1, nv);            // the MSM scalars: canonical
  // a: coefficients (bit-reversed, times n) -> keep 2 d1 a(x) in natural order, then the coset evaluations
  ntt_dif(va.p, d.tw_inv.p, lg);
  HFr hd1, hd2, hr;
  memcpy(hd1.v, d1p, 32); memcpy(hd2.v, d2p, 32); memcpy(hr.v, rp, 32);
  Fr d1m, d2m;
  { HFr t = HFr::to_mont(hd1); memcpy(d1m.v, t.v, 32); t = HFr::to_mont(hd2); memcpy(d2m.v, t.v, 32); }
  {
    const Fr twod1n = Fr::mul(Fr::dbl(d1m), d.ninv);
    const Fr* src = va.p; Fr* dst = a2.p;
    launch<k_ntt_brev>(st_, n, ZKB_LAMBDA(size_t t) { dst[bitrev32((uint32_t)t, lg)] = Fr::mul(src[t], twod1n); });
  }
  ntt_dit(va.p, d.tw_fwd.p, lg, d.cos_fwd.p);
  ntt_dif(vc.p, d.tw_inv.p, lg);
  ntt_dit(vc.p, d.tw_fwd.p, lg, d.cos_fwd.p);
  {
    Fr* pa = va.p; const Fr* pc = vc.p; const Fr zinv = d.zinv;
    launch<k_qap_pointwise>(st_, n, ZKB_LAMBDA(size_t t) { pa[t] = Fr::mul(Fr::sub(Fr::sqr(pa[t]), pc[t]), zinv); });
  }
  ntt_dif(va.p, d.tw_inv.p, lg);
  {
    const Fr* pa = va.p; Fr* pq = vq.p; const Fr* t2c = d.cos_inv.p;
    launch<k_ntt_brev>(st_, n, ZKB_LAMBDA(size_t t) { ntt_brev_copy_body<Fr>(pa, pq, t2c, lg, 0, (uint32_t)t); });
  }
  {  // h = quotient (n - 1 coefficients) + 2 d1 a(x) - d2 - d1^2 + d1^2 x^n, canonical
    const Fr* pq = vq.p; const Fr* p2 = a2.p; Fr* ph = hc.p;
    const Fr d1sq = Fr::sqr(d1m), dd2 = d2m;
    const size_t nn = n;
    launch<k_gm17_h>(st_, n + 1, ZKB_LAMBDA(size_t t) {
      Fr v;
      if (t == nn) v = d1sq;
      else {
        v = p2[t];
        if (t + 1 < nn) v = Fr::add(v, pq[t]);
        if (t == 0) v = Fr::sub(Fr::sub(v, dd2), d1sq);
      }
      ph[t] = Fr::from_mont(v);
    });
  }
  tm.end();
  tm.begin("gm17_msms");
  const HG1X s_a = gm17_msm<Fq, HG1X>(full_c.p + 1, pk.a.p, nv - 1, true);
  const HG1X s_c2 = gm17_msm<Fq, HG1X>(full_c.p + 1, pk.c2.p, nv - 1, false);
  const HG2X s_b = gm17_msm<Fq2, HG2X>(full_c.p + 1, pk.b.p, nv - 1, false);
  const HG1X s_c1 = gm17_msm<Fq, HG1X>(full_c.p + ni, pk.c1.p, nv - ni, true);
  const HG1X s_h = gm17_msm<Fq, HG1X>(hc.p, pk.gz.p, n + 1, true);
  tm.end();
  tm.collect(timings);
  // final combination on the host (ark does the same serially):
  //   A = (r + d1) g_gamma_z + a_0 + S_a;   B likewise in G2;
  //   C = S_c1 + (r^2 + 2 r d1) g_gamma2_z2 + (r + d1) g_ab_gamma_z + r (c2_0 + S_c2) + d2 g_gamma2_z_t[0] + S_h
  const HG1A &a0 = pk.h1[0], &c20 = pk.h1[1], &g_gamma_z = pk.h1[2], &g_ab = pk.h1[3], &g_g2z2 = pk.h1[4], &gz0 = pk.h1[5];
  const HG2A &b0 = pk.h2[0], &h_gamma_z = pk.h2[1];
  const HFr rm = HFr::to_mont(hr), d1h = HFr::to_mont(hd1);
  const HFr rd1 = HFr::from_mont(HFr::add(rm, d1h));                                   // canonical r + d1
  const HFr k2 = HFr::from_mont(HFr::add(HFr::mul(rm, rm), HFr::dbl(HFr::mul(rm, d1h))));   // canonical r^2 + 2 r d1
  HG1X ga = HG1X::madd(HG1X::add(HG1X::mul_affine(g_gamma_z, (const uint32_t*)rd1.v, 8), s_a), a0);
  HG2X gb = HG2X::madd(HG2X::add(HG2X::mul_affine(h_gamma_z, (const uint32_t*)rd1.v, 8), s_b), b0);
  HG1X gc = HG1X::add(s_c1, HG1X::mul_affine(g_g2z2, (const uint32_t*)k2.v, 8));
  gc = HG1X::add(gc, HG1X::mul_affine(g_ab, (const uint32_t*)rd1.v, 8));
  gc = HG1X::add(gc, HG1X::mul_xyzz(HG1X::madd(s_c2, c20), (const uint32_t*)hr.v, 8));
  gc = HG1X::add(gc, HG1X::mul_affine(gz0, (const uint32_t*)hd2.v, 8));
  gc = HG1X::add(gc, s_h);
  const HG1A pa = HG1X::to_affine(ga), pcc = HG1X::to_affine(gc);
  const HG2A pb = HG2X::to_affine(gb);
  write_proof(proof_out, pa, pb, pcc);
}

// ---- circuit-specific GM17 setup from an explicit trapdoor (alpha, beta, gamma, tau, g1_k, g2_k) ---------------------------------
// `impl NonUniversalBackend<T, GM17> for Ark`::setup (zokrates_ark/src/gm17.rs:19-41) -> ark-gm17 `generate_parameters`; the trapdoor
// is explicit as in zkb_groth16_setup (the reference draws it from its rng).  u = Lagrange coefficients at tau over the SAP domain;
// per SAP variable  a_i = sum_rows (u_2r + u_2r+1) A_r[i] + (u_2r - u_2r+1) B_r[i] (+ the input-consistency rows),
// c_i = sum_rows 4 u_2r C_r[i] (+ ...), extra variables x_r: c = u_2r + u_2r+1, y_j: c = u_(e+2j-1) + u_(e+2j); then every key element is a
// fixed-base multiple of g or h (same window tables as the Groth16 setup).  Key bytes: ark's `serialize_unchecked` field order.
template <class C>
size_t Engine<C>::gm17_setup_size(uint64_t rh) {
  R1cs& r = get_r1cs(rh);
  const uint64_t rows = 2 * r.N + 2 * (r.ni - 1) + 1, nv = r.m + r.N + (r.ni - 1);
  size_t n = 1;
  while (n < rows) n <<= 1;
  return 3 * G2B + 2 * G1B + (8 + r.ni * G1B) + (8 + nv * G1B) + (8 + nv * G2B) + (8 + (nv - r.ni) * G1B) + (8 + nv * G1B) + 3 * G1B + G2B +
         (8 + (n + 1) * G1B);
}

template <class C>
void Engine<C>::gm17_setup(uint64_t rh, const uint64_t* trapdoor6, uint8_t* pk_out, size_t cap, size_t* len) {
  typedef typename GenOf<C>::T Gen;
  R1cs& r = get_r1cs(rh);
  const uint32_t N = (uint32_t)r.N, ni = (uint32_t)r.ni, m = (uint32_t)r.m;
  const uint64_t rows = 2 * (uint64_t)N + 2 * (ni - 1) + 1;
  const uint32_t nv = m + N + (ni - 1);
  uint32_t lg = 0;
  while (((uint64_t)1 << lg) < rows) lg++;
  const size_t n = (size_t)1 << lg;
  const size_t total = gm17_setup_size(rh);
  if (cap < total) throw Error(ZKB_E_ARG, "pk_out too small");
  DomainT& d = domain(lg);
  Fr td[4];
  for (int k = 0; k < 4; k++) {
    Fr c;
    for (int i = 0; i < 8; i++) c.v[i] = ((const uint32_t*)trapdoor6)[k * 8 + i];
    td[k] = Fr::to_mont(c);
  }
  const Fr alpha = td[0], beta = td[1], gamma = td[2], tau = td[3];
  Fr tn = tau;
  for (uint32_t i = 0; i < lg; i++) tn = Fr::sqr(tn);
  const Fr zt = Fr::sub(tn, Fr::one());
  const Fr ab = Fr::add(alpha, beta), g2 = Fr::sqr(gamma), abg = Fr::mul(ab, gamma), gz = Fr::mul(gamma, zt);
  const Fr g2z = Fr::mul(g2, zt), g2z2x2 = Fr::dbl(g2z);
  // u = ifft(powers of tau) in natural order; powers up to tau^n scaled by gamma^2 Z for g_gamma2_z_t
  DevBuf<Fr> pw(n), u(n), pwz(n + 1);
  {
    Fr one = Fr::one();
    Fr* pp = pw.p; Fr* pz = pwz.p;
    launch<k_ntt_table>(st_, n, ZKB_LAMBDA(size_t t) { ntt_powers_body<Fr>(tau, one, pp, (uint32_t)n, (uint32_t)t); });
    launch<k_ntt_table>(st_, n + 1, ZKB_LAMBDA(size_t t) { ntt_powers_body<Fr>(tau, g2z, pz, (uint32_t)n + 1, (uint32_t)t); });
    d2d(st_, u.p, pw.p, n * FRB);
    ntt_dif(u.p, d.tw_inv.p, lg);
    scratch_a_.ensure(n);
    Fr* src = u.p; Fr* dst = scratch_a_.p;
    Fr ninv = d.ninv;
    launch<k_ntt_brev>(st_, n, ZKB_LAMBDA(size_t t) { dst[bitrev32((uint32_t)t, lg)] = Fr::mul(src[t], ninv); });
    d2d(st_, u.p, scratch_a_.p, n * FRB);
  }
  // per R1CS row: u_2r + u_2r+1, u_2r - u_2r+1, 4 u_2r
  DevBuf<Fr> urow[3];
  for (int k = 0; k < 3; k++) urow[k].alloc(N ? N : 1);
  {
    const Fr* uu = u.p; Fr* p0 = urow[0].p; Fr* p1 = urow[1].p; Fr* p2 = urow[2].p;
    launch<k_setup_scalars>(st_, N, ZKB_LAMBDA(size_t i) {
      p0[i] = Fr::add(uu[2 * i], uu[2 * i + 1]);
      p1[i] = Fr::sub(uu[2 * i], uu[2 * i + 1]);
      p2[i] = Fr::dbl(Fr::dbl(uu[2 * i]));
    });
  }
  // transposed products (CSC built on the host, as in the Groth16 setup)
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
    DevBuf<uint32_t> d_colptr(m + 1), d_rowidx(nnz ? nnz : 1), d_perm(nnz ? nnz : 1);
    h2d(st_, d_colptr.p, colptr.data(), (m + 1) * 4);
    h2d(st_, d_rowidx.p, rowidx.data(), nnz * 4);
    h2d(st_, d_perm.p, perm.data(), nnz * 4);
    abc[k].alloc(m);
    Fr* out = abc[k].p;
    const uint32_t* cp = d_colptr.p; const uint32_t* ri = d_rowidx.p; const uint32_t* pm = d_perm.p;
    const Fr* vl = r.val[k].p; const Fr* uu = urow[k].p;
    launch<k_setup_scalars>(st_, m, ZKB_LAMBDA(size_t t) {
      Fr acc = Fr::zero();
      for (uint32_t e = cp[t]; e < cp[t + 1]; e++) acc = Fr::add(acc, Fr::mul(vl[pm[e]], uu[ri[e]]));
      out[t] = acc;
    });
    stream_sync(st_);
  }
  // a_i and c_i of every SAP variable
  DevBuf<Fr> va(nv), vc(nv);
  {
    const Fr* pA = abc[0].p; const Fr* pB = abc[1].p; const Fr* pC = abc[2].p; const Fr* uu = u.p; const Fr* uadd = urow[0].p;
    Fr* pa = va.p; Fr* pc = vc.p;
    const uint32_t e_off = 2 * N;
    launch<k_setup_scalars>(st_, nv, ZKB_LAMBDA(size_t t) {
      Fr a = Fr::zero(), c = Fr::zero();
      if (t < m) {
        a = Fr::add(pA[t], pB[t]);
        c = pC[t];
        if (t == 0) {
          a = Fr::add(a, uu[e_off]);
          c = Fr::add(c, uu[e_off]);
          for (uint32_t j = 1; j < ni; j++) a = Fr::add(a, Fr::sub(uu[e_off + 2 * j - 1], uu[e_off + 2 * j]));
        } else if (t < ni) {
          a = Fr::add(a, Fr::add(uu[e_off + 2 * t - 1], uu[e_off + 2 * t]));
          c = Fr::add(c, Fr::dbl(Fr::dbl(uu[e_off + 2 * t - 1])));
        }
      } else if (t < m + N) {
        c = uadd[t - m];
      } else {
        const uint32_t j = (uint32_t)t - (m + N) + 1;
        c = Fr::add(uu[e_off + 2 * j - 1], uu[e_off + 2 * j]);
      }
      pa[t] = a; pc[t] = c;
    });
  }
  // scalar vectors of the queries
  DevBuf<Fr> s_a(nv), s_q(ni), s_c1(nv - ni ? nv - ni : 1), s_c2(nv), ks(9);
  {
    const Fr* pa = va.p; const Fr* pc = vc.p;
    Fr* oa = s_a.p; Fr* oq = s_q.p; Fr* o1 = s_c1.p; Fr* o2 = s_c2.p;
    launch<k_setup_scalars>(st_, nv, ZKB_LAMBDA(size_t t) {
      oa[t] = Fr::mul(gamma, pa[t]);
      o2[t] = Fr::mul(g2z2x2, pa[t]);
      const Fr mix = Fr::add(Fr::mul(g2, pc[t]), Fr::mul(abg, pa[t]));
      if (t < ni) oq[t] = Fr::add(Fr::mul(gamma, pc[t]), Fr::mul(ab, pa[t]));
      else o1[t - ni] = mix;
    });
    Fr hostk[9] = {Fr::one(), alpha, beta, gamma, gz, Fr::mul(abg, zt), Fr::mul(g2z, zt), Fr::zero(), Fr::zero()};
    h2d(st_, ks.p, hostk, sizeof(hostk));
  }
  FixedBase<Fq> fb1;
  FixedBase<Fq2> fb2;
  DevBuf<uint32_t> gk(16);
  h2d(st_, gk.p, trapdoor6 + 4 * 4, 64);
  fb_build<Fq>(fb1, std_g1<Gen, Fq>(), gk.p);
  fb_build<Fq2>(fb2, std_g2<Gen, Fq2>(), gk.p + 8);
  DevBuf<uint8_t> out(total);
  uint8_t* ob = out.p;
  auto emit = [&](auto& fb, const Fr* scalars, size_t count, size_t byte_off) { fb_emit(fb, scalars, count, (uint32_t*)(ob + byte_off)); };
  auto put_len = [&](uint64_t v, size_t byte_off) { h2d(st_, ob + byte_off, &v, 8); stream_sync(st_); };
  size_t off = 0;
  emit(fb2, ks.p + 0, 1, off); off += G2B;                     // vk.h_g2
  emit(fb1, ks.p + 1, 1, off); off += G1B;                     // vk.g_alpha_g1
  emit(fb2, ks.p + 2, 1, off); off += G2B;                     // vk.h_beta_g2
  emit(fb1, ks.p + 3, 1, off); off += G1B;                     // vk.g_gamma_g1
  emit(fb2, ks.p + 3, 1, off); off += G2B;                     // vk.h_gamma_g2
  put_len(ni, off); off += 8;
  emit(fb1, s_q.p, ni, off); off += (size_t)ni * G1B;          // vk.query
  put_len(nv, off); off += 8;
  emit(fb1, s_a.p, nv, off); off += (size_t)nv * G1B;          // a_query
  put_len(nv, off); off += 8;
  emit(fb2, s_a.p, nv, off); off += (size_t)nv * G2B;          // b_query
  put_len(nv - ni, off); off += 8;
  emit(fb1, s_c1.p, nv - ni, off); off += (size_t)(nv - ni) * G1B;   // c_query_1
  put_len(nv, off); off += 8;
  emit(fb1, s_c2.p, nv, off); off += (size_t)nv * G1B;         // c_query_2
  emit(fb1, ks.p + 4, 1, off); off += G1B;                     // g_gamma_z
  emit(fb2, ks.p + 4, 1, off); off += G2B;                     // h_gamma_z
  emit(fb1, ks.p + 5, 1, off); off += G1B;                     // g_ab_gamma_z
  emit(fb1, ks.p + 6, 1, off); off += G1B;                     // g_gamma2_z2
  put_len(n + 1, off); off += 8;
  emit(fb1, pwz.p, n + 1, off); off += (n + 1) * G1B;          // g_gamma2_z_t
  if (off != total) throw Error(ZKB_E_INTERNAL, "gm17 setup size mismatch");
  d2h(st_, pk_out, ob, total);
  stream_sync(st_);
  *len = total;
}

}  // namespace zkb
