#define _GNU_SOURCE
/* zkoracle.c — CPU restatement (C, OpenMP) of the reference's Groth16 proving path.
 *
 * TEST INFRASTRUCTURE / CPU BASELINE ONLY: loaded by tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs.  Never linked or loaded by the product (zokrates_b200/).
 *
 * The arithmetic of this path is not in /root/reference: zokrates_ark (zokrates_ark/src/groth16.rs:21-53)
 * calls arkworks 0.3.0 crates pinned in /root/reference/Cargo.lock (ark-groth16 :221, ark-ec :146,
 * ark-ff :161, ark-poly :282) which are not vendored and cannot be built here (no rustc).  This file
 * restates their published algorithms (SURVEY.md App. B):
 *   - ark-ff   Fp256/Fp384 Montgomery arithmetic on 64-bit limbs
 *   - ark-ec   short-Weierstrass Jacobian add / mixed add / double; VariableBaseMSM::multi_scalar_mul
 *              with ark's window rule c = (size < 32 ? 3 : ceil(log2 size)*69/100 + 2), unsigned windows,
 *              unit scalars added once, parallel over windows only (rayon cfg_into_iter over window_starts)
 *   - ark-poly Radix2EvaluationDomain fft / ifft / coset variants
 *   - ark-groth16 LibsnarkReduction::witness_map and create_proof_with_reduction
 *   - ark-serialize ProvingKey::deserialize_unchecked layout
 *   - GM17's square arithmetic program at tau and its trapdoor-predicted proof (restating oracle/gm17.py)
 * Parity status: field arithmetic and formats pinned by the reference's KATs via the python oracle
 * (tests/test_oracle_pins.py cross-checks this file against it); proof values "parity unpinned"
 * (no golden proof exists in the reference) — validated by the pairing/trapdoor checks in oracle/ark.py.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <time.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef unsigned __int128 u128;
static int zko_pool_threads(void);
#define MAXL 6

typedef struct { uint64_t l[MAXL]; } fe;

typedef struct {
  int n;             /* 64-bit limbs */
  int bits;
  fe p, r1, r2;      /* modulus, R mod p, R^2 mod p */
  uint64_t inv;      /* -p^-1 mod 2^64 */
} fctx;

/* ------------------------------------------------------------------------------------------- */
static inline int fe_is_zero(const fctx* f, const fe* a) { uint64_t t = 0; for (int i = 0; i < f->n; i++) t |= a->l[i]; return t == 0; }
static inline int fe_eq(const fctx* f, const fe* a, const fe* b) { uint64_t t = 0; for (int i = 0; i < f->n; i++) t |= a->l[i] ^ b->l[i]; return t == 0; }
static inline int fe_geq(const fctx* f, const fe* a, const fe* b) {
  for (int i = f->n - 1; i >= 0; i--) { if (a->l[i] > b->l[i]) return 1; if (a->l[i] < b->l[i]) return 0; }
  return 1;
}
static inline void fe_sub_raw(const fctx* f, fe* r, const fe* a, const fe* b) {
  uint64_t borrow = 0;
  for (int i = 0; i < f->n; i++) { u128 t = (u128)a->l[i] - b->l[i] - borrow; r->l[i] = (uint64_t)t; borrow = (uint64_t)(t >> 64) & 1; }
}
static inline void fe_add(const fctx* f, fe* r, const fe* a, const fe* b) {
  uint64_t carry = 0; fe t;
  for (int i = 0; i < f->n; i++) { u128 s = (u128)a->l[i] + b->l[i] + carry; t.l[i] = (uint64_t)s; carry = (uint64_t)(s >> 64); }
  for (int i = f->n; i < MAXL; i++) t.l[i] = 0;
  if (carry || fe_geq(f, &t, &f->p)) fe_sub_raw(f, &t, &t, &f->p);
  *r = t;
}
static inline void fe_sub(const fctx* f, fe* r, const fe* a, const fe* b) {
  fe t; uint64_t borrow = 0;
  for (int i = 0; i < f->n; i++) { u128 d = (u128)a->l[i] - b->l[i] - borrow; t.l[i] = (uint64_t)d; borrow = (uint64_t)(d >> 64) & 1; }
  for (int i = f->n; i < MAXL; i++) t.l[i] = 0;
  if (borrow) { uint64_t carry = 0; for (int i = 0; i < f->n; i++) { u128 s = (u128)t.l[i] + f->p.l[i] + carry; t.l[i] = (uint64_t)s; carry = (uint64_t)(s >> 64); } }
  *r = t;
}
static inline void fe_neg(const fctx* f, fe* r, const fe* a) { if (fe_is_zero(f, a)) { *r = *a; return; } fe_sub_raw(f, r, &f->p, a); for (int i = f->n; i < MAXL; i++) r->l[i] = 0; }
static inline void fe_dbl(const fctx* f, fe* r, const fe* a) { fe_add(f, r, a, a); }

#define MONT_MUL(N)                                                                                   \
  static inline void mont_mul_##N(const fctx* f, fe* r, const fe* a, const fe* b) {                   \
    uint64_t t[N + 2];                                                                                \
    for (int i = 0; i < N + 2; i++) t[i] = 0;                                                         \
    for (int i = 0; i < N; i++) {                                                                     \
      uint64_t c = 0;                                                                                 \
      for (int j = 0; j < N; j++) { u128 s = (u128)a->l[j] * b->l[i] + t[j] + c; t[j] = (uint64_t)s; c = (uint64_t)(s >> 64); } \
      u128 s2 = (u128)t[N] + c; t[N] = (uint64_t)s2; t[N + 1] = (uint64_t)(s2 >> 64);                  \
      uint64_t m = t[0] * f->inv;                                                                     \
      u128 s = (u128)m * f->p.l[0] + t[0]; c = (uint64_t)(s >> 64);                                   \
      for (int j = 1; j < N; j++) { s = (u128)m * f->p.l[j] + t[j] + c; t[j - 1] = (uint64_t)s; c = (uint64_t)(s >> 64); } \
      s2 = (u128)t[N] + c; t[N - 1] = (uint64_t)s2; t[N] = t[N + 1] + (uint64_t)(s2 >> 64);            \
    }                                                                                                 \
    fe o; for (int i = 0; i < N; i++) o.l[i] = t[i]; for (int i = N; i < MAXL; i++) o.l[i] = 0;       \
    if (t[N] || fe_geq(f, &o, &f->p)) fe_sub_raw(f, &o, &o, &f->p);                                    \
    *r = o;                                                                                           \
  }
MONT_MUL(4)
MONT_MUL(6)
static inline void fe_mul(const fctx* f, fe* r, const fe* a, const fe* b) { if (f->n == 4) mont_mul_4(f, r, a, b); else mont_mul_6(f, r, a, b); }
static inline void fe_sqr(const fctx* f, fe* r, const fe* a) { fe_mul(f, r, a, a); }
static void fe_to_mont(const fctx* f, fe* r, const fe* a) { fe_mul(f, r, a, &f->r2); }
static void fe_from_mont(const fctx* f, fe* r, const fe* a) { fe one; memset(&one, 0, sizeof one); one.l[0] = 1; fe_mul(f, r, a, &one); }
static void fe_pow(const fctx* f, fe* r, const fe* a, const uint64_t* e, int nl) {
  fe acc = f->r1;
  for (int i = nl - 1; i >= 0; i--) for (int b = 63; b >= 0; b--) { fe_sqr(f, &acc, &acc); if ((e[i] >> b) & 1) fe_mul(f, &acc, &acc, a); }
  *r = acc;
}
static void fe_inv(const fctx* f, fe* r, const fe* a) {
  fe e = f->p; /* p - 2 */
  uint64_t borrow = 2;
  for (int i = 0; i < f->n && borrow; i++) { uint64_t o = e.l[i]; e.l[i] = o - borrow; borrow = o < borrow; }
  fe_pow(f, r, a, e.l, f->n);
}
static void fe_from_u64(const fctx* f, fe* r, uint64_t v) { fe t; memset(&t, 0, sizeof t); t.l[0] = v; fe_to_mont(f, r, &t); }

/* context construction from the modulus alone */
static void fctx_init(fctx* f, int n, const uint64_t* p) {
  memset(f, 0, sizeof *f);
  f->n = n;
  for (int i = 0; i < n; i++) f->p.l[i] = p[i];
  int bits = 0;
  for (int i = n - 1; i >= 0 && !bits; i--) if (p[i]) bits = 64 * i + (64 - __builtin_clzll(p[i]));
  f->bits = bits;
  uint64_t inv = 1;
  for (int i = 0; i < 63; i++) { inv *= inv; inv *= p[0]; }   /* p^-1 mod 2^64 */
  f->inv = (uint64_t)0 - inv;
  /* R mod p by doubling 1 (64 n) times; R^2 by doubling on */
  fe x; memset(&x, 0, sizeof x); x.l[0] = 1;
  for (int i = 0; i < 64 * n; i++) fe_add(f, &x, &x, &x);
  f->r1 = x;
  for (int i = 0; i < 64 * n; i++) fe_add(f, &x, &x, &x);
  f->r2 = x;
}

/* ------------------------------------------------------------------------------------------- Fq2 */
typedef struct { fe c0, c1; } fe2;
static inline int fe2_is_zero(const fctx* f, const fe2* a) { return fe_is_zero(f, &a->c0) && fe_is_zero(f, &a->c1); }
static inline int fe2_eq(const fctx* f, const fe2* a, const fe2* b) { return fe_eq(f, &a->c0, &b->c0) && fe_eq(f, &a->c1, &b->c1); }
static inline void fe2_add(const fctx* f, fe2* r, const fe2* a, const fe2* b) { fe_add(f, &r->c0, &a->c0, &b->c0); fe_add(f, &r->c1, &a->c1, &b->c1); }
static inline void fe2_sub(const fctx* f, fe2* r, const fe2* a, const fe2* b) { fe_sub(f, &r->c0, &a->c0, &b->c0); fe_sub(f, &r->c1, &a->c1, &b->c1); }
static inline void fe2_neg(const fctx* f, fe2* r, const fe2* a) { fe_neg(f, &r->c0, &a->c0); fe_neg(f, &r->c1, &a->c1); }
static inline void fe2_dbl(const fctx* f, fe2* r, const fe2* a) { fe2_add(f, r, a, a); }
static inline void fe2_mul(const fctx* f, fe2* r, const fe2* a, const fe2* b) {
  fe v0, v1, s, t, u;
  fe_mul(f, &v0, &a->c0, &b->c0); fe_mul(f, &v1, &a->c1, &b->c1);
  fe_add(f, &s, &a->c0, &a->c1); fe_add(f, &t, &b->c0, &b->c1); fe_mul(f, &u, &s, &t);
  fe_sub(f, &r->c0, &v0, &v1); fe_sub(f, &u, &u, &v0); fe_sub(f, &r->c1, &u, &v1);
}
static inline void fe2_sqr(const fctx* f, fe2* r, const fe2* a) { fe2_mul(f, r, a, a); }
static void fe2_inv(const fctx* f, fe2* r, const fe2* a) {
  fe t0, t1, d;
  fe_sqr(f, &t0, &a->c0); fe_sqr(f, &t1, &a->c1); fe_add(f, &d, &t0, &t1); fe_inv(f, &d, &d);
  fe_mul(f, &r->c0, &a->c0, &d); fe_mul(f, &t0, &a->c1, &d); fe_neg(f, &r->c1, &t0);
}
static void fe2_one(const fctx* f, fe2* r) { r->c0 = f->r1; memset(&r->c1, 0, sizeof(fe)); }
static void fe_one(const fctx* f, fe* r) { *r = f->r1; }

/* ------------------------------------------------------------------------------------------- curves
 * Jacobian arithmetic instantiated twice (coordinates in Fq and in Fq2) by textual templating. */
#define FT fe
#define PFX g1
#define F_(op) fe_##op
#include "zkoracle_ec.inc"
#undef FT
#undef PFX
#undef F_
#define FT fe2
#define PFX g2
#define F_(op) fe2_##op
#include "zkoracle_ec.inc"
#undef FT
#undef PFX
#undef F_

/* ------------------------------------------------------------------------------------------- curve table */
typedef struct { fctx fr, fq; fe root; /* 2-adic root of unity (Montgomery) */ fe gen; int two_adicity; int fq_bytes; } curve_t;
static curve_t CURVES[2];
static int curves_ready = 0;

static void curves_init(void) {
  if (curves_ready) return;
  zko_pool_threads();
  static const uint64_t bn_r[4] = {0x43e1f593f0000001ull, 0x2833e84879b97091ull, 0xb85045b68181585dull, 0x30644e72e131a029ull};
  static const uint64_t bn_p[4] = {0x3c208c16d87cfd47ull, 0x97816a916871ca8dull, 0xb85045b68181585dull, 0x30644e72e131a029ull};
  static const uint64_t bls_r[4] = {0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull};
  static const uint64_t bls_p[6] = {0xb9feffffffffaaabull, 0x1eabfffeb153ffffull, 0x6730d2a0f6b0f624ull, 0x64774b84f38512bfull,
                                    0x4b1ba7b6434bacd7ull, 0x1a0111ea397fe69aull};
  fctx_init(&CURVES[0].fr, 4, bn_r); fctx_init(&CURVES[0].fq, 4, bn_p); CURVES[0].two_adicity = 28; CURVES[0].fq_bytes = 32;
  fctx_init(&CURVES[1].fr, 4, bls_r); fctx_init(&CURVES[1].fq, 6, bls_p); CURVES[1].two_adicity = 32; CURVES[1].fq_bytes = 48;
  const uint64_t gens[2] = {5, 7};
  for (int k = 0; k < 2; k++) {
    curve_t* c = &CURVES[k];
    fe_from_u64(&c->fr, &c->gen, gens[k]);
    /* root = gen^((r-1) >> S) */
    fe e = c->fr.p; e.l[0] -= 1;
    int s = c->two_adicity;
    for (int i = 0; i < 4; i++) { e.l[i] = (e.l[i] >> s) | (i + 1 < 4 ? e.l[i + 1] << (64 - s) : 0); }
    fe_pow(&c->fr, &c->root, &c->gen, e.l, 4);
  }
  curves_ready = 1;
}

/* OpenMP team size: never more than the CPUs this process may actually run on (affinity mask and cgroup quota) —
 * an oversubscribed team spends its time in barriers. */
#include <sched.h>
static int zko_threads_cached = 0;
static int zko_pool_threads(void) {
#define cached zko_threads_cached
  if (cached) return cached;
  int n = 1;
#ifdef _OPENMP
  n = omp_get_num_procs();     /* NOT omp_get_max_threads(): launchers export OMP_NUM_THREADS=1 (torchrun does for every rank) */
  { const char* e = getenv("ZKO_THREADS"); if (e && atoi(e) > 0) n = atoi(e); }
#endif
  cpu_set_t set;
  if (sched_getaffinity(0, sizeof set, &set) == 0) { int k = CPU_COUNT(&set); if (k > 0 && k < n) n = k; }
  FILE* fp = fopen("/sys/fs/cgroup/cpu.max", "r");
  if (fp) { long long q = -1, per = 0; char buf[64]; if (fscanf(fp, "%63s %lld", buf, &per) == 2 && strcmp(buf, "max") != 0) { q = atoll(buf); if (q > 0 && per > 0) { int k = (int)((q + per - 1) / per); if (k >= 1 && k < n) n = k; } } fclose(fp); }
  if (n < 1) n = 1;
#ifdef _OPENMP
  omp_set_num_threads(n);
#endif
  cached = n;
  return n;
#undef cached
}
static double now_s(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec + 1e-9 * ts.tv_nsec; }

/* canonical little-endian bytes <-> Montgomery element */
static void fe_read(const fctx* f, fe* r, const uint8_t* b, int nbytes) {
  fe t; memset(&t, 0, sizeof t);
  for (int i = 0; i < nbytes; i++) t.l[i >> 3] |= (uint64_t)b[i] << (8 * (i & 7));
  fe_to_mont(f, r, &t);
}
static void fe_write(const fctx* f, uint8_t* b, const fe* a, int nbytes) {
  fe t; fe_from_mont(f, &t, a);
  for (int i = 0; i < nbytes; i++) b[i] = (uint8_t)(t.l[i >> 3] >> (8 * (i & 7)));
}

/* ark uncompressed point encodings (SURVEY.md App. A.3) */
static void g1_read(const curve_t* c, g1_aff* p, const uint8_t* b) {
  int n = c->fq_bytes; uint8_t tmp[96]; memcpy(tmp, b, 2 * n);
  int inf = (tmp[2 * n - 1] >> 6) & 1; tmp[2 * n - 1] &= 0x3f;
  p->inf = inf;
  if (inf) { memset(&p->x, 0, sizeof p->x); memset(&p->y, 0, sizeof p->y); return; }
  fe_read(&c->fq, &p->x, tmp, n); fe_read(&c->fq, &p->y, tmp + n, n);
}
static void g1_write(const curve_t* c, uint8_t* b, const g1_aff* p) {
  int n = c->fq_bytes;
  if (p->inf) { memset(b, 0, 2 * n); b[2 * n - 1] = 0x40; return; }
  fe_write(&c->fq, b, &p->x, n); fe_write(&c->fq, b + n, &p->y, n);
}
static void g2_read(const curve_t* c, g2_aff* p, const uint8_t* b) {
  int n = c->fq_bytes; uint8_t tmp[192]; memcpy(tmp, b, 4 * n);
  int inf = (tmp[4 * n - 1] >> 6) & 1; tmp[4 * n - 1] &= 0x3f;
  p->inf = inf;
  if (inf) { memset(&p->x, 0, sizeof p->x); memset(&p->y, 0, sizeof p->y); return; }
  fe_read(&c->fq, &p->x.c0, tmp, n); fe_read(&c->fq, &p->x.c1, tmp + n, n);
  fe_read(&c->fq, &p->y.c0, tmp + 2 * n, n); fe_read(&c->fq, &p->y.c1, tmp + 3 * n, n);
}
static void g2_write(const curve_t* c, uint8_t* b, const g2_aff* p) {
  int n = c->fq_bytes;
  if (p->inf) { memset(b, 0, 4 * n); b[4 * n - 1] = 0x40; return; }
  fe_write(&c->fq, b, &p->x.c0, n); fe_write(&c->fq, b + n, &p->x.c1, n);
  fe_write(&c->fq, b + 2 * n, &p->y.c0, n); fe_write(&c->fq, b + 3 * n, &p->y.c1, n);
}

/* ------------------------------------------------------------------------------------------- FFT (ark-poly radix-2) */
static void fr_fft(const curve_t* c, fe* a, int log_n, const fe* omega) {
  const fctx* f = &c->fr;
  size_t n = (size_t)1 << log_n;
  if (n == 1) return;
  /* twiddles w^k, k < n/2, built in parallel chunks (ark: roots of unity computed with rayon per call) */
  size_t half_n = n >> 1;
  fe* tw = (fe*)malloc(half_n * sizeof(fe));
  int nt = zko_pool_threads();
  size_t chunk = (half_n + nt - 1) / nt;
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int t = 0; t < nt; t++) {
    size_t lo = (size_t)t * chunk, hi = lo + chunk < half_n ? lo + chunk : half_n;
    if (lo >= hi) continue;
    uint64_t e[1] = {lo};
    fe p; fe_pow(f, &p, omega, e, 1);
    for (size_t k = lo; k < hi; k++) { tw[k] = p; fe_mul(f, &p, &p, omega); }
  }
#pragma omp parallel num_threads(nt)
  {
#pragma omp for schedule(static)
    for (size_t k = 0; k < n; k++) {  /* bit-reversal permutation */
      size_t rk = 0; for (int b = 0; b < log_n; b++) rk |= ((k >> b) & 1) << (log_n - 1 - b);
      if (k < rk) { fe t = a[k]; a[k] = a[rk]; a[rk] = t; }
    }
    for (int s = 1; s <= log_n; s++) {
      size_t m = (size_t)1 << s, half = m >> 1, stride = n / m;
#pragma omp for schedule(static)
      for (size_t k = 0; k < n / 2; k++) {
        size_t blk = k / half, j = k % half, i0 = blk * m + j;
        fe t, u = a[i0];
        fe_mul(f, &t, &a[i0 + half], &tw[j * stride]);
        fe_add(f, &a[i0], &u, &t);
        fe_sub(f, &a[i0 + half], &u, &t);
      }
    }
  }
  free(tw);
}
static void domain_omega(const curve_t* c, int log_n, fe* w) {
  *w = c->root;
  for (int i = log_n; i < c->two_adicity; i++) fe_sqr(&c->fr, w, w);
}
static void fr_scale_powers(const curve_t* c, fe* a, size_t n, const fe* g, const fe* scale) {
  /* a[i] *= scale * g^i, chunked so that it parallelises */
  const fctx* f = &c->fr;
  int nt = zko_pool_threads();
  size_t chunk = (n + nt - 1) / nt;
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int t = 0; t < nt; t++) {
    size_t lo = (size_t)t * chunk, hi = lo + chunk < n ? lo + chunk : n;
    if (lo >= hi) continue;
    uint64_t e[1] = {lo};
    fe p; fe_pow(f, &p, g, e, 1); fe_mul(f, &p, &p, scale);
    for (size_t i = lo; i < hi; i++) { fe_mul(f, &a[i], &a[i], &p); fe_mul(f, &p, &p, g); }
  }
}
/* mode bits: 1 = inverse, 2 = coset */
static void fr_transform(const curve_t* c, fe* a, int log_n, int inverse, int coset) {
  const fctx* f = &c->fr;
  size_t n = (size_t)1 << log_n;
  fe w; domain_omega(c, log_n, &w);
  if (!inverse) {
    if (coset) fr_scale_powers(c, a, n, &c->gen, &f->r1);
    fr_fft(c, a, log_n, &w);
  } else {
    fe wi, ninv, nn; fe_inv(f, &wi, &w);
    fr_fft(c, a, log_n, &wi);
    fe_from_u64(f, &nn, n); fe_inv(f, &ninv, &nn);
    if (coset) { fe gi; fe_inv(f, &gi, &c->gen); fr_scale_powers(c, a, n, &gi, &ninv); }
    else {
#pragma omp parallel for schedule(static)
      for (size_t i = 0; i < n; i++) fe_mul(f, &a[i], &a[i], &ninv);
    }
  }
}

/* ------------------------------------------------------------------------------------------- witness_map */
typedef struct { uint64_t N, ni, nw; const uint64_t* rowptr[3]; const uint32_t* col[3]; const uint64_t* val[3]; } r1cs_t;

static void eval_rows(const curve_t* c, const r1cs_t* r, int k, const fe* z, fe* out) {
  const fctx* f = &c->fr;
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < r->N; i++) {
    fe acc; memset(&acc, 0, sizeof acc);
    for (uint64_t e = r->rowptr[k][i]; e < r->rowptr[k][i + 1]; e++) {
      fe v, t; memset(&v, 0, sizeof v);
      memcpy(v.l, r->val[k] + 4 * e, 32);
      fe_to_mont(f, &v, &v);
      fe_mul(f, &t, &v, &z[r->col[k][e]]);
      fe_add(f, &acc, &acc, &t);
    }
    out[i] = acc;
  }
}

/* h (Montgomery, length n) ; z Montgomery */
static fe* witness_map(const curve_t* c, const r1cs_t* r, const fe* z, int* log_n_out) {
  const fctx* f = &c->fr;
  uint64_t dom = r->N + r->ni; size_t n = 1; int lg = 0;
  while (n < dom) { n <<= 1; lg++; }
  *log_n_out = lg;
  fe* a = (fe*)calloc(n, sizeof(fe)); fe* b = (fe*)calloc(n, sizeof(fe)); fe* cc = (fe*)calloc(n, sizeof(fe));
  eval_rows(c, r, 0, z, a); eval_rows(c, r, 1, z, b);
  for (uint64_t j = 0; j < r->ni; j++) a[r->N + j] = z[j];
  fr_transform(c, a, lg, 1, 0); fr_transform(c, b, lg, 1, 0);
  fr_transform(c, a, lg, 0, 1); fr_transform(c, b, lg, 0, 1);
#pragma omp parallel for schedule(static)
  for (size_t i = 0; i < n; i++) fe_mul(f, &a[i], &a[i], &b[i]);
  eval_rows(c, r, 2, z, cc);
  fr_transform(c, cc, lg, 1, 0); fr_transform(c, cc, lg, 0, 1);
  fe gn = c->gen, zinv;
  for (int i = 0; i < lg; i++) fe_sqr(f, &gn, &gn);
  fe_sub(f, &gn, &gn, &f->r1); fe_inv(f, &zinv, &gn);
#pragma omp parallel for schedule(static)
  for (size_t i = 0; i < n; i++) { fe_sub(f, &a[i], &a[i], &cc[i]); fe_mul(f, &a[i], &a[i], &zinv); }
  fr_transform(c, a, lg, 1, 1);
  free(b); free(cc);
  return a;
}

/* ------------------------------------------------------------------------------------------- exported API */
#define EXPORT __attribute__((visibility("default")))

EXPORT int zko_threads(void) { return zko_pool_threads(); }
/* explicit team size (bench.py passes the usable core count so that a launcher's OMP_NUM_THREADS=1 — torchrun sets it for
 * every rank — cannot starve the CPU arm) */
EXPORT void zko_set_threads(int n) {
#ifdef _OPENMP
  if (n > 0) { omp_set_num_threads(n); zko_threads_cached = n; }
#else
  (void)n;
#endif
}

/* field 0 = Fr, 1 = Fq; op 0 mul, 1 add, 2 sub, 3 inv; canonical LE limbs in/out (4 or 6 u64 each) */
EXPORT int zko_field_op(int curve, int field, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n) {
  curves_init();
  const fctx* f = field == 0 ? &CURVES[curve].fr : &CURVES[curve].fq;
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < n; i++) {
    fe x, y, r; memset(&x, 0, sizeof x); memset(&y, 0, sizeof y);
    memcpy(x.l, a + i * f->n, 8 * f->n); if (b) memcpy(y.l, b + i * f->n, 8 * f->n);
    fe_to_mont(f, &x, &x); fe_to_mont(f, &y, &y);
    switch (op) { case 0: fe_mul(f, &r, &x, &y); break; case 1: fe_add(f, &r, &x, &y); break; case 2: fe_sub(f, &r, &x, &y); break; default: fe_inv(f, &r, &x); }
    fe_from_mont(f, &r, &r);
    memcpy(out + i * f->n, r.l, 8 * f->n);
  }
  return 0;
}

EXPORT int zko_ntt(int curve, uint64_t* data, uint32_t log_n, int inverse, int coset) {
  curves_init();
  const curve_t* c = &CURVES[curve];
  size_t n = (size_t)1 << log_n;
  fe* a = (fe*)calloc(n, sizeof(fe));
  for (size_t i = 0; i < n; i++) { memcpy(a[i].l, data + 4 * i, 32); fe_to_mont(&c->fr, &a[i], &a[i]); }
  fr_transform(c, a, (int)log_n, inverse, coset);
  for (size_t i = 0; i < n; i++) { fe t; fe_from_mont(&c->fr, &t, &a[i]); memcpy(data + 4 * i, t.l, 32); }
  free(a);
  return 0;
}

EXPORT int zko_msm(int curve, int group, const uint8_t* points, const uint64_t* scalars, uint64_t n, uint8_t* out) {
  curves_init();
  const curve_t* c = &CURVES[curve];
  if (group == 1) {
    g1_aff* p = (g1_aff*)malloc((n ? n : 1) * sizeof(g1_aff));
#pragma omp parallel for schedule(static)
    for (uint64_t i = 0; i < n; i++) g1_read(c, &p[i], points + i * 2 * c->fq_bytes);
    g1_jac r; g1_msm(&c->fq, c->fr.bits, &r, p, scalars, n);
    g1_aff ra; g1_to_affine(&c->fq, &ra, &r); g1_write(c, out, &ra);
    free(p);
  } else {
    g2_aff* p = (g2_aff*)malloc((n ? n : 1) * sizeof(g2_aff));
#pragma omp parallel for schedule(static)
    for (uint64_t i = 0; i < n; i++) g2_read(c, &p[i], points + i * 4 * c->fq_bytes);
    g2_jac r; g2_msm(&c->fq, c->fr.bits, &r, p, scalars, n);
    g2_aff ra; g2_to_affine(&c->fq, &ra, &r); g2_write(c, out, &ra);
    free(p);
  }
  return 0;
}

static fe* load_z(const curve_t* c, const uint64_t* z, uint64_t m) {
  fe* zm = (fe*)calloc(m ? m : 1, sizeof(fe));
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < m; i++) { memcpy(zm[i].l, z + 4 * i, 32); fe_to_mont(&c->fr, &zm[i], &zm[i]); }
  return zm;
}

EXPORT int zko_witness_map(int curve, uint64_t N, uint64_t ni, uint64_t nw, const uint64_t* a_rowptr, const uint32_t* a_col,
                           const uint64_t* a_val, const uint64_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val,
                           const uint64_t* c_rowptr, const uint32_t* c_col, const uint64_t* c_val, const uint64_t* z,
                           uint64_t* h_out) {
  curves_init();
  const curve_t* c = &CURVES[curve];
  r1cs_t r = {N, ni, nw, {a_rowptr, b_rowptr, c_rowptr}, {a_col, b_col, c_col}, {a_val, b_val, c_val}};
  fe* zm = load_z(c, z, ni + nw);
  int lg; fe* h = witness_map(c, &r, zm, &lg);
  size_t n = (size_t)1 << lg;
  for (size_t i = 0; i < n; i++) { fe t; fe_from_mont(&c->fr, &t, &h[i]); memcpy(h_out + 4 * i, t.l, 32); }
  free(h); free(zm);
  return 0;
}

/* ark-groth16 create_proof_with_reduction; times[0..4] = deserialize, witness_map, msm G1 total, msm G2, total (seconds) */
EXPORT int zko_groth16_prove(int curve, const uint8_t* pk, uint64_t pk_len, uint64_t N, uint64_t ni, uint64_t nw,
                             const uint64_t* a_rowptr, const uint32_t* a_col, const uint64_t* a_val,
                             const uint64_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val,
                             const uint64_t* c_rowptr, const uint32_t* c_col, const uint64_t* c_val,
                             const uint64_t* z, const uint64_t* r_s, const uint64_t* s_s, uint8_t* proof_out, double* times) {
  curves_init();
  const curve_t* c = &CURVES[curve];
  const fctx* fq = &c->fq;
  const int g1b = 2 * c->fq_bytes, g2b = 4 * c->fq_bytes;
  double t0 = now_s();
  /* ProvingKey::deserialize_unchecked */
  uint64_t off = 0;
#define NEED(k) do { if (off + (k) > pk_len) return 2; } while (0)
  g1_aff alpha1, beta1, delta1; g2_aff beta2, delta2;
  NEED(g1b); g1_read(c, &alpha1, pk + off); off += g1b;
  NEED(3 * g2b); g2_read(c, &beta2, pk + off); off += g2b; off += g2b; g2_read(c, &delta2, pk + off); off += g2b;
  uint64_t nabc; NEED(8); memcpy(&nabc, pk + off, 8); off += 8; NEED(nabc * g1b); off += nabc * g1b;
  NEED(2 * g1b); g1_read(c, &beta1, pk + off); off += g1b; g1_read(c, &delta1, pk + off); off += g1b;
  uint64_t m; NEED(8); memcpy(&m, pk + off, 8); off += 8; NEED(m * g1b);
  if (m != ni + nw || nabc != ni) return 2;
  g1_aff* aq = (g1_aff*)malloc((m + 1) * sizeof(g1_aff));
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < m; i++) g1_read(c, &aq[i], pk + off + i * g1b);
  off += m * g1b;
  uint64_t m1; NEED(8); memcpy(&m1, pk + off, 8); off += 8; NEED(m1 * g1b); if (m1 != m) return 2;
  g1_aff* b1q = (g1_aff*)malloc((m + 1) * sizeof(g1_aff));
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < m; i++) g1_read(c, &b1q[i], pk + off + i * g1b);
  off += m * g1b;
  uint64_t m2; NEED(8); memcpy(&m2, pk + off, 8); off += 8; NEED(m2 * g2b); if (m2 != m) return 2;
  g2_aff* b2q = (g2_aff*)malloc((m + 1) * sizeof(g2_aff));
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < m; i++) g2_read(c, &b2q[i], pk + off + i * g2b);
  off += m * g2b;
  uint64_t hl; NEED(8); memcpy(&hl, pk + off, 8); off += 8; NEED(hl * g1b);
  g1_aff* hq = (g1_aff*)malloc((hl + 1) * sizeof(g1_aff));
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < hl; i++) g1_read(c, &hq[i], pk + off + i * g1b);
  off += hl * g1b;
  uint64_t ll; NEED(8); memcpy(&ll, pk + off, 8); off += 8; NEED(ll * g1b);
  g1_aff* lq = (g1_aff*)malloc((ll + 1) * sizeof(g1_aff));
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < ll; i++) g1_read(c, &lq[i], pk + off + i * g1b);
  off += ll * g1b;
  if (off != pk_len || ll != m - ni) return 2;
  double t1 = now_s();

  r1cs_t r = {N, ni, nw, {a_rowptr, b_rowptr, c_rowptr}, {a_col, b_col, c_col}, {a_val, b_val, c_val}};
  fe* zm = load_z(c, z, m);
  int lg; fe* h = witness_map(c, &r, zm, &lg);
  size_t n = (size_t)1 << lg;
  if (hl + 1 != n && !(n == 1 && hl == 0)) return 2;
  uint64_t* hs = (uint64_t*)malloc((n + 1) * 32);
#pragma omp parallel for schedule(static)
  for (size_t i = 0; i < n; i++) { fe t; fe_from_mont(&c->fr, &t, &h[i]); memcpy(hs + 4 * i, t.l, 32); }
  double t2 = now_s();

  g1_jac h_acc, l_acc, a_acc, b1_acc; g2_jac b2_acc;
  uint64_t hcnt = hl < n ? hl : n;
  g1_msm(fq, c->fr.bits, &h_acc, hq, hs, hcnt);
  g1_msm(fq, c->fr.bits, &l_acc, lq, z + 4 * ni, ll);
  g1_msm(fq, c->fr.bits, &a_acc, aq + 1, z + 4, m - 1);
  g1_msm(fq, c->fr.bits, &b1_acc, b1q + 1, z + 4, m - 1);
  double t3 = now_s();
  g2_msm(fq, c->fr.bits, &b2_acc, b2q + 1, z + 4, m - 1);
  double t4 = now_s();

  /* r*s (canonical) */
  fe rm, sm, rsm, rs; memset(&rm, 0, sizeof rm); memset(&sm, 0, sizeof sm);
  memcpy(rm.l, r_s, 32); memcpy(sm.l, s_s, 32);
  fe_to_mont(&c->fr, &rm, &rm); fe_to_mont(&c->fr, &sm, &sm); fe_mul(&c->fr, &rsm, &rm, &sm); fe_from_mont(&c->fr, &rs, &rsm);
  g1_jac d1, t, ga, gb1, gc; g2_jac d2, gb2;
  g1_from_affine(fq, &d1, &delta1);
  /* g_a = r*delta1 + a_query[0] + a_acc + alpha1 */
  g1_mul(fq, &ga, &d1, r_s, 4); g1_add_mixed(fq, &ga, &ga, &aq[0]); g1_add(fq, &ga, &ga, &a_acc); g1_add_mixed(fq, &ga, &ga, &alpha1);
  g1_mul(fq, &gb1, &d1, s_s, 4); g1_add_mixed(fq, &gb1, &gb1, &b1q[0]); g1_add(fq, &gb1, &gb1, &b1_acc); g1_add_mixed(fq, &gb1, &gb1, &beta1);
  g2_from_affine(fq, &d2, &delta2);
  g2_mul(fq, &gb2, &d2, s_s, 4); g2_add_mixed(fq, &gb2, &gb2, &b2q[0]); g2_add(fq, &gb2, &gb2, &b2_acc); g2_add_mixed(fq, &gb2, &gb2, &beta2);
  g1_mul(fq, &gc, &ga, s_s, 4);
  g1_mul(fq, &t, &gb1, r_s, 4); g1_add(fq, &gc, &gc, &t);
  g1_mul(fq, &t, &d1, rs.l, 4); g1_neg(fq, &t, &t); g1_add(fq, &gc, &gc, &t);
  g1_add(fq, &gc, &gc, &l_acc); g1_add(fq, &gc, &gc, &h_acc);
  g1_aff pa, pc; g2_aff pb;
  g1_to_affine(fq, &pa, &ga); g2_to_affine(fq, &pb, &gb2); g1_to_affine(fq, &pc, &gc);
  g1_write(c, proof_out, &pa); g2_write(c, proof_out + g1b, &pb); g1_write(c, proof_out + g1b + g2b, &pc);
  double t5 = now_s();
  if (times) { times[0] = t1 - t0; times[1] = t2 - t1; times[2] = t3 - t2; times[3] = t4 - t3; times[4] = t5 - t0; }
  free(aq); free(b1q); free(b2q); free(hq); free(lq); free(zm); free(h); free(hs);
  return 0;
}

/* ------------------------------------------------------------------------------------------- setup
 * ark-groth16 0.3.0 generate_parameters with an explicit trapdoor (SURVEY.md App. B.6):
 * trapdoor7 = alpha, beta, gamma, delta, tau, g1_k, g2_k (canonical LE), generators g1 = g1_k*G1, g2 = g2_k*G2.
 * Writes ProvingKey::serialize_unchecked bytes.  Returns 0, or 2 if pk_cap is too small. */
static void read_fr(const curve_t* c, fe* r, const uint64_t* p) { memset(r, 0, sizeof *r); memcpy(r->l, p, 32); fe_to_mont(&c->fr, r, r); }

static void std_generators(int curve, const curve_t* c, g1_aff* g1, g2_aff* g2) {
  static const char* BN_G2[4] = {
    "1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed", "198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2",
    "12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa", "090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b"};
  static const char* BLS_G1[2] = {
    "17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb",
    "08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1"};
  static const char* BLS_G2[4] = {
    "024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8",
    "13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e",
    "0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801",
    "0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be"};
  const fctx* f = &c->fq;
  #define HEXFE(dst, str) do { fe t_; memset(&t_, 0, sizeof t_); size_t L_ = strlen(str); for (size_t i_ = 0; i_ < L_; i_++) { char ch = (str)[L_ - 1 - i_]; uint64_t v_ = ch <= '9' ? ch - '0' : ch - 'a' + 10; t_.l[i_ >> 4] |= v_ << (4 * (i_ & 15)); } fe_to_mont(f, &(dst), &t_); } while (0)
  g1->inf = 0; g2->inf = 0;
  if (curve == 0) {
    fe_from_u64(f, &g1->x, 1); fe_from_u64(f, &g1->y, 2);
    HEXFE(g2->x.c0, BN_G2[0]); HEXFE(g2->x.c1, BN_G2[1]); HEXFE(g2->y.c0, BN_G2[2]); HEXFE(g2->y.c1, BN_G2[3]);
  } else {
    HEXFE(g1->x, BLS_G1[0]); HEXFE(g1->y, BLS_G1[1]);
    HEXFE(g2->x.c0, BLS_G2[0]); HEXFE(g2->x.c1, BLS_G2[1]); HEXFE(g2->y.c0, BLS_G2[2]); HEXFE(g2->y.c1, BLS_G2[3]);
  }
}

/* fixed-base multiples with an 8-bit window table (ark uses FixedBaseMSM; the points are the same) */
static void g1_fixed_base(const curve_t* c, const g1_jac* g, const fe* scalars_mont, uint64_t n, uint8_t* out) {
  const fctx* fq = &c->fq;
  g1_aff* table = (g1_aff*)malloc(32 * 256 * sizeof(g1_aff));
  g1_jac base = *g;
  for (int j = 0; j < 32; j++) {
    g1_jac acc; g1_set_inf(fq, &acc);
    for (int d = 0; d < 256; d++) { g1_to_affine(fq, &table[j * 256 + d], &acc); g1_add(fq, &acc, &acc, &base); }
    for (int b = 0; b < 8; b++) g1_dbl(fq, &base, &base);
  }
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < n; i++) {
    fe s; fe_from_mont(&c->fr, &s, &scalars_mont[i]);
    g1_jac acc; g1_set_inf(fq, &acc);
    for (int j = 0; j < 32; j++) { unsigned d = (unsigned)(s.l[j >> 3] >> (8 * (j & 7))) & 255u; if (d) g1_add_mixed(fq, &acc, &acc, &table[j * 256 + d]); }
    g1_aff a; g1_to_affine(fq, &a, &acc); g1_write(c, out + i * 2 * c->fq_bytes, &a);
  }
  free(table);
}
static void g2_fixed_base(const curve_t* c, const g2_jac* g, const fe* scalars_mont, uint64_t n, uint8_t* out) {
  const fctx* fq = &c->fq;
  g2_aff* table = (g2_aff*)malloc(32 * 256 * sizeof(g2_aff));
  g2_jac base = *g;
  for (int j = 0; j < 32; j++) {
    g2_jac acc; g2_set_inf(fq, &acc);
    for (int d = 0; d < 256; d++) { g2_to_affine(fq, &table[j * 256 + d], &acc); g2_add(fq, &acc, &acc, &base); }
    for (int b = 0; b < 8; b++) g2_dbl(fq, &base, &base);
  }
#pragma omp parallel for schedule(static)
  for (uint64_t i = 0; i < n; i++) {
    fe s; fe_from_mont(&c->fr, &s, &scalars_mont[i]);
    g2_jac acc; g2_set_inf(fq, &acc);
    for (int j = 0; j < 32; j++) { unsigned d = (unsigned)(s.l[j >> 3] >> (8 * (j & 7))) & 255u; if (d) g2_add_mixed(fq, &acc, &acc, &table[j * 256 + d]); }
    g2_aff a; g2_to_affine(fq, &a, &acc); g2_write(c, out + i * 4 * c->fq_bytes, &a);
  }
  free(table);
}

EXPORT int zko_groth16_setup(int curve, uint64_t N, uint64_t ni, uint64_t nw, const uint64_t* a_rowptr, const uint32_t* a_col,
                             const uint64_t* a_val, const uint64_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val,
                             const uint64_t* c_rowptr, const uint32_t* c_col, const uint64_t* c_val, const uint64_t* trapdoor7,
                             uint8_t* pk_out, uint64_t pk_cap, uint64_t* pk_len) {
  curves_init();
  const curve_t* c = &CURVES[curve];
  const fctx* f = &c->fr;
  const int g1b = 2 * c->fq_bytes, g2b = 4 * c->fq_bytes;
  uint64_t m = ni + nw, dom = N + ni; size_t n = 1; int lg = 0;
  while (n < dom) { n <<= 1; lg++; }
  uint64_t total = g1b + 3 * g2b + 8 + ni * g1b + 2 * g1b + 2 * (8 + m * g1b) + 8 + m * g2b + 8 + (n - 1) * g1b + 8 + (m - ni) * g1b;
  *pk_len = total;
  if (pk_cap < total) return 2;
  fe alpha, beta, gamma, delta, tau; uint64_t gk[2][4];
  read_fr(c, &alpha, trapdoor7); read_fr(c, &beta, trapdoor7 + 4); read_fr(c, &gamma, trapdoor7 + 8);
  read_fr(c, &delta, trapdoor7 + 12); read_fr(c, &tau, trapdoor7 + 16);
  memcpy(gk[0], trapdoor7 + 20, 32); memcpy(gk[1], trapdoor7 + 24, 32);
  /* u = ifft(tau^k) = Lagrange coefficients at tau */
  fe* pw = (fe*)malloc(n * sizeof(fe)); fe* u = (fe*)malloc(n * sizeof(fe));
  pw[0] = f->r1; for (size_t i = 1; i < n; i++) fe_mul(f, &pw[i], &pw[i - 1], &tau);
  memcpy(u, pw, n * sizeof(fe));
  fr_transform(c, u, lg, 1, 0);
  fe* abc[3];
  const uint64_t* rp[3] = {a_rowptr, b_rowptr, c_rowptr}; const uint32_t* cl[3] = {a_col, b_col, c_col}; const uint64_t* vl[3] = {a_val, b_val, c_val};
  for (int k = 0; k < 3; k++) {
    abc[k] = (fe*)calloc(m ? m : 1, sizeof(fe));
    if (k == 0) for (uint64_t i = 0; i < ni; i++) abc[0][i] = u[N + i];
    for (uint64_t row = 0; row < N; row++)
      for (uint64_t e = rp[k][row]; e < rp[k][row + 1]; e++) {
        fe v, t; read_fr(c, &v, vl[k] + 4 * e); fe_mul(f, &t, &v, &u[row]); fe_add(f, &abc[k][cl[k][e]], &abc[k][cl[k][e]], &t);
      }
  }
  fe ginv, dinv, zt, hs; fe_inv(f, &ginv, &gamma); fe_inv(f, &dinv, &delta);
  zt = tau; for (int i = 0; i < lg; i++) fe_sqr(f, &zt, &zt);
  fe_sub(f, &zt, &zt, &f->r1); fe_mul(f, &hs, &zt, &dinv);
  fe* lq = (fe*)malloc((m ? m : 1) * sizeof(fe)); fe* hq = (fe*)malloc(n * sizeof(fe));
  for (uint64_t i = 0; i < m; i++) {
    fe t1, t2; fe_mul(f, &t1, &beta, &abc[0][i]); fe_mul(f, &t2, &alpha, &abc[1][i]); fe_add(f, &t1, &t1, &t2); fe_add(f, &t1, &t1, &abc[2][i]);
    fe_mul(f, &lq[i], &t1, i < ni ? &ginv : &dinv);
  }
  for (size_t i = 0; i < n; i++) fe_mul(f, &hq[i], &pw[i], &hs);
  g1_aff s1; g2_aff s2; std_generators(curve, c, &s1, &s2);
  g1_jac j1, g1; g2_jac j2, g2;
  g1_from_affine(&c->fq, &j1, &s1); g2_from_affine(&c->fq, &j2, &s2);
  g1_mul(&c->fq, &g1, &j1, gk[0], 4); g2_mul(&c->fq, &g2, &j2, gk[1], 4);
  uint8_t* o = pk_out; uint64_t len;
  g1_fixed_base(c, &g1, &alpha, 1, o); o += g1b;
  g2_fixed_base(c, &g2, &beta, 1, o); o += g2b;
  g2_fixed_base(c, &g2, &gamma, 1, o); o += g2b;
  g2_fixed_base(c, &g2, &delta, 1, o); o += g2b;
  len = ni; memcpy(o, &len, 8); o += 8; g1_fixed_base(c, &g1, lq, ni, o); o += ni * g1b;
  g1_fixed_base(c, &g1, &beta, 1, o); o += g1b;
  g1_fixed_base(c, &g1, &delta, 1, o); o += g1b;
  len = m; memcpy(o, &len, 8); o += 8; g1_fixed_base(c, &g1, abc[0], m, o); o += m * g1b;
  memcpy(o, &len, 8); o += 8; g1_fixed_base(c, &g1, abc[1], m, o); o += m * g1b;
  memcpy(o, &len, 8); o += 8; g2_fixed_base(c, &g2, abc[1], m, o); o += m * g2b;
  len = n - 1; memcpy(o, &len, 8); o += 8; g1_fixed_base(c, &g1, hq, n - 1, o); o += (n - 1) * g1b;
  len = m - ni; memcpy(o, &len, 8); o += 8; g1_fixed_base(c, &g1, lq + ni, m - ni, o); o += (m - ni) * g1b;
  free(pw); free(u); free(abc[0]); free(abc[1]); free(abc[2]); free(lq); free(hq);
  return (uint64_t)(o - pk_out) == total ? 0 : 6;
}

/* ------------------------------------------------------------------------------------------- Lagrange coefficients
 * u[j] = L_j(tau) = Z(tau)/n * w^j / (tau - w^j) over the domain of size 2^lg (closed form, NOT an inverse FFT), and
 * zt = Z(tau) = tau^n - 1, all Montgomery.  Chunked over the pool: per chunk w^j by one exponentiation and a running product,
 * one inversion per chunk (Montgomery's trick).  Returns 0, or 3 if tau lies in the domain. */
static int lagrange_at_tau(const curve_t* c, int lg, const fe* tau, fe* u, fe* zt_out) {
  const fctx* f = &c->fr;
  const size_t n = (size_t)1 << lg;
  fe w; domain_omega(c, lg, &w);
  fe zt = *tau; for (int i = 0; i < lg; i++) fe_sqr(f, &zt, &zt);
  fe_sub(f, &zt, &zt, &f->r1);
  *zt_out = zt;
  fe nn, ninv, scale; fe_from_u64(f, &nn, n); fe_inv(f, &ninv, &nn); fe_mul(f, &scale, &zt, &ninv);
  fe* pre = (fe*)malloc(n * sizeof(fe));
  const int nt = zko_pool_threads();
  const size_t chunk = (n + nt - 1) / nt;
  int bad = 0;
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int t = 0; t < nt; t++) {
    size_t lo = (size_t)t * chunk, hi = lo + chunk < n ? lo + chunk : n;
    if (lo >= hi) continue;
    uint64_t e[1] = {lo};
    fe wj; fe_pow(f, &wj, &w, e, 1);
    fe run = f->r1;
    for (size_t j = lo; j < hi; j++) {              /* u[j] = w^j (kept), pre[j] = prod_{k<j} (tau - w^k) */
      fe d; fe_sub(f, &d, tau, &wj);
      if (fe_is_zero(f, &d)) { bad = 1; d = f->r1; }
      u[j] = wj; pre[j] = run;
      fe_mul(f, &run, &run, &d);
      fe_mul(f, &wj, &wj, &w);
    }
    fe inv; fe_inv(f, &inv, &run);
    for (size_t j = hi; j-- > lo;) {
      fe d, dinv; fe_sub(f, &d, tau, &u[j]);
      fe_mul(f, &dinv, &inv, &pre[j]);              /* 1 / (tau - w^j) */
      fe_mul(f, &inv, &inv, &d);
      fe_mul(f, &u[j], &u[j], &dinv);
      fe_mul(f, &u[j], &u[j], &scale);
    }
  }
  free(pre);
  return bad ? 3 : 0;
}

/* g1 = g1_k G1, g2 = g2_k G2 (the generators a key made from this trapdoor uses) */
static void key_generators(int curve, const curve_t* c, const uint64_t* g1_k, const uint64_t* g2_k, g1_jac* g1, g2_jac* g2) {
  g1_aff s1; g2_aff s2; std_generators(curve, c, &s1, &s2);
  g1_jac j1; g2_jac j2;
  g1_from_affine(&c->fq, &j1, &s1); g2_from_affine(&c->fq, &j2, &s2);
  g1_mul(&c->fq, g1, &j1, g1_k, 4); g2_mul(&c->fq, g2, &j2, g2_k, 4);
}

/* ------------------------------------------------------------------------------------------- trapdoor prediction
 * Expected Groth16 proof (A, B, C) for a key made by zko_groth16_setup / zkb_groth16_setup from the SAME explicit
 * trapdoor, computed with Fr arithmetic only plus one scalar multiplication of the generator per proof element —
 * no NTT, no MSM, no proving key (restates oracle/ark.py::trapdoor_expected_proof; Groth16 [ePrint 2016/260] §3.2 with
 * ark-groth16 0.3.0's element order, SURVEY.md App. B.1/B.6):
 *   u_j   = L_j(tau) = Z(tau)/n * w^j / (tau - w^j)            (closed form, batch inversion; NOT an inverse FFT)
 *   Az    = sum_j u_j <A_j, z> + sum_{i<ni} u_{N+i} z_i ;  Bz, Cz likewise (without the instance rows)
 *   a     = alpha + Az + r delta ;  b = beta + Bz + s delta
 *   l     = [ beta (Az - Az|inst) + alpha (Bz - Bz|inst) + (Cz - Cz|inst) ] / delta     (aux variables only)
 *   h     = (Az Bz - Cz) / delta                                  ( = h(tau) Z(tau) / delta )
 *   c     = l + h + s a + r b - r s delta
 *   proof = (a g1, b g2, c g1),  g1 = g1_k G1, g2 = g2_k G2.
 * Returns 0, or 3 if tau lies in the evaluation domain. */
EXPORT int zko_trapdoor_expected(int curve, uint64_t N, uint64_t ni, uint64_t nw, const uint64_t* a_rowptr, const uint32_t* a_col,
                                 const uint64_t* a_val, const uint64_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val,
                                 const uint64_t* c_rowptr, const uint32_t* c_col, const uint64_t* c_val, const uint64_t* trapdoor7,
                                 const uint64_t* z, const uint64_t* r_s, const uint64_t* s_s, uint8_t* proof_out) {
  curves_init();
  const curve_t* c = &CURVES[curve];
  const fctx* f = &c->fr;
  const int g1b = 2 * c->fq_bytes, g2b = 4 * c->fq_bytes;
  const uint64_t m = ni + nw, dom = N + ni; size_t n = 1; int lg = 0;
  while (n < dom) { n <<= 1; lg++; }
  fe alpha, beta, delta, tau, rr, ss; uint64_t gk[2][4];
  read_fr(c, &alpha, trapdoor7); read_fr(c, &beta, trapdoor7 + 4); read_fr(c, &delta, trapdoor7 + 12); read_fr(c, &tau, trapdoor7 + 16);
  memcpy(gk[0], trapdoor7 + 20, 32); memcpy(gk[1], trapdoor7 + 24, 32);
  read_fr(c, &rr, r_s); read_fr(c, &ss, s_s);
  fe* u = (fe*)malloc(n * sizeof(fe));
  fe zt;
  if (lagrange_at_tau(c, lg, &tau, u, &zt)) { free(u); return 3; }
  const int nt = zko_pool_threads();
  fe* zm = load_z(c, z, m);
  const uint64_t* rp[3] = {a_rowptr, b_rowptr, c_rowptr}; const uint32_t* cl[3] = {a_col, b_col, c_col}; const uint64_t* vl[3] = {a_val, b_val, c_val};
  fe all[3], inst[3];
  for (int k = 0; k < 3; k++) {
    fe* pa = (fe*)calloc(nt, sizeof(fe)); fe* pi = (fe*)calloc(nt, sizeof(fe));
    const size_t rchunk = (N + nt - 1) / nt;
#pragma omp parallel for schedule(static) num_threads(nt)
    for (int t = 0; t < nt; t++) {
      size_t lo = (size_t)t * rchunk, hi = lo + rchunk < N ? lo + rchunk : N;
      fe sa, si; memset(&sa, 0, sizeof sa); memset(&si, 0, sizeof si);
      for (size_t row = lo; row < hi; row++) {
        fe ra, ri; memset(&ra, 0, sizeof ra); memset(&ri, 0, sizeof ri);
        for (uint64_t e = rp[k][row]; e < rp[k][row + 1]; e++) {
          fe v, p; read_fr(c, &v, vl[k] + 4 * e);
          fe_mul(f, &p, &v, &zm[cl[k][e]]);
          fe_add(f, &ra, &ra, &p);
          if (cl[k][e] < ni) fe_add(f, &ri, &ri, &p);
        }
        fe_mul(f, &ra, &ra, &u[row]); fe_mul(f, &ri, &ri, &u[row]);
        fe_add(f, &sa, &sa, &ra); fe_add(f, &si, &si, &ri);
      }
      pa[t] = sa; pi[t] = si;
    }
    memset(&all[k], 0, sizeof(fe)); memset(&inst[k], 0, sizeof(fe));
    for (int t = 0; t < nt; t++) { fe_add(f, &all[k], &all[k], &pa[t]); fe_add(f, &inst[k], &inst[k], &pi[t]); }
    free(pa); free(pi);
  }
  for (uint64_t i = 0; i < ni; i++) {               /* the extra rows a[N + i] = z_i of the instance variables */
    fe p; fe_mul(f, &p, &u[N + i], &zm[i]);
    fe_add(f, &all[0], &all[0], &p); fe_add(f, &inst[0], &inst[0], &p);
  }
  free(u); free(zm);
  fe dinv; fe_inv(f, &dinv, &delta);
  fe ad, bd, l, h, cd, t1, t2;
  fe_mul(f, &t1, &rr, &delta); fe_add(f, &ad, &alpha, &all[0]); fe_add(f, &ad, &ad, &t1);
  fe_mul(f, &t1, &ss, &delta); fe_add(f, &bd, &beta, &all[1]); fe_add(f, &bd, &bd, &t1);
  fe_sub(f, &t1, &all[0], &inst[0]); fe_mul(f, &l, &beta, &t1);
  fe_sub(f, &t1, &all[1], &inst[1]); fe_mul(f, &t2, &alpha, &t1); fe_add(f, &l, &l, &t2);
  fe_sub(f, &t1, &all[2], &inst[2]); fe_add(f, &l, &l, &t1);
  fe_mul(f, &l, &l, &dinv);
  fe_mul(f, &h, &all[0], &all[1]); fe_sub(f, &h, &h, &all[2]); fe_mul(f, &h, &h, &dinv);
  fe_add(f, &cd, &l, &h);
  fe_mul(f, &t1, &ss, &ad); fe_add(f, &cd, &cd, &t1);
  fe_mul(f, &t1, &rr, &bd); fe_add(f, &cd, &cd, &t1);
  fe_mul(f, &t1, &rr, &ss); fe_mul(f, &t1, &t1, &delta); fe_sub(f, &cd, &cd, &t1);
  fe ac, bc, cc; fe_from_mont(f, &ac, &ad); fe_from_mont(f, &bc, &bd); fe_from_mont(f, &cc, &cd);
  g1_jac g1, pa1, pc1; g2_jac g2, pb2;
  key_generators(curve, c, gk[0], gk[1], &g1, &g2);
  g1_mul(&c->fq, &pa1, &g1, ac.l, 4); g2_mul(&c->fq, &pb2, &g2, bc.l, 4); g1_mul(&c->fq, &pc1, &g1, cc.l, 4);
  g1_aff oa, oc; g2_aff ob;
  g1_to_affine(&c->fq, &oa, &pa1); g2_to_affine(&c->fq, &ob, &pb2); g1_to_affine(&c->fq, &oc, &pc1);
  g1_write(c, proof_out, &oa); g2_write(c, proof_out + g1b, &ob); g1_write(c, proof_out + g1b + g2b, &oc);
  return 0;
}

/* ------------------------------------------------------------------------------------------- GM17 (Groth-Maller 2017)
 * The square arithmetic program of ark-gm17's R1CStoSAP (restated in oracle/gm17.py): R1CS row i becomes SAP rows 2i, 2i + 1
 *   (A_i + B_i)^2 = 4 C_i + x_i,   (A_i - B_i)^2 = x_i,     x_i = (A_i z - B_i z)^2 at SAP column m + i,
 * then the constant row e = 2N (1^2 = 1) and per public input j >= 1 rows e + 2j - 1, e + 2j
 *   (z_j + 1)^2 = 4 z_j + y_j,     (z_j - 1)^2 = y_j,       y_j = (z_j - 1)^2 at SAP column m + N - 1 + j,
 * over a domain of n = 2^lg >= 2N + 2(ni - 1) + 1 points; nv = m + N + ni - 1 SAP variables (the constant included).
 * trapdoor6 = alpha, beta, gamma, tau, g1_k, g2_k (canonical LE). */
static void gm17_domain(uint64_t N, uint64_t ni, size_t* n, int* lg) {
  const uint64_t rows = 2 * N + 2 * (ni - 1) + 1;
  *n = 1; *lg = 0;
  while (*n < rows) { *n <<= 1; (*lg)++; }
}

/* <M_row, z> over all columns and over the instance columns (< ni) alone */
static void row_dot(const curve_t* c, const r1cs_t* r, int k, uint64_t row, const fe* zm, fe* all, fe* inst) {
  const fctx* f = &c->fr;
  memset(all, 0, sizeof *all); memset(inst, 0, sizeof *inst);
  for (uint64_t e = r->rowptr[k][row]; e < r->rowptr[k][row + 1]; e++) {
    fe v, p; read_fr(c, &v, r->val[k] + 4 * e);
    fe_mul(f, &p, &v, &zm[r->col[k][e]]);
    fe_add(f, all, all, &p);
    if (r->col[k][e] < r->ni) fe_add(f, inst, inst, &p);
  }
}

/* u_i(tau) ("a") and w_i(tau) ("c") of every SAP variable (canonical, nv x 4 limbs each) and Z(tau): R1CStoSAP's
 * instance_map_with_evaluation, with the Lagrange coefficients in closed form.  Returns 0, or 3 if tau lies in the domain. */
EXPORT int zko_gm17_sap_at_tau(int curve, uint64_t N, uint64_t ni, uint64_t nw, const uint64_t* a_rowptr, const uint32_t* a_col,
                               const uint64_t* a_val, const uint64_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val,
                               const uint64_t* c_rowptr, const uint32_t* c_col, const uint64_t* c_val, const uint64_t* tau_s,
                               uint64_t* a_out, uint64_t* c_out, uint64_t* zt_out) {
  curves_init();
  const curve_t* c = &CURVES[curve];
  const fctx* f = &c->fr;
  const uint64_t m = ni + nw, nv = m + N + ni - 1, e_off = 2 * N;
  size_t n; int lg; gm17_domain(N, ni, &n, &lg);
  fe tau, zt; read_fr(c, &tau, tau_s);
  fe* u = (fe*)malloc(n * sizeof(fe));
  if (lagrange_at_tau(c, lg, &tau, u, &zt)) { free(u); return 3; }
  fe* a = (fe*)calloc(nv, sizeof(fe)); fe* cc = (fe*)calloc(nv, sizeof(fe));
  const uint64_t* rp[3] = {a_rowptr, b_rowptr, c_rowptr}; const uint32_t* cl[3] = {a_col, b_col, c_col}; const uint64_t* vl[3] = {a_val, b_val, c_val};
  for (uint64_t row = 0; row < N; row++) {
    fe w[3];
    fe_add(f, &w[0], &u[2 * row], &u[2 * row + 1]);              /* A: u_2i + u_2i+1 */
    fe_sub(f, &w[1], &u[2 * row], &u[2 * row + 1]);              /* B: u_2i - u_2i+1 */
    fe_dbl(f, &w[2], &u[2 * row]); fe_dbl(f, &w[2], &w[2]);      /* C: 4 u_2i */
    for (int k = 0; k < 3; k++) {
      fe* dst = k == 2 ? cc : a;
      for (uint64_t e = rp[k][row]; e < rp[k][row + 1]; e++) {
        fe v, p; read_fr(c, &v, vl[k] + 4 * e); fe_mul(f, &p, &v, &w[k]); fe_add(f, &dst[cl[k][e]], &dst[cl[k][e]], &p);
      }
    }
    fe_add(f, &cc[m + row], &cc[m + row], &w[0]);                /* x_i */
  }
  fe_add(f, &a[0], &a[0], &u[e_off]); fe_add(f, &cc[0], &cc[0], &u[e_off]);
  for (uint64_t j = 1; j < ni; j++) {
    const fe* u1 = &u[e_off + 2 * j - 1]; const fe* u2 = &u[e_off + 2 * j];
    fe s, d, q; fe_add(f, &s, u1, u2); fe_sub(f, &d, u1, u2); fe_dbl(f, &q, u1); fe_dbl(f, &q, &q);
    fe_add(f, &a[j], &a[j], &s); fe_add(f, &a[0], &a[0], &d);
    fe_add(f, &cc[j], &cc[j], &q); fe_add(f, &cc[m + N - 1 + j], &cc[m + N - 1 + j], &s);
  }
  for (uint64_t i = 0; i < nv; i++) {
    fe t; fe_from_mont(f, &t, &a[i]); memcpy(a_out + 4 * i, t.l, 32);
    fe_from_mont(f, &t, &cc[i]); memcpy(c_out + 4 * i, t.l, 32);
  }
  fe t; fe_from_mont(f, &t, &zt); memcpy(zt_out, t.l, 32);
  free(u); free(a); free(cc);
  return 0;
}

/* Expected GM17 proof (A, B, C) for a key made by zkb_gm17_setup from the SAME explicit trapdoor, with Fr arithmetic and three
 * generator multiplications — no NTT, no MSM, no key (restates oracle/gm17.py::trapdoor_expected_proof; Groth-Maller Fig. 4 with
 * a(x) masked by d1 Z and c(x) by d2 Z):
 *   a0    = sum_i u_i(tau) s_i,  c0 = sum_i w_i(tau) s_i     over the full SAP assignment s = [z | x | y]
 *           (per R1CS row: (u_2i + u_2i+1) A_i z + (u_2i - u_2i+1) B_i z, and 4 u_2i C_i z + (u_2i + u_2i+1) x_i; then the extra rows)
 *   at    = a0 + d1 Z,  ct = c0 + d2 Z,  ht = (at^2 - ct) / Z
 *   aux   = sum_(i >= ni) (gamma^2 w_i + (alpha + beta) gamma u_i) s_i       (a0, c0 minus their instance-column parts)
 *   A     = gamma (at + r Z) g1,  B = the same dlog times g2
 *   C     = [aux + d1 (alpha + beta) gamma Z + d2 gamma^2 Z + r^2 gamma^2 Z^2 + r (alpha + beta) gamma Z + gamma^2 Z (ht + 2 r at)] g1
 * Returns 0, or 3 if tau lies in the SAP domain. */
EXPORT int zko_gm17_trapdoor_expected(int curve, uint64_t N, uint64_t ni, uint64_t nw, const uint64_t* a_rowptr, const uint32_t* a_col,
                                      const uint64_t* a_val, const uint64_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val,
                                      const uint64_t* c_rowptr, const uint32_t* c_col, const uint64_t* c_val, const uint64_t* trapdoor6,
                                      const uint64_t* z, const uint64_t* d1_s, const uint64_t* d2_s, const uint64_t* r_s,
                                      uint8_t* proof_out) {
  curves_init();
  const curve_t* c = &CURVES[curve];
  const fctx* f = &c->fr;
  const int g1b = 2 * c->fq_bytes, g2b = 4 * c->fq_bytes;
  const uint64_t m = ni + nw, e_off = 2 * N;
  size_t n; int lg; gm17_domain(N, ni, &n, &lg);
  fe alpha, beta, gamma, tau, d1, d2, rr;
  read_fr(c, &alpha, trapdoor6); read_fr(c, &beta, trapdoor6 + 4); read_fr(c, &gamma, trapdoor6 + 8); read_fr(c, &tau, trapdoor6 + 12);
  read_fr(c, &d1, d1_s); read_fr(c, &d2, d2_s); read_fr(c, &rr, r_s);
  fe* u = (fe*)malloc(n * sizeof(fe));
  fe zt;
  if (lagrange_at_tau(c, lg, &tau, u, &zt)) { free(u); return 3; }
  fe* zm = load_z(c, z, m);
  r1cs_t r = {N, ni, nw, {a_rowptr, b_rowptr, c_rowptr}, {a_col, b_col, c_col}, {a_val, b_val, c_val}};
  /* per-row sums: [0] a0, [1] a0 over instance columns, [2] c0, [3] c0 over instance columns; per-thread partials */
  const int nt = zko_pool_threads();
  fe* part = (fe*)calloc(4 * (size_t)nt, sizeof(fe));
  const size_t rchunk = (N + nt - 1) / nt;
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int t = 0; t < nt; t++) {
    size_t lo = (size_t)t * rchunk, hi = lo + rchunk < N ? lo + rchunk : N;
    fe s[4]; memset(s, 0, sizeof s);
    for (size_t row = lo; row < hi; row++) {
      fe az, azi, bz, bzi, cz, czi, ua, us, u4, x, p;
      row_dot(c, &r, 0, row, zm, &az, &azi); row_dot(c, &r, 1, row, zm, &bz, &bzi); row_dot(c, &r, 2, row, zm, &cz, &czi);
      fe_add(f, &ua, &u[2 * row], &u[2 * row + 1]); fe_sub(f, &us, &u[2 * row], &u[2 * row + 1]);
      fe_dbl(f, &u4, &u[2 * row]); fe_dbl(f, &u4, &u4);
      fe_mul(f, &p, &ua, &az); fe_add(f, &s[0], &s[0], &p); fe_mul(f, &p, &us, &bz); fe_add(f, &s[0], &s[0], &p);
      fe_mul(f, &p, &ua, &azi); fe_add(f, &s[1], &s[1], &p); fe_mul(f, &p, &us, &bzi); fe_add(f, &s[1], &s[1], &p);
      fe_sub(f, &x, &az, &bz); fe_sqr(f, &x, &x);
      fe_mul(f, &p, &u4, &cz); fe_add(f, &s[2], &s[2], &p); fe_mul(f, &p, &ua, &x); fe_add(f, &s[2], &s[2], &p);
      fe_mul(f, &p, &u4, &czi); fe_add(f, &s[3], &s[3], &p);
    }
    for (int k = 0; k < 4; k++) part[4 * t + k] = s[k];
  }
  fe a0, ai, c0, ci, p;
  memset(&a0, 0, sizeof a0); memset(&ai, 0, sizeof ai); memset(&c0, 0, sizeof c0); memset(&ci, 0, sizeof ci);
  for (int t = 0; t < nt; t++) {
    fe_add(f, &a0, &a0, &part[4 * t]); fe_add(f, &ai, &ai, &part[4 * t + 1]);
    fe_add(f, &c0, &c0, &part[4 * t + 2]); fe_add(f, &ci, &ci, &part[4 * t + 3]);
  }
  free(part);
  /* the extra rows: every column they touch is an instance column except y_j's */
  fe_mul(f, &p, &u[e_off], &zm[0]);
  fe_add(f, &a0, &a0, &p); fe_add(f, &ai, &ai, &p); fe_add(f, &c0, &c0, &p); fe_add(f, &ci, &ci, &p);
  for (uint64_t j = 1; j < ni; j++) {
    const fe* u1 = &u[e_off + 2 * j - 1]; const fe* u2 = &u[e_off + 2 * j];
    fe s, d, q, y;
    fe_add(f, &s, u1, u2); fe_sub(f, &d, u1, u2); fe_dbl(f, &q, u1); fe_dbl(f, &q, &q);
    fe_sub(f, &y, &zm[j], &f->r1); fe_sqr(f, &y, &y);
    fe ta; fe_mul(f, &ta, &s, &zm[j]); fe_mul(f, &p, &d, &zm[0]); fe_add(f, &ta, &ta, &p);
    fe_add(f, &a0, &a0, &ta); fe_add(f, &ai, &ai, &ta);
    fe tc; fe_mul(f, &tc, &q, &zm[j]);
    fe_add(f, &c0, &c0, &tc); fe_add(f, &ci, &ci, &tc);
    fe_mul(f, &p, &s, &y); fe_add(f, &c0, &c0, &p);
  }
  free(u); free(zm);
  fe ab, g2, abg, at, ct, ht, zinv, aux, t1, t2;
  fe_add(f, &ab, &alpha, &beta); fe_sqr(f, &g2, &gamma); fe_mul(f, &abg, &ab, &gamma);
  fe_mul(f, &t1, &d1, &zt); fe_add(f, &at, &a0, &t1);
  fe_mul(f, &t1, &d2, &zt); fe_add(f, &ct, &c0, &t1);
  fe_inv(f, &zinv, &zt);
  fe_sqr(f, &ht, &at); fe_sub(f, &ht, &ht, &ct); fe_mul(f, &ht, &ht, &zinv);
  fe_sub(f, &t1, &c0, &ci); fe_mul(f, &aux, &g2, &t1);
  fe_sub(f, &t1, &a0, &ai); fe_mul(f, &t1, &abg, &t1); fe_add(f, &aux, &aux, &t1);
  fe adl, cdl;
  fe_mul(f, &t1, &rr, &zt); fe_add(f, &t1, &at, &t1); fe_mul(f, &adl, &gamma, &t1);         /* gamma (at + r Z) */
  cdl = aux;
  fe_mul(f, &t1, &d1, &abg); fe_mul(f, &t1, &t1, &zt); fe_add(f, &cdl, &cdl, &t1);
  fe_mul(f, &t1, &d2, &g2); fe_mul(f, &t1, &t1, &zt); fe_add(f, &cdl, &cdl, &t1);
  fe_sqr(f, &t1, &rr); fe_mul(f, &t1, &t1, &g2); fe_mul(f, &t1, &t1, &zt); fe_mul(f, &t1, &t1, &zt); fe_add(f, &cdl, &cdl, &t1);
  fe_mul(f, &t1, &rr, &abg); fe_mul(f, &t1, &t1, &zt); fe_add(f, &cdl, &cdl, &t1);
  fe_mul(f, &t2, &rr, &at); fe_dbl(f, &t2, &t2); fe_add(f, &t2, &t2, &ht);
  fe_mul(f, &t1, &g2, &zt); fe_mul(f, &t1, &t1, &t2); fe_add(f, &cdl, &cdl, &t1);
  fe ac, cc; fe_from_mont(f, &ac, &adl); fe_from_mont(f, &cc, &cdl);
  g1_jac g1, pa1, pc1; g2_jac g2g, pb2;
  key_generators(curve, c, trapdoor6 + 16, trapdoor6 + 20, &g1, &g2g);
  g1_mul(&c->fq, &pa1, &g1, ac.l, 4); g2_mul(&c->fq, &pb2, &g2g, ac.l, 4); g1_mul(&c->fq, &pc1, &g1, cc.l, 4);
  g1_aff oa, oc; g2_aff ob;
  g1_to_affine(&c->fq, &oa, &pa1); g2_to_affine(&c->fq, &ob, &pb2); g1_to_affine(&c->fq, &oc, &pc1);
  g1_write(c, proof_out, &oa); g2_write(c, proof_out + g1b, &ob); g1_write(c, proof_out + g1b + g2b, &oc);
  return 0;
}
