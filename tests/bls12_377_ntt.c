/* Radix-2 NTT over the BLS12-377 scalar field (TEST ONLY): the independent answer for zkb_ntt on this curve at sizes where
 * the Python domain of oracle/ark.py is too slow.  A plain restatement of ark-poly's Radix2EvaluationDomain as
 * oracle/ark.py writes it (bit reversal, iterative DIT; inverse = transform with w^-1 times 1/n; coset = scaling by g^i
 * before / by g^-i after), on 4 x 64-bit Montgomery limbs with unsigned __int128, written apart from the product's fields.
 * Every constant that depends on the domain (w, 1/n, g, 1/g) is passed in canonical form by the caller.
 * Build: gcc -O2 -fopenmp -shared -fPIC.  Data: n elements of 4 little-endian uint64 limbs, canonical, in place. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef unsigned __int128 u128;
typedef struct { uint64_t v[4]; } fe;

static const uint64_t MOD[4] = {0x0a11800000000001ull, 0x59aa76fed0000001ull, 0x60b44d1e5c37b001ull, 0x12ab655e9a2ca556ull};
static uint64_t NINV;   /* -r^-1 mod 2^64 */
static fe R2;           /* 2^512 mod r */

static int geq_mod(const uint64_t* a) {
  for (int i = 3; i >= 0; i--) {
    if (a[i] > MOD[i]) return 1;
    if (a[i] < MOD[i]) return 0;
  }
  return 1;
}
static void sub_mod_inplace(uint64_t* a) {
  uint64_t b = 0;
  for (int i = 0; i < 4; i++) {
    u128 d = (u128)a[i] - MOD[i] - b;
    a[i] = (uint64_t)d;
    b = (uint64_t)(d >> 64) & 1;
  }
}
static fe add(fe a, fe b) {
  fe r;
  uint64_t c = 0;
  for (int i = 0; i < 4; i++) {
    u128 s = (u128)a.v[i] + b.v[i] + c;
    r.v[i] = (uint64_t)s;
    c = (uint64_t)(s >> 64);
  }
  if (c || geq_mod(r.v)) sub_mod_inplace(r.v);
  return r;
}
static fe sub(fe a, fe b) {
  fe r;
  uint64_t br = 0;
  for (int i = 0; i < 4; i++) {
    u128 d = (u128)a.v[i] - b.v[i] - br;
    r.v[i] = (uint64_t)d;
    br = (uint64_t)(d >> 64) & 1;
  }
  if (br) {
    uint64_t c = 0;
    for (int i = 0; i < 4; i++) {
      u128 s = (u128)r.v[i] + MOD[i] + c;
      r.v[i] = (uint64_t)s;
      c = (uint64_t)(s >> 64);
    }
  }
  return r;
}
/* Montgomery product a b 2^-256 mod r (CIOS, r < 2^253 so no extra word overflows) */
static fe mul(fe a, fe b) {
  uint64_t t[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; i++) {
    uint64_t c = 0;
    for (int j = 0; j < 4; j++) {
      u128 s = (u128)a.v[j] * b.v[i] + t[j] + c;
      t[j] = (uint64_t)s;
      c = (uint64_t)(s >> 64);
    }
    u128 s = (u128)t[4] + c;
    t[4] = (uint64_t)s;
    t[5] = (uint64_t)(s >> 64);
    uint64_t m = t[0] * NINV;
    s = (u128)m * MOD[0] + t[0];
    c = (uint64_t)(s >> 64);
    for (int j = 1; j < 4; j++) {
      s = (u128)m * MOD[j] + t[j] + c;
      t[j - 1] = (uint64_t)s;
      c = (uint64_t)(s >> 64);
    }
    s = (u128)t[4] + c;
    t[3] = (uint64_t)s;
    t[4] = t[5] + (uint64_t)(s >> 64);
  }
  fe r;
  memcpy(r.v, t, 32);
  if (t[4] || geq_mod(r.v)) sub_mod_inplace(r.v);
  return r;
}
static void init(void) {
  uint64_t x = 1;                                  /* r^-1 mod 2^64 by Newton */
  for (int i = 0; i < 7; i++) x *= 2 - MOD[0] * x;
  NINV = (uint64_t)0 - x;
  fe one = {{1, 0, 0, 0}};
  R2 = one;
  for (int i = 0; i < 512; i++) R2 = add(R2, R2);
}
static fe to_m(const uint64_t* a) { fe x; memcpy(x.v, a, 32); return mul(x, R2); }
static void from_m(fe a, uint64_t* out) { fe one = {{1, 0, 0, 0}}; fe x = mul(a, one); memcpy(out, x.v, 32); }

static void fft(fe* a, uint64_t n, int log_n, fe w) {
  for (uint64_t i = 1, j = 0; i < n; i++) {
    uint64_t bit = n >> 1;
    for (; j & bit; bit >>= 1) j ^= bit;
    j |= bit;
    if (i < j) { fe t = a[i]; a[i] = a[j]; a[j] = t; }
  }
  fe* tw = (fe*)malloc(sizeof(fe) * (n / 2 + 1));   /* w^k, k < n/2 */
  tw[0] = to_m((const uint64_t[4]){1, 0, 0, 0});
  for (uint64_t k = 1; k < n / 2; k++) tw[k] = mul(tw[k - 1], w);
  for (int st = 1; st <= log_n; st++) {
    const uint64_t len = (uint64_t)1 << st, half = len / 2, stride = n / len;
#pragma omp parallel for schedule(static)
    for (int64_t jj = 0; jj < (int64_t)(n / 2); jj++) {
      const uint64_t j = (uint64_t)jj, s = (j / half) * len, k = j % half;
      fe u = a[s + k], v = mul(a[s + k + half], tw[k * stride]);
      a[s + k] = add(u, v);
      a[s + k + half] = sub(u, v);
    }
  }
  free(tw);
}

/* w: the domain's root for this direction (w or w^-1); scale: 1/n for the inverse, else 1; g_pre / g_post: the coset
 * factor applied before / after the transform (g, g^-1, or 0 for none) */
void ref_ntt377(uint64_t* data, uint32_t log_n, const uint64_t* w_c, const uint64_t* scale_c, const uint64_t* g_pre_c,
                const uint64_t* g_post_c) {
  if (!NINV) init();
  const uint64_t n = (uint64_t)1 << log_n;
  fe* a = (fe*)malloc(sizeof(fe) * n);
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < (int64_t)n; i++) a[i] = to_m(data + 4 * i);
  fe one = to_m((const uint64_t[4]){1, 0, 0, 0});
  if (g_pre_c) {   /* x_i g^i: sequential powers (independent of the transform) */
    fe g = to_m(g_pre_c), gp = one;
    for (uint64_t i = 0; i < n; i++) { a[i] = mul(a[i], gp); gp = mul(gp, g); }
  }
  fft(a, n, (int)log_n, to_m(w_c));
  fe sc = to_m(scale_c);
  if (g_post_c) {
    fe g = to_m(g_post_c), gp = sc;
    for (uint64_t i = 0; i < n; i++) { a[i] = mul(a[i], gp); gp = mul(gp, g); }
  } else {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) a[i] = mul(a[i], sc);
  }
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < (int64_t)n; i++) from_m(a[i], data + 4 * i);
  free(a);
}
