// Host emulation harness (TEST ONLY) for BLS12-377: the op wrappers of wide_ops.cuh over Bls377Fr / Bls377Fq, its
// Fq2 = Fq[u]/(u^2 + 5) and G1 / G2, compiled as plain C++.  Same entry-point arguments as emu_wide.cpp; the field / curve
// argument selects within BLS12-377 only (field 0: Fr, 1: Fq; curve ignored).  Fq2 ops beyond wide_ops.cuh's 0-2:
// 3 inv; and the host tail of the prover (fp64.cuh, Fp2T over Fp64, every product reduced): 4 mul_v, 5 sqr_v, 6 inv.
#include <string.h>

#include "fp64.cuh"
#include "wide_ops.cuh"
using namespace zkb;
using namespace zkb::wide;

extern "C" void emu_wide_fp(int field, int op, size_t count, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                            const uint32_t* d, uint32_t* o) {
  for (size_t i = 0; i < count; i++) {
    if (field == 0) fp_case<Bls377Fr>(op, i, a, b, c, d, o);
    else fp_case<Bls377Fq>(op, i, a, b, c, d, o);
  }
}
typedef Fp2T<Fp64<Bls377Fq>> H2;
static H2 ld_h2(const uint32_t* a) { H2 x; memcpy(x.c0.v, a, 48); memcpy(x.c1.v, a + 12, 48); return x; }
static void st_h2(const H2& x, uint32_t* o) { memcpy(o, x.c0.v, 48); memcpy(o + 12, x.c1.v, 48); }

extern "C" void emu_wide_fp2(int, int op, size_t count, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                             const uint32_t* d, uint32_t* o) {
  const size_t s = 24;
  for (size_t i = 0; i < count; i++) {
    const uint32_t* ai = a + s * i;
    uint32_t* oi = o + s * i;
    switch (op) {
      case 3: st2<Bls377Fq>(Fp2<Bls377Fq>::inv(ld2<Bls377Fq>(ai)), oi); break;
      case 4: st_h2(H2::mul_v(ld_h2(ai), ld_h2(b + s * i)), oi); break;
      case 5: st_h2(H2::sqr_v(ld_h2(ai)), oi); break;
      case 6: st_h2(H2::inv(ld_h2(ai)), oi); break;
      default: fp2_case<Bls377Fq>(op, i, a, b, c, d, o);
    }
  }
}
// group 1: G1, 2: G2
extern "C" void emu_wide_ec(int, int group, int op, size_t count, const uint32_t* a, const uint32_t* b, uint32_t* o) {
  for (size_t i = 0; i < count; i++) {
    if (group == 1) ec_case<Fp<Bls377Fq>, 1, Bls377Fq>(op, i, a, b, o);
    else ec_case<Fp2<Bls377Fq>, 2, Bls377Fq>(op, i, a, b, o);
  }
}
