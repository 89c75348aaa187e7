// Host emulation harness (TEST ONLY) for the separated Montgomery arithmetic of fp.cuh / fp2.cuh and the
// point additions of ec.cuh: the device headers compiled as plain C++.  The op wrappers live in wide_ops.cuh,
// shared with the device harness dev_wide.cu; each entry point runs `count` cases (strides in wide_ops.cuh).
#include "wide_ops.cuh"
using namespace zkb;
using namespace zkb::wide;

// field 0: BN254 Fr, 1: BN254 Fq, 2: BLS12-381 Fr, 3: BLS12-381 Fq
extern "C" void emu_wide_fp(int field, int op, size_t count, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                            const uint32_t* d, uint32_t* o) {
  for (size_t i = 0; i < count; i++) {
    switch (field) {
      case 0: fp_case<Bn254Fr>(op, i, a, b, c, d, o); break;
      case 1: fp_case<Bn254Fq>(op, i, a, b, c, d, o); break;
      case 2: fp_case<Bls381Fr>(op, i, a, b, c, d, o); break;
      case 3: fp_case<Bls381Fq>(op, i, a, b, c, d, o); break;
    }
  }
}
// curve 0: BN254 Fq2, 1: BLS12-381 Fq2
extern "C" void emu_wide_fp2(int curve, int op, size_t count, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                             const uint32_t* d, uint32_t* o) {
  for (size_t i = 0; i < count; i++) {
    if (curve == 0) fp2_case<Bn254Fq>(op, i, a, b, c, d, o);
    else fp2_case<Bls381Fq>(op, i, a, b, c, d, o);
  }
}
// curve 0: BN254, 1: BLS12-381; group 1: G1, 2: G2
extern "C" void emu_wide_ec(int curve, int group, int op, size_t count, const uint32_t* a, const uint32_t* b, uint32_t* o) {
  for (size_t i = 0; i < count; i++) {
    if (curve == 0) {
      if (group == 1) ec_case<Fp<Bn254Fq>, 1, Bn254Fq>(op, i, a, b, o);
      else ec_case<Fp2<Bn254Fq>, 2, Bn254Fq>(op, i, a, b, o);
    } else {
      if (group == 1) ec_case<Fp<Bls381Fq>, 1, Bls381Fq>(op, i, a, b, o);
      else ec_case<Fp2<Bls381Fq>, 2, Bls381Fq>(op, i, a, b, o);
    }
  }
}
