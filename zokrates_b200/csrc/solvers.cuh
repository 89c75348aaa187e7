// Solver directives on the device: one thread per directive of a dependency level and input set.
//
// Restates `Interpreter::execute_solver` (/root/reference/zokrates_interpreter/src/lib.rs:249-307) and the out-of-range
// `Bits` path (`try_solve_with_out_of_range_bits`, :140-165, taken when `should_try_out_of_range` is set and the width
// covers the field, :94-101) for the simple solvers; `Zir` folded functions and the embed gadgets are front-end code and
// have no device path (SOLVER_UNSUPPORTED).  Inputs are QuadCombs (left * right of two linear combinations, evaluated
// like `evaluate_quad`, :366-378); outputs are written straight into the assignment vector (Montgomery form).
// A batch of K input sets uses witness_level_body's layout (ntt.cuh): z[col * K + k], thread t runs directive lo + t / K for
// set t % K; `flags` applies to the whole batch.
#pragma once
#include "fp.cuh"
#include "prog.cuh"

namespace zkb {

template <class Fr>
ZKB_HDN inline Fr lc_dot(const uint32_t* ptr, const uint32_t* col, const Fr* val, const Fr* z, uint32_t K, uint32_t k, uint32_t q) {
  Fr acc = Fr::zero();
  for (uint32_t e = ptr[q]; e < ptr[q + 1]; e++) acc = Fr::add(acc, Fr::mul(val[e], z[(size_t)col[e] * K + k]));
  return acc;
}

// 256-bit helpers on canonical little-endian limbs (plain C: the same code runs in the CPU test build)
ZKB_HD bool u256_geq(const uint32_t* a, const uint32_t* b) {
  for (int i = 7; i >= 0; i--) if (a[i] != b[i]) return a[i] > b[i];
  return true;
}
ZKB_HD void u256_sub(uint32_t* a, const uint32_t* b) {
  uint64_t borrow = 0;
  for (int i = 0; i < 8; i++) {
    const uint64_t t = (uint64_t)a[i] - b[i] - borrow;
    a[i] = (uint32_t)t;
    borrow = (t >> 63) & 1u;
  }
}

static constexpr uint32_t SOLVE_TRY_OUT_OF_RANGE = 1u;   // flags: Interpreter::try_out_of_range()

template <class Fr>
ZKB_HDN inline void solver_body(const uint32_t* kind, const uint32_t* arg, const uint32_t* in_ptr, const uint32_t* out_ptr,
                                const uint32_t* out_cols, const uint32_t* lc_ptr, const uint32_t* lc_col, const Fr* lc_val, Fr* z,
                                const uint32_t* dirs, uint32_t lo, uint32_t hi, uint32_t K, uint32_t flags, uint32_t t) {
  const uint32_t i = lo + t / K, kz = t % K;
  if (i >= hi) return;
  const uint32_t d = dirs[i];
  const uint32_t n_in = in_ptr[d + 1] - in_ptr[d];
  Fr x[3];
  for (uint32_t j = 0; j < 3; j++) {
    if (j < n_in) {
      const uint32_t q = in_ptr[d] + j;
      x[j] = Fr::mul(lc_dot<Fr>(lc_ptr, lc_col, lc_val, z, K, kz, 2 * q), lc_dot<Fr>(lc_ptr, lc_col, lc_val, z, K, kz, 2 * q + 1));
    } else {
      x[j] = Fr::zero();
    }
  }
  const uint32_t* oc = out_cols + out_ptr[d];
  const uint32_t n_out = out_ptr[d + 1] - out_ptr[d];
  const Fr one = Fr::one();
  switch (kind[d]) {
    case SOLVER_CONDITION_EQ: {          // x == 0 ? [0, 1] : [1, 1 / x]
      if (n_out < 2) return;
      if (x[0].is_zero()) { z[(size_t)oc[0] * K + kz] = Fr::zero(); z[(size_t)oc[1] * K + kz] = one; }
      else { z[(size_t)oc[0] * K + kz] = one; z[(size_t)oc[1] * K + kz] = Fr::inv(x[0]); }
      return;
    }
    case SOLVER_BITS: {                  // big-endian bits, exactly `w` of them (the low w bits, zero-padded on the left)
      const uint32_t w = arg[d];
      Fr c = Fr::from_mont(x[0]);
      uint32_t v[8];
      for (int k = 0; k < 8; k++) v[k] = c.v[k];
      if ((flags & SOLVE_TRY_OUT_OF_RANGE) && w >= (uint32_t)Fr::Params::BITS) {
        // candidate = x + r; used when it still fits the field's bit length (a second, non-canonical decomposition)
        uint32_t cand[8];
        uint64_t carry = 0;
        for (int k = 0; k < 8; k++) { const uint64_t s = (uint64_t)v[k] + Fr::Params::mod(k) + carry; cand[k] = (uint32_t)s; carry = s >> 32; }
        bool fits = carry == 0;
        for (uint32_t b = (uint32_t)Fr::Params::BITS; b < 256 && fits; b++) fits = !((cand[b >> 5] >> (b & 31)) & 1u);
        if (fits) for (int k = 0; k < 8; k++) v[k] = cand[k];
      }
      for (uint32_t k = 0; k < w && k < n_out; k++) {
        const uint32_t b = w - 1 - k;
        const uint32_t bit = b < 256 ? (v[b >> 5] >> (b & 31)) & 1u : 0u;
        z[(size_t)oc[k] * K + kz] = bit ? one : Fr::zero();
      }
      return;
    }
    case SOLVER_DIV:                     // x / y, 1 when y == 0 (checked_div(..).unwrap_or_else(T::one))
      if (n_out) z[(size_t)oc[0] * K + kz] = x[1].is_zero() ? one : Fr::mul(x[0], Fr::inv(x[1]));
      return;
    case SOLVER_XOR:                     // x + y - 2 x y
      if (n_out) { Fr xy = Fr::mul(x[0], x[1]); z[(size_t)oc[0] * K + kz] = Fr::sub(Fr::add(x[0], x[1]), Fr::dbl(xy)); }
      return;
    case SOLVER_OR:                      // x + y - x y
      if (n_out) z[(size_t)oc[0] * K + kz] = Fr::sub(Fr::add(x[0], x[1]), Fr::mul(x[0], x[1]));
      return;
    case SOLVER_SHA_AXXA: {              // b c - (2 b c - b - c) a
      if (!n_out) return;
      Fr bc = Fr::mul(x[1], x[2]);
      Fr u = Fr::sub(Fr::sub(Fr::dbl(bc), x[1]), x[2]);
      z[(size_t)oc[0] * K + kz] = Fr::sub(bc, Fr::mul(u, x[0]));
      return;
    }
    case SOLVER_SHA_CH:                  // a (b - c) + c
      if (n_out) z[(size_t)oc[0] * K + kz] = Fr::add(Fr::mul(x[0], Fr::sub(x[1], x[2])), x[2]);
      return;
    case SOLVER_EUCLIDEAN_DIV: {         // integers: q = n / d (0 when d == 0), r = n - d q
      if (n_out < 2) return;
      Fr nc = Fr::from_mont(x[0]), dc = Fr::from_mont(x[1]);
      uint32_t q[8], rem[8];
      for (int k = 0; k < 8; k++) { q[k] = 0; rem[k] = 0; }
      if (dc.is_zero()) {
        for (int k = 0; k < 8; k++) rem[k] = nc.v[k];
      } else {
        for (int b = 255; b >= 0; b--) {   // shift-subtract; rem < d < 2^255 so the shift cannot overflow
          for (int k = 7; k > 0; k--) rem[k] = (rem[k] << 1) | (rem[k - 1] >> 31);
          rem[0] = (rem[0] << 1) | ((nc.v[b >> 5] >> (b & 31)) & 1u);
          if (u256_geq(rem, dc.v)) { u256_sub(rem, dc.v); q[b >> 5] |= 1u << (b & 31); }
        }
      }
      Fr qf, rf;
      for (int k = 0; k < 8; k++) { qf.v[k] = q[k]; rf.v[k] = rem[k]; }
      z[(size_t)oc[0] * K + kz] = Fr::to_mont(qf);
      z[(size_t)oc[1] * K + kz] = Fr::to_mont(rf);
      return;
    }
    default: return;                     // SOLVER_UNSUPPORTED: refused before the launch
  }
}

}  // namespace zkb
