// C ABI of libzkb200.so (include/zkb.h).  No exception or CUDA type crosses this boundary.
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include "zkb.h"
#include "engine_base.cuh"
#include "probe.cuh"
#if defined(ZKB_EMU)  // the host-emulation test build is a single translation unit
#include "engine_bn254.cu"
#include "engine_bls12_381.cu"
#include "engine_bls12_377.cu"
#endif

using namespace zkb;

struct zkb_ctx {
  int curve = 0;
  int device = 0;
  Stream st;
  std::unique_ptr<EngineBase> eng;
  uint64_t launches0 = 0;
  // The reference's static `Backend::generate_proof` is thread-safe; here the engine keeps per-context scratch (sort plans,
  // bucket sets, timers), so every entry point holds this lock for its whole duration: concurrent callers on one context
  // are serialised, never interleaved.  (begin/end pairs are additionally guarded by the caller, see _lib.Context.lock.)
  std::recursive_mutex mu;
};

static thread_local std::string g_err;

template <class Fn>
static int32_t guard(zkb_ctx* ctx, Fn fn) {
  try {
    if (!ctx || !ctx->eng) throw Error(ZKB_E_ARG, "null context");
    std::lock_guard<std::recursive_mutex> lock(ctx->mu);
    device_select(ctx->device);
    fn();
    return ZKB_OK;
  } catch (const Error& e) {
    g_err = e.what();
    clear_device_error();
    return e.code;
  } catch (const std::bad_alloc&) {
    g_err = "host allocation failed";
    return ZKB_E_OOM;
  } catch (const std::exception& e) {
    g_err = e.what();
    return ZKB_E_INTERNAL;
  } catch (...) {
    g_err = "unknown error";
    return ZKB_E_INTERNAL;
  }
}

extern "C" {

const char* zkb_last_error(void) { return g_err.c_str(); }
uint32_t zkb_abi_version(void) { return 1; }

int32_t zkb_device_count(void) {
  const char* why = "";
  const int n = device_count(&why);
  if (n < 0) g_err = std::string("cudaGetDeviceCount: ") + why;
  return n;
}

int32_t zkb_ctx_create(int32_t curve, int32_t device, zkb_ctx** out) {
  if (!out) { g_err = "out is null"; return ZKB_E_ARG; }
  *out = nullptr;
  try {
    if (curve != ZKB_CURVE_BN128 && curve != ZKB_CURVE_BLS12_381 && curve != ZKB_CURVE_BLS12_377)
      throw Error(ZKB_E_ARG, "unknown curve id");
    std::unique_ptr<zkb_ctx> c(new zkb_ctx());
    c->curve = curve;
    c->device = device;
    const char* why = "device count is 0";
    const int n = device_count(&why);
    if (n <= 0) throw Error(ZKB_E_CUDA, std::string("no usable CUDA device (libzkb200 has no CPU fallback): ") + why);
    if (device < 0 || device >= n) throw Error(ZKB_E_ARG, "device index out of range");
    device_select(device);
    c->st = stream_create();
    c->eng.reset(curve == ZKB_CURVE_BN128       ? make_engine_bn254(c->st)
                 : curve == ZKB_CURVE_BLS12_381 ? make_engine_bls12_381(c->st)
                                                : make_engine_bls12_377(c->st));
    c->launches0 = launch_counter();
    *out = c.release();
    return ZKB_OK;
  } catch (const Error& e) {
    g_err = e.what();
    return e.code;
  } catch (const std::exception& e) {
    g_err = e.what();
    return ZKB_E_INTERNAL;
  }
}

void zkb_ctx_destroy(zkb_ctx* ctx) {
  if (!ctx) return;
  device_drain(ctx->device, ctx->st);
  ctx->eng.reset();
  stream_destroy(ctx->st);
  delete ctx;
}

int32_t zkb_curve_sizes(int32_t curve, uint64_t out[4]) {
  if (!out) { g_err = "out is null"; return ZKB_E_ARG; }
  if (curve == ZKB_CURVE_BN128) {
    out[0] = 32; out[1] = 32; out[2] = 256; out[3] = partial_bytes_bn254();
  } else if (curve == ZKB_CURVE_BLS12_381) {
    out[0] = 32; out[1] = 48; out[2] = 384; out[3] = partial_bytes_bls12_381();
  } else if (curve == ZKB_CURVE_BLS12_377) {
    out[0] = 32; out[1] = 48; out[2] = 384; out[3] = partial_bytes_bls12_377();
  } else {
    g_err = "unknown curve id";
    return ZKB_E_ARG;
  }
  return ZKB_OK;
}

int32_t zkb_pk_load(zkb_ctx* ctx, const uint8_t* pk, size_t len, uint32_t rank, uint32_t world, uint64_t* h) {
  return guard(ctx, [&] {
    if (!pk || !h) throw Error(ZKB_E_ARG, "null argument");
    *h = ctx->eng->pk_load(pk, len, rank, world);
  });
}
int32_t zkb_pk_info(zkb_ctx* ctx, uint64_t h, uint64_t out[4]) {
  return guard(ctx, [&] { if (!out) throw Error(ZKB_E_ARG, "null"); ctx->eng->pk_info(h, out); });
}
int32_t zkb_pk_table_info(zkb_ctx* ctx, uint64_t h, uint64_t out[8]) {
  return guard(ctx, [&] { if (!out) throw Error(ZKB_E_ARG, "null"); ctx->eng->pk_table_info(h, out); });
}
int32_t zkb_ctx_set_option(zkb_ctx* ctx, int32_t opt, int64_t value) {
  return guard(ctx, [&] {
    Options& o = ctx->eng->opts;
    switch (opt) {
      case ZKB_OPT_TABLES: if (value < 0 || value > 2) throw Error(ZKB_E_ARG, "ZKB_OPT_TABLES: 0, 1 or 2"); o.tables = value; break;
      case ZKB_OPT_TABLE_MIN_LOG: if (value < 0 || value > 40) throw Error(ZKB_E_ARG, "ZKB_OPT_TABLE_MIN_LOG"); o.table_min_log = value; break;
      case ZKB_OPT_TABLE_C: if (value < 0 || value > 22) throw Error(ZKB_E_ARG, "ZKB_OPT_TABLE_C: 0 or 4..22"); o.table_c = value; break;
      case ZKB_OPT_Z_MODE: if (value < 0 || value > 2) throw Error(ZKB_E_ARG, "ZKB_OPT_Z_MODE: 0, 1 or 2"); o.z_mode = value; break;
      case ZKB_OPT_NTT_TILE_MIN: if (value < 0 || value > 64) throw Error(ZKB_E_ARG, "ZKB_OPT_NTT_TILE_MIN"); o.ntt_tile_min = value; break;
      case ZKB_OPT_NTT_MAX_S: if (value < 1 || value > 10) throw Error(ZKB_E_ARG, "ZKB_OPT_NTT_MAX_S: 1..10"); o.ntt_max_s = value; break;
      case ZKB_OPT_BATCH_AFFINE: if (value < 0 || value > 8) throw Error(ZKB_E_ARG, "ZKB_OPT_BATCH_AFFINE: 0..8"); o.batch_affine = value; break;
      case ZKB_OPT_BATCH_AFFINE_MIN_LOG: if (value < 0 || value > 40) throw Error(ZKB_E_ARG, "ZKB_OPT_BATCH_AFFINE_MIN_LOG"); o.batch_affine_min_log = value; break;
      case ZKB_OPT_PLAN_STREAM: if (value < 0 || value > 1) throw Error(ZKB_E_ARG, "ZKB_OPT_PLAN_STREAM: 0 or 1"); o.plan_stream = value; break;
      case ZKB_OPT_CHUNK_TARGET: if (value < 1000 || value > 100000000) throw Error(ZKB_E_ARG, "ZKB_OPT_CHUNK_TARGET: 1e3 .. 1e8"); o.chunk_target = value; break;
      case ZKB_OPT_CHAIN_SHARE: if (value < -1 || value > 500) throw Error(ZKB_E_ARG, "ZKB_OPT_CHAIN_SHARE: -1, 0 or 1..500"); o.chain_share = value; break;
      case ZKB_OPT_NTT_KERNEL: if (value != 1 && value != 2) throw Error(ZKB_E_ARG, "ZKB_OPT_NTT_KERNEL: 1 or 2"); o.ntt_kernel = value; break;
      case ZKB_OPT_PK_CACHE: if (value < 0 || value > 1) throw Error(ZKB_E_ARG, "ZKB_OPT_PK_CACHE: 0 or 1"); o.pk_cache = value; break;
      case ZKB_OPT_BITSUM_RADIX: if (value != 2 && value != 8) throw Error(ZKB_E_ARG, "ZKB_OPT_BITSUM_RADIX: 2 or 8"); o.bitsum_radix = value; break;
      case ZKB_OPT_BATCH_PASS_MAX: if (value < 0 || value > 0xFFFFFFFFll) throw Error(ZKB_E_ARG, "ZKB_OPT_BATCH_PASS_MAX: 0 or a proof count"); o.batch_pass_max = value; break;
      default: throw Error(ZKB_E_ARG, "unknown option");
    }
  });
}
int32_t zkb_pk_free(zkb_ctx* ctx, uint64_t h) { return guard(ctx, [&] { ctx->eng->pk_free(h); }); }

int32_t zkb_r1cs_load(zkb_ctx* ctx, uint64_t N, uint64_t ni, uint64_t nw, const uint64_t* a_rowptr, const uint32_t* a_col,
                      const uint64_t* a_val, const uint64_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val,
                      const uint64_t* c_rowptr, const uint32_t* c_col, const uint64_t* c_val, uint64_t* h) {
  return guard(ctx, [&] {
    if (!a_rowptr || !b_rowptr || !c_rowptr || !h) throw Error(ZKB_E_ARG, "null argument");
    const uint64_t* rp[3] = {a_rowptr, b_rowptr, c_rowptr};
    const uint32_t* cl[3] = {a_col, b_col, c_col};
    const uint64_t* vl[3] = {a_val, b_val, c_val};
    *h = ctx->eng->r1cs_load(N, ni, nw, rp, cl, vl);
  });
}
int32_t zkb_r1cs_free(zkb_ctx* ctx, uint64_t h) { return guard(ctx, [&] { ctx->eng->r1cs_free(h); }); }

int32_t zkb_r1cs_set_assignment(zkb_ctx* ctx, uint64_t h, const uint64_t* z) {
  return guard(ctx, [&] { if (!z) throw Error(ZKB_E_ARG, "null"); ctx->eng->set_assignment(h, z); });
}

static void check_proof_cap(zkb_ctx* ctx, size_t cap) {
  uint64_t sz[4];
  ctx->eng->sizes(sz);
  if (cap < sz[2]) throw Error(ZKB_E_ARG, "proof_out too small");
}

static void prove_common(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, const uint64_t* z, const uint64_t* r, const uint64_t* s,
                         uint8_t* proof_out, size_t cap) {
  if (!r || !s || !proof_out) throw Error(ZKB_E_ARG, "null argument");
  check_proof_cap(ctx, cap);
  ctx->eng->prove_full(pk, r1cs, z, r, s, proof_out);
}

int32_t zkb_groth16_prove(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, const uint64_t* z, const uint64_t* r, const uint64_t* s,
                          uint8_t* proof_out, size_t cap) {
  return guard(ctx, [&] {
    if (!z) throw Error(ZKB_E_ARG, "null assignment");
    prove_common(ctx, pk, r1cs, z, r, s, proof_out, cap);
  });
}
int32_t zkb_groth16_prove_batch(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, uint32_t count, const uint64_t* z, const uint64_t* r,
                                const uint64_t* s, uint8_t* proofs_out, size_t cap) {
  return guard(ctx, [&] {
    if (count == 0) throw Error(ZKB_E_ARG, "empty batch");
    if (!z || !r || !s || !proofs_out) throw Error(ZKB_E_ARG, "null argument");
    uint64_t sz[4];
    ctx->eng->sizes(sz);
    if (cap / count < sz[2]) throw Error(ZKB_E_ARG, "proofs_out too small");
    ctx->eng->prove_batch(pk, r1cs, count, z, r, s, proofs_out);
  });
}
int32_t zkb_groth16_prove_resident(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, const uint64_t* r, const uint64_t* s,
                                   uint8_t* proof_out, size_t cap) {
  return guard(ctx, [&] { prove_common(ctx, pk, r1cs, nullptr, r, s, proof_out, cap); });
}
int32_t zkb_groth16_prove_partial(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, const uint64_t* z, uint8_t* partial_out,
                                  size_t cap) {
  return guard(ctx, [&] {
    uint64_t sz[4];
    ctx->eng->sizes(sz);
    if (!partial_out || cap < sz[3]) throw Error(ZKB_E_ARG, "partial_out too small");
    ctx->eng->prove_partial(pk, r1cs, z, partial_out);
  });
}
int32_t zkb_groth16_prove_begin(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, const uint64_t* z, uint32_t chain_mask,
                                void* chain_dev_ptrs[3], uint64_t* chain_bytes) {
  return guard(ctx, [&] {
    if (!chain_dev_ptrs || !chain_bytes) throw Error(ZKB_E_ARG, "null argument");
    ctx->eng->prove_begin(pk, r1cs, z, chain_mask, chain_dev_ptrs, chain_bytes);
  });
}
int32_t zkb_groth16_prove_end(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, uint8_t* partial_out, size_t cap) {
  return guard(ctx, [&] {
    uint64_t sz[4];
    ctx->eng->sizes(sz);
    if (!partial_out || cap < sz[3]) throw Error(ZKB_E_ARG, "partial_out too small");
    ctx->eng->prove_end(pk, r1cs, partial_out);
  });
}
int32_t zkb_groth16_prove_begin_async(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, const uint64_t* z, uint32_t chain_mask,
                                      void* chain_dev_ptrs[3], uint64_t* chain_bytes, uint64_t* ticket) {
  return guard(ctx, [&] {
    if (!chain_dev_ptrs || !chain_bytes || !ticket) throw Error(ZKB_E_ARG, "null argument");
    *ticket = ctx->eng->prove_begin_async(pk, r1cs, z, chain_mask, chain_dev_ptrs, chain_bytes);
  });
}
int32_t zkb_groth16_prove_chains_to_stream(zkb_ctx* ctx, uint64_t ticket, void* cuda_stream) {
  return guard(ctx, [&] { ctx->eng->prove_chains_to_stream(ticket, cuda_stream); });
}
int32_t zkb_groth16_prove_stream_to_finish(zkb_ctx* ctx, uint64_t ticket, void* cuda_stream) {
  return guard(ctx, [&] { ctx->eng->prove_stream_to_finish(ticket, cuda_stream); });
}
int32_t zkb_groth16_prove_end_async(zkb_ctx* ctx, uint64_t ticket) {
  return guard(ctx, [&] { ctx->eng->prove_end_async(ticket); });
}
int32_t zkb_groth16_prove_submit(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, const uint64_t* z, const uint64_t* r, const uint64_t* s,
                                 uint64_t* ticket) {
  return guard(ctx, [&] {
    if (!ticket || (!r) != (!s)) throw Error(ZKB_E_ARG, "null argument");
    *ticket = ctx->eng->prove_submit(pk, r1cs, z, r, s);
  });
}
int32_t zkb_groth16_prove_collect(zkb_ctx* ctx, uint64_t ticket, uint8_t* proof_out, size_t cap) {
  return guard(ctx, [&] {
    if (!proof_out) throw Error(ZKB_E_ARG, "null argument");
    check_proof_cap(ctx, cap);
    ctx->eng->prove_collect(ticket, proof_out);
  });
}
int32_t zkb_groth16_prove_collect_partial(zkb_ctx* ctx, uint64_t ticket, uint8_t* partial_out, size_t cap) {
  return guard(ctx, [&] {
    uint64_t sz[4];
    ctx->eng->sizes(sz);
    if (!partial_out || cap < sz[3]) throw Error(ZKB_E_ARG, "partial_out too small");
    ctx->eng->prove_collect_partial(ticket, partial_out);
  });
}
int32_t zkb_groth16_finalize_prepare(zkb_ctx* ctx, uint64_t pk, const uint64_t* r, const uint64_t* s) {
  return guard(ctx, [&] {
    if (!r || !s) throw Error(ZKB_E_ARG, "null argument");
    ctx->eng->finalize_prepare(pk, r, s);
  });
}
int32_t zkb_groth16_finalize(zkb_ctx* ctx, uint64_t pk, const uint8_t* partials, uint32_t world, const uint64_t* r,
                             const uint64_t* s, uint8_t* proof_out, size_t cap) {
  return guard(ctx, [&] {
    if (!partials || !r || !s || !proof_out) throw Error(ZKB_E_ARG, "null argument");
    check_proof_cap(ctx, cap);
    ctx->eng->timings.clear();
    ctx->eng->finalize(pk, partials, world, r, s, proof_out);
  });
}

int32_t zkb_msm_g1(zkb_ctx* ctx, const uint8_t* points, const uint64_t* scalars, uint64_t n, uint8_t* out) {
  return guard(ctx, [&] {
    if (!out || (n && (!points || !scalars))) throw Error(ZKB_E_ARG, "null argument");
    ctx->eng->msm(1, points, scalars, n, out);
  });
}
int32_t zkb_msm_g2(zkb_ctx* ctx, const uint8_t* points, const uint64_t* scalars, uint64_t n, uint8_t* out) {
  return guard(ctx, [&] {
    if (!out || (n && (!points || !scalars))) throw Error(ZKB_E_ARG, "null argument");
    ctx->eng->msm(2, points, scalars, n, out);
  });
}
int32_t zkb_ntt(zkb_ctx* ctx, uint64_t* data, uint32_t log_n, int32_t inverse, int32_t coset) {
  return guard(ctx, [&] { if (!data) throw Error(ZKB_E_ARG, "null"); ctx->eng->ntt(data, log_n, inverse, coset); });
}
int32_t zkb_witness_map(zkb_ctx* ctx, uint64_t r1cs, const uint64_t* z, uint64_t* h_out, uint64_t cap) {
  return guard(ctx, [&] { if (!z || !h_out) throw Error(ZKB_E_ARG, "null"); ctx->eng->witness_map(r1cs, z, h_out, cap); });
}
int32_t zkb_r1cs_check(zkb_ctx* ctx, uint64_t r1cs, const uint64_t* z, uint64_t* first_unsatisfied) {
  return guard(ctx, [&] {
    uint64_t f = ctx->eng->witness_eval(r1cs, const_cast<uint64_t*>(z), 0, nullptr, nullptr, nullptr);
    if (first_unsatisfied) *first_unsatisfied = f;
    if (f != ~0ull) throw Error(ZKB_E_UNSAT, "constraint " + std::to_string(f) + " is not satisfied");
  });
}
int32_t zkb_witness_eval(zkb_ctx* ctx, uint64_t r1cs, uint64_t* z_inout, uint32_t n_levels, const uint32_t* level_ptr,
                         const uint32_t* rows, const uint32_t* out_var, uint64_t* first_unsatisfied) {
  return guard(ctx, [&] {
    if (!z_inout || !n_levels) throw Error(ZKB_E_ARG, "null argument");
    uint64_t f = ctx->eng->witness_eval(r1cs, z_inout, n_levels, level_ptr, rows, out_var);
    if (first_unsatisfied) *first_unsatisfied = f;
    if (f != ~0ull) throw Error(ZKB_E_UNSAT, "constraint " + std::to_string(f) + " is not satisfied");
  });
}
int32_t zkb_prog_load(zkb_ctx* ctx, const uint8_t* out_bytes, size_t len, uint64_t* h) {
  return guard(ctx, [&] {
    if (!out_bytes || !h) throw Error(ZKB_E_ARG, "null argument");
    *h = ctx->eng->prog_load(out_bytes, len, ctx->curve);
  });
}
int32_t zkb_prog_info(zkb_ctx* ctx, uint64_t h, uint64_t out[12]) {
  return guard(ctx, [&] { if (!out) throw Error(ZKB_E_ARG, "null"); ctx->eng->prog_info(h, out); });
}
int32_t zkb_prog_free(zkb_ctx* ctx, uint64_t h) { return guard(ctx, [&] { ctx->eng->prog_free(h); }); }
int32_t zkb_prog_compute_witness(zkb_ctx* ctx, uint64_t h, const uint64_t* inputs, uint64_t n_inputs, uint32_t flags,
                                 uint8_t* witness_out, size_t witness_cap, size_t* witness_len, uint64_t* first_unsatisfied) {
  return guard(ctx, [&] {
    if (!inputs && n_inputs) throw Error(ZKB_E_ARG, "null argument");
    uint64_t f = ctx->eng->prog_compute_witness(h, inputs, n_inputs, flags, witness_out, witness_cap, witness_len);
    if (first_unsatisfied) *first_unsatisfied = f;
    if (f != ~0ull) throw Error(ZKB_E_UNSAT, "constraint " + std::to_string(f) + " is not satisfied");
  });
}
int32_t zkb_prog_compute_witness_batch(zkb_ctx* ctx, uint64_t h, uint32_t count, const uint64_t* inputs, uint64_t n_inputs,
                                       uint32_t flags, uint8_t* witness_out, size_t witness_cap, size_t* witness_len,
                                       uint64_t* first_unsatisfied) {
  return guard(ctx, [&] {
    if ((!inputs && n_inputs && count) || !first_unsatisfied) throw Error(ZKB_E_ARG, "null argument");
    if (!ctx->eng->prog_compute_witness_batch(h, count, inputs, n_inputs, flags, witness_out, witness_cap, witness_len, first_unsatisfied))
      throw Error(ZKB_E_UNSAT, "an input set does not satisfy the constraints (see first_unsatisfied)");
  });
}
int32_t zkb_prog_prove_batch(zkb_ctx* ctx, uint64_t prog_handle, uint64_t pk_handle, uint32_t count, const uint64_t* inputs,
                             uint64_t n_inputs, uint32_t flags, const uint64_t* r, const uint64_t* s, uint8_t* proofs_out,
                             size_t proofs_cap, uint64_t* public_out, uint64_t public_cap, uint64_t* first_unsatisfied) {
  return guard(ctx, [&] {
    if ((!inputs && n_inputs && count) || !r || !s || !proofs_out || !first_unsatisfied) throw Error(ZKB_E_ARG, "null argument");
    uint64_t sz[4];
    ctx->eng->sizes(sz);
    if (proofs_cap < (size_t)count * sz[2]) throw Error(ZKB_E_ARG, "proof buffer too small");
    if (!ctx->eng->prog_prove_batch(prog_handle, pk_handle, count, inputs, n_inputs, flags, r, s, proofs_out, public_out, public_cap,
                                    first_unsatisfied))
      throw Error(ZKB_E_UNSAT, "an input set does not satisfy the constraints (see first_unsatisfied)");
  });
}
int32_t zkb_prog_set_witness(zkb_ctx* ctx, uint64_t h, const uint8_t* witness_bytes, size_t len) {
  return guard(ctx, [&] {
    if (!witness_bytes) throw Error(ZKB_E_ARG, "null argument");
    ctx->eng->prog_set_witness(h, witness_bytes, len);
  });
}
int32_t zkb_prog_public_inputs(zkb_ctx* ctx, uint64_t h, uint64_t* out, uint64_t cap, uint64_t* count) {
  return guard(ctx, [&] {
    uint64_t n = ctx->eng->prog_public_inputs(h, out, cap);
    if (count) *count = n;
  });
}
int32_t zkb_prog_assignment(zkb_ctx* ctx, uint64_t h, uint64_t* z_out, uint64_t cap_elems) {
  return guard(ctx, [&] {
    if (!z_out) throw Error(ZKB_E_ARG, "null argument");
    ctx->eng->prog_assignment(h, z_out, cap_elems);
  });
}
int32_t zkb_gm17_pk_load(zkb_ctx* ctx, const uint8_t* pk_bytes, size_t len, uint64_t* h) {
  return guard(ctx, [&] {
    if (!pk_bytes || !h) throw Error(ZKB_E_ARG, "null argument");
    *h = ctx->eng->gm17_pk_load(pk_bytes, len);
  });
}
int32_t zkb_gm17_pk_free(zkb_ctx* ctx, uint64_t h) { return guard(ctx, [&] { ctx->eng->gm17_pk_free(h); }); }
int32_t zkb_gm17_prove(zkb_ctx* ctx, uint64_t pk, uint64_t r1cs, const uint64_t* z, const uint64_t d1[4], const uint64_t d2[4],
                       const uint64_t r[4], uint8_t* proof_out, size_t proof_cap) {
  return guard(ctx, [&] {
    if (!d1 || !d2 || !r || !proof_out) throw Error(ZKB_E_ARG, "null argument");
    uint64_t sz[4];
    ctx->eng->sizes(sz);
    if (proof_cap < sz[2]) throw Error(ZKB_E_ARG, "proof buffer too small");
    ctx->eng->gm17_prove(pk, r1cs, z, d1, d2, r, proof_out);
  });
}
int32_t zkb_gm17_setup_size(zkb_ctx* ctx, uint64_t r1cs, size_t* len) {
  return guard(ctx, [&] { if (!len) throw Error(ZKB_E_ARG, "null"); *len = ctx->eng->gm17_setup_size(r1cs); });
}
int32_t zkb_gm17_setup(zkb_ctx* ctx, uint64_t r1cs, const uint64_t* trapdoor6, uint8_t* pk_out, size_t cap, size_t* len) {
  return guard(ctx, [&] {
    if (!trapdoor6 || !pk_out || !len) throw Error(ZKB_E_ARG, "null argument");
    ctx->eng->gm17_setup(r1cs, trapdoor6, pk_out, cap, len);
  });
}
int32_t zkb_field_op(zkb_ctx* ctx, int32_t field, int32_t op, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n) {
  return guard(ctx, [&] {
    if (!a || !out) throw Error(ZKB_E_ARG, "null argument");
    if (n) ctx->eng->field_op(field, op, a, b, out, n);
  });
}

int32_t zkb_groth16_setup_size(zkb_ctx* ctx, uint64_t r1cs, size_t* len) {
  return guard(ctx, [&] { if (!len) throw Error(ZKB_E_ARG, "null"); *len = ctx->eng->setup_size(r1cs); });
}
int32_t zkb_groth16_setup(zkb_ctx* ctx, uint64_t r1cs, const uint64_t* trapdoor7, uint8_t* pk_out, size_t cap, size_t* len) {
  return guard(ctx, [&] {
    if (!trapdoor7 || !pk_out || !len) throw Error(ZKB_E_ARG, "null argument");
    ctx->eng->setup(r1cs, trapdoor7, pk_out, cap, len);
  });
}

int32_t zkb_last_timings(zkb_ctx* ctx, double* ms_out, const char** names_out, int32_t cap) {
  if (!ctx || !ctx->eng) return 0;
  std::lock_guard<std::recursive_mutex> lock(ctx->mu);
  int32_t k = 0;
  for (auto& e : ctx->eng->timings) {
    if (k >= cap) break;
    if (ms_out) ms_out[k] = e.second;
    if (names_out) names_out[k] = e.first;
    k++;
  }
  return k;
}
uint64_t zkb_launch_count(zkb_ctx* ctx) { return ctx ? launch_counter() - ctx->launches0 : 0; }

#if defined(ZKB_EMU)
// Test build only (not in zkb.h): the order in which the emulation runs threads and blocks, process-wide (rt.cuh).
int32_t zkb_emu_launch_order(uint32_t mode, uint64_t seed) {
  if (mode > EMU_ORDER_SEEDED) { g_err = "unknown launch order"; return ZKB_E_ARG; }
  emu_order().mode = mode;
  emu_order().seed = seed;
  return ZKB_OK;
}
// Test build only: the stream policy (rt.cuh EMU_STREAMS_*: 0 eager, 1 lazy, 2 seeded) and flags (1: poison new device and
// pinned memory), process-wide.  Drains whatever the previous policy left queued and resets the statistics.
int32_t zkb_emu_stream_order(uint32_t mode, uint64_t seed, uint32_t flags) {
  if (mode > EMU_STREAMS_SEEDED || flags > EMU_STREAM_POISON) { g_err = "unknown stream policy"; return ZKB_E_ARG; }
  try {
    emu_set_streams(mode, seed, flags);
  } catch (const std::exception& e) {
    g_err = e.what();
    return ZKB_E_INTERNAL;
  }
  return ZKB_OK;
}
// out[0]: operations run after an operation enqueued later; out[1]: the most operations queued at once (since the policy was set)
int32_t zkb_emu_stream_stats(uint64_t out[2]) {
  if (!out) { g_err = "null"; return ZKB_E_ARG; }
  EmuStreams& E = emu_streams();
  std::lock_guard<std::recursive_mutex> lock(E.mu);
  out[0] = E.reordered;
  out[1] = E.peak;
  return ZKB_OK;
}
// An emulated stream outside any context, standing in for a caller's stream (torch / NCCL) in the stream-ordered chain
// exchange (zkb_groth16_prove_chains_to_stream / _stream_to_finish); zkb_emu_stream_copy queues a copy on it.
int32_t zkb_emu_stream_create(void** out) {
  if (!out) { g_err = "null"; return ZKB_E_ARG; }
  *out = (void*)(intptr_t)stream_create().s;
  return ZKB_OK;
}
int32_t zkb_emu_stream_destroy(void* h) {
  stream_destroy(stream_from_handle(h));
  return ZKB_OK;
}
int32_t zkb_emu_stream_copy(void* h, void* dst, const void* src, uint64_t bytes) {
  if (!dst || !src) { g_err = "null"; return ZKB_E_ARG; }
  d2d(stream_from_handle(h), dst, src, bytes);
  return ZKB_OK;
}
#endif

int32_t zkb_peak_probe(zkb_ctx* ctx, int32_t kind, uint32_t iters, double* out) {
  return guard(ctx, [&] {
    if (!out) throw Error(ZKB_E_ARG, "null");
    *out = peak_probe(ctx->st, kind, iters);
  });
}

}  // extern "C"
