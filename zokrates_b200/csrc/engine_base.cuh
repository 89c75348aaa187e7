// Curve-independent interface of the proving engine (one instance per zkb_ctx).
#pragma once
#include <utility>
#include <vector>
#include "rt.cuh"

namespace zkb {

// Per-context tuning / test options (zkb_ctx_set_option).  Defaults are the product configuration; nothing on a hot path
// reads the environment.
struct Options {
  int64_t tables = 1;         // ZKB_OPT_TABLES: 0 never build window tables, 1 auto (build when they fit), 2 build or fail with ZKB_E_OOM
  int64_t table_min_log = 14; // ZKB_OPT_TABLE_MIN_LOG: smallest MSM (log2 pairs) that gets tables
  int64_t table_c = 0;        // ZKB_OPT_TABLE_C: forced window width (0: cost model)
  int64_t z_mode = 0;         // ZKB_OPT_Z_MODE: 0 sample the assignment, 1 always the shared-bucket table mode, 2 always per-window buckets
  int64_t ntt_tile_min = 10;  // ZKB_OPT_NTT_TILE_MIN: transforms of 2^k points and more use the shared-memory tile passes
  int64_t ntt_max_s = 10;     // ZKB_OPT_NTT_MAX_S: stage bits per tile pass
  int64_t batch_affine = 0;   // ZKB_OPT_BATCH_AFFINE: rounds of pairwise affine additions (shared inversion) before the XYZZ accumulation; 0 = off
                              // (default: slower than the direct path as implemented, see msm_affine.cuh)
  int64_t batch_affine_min_log = 16;   // ZKB_OPT_BATCH_AFFINE_MIN_LOG: only for lists of 2^k (pair, window) entries and more
  int64_t chain_share = -1;   // ZKB_OPT_CHAIN_SHARE: MSM share taken off the ranks that compute a witness-map chain (world >= 3): -1 model, 0 none, > 0 per mille
  int64_t plan_stream = 0;    // ZKB_OPT_PLAN_STREAM: 1 = the z digit/sort plan runs on its own stream (overlaps the previous proof), 0 = heads the main
                              // stream (default: with two proofs in flight the GPU is work-bound, the overlap only slows the accumulate kernels)
  int64_t chunk_target = 600000;   // ZKB_OPT_CHUNK_TARGET: aimed-at number of accumulate chunks (threads) per MSM; chunk = entries / target, 8..64
  int64_t ntt_kernel = 2;     // ZKB_OPT_NTT_KERNEL: 2 = four-step twiddles / cp.async tile load (ntt_tile.cuh), 1 = the round-1 tile pass
  int64_t pk_cache = 1;       // ZKB_OPT_PK_CACHE: share proving keys by content and keep the last released one resident
  int64_t bitsum_radix = 2;   // ZKB_OPT_BITSUM_RADIX: bucket-reduction levels of radix 2 (1 dependent addition per launch) or 8 (7)
  int64_t batch_pass_max = 0; // ZKB_OPT_BATCH_PASS_MAX: most proofs or input sets of one batch pass; 0 = as many as fit in HBM
};

struct EngineBase {
  virtual ~EngineBase() {}
  Options opts;
  virtual void pk_table_info(uint64_t h, uint64_t out[8]) = 0;
  virtual void sizes(uint64_t out[4]) = 0;
  virtual uint64_t pk_load(const uint8_t* pk, size_t len, uint32_t rank, uint32_t world) = 0;
  virtual void pk_info(uint64_t h, uint64_t out[4]) = 0;
  virtual void pk_free(uint64_t h) = 0;
  virtual uint64_t r1cs_load(uint64_t N, uint64_t ni, uint64_t nw, const uint64_t* const rowptr[3],
                             const uint32_t* const col[3], const uint64_t* const val[3]) = 0;
  virtual void r1cs_free(uint64_t h) = 0;
  virtual void set_assignment(uint64_t r1cs, const uint64_t* z) = 0;
  virtual void prove_partial(uint64_t pk, uint64_t r1cs, const uint64_t* z, uint8_t* partial_out) = 0;
  virtual void prove_begin(uint64_t pk, uint64_t r1cs, const uint64_t* z, uint32_t chain_mask, void* chain_ptrs[3],
                           uint64_t* chain_bytes) = 0;
  virtual void prove_end(uint64_t pk, uint64_t r1cs, uint8_t* partial_out) = 0;
  virtual uint64_t prove_begin_async(uint64_t pk, uint64_t r1cs, const uint64_t* z, uint32_t chain_mask, void* chain_ptrs[3],
                                     uint64_t* chain_bytes) = 0;
  virtual void prove_end_async(uint64_t ticket) = 0;
  virtual void prove_chains_to_stream(uint64_t ticket, void* ext_stream) = 0;
  virtual void prove_stream_to_finish(uint64_t ticket, void* ext_stream) = 0;
  virtual uint64_t prove_submit(uint64_t pk, uint64_t r1cs, const uint64_t* z, const uint64_t* r, const uint64_t* s) = 0;
  virtual void prove_collect_partial(uint64_t ticket, uint8_t* partial_out) = 0;
  virtual void prove_collect(uint64_t ticket, uint8_t* proof_out) = 0;
  virtual void finalize_prepare(uint64_t pk, const uint64_t* r, const uint64_t* s) = 0;
  virtual void finalize(uint64_t pk, const uint8_t* partials, uint32_t world, const uint64_t* r, const uint64_t* s,
                        uint8_t* proof_out) = 0;
  virtual void prove_full(uint64_t pk, uint64_t r1cs, const uint64_t* z, const uint64_t* r, const uint64_t* s,
                          uint8_t* proof_out) = 0;
  virtual void prove_batch(uint64_t pk, uint64_t r1cs, uint32_t count, const uint64_t* z, const uint64_t* r, const uint64_t* s,
                           uint8_t* proofs_out) = 0;
  virtual void msm(int group, const uint8_t* points, const uint64_t* scalars, uint64_t n, uint8_t* out) = 0;
  virtual void ntt(uint64_t* data, uint32_t log_n, int inverse, int coset) = 0;
  virtual void witness_map(uint64_t r1cs, const uint64_t* z, uint64_t* h_out, uint64_t cap) = 0;
  virtual uint64_t witness_eval(uint64_t r1cs, uint64_t* z_io, uint32_t n_levels, const uint32_t* level_ptr,
                                const uint32_t* rows, const uint32_t* out_var) = 0;
  virtual uint64_t prog_load(const uint8_t* data, size_t len, int curve) = 0;
  virtual void prog_info(uint64_t h, uint64_t out[12]) = 0;
  virtual void prog_free(uint64_t h) = 0;
  virtual uint64_t prog_compute_witness(uint64_t h, const uint64_t* inputs, uint64_t n_inputs, uint32_t flags, uint8_t* wit_out,
                                        size_t cap, size_t* wit_len) = 0;
  virtual bool prog_compute_witness_batch(uint64_t h, uint32_t count, const uint64_t* inputs, uint64_t n_inputs, uint32_t flags,
                                          uint8_t* wit_out, size_t cap, size_t* wit_len, uint64_t* first_unsat) = 0;
  virtual bool prog_prove_batch(uint64_t h, uint64_t pk, uint32_t count, const uint64_t* inputs, uint64_t n_inputs, uint32_t flags,
                                const uint64_t* r, const uint64_t* s, uint8_t* proofs_out, uint64_t* public_out, uint64_t public_cap,
                                uint64_t* first_unsat) = 0;
  virtual void prog_set_witness(uint64_t h, const uint8_t* wit, size_t len) = 0;
  virtual uint64_t prog_public_inputs(uint64_t h, uint64_t* out, uint64_t cap) = 0;
  virtual void prog_assignment(uint64_t h, uint64_t* z_out, uint64_t cap_elems) = 0;
  virtual void field_op(int field, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n) = 0;
  virtual uint64_t gm17_pk_load(const uint8_t* pk, size_t len) = 0;
  virtual void gm17_pk_free(uint64_t h) = 0;
  virtual void gm17_prove(uint64_t pk, uint64_t r1cs, const uint64_t* z, const uint64_t* d1, const uint64_t* d2, const uint64_t* r,
                          uint8_t* proof_out) = 0;
  virtual size_t gm17_setup_size(uint64_t r1cs) = 0;
  virtual void gm17_setup(uint64_t r1cs, const uint64_t* trapdoor6, uint8_t* pk_out, size_t cap, size_t* len) = 0;
  virtual size_t setup_size(uint64_t r1cs) = 0;
  virtual void setup(uint64_t r1cs, const uint64_t* trapdoor7, uint8_t* pk_out, size_t cap, size_t* len) = 0;
  std::vector<std::pair<const char*, double>> timings;
};


// one translation unit per curve (engine_bn254.cu / engine_bls12_381.cu / engine_bls12_377.cu)
EngineBase* make_engine_bn254(Stream st);
EngineBase* make_engine_bls12_381(Stream st);
EngineBase* make_engine_bls12_377(Stream st);
size_t partial_bytes_bn254();
size_t partial_bytes_bls12_381();
size_t partial_bytes_bls12_377();

}  // namespace zkb
