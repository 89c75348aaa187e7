/* zkb.h — C ABI of the B200-native Groth16 proving backend (libzkb200.so).
 *
 * This is the drop-in boundary for ZoKrates' proving hot path.  A `zokrates_b200` Rust crate
 * implementing `zokrates_proof_systems::Backend<T, G16>` binds exactly these entry points through
 * `extern "C"` (see INTEGRATION.md for the bindgen-style stub and the CLI patch); the Python host
 * mirror in zokrates_b200/backend.py binds the same symbols with ctypes.
 *
 * Conventions
 *   - every function returns an int32 status (ZKB_OK = 0); zkb_last_error() gives the message of the
 *     last failure on the calling thread.  Nothing throws or aborts across this boundary; the
 *     reference panics on failure (zokrates_ark/src/groth16.rs:42,44), the shim turns a non-zero
 *     status into the same panic.
 *   - the caller owns every buffer; the callee copies what it needs before returning.
 *   - field elements cross the boundary as canonical little-endian bytes, exactly what
 *     `Field::write` / ark `CanonicalSerialize` produce (zokrates_field/src/lib.rs:215-233).
 *   - one context drives one GPU (one process per GPU); multi-GPU proving shards every MSM by index
 *     range (`rank`, `world` at zkb_pk_load) and exchanges 5 partial sums per proof.
 *   - there is no CPU fallback: without a usable CUDA device zkb_ctx_create fails with ZKB_E_CUDA.
 */
#ifndef ZKB_H
#define ZKB_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ZKB_OK 0
#define ZKB_E_ARG 1
#define ZKB_E_FORMAT 2
#define ZKB_E_CUDA 3
#define ZKB_E_OOM 4
#define ZKB_E_UNSAT 5
#define ZKB_E_INTERNAL 6

/* curve ids: the curves of BASELINE.json and BLS12-377; names as zokrates_field `Field::name()`
 * (zokrates_field/src/bn128.rs:1-13, bls12_381.rs:1-13, bls12_377.rs:1-13) */
#define ZKB_CURVE_BN128 0
#define ZKB_CURVE_BLS12_381 1
#define ZKB_CURVE_BLS12_377 2

typedef struct zkb_ctx zkb_ctx;

const char* zkb_last_error(void);
/* ABI version of this header */
uint32_t zkb_abi_version(void);
/* number of CUDA devices visible; <0 on CUDA failure */
int32_t zkb_device_count(void);

/* Replaces the implicit global state of the reference's static `Backend` methods
 * (zokrates_proof_systems/src/lib.rs:98-112 have no `self`): the Rust shim keeps one lazily
 * created context per (curve, device). */
int32_t zkb_ctx_create(int32_t curve, int32_t device, zkb_ctx** out);
void zkb_ctx_destroy(zkb_ctx* ctx);

/* Sizes in bytes for `curve`: out[0] = |Fr|, out[1] = |Fq|, out[2] = proof bytes (8 |Fq|),
 * out[3] = partial-sum blob bytes (zkb_groth16_prove_partial). */
int32_t zkb_curve_sizes(int32_t curve, uint64_t out[4]);

/* ---- proving key ------------------------------------------------------------------------------
 * pk_bytes: exactly what ark's `ProvingKey::serialize_unchecked` wrote, i.e. the `proving.key`
 * file (zokrates_ark/src/groth16.rs:97-98; read back unchecked at :40-42; layout SURVEY.md A.3).
 * rank/world: this context keeps rank's share of every query vector resident in HBM (world = 1 for
 * single-GPU): contiguous index ranges, cut where the WORK is equal (a_query / b_query are sparse — points at
 * infinity are skipped — and the sparsity is not uniform over the index); every rank derives the same cuts
 * from the key bytes.  The shares also hold the window tables 2^(c w) P built at load time. */
int32_t zkb_pk_load(zkb_ctx* ctx, const uint8_t* pk_bytes, size_t len, uint32_t rank, uint32_t world,
                    uint64_t* pk_handle);
/* out[0]=gamma_abc len (= instance count incl. one), out[1]=a_query len (= variables), out[2]=h_query len,
 * out[3]=l_query len */
int32_t zkb_pk_info(zkb_ctx* ctx, uint64_t pk_handle, uint64_t out[4]);
int32_t zkb_pk_free(zkb_ctx* ctx, uint64_t pk_handle);
/* HBM-resident window tables 2^(c w) P of this key share (a deliberate bytes-for-multiplications trade, DESIGN.md §4):
 * out[0] = c of the a/b1/b2/l tables (0: none), out[1] = their W, out[2] = c of the h table, out[3] = its W,
 * out[4] = table bytes, out[5] = resident key bytes (tables included),
 * out[6] / out[7] = status of the z / h tables: 1 built, 2 MSM below ZKB_OPT_TABLE_MIN_LOG, 3 did not fit in HBM
 * (the prover then runs the same MSM with per-window bucket sets: slower, never wrong), 4 disabled, 5 no admissible window. */
int32_t zkb_pk_table_info(zkb_ctx* ctx, uint64_t pk_handle, uint64_t out[8]);

/* Per-context options (the reference has none; its equivalents are cargo features, zokrates_ark/Cargo.toml:8-18).
 * Defaults are the product configuration; the tests use them to force every code path. */
#define ZKB_OPT_TABLES 1        /* 0 never build window tables, 1 build them when they fit (default), 2 build or fail ZKB_E_OOM */
#define ZKB_OPT_TABLE_MIN_LOG 2 /* smallest MSM (log2 pairs) that gets tables; default 14 */
#define ZKB_OPT_TABLE_C 3       /* forced window width of the tables, 0 = cost model (default) */
#define ZKB_OPT_Z_MODE 4        /* assignment MSMs: 0 sample z and choose (default), 1 shared-bucket table mode, 2 per-window buckets */
#define ZKB_OPT_NTT_TILE_MIN 5  /* transforms of 2^k points and more use the shared-memory tile passes; default 10 */
#define ZKB_OPT_NTT_MAX_S 6     /* stage bits per tile pass, 1..10; default 10 */
#define ZKB_OPT_BITSUM_RADIX 7  /* bucket reduction by bit sums: levels of radix 2 (default) or 8 */
#define ZKB_OPT_BATCH_AFFINE 10 /* rounds of pairwise AFFINE additions inside the buckets (one shared inversion per block, 6 instead of
                                 * 10 multiplications per addition) in front of the XYZZ bucket accumulation; default 0 = off: the
                                 * one serial inversion per block makes it slower than the direct path as implemented
                                 * (csrc/msm_affine.cuh); kept as a tested experimental path */
#define ZKB_OPT_BATCH_AFFINE_MIN_LOG 11 /* smallest sorted list (log2 entries) that gets the affine rounds; default 16 */
#define ZKB_OPT_PLAN_STREAM 12  /* 1: the digit/sort plan of the assignment MSMs runs on its own stream and overlaps the previous proof's
                                 * accumulate kernels; 0 (default): it heads the main stream (with two proofs in flight the GPU is work-bound) */
#define ZKB_OPT_CHUNK_TARGET 13 /* aimed-at number of accumulate chunks per MSM (default 600000); chunk length = entries / target in 8..64 */
#define ZKB_OPT_CHAIN_SHARE 14  /* multi-GPU, world >= 3: the ranks that compute a witness-map chain (0, 1, 2) get a smaller slice of every
                                 * query vector at zkb_pk_load; -1 (default) from a cost model, 0 equal shares, > 0 the chain's cost in
                                 * 1/1000 of the whole MSM work.  Must be equal on all ranks (the cuts are derived independently). */
#define ZKB_OPT_NTT_KERNEL 9    /* tile pass of the NTT: 2 (default) four-step twiddles + cp.async tile load, 1 the round-1 pass */
#define ZKB_OPT_BATCH_PASS_MAX 15 /* most proofs zkb_groth16_prove_batch / zkb_prog_prove_batch, and most input sets
                                   * zkb_prog_compute_witness_batch, run as one pass (one set of launches); 0 (default) = as many as
                                   * fit in free HBM and in the 32-bit indices of the sorted MSM lists.  Larger batches run as several
                                   * passes with the same results; tests use it to force several passes */
#define ZKB_OPT_PK_CACHE 8      /* 1 (default): zkb_pk_load of bytes that are already resident returns a handle onto the same key
                                 * (content fingerprint), and the last key released by zkb_pk_free stays resident until another
                                 * key is loaded — the per-call pk_load / prove / pk_free of the static trait method then builds
                                 * the window tables once; 0: every load builds, every free releases */
int32_t zkb_ctx_set_option(zkb_ctx* ctx, int32_t option, int64_t value);

/* ---- R1CS -------------------------------------------------------------------------------------
 * Matrices A, B, C in CSR form with columns in ark-relations order (0 = one, then instance
 * variables, then witness variables — the order `Computation::generate_constraints` allocates,
 * zokrates_ark/src/lib.rs:80-130).  Coefficients canonical LE, 4 x u64 each. */
int32_t zkb_r1cs_load(zkb_ctx* ctx, uint64_t n_constraints, uint64_t n_instance /* incl. one */,
                      uint64_t n_witness,
                      const uint64_t* a_rowptr, const uint32_t* a_col, const uint64_t* a_val,
                      const uint64_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val,
                      const uint64_t* c_rowptr, const uint32_t* c_col, const uint64_t* c_val,
                      uint64_t* r1cs_handle);
int32_t zkb_r1cs_free(zkb_ctx* ctx, uint64_t r1cs_handle);

/* ---- Groth16 prover ---------------------------------------------------------------------------
 * Replaces `Groth16::<E>::prove(&pk, computation, rng)` (zokrates_ark/src/groth16.rs:44).
 * z: full assignment [1, instance.., witness..] (n_instance + n_witness elements, canonical LE).
 * r, s: the two blinding scalars, canonical LE, drawn by the caller with ark semantics
 *       (`Fr::rand(rng)` twice, SURVEY.md App. B.5) so the RNG stays on the Rust side.
 * proof_out: A.x | A.y | B.x.c0 | B.x.c1 | B.y.c0 | B.y.c1 | C.x | C.y, canonical LE (8 |Fq| bytes) —
 *       the coordinate order `parse_g1`/`parse_g2` hex-encode (zokrates_ark/src/lib.rs:150-218). */
int32_t zkb_groth16_prove(zkb_ctx* ctx, uint64_t pk_handle, uint64_t r1cs_handle, const uint64_t* z,
                          const uint64_t* r, const uint64_t* s, uint8_t* proof_out, size_t proof_cap);

/* Same with the assignment already resident in HBM (set by zkb_r1cs_set_assignment): the
 * kernel-only timing region of bench.py. */
int32_t zkb_r1cs_set_assignment(zkb_ctx* ctx, uint64_t r1cs_handle, const uint64_t* z);
int32_t zkb_groth16_prove_resident(zkb_ctx* ctx, uint64_t pk_handle, uint64_t r1cs_handle,
                                   const uint64_t* r, const uint64_t* s, uint8_t* proof_out, size_t proof_cap);

/* K proofs of one circuit under one key.  z: K full assignments back to back (K x (n_instance + n_witness) elements,
 * canonical LE); r, s: K scalars each, canonical LE; proofs_out: K x zkb_curve_sizes()[2] bytes, proof k byte-identical
 * to zkb_groth16_prove(pk, r1cs, z_k, r_k, s_k).
 * The proofs share the key, its window tables, the matrices and the domain, so the device work of a PASS of proofs is one
 * set of launches: one SpMV over all assignments, the transforms of all chain vectors at once, and MSMs with one bucket set
 * per proof over the shared points.  A pass holds as many proofs as fit in free HBM (see ZKB_OPT_BATCH_PASS_MAX); the host
 * tails of its proofs run in parallel on host threads.  From a domain of 2^18 on, where a batch gains nothing over the pipeline, and
 * for count 1 the proofs run one after the other through the two-slot pipeline (zkb_groth16_prove_submit / _collect): same bytes.
 * ZKB_E_ARG: count 0, proofs_out too small, a key loaded with world > 1, a proof in flight on this context (it stays
 * collectable), a key that does not match the R1CS.  ZKB_E_OOM when not even one proof fits. */
int32_t zkb_groth16_prove_batch(zkb_ctx* ctx, uint64_t pk_handle, uint64_t r1cs_handle, uint32_t count,
                                const uint64_t* z, const uint64_t* r, const uint64_t* s, uint8_t* proofs_out, size_t cap);

/* Multi-GPU: every rank computes the partial sums of its index slice (opaque blob, host memory,
 * zkb_curve_sizes()[3] bytes: five projective points — their representation depends on the order the sort's
 * atomics produced, so blobs are not comparable byte for byte, only the finished proofs are); the host gathers
 * the `world` blobs (torch.distributed all_gather over NCCL) and any rank finishes the proof. */
int32_t zkb_groth16_prove_partial(zkb_ctx* ctx, uint64_t pk_handle, uint64_t r1cs_handle, const uint64_t* z,
                                  uint8_t* partial_out, size_t partial_cap);
int32_t zkb_groth16_finalize(zkb_ctx* ctx, uint64_t pk_handle, const uint8_t* partials, uint32_t world,
                             const uint64_t* r, const uint64_t* s, uint8_t* proof_out, size_t proof_cap);
/* Optional, on the rank that will call zkb_groth16_finalize: announce (r, s) before starting this rank's share so that
 * r*delta1, s*delta1, rs*delta1 and s*delta2 (ark-groth16 create_proof_with_reduction; they need nothing from the GPU) are
 * computed on host threads underneath the kernels.  Returns at once; finalize with the same (pk, r, s) picks them up. */
int32_t zkb_groth16_finalize_prepare(zkb_ctx* ctx, uint64_t pk_handle, const uint64_t* r, const uint64_t* s);

/* Multi-GPU, shared witness map.  The three chains of ark-groth16's `witness_map` (k = 0, 1, 2:
 * coset_fft(ifft(A z)), ...(B z), ...(C z); external crate reached from zokrates_ark/src/groth16.rs:44) are
 * independent, so with three or more ranks each chain is computed once instead of on every rank:
 *   zkb_groth16_prove_begin  starts the proof (z upload, the z-dependent MSMs) and computes the chains in
 *                            `chain_mask` (bit k = chain k) into DEVICE buffers whose addresses are returned in
 *                            chain_dev_ptrs[0..2] (`*chain_bytes` bytes each); when the mask is not 7 it returns
 *                            after this rank's chains are complete in memory;
 *   the host then broadcasts every chain buffer from the rank that computed it (NCCL over NVLink on the
 *   device pointers; zokrates_b200/distributed.py) and synchronises that transfer;
 *   zkb_groth16_prove_end    finishes the witness map, the h MSM and the reductions and returns the same
 *                            partial blob as zkb_groth16_prove_partial (= begin with mask 7 + end). */
int32_t zkb_groth16_prove_begin(zkb_ctx* ctx, uint64_t pk_handle, uint64_t r1cs_handle, const uint64_t* z,
                                uint32_t chain_mask, void* chain_dev_ptrs[3], uint64_t* chain_bytes);
int32_t zkb_groth16_prove_end(zkb_ctx* ctx, uint64_t pk_handle, uint64_t r1cs_handle, uint8_t* partial_out,
                              size_t partial_cap);

/* Pipelined proving: TWO proofs may be in flight per context.  `submit` enqueues a proof's whole device work and returns
 * without synchronising; `collect` waits for it and runs the host tail.  While the host finishes proof i (the last additions
 * of each MSM, the final combination, a multi-GPU gather) the GPU already runs proof i + 1, whose digit plans and
 * accumulate kernels overlap the latency-bound reduction tails of proof i — the reference proves strictly one at a time
 * (zokrates_cli/src/ops/generate_proof.rs:152-202 is one process per proof).
 *   submit: z may be NULL (resident assignment); r, s both NULL (partial only) or both given (finished proof).
 *   collect / collect_partial: in any order, each ticket once.  A third submit before a collect fails with ZKB_E_ARG.
 *   begin_async / end_async: the chain-exchange form (see above) without the synchronising collect. */
int32_t zkb_groth16_prove_submit(zkb_ctx* ctx, uint64_t pk_handle, uint64_t r1cs_handle, const uint64_t* z,
                                 const uint64_t* r, const uint64_t* s, uint64_t* ticket);
int32_t zkb_groth16_prove_collect(zkb_ctx* ctx, uint64_t ticket, uint8_t* proof_out, size_t proof_cap);
int32_t zkb_groth16_prove_collect_partial(zkb_ctx* ctx, uint64_t ticket, uint8_t* partial_out, size_t partial_cap);
int32_t zkb_groth16_prove_begin_async(zkb_ctx* ctx, uint64_t pk_handle, uint64_t r1cs_handle, const uint64_t* z,
                                      uint32_t chain_mask, void* chain_dev_ptrs[3], uint64_t* chain_bytes, uint64_t* ticket);
int32_t zkb_groth16_prove_end_async(zkb_ctx* ctx, uint64_t ticket);
/* Stream-ordered chain exchange: with ZKB_CHAIN_NO_HOST_SYNC or-ed into chain_mask, begin_async returns without waiting for this
 * rank's chains; `chains_to_stream` makes `cuda_stream` (a cudaStream_t: the stream the caller's NCCL broadcasts are ordered on)
 * wait for them, and `stream_to_finish` makes the finish step (end_async) wait for everything enqueued on `cuda_stream` so far —
 * the host never blocks between two proofs. */
#define ZKB_CHAIN_NO_HOST_SYNC 0x80000000u
int32_t zkb_groth16_prove_chains_to_stream(zkb_ctx* ctx, uint64_t ticket, void* cuda_stream);
int32_t zkb_groth16_prove_stream_to_finish(zkb_ctx* ctx, uint64_t ticket, void* cuda_stream);

/* ---- witness side (SURVEY.md §8 rows a9-a11) -------------------------------------------------
 * zkb_r1cs_check: (A z) o (B z) == C z for every constraint, on the device; z = NULL checks the resident assignment.
 *   Returns ZKB_E_UNSAT and the first violated constraint index (the interpreter's `UnsatisfiedConstraint`,
 *   zokrates_interpreter/src/lib.rs:95-104), ZKB_OK and UINT64_MAX otherwise.
 * zkb_witness_eval: witness generation for constraint-defined programs by dependency levels, following the rule of
 *   `Interpreter::execute_with_log_stream` (zokrates_interpreter/src/lib.rs:61-138): a constraint whose linear side is one
 *   fresh variable with coefficient one assigns it the value of the quadratic side, any other constraint is checked.
 *   z_inout: m x 32 bytes canonical LE, inputs (and `~one`) filled in, in the column order of zkb_r1cs_load; level l owns
 *   entries [level_ptr[l], level_ptr[l+1]) of rows[] (constraint indices) / out_var[] (assigned column or 0xFFFFFFFF = check).
 *   Directives (solvers) have no device path: the host interpreter handles programs that use them.  The finished
 *   assignment is written back and stays resident for zkb_groth16_prove_resident. */
int32_t zkb_r1cs_check(zkb_ctx* ctx, uint64_t r1cs_handle, const uint64_t* z, uint64_t* first_unsatisfied);
int32_t zkb_witness_eval(zkb_ctx* ctx, uint64_t r1cs_handle, uint64_t* z_inout, uint32_t n_levels,
                         const uint32_t* level_ptr, const uint32_t* rows, const uint32_t* out_var,
                         uint64_t* first_unsatisfied);

/* ---- compiled programs: the native front door (SURVEY.md §8 rows a10, f2) --------------------------------
 * zkb_prog_load: `out_bytes` is the compiled-program file `zokrates compile` writes and `generate-proof -i out` /
 *   `compute-witness -i out` read (header + serde_cbor sections, zokrates_ast/src/ir/serialize.rs:124-189,295-391).  The
 *   library parses it natively, synthesises the R1CS in ark variable order (`Computation::generate_constraints`,
 *   zokrates_ark/src/lib.rs:41-130) and keeps it resident: info[7] is an ordinary R1CS handle (owned by the program) for
 *   zkb_groth16_prove* / zkb_groth16_setup.  It also schedules the statements by dependency level.
 * zkb_prog_info: out[0] constraints, [1] instance variables incl. one, [2] witness variables, [3] arguments, [4] return
 *   values, [5] directives, [6] levels, [7] R1CS handle, [8] variables only directives touch, [9] directives whose solver has
 *   no device path (Zir functions, embed gadgets), [10] public arguments, [11] 1 if the statements can be scheduled.
 * zkb_prog_compute_witness: `Interpreter::execute` on the device (zokrates_interpreter/src/lib.rs:40-138): constraints assign
 *   or check, directives run the solver kernels (ConditionEq, Bits incl. the out-of-range path with flag 1 =
 *   `try_out_of_range`, Div, Xor, Or, ShaAndXorAndXorAnd, ShaCh, EuclideanDiv; :140-165,249-307).  inputs: n_inputs canonical
 *   field elements (32 bytes each), one per argument.  witness_out (may be NULL) receives the witness FILE bytes
 *   (`Witness::write`, zokrates_ast/src/ir/witness.rs:44-53); *witness_len its length.  The assignment stays resident for
 *   zkb_groth16_prove_resident.  ZKB_E_UNSAT + *first_unsatisfied on a violated constraint; ZKB_E_ARG "WrongInputCount".
 * zkb_prog_set_witness: `Witness::read` (:55-71) of a witness file into the resident assignment (ark column order).
 * zkb_prog_public_inputs: public arguments in declaration order, then ~out_0.. (ir/mod.rs:278-288) of the current
 *   assignment, canonical, 32 bytes each; out may be NULL to query *count.
 * zkb_prog_assignment: the program's current assignment (after zkb_prog_set_witness / zkb_prog_compute_witness) in ark
 *   column order, host copy: n_instance + n_witness canonical LE elements (4 x u64 each); cap_elems counts elements. */
int32_t zkb_prog_load(zkb_ctx* ctx, const uint8_t* out_bytes, size_t len, uint64_t* prog_handle);
int32_t zkb_prog_info(zkb_ctx* ctx, uint64_t prog_handle, uint64_t out[12]);
int32_t zkb_prog_free(zkb_ctx* ctx, uint64_t prog_handle);
int32_t zkb_prog_compute_witness(zkb_ctx* ctx, uint64_t prog_handle, const uint64_t* inputs, uint64_t n_inputs, uint32_t flags,
                                 uint8_t* witness_out, size_t witness_cap, size_t* witness_len, uint64_t* first_unsatisfied);
int32_t zkb_prog_set_witness(zkb_ctx* ctx, uint64_t prog_handle, const uint8_t* witness_bytes, size_t len);

/* Batches of input sets of one program.  inputs: count sets of n_inputs canonical elements back to back; flags as in
 * zkb_prog_compute_witness, for every set.  One level sweep serves all sets: the launch count does not grow with count.
 * first_unsatisfied[count]: set k's first violated constraint (the index zkb_prog_compute_witness reports for the same
 * inputs), UINT64_MAX when it is satisfied.  When some set fails the call returns ZKB_E_UNSAT; every other set's results are
 * complete and the failing sets' output slots are zero-filled.  Refused as a whole, before any launch, with the codes of the
 * single call: count 0, a wrong n_inputs, a non-canonical input in any set, a program that cannot be scheduled or calls a
 * solver without a device path, a short buffer.  Neither call changes the program's resident assignment (what
 * zkb_prog_public_inputs, zkb_prog_assignment and zkb_groth16_prove_resident read).
 * zkb_prog_compute_witness_batch: witness_out (may be NULL) receives count witness FILES back to back, all of one length
 *   *witness_len (8 + 40 x defined variables), file k byte-identical to zkb_prog_compute_witness on set k.
 * zkb_prog_prove_batch: inputs -> count Groth16 proofs under pk_handle, the assignments never leaving the device below a 2^18
 *   domain (the witness sweep writes the batched prover's interleaved assignment; from 2^18 on, and for count 1, the proofs
 *   run through the two-slot pipeline as in zkb_groth16_prove_batch).  r, s: count scalars each; proofs_out: count x
 *   zkb_curve_sizes()[2] bytes, proof k byte-identical to zkb_prog_compute_witness on set k + zkb_groth16_prove_resident
 *   with (r_k, s_k).  public_out (may be NULL): count x (public inputs) elements, set k's in the order of
 *   zkb_prog_public_inputs; public_cap counts elements.  Further ZKB_E_ARG refusals are zkb_groth16_prove_batch's: a key
 *   loaded with world > 1, a proof in flight (it stays collectable), a key that does not match the program's R1CS. */
int32_t zkb_prog_compute_witness_batch(zkb_ctx* ctx, uint64_t prog_handle, uint32_t count, const uint64_t* inputs, uint64_t n_inputs,
                                       uint32_t flags, uint8_t* witness_out, size_t witness_cap, size_t* witness_len,
                                       uint64_t* first_unsatisfied);
int32_t zkb_prog_prove_batch(zkb_ctx* ctx, uint64_t prog_handle, uint64_t pk_handle, uint32_t count, const uint64_t* inputs,
                             uint64_t n_inputs, uint32_t flags, const uint64_t* r, const uint64_t* s, uint8_t* proofs_out,
                             size_t proofs_cap, uint64_t* public_out, uint64_t public_cap, uint64_t* first_unsatisfied);
int32_t zkb_prog_public_inputs(zkb_ctx* ctx, uint64_t prog_handle, uint64_t* out, uint64_t cap, uint64_t* count);
int32_t zkb_prog_assignment(zkb_ctx* ctx, uint64_t prog_handle, uint64_t* z_out, uint64_t cap_elems);

/* ---- GM17 (SURVEY.md §8 row f3) ------------------------------------------------------------------------
 * The second proving scheme of the same trait: `impl Backend<T, GM17> for Ark` (zokrates_ark/src/gm17.rs:43-75 ->
 * ark-gm17 0.3.0 `ProvingKey::deserialize_unchecked`, `create_proof`).  pk_bytes: ark's `serialize_unchecked` of the GM17
 * `ProvingKey` (vk{h_g2, g_alpha_g1, h_beta_g2, g_gamma_g1, h_gamma_g2, query}, a_query, b_query, c_query_1, c_query_2,
 * g_gamma_z, h_gamma_z, g_ab_gamma_z, g_gamma2_z2, g_gamma2_z_t).  zkb_gm17_prove: z as in zkb_groth16_prove (NULL: the resident
 * assignment of the R1CS); d1, d2, r: the three masks `create_random_proof` draws in that order, canonical LE;
 * proof_out = A.x | A.y | B.x.c0 | B.x.c1 | B.y.c0 | B.y.c1 | C.x | C.y like the Groth16 proof.  The R1CS -> SAP witness map, the
 * five MSMs and the transforms run on the device with the Groth16 kernels.  ark-gm17's sources are not part of the reference
 * tree: restated in oracle/gm17.py, parity unpinned against real ark-gm17 output. */
/* zkb_gm17_setup: `impl NonUniversalBackend<T, GM17> for Ark`::setup (gm17.rs:19-41 -> ark-gm17 generate_parameters) from an explicit
 * trapdoor (alpha, beta, gamma, tau, g1 generator scalar, g2 generator scalar; 6 x 32 bytes canonical LE) — fixed-base multiples on
 * the device, key written in ark's serialize_unchecked layout.  The verifying key is the head of the proving key. */
int32_t zkb_gm17_setup_size(zkb_ctx* ctx, uint64_t r1cs_handle, size_t* len);
int32_t zkb_gm17_setup(zkb_ctx* ctx, uint64_t r1cs_handle, const uint64_t* trapdoor6, uint8_t* pk_out, size_t cap, size_t* len);
int32_t zkb_gm17_pk_load(zkb_ctx* ctx, const uint8_t* pk_bytes, size_t len, uint64_t* pk_handle);
int32_t zkb_gm17_pk_free(zkb_ctx* ctx, uint64_t pk_handle);
int32_t zkb_gm17_prove(zkb_ctx* ctx, uint64_t pk_handle, uint64_t r1cs_handle, const uint64_t* z, const uint64_t d1[4],
                       const uint64_t d2[4], const uint64_t r[4], uint8_t* proof_out, size_t proof_cap);

/* ---- building blocks (micro-benchmarks and parity tests; BASELINE.json config 5) ---------------
 * points: ark uncompressed affine encoding (x | y, canonical LE, infinity flag 0x40 in the last
 * byte) as in proving.key; scalars canonical LE 32 bytes; out: one point in the same encoding.
 * Replaces `VariableBaseMSM::multi_scalar_mul` (ark-ec 0.3.0). */
int32_t zkb_msm_g1(zkb_ctx* ctx, const uint8_t* points, const uint64_t* scalars, uint64_t n, uint8_t* out);
int32_t zkb_msm_g2(zkb_ctx* ctx, const uint8_t* points, const uint64_t* scalars, uint64_t n, uint8_t* out);
/* In-place size-2^log_n transform of canonical LE Fr elements, natural order in and out.
 * Replaces ark-poly `Radix2EvaluationDomain::{fft,ifft,coset_fft,coset_ifft}_in_place`. */
int32_t zkb_ntt(zkb_ctx* ctx, uint64_t* data, uint32_t log_n, int32_t inverse, int32_t coset);
/* h = witness_map(r1cs, z): domain-size canonical LE coefficients (ark `R1CSToQAP::witness_map`). */
int32_t zkb_witness_map(zkb_ctx* ctx, uint64_t r1cs_handle, const uint64_t* z, uint64_t* h_out, uint64_t h_cap_elems);
/* Batched field arithmetic on canonical LE operands: field 0 = Fr, 1 = Fq; op 0 = mul, 1 = add,
 * 2 = sub, 3 = inverse(a).  Replaces the `Field` ops of zokrates_field/src/lib.rs:407-503. */
int32_t zkb_field_op(zkb_ctx* ctx, int32_t field, int32_t op, const uint64_t* a, const uint64_t* b, uint64_t* out,
                     uint64_t n);

/* ---- setup ("next" row: NonUniversalBackend::setup, zokrates_ark/src/groth16.rs:90-109) ---------
 * Deterministic circuit-specific setup from an explicit trapdoor (alpha, beta, gamma, delta, tau and
 * the discrete logs of the two generators w.r.t. the standard ones), all canonical LE Fr.  Writes an
 * ark-format proving key (same bytes `serialize_unchecked` would produce for these parameters). */
int32_t zkb_groth16_setup(zkb_ctx* ctx, uint64_t r1cs_handle, const uint64_t* trapdoor7, uint8_t* pk_out,
                          size_t pk_cap, size_t* pk_len);
/* bytes zkb_groth16_setup will write for this R1CS */
int32_t zkb_groth16_setup_size(zkb_ctx* ctx, uint64_t r1cs_handle, size_t* pk_len);

/* ---- measurement ------------------------------------------------------------------------------
 * Per-stage device times (ms, CUDA events on the engine's stream) of the last prove/msm/ntt call.
 * names: static strings, one per slot; returns the number of slots filled. */
int32_t zkb_last_timings(zkb_ctx* ctx, double* ms_out, const char** names_out, int32_t cap);
/* Kernels launched by this context so far (bench.py's gpu_launches). */
uint64_t zkb_launch_count(zkb_ctx* ctx);
/* Integer-pipe peak probes used as roofline denominators: kind 0 = dependent-free IMAD.WIDE.U32
 * chain (returns 32x32+64 MAD/s), kind 1 = register-resident Montgomery multiplications in Fq
 * (returns field-mul/s).  `iters` controls the duration. */
int32_t zkb_peak_probe(zkb_ctx* ctx, int32_t kind, uint32_t iters, double* out_per_sec);

#ifdef __cplusplus
}
#endif
#endif /* ZKB_H */
