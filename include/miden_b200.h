/*
 * miden_b200.h -- C ABI of the H100 (sm_90a) STARK proving backend for Miden VM.
 *
 * Drop-in boundary: everything beneath `miden_prover::prove_stark()` (reference
 * prover/src/lib.rs:317-355), i.e. `ProverInstance::new(config, statement, None)?.prove(challenger)`
 * (crates/lifted-stark/src/prover/mod.rs:139,157,230-578).  The Rust host keeps trace generation,
 * the AIR (lowered once to an op-list, see mdn_air.program), the LogUp aux-trace builder
 * (a callback) and wincode serialisation of the returned streams.  INTEGRATION.md shows the
 * Rust `extern "C"` binding.  Beside the proof, mdn_check_constraints restates `debug::check_constraints`
 * (crates/lifted-stark/src/debug.rs:70-214): every constraint on every trace row, no proof.
 *
 * Conventions
 *   - every field element is a canonical Goldilocks u64 (< 2^64 - 2^32 + 1); quadratic-extension
 *     elements are two consecutive u64 (c0, c1), u^2 = 7 -- the layout of the reference's
 *     `Felt` / `QuadFelt` (crates/field/src/native/mod.rs:58, flatten_to_base order).
 *   - matrices are row-major exactly like p3 `RowMajorMatrix<Felt>`; the library transposes on
 *     the device.  Traces already on the device may also be column-major (MDN_FLAG_COLUMN_MAJOR).
 *   - functions return 0 on success and a negative mdn_status otherwise; the message is
 *     available through mdn_last_error().  Errors mirror `ProverError` / `ExecutionError::
 *     ProvingError(String)` (prover/mod.rs:582-596, prover/src/lib.rs:336-345).
 *   - a session is bound to one CUDA device and is not thread-safe; sessions are independent.
 *   - there is NO CPU fallback: if no CUDA device is usable, mdn_session_create fails.
 */
#ifndef MIDEN_B200_H
#define MIDEN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mdn_session mdn_session;

typedef enum {
    MDN_OK = 0,
    MDN_ERR_INVALID_ARG = -1,      /* malformed statement / trace shape (InstanceError) */
    MDN_ERR_DOMAIN = -2,           /* DomainError: LDE order too large, degree > blowup */
    MDN_ERR_CUDA = -3,             /* device error (message carries the CUDA string) */
    MDN_ERR_UNSUPPORTED = -4,      /* e.g. log_blowup > 4, > 1024 live constraint values */
    MDN_ERR_AUX_BUILDER = -5,      /* aux-trace callback failed */
    MDN_ERR_NO_DEVICE = -6,
    MDN_ERR_EXTERNAL_ASSERTION = -7,   /* ProverError::ExternalAssertionFailed / ::Reduction (prover/mod.rs:383-395) */
    MDN_ERR_CONSTRAINT_VIOLATED = -8,  /* the constraint guard refused the proof (mdn_session_set_constraint_guard) */
} mdn_status;

/* PcsParams::new(log_blowup, log_folding_arity, log_final_degree, folding_pow_bits,
 * deep_pow_bits, num_queries, query_pow_bits) -- crates/lifted-stark/src/pcs/params.rs:53-99.
 * Miden production values: air/src/config.rs:55-67 = {3, 2, 7, 4, 12, 27, 16}. */
typedef struct {
    uint32_t log_blowup;
    uint32_t log_folding_arity;
    uint32_t log_final_degree;
    uint32_t folding_pow_bits;
    uint32_t deep_pow_bits;
    uint32_t num_queries;
    uint32_t query_pow_bits;
} mdn_pcs_params;

/* p3 `DuplexChallenger<Felt, Poseidon2, 12, 8>` state (public fields used at
 * air/src/config.rs:264-271): sponge_state, input_buffer, output_buffer.  output_len counts the
 * unread rate elements; the next sample returns sponge_state[output_len - 1]. */
typedef struct {
    uint64_t sponge_state[12];
    uint64_t input_buffer[8];
    uint32_t input_len;
    uint32_t output_len;
} mdn_challenger;

/* Lowering of `LookupAir::eval` (air/src/lookup/builder.rs) for AIRs whose `build_aux_trace` is
 * `build_logup_aux_trace` (air/src/lookup/aux_builder.rs:49-97).  When `mdn_air.lookup` is set, the aux trace
 * and its committed final are built ON THE DEVICE from the resident main trace right after the randomness is
 * sampled -- no host callback, no aux-trace upload for that AIR.
 *   program words[0..5) = { 0x504B4C4D ("MLKP"), 1, n_nodes, n_interactions, n_consts }
 *   nodes        : as in mdn_air.program, restricted to what a LookupBuilder exposes: MAIN, PUBLIC,
 *                  CHALLENGE (0 = alpha, 1 = beta), CONST, EXT_CONST, ADD, SUB, MUL, NEG, PERIODIC, and
 *                  PREPROCESSED (a = row offset 0|1, b = column < preprocessed_width; an AIR without preprocessed
 *                  columns is refused with MDN_ERR_INVALID_ARG) -- the `CombinedWindow` reads of a preprocessed
 *                  lookup table.  AUX, AUX_VALUE and the selectors are refused.
 *   interactions : 4 words { aux column, flag node | 0xFFFFFFFF, multiplicity node, denominator node } --
 *                  one per `LookupGroup::insert` / `LookupBatch::insert` after `LookupMessage::encode`; it
 *                  contributes multiplicity/denominator to its column on every row where the (0/1) flag is
 *                  non-zero (air/src/lookup/prover.rs:338-362,421-444)
 *   consts       : (lo, hi) word pairs
 * Output (aux_builder.rs:1-20,215-268): f_c(r) = sum of m/d over column c's active interactions at row r;
 * aux[r][c] = f_c(r) for c > 0; aux[r][0] = sum_{r' < r} sum_c f_c(r'); aux value 0 = the total over all rows.
 * Requires aux_width == num_columns (<= 16) and num_aux_values == 1; a zero denominator is an error.
 * PREPROCESSED reads the raw preprocessed rows r and (r + 1) mod N of the trace domain, as mdn_check_constraints does.
 * Where each call takes them from:
 *   mdn_prove, mdn_prove_begin / commit_aux, the constraint guard : the installed bundle (mdn_session_set_preprocessed),
 *       which such a proof requires anyway; one derivation serves the LogUp build and the guard
 *   mdn_check_constraints, mdn_constraint_census                   : the call's own `preprocessed` argument
 *   mdn_check_trace_balance, mdn_check_lookup_folds, mdn_lookup_fold_census : the installed bundle, which must hold
 *       each AIR whose lookup program reads PREPROCESSED at that AIR's height and width (MDN_ERR_INVALID_ARG naming
 *       the AIR otherwise, before any device work); calls whose lookup programs read none do not consult it.
 * Version 2 adds register columns after the LogUp ones (the uint chiplets' Schwartz-Zippel columns; the reference's
 * `num_logup_cols` layout):
 *   program words[0..6) = { 0x504B4C4D, 2, n_nodes, n_interactions, n_consts, n_registers }
 *   nodes        : as version 1, plus AUX(a = 0, b = c) with num_columns <= c < aux_width: register c - num_columns's
 *                  value on the current row
 *   interactions : as version 1
 *   registers    : n_registers words, the update node of register i; register i is aux column num_columns + i
 *   consts       : (lo, hi) pairs
 * reg_i[0] = 0 and reg_i[r+1] = U_i evaluated on row r (every register read at its row-r value); the LogUp columns and
 * aux value 0 are what version 1 makes of the same interactions, and the registers take no part in them.  Refused with
 * MDN_ERR_INVALID_ARG naming the AIR, before any device work: aux_width != num_columns + n_registers; n_registers
 * outside 1..=4; num_aux_values != 1; an AUX leaf with offset 1 or on a LogUp column; an interaction whose flag,
 * multiplicity or denominator reaches an AUX leaf; an update not syntactically affine in the registers (register degree:
 * AUX 1, other leaves 0, ADD / SUB the max, MUL the sum, NEG the same; an update of degree > 1 is refused even where it
 * cancels).  Version 1 still refuses AUX.  mdn_check_trace_balance runs the interactions only (registers push
 * nothing); mdn_check_lookup_folds and mdn_lookup_fold_census compare the num_columns LogUp columns only (a given aux
 * trace still has 2 * aux_width base columns; folds_out stays num_columns wide); the AIR's own constraints check the
 * registers through mdn_check_constraints.  mdn_jit_compile_check compiles a version-2 program's interaction part. */
typedef struct {
    uint32_t num_columns;           /* LookupAir::num_columns() */
    uint32_t program_words;
    const uint32_t* program;
} mdn_lookup;

/* One AIR of the MultiAir (crates/lifted-air/src/air.rs:47-202 `LiftedAir`): shape + constraint
 * program.  `program` is the op-list lowering of `air.eval()`:
 *   words[0..5) = { 0x5249414D ("MAIR"), 1, n_nodes, n_constraints, n_consts }
 *   nodes: 3 words each { op, a, b }; constraints: node ids in emission order;
 *   consts: (lo, hi) word pairs.
 * Ops (leaf vocabulary of crates/ace-codegen/src/dag/lower.rs:109-210):
 *   0 MAIN(a=row offset 0|1, b=col)  1 AUX(a=offset, b=EF col)  2 PUBLIC(a)  3 CHALLENGE(a)
 *   4 AUX_VALUE(a)  5 IS_FIRST_ROW  6 IS_LAST_ROW  7 IS_TRANSITION  8 CONST(a)  9 EXT_CONST(a)
 *   10 ADD(a,b)  11 SUB(a,b)  12 MUL(a,b)  13 NEG(a)  14 PERIODIC(a=periodic column)
 *   15 PREPROCESSED(a=row offset 0|1, b=col)
 * Constraints are folded as acc <- acc*alpha + C_k in emission order
 * (crates/lifted-stark/src/verifier/constraints.rs:83,108). */
typedef struct {
    uint32_t width;                 /* BaseAir::width -- main trace columns */
    uint32_t aux_width;             /* LiftedAir::aux_width -- EF columns */
    uint32_t num_aux_values;        /* LiftedAir::num_aux_values */
    uint32_t num_randomness;        /* LiftedAir::num_randomness */
    uint32_t log_quotient_degree;   /* domain.rs:585-598 (symbolic degree analysis stays host-side) */
    uint32_t program_words;
    const uint32_t* program;
    /* `BaseAir::periodic_columns_matrix()` (crates/lifted-stark/src/prover/periodic.rs:49-98): row-major
     * (1 << log_max_period) x num_periodic_columns, every column repeated to the maximum period.
     * NULL / 0 when the AIR has no periodic columns. */
    const uint64_t* periodic_values;
    uint32_t num_periodic_columns;
    uint32_t log_max_period;
    uint32_t preprocessed_width;    /* BaseAir::preprocessed_width(): 0 = the AIR declares no preprocessed columns */
    const mdn_lookup* lookup;       /* NULL: the aux trace comes from the host (mdn_aux_builder / commit_aux) */
} mdn_air;

/* p3 RowMajorMatrix<Felt>: `values` has (1 << log_height) * width entries.  With
 * MDN_FLAG_DEVICE_TRACES `values` is a device pointer on the session's device. */
typedef struct {
    const uint64_t* values;
    uint32_t log_height;
    uint32_t width;
} mdn_matrix;

/* crates/lifted-air/src/statement.rs `Statement`: AIRs in instance order, shared air_inputs, and
 * the exact felts `Statement::observe` absorbs (AIR-specific, e.g. air/src/lib.rs:817-847). */
typedef struct {
    const mdn_air* airs;
    uint32_t n_airs;
    const uint64_t* public_values;
    uint32_t n_public_values;
    const uint64_t* observe_felts;
    uint32_t n_observe_felts;
} mdn_statement;

/* `LiftedAir::build_aux_trace(main, air_inputs, aux_inputs, challenges)` (prover/mod.rs:357-381),
 * called once per AIR in instance order after the main root is observed.
 *   randomness : 2 * num_randomness u64
 *   aux_out    : (1 << log_height) x (2 * aux_width) row-major, EF flattened to base
 *   aux_values : 2 * num_aux_values u64
 * Return 0 on success.  A NULL builder means all-zero aux traces and values
 * (crates/lifted-stark/src/testing/airs/miden.rs:84-94). */
typedef int (*mdn_aux_builder)(void* ctx, uint32_t instance, const mdn_matrix* main,
                               const uint64_t* randomness, uint64_t* aux_out, uint64_t* aux_values);

/* `StarkProofData { log_trace_heights, transcript: TranscriptData { fields, commitments } }`
 * (crates/lifted-stark/src/proof.rs:57-63, crates/stark-transcript/src/data.rs:11-15).
 * Memory is owned by the session and valid until the next prove on it or its destruction. */
typedef struct {
    const uint8_t* log_trace_heights;
    size_t n_heights;
    const uint64_t* fields;
    size_t n_fields;
    const uint64_t* commitments;    /* 4 u64 per commitment */
    size_t n_commitments;
} mdn_proof;

enum {
    MDN_FLAG_DEVICE_TRACES = 1u,    /* trace matrices already resident in device memory */
    MDN_FLAG_COLUMN_MAJOR = 2u,     /* with MDN_FLAG_DEVICE_TRACES only: the device matrices are column-major (below) */
};

/* ---- traces that already live on the GPU, column-major (MDN_FLAG_DEVICE_TRACES | MDN_FLAG_COLUMN_MAJOR) ----------
 * Accepted by mdn_prove, mdn_prove_begin and mdn_check_constraints.  Each mdn_matrix.values is then a device pointer on
 * the session's device, 16-byte aligned, and entry (row r, column c) is at values[(size_t)c << log_height | r] -- the
 * layout a trace builder on the GPU writes naturally.  The library copies it into its coefficient buffer (no transpose;
 * the per-kernel class 0 "transpose" of mdn_timings covers this ingest), a LogUp build (mdn_air.lookup) and the row
 * checks of mdn_check_constraints read it in place, and nothing ever writes to it.  Lifetime: the buffers must stay
 * valid and unchanged until mdn_prove / mdn_check_constraints returns; in the staged API until mdn_prove_commit_aux
 * returns.  There, the `aux` matrices of mdn_prove_commit_aux are column-major device matrices too (aux_values stay on
 * the host).  MDN_FLAG_COLUMN_MAJOR without MDN_FLAG_DEVICE_TRACES, or a misaligned pointer: MDN_ERR_INVALID_ARG.
 * The preprocessed traces (mdn_session_set_preprocessed, mdn_check_constraints) stay host row-major.
 * mdn_check_lookup_folds takes its `aux` matrices in the same layout (width 2 * aux_width: coordinate k of aux column c
 * is column 2c + k) and reads them in place; its `folds_out` buffers are then device buffers of 4 * num_columns columns
 * of 2^log_height rows, column 4c + w holding word w of (V c0, V c1, U c0, U c1) of aux column c:
 * folds_out[i][(size_t)(4 * c + w) << log_height | r].
 *
 * Aux traces of such calls come from the session's device aux builder, called in instance order for every AIR without
 * mdn_air.lookup, after the randomness is sampled:
 *   main       : the AIR's trace as passed (device, column-major)
 *   randomness : host, 2 * num_randomness u64
 *   aux_out    : device, column-major, 2 * aux_width columns of 2^log_height rows (EF flattened to base) -- the aux
 *                coefficient slot of that AIR itself, NULL when aux_width is 0
 *   aux_values : host, 2 * num_aux_values u64
 *   stream     : the session's cudaStream_t.  The builder enqueues its work on it or finishes it before returning; the
 *                library does not synchronise in between.  What it wrote is checked to be canonical.
 * Return 0 on success; otherwise the call fails with MDN_ERR_AUX_BUILDER.  The `build_aux` argument of those calls
 * must be NULL (MDN_ERR_INVALID_ARG otherwise).  With no device builder installed the aux traces and values are zero.
 * Calls without MDN_FLAG_COLUMN_MAJOR never consult it.  fn = NULL removes it. */
typedef int (*mdn_aux_builder_device)(void* ctx, uint32_t instance, const mdn_matrix* main, const uint64_t* randomness,
                                      uint64_t* aux_out, uint64_t* aux_values, void* stream);
int mdn_session_set_device_aux_builder(mdn_session* s, mdn_aux_builder_device fn, void* ctx);

/* ---- session ------------------------------------------------------------------------------ */
int mdn_session_create(const mdn_pcs_params* params, int cuda_device, mdn_session** out);
void mdn_session_destroy(mdn_session* s);
const char* mdn_last_error(const mdn_session* s);   /* s may be NULL: last create error */

/* ---- one proof on several GPUs ---------------------------------------------------------------------
 * One process per GPU of one NVLink/NVSwitch box; every rank calls mdn_prove (or the staged calls) with the SAME
 * statement / traces / challenger / flags and every rank returns the byte-identical proof.  The work of the ONE proof
 * is partitioned (the reference has no counterpart: it is single-process rayon; the loops that are split are
 * prover/commit.rs:142-180, lmcs/lifted_tree.rs:394-406, prover/constraints/mod.rs:246-259, prover/quotient.rs:163,
 * pcs/deep/prover.rs:214-312, pcs/fri/prover.rs:137-211):
 *   - rank g owns LDE cosets [g*B/G, (g+1)*B/G) of every committed column: forward coset NTTs, leaf sponge,
 *     constraint evaluation, quotient-chunk interpolation, DEEP quotient and FRI folds of those cosets;
 *   - rank g owns the Merkle sub-tree over leaves [g*L/G, (g+1)*L/G) of every commitment (input and FRI trees).
 * Data crosses ranks as peer-memory stores inside the producing kernels (CUDA IPC mappings of each rank's proof
 * arena over NVLink: leaf digests to the sub-tree owner, sub-roots / quotient chunk coefficients / the first small
 * FRI layer / opened values to every rank), ordered by a device-side flag barrier; there is no host round trip and
 * no library collective on the data path.  `fn` is only the bootstrap transport: it must gather `n_u64` words from
 * every rank into `recv` (rank-major) -- e.g. torch.distributed.all_gather -- and carries the 64-byte CUDA IPC
 * handles when an arena slab is created (first proof of a shape) and one word of rendezvous when slabs are
 * released.  world must be a power of two <= min(8, 2^log_blowup); world = 1 turns the partition off.  Collective:
 * every rank must call it at the same point.  The preprocessed bundle (mdn_session_set_preprocessed) and the
 * utility entry points (mdn_coset_lde_batch, mdn_lmcs_commit) are not partitioned. */
typedef int (*mdn_allgather_fn)(void* ctx, const uint64_t* send, uint64_t* recv, size_t n_u64);
int mdn_session_set_shard(mdn_session* s, uint32_t rank, uint32_t world, mdn_allgather_fn fn, void* ctx);

/* ---- Statement::eval_external (crates/lifted-air/src/air.rs:272-288, statement.rs:94-110) -------------------
 * Cross-AIR assertions are host code of the statement.  When a callback is installed the prover calls it once per
 * proof, after the aux traces are built -- on the host or on the device (mdn_air.lookup) -- and BEFORE the aux
 * commitment, exactly where the reference evaluates them (prover/mod.rs:383-395):
 *   challenges  : the shared randomness pool, 2 u64 per EF challenge          aux_values[i] : AIR i's aux values
 *   (instance order, 2 u64 per EF value, n_aux_values[i] of them)            log_trace_heights : instance order
 * Return 0 when every assertion evaluates to zero; > 0 with *failed_assertion = k for
 * `ProverError::ExternalAssertionFailed { assertion: k }`; < 0 for a `ReductionError`.  mdn_prove* then returns
 * MDN_ERR_EXTERNAL_ASSERTION and nothing of the aux phase is committed.  NULL (default) = no assertions. */
typedef int (*mdn_external_check)(void* ctx, const uint64_t* challenges, uint32_t n_challenges,
                                  const uint64_t* const* aux_values, const uint32_t* n_aux_values,
                                  const uint8_t* log_trace_heights, uint32_t n_airs, uint32_t* failed_assertion);
int mdn_session_set_external_check(mdn_session* s, mdn_external_check fn, void* ctx);

/* ---- STARK hash configuration (miden_air::config, air/src/config.rs) ----------------------------------------
 * MDN_HASH_POSEIDON2 (default): `poseidon2_config` (:241-273) -- StatefulSponge<Poseidon2, 12, 8, 4> leaves (alignment 8),
 *   TruncatedPermutation nodes, DuplexChallenger; the pre-bound challenger is the `mdn_challenger` argument of mdn_prove*.
 * MDN_HASH_BLAKE3: `blake3_256_config` (:276-307), the CLI's default hasher (miden-vm/src/cli/prove.rs:51) --
 *   ChainingHasher<Blake3> leaves (state <- blake3(state || little-endian u64 of every felt of the row); alignment 1, so
 *   opened rows and the OOD evaluation lists carry no zero padding), blake3(left || right) nodes,
 *   SerializingChallenger64<Felt, HashChallenger<u8, Blake3, 32>>.  Commitments are 32-byte digests carried as four
 *   little-endian u64 per commitment in `mdn_proof.commitments`.  The pre-bound challenger is the HashChallenger state
 *   installed with mdn_session_set_hash_challenger (after `config.challenger()` + `observe_protocol_params` that is the
 *   input buffer: 32 bytes of relation digest + 8 parameter felts as little-endian u64, and an empty output buffer); the
 *   `challenger` argument of mdn_prove* is ignored and may be NULL.  A preprocessed bundle belongs to the hash it was
 *   committed under.
 * MDN_HASH_KECCAK: `keccak_config` (:309-353) -- SerializingStatefulSponge<StatefulSponge<KeccakF, 25, 17, 4>> leaves (the
 *   overwrite-mode sponge over the canonical u64 of every felt; alignment 17: opened rows and the OOD lists are zero-padded
 *   to multiples of 17), PaddingFreeSponge<KeccakF, 25, 17, 4> nodes, SerializingChallenger64<Felt, HashChallenger<u8,
 *   Keccak256Hash, 32>>.  Digests are four u64 lanes; the challenger is installed like the Blake3 one (its input buffer must
 *   be whole 64-bit words, which `observe_slice(&relation_digest)` + `observe_protocol_params` always gives).
 * MDN_HASH_RPO / MDN_HASH_RPX: `rpo_config` / `rpx_config` (:225-248) -- the Poseidon2 configuration with the permutation
 *   replaced (`alg_config<P>` is generic in it, :255-273): same LMCS, alignment, duplex challenger (pass the `mdn_challenger`
 *   built with that permutation) and proof layout.  Functional coverage: an RPO permutation costs ~9x a Poseidon2 one. */
typedef enum { MDN_HASH_POSEIDON2 = 0, MDN_HASH_BLAKE3 = 1, MDN_HASH_KECCAK = 2, MDN_HASH_RPO = 3, MDN_HASH_RPX = 4 } mdn_hash_kind;
int mdn_session_set_hash(mdn_session* s, mdn_hash_kind kind);
/* p3 `HashChallenger<u8, Blake3 | Keccak256Hash, 32>`: `input_buffer`, `output_buffer` (bytes are sampled from its back). */
typedef struct {
    const uint8_t* input_buffer;
    size_t input_len;
    const uint8_t* output_buffer;
    size_t output_len;
} mdn_hash_challenger;
int mdn_session_set_hash_challenger(mdn_session* s, const mdn_hash_challenger* c);

/* ---- preprocessed columns: Preprocessed::build (crates/lifted-stark/src/preprocessed.rs:63-131) -----
 * `preprocessed[i]` = `BaseAir::preprocessed_trace()` of AIR i (HOST pointer; width 0 where the AIR declares
 * none, otherwise width == airs[i].preprocessed_width).  The declared matrices are sorted by (height, AIR
 * index), LDE'd on the canonical coset of their own height and committed in one aligned LMCS tree that stays
 * on the device and is borrowed by every later proof of this session (prover/mod.rs:118-123), until replaced.
 * `commitment_out` receives `Preprocessed::commitment()` -- the value the verifier is constructed with
 * (verifier/mod.rs:101-121).  A bundle must be installed exactly when some AIR of the proved statement
 * declares preprocessed columns, and each preprocessed height must equal the AIR's main trace height
 * (validate_preprocessed, preprocessed.rs:147-260): otherwise mdn_prove returns MDN_ERR_INVALID_ARG.
 * preprocessed == NULL removes the bundle. */
int mdn_session_set_preprocessed(mdn_session* s, const mdn_statement* st, const mdn_matrix* preprocessed,
                                 uint64_t commitment_out[4]);

/* ---- the drop-in: ProverInstance::prove (prover/mod.rs:230-578) ------------------------------
 * `challenger` is the caller's pre-bound challenger (protocol params observed,
 * prover/src/lib.rs:329-330); the statement felts and instance shape are observed inside, as the
 * reference does (mod.rs:290-291). */
int mdn_prove(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces /* instance order */,
              const mdn_challenger* challenger, mdn_aux_builder build_aux, void* aux_ctx,
              uint32_t flags, mdn_proof* out);

/* ---- the same path, staged (for hosts that prefer to drive the aux build themselves) -------- */
int mdn_prove_begin(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces,
                    const mdn_challenger* challenger, uint32_t flags,
                    uint64_t main_root[4], uint64_t* randomness_out /* 2*max num_randomness */);
int mdn_prove_commit_aux(mdn_session* s, const mdn_matrix* aux /* instance order, base-flattened */,
                         const uint64_t* const* aux_values /* per instance, 2*num_aux_values */,
                         uint64_t aux_root[4]);
int mdn_prove_finish(mdn_session* s, mdn_proof* out);

/* ---- check every constraint on every row, without proving: debug::check_constraints ----------------------------
 * (crates/lifted-stark/src/debug.rs:70-214; ExecutionTrace::check_constraints, processor/src/trace/mod.rs:251-278).
 *   1. challenges: the caller's challenger (or the installed hash challenger for Blake3 / Keccak, as in mdn_prove)
 *      observes observe_felts, the instance count and the log heights in instance order -- and NO commitment (neither
 *      the preprocessed one nor any root) -- then max num_randomness EF challenges are sampled into randomness_out.
 *      ExecutionTrace::check_constraints passes `config.challenger()` WITHOUT observe_protocol_params: the caller
 *      chooses the seed, and the challenges need not equal those of a proof.
 *   2. aux traces with those challenges: a lowered mdn_air.lookup is built on the device; otherwise `build_aux` is
 *      called (host-resident traces only, as in mdn_prove), or with MDN_FLAG_COLUMN_MAJOR the session's device aux
 *      builder; no builder means all-zero aux traces and values.  Column-major device traces are checked and read in
 *      place: nothing of them is uploaded or copied.
 *   3. the session's mdn_external_check, before the row checks (debug.rs:108-118): a non-zero assertion k makes
 *      the report kind 2; the row checks still run so that failing_rows is filled.  A callback returning < 0
 *      (ReductionError) makes the call return MDN_ERR_EXTERNAL_ASSERTION.
 *   4. for every instance (instance order), row r < N and constraint k (emission order): next row (r + 1) mod N,
 *      is_first = [r == 0], is_last = [r == N-1], is_transition = [r != N-1] exactly, periodic values = row
 *      r mod 2^log_max_period of periodic_values, PREPROCESSED = rows r and next of `preprocessed`.  A constraint
 *      fails when it is non-zero (in either coordinate); the first failure is the least (instance, row, k).
 * Returns MDN_OK whenever the check ran, whatever it found; malformed input gets mdn_prove's statuses and messages.
 * Refused before any device work: a call between mdn_prove_begin and mdn_prove_finish (MDN_ERR_INVALID_ARG) and a
 * session split over ranks (MDN_ERR_UNSUPPORTED).  The check uses the proof arena and releases it; it changes nothing
 * mdn_get_info / mdn_get_timings report about the last proof (MDN_INFO_JIT_CHECK is about the checks), and proofs
 * after it are unchanged.
 * The row pass of a program with at least the mdn_session_set_jit threshold of nodes runs on an NVRTC-specialised
 * kernel (k_jit_check), self-checked against the interpreter on its first use; the one-row probe of the reported value
 * stays on the interpreter.  mdn_get_info(MDN_INFO_JIT_CHECK) says which AIRs used it. */
typedef struct {
    uint32_t holds;          /* 1: every constraint is zero on every row and every external assertion is zero */
    uint32_t kind;           /* 0 none, 1 AIR constraint, 2 external assertion: the failure the reference panics on first */
    uint32_t instance;       /* kind 1: AIR index in INSTANCE order (statement order, not proof/height order) */
    uint32_t constraint;     /* kind 1: emission index in the AIR's program; kind 2: assertion index */
    uint64_t row;            /* kind 1 */
    uint64_t value[2];       /* kind 1: EF value (c0, c1) of that constraint at that row; c1 = 0 for base constraints */
    uint64_t failing_rows;   /* (instance, row) pairs, over all AIRs, where at least one constraint is non-zero */
} mdn_constraint_report;
int mdn_check_constraints(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces,
                          const mdn_matrix* preprocessed /* instance order, HOST, width 0 where none; NULL if no AIR declares any */,
                          const mdn_challenger* challenger, mdn_aux_builder build_aux, void* aux_ctx,
                          uint32_t flags, uint64_t* randomness_out /* 2*max num_randomness, may be NULL */,
                          mdn_constraint_report* out);

/* ---- refuse to prove a statement that does not hold: the constraint guard ---------------------------------------
 * enable = 1 makes every later mdn_prove / mdn_prove_commit_aux of this session check every constraint of every AIR on
 * every trace row before anything of the aux phase is committed; 0 (the default) turns it off.  Any other value, and a
 * call between mdn_prove_begin and mdn_prove_finish, is MDN_ERR_INVALID_ARG.
 * When: after the aux traces and aux values are final (host builder, device aux builder, device LogUp build, the
 * caller's aux of mdn_prove_commit_aux, or zeros) and the external assertions hold -- a failing assertion is still
 * MDN_ERR_EXTERNAL_ASSERTION and the guard does not run -- and before the aux commitment.
 * What it reads: the raw main traces (a copy kept from before the inverse NTT, or a column-major device trace in place,
 * which the caller keeps unchanged until mdn_prove_commit_aux returns, as for a LogUp build), the raw aux traces and aux
 * values about to be committed, the raw preprocessed rows (re-derived on the device from the installed bundle) and the
 * raw periodic matrices.  The challenges are the PROOF's randomness, sampled after the main commitment (what
 * mdn_prove_begin writes to randomness_out), and the proof's public values -- not the debug challenges of
 * mdn_check_constraints, which observe no commitment.  Rows, next row, selectors and the first failure (least
 * (instance, row, constraint)) are exactly those of mdn_check_constraints.
 * A non-zero constraint makes the call return MDN_ERR_CONSTRAINT_VIOLATED: mdn_last_error names the instance, row and
 * constraint, nothing is committed and the proof is abandoned, as after a failing external assertion.  A statement that
 * holds gets the byte-identical proof it gets with the guard off: the guard observes and samples nothing.
 * Cost: the raw main copies (N x width x 8 bytes per AIR of the proof arena) and one row pass per AIR -- k_jit_check
 * for programs at or above the mdn_session_set_jit threshold (its cubin is compiled and loaded by mdn_prove_begin only
 * while the guard is on), k_check_rows below it; its launches count in mdn_timings.kernel_launches and its time in
 * kernel class 4 and in commit_aux.  mdn_get_info(MDN_INFO_JIT_CHECK) says which AIRs the last guard run specialised.
 * A session split over ranks (mdn_session_set_shard): every rank holds the whole raw main and aux traces and runs the
 * whole check on them, with no communication; every rank returns the same status and report. */
int mdn_session_set_constraint_guard(mdn_session* s, uint32_t enable);
/* The report of the last guard run: kind 1 with instance, row, constraint, value and failing_rows (over all AIRs) as
 * mdn_check_constraints fills them, holds = 0, after a refusal; holds = 1, kind = 0 and every other field 0 after a
 * guard run that passed and before any guard run.  Proofs with the guard off, proofs that fail before the guard and
 * mdn_check_constraints leave it unchanged.  NULL s or out: MDN_ERR_INVALID_ARG. */
int mdn_last_constraint_report(const mdn_session* s, mdn_constraint_report* out);

/* ---- list every violated constraint, without proving: the census of mdn_check_constraints ----------------------
 * The same inputs, challenges, aux traces, external check, trace layouts and refusals as mdn_check_constraints; the row
 * pass keeps every (instance, row, constraint) whose value is non-zero instead of stopping at the first.
 *   failures : host, room for max_failures (NULL iff max_failures == 0): the first max_failures violations in
 *              (instance, row, constraint) order, instance order as in mdn_check_constraints -- the failures the
 *              reference would panic on one after another if each were fixed in turn.
 *   tallies  : host, room for max_tallies (NULL iff max_tallies == 0): each (instance, constraint) that is non-zero on
 *              at least one row, in (instance, constraint) order, truncated to max_tallies.
 *   out      : the counts; out->first is field for field the report mdn_check_constraints gives for the same call
 *              (its least failure and value come from the tallies; a failing external assertion takes precedence).
 * A NULL list with a non-zero capacity, or a NULL out, is MDN_ERR_INVALID_ARG before any device work.  The outputs do
 * not depend on the order in which device atomics ran: two calls on the same inputs give byte-identical outputs.
 * Refused, as mdn_check_constraints, inside a staged proof and on a session split over ranks; uses and releases the
 * proof arena; leaves mdn_get_info (but for MDN_INFO_JIT_CHECK), mdn_get_timings and later proofs unchanged.
 * The per-row count and tally pass runs on the NVRTC kernel k_jit_census for programs at or above the mdn_session_set_jit
 * threshold, as for mdn_check_constraints; the listing of the failures and the values at the tallies' first rows stay on
 * the interpreter. */
typedef struct {                 /* one violation: constraint `constraint` of instance `instance` is non-zero at `row` */
    uint32_t instance, constraint;
    uint64_t row;
    uint64_t value[2];           /* EF (c0, c1); c1 = 0 for base constraints */
} mdn_constraint_failure;        /* 32 bytes */
typedef struct {                 /* one (instance, constraint) that is non-zero on at least one row */
    uint32_t instance, constraint;
    uint64_t failing_rows;       /* rows where it is non-zero */
    uint64_t first_row, last_row;
    uint64_t first_value[2];     /* its value at first_row */
} mdn_constraint_tally;          /* 48 bytes */
typedef struct mdn_constraint_census {   /* the typedef cannot share the function's name in C */
    mdn_constraint_report first; /* field for field what mdn_check_constraints returns for the same call */
    uint64_t violations;         /* (instance, row, constraint) triples that are non-zero */
    uint64_t n_failures;         /* written to failures[] = min(violations, max_failures) */
    uint64_t failing_constraints;/* (instance, constraint) pairs with failing_rows > 0 */
    uint64_t n_tallies;          /* written to tallies[] = min(failing_constraints, max_tallies) */
} mdn_constraint_census_report;
int mdn_constraint_census(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces,
                          const mdn_matrix* preprocessed, const mdn_challenger* challenger,
                          mdn_aux_builder build_aux, void* aux_ctx, uint32_t flags, uint64_t* randomness_out,
                          mdn_constraint_failure* failures, uint64_t max_failures,
                          mdn_constraint_tally* tallies, uint64_t max_tallies,
                          mdn_constraint_census_report* out);

/* ---- find unbalanced LogUp bus messages, without proving: check_trace_balance ----------------------------------
 * (air/src/lookup/debug/trace/mod.rs:169-309, builder.rs:201-375).  Walks every row of every AIR of the statement that
 * carries a lowered mdn_air.lookup, keys every active push by its encoded denominator and sums the multiplicities
 * jointly over those AIRs (Miden's buses close across AIRs; a one-AIR statement gives the reference's per-AIR report).
 * AIRs without mdn_air.lookup are skipped and counted.  Per push, exactly as the reference's DebugTraceBuilder:
 * interaction k of the lookup program pushes (multiplicity, denominator) at row r when its flag is non-zero (or it has
 * none); the multiplicity is recorded as given, not multiplied by the flag; a zero denominator is an ordinary key (the
 * aux build refuses it); the next row wraps; periodic values are row r mod 2^log_max_period of periodic_values;
 * preprocessed columns are read from the installed bundle (see mdn_lookup).
 *   randomness : 2 * max num_randomness u64 (alpha, beta, ...: EF pairs), canonical -- e.g. the randomness_out of
 *                mdn_check_constraints or mdn_prove_begin.  Nothing is observed; no hash configuration is consulted.
 *   boundary   : n_boundary triples {denominator c0, c1, multiplicity}, canonical: the output of LookupAir::eval_boundary
 *                (DebugBoundaryEmitter, builder.rs:401-415).  Emission i is tagged instance 0xFFFFFFFF,
 *                row UINT64_MAX, column 0xFFFFFFFF, interaction i.
 *   mutex_sites: NULL, or per AIR (instance order) NULL or one word per interaction of its lookup program: 0xFFFFFFFF
 *                when the interaction is not in a group_with_cached_encoding, else (g << 16) | site with g the group's
 *                index within its column (the reference's group_idx) and site one insert / insert_encoded / batch call
 *                of that group (every interaction of a batch carries the batch's site, so all of them share one flag
 *                node).  A row violates group g of column c when more than one distinct site of it has a non-zero flag
 *                (track_mutex, builder.rs:204-208).  At most 1024 annotated interactions per AIR.
 *   max_contributions : the pushes of the unmatched denominators are listed when there are at most this many.
 *   flags      : as mdn_check_constraints: host row-major traces, MDN_FLAG_DEVICE_TRACES, | MDN_FLAG_COLUMN_MAJOR (read
 *                in place).
 * Orders.  unmatched: ascending denominator (c0, then c1) -- the derived Ord of p3's BinomialExtensionField over
 * Felt::cmp (crates/field/src/native/mod.rs:681); p3 is not vendored, so this order is not pinned by the reference's own
 * sources.  contributions: grouped in unmatched order, in emission order (instance, row, interaction) inside a group,
 * boundary emissions last.  mutex_violations: (instance, row, column, group).  The report does not depend on the order
 * in which the device's atomics ran.
 * Returns MDN_OK whenever the check ran, whatever it found.  Refused before any device work: a call between
 * mdn_prove_begin and mdn_prove_finish (MDN_ERR_INVALID_ARG) and a session split over ranks (MDN_ERR_UNSUPPORTED).
 * Malformed or non-canonical randomness, boundary triples or annotations: MDN_ERR_INVALID_ARG; a table larger than the
 * free device memory: MDN_ERR_UNSUPPORTED.  The report's memory is owned by the session and valid until the next call
 * on it.  Nothing mdn_get_info / mdn_get_timings report about the last proof changes, and later proofs are unchanged.
 * The three row passes (count, insert, collect) of a lookup program at or above the mdn_session_set_jit threshold run
 * on the NVRTC kernel k_jit_balance; on its first use in a session the interpreter repeats every pass into a second
 * table and lists of its own, which must agree (when that table does not fit in free device memory the call runs the
 * interpreter and the kernel stays unchecked).  MDN_INFO_JIT_LOOKUP_CHECK says which AIRs used it; the same holds for
 * mdn_check_lookup_folds (k_jit_fold) and mdn_lookup_fold_census (k_jit_fold_census). */
typedef struct {
    uint64_t denom[2];               /* encoded denominator (c0, c1) */
    uint64_t net_multiplicity;       /* sum of its multiplicities mod p, non-zero */
    uint64_t n_pushes;               /* pushes that landed on it */
    uint64_t first_row;              /* its least push (instance, row, interaction); UINT64_MAX for a boundary emission */
    uint32_t first_instance;         /* instance order; 0xFFFFFFFF: boundary */
    uint32_t first_interaction;      /* interaction index in the AIR's lookup program; boundary: index in `boundary` */
} mdn_unmatched;
typedef struct {
    uint64_t row;                    /* UINT64_MAX: boundary */
    uint64_t multiplicity;           /* as pushed */
    uint32_t instance;               /* 0xFFFFFFFF: boundary */
    uint32_t column;                 /* aux column of the interaction; 0xFFFFFFFF: boundary */
    uint32_t interaction;
    uint32_t reserved;
} mdn_balance_push;
typedef struct {
    uint64_t row;
    uint32_t instance, column, group, active_flags;   /* active_flags: distinct sites of the group with a non-zero flag */
} mdn_mutex_violation;
typedef struct {
    uint32_t holds;                  /* 1: nothing unmatched and no mutex violation */
    uint32_t contributions_complete; /* 1: contributions lists every push of every unmatched denominator */
    uint64_t n_pushes;               /* active pushes, boundary emissions included */
    uint64_t n_denominators;         /* distinct denominators pushed */
    uint64_t n_unmatched;
    uint64_t n_mutex_violations;
    uint64_t n_contributions;        /* pushes of the unmatched denominators (= sum of their n_pushes) */
    uint32_t n_skipped_airs;         /* AIRs without mdn_air.lookup */
    uint32_t reserved;
    const mdn_unmatched* unmatched;               /* n_unmatched */
    const mdn_balance_push* contributions;        /* n_contributions when contributions_complete, else NULL */
    const mdn_mutex_violation* mutex_violations;  /* the first min(n_mutex_violations, max_contributions) */
    uint64_t n_mutex_listed;
} mdn_balance_report;
int mdn_check_trace_balance(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces /* instance order */,
                            const uint64_t* randomness /* 2 * max num_randomness: alpha, beta, ... */,
                            const uint64_t* boundary, size_t n_boundary /* n x {denom c0, denom c1, multiplicity} */,
                            const uint32_t* const* mutex_sites /* per AIR, NULL or one word per interaction; NULL = none */,
                            uint64_t max_contributions, uint32_t flags, mdn_balance_report* out);

/* ---- cross-check a LogUp aux trace against the constraint path, without proving: collect_column_oracle_folds -----
 * (air/src/lookup/debug/trace/mod.rs:191-207 with run_trace_walk :220-282, filled by DebugTraceBuilder,
 * debug/trace/builder.rs:114-149,234-372; compared as assert_prover_matches_oracle does,
 * processor/src/trace/tests/lookup.rs:185-265).  For every row r of every AIR that carries a lowered mdn_air.lookup and
 * every aux column c it computes the constraint-path fold (V_c(r), U_c(r)), starting from (0, 1) each row, and checks
 * the aux trace against it:
 *   aux[r][c]               == V_c(r) / U_c(r)            for c >= 1           (kind 1 otherwise)
 *   aux[r+1][0] - aux[r][0] == sum over c of V_c(r)/U_c(r)                     (kind 2 otherwise)
 *   U_c(r) != 0                                                                (kind 3 otherwise: reported, not divided)
 * A column whose U is zero is left out of the kind 1 comparison, and a row with any zero U out of the kind 2 comparison.
 * Rows, the next-row wrap, periodic values, flags and the "multiplicity as given" rule are those of
 * mdn_check_trace_balance, preprocessed columns included; nothing is observed and no hash configuration is consulted.  Boundary emissions do not enter
 * the folds (mod.rs:194-195).  AIRs without mdn_air.lookup are skipped and counted.
 * The fold is the builder's, which (V, U) is compared with as a pair, not "sum m/d, then split":
 *   batch  : (N, D) <- (N * d + D * m, D * d) per interaction, from (0, 1)              (builder.rs:353-355,369-371)
 *   group  : (V_g, U_g) <- (V_g + N * flag, U_g + (D - 1) * flag) per insert / insert_encoded / batch call, from (0, 1),
 *            a single insert being the batch of its one interaction; the flag enters as a field element (an
 *            interaction without a flag node has flag 1) and a zero flag adds nothing   (builder.rs:245-252,278-279)
 *   column : (V, U) <- (V * U_g + V_g * U, U * U_g) per group, from (0, 1)              (builder.rs:144-146)
 * Of a group_with_cached_encoding only the canonical closure is folded, which is the one the lowered program carries
 * (builder.rs:177-181).  With boolean flags of which at most one is set per group this equals the prover path
 * (k_logup_rows: one rational per column over the active pushes); where a flag is not boolean or two flags of a group
 * are set together the two paths differ, and this call says where.
 * The lowered mdn_lookup program carries column, flag, multiplicity and denominator per interaction but not where a
 * group or a batch begins, so that comes as an optional per-interaction argument (as mutex_sites does for
 * mdn_check_trace_balance; mdn_lookup is unchanged):
 *   fold_marks : NULL, or per AIR (instance order) NULL or one word per interaction of its lookup program, emission
 *                order: 3 = the interaction opens a new group (and the first insert / batch call of it), 1 = it opens a
 *                new insert / insert_encoded / batch call in the open group, 0 = it continues the batch of the previous
 *                interaction.  Interaction 0 and every interaction whose column differs from its predecessor's carry
 *                3; an interaction marked 0 shares its predecessor's flag node.  NULL: every interaction is a group of
 *                its own, i.e. (V, U) <- (V * (1 + (d - 1) * flag) + m * flag * U, U * (1 + (d - 1) * flag)).
 *   randomness : as mdn_check_trace_balance (2 * max num_randomness u64, canonical).
 *   aux        : NULL, or per AIR (instance order; entries of AIRs without mdn_air.lookup are ignored) the aux trace
 *                in this library's layout: 2^log_height rows (the reference's (n+1)-row `accumulate` output without
 *                its last row, aux_builder.rs:49-97), base-flattened EF, width 2 * aux_width, canonical; host row-major,
 *                or on the device as the traces are (MDN_FLAG_DEVICE_TRACES, | MDN_FLAG_COLUMN_MAJOR: read in place).
 *                NULL: the call first runs the device LogUp build (k_logup_rows + k_scan_*) on the same traces and
 *                challenges and checks that -- the prover path against the constraint path.  That build refuses a zero
 *                denominator (MDN_ERR_INVALID_ARG), so a kind 3 report needs an explicit aux.
 *   aux_finals : with aux, per AIR 2 u64 (host, canonical): the value aux[n][0] would hold (aux value 0), which closes
 *                the last row's delta: aux_finals[i] - aux[n-1][0].  Must be NULL when aux is NULL.
 *   folds_out  : NULL, or per AIR NULL or a buffer of rows x num_columns x 4 u64, entry (r, c) = (V c0, V c1, U c0, U c1)
 *                at folds_out[i][4 * (r * num_columns + c)]: host memory, device memory with MDN_FLAG_DEVICE_TRACES
 *                (16-byte aligned), column-major planes with | MDN_FLAG_COLUMN_MAJOR (layout above).
 * First failure: the least (instance, row, column) in instance order; failing_rows and zero_u count over all AIRs.
 * Returns MDN_OK whenever the check ran, whatever it found.  Refusals and statuses as mdn_check_trace_balance: malformed
 * or non-canonical randomness, aux, finals or marks MDN_ERR_INVALID_ARG; a call between mdn_prove_begin and
 * mdn_prove_finish MDN_ERR_INVALID_ARG and a session split over ranks MDN_ERR_UNSUPPORTED, both before any device work;
 * a host folds_out whose device staging is larger than the free device memory MDN_ERR_UNSUPPORTED.  Nothing
 * mdn_get_info / mdn_get_timings report about the last proof changes, and later proofs are unchanged. */
typedef struct {
    uint32_t holds;            /* 1: every checked (row, column) agrees and no U is zero */
    uint32_t kind;             /* 0 none, 1 fraction column mismatch (c >= 1), 2 accumulator mismatch (c = 0), 3 zero U */
    uint32_t instance;         /* first failure: least (instance, row, column), instance order */
    uint32_t column;
    uint64_t row;
    uint64_t fold[4];          /* (V c0,c1, U c0,c1) of that (row, column) */
    uint64_t expected[2];      /* kind 1: V/U; kind 2: sum_c V_c/U_c; kind 3: 0 (c >= 1) or the sum over the non-zero U (c = 0) */
    uint64_t actual[2];        /* kind 1, 3 (c >= 1): aux[r][c]; kind 2, 3 (c = 0): aux[r+1][0] - aux[r][0] */
    uint64_t failing_rows;     /* (instance, row) pairs with at least one disagreement or zero U, over all AIRs */
    uint64_t zero_u;           /* (instance, row, column) triples with U == 0 */
    uint32_t n_skipped_airs;   /* AIRs without mdn_air.lookup */
    uint32_t reserved;
} mdn_fold_report;
int mdn_check_lookup_folds(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces /* instance order */,
                           const uint64_t* randomness /* 2 * max num_randomness: alpha, beta, ... */,
                           const uint32_t* const* fold_marks /* per AIR, NULL or one word per interaction; NULL = none */,
                           const mdn_matrix* aux /* instance order, width 2 * aux_width; NULL: the device LogUp build */,
                           const uint64_t* const* aux_finals /* per AIR 2 u64; NULL with aux == NULL */,
                           uint64_t* const* folds_out /* NULL, or per AIR NULL or rows x num_columns x 4 u64 */,
                           uint32_t flags, mdn_fold_report* out);

/* ---- list every disagreement between an aux trace and its lookup program, without proving: the census of
 * mdn_check_lookup_folds ----------------------------------------------------------------------------------------
 * The same inputs, validation, messages, trace layouts and refusals as mdn_check_lookup_folds without folds_out (aux ==
 * NULL: the device LogUp build of the same call, so that every row where a flag is not boolean or two flags of a group
 * are set together is listed); the verdict of every (instance, row, column) is the one mdn_check_lookup_folds gives:
 * kind 3 where U_c is zero, kind 1 for a fraction column that differs, kind 2 for column 0 when its delta differs and no
 * U of that row is zero (a row with a zero U lists no column-0 entry).  Every one with kind != 0 is kept:
 *   failures : host, room for max_failures (NULL iff max_failures == 0): the first max_failures disagreements in
 *              (instance, row, column) order, instance order as in mdn_check_lookup_folds.
 *   tallies  : host, room for max_tallies (NULL iff max_tallies == 0): each (instance, column) that disagrees on at least
 *              one row, in (instance, column) order, truncated to max_tallies.
 *   out      : the counts; out->first is field for field the report mdn_check_lookup_folds gives for the same call (the
 *              first failing instance's least (first_row, column) of the tallies, its values probed at that row).
 * A NULL list with a non-zero capacity, or a NULL out, is MDN_ERR_INVALID_ARG before any device work; a failure list
 * whose device staging is larger than the free device memory MDN_ERR_UNSUPPORTED.  The outputs do not depend on the
 * order in which device atomics ran: two calls on the same inputs give byte-identical outputs.  Refused, as
 * mdn_check_lookup_folds, inside a staged proof and on a session split over ranks; uses and releases the proof arena;
 * leaves mdn_get_info (but for MDN_INFO_JIT_LOOKUP_CHECK), mdn_get_timings and later proofs unchanged.  The per-row count
 * and tally pass runs on the NVRTC kernel k_jit_fold_census for lookup programs at or above the mdn_session_set_jit
 * threshold (self-checked against k_fold_census_rows on its first use); the failure listing and its probes stay on the
 * interpreter. */
typedef struct {                 /* one (instance, row, column) where the aux trace departs from the fold */
    uint32_t instance, column;
    uint32_t kind;               /* 1, 2 or 3 exactly as mdn_fold_report.kind */
    uint32_t reserved;
    uint64_t row;
    uint64_t fold[4];            /* (V c0, V c1, U c0, U c1) of that (row, column) */
    uint64_t expected[2], actual[2];   /* as mdn_fold_report: the same conventions for every kind and column */
} mdn_fold_failure;              /* 88 bytes */
typedef struct {                 /* one (instance, column) that disagrees on at least one row */
    uint32_t instance, column;
    uint64_t failing_rows;       /* rows where this column has kind != 0 */
    uint64_t zero_u_rows;        /* of those, rows of kind 3 (U_c == 0) */
    uint64_t first_row, last_row;
    uint32_t first_kind, reserved;
    uint64_t first_expected[2], first_actual[2];   /* at first_row */
} mdn_fold_tally;                /* 80 bytes */
typedef struct {
    mdn_fold_report first;       /* field for field what mdn_check_lookup_folds returns for the same call */
    uint64_t disagreements;      /* (instance, row, column) triples with kind != 0 */
    uint64_t n_failures;         /* = min(disagreements, max_failures) written to failures[] */
    uint64_t failing_columns;    /* (instance, column) pairs with failing_rows > 0 */
    uint64_t n_tallies;          /* = min(failing_columns, max_tallies) written to tallies[] */
} mdn_fold_census_report;
int mdn_lookup_fold_census(mdn_session* s, const mdn_statement* st, const mdn_matrix* traces /* instance order */,
                           const uint64_t* randomness /* 2 * max num_randomness: alpha, beta, ... */,
                           const uint32_t* const* fold_marks /* per AIR, NULL or one word per interaction; NULL = none */,
                           const mdn_matrix* aux /* instance order, width 2 * aux_width; NULL: the device LogUp build */,
                           const uint64_t* const* aux_finals /* per AIR 2 u64; NULL with aux == NULL */, uint32_t flags,
                           mdn_fold_failure* failures, uint64_t max_failures,
                           mdn_fold_tally* tallies, uint64_t max_tallies,
                           mdn_fold_census_report* out);

/* wincode/bincode-default layout of StarkProofData (prover/src/lib.rs:347-354): u64-LE length +
 * height bytes; u64-LE length + u64-LE felts; u64-LE length + 32-byte commitments.  Returns the
 * number of bytes needed; writes only if cap is large enough.  (Layout unpinned in-tree.) */
size_t mdn_proof_serialize(const mdn_proof* p, uint8_t* out, size_t cap);

/* ---- the two trait seams of StarkConfig (crates/lifted-stark/src/config.rs:26-45) ----------- */
/* Dft::coset_lde_batch(mat, added_bits, shift) as used at prover/commit.rs:173.  `out` receives
 * the (1 << (log_height+added_bits)) x width result, row-major, rows in bit-reversed order. */
int mdn_coset_lde_batch(mdn_session* s, const mdn_matrix* mat, uint32_t added_bits, uint64_t shift,
                        uint64_t* out);
/* Lmcs::build_aligned_tree(ldes).root() (lmcs/config.rs:125-139) for matrices given in domain
 * (natural) order, ascending heights.  */
int mdn_lmcs_commit(mdn_session* s, const mdn_matrix* mats_domain_order, uint32_t n_mats,
                    uint64_t root[4]);
/* Poseidon2 permutation on `n` independent 12-element states (crates/crypto/src/hash/
 * algebraic_sponge/poseidon2/mod.rs:31-37), device-computed. */
int mdn_poseidon2_permute(mdn_session* s, uint64_t* states /* n x 12 */, size_t n);

/* ---- host-side transcript helpers -----------------------------------------------------------
 * `CanObserve::observe` / `CanSample::sample` of the duplex challenger for hosts without p3
 * (tests, bench); sequential sponge steps on the CPU, exactly what the reference's host does.
 * Semantics: crates/lib/core/asm/stark/random_coin.masm:103-115,128-135,181-210,272-296. */
void mdn_challenger_observe(mdn_challenger* c, const uint64_t* felts, size_t n);
uint64_t mdn_challenger_sample(mdn_challenger* c);

/* ---- introspection for stage-level parity tests and the benchmark ---------------------------- */
typedef enum {
    MDN_INFO_MAIN_ROOT = 0,        /* 4 u64 */
    MDN_INFO_AUX_ROOT = 1,         /* 4 u64 */
    MDN_INFO_QUOTIENT_ROOT = 2,    /* 4 u64 */
    MDN_INFO_OOD_POINT = 3,        /* 2 u64 */
    MDN_INFO_QUOTIENT_ACC = 4,     /* N_max*D EF values, natural order on gJ */
    MDN_INFO_DEEP_EVALS = 5,       /* L EF values, bit-reversed order */
    MDN_INFO_FRI_ROOTS = 6,        /* 4 u64 per round */
    MDN_INFO_QUERY_INDICES = 7,    /* num_queries u64 */
    MDN_INFO_JIT = 8,              /* per AIR (proof order) of the last proof: 1 = NVRTC kernel, 0 = interpreter */
    MDN_INFO_POOL = 9,             /* cudaMallocAsync pool reserved now / high, used now / high (bytes); proof arena capacity (bytes), slabs, driver allocations so far, live blocks */
    MDN_INFO_BUILD = 10,           /* { generation of the field arithmetic, generation of the NTT kernels }: always { 2, 2 } (poseidon2_fast2.cuh, ntt2.cuh) */
    MDN_INFO_JIT_CHECK = 11,       /* per AIR (instance order) of the last mdn_check_constraints / mdn_constraint_census call or constraint-guard run: 1 = NVRTC row kernel, 0 = interpreter */
    MDN_INFO_JIT_LOOKUP_CHECK = 12, /* per AIR (instance order) of the last mdn_check_trace_balance / mdn_check_lookup_folds / mdn_lookup_fold_census call: 1 = NVRTC row kernel, 0 = interpreter (also for an AIR without mdn_air.lookup) */
    MDN_INFO_JIT_CACHE = 13,       /* process-wide, session may be NULL: { disk hits, disk misses (no usable file: compiled), rejected files, write failures, NVRTC compiles, NVRTC wall ms } (mdn_jit_set_cache_dir); the last two count every compile, cache on or off */
} mdn_info;
/* QUOTIENT_ACC / DEEP_EVALS are only recorded (extra device->host copies) after mdn_set_debug(s, 1). */
int mdn_set_debug(mdn_session* s, int enable);
/* Layout self-description for binding authors: { sizeof pcs_params, challenger, lookup, air; offsetof air.program,
 * .periodic_values, .preprocessed_width, .lookup; sizeof matrix, statement, proof, timings; offsetof
 * timings.kernel_ms, .permutations }.  Returns the number of entries. */
size_t mdn_abi_layout(uint32_t* out, size_t cap);

/* ---- run-time specialisation of the constraint evaluator -------------------------------------------
 * AIR programs with at least `min_nodes` nodes (default 256; 0 = never) are lowered to straight-line CUDA,
 * compiled once per program with NVRTC for sm_90a and cached; smaller ones (and all of them when libnvrtc
 * is absent) run on the op-list interpreter.  Both produce identical values.  Specialised: the proof's constraint
 * evaluation and LogUp row build (MDN_INFO_JIT), the row pass of mdn_check_constraints, mdn_constraint_census and
 * the constraint guard (MDN_INFO_JIT_CHECK), and the row passes of the lookup checks mdn_check_trace_balance,
 * mdn_check_lookup_folds and mdn_lookup_fold_census (MDN_INFO_JIT_LOOKUP_CHECK; the lookup program's node count decides,
 * and only these three calls compile or load its kernels).  Interpreted whatever the size: the censuses' failure
 * listings, the checks' one-row probes and the register program of a version-2 lookup program.
 * Each compiled kernel is compared with the interpreter on its first use in a session: word for word, and for the
 * balance table slot by slot (slot placement follows the order of the atomics). */
int mdn_session_set_jit(mdn_session* s, uint32_t min_nodes);
/* "nvrtc <version>" or why it is unavailable, plus the reason the last JIT attempt was dropped (compile error,
 * or the first-use comparison against the interpreter failed -- the interpreter's result is then kept). */
const char* mdn_jit_status(mdn_session* s);
/* Codegen + NVRTC only, no device needed: cubin size (> 0) or a negative mdn_status with *err set.  Fills the
 * mdn_jit_set_cache_dir cache for the constraint mode (a constraint program) or the LogUp mode (a lookup program). */
long long mdn_jit_compile_check(const uint32_t* program, uint32_t program_words, const char** err);
/* Keeps the NVRTC cubins on disk, so that later processes load them instead of compiling again (a Miden-size program
 * takes NVRTC tens of seconds per mode).  Process-wide, like the in-memory cubin cache it extends: call it once at
 * start-up.  `dir` must be an existing directory; NULL or "" turns the disk cache off, which is the default.  A bad
 * `dir` returns MDN_ERR_INVALID_ARG with the reason in mdn_last_error(NULL).  The setting applies to later cubins the
 * process has not compiled or read yet.
 * Each cubin is <dir>/<key>.cubin, the key a BLAKE3 digest of the file format version, the NVRTC version, the
 * compile options (MDN_JIT_PTXAS applied) and the generated source, so a changed program, generator, chunk size
 * (MDN_JIT_CHUNK) or NVRTC gives a new file.  A file that fails its header, size or BLAKE3 check is ignored, and the
 * cubin is compiled and the file replaced; a file is written through a temporary file and rename(2), so concurrent
 * processes leave one whole file; a failed write (read-only directory, full disk) is counted and is not an error.
 * mdn_get_info(NULL, MDN_INFO_JIT_CACHE) counts all of this.
 * Trust: the BLAKE3 check detects corruption, not a hostile writer.  The files are loaded as GPU code, so only trusted
 * users may be able to write to `dir`.  Each kernel, fresh or read from disk, is still compared with the interpreter on
 * its first use in each session. */
int mdn_jit_set_cache_dir(const char* dir);
/* Copies at most cap u64 into out; returns the number of u64 available (or <0).  s may be NULL only for
 * MDN_INFO_JIT_CACHE. */
long long mdn_get_info(mdn_session* s, mdn_info what, uint64_t* out, size_t cap);

/* Per-phase device timings of the last prove, in milliseconds (CUDA events on the session's
 * stream).  Names follow the reference's tracing spans (prover/mod.rs:339,412,445,542,561). */
typedef struct {
    float h2d_transpose, commit_main, commit_aux, evaluate_constraints, commit_quotient, open, total;
    float lde_main, hash_main;          /* inside commit_main */
    /* per kernel class, summed over the last prove's launches (CUDA events on the session stream):
     * 0 transpose (or the ingest of column-major device traces), 1 NTT/LDE, 2 leaf sponge, 3 Merkle compress, 4 constraints, 5 OOD dot products,
     * 6 DEEP quotient, 7 FRI (leaf+compress+fold), 8 PoW grind, 9 opening gather.  The constraint guard's row check (and
     * the re-derivation of the preprocessed rows it reads) is one more region of class 4 and is inside commit_aux. */
    float kernel_ms[10];
    unsigned kernel_regions[10];        /* timed regions per class */
    unsigned long long kernel_launches; /* kernels launched by the last prove */
    unsigned long long permutations;    /* Poseidon2 permutations executed for commitments */
    double leaf_hash_bytes;             /* algorithmic bytes of the leaf-sponge launches (LDE read + state/digest write) */
    double ntt_bytes;                   /* algorithmic bytes of the LDE: (N + L) * width * 8 per matrix */
} mdn_timings;
int mdn_get_timings(mdn_session* s, mdn_timings* out);

#ifdef __cplusplus
}
#endif
#endif /* MIDEN_B200_H */
