/* sp1b200.h — C ABI of the H100-native SP1 (Hypercube, v6) core-shard prover hot path.
 *
 * This is the drop-in boundary: a Rust shim implementing `sp1_hypercube::prover::AirProver`
 * (reference: crates/hypercube/src/prover/shard.rs:45-101), selected through
 * `SP1ProverComponents::CoreProver` (crates/prover/src/components.rs:148-198), binds these symbols the way
 * sp1-gpu's own FFI binds its kernels (sp1-gpu/crates/sys/src/runtime.rs:5-20,151-158).  See INTEGRATION.md.
 *
 * Conventions (mirroring the reference FFI):
 *  - every fallible call returns NULL on success or a NUL-terminated message owned by the library
 *    (valid until the next call on the same thread)            [CudaRustError, sys/src/runtime.rs:5-20]
 *  - field elements are u32 KoalaBear Montgomery words (R = 2^32), byte-compatible with p3's KoalaBear;
 *    extension elements are 4 consecutive words; digests are 8 words   [kb31_t.cuh:76-85, kb31_extension_t.cuh:6-63]
 *  - matrices are column-major: column c occupies [c*height, (c+1)*height)      [sp1-gpu/crates/utils/src/traces.rs:48-75]
 *  - pointers named `*_any` may be host or device pointers (resolved with cudaPointerGetAttributes);
 *    `d_*` must be device pointers, `h_*` host pointers
 *  - all work is enqueued on the context's stream; calls that return data to the host synchronise it
 *  - the Fiat-Shamir challenger crosses the boundary as 34 words: sponge[16] input[8] output[8] n_in n_out
 *    (same struct the reference ships to the device, sys/include/challenger/challenger.cuh:13-60)
 */
#ifndef SP1B200_H
#define SP1B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sp1b200_ctx sp1b200_ctx;
typedef const char* sp1b200_err; /* NULL == ok */

/* protocol parameters: crates/prover/src/components.rs:16-17, crates/primitives/src/fri_params.rs:5-58,
 * slop/crates/basefold/src/verifier.rs:16, crates/hypercube/src/verifier/shard.rs:41 */
typedef struct sp1b200_params {
    uint32_t log_stacking_height; /* 21 */
    uint32_t max_log_row_count;   /* 22 */
    uint32_t log_blowup;          /* 2  */
    uint32_t num_queries;         /* 124 */
    uint32_t pow_bits;            /* 16 */
    uint32_t batch_pow_bits;      /* 5  */
    uint32_t gkr_pow_bits;        /* 12 */
    uint32_t grind_mode;          /* 0 = canonical-min witness (deterministic), 1 = replay supplied witnesses */
} sp1b200_params;

#define SP1B200_CHALLENGER_WORDS 34
#define SP1B200_DIGEST_WORDS 8

/* ---- context / runtime (replaces sp1-gpu/crates/cuda TaskScope + sys/lib/runtime/{all}.cu) ---------------- */
sp1b200_err sp1b200_ctx_create(int device, const sp1b200_params* params, sp1b200_ctx** out);
void sp1b200_ctx_destroy(sp1b200_ctx* ctx);
sp1b200_err sp1b200_ctx_sync(sp1b200_ctx* ctx);
void sp1b200_default_core_params(sp1b200_params* out);
const char* sp1b200_version(void);
/* raw cudaStream_t of the context (so a host runtime can order its own copies against it) */
void* sp1b200_ctx_stream(sp1b200_ctx* ctx);
/* stream-ordered device memory (replaces cuda_malloc_async / cuda_free_async, sys/lib/runtime/memory.cu) */
sp1b200_err sp1b200_malloc(sp1b200_ctx* ctx, size_t bytes, void** d_out);
sp1b200_err sp1b200_free(sp1b200_ctx* ctx, void* d_ptr);
sp1b200_err sp1b200_memcpy_h2d(sp1b200_ctx* ctx, void* d_dst, const void* h_src, size_t bytes);
sp1b200_err sp1b200_memcpy_d2h(sp1b200_ctx* ctx, void* h_dst, const void* d_src, size_t bytes);
/* Row-major chip traces -> the dense column-major layout every commit / prove entry point takes (TraceDenseData,
 * sp1-gpu/crates/utils/src/traces.rs:48-75).  The reference's CPU trace generator yields one row-major [rows x cols] matrix
 * per chip (crates/hypercube/src/prover/trace.rs:126-201) and its GPU prover transposes on the device; this is that step.
 * rows_any: the tables back to back, each row-major (host or device); d_dense_out: device buffer of the same total size, tables
 * back to back, each column-major. */
sp1b200_err sp1b200_pack_row_major(sp1b200_ctx* ctx, const uint32_t* rows_any, uint32_t n_tables, const uint64_t* rows,
                                   const uint64_t* cols, uint32_t* d_dense_out);
/* Double-buffered asynchronous upload (replaces the host->device trace transfer the reference does per shard in
 * sp1-gpu/crates/jagged_tracegen: traces of shard k+1 are moved while shard k is proven).  Copies n_words words from
 * (ideally pinned) host memory into library-owned slot 0 or 1 on a separate copy stream and returns the slot's device
 * pointer; pass that pointer as main_dense_any to sp1b200_prove_shard / sp1b200_jagged_commit, which wait for the copy in
 * stream order.  The slot is reused only after its previous consumer finished. */
sp1b200_err sp1b200_upload_begin(sp1b200_ctx* ctx, const uint32_t* h_src, uint64_t n_words, int slot, uint32_t** d_out);
/* number of kernels this library has launched on ctx since creation (bench.py's gpu_launches) */
uint64_t sp1b200_launch_count(sp1b200_ctx* ctx);
/* device time in ms of the most recent call of the named phase ("rs_encode", "leaf_hash", "compress", ...),
 * measured with CUDA events on the context stream; -1 if unknown */
float sp1b200_last_phase_ms(sp1b200_ctx* ctx, const char* phase);

/* ---- kernel-level entry points (replace the per-kernel FFI of sp1-gpu/crates/sys/src/{all}.rs) ------------- */

/* Poseidon2 permutation of n independent 16-word states (poseidon2.cuh:46-80). */
sp1b200_err sp1b200_poseidon2_permute(sp1b200_ctx* ctx, uint32_t* states_any, uint64_t n);

/* Reed-Solomon encode: per column zero-pad x 2^log_blowup, forward DFT, rows bit-reversed
 * (replaces batch_coset_dft, sys/include/ntt/sppark.cuh:49-107; semantics slop/crates/dft/src/p3.rs:11-48).
 * msg: [ncols x 2^log_h], out: [ncols x 2^(log_h+log_blowup)], both column-major. */
sp1b200_err sp1b200_rs_encode(sp1b200_ctx* ctx, const uint32_t* msg_any, uint64_t ncols, uint32_t log_h,
                              uint32_t log_blowup, uint32_t* out_any);

/* Merkle tensor commitment of a column-major [width x 2^log_h] matrix: leaf i = sponge(row i), binary
 * compress layers, commitment = compress(root, hash([log_h, width]))
 * (replaces leafHashPacked/compress, sys/lib/merkle_tree/merkle_tree.cu:27-94; semantics
 * slop/crates/merkle-tree/src/p3sync.rs:40-143).  d_layers_out (optional, device): all 2^(log_h+1)-1 digests,
 * bottom-up (layer k of 2^(log_h-k) digests after layers 0..k-1).  root/commit: 8 words each, host. */
sp1b200_err sp1b200_merkle_commit(sp1b200_ctx* ctx, const uint32_t* mat_any, uint64_t width, uint32_t log_h,
                                  uint32_t* d_layers_out, uint32_t* h_root8, uint32_t* h_commit8);

/* Proof-of-work grind on a challenger state (replaces grindKernel, sys/include/challenger/challenger.cuh:114-158;
 * semantics p3 DuplexChallenger::grind).  Returns the MINIMUM canonical witness (deterministic) and leaves
 * `state` in the post-check_witness state (sp1-gpu/crates/challenger/src/grinding_challenger.rs:70-74). */
sp1b200_err sp1b200_grind(sp1b200_ctx* ctx, uint32_t* h_state34, uint32_t bits, uint32_t* h_witness);

/* Host-side transcript helpers on the 34-word state (no device work; semantics challenger.cuh:22-112,
 * slop/crates/challenger/src/lib.rs:54-82).  Provided so a shim can keep its challenger in this format. */
void sp1b200_challenger_init(uint32_t* h_state34);
void sp1b200_challenger_observe(uint32_t* h_state34, const uint32_t* h_vals, uint64_t n);
void sp1b200_challenger_sample(uint32_t* h_state34, uint32_t* h_out, uint64_t n);
uint32_t sp1b200_challenger_sample_bits(uint32_t* h_state34, uint32_t bits);
int sp1b200_challenger_check_witness(uint32_t* h_state34, uint32_t bits, uint32_t witness);

/* ---- PCS-level entry points (replace sp1-gpu/crates/{commit,basefold}) -------------------------------- */

typedef struct sp1b200_commit sp1b200_commit; /* device-resident prover data of one commitment round */

/* Stacked-PCS commit of a dense buffer already laid out as [ncols x 2^log_stacking_height] column-major
 * (zero padding applied by the caller or by sp1b200_jagged_commit): RS-encode + Merkle commit
 * (slop/crates/stacked/src/prover.rs:59-94 -> basefold-prover/src/prover.rs:78-99).
 * keep_codeword != 0 keeps the 2^log_blowup x larger codeword resident for the query phase; otherwise it is
 * recomputed on demand (the reference's drop_ldes, sp1-gpu/crates/basefold/src/fri.rs:333-359). */
sp1b200_err sp1b200_stacked_commit(sp1b200_ctx* ctx, const uint32_t* dense_any, uint64_t ncols, int keep_codeword,
                                   uint32_t* h_commit8, sp1b200_commit** out);
void sp1b200_commit_free(sp1b200_ctx* ctx, sp1b200_commit* c);

/* Stacked-PCS + BaseFold evaluation proof at `point` (n_point ext elements, the last log_stacking_height of
 * which are the stack point) over `n_rounds` commitment rounds
 * (slop/crates/stacked/src/prover.rs:111-160 -> basefold-prover/src/prover.rs:102-270).
 * h_replay_witnesses: {batch_grinding_witness, pow_witness} when params.grind_mode == 1, else NULL.
 * Proof is written as flat words in the field order of StackedBasefoldProof/BasefoldProof
 * (slop/crates/stacked/src/verifier.rs:27-31, slop/crates/basefold/src/verifier.rs:97-116):
 *   univariate_messages[d][2] ext | fri_commitments[d] digest | per commit round {values[q][ncols], root, log_height,
 *   width, paths[q][log_height] digest} | per fold round {values[q][8], root, log_height, width, paths} |
 *   final_poly ext | pow_witness | batch_grinding_witness | batch_evaluations[round][ncols] ext.
 * *h_proof_words receives the number of words; returns an error if proof_cap_words is too small. */
sp1b200_err sp1b200_stacked_prove(sp1b200_ctx* ctx, sp1b200_commit* const* rounds, uint32_t n_rounds,
                                  const uint32_t* h_point, uint32_t n_point, const uint32_t* h_replay_witnesses,
                                  uint32_t* h_challenger34, uint32_t* h_proof, uint64_t proof_cap_words,
                                  uint64_t* h_proof_words);

/* ---- jagged PCS (replaces sp1-gpu/crates/{jagged_sumcheck,jagged_assist} + the jagged part of shard_prover) -------- */

typedef struct sp1b200_jagged_round sp1b200_jagged_round; /* one commitment round: tables, dense buffer, stacked data */

/* JaggedProver::commit_multilinears (slop/crates/jagged/src/prover.rs:106-160) for one round of chip tables.
 * dense_any: the tables' real cells back to back in table order, each table column-major [cols x rows]
 * (tables with rows == 0 contribute no data but do enter the row/column counts), host or device memory; this is the
 * reference's TraceDenseData layout (sp1-gpu/crates/utils/src/traces.rs:48-75).  The library keeps its own copy,
 * zero-padded to a multiple of 2^log_stacking_height, appends the two dummy tables to the counts and returns
 * commit = compress(stacked_commit, hash(n, rows.., cols..)). */
sp1b200_err sp1b200_jagged_commit(sp1b200_ctx* ctx, const uint32_t* dense_any, uint32_t n_tables, const uint64_t* h_rows,
                                  const uint64_t* h_cols, int keep_codeword, uint32_t* h_commit8, sp1b200_jagged_round** out);
void sp1b200_jagged_round_free(sp1b200_ctx* ctx, sp1b200_jagged_round* round);

/* Evaluations at z_row (max_log_row_count ext elements) of every table column of the round, zero-extended to
 * 2^max_log_row_count rows: the per-column claims zerocheck hands to the PCS
 * (crates/hypercube/src/prover/shard.rs:736-767).  h_out: sum(cols) ext elements in table/column order. */
sp1b200_err sp1b200_jagged_column_claims(sp1b200_ctx* ctx, const sp1b200_jagged_round* round, const uint32_t* h_z_row,
                                         uint32_t* h_out);

/* JaggedProver::prove_trusted_evaluations (slop/crates/jagged/src/prover.rs:162-328): sample z_col, Hadamard sumcheck
 * of the dense trace against the jagged little polynomial, branching-program evaluation sumcheck, stacked/BaseFold
 * proof at the sumcheck point.  h_claims: per round, that round's column claims back to back (ext each).
 * Proof words (field order of JaggedPcsProof, slop/crates/jagged/src/verifier.rs:17-27):
 *   stacked proof (see sp1b200_stacked_prove) | sumcheck {n_polys, per poly {n_coeffs, coeffs ext}, claimed_sum ext,
 *   point ext[n_polys], eval ext} | jagged_eval (same layout) | per round {n_tables, (rows, cols) per table} |
 *   original commitments digest[n_rounds] | expected_eval ext | max_log_row_count | log_m */
sp1b200_err sp1b200_jagged_prove(sp1b200_ctx* ctx, sp1b200_jagged_round* const* rounds, uint32_t n_rounds,
                                 const uint32_t* h_z_row, const uint32_t* h_claims, const uint32_t* h_replay_witnesses,
                                 uint32_t* h_challenger34, uint32_t* h_proof, uint64_t proof_cap_words,
                                 uint64_t* h_proof_words);

/* ---- zerocheck (replaces sp1-gpu/crates/zerocheck + sys/lib/zerocheck/{all}.cu) ------------------------------------ */

typedef struct sp1b200_machine sp1b200_machine; /* the machine's AIR constraints, uploaded once */

/* Upload the constraint bytecode of every chip (replaces upload_machine_bytecode, sp1-gpu/crates/zerocheck/src/prover.rs).
 * The instruction set and record layouts are the reference GPU prover's (sys/include/zerocheck/sequential.cuh:13-49):
 *   DagInstr {u8 opcode, u8 pad, u16 out, u16 a, u16 b}, LeafRef {u8 source(2 = preprocessed, 4 = main), u8 pad, u16 pad, u32 col},
 *   opcodes LOAD_LEAF 0, LOAD_CONST 1, LOAD_PUBLIC 2, ADD 3, SUB 4, MUL 5, NEG 6; asserts = (register, alpha index) pairs
 *   with alpha index i <-> alpha^(n_constraints-1-i) (Horner order of the verifier folder).
 * Blob words: [n_chips] then per chip (chips in BTreeSet/name order):
 *   main_w prep_w n_constraints n_regs n_instrs n_leaves n_consts n_publics n_asserts,
 *   instrs (2 words each), leaves (2 words each), consts (Montgomery), publics (indices), assert_regs, assert_alphas. */
sp1b200_err sp1b200_machine_create(sp1b200_ctx* ctx, const uint32_t* h_blob, uint64_t n_words, sp1b200_machine** out);
void sp1b200_machine_free(sp1b200_ctx* ctx, sp1b200_machine* machine);
uint32_t sp1b200_machine_num_chips(const sp1b200_machine* machine);
/* diagnostic: peak number of live registers of a chip's re-scheduled constraint program (selects the register-file tier of the
 * zerocheck kernels: <= 32 shared memory, <= 128 local memory, <= 1024 global-memory workspace - the reference's largest tier,
 * sys/lib/zerocheck/sequential.cu:298-335; more is rejected by sp1b200_zerocheck); 0 if chip is out of range */
uint32_t sp1b200_machine_chip_regs(const sp1b200_machine* machine, uint32_t chip);

/* ShardProver::zerocheck (crates/hypercube/src/prover/shard.rs:474-646): samples lambda, runs the max_log_row_count-round
 * sumcheck over all chips (round polynomial through nodes {0,1,2,4,b}, crates/hypercube/src/prover/zerocheck/sum_as_poly.rs:187-287),
 * observes and returns the opened values.  d_main[k]/d_prep[k]: device pointers to chip k's columns, column-major
 * [w x h_heights[k]] (d_prep[k] may be NULL when the chip has no preprocessed columns); h_alpha/h_gamma: the two ext
 * challenges the caller sampled after LogUp-GKR (shard.rs:707-709); h_claims: per chip sum_j gamma^(j+1) * opening_j
 * (main columns then preprocessed) of the LogUp-GKR openings at h_gkr_point.
 * Output words: sumcheck proof {n_polys, per poly {n_coeffs, coeffs ext}, claimed_sum, point, eval} |
 *               per chip {preprocessed evaluations ext[prep_w], main evaluations ext[main_w]} at the sumcheck point. */
sp1b200_err sp1b200_zerocheck(sp1b200_ctx* ctx, const sp1b200_machine* machine, const uint64_t* h_heights,
                              const uint32_t* const* d_main, const uint32_t* const* d_prep, const uint32_t* h_public_values,
                              uint32_t n_public_values, const uint32_t* h_gkr_point, const uint32_t* h_alpha,
                              const uint32_t* h_gamma, const uint32_t* h_claims, uint32_t* h_challenger34, uint32_t* h_out,
                              uint64_t out_cap_words, uint64_t* h_out_words);

/* ---- LogUp-GKR (replaces sp1-gpu/crates/logup_gkr + sys/lib/logup_gkr/{all}.cu) ---------------------------------------- */

/* The machine blob of sp1b200_machine_create may carry an interactions section after the AIR records
 * (crates/hypercube/src/lookup/interaction.rs:11-22; VirtualPairCol = sum weight * column + constant):
 *   per chip: [n_interactions] then per interaction (sends first, then receives):
 *     is_send arg_index(InteractionKind) n_values, multiplicity vcol, n_values value vcols
 *   vcol: n_terms constant(Montgomery) { source(2 = preprocessed, 4 = main) col weight(Montgomery) } x n_terms */

/* GkrProverImpl::prove_logup_gkr (crates/hypercube/src/logup_gkr/prover.rs:70-215): grind(gkr_pow_bits), sample alpha / beta seed,
 * build the fraction-sum circuit over the row variables, observe the circuit output, prove max_log_row_count-1 layers
 * (logup_poly.rs:230-552), open every chip column at the final trace point.
 * Output words: n_out | numerator ext[n_out] | denominator ext[n_out] | n_rounds | per round {numerator_0 numerator_1
 *   denominator_0 denominator_1 ext, sumcheck {n_polys, per poly {n_coeffs, coeffs}, claimed_sum, point, eval}} |
 *   evaluation point ext[max_log_row_count] | per chip {main openings ext[main_w], preprocessed openings ext[prep_w]} | witness */
sp1b200_err sp1b200_logup_gkr(sp1b200_ctx* ctx, const sp1b200_machine* machine, const uint64_t* h_heights,
                              const uint32_t* const* d_main, const uint32_t* const* d_prep, const uint32_t* h_replay_witness,
                              uint32_t* h_challenger34, uint32_t* h_out, uint64_t out_cap_words, uint64_t* h_out_words);

/* ---- whole shard (the AirProver::prove_shard_with_pk body; replaces CudaShardProver::prove_shard_with_data,
 *      sp1-gpu/crates/shard_prover/src/prover.rs:618-763) -------------------------------------------------------------- */

/* ShardProver::prove_shard_with_data (crates/hypercube/src/prover/shard.rs:650-792): observe public values, commit the main
 * traces, observe the commitment and every chip's (height, name), LogUp-GKR, sample alpha and gamma, zerocheck, jagged
 * evaluation proof at the zerocheck point over {preprocessed round, main round}.
 * machine: chips in BTreeSet (name) order; prep_round: the preprocessed commitment made at setup with
 * sp1b200_jagged_commit over the chips with preprocessed columns (NULL if the machine has none; heights must equal the
 * main heights, as the reference verifier requires, verifier/shard.rs:690-720); main_dense_any: main tables back to back
 * (TraceDenseData layout); chip_names: NUL-terminated names in chip order; h_challenger34: the transcript after the
 * verifying key has been observed (crates/hypercube/src/verifier/config.rs:97-112), updated in place.
 * h_replay_witnesses (grind_mode == 1): {gkr, batch grinding, pow}.
 * Proof words: [5][len_0..len_4] then  main commitment (8) | LogUp-GKR (sp1b200_logup_gkr words) | zerocheck + opened values
 * (sp1b200_zerocheck words) | evaluation proof (sp1b200_jagged_prove words) | public values
 * = the fields of ShardProof (crates/hypercube/src/verifier/proof.rs:47-61). */
sp1b200_err sp1b200_prove_shard(sp1b200_ctx* ctx, const sp1b200_machine* machine, sp1b200_jagged_round* prep_round,
                                const uint32_t* main_dense_any, const uint64_t* h_heights, const char* const* chip_names,
                                const uint32_t* h_public_values, uint32_t n_public_values, const uint32_t* h_replay_witnesses,
                                uint32_t* h_challenger34, uint32_t* h_proof, uint64_t proof_cap_words, uint64_t* h_proof_words);

/* AirProver::setup_and_prove_shard (crates/hypercube/src/prover/shard.rs:56-68), the vk-less path: setup (commit the preprocessed
 * traces = the device part of the proving key), observe the verifying key, prove the shard.
 * prep_dense_any / h_prep_rows / h_prep_cols (n_prep tables): as sp1b200_jagged_commit, the tables of the chips with preprocessed columns
 * in chip order.  The verifying key enters a FRESH transcript the way MachineVerifyingKey::observe_into does
 * (crates/hypercube/src/verifier/config.rs:97-112): the preprocessed commitment (8 words, produced here) followed by h_vk_tail - the
 * words the shim builds from the program: pc_start[3], initial_global_cumulative_sum x[7] y[7], enable_untrusted_programs, six zero
 * padding words - so h_challenger34 is the state BEFORE the key is observed (sp1b200_challenger_init for a new proof).
 * h_prep_commit8 receives the commitment (MachineVerifyingKey::preprocessed_commit); *prep_round_out receives the committed round
 * (keep it for later sp1b200_prove_shard calls of the same program, free it with sp1b200_jagged_round_free).  Everything else as
 * sp1b200_prove_shard. */
sp1b200_err sp1b200_setup_and_prove_shard(sp1b200_ctx* ctx, const sp1b200_machine* machine, const uint32_t* prep_dense_any, uint32_t n_prep,
                                          const uint64_t* h_prep_rows, const uint64_t* h_prep_cols, const uint32_t* h_vk_tail,
                                          uint32_t n_vk_tail, const uint32_t* main_dense_any, const uint64_t* h_heights,
                                          const char* const* chip_names, const uint32_t* h_public_values, uint32_t n_public_values,
                                          const uint32_t* h_replay_witnesses, uint32_t* h_challenger34, uint32_t* h_prep_commit8,
                                          sp1b200_jagged_round** prep_round_out, uint32_t* h_proof, uint64_t proof_cap_words,
                                          uint64_t* h_proof_words);

/* ---- shard checks (the reference's cfg(sp1_debug_constraints) build; nothing of the transcript is touched) -------------------------
 * Both take the shard inputs of sp1b200_prove_shard (same validation: prep_round = the round committed at setup or NULL, its heights
 * equal to the main heights, every height <= 2^max_log_row_count; main_dense_any = host pointer, device pointer or upload slot), so a
 * shim can call them right before proving.  A failing check is not an error: the call returns NULL and writes the report.  Errors
 * are malformed input and out_cap_words too small (*h_out_words then holds the size needed; the context stays usable).  Every
 * device allocation comes from the context's pool and is returned before the call ends.  Field words are Montgomery words. */

/* debug_constraints_all_chips (crates/hypercube/src/debug.rs:27-130): every real row 0 .. h-1 of every chip (height 0 = skipped)
 * through the chip's constraints in the base field, over main columns, preprocessed columns and public values.  A constraint is
 * named by its assert's alpha index (alpha index i <-> alpha^(n_constraints-1-i): the constraint's position in the chip's eval order).
 * Report words: n_failing_chips | per failing chip, ascending: chip | n_failing_rows | n_listed = min(n_failing_rows,
 * max_rows_per_chip) | per listed row (the lowest failing rows, ascending): row | n_failed | failed constraint indices, ascending. */
sp1b200_err sp1b200_debug_constraints(sp1b200_ctx* ctx, const sp1b200_machine* machine, sp1b200_jagged_round* prep_round,
                                      const uint32_t* main_dense_any, const uint64_t* h_heights, const uint32_t* h_public_values,
                                      uint32_t n_public_values, uint32_t max_rows_per_chip, uint32_t* h_out, uint64_t out_cap_words,
                                      uint64_t* h_out_words);

/* debug_interactions_with_all_chips (crates/hypercube/src/lookup/debug.rs:48-200): over rows 0 .. h-1 and the (row, interaction)
 * pairs with a non-zero multiplicity, the net multiplicity (sends - receives, in F) of every distinct key (kind = arg_index,
 * n_values, values); a key is unbalanced when its net is not zero.  Keys are listed in order of first occurrence, records ranked by
 * (chip, row, interaction index in the blob: sends, then receives); the chip list holds every chip with a record of the key.
 * Report words: n_unbalanced (u64: lo, hi) | n_listed = min(n_unbalanced, max_keys) | per listed key: kind | n_values |
 * values[n_values] | net | first chip | first interaction index | first row | n_chips | per chip, ascending: chip | net. */
sp1b200_err sp1b200_debug_interactions(sp1b200_ctx* ctx, const sp1b200_machine* machine, sp1b200_jagged_round* prep_round,
                                       const uint32_t* main_dense_any, const uint64_t* h_heights, uint32_t max_keys, uint32_t* h_out,
                                       uint64_t out_cap_words, uint64_t* h_out_words);

/* ---- ShardProof wire format (SURVEY 8f.4) ----------------------------------------------------------------------------------------
 * The reference moves shard proofs between prover workers, the recursion tree and the verifier as bincode(ShardProof)
 * (crates/hypercube/src/verifier/proof.rs:47-61 and the nested types listed in csrc/wire.cu; bincode 1.3 default configuration:
 * little endian, fixed-width integers, u64 lengths, Option tag u8).  Field elements travel as CANONICAL u32 words (pinned by the
 * reference-held crates/prover/src/vk_map_dummy.bin, tests/golden/bincode_pins.json), extension elements as 4 of them, chip maps in
 * name order with the names as strings, chip heights as the `degree` bit points.  Host-only calls: no context, no device work.
 * n_chips / chip_names (strictly ascending) / h_main_w / h_prep_w describe the shard's chips (the machine passed to sp1b200_prove_shard). */

/* flat words of sp1b200_prove_shard -> bincode(ShardProof).  h_out may be NULL to query *h_out_bytes. */
sp1b200_err sp1b200_shard_proof_to_bincode(const sp1b200_params* params, uint32_t n_chips, const char* const* chip_names,
                                           const uint64_t* h_heights, const uint32_t* h_main_w, const uint32_t* h_prep_w,
                                           const uint32_t* h_proof, uint64_t n_words, uint8_t* h_out, uint64_t cap_bytes,
                                           uint64_t* h_out_bytes);
/* bincode(ShardProof) -> flat words; every length prefix, tensor dimension, chip name / width and the canonical range of every field
 * element is checked.  h_heights_out (n_chips, optional) receives the heights decoded from the degree points; h_proof may be NULL to
 * query *h_words. */
sp1b200_err sp1b200_shard_proof_from_bincode(const sp1b200_params* params, uint32_t n_chips, const char* const* chip_names,
                                             const uint32_t* h_main_w, const uint32_t* h_prep_w, const uint8_t* h_bytes, uint64_t n_bytes,
                                             uint64_t* h_heights_out, uint32_t* h_proof, uint64_t cap_words, uint64_t* h_words);

/* ---- shard verifier (ShardVerifier::verify_shard, crates/hypercube/src/verifier/shard.rs:437-750) ---------------------------------
 * Checks the flat words of sp1b200_prove_shard against the machine, the chip heights and names and the context's parameters
 * (log_stacking_height, max_log_row_count, log_blowup, num_queries and the three PoW bit counts) the prover used.
 * h_prep_commit8: the verifying key's preprocessed commitment (NULL when no chip has preprocessed columns).  h_challenger34: the
 * transcript after the caller observed the verifying key (the state sp1b200_prove_shard starts from).  Heights come from the caller:
 * the flat words do not carry the proof's `degree` points (sp1b200_shard_proof_from_bincode recovers them from bincode(ShardProof)).
 * Every Merkle opening, the BaseFold query fold chains and the jagged evaluation's column sum run on the device (context stream and
 * pool); the transcript, the PoW checks, the sumcheck rounds and the constraints at the zerocheck point run on the host.
 *
 * *h_verdict = SP1B200_VERDICT_ACCEPT: the proof is valid and h_challenger34 holds the verifier's final state (equal to the prover's).
 * Any other verdict rejects the proof and names the first failing check, in verify_shard's order; h_challenger34 is then left
 * unchanged.  A rejection is not an error.  Errors: the words do not parse as a proof of this machine's shape (section lengths,
 * counts beyond the layout's limits, opening heights other than the context's, trailing words, a field word >= p), malformed
 * arguments (a height >= 2^(max_log_row_count+1), a public value index beyond the proof's public values, NULL pointers), device
 * failures.  The context stays usable after a rejection or an error.
 * Not checked, as they need the Rust machine definition: the public-values length against PROOF_MAX_NUM_PVS, chip clusters, and the
 * machine-specific public-values interactions (the expected LogUp cumulative sum is 0). */
#define SP1B200_VERDICT_ACCEPT 0u
#define SP1B200_VERDICT_POW 1u                          /* "Pow": the LogUp-GKR or the BaseFold query grinding witness */
#define SP1B200_VERDICT_INVALID_SHAPE 2u                /* "InvalidShape": GKR output length, zerocheck rounds */
#define SP1B200_VERDICT_ZERO_DENOMINATOR 3u             /* "ZeroDenominator" */
#define SP1B200_VERDICT_CUMULATIVE_SUM_MISMATCH 4u      /* "CumulativeSumMismatch" */
#define SP1B200_VERDICT_INVALID_SHAPE_ROUNDS 5u         /* "InvalidShape(rounds)": GKR layer count */
#define SP1B200_VERDICT_INCONSISTENT_SUMCHECK_CLAIM 6u  /* "InconsistentSumcheckClaim": GKR layer claim */
#define SP1B200_VERDICT_SUMCHECK_PROOF_SHAPE 7u         /* "InvalidProofShape": a sumcheck's round count or degree */
#define SP1B200_VERDICT_SUMCHECK_CLAIMED_SUM 8u         /* "InconsistencyWithClaimedSum": a sumcheck's first round */
#define SP1B200_VERDICT_SUMCHECK_ROUND 9u               /* "SumcheckRoundInconsistency" */
#define SP1B200_VERDICT_SUMCHECK_POINT 10u              /* "InvalidProofShape(point)" */
#define SP1B200_VERDICT_SUMCHECK_EVAL 11u               /* "InconsistencyWithEval": a sumcheck's final evaluation */
#define SP1B200_VERDICT_INCONSISTENT_EVALUATION 12u     /* "InconsistentEvaluation": GKR layer evaluation */
#define SP1B200_VERDICT_LAST_LAYER_DIMENSION 13u        /* "InvalidLastLayerDimension" */
#define SP1B200_VERDICT_TRACE_POINT_MISMATCH 14u        /* "TracePointMismatch" */
#define SP1B200_VERDICT_INVALID_SHAPE_OPENINGS 15u      /* "InvalidShape(openings)" */
#define SP1B200_VERDICT_NUMERATOR_EVALUATION 16u        /* "NumeratorEvaluationMismatch" */
#define SP1B200_VERDICT_DENOMINATOR_EVALUATION 17u      /* "DenominatorEvaluationMismatch" */
#define SP1B200_VERDICT_OPENING_SHAPE 18u               /* "OpeningShape" */
#define SP1B200_VERDICT_HEIGHT_BITS 19u                 /* "InvalidHeightBitDecomposition" */
#define SP1B200_VERDICT_HEIGHT_TOO_LARGE 20u            /* "HeightTooLarge": a height above 2^max_log_row_count */
#define SP1B200_VERDICT_CONSTRAINTS_EVAL 21u            /* "ConstraintsCheckFailed(InconsistencyWithEval)" */
#define SP1B200_VERDICT_CONSTRAINTS_CLAIMED_SUM 22u     /* "ConstraintsCheckFailed(InconsistencyWithClaimedSum)" */
#define SP1B200_VERDICT_INCORRECT_SHAPE 23u             /* "IncorrectShape": jagged / stacked shapes */
#define SP1B200_VERDICT_INCORRECT_TABLE_SIZES 24u       /* "IncorrectTableSizes": row/column counts or commitments */
#define SP1B200_VERDICT_AREA_OUT_OF_BOUNDS 25u          /* "AreaOutOfBounds" */
#define SP1B200_VERDICT_DUMMY_TABLES 26u                /* "IncorrectShape(dummy tables)" */
#define SP1B200_VERDICT_SUMCHECK_CLAIM_MISMATCH 27u     /* "SumcheckClaimMismatch": jagged claim */
#define SP1B200_VERDICT_MONOTONICITY 28u                /* "MonotonicityCheckFailed" */
#define SP1B200_VERDICT_JAGGED_EVALUATION 29u           /* "JaggedEvaluationFailed" */
#define SP1B200_VERDICT_JAGGED_EVAL_PROOF 30u           /* "JaggedEvalProofVerificationFailed" */
#define SP1B200_VERDICT_STACKING 31u                    /* "StackingError" */
#define SP1B200_VERDICT_BATCH_POW 32u                   /* "BatchPow" */
#define SP1B200_VERDICT_FRI_LENGTH 33u                  /* "SumcheckFriLengthMismatch" */
#define SP1B200_VERDICT_BASEFOLD_SUMCHECK 34u           /* "Sumcheck": a BaseFold univariate message */
#define SP1B200_VERDICT_TWO_ADICITY 35u                 /* "TwoAdicityOverflow" */
#define SP1B200_VERDICT_TCS_COMPONENT 36u               /* "TcsError(component)": a commitment round's opening */
#define SP1B200_VERDICT_QUERY_VALUE 37u                 /* "QueryValueMismatch" */
#define SP1B200_VERDICT_TCS_QUERY 38u                   /* "TcsError(query)": a fold round's opening */
#define SP1B200_VERDICT_QUERY_FINAL_POLY 39u            /* "QueryFinalPolyMismatch" */
#define SP1B200_VERDICT_SUMCHECK_FINAL_POLY 40u         /* "SumcheckFinalPolyMismatch" */
#define SP1B200_VERDICT_PREPROCESSED_WIDTHS 41u         /* "InvalidShape(preprocessed widths)": the preprocessed round's leading
                                                           column counts differ from the chips' preprocessed widths (shard.rs:506-523) */
#define SP1B200_VERDICT_CHIP_TABLES 42u                 /* "InvalidShape(chip tables)": a round's table row counts differ from the
                                                           chip heights or its column counts from the chip widths (shard.rs:662-742) */
sp1b200_err sp1b200_verify_shard(sp1b200_ctx* ctx, const sp1b200_machine* machine, const uint32_t* h_prep_commit8,
                                 const uint64_t* h_heights, const char* const* chip_names, const uint32_t* h_proof, uint64_t n_words,
                                 uint32_t* h_challenger34, uint32_t* h_verdict);
/* the name of a verdict code (the reason string above; "Accepted" for 0, "Unknown" beyond the list) */
const char* sp1b200_verdict_name(uint32_t verdict);

#ifdef __cplusplus
}
#endif
#endif /* SP1B200_H */
