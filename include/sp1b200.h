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

/* Alignment of caller device buffers: the Poseidon2 states of sp1b200_poseidon2_permute, the output of sp1b200_rs_encode and the
 * d_layers_out digests of sp1b200_merkle_commit are read or written with 16-byte vector accesses, so a device pointer passed there
 * must be 16-byte aligned.  A pointer from sp1b200_malloc or cudaMalloc (256-byte aligned), or one a multiple of 4 words into
 * such a buffer, is. */

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

/* ---- program setup (the part of AirProver::setup that depends on the program, crates/hypercube/src/prover/shard.rs:259-290) --------
 * MachineProgram::pc_start + initial_global_cumulative_sum + untrusted_config for a core program (crates/core/executor/src/program.rs:
 * 161-229), as the 24-word vk_tail that sp1b200_setup_and_prove_shard, sp1b200_verify_core_proof and sp1b200_vk_hash take:
 *   pc_start = the 16-bit limbs 0..16 / 16..32 / 32..48 of pc_start_abs | initial_global_cumulative_sum x[7] y[7] |
 *   enable_untrusted_programs | 6 zeros (Montgomery words).
 * The sum is SepticDigest::zero() plus the negation of SepticCurve::lift_x of one message per memory entry (address mem_addrs_any[i],
 * word mem_words_any[i]: [Memory << 24, 0, address limbs 0..16 / 16..32 / 32..48, (w & 0xFFFF) + 2^16 ((w >> 32) & 0xFF),
 * ((w >> 16) & 0xFFFF) + 2^16 ((w >> 40) & 0xFF), w >> 48]) and, only when enable_untrusted_programs is 1, one per page entry (index
 * page_idx_any[i], protection page_prot_any[i]: [PageProtAccess << 24, 0, index bits 0..4 / 4..20 / 20..36, prot, 0, 0]), summed under
 * the complete addition law; with enable_untrusted_programs 0 the page image is not read.  An empty image gives SepticDigest::zero().
 * The arrays are host or device memory; device memory comes from the context's pool and is returned before the call ends.
 * Errors: a duplicate memory address or page index (the image is a map; the message names the key), an entry none of whose 256 lift
 * offsets gives a point, a sum at infinity, NULL arrays with a non-zero count, enable_untrusted_programs other than 0 or 1, 2^31 - 1
 * entries or more.  The context stays usable after an error.  Phases: "program_vk_tail", "program_vk_tail.lift", ".sum". */
sp1b200_err sp1b200_program_vk_tail(sp1b200_ctx* ctx, uint64_t pc_start_abs, const uint64_t* mem_addrs_any, const uint64_t* mem_words_any,
                                    uint64_t n_mem, const uint64_t* page_idx_any, const uint8_t* page_prot_any, uint64_t n_pages,
                                    int enable_untrusted_programs, uint32_t* h_vk_tail24);

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
 * Not checked, as they need the Rust machine definition: chip clusters and the machine-specific public-values interactions (the expected
 * LogUp cumulative sum is 0).  The public-values length against PROOF_MAX_NUM_PVS and the checks across shards are made by
 * sp1b200_verify_core_proof. */
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
/* the name of a verdict code of sp1b200_verify_shard or sp1b200_verify_core_proof (the reason strings; "Accepted" for 0, "Unknown"
 * beyond the lists) */
const char* sp1b200_verdict_name(uint32_t verdict);

/* ---- core-proof verifier (SP1Prover::verify, crates/prover/src/verify.rs:109-524) --------------------------------------------------
 * Verifies a core proof: the n_shards flat proofs (sp1b200_prove_shard words) of one execution, all of the same machine, chip names
 * and context parameters; h_heights[s * n_chips + k] = chip k's height in shard s.  The verifying key is h_prep_commit8 (always
 * observed; passed on to the shard checks only when a chip has preprocessed columns) followed by h_vk_tail, the words
 * sp1b200_setup_and_prove_shard takes: pc_start[3] | initial_global_cumulative_sum x[7] y[7] | enable_untrusted_programs | 6 zeros,
 * so n_vk_tail must be 24 (the build without mprotect).  Field words are Montgomery words.
 * Order of checks, as the reference's: every shard parses (else an error, as sp1b200_verify_shard); EmptyProof; the public values
 * across shards (PublicValues<[F;4],[F;3],[F;4],F> without mprotect: length PROOF_MAX_NUM_PVS = 187; one first execution shard;
 * timestamps from [0,0,0,1]; program counters from vk.pc_start to HALT_PC = [1,0,0]; exit codes; one proof nonce; memory
 * init/finalize addresses and page indices; committed-value and deferred-proof digests and commit-syscall flags); TooManyShards;
 * the global cumulative sum (vk.initial_global_cumulative_sum plus every shard's digest, one septic-curve SepticDigest addition per
 * shard, must be the zero digest); then every shard's verify_shard from a fresh transcript that observed the verifying key.
 * The one deviation from the reference: where an incomplete curve addition meets a zero denominator the reference panics; this
 * returns SP1B200_VERDICT_PV_EXCEPTIONAL_ADDITION.
 * *h_verdict: 0 accepts; otherwise the first failing check (names: sp1b200_verdict_name, "InvalidPublicValues(<reason>)" with the
 * reference's reason strings).  *h_shard: the shard at which the failing check's loop stopped; n_shards for the end-of-chain checks
 * (first execution shard not set, not halted, zero address never initialised / finalised, COMMIT syscalls never called,
 * TooManyShards, cumulative sum not zero); for InvalidShardProof the lowest failing shard, and *h_shard_verdict that shard's own
 * verify_shard code (0 for every other verdict; the two code spaces stay apart).  On accept h_final_challengers (optional,
 * [n_shards][34]) receives every shard verifier's final transcript state.
 * The shards' host phases run on host_threads threads (0 = the hardware concurrency); their device work runs in one launch per kernel
 * for each batch of consecutive shards with at most 2^26 proof words (the environment variable SP1B200_VERIFY_BATCH_WORDS can lower
 * the cap; batching never changes a verdict).  A rejection is not an error; the context stays usable after either. */
#define SP1B200_VERDICT_EMPTY_PROOF 43u                 /* EmptyProof: a core proof without shards */
#define SP1B200_VERDICT_TOO_MANY_SHARDS 44u             /* TooManyShards: 2^24 shards or more */
#define SP1B200_VERDICT_INVALID_SHARD_PROOF 45u         /* InvalidShardProof: *h_shard_verdict holds the shard's verify_shard code */
#define SP1B200_VERDICT_PV_LENGTH 46u                   /* invalid public values length */
#define SP1B200_VERDICT_PV_FIRST_SHARD_MULTIPLE 47u     /* is_first_execution_shard is set to one for multiple shards */
#define SP1B200_VERDICT_PV_FIRST_SHARD_NOT_BOOLEAN 48u  /* is_first_execution_shard is not boolean */
#define SP1B200_VERDICT_PV_FIRST_SHARD_NOT_SET 49u      /* first execution shard is not set */
#define SP1B200_VERDICT_PV_INITIAL_TIMESTAMP 50u        /* invalid initial timestamp */
#define SP1B200_VERDICT_PV_TIMESTAMP_UNCHANGED 51u      /* timestamp should change on execution shard */
#define SP1B200_VERDICT_PV_TIMESTAMP_CHANGED 52u        /* timestamp should not change on non-execution shard */
#define SP1B200_VERDICT_PV_PC_START_VK 53u              /* pc_start != vk.pc_start: ... */
#define SP1B200_VERDICT_PV_PC_START_PREV 54u            /* pc_start != prev_next_pc: ... */
#define SP1B200_VERDICT_PV_PC_NON_EXECUTION 55u         /* pc_start != next_pc: ... non-execution shards */
#define SP1B200_VERDICT_PV_NOT_HALTED 56u               /* next_pc != HALT_PC: execution should have halted */
#define SP1B200_VERDICT_PV_PREV_EXIT_CODE 57u           /* public_values.prev_exit_code != prev_exit_code: ... */
#define SP1B200_VERDICT_PV_EXIT_CODE_NON_EXECUTION 58u  /* prev_exit_code != exit_code: exit code should be same in non-execution shards */
#define SP1B200_VERDICT_PV_EXIT_CODE_CHANGED 59u        /* prev_exit_code != exit_code: exit code should change at most once */
#define SP1B200_VERDICT_PV_PROOF_NONCE 60u              /* proof_nonce != proof_nonce_first_shard */
#define SP1B200_VERDICT_PV_INIT_ADDR 61u                /* previous_init_addr != last_init_addr_prev */
#define SP1B200_VERDICT_PV_FINALIZE_ADDR 62u            /* previous_finalize_addr != last_finalize_addr_prev */
#define SP1B200_VERDICT_PV_INIT_PAGE_IDX 63u            /* previous_init_page_idx != last_init_page_idx_prev */
#define SP1B200_VERDICT_PV_FINALIZE_PAGE_IDX 64u        /* previous_finalize_page_idx != last_finalize_page_idx_prev */
#define SP1B200_VERDICT_PV_UNTRUSTED_PROGRAMS 65u       /* public_values.is_untrusted_programs_enabled != vk...enable_untrusted_programs */
#define SP1B200_VERDICT_PV_NEVER_INITIALIZED 66u        /* the zero address was never initialized */
#define SP1B200_VERDICT_PV_NEVER_FINALIZED 67u          /* the zero address was never finalized */
#define SP1B200_VERDICT_PV_COMMITTED_VALUE_DIGEST 68u   /* prev_committed_value_digest doesn't equal the previous shard's ... */
#define SP1B200_VERDICT_PV_DEFERRED_PROOFS_DIGEST 69u   /* prev_deferred_proofs_digest doesn't equal the previous shard's ... */
#define SP1B200_VERDICT_PV_COMMIT_SYSCALL 70u           /* prev_commit_syscall doesn't equal the previous shard's commit_syscall */
#define SP1B200_VERDICT_PV_COMMIT_DEFERRED_SYSCALL 71u  /* prev_commit_deferred_syscall doesn't equal the previous shard's ... */
#define SP1B200_VERDICT_PV_COMMIT_NEVER_CALLED 72u      /* COMMIT syscall was never called */
#define SP1B200_VERDICT_PV_COMMIT_DEFERRED_NEVER_CALLED 73u/* COMMIT_DEFERRED_PROOFS syscall was never called */
#define SP1B200_VERDICT_PV_GLOBAL_CUMULATIVE_SUM 74u    /* global cumulative sum is not zero */
#define SP1B200_VERDICT_PV_EXCEPTIONAL_ADDITION 75u     /* global cumulative sum: exceptional point addition (this library only, see above) */
#define SP1B200_VERDICT_CORE_COUNT 76u                  /* one past the last code */
sp1b200_err sp1b200_verify_core_proof(sp1b200_ctx* ctx, const sp1b200_machine* machine, const uint32_t* h_prep_commit8,
                                      const uint32_t* h_vk_tail, uint32_t n_vk_tail, uint32_t n_shards, const uint64_t* h_heights,
                                      const char* const* chip_names, const uint32_t* const* h_proofs, const uint64_t* h_n_words,
                                      uint32_t host_threads, uint32_t* h_final_challengers, uint32_t* h_verdict, uint32_t* h_shard,
                                      uint32_t* h_shard_verdict);

/* ---- recursion keys, public values and the recursion vk map (host only unless a context is taken) ---------------------------------
 * MachineVerifyingKey::hash_koalabear without mprotect (crates/hypercube/src/verifier/hashable_key.rs:94-118): poseidon2_hash of the 26
 * words prep_commit[8] | pc_start[3] | initial_global_cumulative_sum x[7] y[7] | enable_untrusted_programs, i.e. the commitment and the
 * first 18 words of the 24-word vk_tail that sp1b200_setup_and_prove_shard takes (its 6 padding words are observed, not hashed).
 * n_vk_tail must be 24. */
sp1b200_err sp1b200_vk_hash(const uint32_t* h_prep_commit8, const uint32_t* h_vk_tail, uint32_t n_vk_tail, uint32_t* h_out8);
/* koalabears_to_bn254 (hashable_key.rs:23-33) as 32 big-endian bytes, the vk.bytes32() value: the canonical words concatenated 31 bits
 * apart, first word most significant (248 bits < r, so no reduction; byte 0 is zero). */
sp1b200_err sp1b200_digest_bytes32(const uint32_t* h_digest8, uint8_t* h_out32);
/* recursion_public_values_digest (crates/prover/src/utils.rs:22-28): the sponge over the first NUM_PV_ELMS_TO_HASH = 175 words of the 187
 * words of RecursionPublicValues (crates/recursion/executor/src/public_values.rs:39-143; sp1_vk_digest at 136, vk_root at 144,
 * is_complete at 168, digest at 175, proof_nonce at 183). */
sp1b200_err sp1b200_recursion_pv_digest(const uint32_t* h_pv187, uint32_t* h_out8);

/* RecursionVks::from_map (crates/prover/src/recursion.rs:59-87): the digests (n x 8 words) deduplicated and sorted in canonical
 * lexicographic order, [i; 8] added for every index i below pad_to the keys do not reach (as the development map is padded), then
 * MerkleTree::commit (crates/recursion/circuit/src/basefold/merkle_tree.rs:24-64): key i is leaf i, padded with zero digests to a power
 * of two, leaves stored bit-reversed, layers compressed pairwise on the device (the tree kernels of sp1b200_merkle_commit; memory from the
 * context's pool, returned before the call ends).  The layers are then kept on the host.  Fewer than two keys, more than 2^26, or a
 * non-canonical word is an error.  vk_verification: whether sp1b200_verify_compressed checks a proof's key against the map. */
typedef struct sp1b200_recursion_vks sp1b200_recursion_vks;
sp1b200_err sp1b200_recursion_vks_create(sp1b200_ctx* ctx, const uint32_t* h_digests, uint64_t n, uint64_t pad_to, int vk_verification,
                                         sp1b200_recursion_vks** out);
void sp1b200_recursion_vks_free(sp1b200_recursion_vks* vks);
void sp1b200_recursion_vks_root(const sp1b200_recursion_vks* vks, uint32_t* h_out8);
uint64_t sp1b200_recursion_vks_num_keys(const sp1b200_recursion_vks* vks);
/* RecursionVks::open / MerkleTree::open (recursion.rs:141-170, merkle_tree.rs:66-88): the index of digest8 in the map and its Merkle path
 * (*h_n_path = the tree height digests of 8 words into h_path, path_cap digests of room).  A digest outside the map is an error ("vk not
 * allowed").  The path verifies as verify_merkle_proof (crates/hypercube/src/verifier/proof.rs:121-143) does: reverse_bits_len(index,
 * path length) - index bits above the path length are ignored - then one compression per sibling, the sibling on the left when the low
 * bit is one. */
sp1b200_err sp1b200_recursion_vks_open(const sp1b200_recursion_vks* vks, const uint32_t* h_digest8, uint64_t* h_index, uint32_t* h_path,
                                       uint32_t path_cap, uint32_t* h_n_path);

/* ---- compressed / shrink proof verifier (SP1Prover::verify_compressed / verify_shrink, crates/prover/src/verify.rs:527-642) ---------
 * Verifies n_proofs recursion proofs of one machine at the context's parameters.  Proof s has its own verifying key
 * h_vks[s * 32 ..]: preprocessed commitment[8] | vk_tail[24] (as sp1b200_vk_hash), its chip heights h_heights[s * n_chips ..], its
 * flat proof words (sp1b200_prove_shard words), its vk_merkle_proof (h_vk_index[s], h_vk_path_len[s] <= 64 digests at h_vk_paths[s]) and
 * the digest of the SP1 program key the proof must be for (h_sp1_vk_digests[s * 8 ..], the reference's vk.hash_koalabear()).
 * mode SP1B200_COMPRESSED takes no shrink key (h_shrink_vk must be NULL); mode SP1B200_SHRINK compares every proof's key with
 * h_shrink_vk (32 words as above, NULL = not initialised) word for word.  The Rust key's chip information is not compared: here it is
 * fixed by the machine and heights passed in.  Checks per proof, in the reference's order:
 *   shrink only: UninitializedVerificationKey (h_shrink_vk NULL), InvalidVerificationKey (key differs);
 *   InvalidPublicValues(invalid public values length) (not 187 public values; code 46);
 *   InvalidShardProof (code 45; h_shard_verdicts[s] = the verify_shard code), from a fresh transcript that observed the proof's key;
 *   the public values' digest (words 175..182) is not the digest of words 0..174; vk_root (144..151) is not the map's root;
 *   InvalidVerificationKey when the map has vk_verification on and the Merkle proof of sp1b200_vk_hash(key) does not reach the root;
 *   is_complete (168) is not 1; sp1_vk_digest (136..143) differs from the expected digest.
 * h_verdicts[s] = 0 accepts (h_final_challengers[s * 34 ..], optional, then holds the verifier's final transcript state), else the first
 * failing check (sp1b200_verdict_name).  The host phases run on host_threads threads (0 = the hardware concurrency); the device work of
 * all proofs runs in one launch per kernel for each batch of at most 2^26 proof words (SP1B200_VERIFY_BATCH_WORDS can lower the cap;
 * batching never changes a verdict).  Errors: a proof that does not parse (as sp1b200_verify_shard), a vk Merkle path longer than 64, a
 * non-canonical word in a key, path or expected digest, NULL pointers, n_proofs = 0.  A rejection is not an error; the context stays
 * usable after either. */
#define SP1B200_COMPRESSED 0u
#define SP1B200_SHRINK 1u
#define SP1B200_VERDICT_RECURSION_PV_DIGEST 77u         /* InvalidPublicValues(recursion public values are invalid) */
#define SP1B200_VERDICT_VK_ROOT 78u                     /* InvalidPublicValues(vk_root mismatch) */
#define SP1B200_VERDICT_INVALID_VERIFICATION_KEY 79u    /* InvalidVerificationKey: shrink key differs, or the key is not in the vk map */
#define SP1B200_VERDICT_IS_COMPLETE 80u                 /* InvalidPublicValues(is_complete is not 1) */
#define SP1B200_VERDICT_SP1_VK_DIGEST 81u               /* InvalidPublicValues(sp1 vk hash mismatch) */
#define SP1B200_VERDICT_UNINITIALIZED_VERIFICATION_KEY 82u /* UninitializedVerificationKey: shrink mode without a shrink key */
#define SP1B200_VERDICT_COMPRESSED_COUNT 83u            /* one past the last code */
sp1b200_err sp1b200_verify_compressed(sp1b200_ctx* ctx, const sp1b200_machine* machine, const sp1b200_recursion_vks* vks, uint32_t mode,
                                      const uint32_t* h_shrink_vk, uint32_t n_proofs, const uint32_t* h_vks, const uint64_t* h_heights,
                                      const char* const* chip_names, const uint32_t* const* h_proofs, const uint64_t* h_n_words,
                                      const uint64_t* h_vk_index, const uint32_t* const* h_vk_paths, const uint32_t* h_vk_path_len,
                                      const uint32_t* h_sp1_vk_digests, uint32_t host_threads, uint32_t* h_final_challengers,
                                      uint32_t* h_verdicts, uint32_t* h_shard_verdicts);

#ifdef __cplusplus
}
#endif
#endif /* SP1B200_H */
