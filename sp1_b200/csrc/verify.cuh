// The shard verifier's interface inside the library (verify.cu): sp1b200_verify_shard, sp1b200_verify_core_proof (verify_core.cu) and
// sp1b200_verify_compressed (recursion_vks.cu) parse each shard with verify_parse_shard and verify a list of parsed shards with
// verify_shards.
#pragma once
#include "ctx.cuh"
#include "machine.cuh"
#include "proof_layout.hpp"
#include <string>
#include <vector>

// the verifying key's words after the preprocessed commitment (without mprotect): pc_start[3] | initial_global_cumulative_sum x[7] y[7] |
// enable_untrusted_programs | 6 zeros
constexpr uint32_t VK_TAIL_WORDS = 24;

// one shard's flat proof words, parsed and checked against the machine, its heights and the context's parameters
struct VerifyShardIn {
    const uint64_t* heights = nullptr;
    const uint32_t* prep_commit8 = nullptr;   // the verifying key's preprocessed commitment (NULL when no chip has preprocessed columns)
    std::vector<uint32_t> mw, pw;
    layout::Shape shape;     // points into mw / pw: not copyable
    layout::ShardProof p;
    VerifyShardIn() = default;
    VerifyShardIn(const VerifyShardIn&) = delete;
    VerifyShardIn& operator=(const VerifyShardIn&) = delete;
};

// Errors (prefixed with `who`): parameters out of range, a chip without a name, a height beyond max_log_row_count + 1 bits, a machine
// that is not initialised, preprocessed columns without h_prep_commit8, words that do not parse, non-canonical field words, a public
// value index beyond the proof's, more GKR outputs or tables than this library's shards can have.
sp1b200_err verify_parse_shard(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint32_t* h_prep_commit8, const uint64_t* h_heights,
                               const char* const* chip_names, const uint32_t* h_proof, uint64_t n_words, const std::string& who,
                               VerifyShardIn& out);

struct VerifyTimes { double host_ms = 0; float merkle = 0, fold = 0, jagged = 0; bool fold_ran = false, jagged_ran = false; };

// verify_shard of every shard, shard s from the transcript state starts[s] (34 words) under its own preprocessed commitment.  The
// host phases run on host_threads threads (at least 1); the device work of all shards then runs in one launch per kernel, with one
// copy back.  verdicts[s] = the shard's verdict; finals (optional): the verifier's final state of every accepted shard at
// finals + 34 s.  Times are added to t.
sp1b200_err verify_shards(sp1b200_ctx* ctx, const sp1b200_machine* m, const char* const* chip_names,
                          const std::vector<const VerifyShardIn*>& shards, const std::vector<const uint32_t*>& starts, uint32_t host_threads,
                          uint32_t* verdicts, uint32_t* finals, VerifyTimes& t);

// the name of a verdict of sp1b200_verify_core_proof beyond the shard verdicts (verify_core.cu); NULL outside that range
const char* verify_core_verdict_name(uint32_t verdict);
// the name of a verdict of sp1b200_verify_compressed beyond the core-proof verdicts (recursion_vks.cu); NULL outside that range
const char* verify_compressed_verdict_name(uint32_t verdict);

// SP1B200_VERIFY_BATCH_WORDS, capped at (and by default) 2^26 proof words per batch of verify_shards
uint64_t verify_batch_words_cap();
