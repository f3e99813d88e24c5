// SP1Prover::verify (crates/prover/src/verify.rs:109-524) for a core proof: the list of flat shard proofs of one execution.
// The checks across shards read the public values (the last section of every shard's words) and run on the host; the shards
// themselves are verified by verify_shards (verify.cu), whose host phases run on several threads and whose device work for a whole
// batch of shards runs in one launch per kernel.
#include "ctx.cuh"
#include "challenger.cuh"
#include "hostfield.hpp"
#include "public_values.hpp"
#include "septic.cuh"
#include "verify.cuh"
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>

namespace {

constexpr uint32_t MAX_LOG_NUMBER_OF_SHARDS = 24;
constexpr uint64_t DEFAULT_BATCH_WORDS = (uint64_t)1 << 26;

const char* const CORE_NAMES[SP1B200_VERDICT_CORE_COUNT - SP1B200_VERDICT_EMPTY_PROOF] = {
    "EmptyProof", "TooManyShards", "InvalidShardProof",
    "InvalidPublicValues(invalid public values length)",
    "InvalidPublicValues(is_first_execution_shard is set to one for multiple shards)",
    "InvalidPublicValues(is_first_execution_shard is not boolean)",
    "InvalidPublicValues(first execution shard is not set)",
    "InvalidPublicValues(invalid initial timestamp)",
    "InvalidPublicValues(timestamp should change on execution shard)",
    "InvalidPublicValues(timestamp should not change on non-execution shard)",
    "InvalidPublicValues(pc_start != vk.pc_start: program counter should start at vk.pc_start)",
    "InvalidPublicValues(pc_start != prev_next_pc: pc_start should equal prev_next_pc for all shards)",
    "InvalidPublicValues(pc_start != next_pc: pc_start should equal next_pc for non-execution shards)",
    "InvalidPublicValues(next_pc != HALT_PC: execution should have halted)",
    "InvalidPublicValues(public_values.prev_exit_code != prev_exit_code: prev_exit_code does not match previous shard's exit_code)",
    "InvalidPublicValues(prev_exit_code != exit_code: exit code should be same in non-execution shards)",
    "InvalidPublicValues(prev_exit_code != exit_code: exit code should change at most once)",
    "InvalidPublicValues(proof_nonce != proof_nonce_first_shard)",
    "InvalidPublicValues(previous_init_addr != last_init_addr_prev)",
    "InvalidPublicValues(previous_finalize_addr != last_finalize_addr_prev)",
    "InvalidPublicValues(previous_init_page_idx != last_init_page_idx_prev)",
    "InvalidPublicValues(previous_finalize_page_idx != last_finalize_page_idx_prev)",
    "InvalidPublicValues(public_values.is_untrusted_programs_enabled != vk.untrusted_config.enable_untrusted_programs)",
    "InvalidPublicValues(the zero address was never initialized)",
    "InvalidPublicValues(the zero address was never finalized)",
    "InvalidPublicValues(prev_committed_value_digest doesn't equal the previous shard's committed_value_digest)",
    "InvalidPublicValues(prev_deferred_proofs_digest doesn't equal the previous shard's deferred_proofs_digest)",
    "InvalidPublicValues(prev_commit_syscall doesn't equal the previous shard's commit_syscall)",
    "InvalidPublicValues(prev_commit_deferred_syscall doesn't equal the previous shard's commit_deferred_syscall)",
    "InvalidPublicValues(COMMIT syscall was never called)",
    "InvalidPublicValues(COMMIT_DEFERRED_PROOFS syscall was never called)",
    "InvalidPublicValues(global cumulative sum is not zero)",
    "InvalidPublicValues(global cumulative sum: exceptional point addition)",
};

bool eqw(const uint32_t* a, const uint32_t* b, size_t n) { return !memcmp(a, b, 4 * n); }
bool zerow(const uint32_t* a, size_t n) { for (size_t i = 0; i < n; i++) if (a[i]) return false; return true; }

// the checks of verify.rs:116-510 on the public values, in the reference's order: -> verdict (0 = all hold), *shard = where it fails.
// Field elements compare as Montgomery words, which are equal exactly when the canonical values are.
uint32_t check_public_values(const std::vector<const uint32_t*>& pvs, const std::vector<uint32_t>& n_pv, const uint32_t* vk_tail, uint32_t* shard) {
    const uint32_t n = (uint32_t)pvs.size();
    const uint32_t ONE = kb::ONE;
    *shard = 0;
    if (n == 0) return SP1B200_VERDICT_EMPTY_PROOF;
    auto fail = [&](uint32_t code, uint32_t s) { *shard = s; return code; };
    for (uint32_t s = 0; s < n; s++)
        if (n_pv[s] != pv::PROOF_MAX_NUM_PVS) return fail(SP1B200_VERDICT_PV_LENGTH, s);
    bool first_set = false;
    for (uint32_t s = 0; s < n; s++) {
        const uint32_t f = pvs[s][pv::IS_FIRST_EXECUTION_SHARD];
        if (f == ONE) {
            if (first_set) return fail(SP1B200_VERDICT_PV_FIRST_SHARD_MULTIPLE, s);
            first_set = true;
        } else if (f != 0) {
            return fail(SP1B200_VERDICT_PV_FIRST_SHARD_NOT_BOOLEAN, s);
        }
    }
    if (!first_set) return fail(SP1B200_VERDICT_PV_FIRST_SHARD_NOT_SET, n);
    // timestamps
    uint32_t prev_ts[4] = {0, 0, 0, ONE};
    for (uint32_t s = 0; s < n; s++) {
        const uint32_t* v = pvs[s];
        const bool same = eqw(v + pv::INITIAL_TIMESTAMP, v + pv::LAST_TIMESTAMP, 4);
        if (!eqw(v + pv::INITIAL_TIMESTAMP, prev_ts, 4)) return fail(SP1B200_VERDICT_PV_INITIAL_TIMESTAMP, s);
        if (v[pv::IS_EXECUTION_SHARD] != 0 && same) return fail(SP1B200_VERDICT_PV_TIMESTAMP_UNCHANGED, s);
        if (v[pv::IS_EXECUTION_SHARD] != ONE && !same) return fail(SP1B200_VERDICT_PV_TIMESTAMP_CHANGED, s);
        memcpy(prev_ts, v + pv::LAST_TIMESTAMP, 16);
    }
    // program counters: vk.pc_start .. HALT_PC = [1, 0, 0]
    uint32_t prev_pc[3];
    memcpy(prev_pc, vk_tail, 12);
    for (uint32_t s = 0; s < n; s++) {
        const uint32_t* v = pvs[s];
        if (!eqw(v + pv::PC_START, prev_pc, 3)) return fail(s == 0 ? SP1B200_VERDICT_PV_PC_START_VK : SP1B200_VERDICT_PV_PC_START_PREV, s);
        if (v[pv::IS_EXECUTION_SHARD] != ONE && !eqw(v + pv::PC_START, v + pv::NEXT_PC, 3)) return fail(SP1B200_VERDICT_PV_PC_NON_EXECUTION, s);
        memcpy(prev_pc, v + pv::NEXT_PC, 12);
    }
    const uint32_t halt_pc[3] = {ONE, 0, 0};
    if (!eqw(prev_pc, halt_pc, 3)) return fail(SP1B200_VERDICT_PV_NOT_HALTED, n);
    // exit codes
    uint32_t prev_exit = 0;
    for (uint32_t s = 0; s < n; s++) {
        const uint32_t* v = pvs[s];
        if (v[pv::PREV_EXIT_CODE] != prev_exit) return fail(SP1B200_VERDICT_PV_PREV_EXIT_CODE, s);
        if (v[pv::IS_EXECUTION_SHARD] != ONE && v[pv::PREV_EXIT_CODE] != v[pv::EXIT_CODE]) return fail(SP1B200_VERDICT_PV_EXIT_CODE_NON_EXECUTION, s);
        if (v[pv::PREV_EXIT_CODE] != 0 && v[pv::PREV_EXIT_CODE] != v[pv::EXIT_CODE]) return fail(SP1B200_VERDICT_PV_EXIT_CODE_CHANGED, s);
        prev_exit = v[pv::EXIT_CODE];
    }
    // one proof nonce
    for (uint32_t s = 1; s < n; s++)
        if (!eqw(pvs[s] + pv::PROOF_NONCE, pvs[0] + pv::PROOF_NONCE, 4)) return fail(SP1B200_VERDICT_PV_PROOF_NONCE, s);
    // memory initialisation and finalisation
    uint32_t ia[3] = {0, 0, 0}, fa[3] = {0, 0, 0}, ip[3] = {0, 0, 0}, fp[3] = {0, 0, 0};
    for (uint32_t s = 0; s < n; s++) {
        const uint32_t* v = pvs[s];
        if (!eqw(v + pv::PREVIOUS_INIT_ADDR, ia, 3)) return fail(SP1B200_VERDICT_PV_INIT_ADDR, s);
        if (!eqw(v + pv::PREVIOUS_FINALIZE_ADDR, fa, 3)) return fail(SP1B200_VERDICT_PV_FINALIZE_ADDR, s);
        if (!eqw(v + pv::PREVIOUS_INIT_PAGE_IDX, ip, 3)) return fail(SP1B200_VERDICT_PV_INIT_PAGE_IDX, s);
        if (!eqw(v + pv::PREVIOUS_FINALIZE_PAGE_IDX, fp, 3)) return fail(SP1B200_VERDICT_PV_FINALIZE_PAGE_IDX, s);
        if (v[pv::IS_UNTRUSTED_PROGRAMS_ENABLED] != vk_tail[17]) return fail(SP1B200_VERDICT_PV_UNTRUSTED_PROGRAMS, s);
        memcpy(ia, v + pv::LAST_INIT_ADDR, 12); memcpy(fa, v + pv::LAST_FINALIZE_ADDR, 12);
        memcpy(ip, v + pv::LAST_INIT_PAGE_IDX, 12); memcpy(fp, v + pv::LAST_FINALIZE_PAGE_IDX, 12);
    }
    if (zerow(ia, 3)) return fail(SP1B200_VERDICT_PV_NEVER_INITIALIZED, n);
    if (zerow(fa, 3)) return fail(SP1B200_VERDICT_PV_NEVER_FINALIZED, n);
    // committed-value and deferred-proof digests, commit-syscall flags
    const uint32_t* cvd = nullptr;   // null = the zero digest
    const uint32_t* dpd = nullptr;
    uint32_t commit = 0, commit_deferred = 0;
    for (uint32_t s = 0; s < n; s++) {
        const uint32_t* v = pvs[s];
        if (cvd ? !eqw(v + pv::PREV_COMMITTED_VALUE_DIGEST, cvd, 32) : !zerow(v + pv::PREV_COMMITTED_VALUE_DIGEST, 32))
            return fail(SP1B200_VERDICT_PV_COMMITTED_VALUE_DIGEST, s);
        if (dpd ? !eqw(v + pv::PREV_DEFERRED_PROOFS_DIGEST, dpd, 8) : !zerow(v + pv::PREV_DEFERRED_PROOFS_DIGEST, 8))
            return fail(SP1B200_VERDICT_PV_DEFERRED_PROOFS_DIGEST, s);
        if (v[pv::PREV_COMMIT_SYSCALL] != commit) return fail(SP1B200_VERDICT_PV_COMMIT_SYSCALL, s);
        if (v[pv::PREV_COMMIT_DEFERRED_SYSCALL] != commit_deferred) return fail(SP1B200_VERDICT_PV_COMMIT_DEFERRED_SYSCALL, s);
        cvd = v + pv::COMMITTED_VALUE_DIGEST; dpd = v + pv::DEFERRED_PROOFS_DIGEST;
        commit = v[pv::COMMIT_SYSCALL]; commit_deferred = v[pv::COMMIT_DEFERRED_SYSCALL];
    }
    if (commit != ONE) return fail(SP1B200_VERDICT_PV_COMMIT_NEVER_CALLED, n);
    if (commit_deferred != ONE) return fail(SP1B200_VERDICT_PV_COMMIT_DEFERRED_NEVER_CALLED, n);
    if ((uint64_t)n >= ((uint64_t)1 << MAX_LOG_NUMBER_OF_SHARDS)) return fail(SP1B200_VERDICT_TOO_MANY_SHARDS, n);
    // the global cumulative sum: vk.initial_global_cumulative_sum + every shard's digest, one SepticDigest addition per shard
    // (verify.rs:498-505), must come back to the zero digest.  Where the reference panics on an incomplete addition with a zero
    // denominator, this rejects the proof with its own verdict.
    s7::Pt sum = s7::load_point(vk_tail + 3);
    for (uint32_t s = 0; s < n; s++)
        if (!s7::digest_add(sum, s7::load_point(pvs[s] + pv::GLOBAL_CUMULATIVE_SUM), sum)) return fail(SP1B200_VERDICT_PV_EXCEPTIONAL_ADDITION, s);
    if (!s7::is_zero_digest(sum)) return fail(SP1B200_VERDICT_PV_GLOBAL_CUMULATIVE_SUM, n);
    return SP1B200_VERDICT_ACCEPT;
}

}  // namespace

uint64_t verify_batch_words_cap() {
    const char* e = getenv("SP1B200_VERIFY_BATCH_WORDS");
    if (!e || !*e) return DEFAULT_BATCH_WORDS;
    const unsigned long long v = strtoull(e, nullptr, 10);
    return v ? std::min<uint64_t>(v, DEFAULT_BATCH_WORDS) : DEFAULT_BATCH_WORDS;
}

const char* verify_core_verdict_name(uint32_t verdict) {
    if (verdict < SP1B200_VERDICT_EMPTY_PROOF || verdict >= SP1B200_VERDICT_CORE_COUNT) return nullptr;
    return CORE_NAMES[verdict - SP1B200_VERDICT_EMPTY_PROOF];
}

extern "C" {

sp1b200_err sp1b200_verify_core_proof(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint32_t* h_prep_commit8, const uint32_t* h_vk_tail,
                                      uint32_t n_vk_tail, uint32_t n_shards, const uint64_t* h_heights, const char* const* chip_names,
                                      const uint32_t* const* h_proofs, const uint64_t* h_n_words, uint32_t host_threads,
                                      uint32_t* h_final_challengers, uint32_t* h_verdict, uint32_t* h_shard, uint32_t* h_shard_verdict) {
    SP1_DEVICE_GUARD(ctx);
    if (!ctx || !m || !h_prep_commit8 || !h_vk_tail || !h_verdict || !h_shard || !h_shard_verdict)
        return sp1b200_set_error("verify_core_proof: NULL argument");
    if (n_shards && (!h_heights || !chip_names || !h_proofs || !h_n_words)) return sp1b200_set_error("verify_core_proof: NULL argument");
    if (n_vk_tail != VK_TAIL_WORDS)
        return sp1b200_set_error("verify_core_proof: n_vk_tail is %u; the verifying key without mprotect has %u words after the commitment", n_vk_tail, VK_TAIL_WORDS);
    if (!hf::canonical(h_prep_commit8, 8)) return sp1b200_set_error("verify_core_proof: the preprocessed commitment is not canonical");
    for (uint32_t i = 0; i < n_vk_tail; i++) if (h_vk_tail[i] >= kb::P) return sp1b200_set_error("verify_core_proof: vk_tail word %u is not canonical", i);
    const auto t0 = std::chrono::steady_clock::now();
    const size_t nch = m->chips.size();
    bool has_prep = false;
    for (auto& c : m->chips) has_prep |= c.prep_w != 0;
    // 1. every shard parses
    std::vector<std::unique_ptr<VerifyShardIn>> in;
    std::vector<const uint32_t*> pvs;
    std::vector<uint32_t> n_pv;
    for (uint32_t s = 0; s < n_shards; s++) {
        if (!h_proofs[s]) return sp1b200_set_error("verify_core_proof: shard %u: NULL proof", s);
        in.emplace_back(new VerifyShardIn);
        SP1_TRY(verify_parse_shard(ctx, m, has_prep ? h_prep_commit8 : nullptr, h_heights + (size_t)s * nch, chip_names, h_proofs[s],
                                   h_n_words[s], "verify_core_proof: shard " + std::to_string(s), *in.back()));
        pvs.push_back(in.back()->p.pv);
        n_pv.push_back(in.back()->p.n_pv);
    }
    *h_shard_verdict = 0;
    // 2-5. EmptyProof, the public values across shards, TooManyShards, the global cumulative sum
    uint32_t shard = 0;
    uint32_t verdict = check_public_values(pvs, n_pv, h_vk_tail, &shard);
    // 6. every shard, each from a fresh transcript that has observed the verifying key (verify.rs:513-521)
    VerifyTimes t;
    std::vector<uint32_t> finals(34 * (size_t)n_shards);
    if (!verdict) {
        HostChallenger ch;
        uint32_t zero[34] = {0}, start[34];
        ch.load(zero);
        ch.observe_n(h_prep_commit8, 8);
        ch.observe_n(h_vk_tail, n_vk_tail);
        ch.store(start);
        if (!host_threads) host_threads = std::max(1u, std::thread::hardware_concurrency());
        // batches of consecutive shards with at most verify_batch_words_cap() proof words (at least one shard each), in order: the
        // first failing shard of the first failing batch is the lowest failing shard
        const uint64_t cap = verify_batch_words_cap();
        std::vector<uint32_t> verdicts(n_shards);
        for (uint32_t a = 0; a < n_shards && !verdict;) {
            uint32_t b = a + 1;
            uint64_t words = h_n_words[a];
            while (b < n_shards && words + h_n_words[b] <= cap) words += h_n_words[b++];
            std::vector<const VerifyShardIn*> batch;
            for (uint32_t s = a; s < b; s++) batch.push_back(in[s].get());
            SP1_TRY(verify_shards(ctx, m, chip_names, batch, std::vector<const uint32_t*>(batch.size(), start), host_threads,
                                  verdicts.data() + a, finals.data() + 34 * (size_t)a, t));
            for (uint32_t s = a; s < b; s++)
                if (verdicts[s]) { verdict = SP1B200_VERDICT_INVALID_SHARD_PROOF; shard = s; *h_shard_verdict = verdicts[s]; break; }
            a = b;
        }
    }
    ctx->phase_ms["verify_core.host"] = (float)t.host_ms;
    ctx->phase_ms["verify_core.merkle"] = t.merkle;
    ctx->phase_ms["verify_core.fold"] = t.fold;
    ctx->phase_ms["verify_core.jagged_eval"] = t.jagged;
    ctx->phase_ms["verify_core.kernels"] = t.merkle + t.fold + t.jagged;
    ctx->phase_ms["verify_core.total"] = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *h_verdict = verdict;
    *h_shard = verdict ? shard : 0;
    if (!verdict && h_final_challengers) memcpy(h_final_challengers, finals.data(), finals.size() * 4);
    return nullptr;
}

}  // extern "C"
