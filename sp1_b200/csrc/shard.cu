// Whole-shard transcript driver: ShardProver::prove_shard_with_data (crates/hypercube/src/prover/shard.rs:650-792; GPU twin
// sp1-gpu/crates/shard_prover/src/prover.rs:618-763) composed from the phase entry points of this library:
// observe public values -> jagged commit of the main traces -> observe commitment and chip table shapes -> LogUp-GKR ->
// sample alpha, gamma -> zerocheck -> jagged evaluation proof at the zerocheck point.
#include "ctx.cuh"
#include "challenger.cuh"
#include "hostfield.hpp"
#include "machine.cuh"
#include "pcs.cuh"
#include "proof_layout.hpp"
#include <cstring>
#include <memory>
#include <string>
#include <vector>

// Chip column pointers inside the dense main buffer (tables back to back) and the preprocessed round, with the checks that the round
// matches the machine and the main heights.  `who` prefixes the error messages.
static sp1b200_err chip_pointers(const char* who, const sp1b200_machine* m, const sp1b200_jagged_round* prep_round, const uint32_t* d_main_dense,
                                 const uint64_t* h_heights, std::vector<const uint32_t*>& d_main, std::vector<const uint32_t*>& d_prep) {
    const size_t nch = m->chips.size();
    d_main.assign(nch, nullptr); d_prep.assign(nch, nullptr);
    uint64_t off = 0, poff = 0; size_t pt = 0;
    // the preprocessed round's chip tables: all of its tables but the two padding tables
    const size_t n_prep_tables = prep_round ? prep_round->tables.size() - 2 : 0;
    for (size_t k = 0; k < nch; k++) {
        d_main[k] = d_main_dense + off;
        off += h_heights[k] * m->chips[k].main_w;
        if (m->chips[k].prep_w) {
            if (pt >= n_prep_tables || prep_round->tables[pt].second != m->chips[k].prep_w)
                return sp1b200_set_error("%s: preprocessed round does not match the machine at chip %zu", who, k);
            const uint64_t rows = prep_round->tables[pt].first;
            if (rows != h_heights[k])
                return sp1b200_set_error("%s: chip %zu: preprocessed height %llu != main height %llu", who, k, (unsigned long long)rows,
                                         (unsigned long long)h_heights[k]);
            d_prep[k] = prep_round->d_dense + poff;
            poff += rows * m->chips[k].prep_w;
            pt++;
        }
    }
    return nullptr;
}

// The inputs of sp1b200_prove_shard for the two shard checks: heights within 2^max_log_row_count, the main tables on the device
// (a host buffer is staged through the pool; an upload slot is waited for in stream order and released after `run`), chip pointers.
template <class Run>
static sp1b200_err with_shard_inputs(const char* who, sp1b200_ctx* ctx, const sp1b200_machine* m, const sp1b200_jagged_round* prep_round,
                                     const uint32_t* main_dense_any, const uint64_t* h_heights, Run run) {
    const size_t nch = m->chips.size();
    const uint32_t mlr = ctx->params.max_log_row_count;
    uint64_t area = 0;
    for (size_t k = 0; k < nch; k++) {
        if (h_heights[k] > ((uint64_t)1 << mlr))
            return sp1b200_set_error("%s: chip %zu has %llu rows > 2^%u", who, k, (unsigned long long)h_heights[k], mlr);
        area += h_heights[k] * m->chips[k].main_w;
    }
    if (area && !main_dense_any) return sp1b200_set_error("%s: main_dense_any is NULL", who);
    const int up_slot = sp1b200_upload_acquire(ctx, main_dense_any);
    DevBuf main;
    sp1b200_err e = main.in(ctx, main_dense_any, area * 4);
    std::vector<const uint32_t*> d_main, d_prep;
    if (!e) e = chip_pointers(who, m, prep_round, static_cast<const uint32_t*>(main.d), h_heights, d_main, d_prep);
    if (!e) e = run(d_main, d_prep);
    sp1b200_upload_release(ctx, up_slot);
    return e;
}

extern "C" {

// debug_constraints_all_chips (crates/hypercube/src/debug.rs:27-130) on the device: report words in include/sp1b200.h
sp1b200_err sp1b200_debug_constraints(sp1b200_ctx* ctx, const sp1b200_machine* m, sp1b200_jagged_round* prep_round, const uint32_t* main_dense_any,
                                      const uint64_t* h_heights, const uint32_t* h_pv, uint32_t n_pv, uint32_t max_rows_per_chip, uint32_t* h_out,
                                      uint64_t out_cap_words, uint64_t* h_out_words) { SP1_DEVICE_GUARD(ctx);
    std::vector<uint32_t> words;
    SP1_TRY(with_shard_inputs("debug_constraints", ctx, m, prep_round, main_dense_any, h_heights,
                              [&](const std::vector<const uint32_t*>& d_main, const std::vector<const uint32_t*>& d_prep) {
                                  return sp1b200_debug_constraints_device(ctx, m, h_heights, d_main.data(), d_prep.data(), h_pv, n_pv,
                                                                          max_rows_per_chip, words);
                              }));
    return layout::deliver("debug_constraints", "report", words, h_out, out_cap_words, h_out_words);
}

// debug_interactions_with_all_chips (crates/hypercube/src/lookup/debug.rs:48-200) on the device: report words in include/sp1b200.h
sp1b200_err sp1b200_debug_interactions(sp1b200_ctx* ctx, const sp1b200_machine* m, sp1b200_jagged_round* prep_round, const uint32_t* main_dense_any,
                                       const uint64_t* h_heights, uint32_t max_keys, uint32_t* h_out, uint64_t out_cap_words,
                                       uint64_t* h_out_words) { SP1_DEVICE_GUARD(ctx);
    std::vector<uint32_t> words;
    SP1_TRY(with_shard_inputs("debug_interactions", ctx, m, prep_round, main_dense_any, h_heights,
                              [&](const std::vector<const uint32_t*>& d_main, const std::vector<const uint32_t*>& d_prep) {
                                  return sp1b200_debug_interactions_device(ctx, m, h_heights, d_main.data(), d_prep.data(), max_keys, words);
                              }));
    return layout::deliver("debug_interactions", "report", words, h_out, out_cap_words, h_out_words);
}

// Proof words (proof_layout.hpp): the main commitment, the sp1b200_logup_gkr, sp1b200_zerocheck and sp1b200_jagged_prove words, the
// public values = the fields of ShardProof (crates/hypercube/src/verifier/proof.rs:47-61); chip degrees are the heights the caller passed.
// h_replay_witnesses (grind_mode == 1): {gkr witness, batch grinding witness, pow witness}.
sp1b200_err sp1b200_prove_shard(sp1b200_ctx* ctx, const sp1b200_machine* m, sp1b200_jagged_round* prep_round, const uint32_t* main_dense_any,
                                const uint64_t* h_heights, const char* const* chip_names, const uint32_t* h_pv, uint32_t n_pv,
                                const uint32_t* h_replay_witnesses, uint32_t* h_chal, uint32_t* h_proof, uint64_t cap, uint64_t* h_words) { SP1_DEVICE_GUARD(ctx);
    using hf::E4;
    const size_t nch = m->chips.size();
    const uint32_t mlr = ctx->params.max_log_row_count;
    PhaseTimer t_all(ctx, "shard.total");
    HostChallenger ch;
    SP1_TRY(ch.init(ctx, h_chal));
    ch.observe_n(h_pv, n_pv);
    // main commit
    std::vector<uint64_t> rows(nch), cols(nch);
    for (size_t k = 0; k < nch; k++) { rows[k] = h_heights[k]; cols[k] = m->chips[k].main_w; }
    uint32_t commit[8];
    sp1b200_jagged_round* main_round = nullptr;
    {
        PhaseTimer t(ctx, "shard.commit");
        SP1_TRY(sp1b200_jagged_commit(ctx, main_dense_any, (uint32_t)nch, rows.data(), cols.data(), 1, commit, &main_round));
        t.stop();
    }
    struct Guard { sp1b200_ctx* c; sp1b200_jagged_round* r; ~Guard() { sp1b200_jagged_round_free(c, r); } } guard{ctx, main_round};
    ch.observe_n(commit, 8);
    observe_chip_shapes(ch, nch, h_heights, chip_names);
    // chip column pointers inside the dense buffers
    std::vector<const uint32_t*> d_main, d_prep;
    SP1_TRY(chip_pointers("prove_shard", m, prep_round, main_round->d_dense, h_heights, d_main, d_prep));
    uint32_t st[34];
    ch.store(st);
    // per-context scratch for the phase outputs, allocated once and reused by every shard proven on this context (uninitialised:
    // zero-filling 3 x 64 MiB per shard would cost more than some of the phases)
    const uint64_t scratch_cap = (uint64_t)1 << 24;
    if (!ctx->shard_scratch) ctx->shard_scratch.reset(new uint32_t[3 * scratch_cap]);
    uint32_t* gkr = ctx->shard_scratch.get();
    uint64_t n_gkr = 0;
    SP1_TRY(sp1b200_logup_gkr(ctx, m, h_heights, d_main.data(), d_prep.data(), h_replay_witnesses, st, gkr, scratch_cap, &n_gkr));
    // the phase outputs are read with the proof layout's section readers
    std::vector<uint32_t> main_w(nch), prep_w(nch);
    for (size_t k = 0; k < nch; k++) { main_w[k] = m->chips[k].main_w; prep_w[k] = m->chips[k].prep_w; }
    layout::Shape shape;
    shape.n_chips = nch; shape.main_w = main_w.data(); shape.prep_w = prep_w.data(); shape.max_log_row_count = mlr;
    layout::ShardProof phases;   // its LogUp-GKR and zerocheck fields
    layout::FlatReader gkr_words{gkr, gkr + n_gkr};
    if (const char* why = layout::read_gkr(gkr_words, shape, phases)) return sp1b200_set_error("prove_shard: %s", why);
    ch.load(st);
    E4 alpha, gamma;
    ch.sample_ext(alpha.c); ch.sample_ext(gamma.c);
    std::vector<uint32_t> claims(nch * 4);
    for (size_t k = 0; k < nch; k++)
        batched_opening_claim(phases.gkr_main[k], main_w[k], phases.gkr_prep[k], prep_w[k], gamma).store(&claims[4 * k]);
    ch.store(st);
    uint32_t* zc = gkr + scratch_cap;
    uint64_t n_zc = 0;
    SP1_TRY(sp1b200_zerocheck(ctx, m, h_heights, d_main.data(), d_prep.data(), h_pv, n_pv, phases.gkr_point, alpha.c, gamma.c, claims.data(), st,
                              zc, scratch_cap, &n_zc));
    layout::FlatReader zc_words{zc, zc + n_zc};
    if (const char* why = layout::read_zerocheck(zc_words, shape, phases)) return sp1b200_set_error("prove_shard: %s", why);
    if (phases.zc.polys.size() != mlr)
        return sp1b200_set_error("prove_shard: zerocheck section: %zu rounds, the point needs %u", phases.zc.polys.size(), mlr);
    // the jagged claims: the opened values of the preprocessed round's columns, then the main round's, in chip order
    std::vector<uint32_t> jclaims;
    if (prep_round)
        for (size_t k = 0; k < nch; k++) jclaims.insert(jclaims.end(), phases.zc_prep[k], phases.zc_prep[k] + 4 * prep_w[k]);
    for (size_t k = 0; k < nch; k++) jclaims.insert(jclaims.end(), phases.zc_main[k], phases.zc_main[k] + 4 * main_w[k]);
    std::vector<sp1b200_jagged_round*> rounds;
    if (prep_round) rounds.push_back(prep_round);
    rounds.push_back(main_round);
    uint32_t* ev = gkr + 2 * scratch_cap;
    uint64_t n_ev = 0;
    SP1_TRY(sp1b200_jagged_prove(ctx, rounds.data(), (uint32_t)rounds.size(), phases.zc.point, jclaims.data(),
                                 h_replay_witnesses ? h_replay_witnesses + 1 : nullptr, st, ev, scratch_cap, &n_ev));
    const uint64_t total = layout::shard_proof_words(n_gkr, n_zc, n_ev, n_pv);
    t_all.stop();
    if (h_words) *h_words = total;
    // the caller's challenger is advanced only together with a delivered proof: on a capacity error h_chal is untouched and
    // *h_words holds the size to retry with
    if (h_proof && total > cap) return sp1b200_set_error("prove_shard: proof needs %llu words, capacity %llu", (unsigned long long)total, (unsigned long long)cap);
    memcpy(h_chal, st, sizeof(st));
    if (h_proof) layout::write_shard_proof(h_proof, commit, gkr, n_gkr, zc, n_zc, ev, n_ev, h_pv, n_pv);
    return nullptr;
}

// AirProver::setup_and_prove_shard (shard.rs:56-68): setup = commit the preprocessed traces, observe the verifying key
// (MachineVerifyingKey::observe_into, verifier/config.rs:97-112: commitment, then the program-dependent words), prove.
sp1b200_err sp1b200_setup_and_prove_shard(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint32_t* prep_dense_any, uint32_t n_prep,
                                          const uint64_t* h_prep_rows, const uint64_t* h_prep_cols, const uint32_t* h_vk_tail, uint32_t n_vk_tail,
                                          const uint32_t* main_dense_any, const uint64_t* h_heights, const char* const* chip_names,
                                          const uint32_t* h_pv, uint32_t n_pv, const uint32_t* h_replay_witnesses, uint32_t* h_chal,
                                          uint32_t* h_prep_commit8, sp1b200_jagged_round** prep_round_out, uint32_t* h_proof, uint64_t cap,
                                          uint64_t* h_words) { SP1_DEVICE_GUARD(ctx);
    if (!prep_round_out) return sp1b200_set_error("setup_and_prove_shard: prep_round_out is NULL");
    *prep_round_out = nullptr;
    uint32_t commit[8] = {0};
    sp1b200_jagged_round* prep = nullptr;
    if (n_prep) SP1_TRY(sp1b200_jagged_commit(ctx, prep_dense_any, n_prep, h_prep_rows, h_prep_cols, 1, commit, &prep));
    HostChallenger ch;
    sp1b200_err e = ch.init(ctx, h_chal);
    if (!e) {
        ch.observe_n(commit, 8);
        ch.observe_n(h_vk_tail, n_vk_tail);
        uint32_t st[34];
        ch.store(st);
        e = sp1b200_prove_shard(ctx, m, prep, main_dense_any, h_heights, chip_names, h_pv, n_pv, h_replay_witnesses, st, h_proof, cap, h_words);
        if (!e) memcpy(h_chal, st, sizeof(st));
    }
    if (e) { sp1b200_jagged_round_free(ctx, prep); return e; }
    if (h_prep_commit8) memcpy(h_prep_commit8, commit, 32);
    *prep_round_out = prep;
    return nullptr;
}
}
