// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header).  C entry points of the restated core-proof verifier (core.hpp), built into
// their own library, oracle/libcoreoracle.so (oracle/core.mk), for tests/core_oracle_lib.py.  The shards are verified by the oracle's
// restated ShardVerifier, orc_verify_shard of liboracle.so.  Field elements cross as u32 Montgomery words.
#include "core.hpp"
#include <cstring>

using namespace orc;

extern "C" {
// liboracle.so
int64_t orc_verify_shard(const uint32_t* machine_blob, const uint64_t* heights, const char* names, uint32_t log_stack, uint32_t max_log_rows,
                         uint32_t log_blowup, uint32_t num_queries, uint32_t pow_bits, uint32_t batch_pow_bits, uint32_t gkr_pow_bits,
                         uint32_t* challenger_state, const uint32_t* prep_commit8, const uint32_t* words, uint64_t n_words);
void orc_challenger_init(uint32_t* st);
void orc_challenger_observe(uint32_t* st, const uint32_t* vals, uint64_t n);

static S7 ld7(const uint32_t* p) { S7 r; for (int i = 0; i < 7; i++) r.c[i] = F::raw(p[i]); return r; }
static void st7(const S7& a, uint32_t* p) { for (int i = 0; i < 7; i++) p[i] = a.c[i].v; }

void orc_septic_mul(const uint32_t* a, const uint32_t* b, uint32_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) st7(ld7(a + 7 * i) * ld7(b + 7 * i), out + 7 * i);
}
void orc_septic_inv(const uint32_t* a, uint32_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) st7(s7_inv(ld7(a + 7 * i)), out + 7 * i);
}
// points: x[7] y[7]; ok[i] = 0 on the exceptional case
void orc_septic_curve_add(const uint32_t* p, const uint32_t* q, uint32_t* out, uint32_t* ok, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        SPoint r;
        ok[i] = s_add(SPoint{ld7(p + 14 * i), ld7(p + 14 * i + 7)}, SPoint{ld7(q + 14 * i), ld7(q + 14 * i + 7)}, r);
        if (ok[i]) { st7(r.x, out + 14 * i); st7(r.y, out + 14 * i + 7); }
    }
}
int orc_septic_digest_add(const uint32_t* a, const uint32_t* b, uint32_t* out) {
    SPoint r;
    if (!digest_add(SPoint{ld7(a), ld7(a + 7)}, SPoint{ld7(b), ld7(b + 7)}, r)) return 0;
    st7(r.x, out); st7(r.y, out + 7);
    return 1;
}

// SP1Prover::verify (verify.rs:109-524): -> 0 (accepted), a verdict code of include/sp1b200.h, or -2 when a shard's words do not
// parse.  *shard: where the failing check stops; for InvalidShardProof *shard_result = the oracle's orc_verify_shard result (-1).
// heights: [n_shards][n_chips]; names: NUL-separated; vk_tail: 24 words.
int64_t orc_verify_core_proof(const uint32_t* machine_blob, uint32_t n_chips, const uint64_t* heights, const char* names, uint32_t log_stack,
                              uint32_t max_log_rows, uint32_t log_blowup, uint32_t num_queries, uint32_t pow_bits, uint32_t batch_pow_bits,
                              uint32_t gkr_pow_bits, const uint32_t* prep_commit8, const uint32_t* vk_tail, uint32_t n_shards,
                              const uint32_t* const* proofs, const uint64_t* n_words, uint32_t* shard, int64_t* shard_result) {
    *shard_result = 0;
    *shard = 0;
    std::vector<const uint32_t*> pvs;
    std::vector<uint64_t> npv;
    for (uint32_t s = 0; s < n_shards; s++) {   // the public values: the last of the five sections
        const uint32_t* w = proofs[s];
        if (n_words[s] < 6 || w[0] != 5) return -2;
        const uint64_t l4 = w[5];
        if (6 + (uint64_t)w[1] + w[2] + w[3] + w[4] + l4 != n_words[s]) return -2;
        pvs.push_back(w + n_words[s] - l4);
        npv.push_back(l4);
    }
    if (const int64_t v = core_public_value_checks(pvs, npv, vk_tail, shard)) return v;
    uint32_t start[34];
    orc_challenger_init(start);
    orc_challenger_observe(start, prep_commit8, 8);
    orc_challenger_observe(start, vk_tail, 24);
    for (uint32_t s = 0; s < n_shards; s++) {
        uint32_t st[34];
        memcpy(st, start, sizeof(st));
        const int64_t r = orc_verify_shard(machine_blob, heights + (size_t)s * n_chips, names, log_stack, max_log_rows, log_blowup, num_queries,
                                           pow_bits, batch_pow_bits, gkr_pow_bits, st, prep_commit8, proofs[s], n_words[s]);
        if (r == -2) return -2;
        if (r != 0) { *shard = s; *shard_result = r; return CORE_INVALID_SHARD_PROOF; }
    }
    return 0;
}
}
