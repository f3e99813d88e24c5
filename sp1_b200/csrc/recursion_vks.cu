// SP1Prover::verify_compressed / verify_shrink (crates/prover/src/verify.rs:527-642) and what they need around one recursion-machine
// verify_shard: the verifying-key hash (MachineVerifyingKey::hash_koalabear), its bytes32 packing (koalabears_to_bn254), the digest of
// RecursionPublicValues, and the recursion vk map (RecursionVks, crates/prover/src/recursion.rs:59-170): a Poseidon2 Merkle tree over the
// digests of every allowed recursion key, built on the device by the commitment code's tree kernels and then kept on the host, where
// opening a key is a lookup.  The shards themselves are verified by verify_shards (verify.cu): host phases on several threads, the device
// work of a whole batch of proofs in one launch per kernel.
#include "ctx.cuh"
#include "challenger.cuh"
#include "hostfield.hpp"
#include "sumcheck.cuh"
#include "verify.cuh"
#include <algorithm>
#include <chrono>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>

struct sp1b200_recursion_vks {
    uint32_t root[8];
    uint32_t log_h = 0;
    bool vk_verification = false;
    std::vector<uint32_t> keys;     // [n][8] Montgomery words, in canonical lexicographic order; key i is leaf i
    std::vector<uint32_t> layers;   // all 2^(log_h+1) - 1 digests bottom-up (merkle.cu's layout), leaves at bit-reversed positions
};

namespace {

// RecursionPublicValues<F> (crates/recursion/executor/src/public_values.rs:39-143): the fields in declaration order and their widths
namespace rpv {
enum Field {
    PREV_COMMITTED_VALUE_DIGEST, COMMITTED_VALUE_DIGEST, PREV_DEFERRED_PROOFS_DIGEST, DEFERRED_PROOFS_DIGEST, PREV_DEFERRED_PROOF,
    DEFERRED_PROOF, PC_START, NEXT_PC, INITIAL_TIMESTAMP, LAST_TIMESTAMP, PREVIOUS_INIT_ADDR, LAST_INIT_ADDR, PREVIOUS_FINALIZE_ADDR,
    LAST_FINALIZE_ADDR, PREVIOUS_INIT_PAGE_IDX, LAST_INIT_PAGE_IDX, PREVIOUS_FINALIZE_PAGE_IDX, LAST_FINALIZE_PAGE_IDX,
    START_RECONSTRUCT_DEFERRED_DIGEST, END_RECONSTRUCT_DEFERRED_DIGEST, SP1_VK_DIGEST, VK_ROOT, GLOBAL_CUMULATIVE_SUM,
    CONTAINS_FIRST_SHARD, NUM_INCLUDED_SHARD, IS_COMPLETE, PREV_EXIT_CODE, EXIT_CODE, PREV_COMMIT_SYSCALL, COMMIT_SYSCALL,
    PREV_COMMIT_DEFERRED_SYSCALL, COMMIT_DEFERRED_SYSCALL, DIGEST, PROOF_NONCE, N_FIELDS
};
constexpr uint32_t WIDTH[N_FIELDS] = {32, 32, 8, 8, 1, 1, 3, 3, 4, 4, 3, 3, 3, 3, 3, 3, 3, 3, 8, 8, 8, 8, 14, 1, 1, 1, 1, 1, 1, 1, 1, 1, 8, 4};
constexpr uint32_t at(int f) { return f == 0 ? 0 : at(f - 1) + WIDTH[f - 1]; }
constexpr uint32_t NUM_ELTS = at(N_FIELDS);   // RECURSIVE_PROOF_NUM_PV_ELTS = PROOF_MAX_NUM_PVS
constexpr uint32_t NUM_TO_HASH = at(DIGEST);  // NUM_PV_ELMS_TO_HASH: every word before `digest`
}  // namespace rpv
static_assert(rpv::NUM_ELTS == 187 && rpv::NUM_TO_HASH == 175 && rpv::at(rpv::PROOF_NONCE) == 183, "recursion public values layout");
static_assert(rpv::at(rpv::SP1_VK_DIGEST) == 136 && rpv::at(rpv::VK_ROOT) == 144 && rpv::at(rpv::IS_COMPLETE) == 168, "recursion public values layout");

constexpr uint32_t VK_HASHED_TAIL = 18;   // the tail words hash_koalabear reads (the padding is observed, not hashed)
constexpr uint32_t VK_WORDS = 8 + VK_TAIL_WORDS;
constexpr uint32_t MAX_PATH = 64;
constexpr uint32_t MAX_LOG_KEYS = 26;     // 2^26 leaves: a 4 GiB tree on the device

const char* const COMPRESSED_NAMES[SP1B200_VERDICT_COMPRESSED_COUNT - SP1B200_VERDICT_RECURSION_PV_DIGEST] = {
    "InvalidPublicValues(recursion public values are invalid)",
    "InvalidPublicValues(vk_root mismatch)",
    "InvalidVerificationKey",
    "InvalidPublicValues(is_complete is not 1)",
    "InvalidPublicValues(sp1 vk hash mismatch)",
    "UninitializedVerificationKey",
};

// reverse_bits_len (crates/primitives): the low `bits` bits of x reversed; higher bits are dropped
uint64_t reverse_bits_len(uint64_t x, uint32_t bits) {
    uint64_t r = 0;
    for (uint32_t i = 0; i < bits; i++) r |= ((x >> i) & 1) << (bits - 1 - i);
    return r;
}

// canonical lexicographic order of two digests (the BTreeMap order of [SP1Field; 8])
bool key_less(const uint32_t* a, const uint32_t* b) {
    for (int i = 0; i < 8; i++) {
        const uint32_t x = kb::to_canonical(a[i]), y = kb::to_canonical(b[i]);
        if (x != y) return x < y;
    }
    return false;
}

// hash_koalabear without mprotect (crates/hypercube/src/verifier/hashable_key.rs:94-118): poseidon2_hash of the preprocessed commitment,
// pc_start, initial_global_cumulative_sum x and y, enable_untrusted_programs
void vk_hash(const uint32_t* commit8, const uint32_t* tail, uint32_t* out8) {
    uint32_t in[8 + VK_HASHED_TAIL];
    memcpy(in, commit8, 32);
    memcpy(in + 8, tail, 4 * VK_HASHED_TAIL);
    host_hash(in, 8 + VK_HASHED_TAIL, out8);
}

// verify_merkle_proof (crates/hypercube/src/verifier/proof.rs:121-143)
bool merkle_proof_holds(const uint32_t* leaf8, uint64_t index, const uint32_t* path, uint32_t n_path, const uint32_t* root8) {
    uint32_t v[8];
    memcpy(v, leaf8, 32);
    uint64_t idx = reverse_bits_len(index, n_path);
    for (uint32_t k = 0; k < n_path; k++, idx >>= 1) {
        if (idx & 1) host_compress(path + 8 * k, v, v); else host_compress(v, path + 8 * k, v);
    }
    return !memcmp(v, root8, 32);
}

// the checks of verify_compressed after verify_shard (verify.rs:549-577) on an accepted proof: -> verdict
uint32_t check_after_shard(const uint32_t* pv, const uint32_t* key, const sp1b200_recursion_vks& vks, uint64_t index, const uint32_t* path,
                           uint32_t n_path, const uint32_t* sp1_vk_digest8) {
    uint32_t d[8];
    host_hash(pv, rpv::NUM_TO_HASH, d);
    if (memcmp(d, pv + rpv::at(rpv::DIGEST), 32)) return SP1B200_VERDICT_RECURSION_PV_DIGEST;
    if (memcmp(pv + rpv::at(rpv::VK_ROOT), vks.root, 32)) return SP1B200_VERDICT_VK_ROOT;
    if (vks.vk_verification) {
        vk_hash(key, key + 8, d);
        if (!merkle_proof_holds(d, index, path, n_path, vks.root)) return SP1B200_VERDICT_INVALID_VERIFICATION_KEY;
    }
    if (pv[rpv::at(rpv::IS_COMPLETE)] != kb::ONE) return SP1B200_VERDICT_IS_COMPLETE;
    if (memcmp(pv + rpv::at(rpv::SP1_VK_DIGEST), sp1_vk_digest8, 32)) return SP1B200_VERDICT_SP1_VK_DIGEST;
    return SP1B200_VERDICT_ACCEPT;
}

}  // namespace

const char* verify_compressed_verdict_name(uint32_t verdict) {
    if (verdict < SP1B200_VERDICT_RECURSION_PV_DIGEST || verdict >= SP1B200_VERDICT_COMPRESSED_COUNT) return nullptr;
    return COMPRESSED_NAMES[verdict - SP1B200_VERDICT_RECURSION_PV_DIGEST];
}

extern "C" {

sp1b200_err sp1b200_vk_hash(const uint32_t* h_prep_commit8, const uint32_t* h_vk_tail, uint32_t n_vk_tail, uint32_t* h_out8) {
    if (!h_prep_commit8 || !h_vk_tail || !h_out8) return sp1b200_set_error("vk_hash: NULL argument");
    if (n_vk_tail != VK_TAIL_WORDS)
        return sp1b200_set_error("vk_hash: n_vk_tail is %u; the verifying key without mprotect has %u words after the commitment", n_vk_tail, VK_TAIL_WORDS);
    if (!hf::canonical(h_prep_commit8, 8) || !hf::canonical(h_vk_tail, n_vk_tail)) return sp1b200_set_error("vk_hash: a key word is not canonical");
    vk_hash(h_prep_commit8, h_vk_tail, h_out8);
    return nullptr;
}

sp1b200_err sp1b200_digest_bytes32(const uint32_t* h_digest8, uint8_t* h_out32) {
    if (!h_digest8 || !h_out32) return sp1b200_set_error("digest_bytes32: NULL argument");
    if (!hf::canonical(h_digest8, 8)) return sp1b200_set_error("digest_bytes32: a digest word is not canonical");
    // Σ_i c_i · 2^(31 (7 - i)) < 2^248 < r: no reduction; big-endian, so byte 0 is always zero
    memset(h_out32, 0, 32);
    for (uint32_t i = 0; i < 8; i++) {
        const uint32_t c = kb::to_canonical(h_digest8[i]);
        for (uint32_t b = 0; b < 31; b++) {
            const uint32_t pos = 31 * (7 - i) + b;
            h_out32[31 - pos / 8] |= (uint8_t)(((c >> b) & 1) << (pos % 8));
        }
    }
    return nullptr;
}

sp1b200_err sp1b200_recursion_pv_digest(const uint32_t* h_pv187, uint32_t* h_out8) {
    if (!h_pv187 || !h_out8) return sp1b200_set_error("recursion_pv_digest: NULL argument");
    host_hash(h_pv187, rpv::NUM_TO_HASH, h_out8);
    return nullptr;
}

sp1b200_err sp1b200_recursion_vks_create(sp1b200_ctx* ctx, const uint32_t* h_digests, uint64_t n, uint64_t pad_to, int vk_verification,
                                         sp1b200_recursion_vks** out) {
    SP1_DEVICE_GUARD(ctx);
    if (!ctx || !out || (n && !h_digests)) return sp1b200_set_error("recursion_vks_create: NULL argument");
    *out = nullptr;
    const uint64_t max_keys = (uint64_t)1 << MAX_LOG_KEYS;
    if (n > max_keys || pad_to > max_keys) return sp1b200_set_error("recursion_vks_create: more than 2^%u keys", MAX_LOG_KEYS);
    if (!hf::canonical(h_digests, 8 * n)) return sp1b200_set_error("recursion_vks_create: a digest word is not canonical");
    // RecursionVks::from_map: the keys, then [i; 8] for every missing index below pad_to, deduplicated and sorted
    std::vector<uint32_t> all(h_digests, h_digests + 8 * n);
    std::vector<uint32_t> order;
    auto sort_unique = [&] {
        order.resize(all.size() / 8);
        for (uint32_t i = 0; i < order.size(); i++) order[i] = i;
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key_less(&all[8 * a], &all[8 * b]); });
        order.erase(std::unique(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return !memcmp(&all[8 * a], &all[8 * b], 32); }), order.end());
    };
    sort_unique();
    for (uint64_t i = order.size(); i < pad_to; i++) all.insert(all.end(), 8, kb::to_monty_c(i));
    if (pad_to > order.size()) sort_unique();
    const uint64_t nk = order.size();
    if (nk < 2) return sp1b200_set_error("recursion_vks_create: %llu key(s); the tree needs at least two", (unsigned long long)nk);
    std::unique_ptr<sp1b200_recursion_vks> v(new sp1b200_recursion_vks);
    v->vk_verification = vk_verification != 0;
    v->keys.resize(8 * nk);
    for (uint64_t i = 0; i < nk; i++) memcpy(&v->keys[8 * i], &all[8 * (size_t)order[i]], 32);
    uint32_t log_h = 0;
    while (((uint64_t)1 << log_h) < nk) log_h++;
    v->log_h = log_h;
    const uint64_t h = (uint64_t)1 << log_h;
    // MerkleTree::commit (crates/recursion/circuit/src/basefold/merkle_tree.rs:24-64): zero-padded, leaves bit-reversed
    v->layers.assign((2 * h - 1) * 8, 0);
    for (uint64_t i = 0; i < nk; i++) memcpy(&v->layers[8 * reverse_bits_len(i, log_h)], &v->keys[8 * i], 32);
    {
        DevFree mem(ctx);
        uint32_t *d_layers, *d_root;
        SP1_TRY(mem.alloc((void**)&d_layers, v->layers.size() * 4));
        SP1_TRY(mem.alloc((void**)&d_root, 16 * 4));
        SP1_CUDA(cudaMemcpyAsync(d_layers, v->layers.data(), h * 32, cudaMemcpyHostToDevice, ctx->stream));
        PhaseTimer t(ctx, "recursion_vks.tree");
        SP1_TRY(sp1b200_merkle_tree_from_leaves_device(ctx, d_layers, log_h, 8, d_root));
        t.stop();
        SP1_CUDA(cudaMemcpyAsync(v->layers.data(), d_layers, v->layers.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
        SP1_CUDA(cudaMemcpyAsync(v->root, d_root, 32, cudaMemcpyDeviceToHost, ctx->stream));
        SP1_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    *out = v.release();
    return nullptr;
}

void sp1b200_recursion_vks_free(sp1b200_recursion_vks* vks) { delete vks; }

void sp1b200_recursion_vks_root(const sp1b200_recursion_vks* vks, uint32_t* h_out8) { memcpy(h_out8, vks->root, 32); }

uint64_t sp1b200_recursion_vks_num_keys(const sp1b200_recursion_vks* vks) { return vks->keys.size() / 8; }

sp1b200_err sp1b200_recursion_vks_open(const sp1b200_recursion_vks* vks, const uint32_t* h_digest8, uint64_t* h_index, uint32_t* h_path,
                                       uint32_t path_cap, uint32_t* h_n_path) {
    if (!vks || !h_digest8 || !h_index || !h_n_path) return sp1b200_set_error("recursion_vks_open: NULL argument");
    if (!hf::canonical(h_digest8, 8)) return sp1b200_set_error("recursion_vks_open: a digest word is not canonical");
    const uint64_t nk = vks->keys.size() / 8;
    uint64_t lo = 0, hi = nk;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        if (key_less(&vks->keys[8 * mid], h_digest8)) lo = mid + 1; else hi = mid;
    }
    if (lo == nk || memcmp(&vks->keys[8 * lo], h_digest8, 32)) return sp1b200_set_error("recursion_vks_open: vk not allowed (the digest is not in the map)");
    *h_index = lo;
    *h_n_path = vks->log_h;
    if (path_cap < vks->log_h) return sp1b200_set_error("recursion_vks_open: path_cap %u is below the path length %u", path_cap, vks->log_h);
    if (!h_path) return sp1b200_set_error("recursion_vks_open: NULL argument");
    // MerkleTree::open (merkle_tree.rs:66-88): from the bit-reversed leaf position, the sibling in every layer
    const uint64_t h = (uint64_t)1 << vks->log_h;
    uint64_t pos = reverse_bits_len(lo, vks->log_h);
    for (uint32_t k = 0; k < vks->log_h; k++, pos >>= 1)
        memcpy(h_path + 8 * k, &vks->layers[8 * ((2 * h - (2 * h >> k)) + (pos ^ 1))], 32);
    return nullptr;
}

sp1b200_err sp1b200_verify_compressed(sp1b200_ctx* ctx, const sp1b200_machine* m, const sp1b200_recursion_vks* vks, uint32_t mode,
                                      const uint32_t* h_shrink_vk, uint32_t n_proofs, const uint32_t* h_vks, const uint64_t* h_heights,
                                      const char* const* chip_names, const uint32_t* const* h_proofs, const uint64_t* h_n_words,
                                      const uint64_t* h_vk_index, const uint32_t* const* h_vk_paths, const uint32_t* h_vk_path_len,
                                      const uint32_t* h_sp1_vk_digests, uint32_t host_threads, uint32_t* h_final_challengers,
                                      uint32_t* h_verdicts, uint32_t* h_shard_verdicts) {
    SP1_DEVICE_GUARD(ctx);
    if (!ctx || !m || !vks || !h_verdicts || !h_shard_verdicts) return sp1b200_set_error("verify_compressed: NULL argument");
    if (!n_proofs) return sp1b200_set_error("verify_compressed: no proofs");
    if (!h_vks || !h_heights || !chip_names || !h_proofs || !h_n_words || !h_vk_index || !h_vk_paths || !h_vk_path_len || !h_sp1_vk_digests)
        return sp1b200_set_error("verify_compressed: NULL argument");
    if (mode != SP1B200_COMPRESSED && mode != SP1B200_SHRINK) return sp1b200_set_error("verify_compressed: mode %u is neither compressed nor shrink", mode);
    if (mode == SP1B200_COMPRESSED && h_shrink_vk) return sp1b200_set_error("verify_compressed: a shrink key in compressed mode");
    if (h_shrink_vk && !hf::canonical(h_shrink_vk, VK_WORDS)) return sp1b200_set_error("verify_compressed: the shrink key is not canonical");
    const auto t0 = std::chrono::steady_clock::now();
    const size_t nch = m->chips.size();
    bool has_prep = false;
    for (auto& c : m->chips) has_prep |= c.prep_w != 0;
    // every proof parses; keys, paths and expected digests are canonical
    std::vector<std::unique_ptr<VerifyShardIn>> in;
    for (uint32_t s = 0; s < n_proofs; s++) {
        const std::string who = "verify_compressed: proof " + std::to_string(s);
        if (!h_proofs[s]) return sp1b200_set_error("%s: NULL proof", who.c_str());
        const uint32_t* key = h_vks + (size_t)VK_WORDS * s;
        if (!hf::canonical(key, VK_WORDS)) return sp1b200_set_error("%s: a verifying-key word is not canonical", who.c_str());
        if (h_vk_path_len[s] > MAX_PATH) return sp1b200_set_error("%s: vk Merkle path of %u digests, more than %u", who.c_str(), h_vk_path_len[s], MAX_PATH);
        if (h_vk_path_len[s] && !h_vk_paths[s]) return sp1b200_set_error("%s: NULL vk Merkle path", who.c_str());
        if (!hf::canonical(h_vk_paths[s], 8 * (size_t)h_vk_path_len[s])) return sp1b200_set_error("%s: a vk Merkle path word is not canonical", who.c_str());
        if (!hf::canonical(h_sp1_vk_digests + 8 * (size_t)s, 8)) return sp1b200_set_error("%s: the SP1 vk digest is not canonical", who.c_str());
        in.emplace_back(new VerifyShardIn);
        SP1_TRY(verify_parse_shard(ctx, m, has_prep ? key : nullptr, h_heights + (size_t)s * nch, chip_names, h_proofs[s], h_n_words[s], who,
                                   *in.back()));
    }
    // verify.rs:582-590 (shrink mode), then the public values' length (verify.rs:535-538)
    std::vector<uint32_t> verdict(n_proofs, SP1B200_VERDICT_ACCEPT), shard_verdict(n_proofs, 0);
    for (uint32_t s = 0; s < n_proofs; s++) {
        if (mode == SP1B200_SHRINK && !h_shrink_vk) verdict[s] = SP1B200_VERDICT_UNINITIALIZED_VERIFICATION_KEY;
        else if (mode == SP1B200_SHRINK && memcmp(h_vks + (size_t)VK_WORDS * s, h_shrink_vk, 4 * VK_WORDS)) verdict[s] = SP1B200_VERDICT_INVALID_VERIFICATION_KEY;
        else if (in[s]->p.n_pv != rpv::NUM_ELTS) verdict[s] = SP1B200_VERDICT_PV_LENGTH;
    }
    // verify_shard of the rest, each from a fresh transcript that observed its own key (observe_into), in batches of at most
    // verify_batch_words_cap() proof words
    std::vector<uint32_t> starts(34 * (size_t)n_proofs), finals(34 * (size_t)n_proofs);
    std::vector<uint32_t> todo;
    for (uint32_t s = 0; s < n_proofs; s++) {
        if (verdict[s]) continue;
        HostChallenger ch;
        uint32_t zero[34] = {0};
        ch.load(zero);
        ch.observe_n(h_vks + (size_t)VK_WORDS * s, VK_WORDS);
        ch.store(&starts[34 * (size_t)s]);
        todo.push_back(s);
    }
    if (!host_threads) host_threads = std::max(1u, std::thread::hardware_concurrency());
    VerifyTimes t;
    const uint64_t cap = verify_batch_words_cap();
    for (size_t a = 0; a < todo.size();) {
        size_t b = a + 1;
        uint64_t words = h_n_words[todo[a]];
        while (b < todo.size() && words + h_n_words[todo[b]] <= cap) words += h_n_words[todo[b++]];
        std::vector<const VerifyShardIn*> batch;
        std::vector<const uint32_t*> st;
        for (size_t i = a; i < b; i++) { batch.push_back(in[todo[i]].get()); st.push_back(&starts[34 * (size_t)todo[i]]); }
        std::vector<uint32_t> vd(batch.size()), fin(34 * batch.size());
        SP1_TRY(verify_shards(ctx, m, chip_names, batch, st, host_threads, vd.data(), fin.data(), t));
        for (size_t i = a; i < b; i++) {
            const uint32_t s = todo[i];
            if (vd[i - a]) { verdict[s] = SP1B200_VERDICT_INVALID_SHARD_PROOF; shard_verdict[s] = vd[i - a]; continue; }
            memcpy(&finals[34 * (size_t)s], &fin[34 * (i - a)], 34 * 4);
            verdict[s] = check_after_shard(in[s]->p.pv, h_vks + (size_t)VK_WORDS * s, *vks, h_vk_index[s], h_vk_paths[s], h_vk_path_len[s],
                                           h_sp1_vk_digests + 8 * (size_t)s);
        }
        a = b;
    }
    ctx->phase_ms["verify_compressed.host"] = (float)t.host_ms;
    ctx->phase_ms["verify_compressed.kernels"] = t.merkle + t.fold + t.jagged;
    ctx->phase_ms["verify_compressed.total"] = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    memcpy(h_verdicts, verdict.data(), 4 * (size_t)n_proofs);
    memcpy(h_shard_verdicts, shard_verdict.data(), 4 * (size_t)n_proofs);
    if (h_final_challengers)
        for (uint32_t s = 0; s < n_proofs; s++)
            if (!verdict[s]) memcpy(h_final_challengers + 34 * (size_t)s, &finals[34 * (size_t)s], 34 * 4);
    return nullptr;
}

}  // extern "C"
