// sp1b200_air_prover.hpp — the host side above the C ABI in C++ (the reference's host language, Rust, is absent from this image).
//
// Mirrors the trait the reference selects its shard prover through, `sp1_hypercube::prover::AirProver<GC, SC>`
// (crates/hypercube/src/prover/shard.rs:45-101): same method names, argument meaning and error behaviour
//   machine()                       -> the chips (name order) this prover was built for
//   setup(...)                      -> setup_from_vk plus the verifying key's words computed from the program's memory image; given the
//                                      instruction list, the core machine's preprocessed tables are generated on the device too
//   setup_from_vk(...)              -> commits the preprocessed traces once per program, returns the proving key
//                                      (`PreprocessedData<ProvingKey>`) and the preprocessed commitment of the verifying key
//   setup_and_prove_shard(...)      -> setup, observe the verifying key, prove (the vk-less path of the first shard of a program)
//   prove_shard_with_pk(pk, record) -> the shard proof for one execution record (here: its main traces in the dense layout)
//   preprocessed_table_heights(pk)  -> chip name -> height of its preprocessed table
// The reference implementations are infallible by signature and panic on failure (worker maps the panic to TaskError::Fatal);
// here every failure throws sp1b200::Error carrying the library's message.  One AirProver owns one context (= one CUDA stream,
// pool, mailbox and pair of upload slots) and proves one shard at a time; hold several per GPU for throughput (DESIGN.md 3.4).
// Header-only over include/sp1b200.h; link with -lsp1b200.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <map>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "sp1b200.h"

namespace sp1b200 {

struct Error : std::runtime_error {
    explicit Error(const char* msg) : std::runtime_error(msg) {}
};
inline void check(sp1b200_err e) {
    if (e) throw Error(e);
}

using Digest = std::array<uint32_t, SP1B200_DIGEST_WORDS>;
using Challenger = std::array<uint32_t, SP1B200_CHALLENGER_WORDS>;  // sponge[16] input[8] output[8] n_in n_out

// one chip of the machine, in the order the reference iterates them (BTreeSet by name)
struct Chip {
    std::string name;
    uint32_t main_width = 0;
    uint32_t preprocessed_width = 0;
};

// `ProvingKey` + device-resident preprocessed data (reference: PreprocessedData<ProvingKey<GC, SC, Self>>)
class ProvingKey {
  public:
    ProvingKey() = default;
    ProvingKey(ProvingKey&& o) noexcept { *this = std::move(o); }
    ProvingKey& operator=(ProvingKey&& o) noexcept {
        release();
        ctx_ = o.ctx_; round_ = o.round_; commit = o.commit; heights = std::move(o.heights);
        o.round_ = nullptr;
        return *this;
    }
    ProvingKey(const ProvingKey&) = delete;
    ProvingKey& operator=(const ProvingKey&) = delete;
    ~ProvingKey() { release(); }

    Digest commit{};                           // preprocessed commitment (MachineVerifyingKey::preprocessed_commit)
    std::map<std::string, uint64_t> heights;   // chip name -> preprocessed table height

  private:
    friend class AirProver;
    void release() {
        if (round_) sp1b200_jagged_round_free(ctx_, round_);
        round_ = nullptr;
    }
    sp1b200_ctx* ctx_ = nullptr;
    sp1b200_jagged_round* round_ = nullptr;
};

// What setup needs of a program (MachineProgram: pc_start_abs, memory_image and page_prot_image as parallel arrays in any order, host or
// device memory, enable_untrusted_programs)
struct ProgramImage {
    uint64_t pc_start_abs = 0;
    const uint64_t* mem_addrs = nullptr;
    const uint64_t* mem_words = nullptr;
    uint64_t n_mem = 0;
    const uint64_t* page_idx = nullptr;
    const uint8_t* page_prot = nullptr;
    uint64_t n_pages = 0;
    bool enable_untrusted_programs = false;
};

// MachineVerifyingKey as the library's calls take it: the preprocessed commitment and the 24 words observed after it
// (pc_start[3], initial_global_cumulative_sum x[7] y[7], enable_untrusted_programs, six zeros)
struct VerifyingKeyWords {
    Digest preprocessed_commit{};
    std::vector<uint32_t> tail;
};

class AirProver {
  public:
    // chips in name order; machine_blob = the constraint bytecode + interactions of every chip (sp1b200_machine_create)
    AirProver(int device, const sp1b200_params& params, std::vector<Chip> chips, const std::vector<uint32_t>& machine_blob)
        : params_(params), chips_(std::move(chips)) {
        check(sp1b200_ctx_create(device, &params, &ctx_));
        sp1b200_err e = sp1b200_machine_create(ctx_, machine_blob.data(), machine_blob.size(), &machine_);
        if (e) { std::string m = e; sp1b200_ctx_destroy(ctx_); throw Error(m.c_str()); }
        if (sp1b200_machine_num_chips(machine_) != chips_.size()) {
            sp1b200_machine_free(ctx_, machine_); sp1b200_ctx_destroy(ctx_);
            throw Error("AirProver: the machine blob and the chip list disagree on the number of chips");
        }
    }
    AirProver(const AirProver&) = delete;
    AirProver& operator=(const AirProver&) = delete;
    ~AirProver() {
        if (machine_) sp1b200_machine_free(ctx_, machine_);
        if (ctx_) sp1b200_ctx_destroy(ctx_);
    }

    static sp1b200_params core_params() {
        sp1b200_params p;
        sp1b200_default_core_params(&p);
        return p;
    }

    const std::vector<Chip>& machine() const { return chips_; }

    // AirProver::setup_from_vk: `prep_dense_any` holds the preprocessed tables of the chips that have preprocessed columns,
    // back to back in chip order, each column-major [preprocessed_width x height]; heights[i] = height of chip i's tables
    // (0 for an absent chip).  Returns the proving key; pk.commit is the preprocessed commitment.
    ProvingKey setup_from_vk(const uint32_t* prep_dense_any, const std::vector<uint64_t>& heights) {
        if (heights.size() != chips_.size()) throw Error("setup_from_vk: one height per chip expected");
        std::vector<uint64_t> rows, cols;
        ProvingKey pk;
        for (size_t k = 0; k < chips_.size(); k++)
            if (chips_[k].preprocessed_width) {
                rows.push_back(heights[k]); cols.push_back(chips_[k].preprocessed_width);
                pk.heights[chips_[k].name] = heights[k];
            }
        pk.ctx_ = ctx_;
        if (!rows.empty())
            check(sp1b200_jagged_commit(ctx_, prep_dense_any, (uint32_t)rows.size(), rows.data(), cols.data(), 1, pk.commit.data(), &pk.round_));
        return pk;
    }

    // AirProver::setup (shard.rs:88-95 -> setup_from_vk(program, None), shard.rs:259-290): the proving key as setup_from_vk makes it and
    // the verifying key, whose initial global cumulative sum is computed from the program's memory image on the device
    // (sp1b200_program_vk_tail).  The image is checked before anything is committed.
    std::pair<ProvingKey, VerifyingKeyWords> setup(const uint32_t* prep_dense_any, const std::vector<uint64_t>& heights, const ProgramImage& program) {
        VerifyingKeyWords vk;
        vk.tail.resize(24);
        check(sp1b200_program_vk_tail(ctx_, program.pc_start_abs, program.mem_addrs, program.mem_words, program.n_mem, program.page_idx,
                                      program.page_prot, program.n_pages, program.enable_untrusted_programs ? 1 : 0, vk.tail.data()));
        ProvingKey pk = setup_from_vk(prep_dense_any, heights);
        vk.preprocessed_commit = pk.commit;
        return {std::move(pk), std::move(vk)};
    }

    // AirProver::setup(program) for a core program given by its instructions (Program::instructions, pc_base; host or device memory) and
    // its image: the Byte, Program and Range preprocessed tables are generated and committed on the device (sp1b200_program_setup), so no
    // trace crosses the bus.  The machine's chips with preprocessed columns must be exactly Byte (7 columns), Program (16) and Range (2).
    // Only Program::preprocessed_shape = None is implemented.  Returns the proving key, the verifying key words and the key's digest
    // (MachineVerifyingKey::hash_koalabear; sp1b200_digest_bytes32 of it is vk.bytes32()).
    struct ProgramSetup {
        ProvingKey pk;
        VerifyingKeyWords vk;
        Digest vk_digest{};
    };
    ProgramSetup setup(uint64_t pc_base, const sp1b200_instruction* instrs_any, uint64_t n_instrs, const ProgramImage& image) {
        static const std::pair<const char*, uint32_t> prep_chips[3] = {
            {"Byte", SP1B200_BYTE_PREP_COLS}, {"Program", SP1B200_PROGRAM_PREP_COLS}, {"Range", SP1B200_RANGE_PREP_COLS}};
        size_t t = 0;
        for (const Chip& c : chips_)
            if (c.preprocessed_width) {
                if (t == 3 || c.name != prep_chips[t].first || c.preprocessed_width != prep_chips[t].second)
                    throw Error("setup(program): the chips with preprocessed columns must be Byte (7), Program (16) and Range (2)");
                t++;
            }
        if (t != 3) throw Error("setup(program): the chips with preprocessed columns must be Byte (7), Program (16) and Range (2)");
        ProgramSetup out;
        out.vk.tail.resize(24);
        uint64_t rows[3];
        check(sp1b200_program_setup(ctx_, pc_base, instrs_any, n_instrs, image.pc_start_abs, image.mem_addrs, image.mem_words, image.n_mem,
                                    image.page_idx, image.page_prot, image.n_pages, image.enable_untrusted_programs ? 1 : 0, 1, rows,
                                    out.pk.commit.data(), out.vk.tail.data(), out.vk_digest.data(), &out.pk.round_));
        out.pk.ctx_ = ctx_;
        for (int k = 0; k < 3; k++) out.pk.heights[prep_chips[k].first] = rows[k];
        out.vk.preprocessed_commit = out.pk.commit;
        return out;
    }

    // The shard's Byte, Program and Range main traces (ByteChip / RangeChip / ProgramChip::generate_trace_into) generated on the device
    // from record.byte_lookups and the pcs of the shard's instruction events (sp1b200_lookup_traces), written straight into their slices
    // of main_dense_any: the dense main buffer of prove_shard_with_pk (device memory, or host memory before an upload), laid out for
    // `heights` in chip order.  public_values non-empty (the 187 words prove_shard_with_pk takes) adds the lookups of the two chips'
    // generate_dependencies.  The chips must include Byte (6 main columns), Program (1) and Range (1) at the heights the call reports.
    void lookup_traces(uint32_t* main_dense_any, const std::vector<uint64_t>& heights, uint64_t pc_base, uint64_t n_instrs,
                       const sp1b200_byte_lookup* lookups_any, uint64_t n_lookups, const sp1b200_pc_count* pcs_any, uint64_t n_pcs,
                       const std::vector<uint32_t>& public_values) {
        if (heights.size() != chips_.size()) throw Error("lookup_traces: one height per chip expected");
        uint64_t rows[3];
        check(sp1b200_lookup_traces(ctx_, pc_base, n_instrs, lookups_any, n_lookups, pcs_any, n_pcs, nullptr, 0, nullptr, nullptr, nullptr,
                                    rows));
        static const std::pair<const char*, uint32_t> chips[3] = {
            {"Byte", SP1B200_BYTE_MULT_COLS}, {"Program", SP1B200_PROGRAM_MULT_COLS}, {"Range", SP1B200_RANGE_MULT_COLS}};
        uint32_t* out[3] = {nullptr, nullptr, nullptr};
        uint64_t off = 0;
        for (size_t k = 0; k < chips_.size(); k++) {
            for (int t = 0; t < 3; t++)
                if (chips_[k].name == chips[t].first) {
                    if (chips_[k].main_width != chips[t].second || heights[k] != rows[t])
                        throw Error((std::string("lookup_traces: chip ") + chips[t].first + " has another main width or height").c_str());
                    out[t] = main_dense_any + off;
                }
            off += heights[k] * chips_[k].main_width;
        }
        if (!out[0] || !out[1] || !out[2]) throw Error("lookup_traces: the machine lacks one of Byte, Program and Range");
        check(sp1b200_lookup_traces(ctx_, pc_base, n_instrs, lookups_any, n_lookups, pcs_any, n_pcs,
                                    public_values.empty() ? nullptr : public_values.data(), (uint32_t)public_values.size(), out[0], out[1],
                                    out[2], nullptr));
    }

    // The shard's MemoryGlobalInit, MemoryGlobalFinalize and MemoryLocal main traces (MemoryGlobalChip / MemoryLocalChip::
    // generate_trace_into) generated on the device from record.global_memory_initialize_events / _finalize_events and
    // get_local_mem_events() (sp1b200_memory_traces), written straight into their slices of main_dense_any (laid out for `heights` in chip
    // order, as for lookup_traces).  previous_*_addr: the shard's public values of those names.  The chips' generate_dependencies go to
    // lookups_out_any (12 records per init / finalize event + 10 per local event: pass them to lookup_traces with the shard's other
    // lookups) and globals_out_any (one record per init / finalize event + 2 per local event, in sections init, finalize, local); both host
    // or device memory.  A chip the machine lacks must have no events; one it has must be at the height the call reports (0 without
    // events).  Returns {lookup records, global records} written.
    std::pair<uint64_t, uint64_t> memory_traces(uint32_t* main_dense_any, const std::vector<uint64_t>& heights,
                                                const sp1b200_memory_event* init_any, uint64_t n_init, const sp1b200_memory_event* finalize_any,
                                                uint64_t n_finalize, uint64_t previous_init_addr, uint64_t previous_finalize_addr,
                                                const sp1b200_memory_local_event* local_any, uint64_t n_local,
                                                sp1b200_byte_lookup* lookups_out_any, sp1b200_global_event* globals_out_any) {
        if (heights.size() != chips_.size()) throw Error("memory_traces: one height per chip expected");
        uint64_t rows[3], n_lookups = 0, n_globals = 0;
        check(sp1b200_memory_traces(ctx_, init_any, n_init, finalize_any, n_finalize, previous_init_addr, previous_finalize_addr, local_any,
                                    n_local, nullptr, nullptr, nullptr, nullptr, nullptr, rows, &n_lookups, &n_globals));
        static const std::pair<const char*, uint32_t> chips[3] = {{"MemoryGlobalInit", SP1B200_MEMORY_GLOBAL_COLS},
                                                                  {"MemoryGlobalFinalize", SP1B200_MEMORY_GLOBAL_COLS},
                                                                  {"MemoryLocal", SP1B200_MEMORY_LOCAL_COLS}};
        uint32_t* out[3] = {nullptr, nullptr, nullptr};
        uint64_t off = 0;
        for (size_t k = 0; k < chips_.size(); k++) {
            for (int t = 0; t < 3; t++)
                if (chips_[k].name == chips[t].first) {
                    if (chips_[k].main_width != chips[t].second || heights[k] != rows[t])
                        throw Error((std::string("memory_traces: chip ") + chips[t].first + " has another main width or height").c_str());
                    out[t] = main_dense_any + off;
                }
            off += heights[k] * chips_[k].main_width;
        }
        for (int t = 0; t < 3; t++)
            if (rows[t] && !out[t]) throw Error((std::string("memory_traces: the machine lacks ") + chips[t].first + ", which has events").c_str());
        check(sp1b200_memory_traces(ctx_, init_any, n_init, finalize_any, n_finalize, previous_init_addr, previous_finalize_addr, local_any,
                                    n_local, out[0], out[1], out[2], lookups_out_any, globals_out_any, nullptr, nullptr, nullptr));
        return {n_lookups, n_globals};
    }

    // AirProver::preprocessed_table_heights
    static const std::map<std::string, uint64_t>& preprocessed_table_heights(const ProvingKey& pk) { return pk.heights; }

    // Asynchronous upload of the NEXT record's main traces from pinned host memory into slot 0 / 1; returns the pointer to
    // hand to prove_shard_with_pk (the reference overlaps trace generation / transfer with proving the same way).
    const uint32_t* upload_begin(const uint32_t* h_main_dense, uint64_t n_words, int slot) {
        uint32_t* d = nullptr;
        check(sp1b200_upload_begin(ctx_, h_main_dense, n_words, slot, &d));
        return d;
    }

    // AirProver::prove_shard_with_pk.  main_dense_any: every chip's main trace back to back in chip order, column-major
    // [main_width x height] (host pointer, device pointer or an upload slot); heights: one per chip (0 = absent, must equal
    // the preprocessed height where the chip has one).  `challenger` is the transcript state on entry (the verifying key has
    // been observed by the caller, shard.rs:660-672) and on return.  Returns the flat proof words:
    // [5][section lengths] main commitment | LogUp-GKR | zerocheck + opened values | evaluation proof | public values.
    std::vector<uint32_t> prove_shard_with_pk(const ProvingKey& pk, const uint32_t* main_dense_any, const std::vector<uint64_t>& heights,
                                              const std::vector<uint32_t>& public_values, Challenger& challenger,
                                              const uint32_t* replay_witnesses = nullptr) {
        if (heights.size() != chips_.size()) throw Error("prove_shard_with_pk: one height per chip expected");
        std::vector<const char*> names;
        for (const Chip& c : chips_) names.push_back(c.name.c_str());
        if (proof_buf_.size() < kCapWords) proof_buf_.resize(kCapWords);
        uint64_t n = 0;
        check(sp1b200_prove_shard(ctx_, machine_, pk.round_, main_dense_any, heights.data(), names.data(), public_values.data(),
                                  (uint32_t)public_values.size(), replay_witnesses, challenger.data(), proof_buf_.data(), kCapWords, &n));
        return std::vector<uint32_t>(proof_buf_.begin(), proof_buf_.begin() + n);
    }

    // AirProver::setup_and_prove_shard (shard.rs:56-68): setup + MachineVerifyingKey::observe_into + prove in one call.
    // `challenger` is the transcript BEFORE the verifying key is observed; vk_tail = the words observed after the preprocessed
    // commitment (pc_start[3], initial_global_cumulative_sum x[7] y[7], enable_untrusted_programs, six zeros; config.rs:97-112).
    // Returns (proving key - its commit is the vk's preprocessed_commit -, proof words).
    std::pair<ProvingKey, std::vector<uint32_t>> setup_and_prove_shard(const uint32_t* prep_dense_any, const uint32_t* main_dense_any,
                                                                       const std::vector<uint64_t>& heights, const std::vector<uint32_t>& vk_tail,
                                                                       const std::vector<uint32_t>& public_values, Challenger& challenger,
                                                                       const uint32_t* replay_witnesses = nullptr) {
        if (heights.size() != chips_.size()) throw Error("setup_and_prove_shard: one height per chip expected");
        std::vector<uint64_t> rows, cols;
        std::vector<const char*> names;
        ProvingKey pk;
        for (size_t k = 0; k < chips_.size(); k++) {
            names.push_back(chips_[k].name.c_str());
            if (chips_[k].preprocessed_width) {
                rows.push_back(heights[k]); cols.push_back(chips_[k].preprocessed_width);
                pk.heights[chips_[k].name] = heights[k];
            }
        }
        pk.ctx_ = ctx_;
        if (proof_buf_.size() < kCapWords) proof_buf_.resize(kCapWords);
        uint64_t n = 0;
        check(sp1b200_setup_and_prove_shard(ctx_, machine_, prep_dense_any, (uint32_t)rows.size(), rows.data(), cols.data(), vk_tail.data(),
                                            (uint32_t)vk_tail.size(), main_dense_any, heights.data(), names.data(), public_values.data(),
                                            (uint32_t)public_values.size(), replay_witnesses, challenger.data(), pk.commit.data(), &pk.round_,
                                            proof_buf_.data(), kCapWords, &n));
        return {std::move(pk), std::vector<uint32_t>(proof_buf_.begin(), proof_buf_.begin() + n)};
    }

    // ShardVerifier::verify_shard (crates/hypercube/src/verifier/shard.rs:437-750) on proof words of prove_shard_with_pk /
    // setup_and_prove_shard (sp1b200_verify_shard).  prep_commit: the verifying key's preprocessed commitment (nullptr when no chip has
    // preprocessed columns); `challenger` is the transcript after the verifying key was observed, the state the prover started from.
    // On acceptance `challenger` becomes the verifier's final state (equal to the prover's); on rejection it is left unchanged and the
    // verdict names the first failing check.  Words that do not parse as a proof of this machine throw.
    struct Verdict {
        uint32_t code = SP1B200_VERDICT_ACCEPT;
        std::string reason;
        bool accepted() const { return code == SP1B200_VERDICT_ACCEPT; }
    };
    Verdict verify_shard(const Digest* prep_commit, const std::vector<uint32_t>& proof_words, const std::vector<uint64_t>& heights,
                         Challenger& challenger) {
        if (heights.size() != chips_.size()) throw Error("verify_shard: one height per chip expected");
        std::vector<const char*> names;
        for (const Chip& c : chips_) names.push_back(c.name.c_str());
        Verdict v;
        check(sp1b200_verify_shard(ctx_, machine_, prep_commit ? prep_commit->data() : nullptr, heights.data(), names.data(), proof_words.data(),
                                   proof_words.size(), challenger.data(), &v.code));
        v.reason = sp1b200_verdict_name(v.code);
        return v;
    }

    // SP1Prover::verify (crates/prover/src/verify.rs:109-524) on a core proof: the proof words of every shard of one execution, with
    // each shard's chip heights, against the verifying key prep_commit + vk_tail (24 words, as setup_and_prove_shard takes them;
    // sp1b200_verify_core_proof).  Shards that do not parse throw.  On acceptance final_challengers holds each shard verifier's final
    // state; for InvalidShardProof, `shard` is the lowest failing shard and shard_code / shard_reason its verify_shard verdict.
    struct CoreVerdict {
        uint32_t code = SP1B200_VERDICT_ACCEPT, shard = 0, shard_code = SP1B200_VERDICT_ACCEPT;
        std::string reason, shard_reason;
        std::vector<Challenger> final_challengers;
        bool accepted() const { return code == SP1B200_VERDICT_ACCEPT; }
    };
    CoreVerdict verify_core_proof(const Digest& prep_commit, const std::vector<uint32_t>& vk_tail,
                                  const std::vector<std::vector<uint32_t>>& shard_words, const std::vector<std::vector<uint64_t>>& heights,
                                  uint32_t host_threads = 0) {
        if (heights.size() != shard_words.size()) throw Error("verify_core_proof: one height list per shard expected");
        std::vector<const char*> names;
        for (const Chip& c : chips_) names.push_back(c.name.c_str());
        std::vector<uint64_t> h, nw;
        std::vector<const uint32_t*> words;
        for (size_t s = 0; s < shard_words.size(); s++) {
            if (heights[s].size() != chips_.size()) throw Error("verify_core_proof: one height per chip expected");
            h.insert(h.end(), heights[s].begin(), heights[s].end());
            words.push_back(shard_words[s].data());
            nw.push_back(shard_words[s].size());
        }
        std::vector<uint32_t> fin(34 * shard_words.size());
        CoreVerdict v;
        check(sp1b200_verify_core_proof(ctx_, machine_, prep_commit.data(), vk_tail.data(), (uint32_t)vk_tail.size(), (uint32_t)shard_words.size(),
                                        h.data(), names.data(), words.data(), nw.data(), host_threads, fin.data(), &v.code, &v.shard,
                                        &v.shard_code));
        v.reason = sp1b200_verdict_name(v.code);
        v.shard_reason = sp1b200_verdict_name(v.shard_code);
        if (v.accepted())
            for (size_t s = 0; s < shard_words.size(); s++) {
                Challenger c;
                std::copy(fin.begin() + 34 * s, fin.begin() + 34 * (s + 1), c.data());
                v.final_challengers.push_back(c);
            }
        return v;
    }

    // SP1Prover::verify_compressed / verify_shrink (crates/prover/src/verify.rs:527-642) of recursion proofs of this machine
    // (sp1b200_verify_compressed): each with its own key (prep_commit[8] | vk_tail[24]), chip heights, proof words, vk Merkle proof
    // (sp1b200_recursion_vks_open) and the SP1 program key digest it must be for.  shrink_vk != nullptr selects shrink mode, checked
    // against *shrink_vk; shrink mode without a key is SP1B200_SHRINK with shrink_vk_missing = true.  Proofs that do not parse throw.
    struct RecursionProof {
        std::vector<uint32_t> vk;                       // 32 words
        std::vector<uint64_t> heights;
        std::vector<uint32_t> words;
        uint64_t vk_index = 0;
        std::vector<Digest> vk_path;
        Digest sp1_vk_digest{};
    };
    struct CompressedVerdict {
        uint32_t code = SP1B200_VERDICT_ACCEPT, shard_code = SP1B200_VERDICT_ACCEPT;
        std::string reason, shard_reason;
        Challenger final_challenger{};
        bool accepted() const { return code == SP1B200_VERDICT_ACCEPT; }
    };
    std::vector<CompressedVerdict> verify_compressed(const sp1b200_recursion_vks* vks, const std::vector<RecursionProof>& proofs,
                                                     const std::vector<uint32_t>* shrink_vk = nullptr, bool shrink_vk_missing = false,
                                                     uint32_t host_threads = 0) {
        std::vector<const char*> names;
        for (const Chip& c : chips_) names.push_back(c.name.c_str());
        std::vector<uint32_t> keys, digests, path_len;
        std::vector<uint64_t> h, nw, index;
        std::vector<const uint32_t*> words, paths;
        for (const RecursionProof& p : proofs) {
            if (p.heights.size() != chips_.size()) throw Error("verify_compressed: one height per chip expected");
            if (p.vk.size() != 32) throw Error("verify_compressed: a verifying key has 32 words");
            keys.insert(keys.end(), p.vk.begin(), p.vk.end());
            h.insert(h.end(), p.heights.begin(), p.heights.end());
            words.push_back(p.words.data());
            nw.push_back(p.words.size());
            index.push_back(p.vk_index);
            paths.push_back(p.vk_path.empty() ? nullptr : p.vk_path[0].data());
            path_len.push_back((uint32_t)p.vk_path.size());
            digests.insert(digests.end(), p.sp1_vk_digest.begin(), p.sp1_vk_digest.end());
        }
        const bool shrink = shrink_vk || shrink_vk_missing;
        if (shrink_vk && shrink_vk->size() != 32) throw Error("verify_compressed: the shrink key has 32 words");
        std::vector<uint32_t> fin(34 * proofs.size()), code(proofs.size()), shard_code(proofs.size());
        check(sp1b200_verify_compressed(ctx_, machine_, vks, shrink ? SP1B200_SHRINK : SP1B200_COMPRESSED, shrink_vk ? shrink_vk->data() : nullptr,
                                        (uint32_t)proofs.size(), keys.data(), h.data(), names.data(), words.data(), nw.data(), index.data(),
                                        paths.data(), path_len.data(), digests.data(), host_threads, fin.data(), code.data(), shard_code.data()));
        std::vector<CompressedVerdict> out(proofs.size());
        for (size_t s = 0; s < proofs.size(); s++) {
            out[s].code = code[s];
            out[s].shard_code = shard_code[s];
            out[s].reason = sp1b200_verdict_name(code[s]);
            out[s].shard_reason = sp1b200_verdict_name(shard_code[s]);
            if (out[s].accepted()) std::copy(fin.begin() + 34 * s, fin.begin() + 34 * (s + 1), out[s].final_challenger.data());
        }
        return out;
    }

    // bincode(ShardProof) of a proof returned by prove_shard_with_pk / setup_and_prove_shard: the bytes the reference's workers, recursion
    // tree and verifier exchange (crates/hypercube/src/verifier/proof.rs:47-61; sp1b200_shard_proof_to_bincode)
    std::vector<uint8_t> to_bincode(const std::vector<uint32_t>& proof_words, const std::vector<uint64_t>& heights) const {
        if (heights.size() != chips_.size()) throw Error("to_bincode: one height per chip expected");
        std::vector<const char*> names; std::vector<uint32_t> mw, pw;
        for (const auto& c : chips_) { names.push_back(c.name.c_str()); mw.push_back(c.main_width); pw.push_back(c.preprocessed_width); }
        uint64_t n = 0;
        check(sp1b200_shard_proof_to_bincode(&params_, (uint32_t)chips_.size(), names.data(), heights.data(), mw.data(), pw.data(), proof_words.data(),
                                             proof_words.size(), nullptr, 0, &n));
        std::vector<uint8_t> out(n);
        check(sp1b200_shard_proof_to_bincode(&params_, (uint32_t)chips_.size(), names.data(), heights.data(), mw.data(), pw.data(), proof_words.data(),
                                             proof_words.size(), out.data(), out.size(), &n));
        return out;
    }

    // The reference's cfg(sp1_debug_constraints) checks on the inputs of prove_shard_with_pk (nothing of the transcript is touched).
    // debug_constraints: chips whose real rows violate a constraint, each with its number of failing rows and the failed constraint
    // indices of its lowest max_rows failing rows (crates/hypercube/src/debug.rs:27-130; the reference prints three rows per chip).
    struct FailingRow { uint32_t row; std::vector<uint32_t> constraints; };
    struct FailingChip { uint32_t chip; uint32_t n_failing_rows; std::vector<FailingRow> rows; };
    std::vector<FailingChip> debug_constraints(const ProvingKey& pk, const uint32_t* main_dense_any, const std::vector<uint64_t>& heights,
                                               const std::vector<uint32_t>& public_values, uint32_t max_rows = 3) {
        if (heights.size() != chips_.size()) throw Error("debug_constraints: one height per chip expected");
        std::vector<uint32_t> w = report([&](uint32_t* out, uint64_t cap, uint64_t* n) {
            return sp1b200_debug_constraints(ctx_, machine_, pk.round_, main_dense_any, heights.data(), public_values.data(),
                                             (uint32_t)public_values.size(), max_rows, out, cap, n);
        });
        std::vector<FailingChip> out(w[0]);
        size_t p = 1;
        for (FailingChip& c : out) {
            c.chip = w[p]; c.n_failing_rows = w[p + 1]; c.rows.resize(w[p + 2]); p += 3;
            for (FailingRow& r : c.rows) { r.row = w[p]; r.constraints.assign(w.begin() + p + 2, w.begin() + p + 2 + w[p + 1]); p += 2 + w[p + 1]; }
        }
        return out;
    }
    // debug_interactions: the keys (kind, values) whose sends and receives do not balance, in order of first occurrence, with every
    // chip that has a record of the key (crates/hypercube/src/lookup/debug.rs:48-200)
    struct UnbalancedKey {
        uint32_t kind; std::vector<uint32_t> values; uint32_t net;
        uint32_t first_chip, first_interaction, first_row;
        std::vector<std::pair<uint32_t, uint32_t>> chips;   // (chip, net)
    };
    struct InteractionReport { uint64_t n_unbalanced = 0; std::vector<UnbalancedKey> keys; };
    InteractionReport debug_interactions(const ProvingKey& pk, const uint32_t* main_dense_any, const std::vector<uint64_t>& heights,
                                         uint32_t max_keys = 16) {
        if (heights.size() != chips_.size()) throw Error("debug_interactions: one height per chip expected");
        std::vector<uint32_t> w = report([&](uint32_t* out, uint64_t cap, uint64_t* n) {
            return sp1b200_debug_interactions(ctx_, machine_, pk.round_, main_dense_any, heights.data(), max_keys, out, cap, n);
        });
        InteractionReport r;
        r.n_unbalanced = w[0] | ((uint64_t)w[1] << 32);
        r.keys.resize(w[2]);
        size_t p = 3;
        for (UnbalancedKey& k : r.keys) {
            k.kind = w[p]; k.values.assign(w.begin() + p + 2, w.begin() + p + 2 + w[p + 1]); p += 2 + w[p + 1];
            k.net = w[p]; k.first_chip = w[p + 1]; k.first_interaction = w[p + 2]; k.first_row = w[p + 3];
            k.chips.resize(w[p + 4]); p += 5;
            for (auto& c : k.chips) { c = {w[p], w[p + 1]}; p += 2; }
        }
        return r;
    }

    sp1b200_ctx* context() const { return ctx_; }

  private:
    // a report call, retried once with the capacity the library asks for
    template <class Call>
    static std::vector<uint32_t> report(Call call) {
        std::vector<uint32_t> w(1 << 16);
        uint64_t n = 0;
        sp1b200_err e = call(w.data(), w.size(), &n);
        if (e && n > w.size()) { w.resize(n); e = call(w.data(), w.size(), &n); }
        check(e);
        w.resize(n);
        return w;
    }
    static constexpr uint64_t kCapWords = 1ull << 24;
    sp1b200_params params_;
    sp1b200_ctx* ctx_ = nullptr;
    sp1b200_machine* machine_ = nullptr;
    std::vector<Chip> chips_;
    std::vector<uint32_t> proof_buf_;
};

}  // namespace sp1b200
