// Host-side Fiat-Shamir transcript object of the library (DuplexChallenger<KoalaBear, Poseidon2-16, 16, 8>).
// Like the reference's GPU prover, the transcript itself lives on the host (it absorbs a few hundred words per
// shard: digests and round polynomials copied back from the device) -- sp1-gpu/crates/shard_prover/src/prover.rs:618-763;
// semantics sp1-gpu/crates/sys/include/challenger/challenger.cuh:22-112.  Only the PoW grind runs on the device.
#pragma once
#include "ctx.cuh"
#include "hostfield.hpp"
#include <cstring>
#include <utility>
#include <vector>

void host_poseidon2_permute(uint32_t* s16);
// PaddingFreeSponge<16, 8, 8> (overwrite mode) and the 2-to-1 compression, with the transcript's permutation
void host_hash(const uint32_t* in, size_t n, uint32_t* out8);
void host_compress(const uint32_t* l8, const uint32_t* r8, uint32_t* out8);
// a jagged round's commitment: compress(original, hash(n_tables | rows of every table | columns of every table)); tables: (rows, cols)
void table_size_commitment(const uint32_t* original8, const std::vector<std::pair<uint64_t, uint64_t>>& tables, uint32_t* out8);

struct HostChallenger {
    sp1b200_ctx* ctx = nullptr;
    uint32_t sponge[16], inbuf[8], outbuf[8];
    uint32_t nin = 0, nout = 0;
    uint32_t* d_scratch = nullptr;

    sp1b200_err init(sp1b200_ctx* c, const uint32_t* st34);
    ~HostChallenger();
    void load(const uint32_t* st34);
    void store(uint32_t* st34) const;
    void duplexing();
    void observe(uint32_t v);
    void observe_n(const uint32_t* v, size_t n);
    uint32_t sample();
    void sample_ext(uint32_t* out4);
    uint32_t sample_bits(uint32_t bits);
    bool check_witness(uint32_t bits, uint32_t w_monty);
    sp1b200_err grind(uint32_t bits, uint32_t* w_monty);  // device search, canonical-min witness
};

// Transcript steps the shard prover and the shard verifier share.
// The chip shapes after the main commitment (shard.rs): the chip count, then per chip its height and its name (length, then bytes).
void observe_chip_shapes(HostChallenger& ch, size_t n_chips, const uint64_t* heights, const char* const* names);
// A chip's γ-batched opening claim Σ_j γ^(j+1) o_j over its opened values, main columns then preprocessed ones (ext each).
hf::E4 batched_opening_claim(const uint32_t* main, uint32_t main_w, const uint32_t* prep, uint32_t prep_w, const hf::E4& gamma);
