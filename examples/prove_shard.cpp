// Compiled host above the C ABI: proves one shard through sp1b200::AirProver (include/sp1b200_air_prover.hpp), the C++ mirror of
// the reference's `AirProver` trait.  Input / output are flat little-endian u32 files (written / read by tests/test_gpu_example.py):
//
//   input : "SP1B" 1 | params[8] | n_chips | per chip { name_len, name bytes (padded to 4), main_w, prep_w, height } |
//           n_blob, blob | n_pv, pv | challenger[34] | n_prep, prep dense | n_main, main dense
//   output: prep commit[8] | n_words, proof words | challenger[34]
//
// build: g++ -O2 -std=c++17 -Iinclude examples/prove_shard.cpp -Lsp1_b200 -lsp1b200 -Wl,-rpath,$PWD/sp1_b200 -o examples/prove_shard
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>

#include "sp1b200_air_prover.hpp"

namespace {
std::vector<uint32_t> read_all(const char* path) {
    std::ifstream f(path, std::ios::binary | std::ios::ate);
    if (!f) throw std::runtime_error(std::string("cannot open ") + path);
    const std::streamsize n = f.tellg();
    f.seekg(0);
    std::vector<uint32_t> w((size_t)n / 4);
    f.read(reinterpret_cast<char*>(w.data()), (std::streamsize)w.size() * 4);
    return w;
}
struct Reader {
    const std::vector<uint32_t>& w; size_t i = 0;
    uint32_t u() { if (i >= w.size()) throw std::runtime_error("truncated input"); return w[i++]; }
    std::vector<uint32_t> vec() { uint32_t n = u(); if (i + n > w.size()) throw std::runtime_error("truncated input"); std::vector<uint32_t> v(w.begin() + i, w.begin() + i + n); i += n; return v; }
};
}  // namespace

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: %s input.bin output.bin\n", argv[0]); return 2; }
    try {
        const std::vector<uint32_t> in = read_all(argv[1]);
        Reader r{in};
        if (r.u() != 0x42315053u || r.u() != 1) throw std::runtime_error("bad magic / version");
        sp1b200_params params;
        uint32_t* pw = reinterpret_cast<uint32_t*>(&params);
        for (int k = 0; k < 8; k++) pw[k] = r.u();
        const uint32_t n_chips = r.u();
        std::vector<sp1b200::Chip> chips(n_chips);
        std::vector<uint64_t> heights(n_chips);
        for (uint32_t c = 0; c < n_chips; c++) {
            const uint32_t len = r.u();
            const size_t words = (len + 3) / 4;
            if (r.i + words > in.size()) throw std::runtime_error("truncated input");
            chips[c].name.assign(reinterpret_cast<const char*>(&in[r.i]), len);
            r.i += words;
            chips[c].main_width = r.u(); chips[c].preprocessed_width = r.u(); heights[c] = r.u();
        }
        const std::vector<uint32_t> blob = r.vec(), pv = r.vec();
        sp1b200::Challenger ch;
        for (auto& x : ch) x = r.u();
        const std::vector<uint32_t> prep = r.vec(), main_dense = r.vec();

        sp1b200::AirProver prover(0, params, chips, blob);
        sp1b200::ProvingKey pk = prover.setup_from_vk(prep.data(), heights);
        sp1b200::Challenger vch = ch;   // the verifier starts from the same post-vk transcript
        const std::vector<uint32_t> proof = prover.prove_shard_with_pk(pk, main_dense.data(), heights, pv, ch);
        // check the proof just made before it leaves this process
        bool has_prep = false;
        for (const auto& c : chips) has_prep |= c.preprocessed_width != 0;
        const sp1b200::AirProver::Verdict verdict = prover.verify_shard(has_prep ? &pk.commit : nullptr, proof, heights, vch);
        std::printf("verify_shard: %s\n", verdict.reason.c_str());
        if (!verdict.accepted() || vch != ch) { std::fprintf(stderr, "prove_shard: the proof does not verify (%s)\n", verdict.reason.c_str()); return 1; }

        std::ofstream out(argv[2], std::ios::binary);
        out.write(reinterpret_cast<const char*>(pk.commit.data()), 32);
        const uint32_t n = (uint32_t)proof.size();
        out.write(reinterpret_cast<const char*>(&n), 4);
        out.write(reinterpret_cast<const char*>(proof.data()), (std::streamsize)proof.size() * 4);
        out.write(reinterpret_cast<const char*>(ch.data()), 34 * 4);
        std::printf("proved %u chips: %u proof words, %zu preprocessed tables (%s)\n", n_chips, n, pk.heights.size(), sp1b200_version());
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "prove_shard: %s\n", e.what());
        return 1;
    }
}
