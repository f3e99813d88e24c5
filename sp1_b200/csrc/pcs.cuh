// Device-resident prover data shared by jagged.cu and shard.cu.
#pragma once
#include "proof_layout.hpp"
#include <cstdint>
#include <vector>

struct sp1b200_commit;

struct sp1b200_jagged_round {
    sp1b200_commit* stacked = nullptr;
    layout::Tables tables;  // including the two padding tables
    uint64_t area = 0, padded_area = 0;
    uint32_t* d_dense = nullptr;  // owned, padded_area words
    uint32_t original_commit[8], commit[8];
};
