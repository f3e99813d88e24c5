// Shapes of the core machine's three lookup-table chips (Byte, Program, Range), shared by the preprocessed tables of a program
// (program_tables.cu) and the multiplicity tables of a shard (lookup_traces.cu): both halves of a chip must have the same height.
#pragma once
#include "ctx.cuh"
#include <algorithm>
#include <cstdint>

namespace core_tables {

constexpr uint64_t BYTE_ROWS = 1u << 16;    // bytes/trace.rs:15 NUM_ROWS
constexpr uint64_t RANGE_ROWS = 1u << 17;   // range/trace.rs:15 NUM_ROWS

// next_multiple_of_32(n, None) (hypercube/src/util.rs:50-59): the Program table's height.  Only Program::preprocessed_shape = None is
// implemented.  For a later fixed-shape path: trusted.rs:91-92 passes `fixed_log2_rows` to next_multiple_of_32 as its fixed *height*;
// read Shape::log2_height before assuming whether a height or its log is meant.
inline uint64_t program_height(uint64_t n) { return std::max<uint64_t>((n + 31) / 32 * 32, 16); }

// a program of n >= 1 instructions at pc_base: its Program table fits 2^max_log_row_count rows and every pc = pc_base + 4 idx is below
// 2^48 (trusted.rs:117-118); `what` prefixes the messages
inline sp1b200_err check_program_window(sp1b200_ctx* ctx, const char* what, uint64_t pc_base, uint64_t n) {
    const uint32_t mlr = ctx->params.max_log_row_count;
    if (n > ((uint64_t)1 << 40) || program_height(n) > ((uint64_t)1 << mlr))
        return sp1b200_set_error("%s: %llu instructions give a Program table of %llu rows > 2^%u (max_log_row_count)", what,
                                 (unsigned long long)n, (unsigned long long)program_height(n), mlr);
    const uint64_t lim = (uint64_t)1 << 48;
    if (pc_base >= lim || 4 * (n - 1) >= lim - pc_base) {
        const uint64_t i = pc_base >= lim ? 0 : (lim - pc_base + 3) / 4;
        return sp1b200_set_error("%s: instruction %llu has pc 0x%llx + 4 * %llu >= 2^48", what, (unsigned long long)i,
                                 (unsigned long long)pc_base, (unsigned long long)i);
    }
    return nullptr;
}

}  // namespace core_tables
