// Program setup from the instruction list: the preprocessed tables of the core machine's three chips with preprocessed columns (Byte,
// Program, Range; generate_preprocessed_trace_into exists only in crates/core/machine/src/{bytes/trace.rs, program/trusted.rs,
// range/trace.rs}), written on the device straight into the dense layout sp1b200_jagged_commit takes, and the whole verifying key built
// on top of them.  One thread writes one row; the commitment that follows dominates the call.
#include "core_tables.hpp"
#include "ctx.cuh"
#include "sumcheck.cuh"
#include <algorithm>
#include <cstddef>
#include <cstring>

static_assert(sizeof(sp1b200_instruction) == 24, "sp1b200_instruction is 24 bytes");
static_assert(offsetof(sp1b200_instruction, opcode) == 0 && offsetof(sp1b200_instruction, op_a) == 1 &&
                  offsetof(sp1b200_instruction, imm_b) == 2 && offsetof(sp1b200_instruction, imm_c) == 3 &&
                  offsetof(sp1b200_instruction, op_b) == 8 && offsetof(sp1b200_instruction, op_c) == 16,
              "sp1b200_instruction field offsets");

namespace {

using core_tables::BYTE_ROWS;
using core_tables::RANGE_ROWS;
using core_tables::program_height;
constexpr uint32_t BYTE_COLS = SP1B200_BYTE_PREP_COLS, PROGRAM_COLS = SP1B200_PROGRAM_PREP_COLS, RANGE_COLS = SP1B200_RANGE_PREP_COLS;
constexpr uint64_t NONE = ~0ull;

// canonical x < p -> Montgomery word
__device__ __forceinline__ uint32_t mont(uint32_t x) { return kb::monty_reduce((uint64_t)x * kb::RR); }

// Byte and Range: thread r < 2^17 writes Range row r and, for r < 2^16, Byte row r.  d_byte: [7 x 2^16], d_range: [2 x 2^17].
__global__ void __launch_bounds__(256) fixed_tables_kernel(uint32_t* __restrict__ d_byte, uint32_t* __restrict__ d_range) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= RANGE_ROWS) return;
    if (r < BYTE_ROWS) {
        // ByteChip::trace (bytes/mod.rs:31-80): row 256 b + c of (0..=255).cartesian_product(0..=255); columns BytePreprocessedCols
        // (bytes/columns.rs) b, c, and, or, xor, ltu, msb for the byte_table opcodes (executor/src/events/byte.rs:166-176); U8Range
        // has no column
        const uint32_t b = r >> 8, c = r & 0xFF;
        const uint32_t v[BYTE_COLS] = {b, c, b & c, b | c, b ^ c, b < c ? 1u : 0u, (b & 0x80) ? 1u : 0u};
#pragma unroll
        for (uint32_t k = 0; k < BYTE_COLS; k++) d_byte[k * BYTE_ROWS + r] = mont(v[k]);
    }
    // RangeChip::trace (range/mod.rs:18-39): row 0 = (0, 0); row 2^bits + a = (a, bits) for 0 <= bits <= 16, a < 2^bits
    const uint32_t bits = r ? 31 - __clz(r) : 0;
    const uint32_t a = r ? r - (1u << bits) : 0;
    d_range[r] = mont(a);
    d_range[RANGE_ROWS + r] = mont(bits);
}

// Program (trusted.rs:80-127 generate_preprocessed_trace_into, instruction.rs:36-45 InstructionCols::populate): row r of h rows, r < n
// the instruction r, every padding row a copy of row 0 (trusted.rs:113-115 resets idx to 0 before pc is computed).  Columns
// ProgramPreprocessedCols: pc[3] (16-bit limbs 0..16 / 16..32 / 32..48 of pc_base + 4 idx), opcode, op_a, op_b[4], op_c[4] (Word::from(u64),
// hypercube/src/word.rs:167-176: 16-bit limbs, low first), op_a_0 = (op_a == X0), imm_b, imm_c.  Malformed instructions leave their index
// in bad[0] (opcode), bad[1] (imm_b), bad[2] (imm_c), the lowest index winning.
__global__ void __launch_bounds__(256) program_table_kernel(const sp1b200_instruction* __restrict__ instrs, uint64_t n, uint64_t h,
                                                            uint64_t pc_base, uint32_t* __restrict__ d_prog, unsigned long long* bad) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= h) return;
    const uint64_t idx = r < n ? r : 0;
    const sp1b200_instruction in = instrs[idx];
    if (r < n) {
        if (in.opcode > SP1B200_MAX_OPCODE) atomicMin(bad, (unsigned long long)r);
        if (in.imm_b > 1) atomicMin(bad + 1, (unsigned long long)r);
        if (in.imm_c > 1) atomicMin(bad + 2, (unsigned long long)r);
    }
    const uint64_t pc = pc_base + 4 * idx;
    const uint32_t v[PROGRAM_COLS] = {
        (uint32_t)(pc & 0xFFFF), (uint32_t)((pc >> 16) & 0xFFFF), (uint32_t)((pc >> 32) & 0xFFFF),
        in.opcode, in.op_a,
        (uint32_t)(in.op_b & 0xFFFF), (uint32_t)((in.op_b >> 16) & 0xFFFF), (uint32_t)((in.op_b >> 32) & 0xFFFF), (uint32_t)(in.op_b >> 48),
        (uint32_t)(in.op_c & 0xFFFF), (uint32_t)((in.op_c >> 16) & 0xFFFF), (uint32_t)((in.op_c >> 32) & 0xFFFF), (uint32_t)(in.op_c >> 48),
        in.op_a == 0 ? 1u : 0u, in.imm_b, in.imm_c};
#pragma unroll
    for (uint32_t k = 0; k < PROGRAM_COLS; k++) d_prog[k * h + r] = mont(v[k]);
}

struct Shapes {
    uint64_t rows[3], cols[3], words;
};
Shapes shapes_of(uint64_t n) {
    Shapes s{{BYTE_ROWS, program_height(n), RANGE_ROWS}, {BYTE_COLS, PROGRAM_COLS, RANGE_COLS}, 0};
    for (int t = 0; t < 3; t++) s.words += s.rows[t] * s.cols[t];
    return s;
}

// the host checks of both entry points; `what` prefixes the messages
sp1b200_err check_program(sp1b200_ctx* ctx, const char* what, uint64_t pc_base, const void* instrs_any, uint64_t n) {
    if (!ctx) return sp1b200_set_error("%s: NULL context", what);
    if (n == 0) return sp1b200_set_error("%s: empty program (no instructions)", what);
    if (!instrs_any) return sp1b200_set_error("%s: NULL instruction list with %llu instructions", what, (unsigned long long)n);
    return core_tables::check_program_window(ctx, what, pc_base, n);
}

// writes the three tables back to back (Byte, Program, Range; each column-major) into d_out, then reports the lowest malformed instruction
sp1b200_err write_tables(sp1b200_ctx* ctx, const char* what, uint64_t pc_base, const sp1b200_instruction* instrs_any, uint64_t n,
                         const Shapes& s, uint32_t* d_out) {
    cudaStream_t st = ctx->stream;
    DevFree mem(ctx);
    DevBuf instrs;
    SP1_TRY(instrs.in(ctx, instrs_any, n * sizeof(sp1b200_instruction)));
    unsigned long long* d_bad;
    SP1_TRY(mem.alloc((void**)&d_bad, 3 * 8));
    SP1_CUDA(cudaMemsetAsync(d_bad, 0xff, 3 * 8, st));
    uint32_t* d_byte = d_out;
    uint32_t* d_prog = d_byte + s.rows[0] * s.cols[0];
    uint32_t* d_range = d_prog + s.rows[1] * s.cols[1];
    SP1_LAUNCH(ctx, fixed_tables_kernel, blocks_for(RANGE_ROWS), 256, 0, d_byte, d_range);
    SP1_LAUNCH(ctx, program_table_kernel, blocks_for(s.rows[1]), 256, 0, (const sp1b200_instruction*)instrs.d, n, s.rows[1], pc_base,
               d_prog, d_bad);
    unsigned long long bad[3];
    SP1_CUDA(cudaMemcpyAsync(bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, st));
    SP1_CUDA(cudaStreamSynchronize(st));
    const uint64_t first = std::min(bad[0], std::min(bad[1], bad[2]));
    if (first != NONE) {
        sp1b200_instruction in;
        SP1_CUDA(cudaMemcpy(&in, (const sp1b200_instruction*)instrs.d + first, sizeof(in), cudaMemcpyDeviceToHost));
        if (bad[0] == first)
            return sp1b200_set_error("%s: instruction %llu has opcode %u (the largest Opcode is %u)", what, (unsigned long long)first,
                                     in.opcode, (unsigned)SP1B200_MAX_OPCODE);
        return sp1b200_set_error("%s: instruction %llu has %s = %u, not 0 or 1", what, (unsigned long long)first,
                                 bad[1] == first ? "imm_b" : "imm_c", bad[1] == first ? in.imm_b : in.imm_c);
    }
    return instrs.finish();
}

}  // namespace

extern "C" sp1b200_err sp1b200_program_preprocessed_traces(sp1b200_ctx* ctx, uint64_t pc_base, const sp1b200_instruction* instrs_any,
                                                           uint64_t n_instrs, uint32_t* out_any, uint64_t cap_words, uint64_t* h_rows3,
                                                           uint64_t* h_cols3, uint64_t* h_words) {
    SP1_DEVICE_GUARD(ctx);
    const char* what = "program_preprocessed_traces";
    SP1_TRY(check_program(ctx, what, pc_base, instrs_any, n_instrs));
    const Shapes s = shapes_of(n_instrs);
    if (h_rows3) for (int t = 0; t < 3; t++) h_rows3[t] = s.rows[t];
    if (h_cols3) for (int t = 0; t < 3; t++) h_cols3[t] = s.cols[t];
    if (h_words) *h_words = s.words;
    if (!out_any) return nullptr;   // a size query
    if (cap_words < s.words)
        return sp1b200_set_error("%s: the tables need %llu words, capacity %llu", what, (unsigned long long)s.words, (unsigned long long)cap_words);
    DevBuf out;
    SP1_TRY(out.out(ctx, out_any, s.words * 4));
    SP1_TRY(write_tables(ctx, what, pc_base, instrs_any, n_instrs, s, (uint32_t*)out.d));
    return out.finish();
}

extern "C" sp1b200_err sp1b200_program_setup(sp1b200_ctx* ctx, uint64_t pc_base, const sp1b200_instruction* instrs_any, uint64_t n_instrs,
                                             uint64_t pc_start_abs, const uint64_t* mem_addrs_any, const uint64_t* mem_words_any,
                                             uint64_t n_mem, const uint64_t* page_idx_any, const uint8_t* page_prot_any, uint64_t n_pages,
                                             int enable_untrusted_programs, int keep_codeword, uint64_t* h_prep_rows3,
                                             uint32_t* h_prep_commit8, uint32_t* h_vk_tail24, uint32_t* h_vk_digest8,
                                             sp1b200_jagged_round** prep_round_out) {
    SP1_DEVICE_GUARD(ctx);
    const char* what = "program_setup";
    SP1_TRY(check_program(ctx, what, pc_base, instrs_any, n_instrs));
    if (!h_prep_commit8 || !h_vk_tail24 || !h_vk_digest8) return sp1b200_set_error("%s: NULL output", what);
    const Shapes s = shapes_of(n_instrs);
    uint32_t tail[24];
    sp1b200_jagged_round* round = nullptr;
    {
        DevFree mem(ctx);
        uint32_t* d_dense;
        SP1_TRY(mem.alloc((void**)&d_dense, s.words * 4));
        PhaseTimer t_all(ctx, "program_setup");
        {
            PhaseTimer t(ctx, "program_setup.tables");
            SP1_TRY(write_tables(ctx, what, pc_base, instrs_any, n_instrs, s, d_dense));
            t.stop();
        }
        // the memory image is checked before anything is committed
        {
            PhaseTimer t(ctx, "program_setup.vk_tail");
            SP1_TRY(sp1b200_program_vk_tail(ctx, pc_start_abs, mem_addrs_any, mem_words_any, n_mem, page_idx_any, page_prot_any, n_pages,
                                            enable_untrusted_programs, tail));
            t.stop();
        }
        {
            PhaseTimer t(ctx, "program_setup.commit");
            SP1_TRY(sp1b200_jagged_commit(ctx, d_dense, 3, s.rows, s.cols, keep_codeword, h_prep_commit8, &round));
            t.stop();
        }
        t_all.stop();
    }
    sp1b200_err e = sp1b200_vk_hash(h_prep_commit8, tail, 24, h_vk_digest8);
    if (e) { sp1b200_jagged_round_free(ctx, round); return e; }
    memcpy(h_vk_tail24, tail, sizeof(tail));
    if (h_prep_rows3) for (int t = 0; t < 3; t++) h_prep_rows3[t] = s.rows[t];
    if (prep_round_out) *prep_round_out = round;
    else sp1b200_jagged_round_free(ctx, round);
    return nullptr;
}
