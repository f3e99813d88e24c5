// A shard's multiplicity traces of the core machine's three lookup-table chips (the main halves of Byte, Program and Range; the
// preprocessed halves come from program_tables.cu), generated on the device from the shard's byte lookups and executed pcs:
// ByteChip / RangeChip::generate_trace_into (crates/core/machine/src/{bytes,range}/trace.rs) read record.byte_lookups,
// ProgramChip::generate_trace_into (program/trusted.rs:134-292) counts the pcs of the shard's instruction events.
//
// The work is a keyed histogram: one pass over each record stream adds every record's count into 64-bit counters in the context's
// pool (Byte 6 x 2^16, Range 2^17, Program h), then one pass checks every counter against p and writes the three column-major tables
// as Montgomery words.  Zero-byte range checks and a loop's pcs take most of the hits, so equal keys are first summed inside the warp
// (__match_any_sync) and one lane per distinct key issues the atomic.  Integer sums make the words independent of the record order.
#include "core_tables.hpp"
#include "ctx.cuh"
#include "public_values.hpp"
#include "sumcheck.cuh"
#include <cstddef>
#include <vector>

static_assert(sizeof(sp1b200_byte_lookup) == 12, "sp1b200_byte_lookup is 12 bytes");
static_assert(offsetof(sp1b200_byte_lookup, a) == 0 && offsetof(sp1b200_byte_lookup, b) == 2 && offsetof(sp1b200_byte_lookup, c) == 3 &&
                  offsetof(sp1b200_byte_lookup, opcode) == 4 && offsetof(sp1b200_byte_lookup, count) == 8,
              "sp1b200_byte_lookup field offsets");
static_assert(sizeof(sp1b200_pc_count) == 16 && offsetof(sp1b200_pc_count, pc) == 0 && offsetof(sp1b200_pc_count, count) == 8,
              "sp1b200_pc_count layout");

namespace {

using core_tables::BYTE_ROWS;
using core_tables::RANGE_ROWS;
constexpr uint32_t BYTE_COLS = SP1B200_BYTE_MULT_COLS;    // ByteMultCols: one multiplicity per ByteOpcode::byte_table() opcode
constexpr uint32_t RANGE_OPCODE = SP1B200_BYTE_OPCODE_RANGE;
constexpr uint32_t MAX_RANGE_BITS = 16;                   // RangeChip: a < 2^bits, bits <= 16
// counter layout: Byte column k row r at k 2^16 + r, then Range row r, then Program row i
constexpr uint64_t RANGE_BASE = BYTE_COLS * BYTE_ROWS;
constexpr uint64_t PROGRAM_BASE = RANGE_BASE + RANGE_ROWS;
constexpr uint32_t NO_KEY = ~0u;
constexpr uint64_t NONE = ~0ull;
constexpr uint64_t MAX_RECORDS = (uint64_t)1 << 32;   // n (2^32 - 1) + the public-value lookups < 2^64: no counter wraps
constexpr unsigned THREADS = 256, WARPS = THREADS / 32;

__device__ __forceinline__ uint32_t mont(uint32_t x) { return kb::monty_reduce((uint64_t)x * kb::RR); }

// Adds `count` at counters[key] for every lane whose key is not NO_KEY; called by all 32 lanes.  Lanes with equal keys are summed
// in 64 bits by the lowest of them, which alone issues the atomic.
__device__ __forceinline__ void warp_add(unsigned long long* __restrict__ counters, uint32_t key, uint32_t count, uint32_t* s_warp) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    s_warp[lane] = count;
    __syncwarp();
    if (key != NO_KEY && lane == (unsigned)(__ffs(peers) - 1)) {
        unsigned long long sum = 0;
        for (unsigned m = peers; m; m &= m - 1) sum += s_warp[__ffs(m) - 1];
        if (sum) atomicAdd(counters + key, sum);
    }
    __syncwarp();
}

// ByteChip::generate_trace_into (bytes/trace.rs:68-92): opcode 0..5 -> Byte row 256 b + c, column opcode (a is not read);
// RangeChip::generate_trace_into (range/trace.rs:98-121): opcode 6 -> Range row a + 2^b.  A record with opcode > 6, or a Range record with
// b > 16, leaves its index in *bad (the lowest index wins) and adds nothing.
__global__ void __launch_bounds__(THREADS) count_lookups_kernel(const sp1b200_byte_lookup* __restrict__ recs, uint64_t n,
                                                                 unsigned long long* __restrict__ counters, unsigned long long* bad) {
    __shared__ uint32_t s_count[WARPS][32];
    const uint64_t stride = (uint64_t)gridDim.x * THREADS;
    for (uint64_t base = (uint64_t)blockIdx.x * THREADS + (threadIdx.x & ~31u); base < n; base += stride) {   // warp-uniform loop
        const uint64_t i = base + (threadIdx.x & 31);
        uint32_t key = NO_KEY, count = 0;
        if (i < n) {
            const sp1b200_byte_lookup r = recs[i];
            if (r.opcode < RANGE_OPCODE) {
                key = (uint32_t)r.opcode * (uint32_t)BYTE_ROWS + ((uint32_t)r.b << 8 | r.c);
            } else if (r.opcode == RANGE_OPCODE && r.b <= MAX_RANGE_BITS) {
                key = (uint32_t)RANGE_BASE + r.a + (1u << r.b);
            } else {
                atomicMin(bad, (unsigned long long)i);
            }
            count = r.count;
        }
        warp_add(counters, key, count, s_count[threadIdx.x >> 5]);
    }
}

// ProgramChip::generate_trace_into (trusted.rs:134-292): a pc = pc_base + 4 i with i < n_instrs adds to Program row i; any other pc is
// dropped, as instruction_counts.get(&pc) never reads it
__global__ void __launch_bounds__(THREADS) count_pcs_kernel(const sp1b200_pc_count* __restrict__ recs, uint64_t n, uint64_t pc_base,
                                                             uint64_t n_instrs, unsigned long long* __restrict__ counters) {
    __shared__ uint32_t s_count[WARPS][32];
    const uint64_t stride = (uint64_t)gridDim.x * THREADS;
    for (uint64_t base = (uint64_t)blockIdx.x * THREADS + (threadIdx.x & ~31u); base < n; base += stride) {
        const uint64_t i = base + (threadIdx.x & 31);
        uint32_t key = NO_KEY, count = 0;
        if (i < n) {
            const uint64_t pc = recs[i].pc;
            count = recs[i].count;
            const uint64_t off = pc - pc_base;
            if (pc >= pc_base && (off & 3) == 0 && (off >> 2) < n_instrs) key = (uint32_t)(PROGRAM_BASE + (off >> 2));
        }
        warp_add(counters, key, count, s_count[threadIdx.x >> 5]);
    }
}

// every counter < p (from_canonical_usize) -> its Montgomery word in the table it belongs to; the lowest counter index >= p goes to *bad
__global__ void __launch_bounds__(256) write_tables_kernel(const unsigned long long* __restrict__ counters, uint64_t total,
                                                            uint32_t* __restrict__ d_byte, uint32_t* __restrict__ d_range,
                                                            uint32_t* __restrict__ d_prog, unsigned long long* bad) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const unsigned long long v = counters[t];
    if (v >= kb::P) atomicMin(bad, (unsigned long long)t);
    const uint32_t w = v < kb::P ? mont((uint32_t)v) : 0u;
    if (t < RANGE_BASE) d_byte[t] = w;
    else if (t < PROGRAM_BASE) d_range[t - RANGE_BASE] = w;
    else d_prog[t - PROGRAM_BASE] = w;
}

// ByteChip / RangeChip::generate_dependencies (bytes/trace.rs:50-66, range/trace.rs:54-96 without the mprotect fields) from the field
// form of the shard's public values (Montgomery words): U8Range checks of the timestamps' middle bytes and of both value digests' bytes,
// 16- and 13-bit Range checks of the timestamps' limbs and 16-bit checks of the six addresses' limbs.  Each value is rebuilt as the
// reference reads it (timestamp_from_limbs, 16-bit address limbs, little-endian digest bytes), so a limb or byte out of its range is an
// error.
sp1b200_err public_value_lookups(const char* what, const uint32_t* pv_words, uint32_t n, std::vector<sp1b200_byte_lookup>& out) {
    if (n != pv::PROOF_MAX_NUM_PVS)
        return sp1b200_set_error("%s: %u public values, a core shard has %u", what, n, pv::PROOF_MAX_NUM_PVS);
    uint32_t v[pv::PROOF_MAX_NUM_PVS];
    for (uint32_t i = 0; i < n; i++) {
        if (pv_words[i] >= kb::P) return sp1b200_set_error("%s: public value %u is not a field element (word 0x%08x >= p)", what, i, pv_words[i]);
        v[i] = kb::monty_reduce(pv_words[i]);
    }
    auto limb = [&](uint32_t at, uint32_t bits, const char* name) -> sp1b200_err {
        if (v[at] >> bits) return sp1b200_set_error("%s: public value %u (%s) = %u does not fit %u bits", what, at, name, v[at], bits);
        return nullptr;
    };
    auto u8_pair = [&](uint32_t b, uint32_t c) { out.push_back(sp1b200_byte_lookup{0, (uint8_t)b, (uint8_t)c, 3, {0, 0, 0}, 1}); };
    auto range = [&](uint32_t a, uint32_t bits) {
        out.push_back(sp1b200_byte_lookup{(uint16_t)a, (uint8_t)bits, 0, (uint8_t)RANGE_OPCODE, {0, 0, 0}, 1});
    };
    uint64_t ts[2];
    for (int k = 0; k < 2; k++) {   // timestamp_from_limbs: limbs[0] << 32 | limbs[1] << 24 | limbs[2] << 16 | limbs[3]
        const uint32_t at = k ? pv::LAST_TIMESTAMP : pv::INITIAL_TIMESTAMP;
        const char* name = k ? "last_timestamp" : "initial_timestamp";
        const uint32_t bits[4] = {16, 8, 8, 16};
        for (uint32_t j = 0; j < 4; j++) SP1_TRY(limb(at + j, bits[j], name));
        ts[k] = ((uint64_t)v[at] << 32) | ((uint64_t)v[at + 1] << 24) | ((uint64_t)v[at + 2] << 16) | v[at + 3];
    }
    for (uint32_t at : {pv::PREV_COMMITTED_VALUE_DIGEST, pv::COMMITTED_VALUE_DIGEST})
        for (uint32_t j = 0; j < 32; j++) SP1_TRY(limb(at + j, 8, at ? "committed_value_digest" : "prev_committed_value_digest"));
    const uint32_t addrs[6] = {pv::PC_START, pv::NEXT_PC, pv::PREVIOUS_INIT_ADDR, pv::LAST_INIT_ADDR, pv::PREVIOUS_FINALIZE_ADDR,
                               pv::LAST_FINALIZE_ADDR};
    for (uint32_t at : addrs)
        for (uint32_t j = 0; j < 3; j++) SP1_TRY(limb(at + j, 16, "address"));
    // ByteChip
    for (int k = 0; k < 2; k++) u8_pair((ts[k] >> 24) & 0xFF, (ts[k] >> 16) & 0xFF);
    for (uint32_t i = 0; i < 8; i++)   // u32::to_le_bytes of word i of each digest, checked two bytes at a time
        for (uint32_t at : {pv::PREV_COMMITTED_VALUE_DIGEST, pv::COMMITTED_VALUE_DIGEST}) {
            u8_pair(v[at + 4 * i], v[at + 4 * i + 1]);
            u8_pair(v[at + 4 * i + 2], v[at + 4 * i + 3]);
        }
    // RangeChip; (limb - 1) / 8 is a u16 subtraction, which wraps to 0xFFFF / 8 at 0 as the release build does
    for (int k = 0; k < 2; k++) {
        range((ts[k] >> 32) & 0xFFFF, 16);
        range((uint16_t)((uint16_t)(ts[k] & 0xFFFF) - 1) / 8, 13);
    }
    for (uint32_t at : addrs) {
        const uint64_t addr = (uint64_t)v[at] | ((uint64_t)v[at + 1] << 16) | ((uint64_t)v[at + 2] << 32);
        for (uint32_t j = 0; j < 3; j++) range((addr >> (16 * j)) & 0xFFFF, 16);
    }
    return nullptr;
}

const char* const TABLE_NAMES[3] = {"Byte", "Range", "Program"};

}  // namespace

extern "C" sp1b200_err sp1b200_lookup_traces(sp1b200_ctx* ctx, uint64_t pc_base, uint64_t n_instrs, const sp1b200_byte_lookup* lookups_any,
                                             uint64_t n_lookups, const sp1b200_pc_count* pcs_any, uint64_t n_pcs,
                                             const uint32_t* h_public_values, uint32_t n_public_values, uint32_t* byte_out_any,
                                             uint32_t* program_out_any, uint32_t* range_out_any, uint64_t* h_rows3) {
    SP1_DEVICE_GUARD(ctx);
    const char* what = "lookup_traces";
    if (!ctx) return sp1b200_set_error("%s: NULL context", what);
    if (n_instrs == 0) return sp1b200_set_error("%s: n_instrs = 0 (a program has at least one instruction)", what);
    SP1_TRY(core_tables::check_program_window(ctx, what, pc_base, n_instrs));
    if (n_lookups && !lookups_any) return sp1b200_set_error("%s: NULL lookup array with %llu records", what, (unsigned long long)n_lookups);
    if (n_pcs && !pcs_any) return sp1b200_set_error("%s: NULL pc array with %llu records", what, (unsigned long long)n_pcs);
    if (n_lookups > MAX_RECORDS || n_pcs > MAX_RECORDS)
        return sp1b200_set_error("%s: %llu lookup and %llu pc records; at most 2^32 of each", what, (unsigned long long)n_lookups,
                                 (unsigned long long)n_pcs);
    std::vector<sp1b200_byte_lookup> pv_recs;
    if (h_public_values) SP1_TRY(public_value_lookups(what, h_public_values, n_public_values, pv_recs));
    const uint64_t h = core_tables::program_height(n_instrs);
    if (h_rows3) { h_rows3[0] = BYTE_ROWS; h_rows3[1] = h; h_rows3[2] = RANGE_ROWS; }
    const bool any_out = byte_out_any || program_out_any || range_out_any;
    if (!any_out) return nullptr;   // a size query
    if (!byte_out_any || !program_out_any || !range_out_any)
        return sp1b200_set_error("%s: the three outputs are all NULL (a size query) or all set", what);

    cudaStream_t st = ctx->stream;
    const uint64_t total = PROGRAM_BASE + h;
    PhaseTimer t_all(ctx, "lookup_traces");
    DevFree mem(ctx);
    unsigned long long *d_counters, *d_bad;
    SP1_TRY(mem.alloc((void**)&d_counters, total * 8));
    SP1_TRY(mem.alloc((void**)&d_bad, 2 * 8));
    SP1_CUDA(cudaMemsetAsync(d_counters, 0, total * 8, st));
    SP1_CUDA(cudaMemsetAsync(d_bad, 0xff, 2 * 8, st));
    DevBuf lookups, pcs, pv_dev;
    SP1_TRY(lookups.in(ctx, lookups_any, n_lookups * sizeof(sp1b200_byte_lookup)));
    SP1_TRY(pcs.in(ctx, pcs_any, n_pcs * sizeof(sp1b200_pc_count)));
    SP1_TRY(pv_dev.in(ctx, pv_recs.data(), pv_recs.size() * sizeof(sp1b200_byte_lookup)));
    const unsigned grid_cap = (unsigned)ctx->num_sms * 16;
    auto grid = [&](uint64_t n) { return std::max(1u, std::min(grid_cap, blocks_for(n, THREADS))); };
    {
        PhaseTimer t(ctx, "lookup_traces.tables");
        if (n_lookups)
            SP1_LAUNCH(ctx, count_lookups_kernel, grid(n_lookups), THREADS, 0, (const sp1b200_byte_lookup*)lookups.d, n_lookups, d_counters,
                       d_bad);
        if (!pv_recs.empty())   // valid by construction: nothing reaches *d_bad from them
            SP1_LAUNCH(ctx, count_lookups_kernel, 1, THREADS, 0, (const sp1b200_byte_lookup*)pv_dev.d, (uint64_t)pv_recs.size(), d_counters,
                       d_bad);
        if (n_pcs)
            SP1_LAUNCH(ctx, count_pcs_kernel, grid(n_pcs), THREADS, 0, (const sp1b200_pc_count*)pcs.d, n_pcs, pc_base, n_instrs, d_counters);
        t.stop();
    }
    unsigned long long bad;
    SP1_CUDA(cudaMemcpyAsync(&bad, d_bad, 8, cudaMemcpyDeviceToHost, st));
    SP1_CUDA(cudaStreamSynchronize(st));
    if (bad != NONE) {
        sp1b200_byte_lookup r;
        SP1_CUDA(cudaMemcpy(&r, (const sp1b200_byte_lookup*)lookups.d + bad, sizeof(r), cudaMemcpyDeviceToHost));
        if (r.opcode > RANGE_OPCODE)
            return sp1b200_set_error("%s: lookup %llu has opcode %u (the largest ByteOpcode is Range = %u)", what, bad, r.opcode, RANGE_OPCODE);
        return sp1b200_set_error("%s: lookup %llu is a Range check of a = %u with b = %u bits > %u", what, bad, r.a, r.b, MAX_RANGE_BITS);
    }
    DevBuf byte_out, prog_out, range_out;
    SP1_TRY(byte_out.out(ctx, byte_out_any, RANGE_BASE * 4));
    SP1_TRY(prog_out.out(ctx, program_out_any, h * 4));
    SP1_TRY(range_out.out(ctx, range_out_any, RANGE_ROWS * 4));
    {
        PhaseTimer t(ctx, "lookup_traces.write");
        SP1_LAUNCH(ctx, write_tables_kernel, blocks_for(total), 256, 0, d_counters, total, (uint32_t*)byte_out.d, (uint32_t*)range_out.d,
                   (uint32_t*)prog_out.d, d_bad + 1);
        t.stop();
    }
    SP1_CUDA(cudaMemcpyAsync(&bad, d_bad + 1, 8, cudaMemcpyDeviceToHost, st));
    SP1_CUDA(cudaStreamSynchronize(st));
    if (bad != NONE) {
        unsigned long long v;
        SP1_CUDA(cudaMemcpy(&v, d_counters + bad, 8, cudaMemcpyDeviceToHost));
        const int table = bad < RANGE_BASE ? 0 : bad < PROGRAM_BASE ? 1 : 2;
        const uint64_t row = table == 0 ? bad % BYTE_ROWS : table == 1 ? bad - RANGE_BASE : bad - PROGRAM_BASE;
        const uint64_t col = table == 0 ? bad / BYTE_ROWS : 0;
        return sp1b200_set_error("%s: %s row %llu column %llu accumulates multiplicity %llu >= p", what, TABLE_NAMES[table],
                                 (unsigned long long)row, (unsigned long long)col, v);
    }
    SP1_TRY(byte_out.finish());
    SP1_TRY(prog_out.finish());
    SP1_TRY(range_out.finish());
    t_all.stop();
    return nullptr;
}
