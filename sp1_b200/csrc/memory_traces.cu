// A shard's memory chips, generated on the device from its memory events: the main traces of MemoryGlobalInit / MemoryGlobalFinalize
// (MemoryGlobalChip::generate_trace_into, crates/core/machine/src/memory/global.rs:155-236) and MemoryLocal (local.rs:166-238), with
// the byte lookups and global interaction events of their generate_dependencies (global.rs:63-142, local.rs:105-157).
//
// Init / finalize: one pass builds the 48-bit address keys with the event indices and checks every address and timestamp; a radix
// sort orders the events by address; one thread per sorted row gathers its event, compares its address with the row before (the
// chip's prev_addr < addr), computes the row's three inverses with one field inversion, and writes each column as its own coalesced
// stream.  The row's lookup and global records go through shared memory so the block stores them as one contiguous run.  Local: one
// streaming pass in input order, the same way.
#include "ctx.cuh"
#include "radix_sort.cuh"
#include "sumcheck.cuh"
#include <cstddef>

static_assert(sizeof(sp1b200_memory_event) == 24 && offsetof(sp1b200_memory_event, addr) == 0 &&
                  offsetof(sp1b200_memory_event, value) == 8 && offsetof(sp1b200_memory_event, timestamp) == 16,
              "sp1b200_memory_event layout");
static_assert(sizeof(sp1b200_memory_local_event) == 40 && offsetof(sp1b200_memory_local_event, addr) == 0 &&
                  offsetof(sp1b200_memory_local_event, initial_timestamp) == 8 &&
                  offsetof(sp1b200_memory_local_event, initial_value) == 16 &&
                  offsetof(sp1b200_memory_local_event, final_timestamp) == 24 && offsetof(sp1b200_memory_local_event, final_value) == 32,
              "sp1b200_memory_local_event layout");
static_assert(sizeof(sp1b200_global_event) == 36 && offsetof(sp1b200_global_event, message) == 0 &&
                  offsetof(sp1b200_global_event, is_receive) == 32 && offsetof(sp1b200_global_event, kind) == 33,
              "sp1b200_global_event layout");
static_assert(sizeof(sp1b200_byte_lookup) == 12, "sp1b200_byte_lookup is 12 bytes");

namespace {

constexpr uint32_t GCOLS = SP1B200_MEMORY_GLOBAL_COLS, LCOLS = SP1B200_MEMORY_LOCAL_COLS;
constexpr uint32_t GLK = SP1B200_MEMORY_GLOBAL_LOOKUPS, LLK = SP1B200_MEMORY_LOCAL_LOOKUPS;
constexpr uint32_t LK_WORDS = sizeof(sp1b200_byte_lookup) / 4, GE_WORDS = sizeof(sp1b200_global_event) / 4;
constexpr uint64_t ADDR_LIMIT = 1ull << 48;   // three 16-bit limbs (u64_to_u16_limbs(addr)[0..3])
// the executor's clock is 48 bits wide: clk_high = timestamp >> 24 and clk_low = timestamp & 0xFFFFFF are 24-bit limbs
constexpr uint64_t TS_LIMIT = 1ull << 48;
constexpr uint64_t MAX_EVENTS = 1ull << 31;
constexpr uint32_t OP_U8RANGE = 3, OP_RANGE = SP1B200_BYTE_OPCODE_RANGE;
constexpr uint32_t KIND_MEMORY = 1;           // InteractionKind::Memory
constexpr unsigned ROWS = 128;                // rows (threads) per block of the row kernels
constexpr uint64_t NONE = ~0ull;

// flags, each the lowest offending index: per init (0) / finalize (1) / local (2) section
enum { F_ADDR = 0, F_TS = 1, F_ORDER = 2, F_PER = 3 };

__device__ __forceinline__ uint32_t mont(uint32_t x) { return kb::monty_reduce((uint64_t)x * kb::RR); }
__device__ __forceinline__ uint32_t limb(uint64_t x, int k) { return (uint32_t)(x >> (16 * k)) & 0xFFFFu; }

__device__ __forceinline__ void put_lookup(uint32_t* s, uint32_t op, uint32_t a, uint32_t b, uint32_t c, uint32_t count) {
    s[0] = a | (b << 16) | (c << 24);
    s[1] = op;
    s[2] = count;
}

// the message of a memory access (global.rs:117-141, local.rs:115-151): value limbs 0 and 1 carry bytes 4 and 5 at 2^16
__device__ __forceinline__ void put_global(uint32_t* s, uint32_t clk_high, uint32_t clk_low, uint64_t addr, uint64_t value,
                                           uint32_t is_receive) {
    s[0] = clk_high;
    s[1] = clk_low;
    for (int k = 0; k < 3; k++) s[2 + k] = limb(addr, k);
    s[5] = limb(value, 0) + (((uint32_t)(value >> 32) & 0xFF) << 16);
    s[6] = limb(value, 1) + (((uint32_t)(value >> 40) & 0xFF) << 16);
    s[7] = limb(value, 3);
    s[8] = is_receive | (KIND_MEMORY << 8);
}

// the block's staged records (rows [row0, row0 + n_rows) of the block, `per_row` words each) -> out, as one contiguous run
__device__ __forceinline__ void flush(const uint32_t* s, uint32_t* __restrict__ out, uint64_t row0, uint32_t n_rows, uint32_t per_row) {
    const uint32_t words = n_rows * per_row;
    uint32_t* dst = out + row0 * per_row;
    for (uint32_t w = threadIdx.x; w < words; w += blockDim.x) dst[w] = s[w];
}

// keys[i] = addr of event i, idx[i] = i; an address or timestamp >= 2^48 leaves i in flags[F_ADDR] / flags[F_TS]
__global__ void __launch_bounds__(256) memory_keys_kernel(const sp1b200_memory_event* __restrict__ ev, uint64_t n, uint64_t* __restrict__ keys,
                                                          uint32_t* __restrict__ idx, unsigned long long* flags) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t addr = ev[i].addr;
    keys[i] = addr;
    idx[i] = (uint32_t)i;
    if (addr >= ADDR_LIMIT) atomicMin(flags + F_ADDR, (unsigned long long)i);
    if (ev[i].timestamp >= TS_LIMIT) atomicMin(flags + F_TS, (unsigned long long)i);
}

// MemoryGlobalChip rows: thread r < h writes row r of the column-major [GCOLS x h] trace; a real row r < n also writes its GLK lookups
// (generate_dependencies' order) and its global event.  A compared row whose address is not above prev_addr leaves r in *bad_order.
__global__ void __launch_bounds__(ROWS) memory_global_rows_kernel(const sp1b200_memory_event* __restrict__ ev, const uint64_t* __restrict__ keys,
                                                                  const uint32_t* __restrict__ idx, uint64_t n, uint64_t h,
                                                                  uint64_t previous_addr, uint32_t is_finalize, uint32_t* __restrict__ out,
                                                                  uint32_t* __restrict__ lookups, uint32_t* __restrict__ globals,
                                                                  unsigned long long* bad_order) {
    __shared__ uint32_t s_lk[ROWS * GLK * LK_WORDS];
    __shared__ uint32_t s_ge[ROWS * GE_WORDS];
    const uint64_t row0 = (uint64_t)blockIdx.x * ROWS;
    const uint64_t r = row0 + threadIdx.x;
    uint32_t c[GCOLS];
    for (uint32_t k = 0; k < GCOLS; k++) c[k] = 0;
    if (r < n) {
        const sp1b200_memory_event e = ev[idx[r]];
        const uint64_t addr = keys[r];
        const uint64_t prev = r ? keys[r - 1] : previous_addr;
        const bool comp = prev != 0 || r != 0;
        if (comp && !(prev < addr)) atomicMin(bad_order, (unsigned long long)r);
        c[0] = mont((uint32_t)(e.timestamp >> 24));
        c[1] = mont((uint32_t)(e.timestamp & 0xFFFFFF));
        c[2] = mont((uint32_t)r);
        for (int k = 0; k < 3; k++) {
            c[3 + k] = mont(limb(prev, k));
            c[6 + k] = mont(limb(addr, k));
        }
        for (int k = 0; k < 4; k++) c[17 + k] = mont(limb(e.value, k));
        const uint32_t lower = (uint32_t)(e.value >> 32) & 0xFF, upper = (uint32_t)(e.value >> 40) & 0xFF;
        c[21] = mont(lower);
        c[22] = mont(upper);
        c[23] = kb::ONE;                                        // is_real
        c[24] = comp ? kb::ONE : 0u;                            // is_comp
        c[25] = (prev == 0 && r != 0) ? 0u : kb::ONE;           // prev_valid
        // LtOperationUnsigned::populate_unsigned(1, prev, addr): the first differing limb from the top
        int k_diff = -1;
        if (comp)
            for (int k = 3; k >= 0; k--)
                if (limb(prev, k) != limb(addr, k)) { k_diff = k; break; }
        const uint32_t pk = k_diff >= 0 ? limb(prev, k_diff) : 0u, ak = k_diff >= 0 ? limb(addr, k_diff) : 0u;
        // the three inverses with one inversion: IsZero of prev's limb sum, IsZero of the index, and (prev_k - addr_k)^-1
        uint32_t x[3] = {mont(limb(prev, 0) + limb(prev, 1) + limb(prev, 2)), c[2], k_diff >= 0 ? kb::sub(mont(pk), mont(ak)) : 0u};
        uint32_t y[3];
        for (int k = 0; k < 3; k++) y[k] = x[k] ? x[k] : kb::ONE;
        const uint32_t p01 = kb::mul(y[0], y[1]);
        const uint32_t inv012 = kb::inv(kb::mul(p01, y[2]));
        const uint32_t inv01 = kb::mul(inv012, y[2]);
        uint32_t xi[3] = {kb::mul(inv01, y[1]), kb::mul(inv01, y[0]), kb::mul(inv012, p01)};
        for (int k = 0; k < 3; k++) xi[k] = x[k] ? xi[k] : 0u;
        c[9] = comp ? kb::ONE : 0u;                             // u16_compare_operation.bit = a = 1
#pragma unroll
        for (int k = 0; k < 4; k++) c[10 + k] = k == k_diff ? kb::ONE : 0u;   // u16_flags
        c[14] = xi[2];                                          // not_eq_inv
        c[15] = mont(pk);                                       // comparison_limbs
        c[16] = mont(ak);
        c[26] = xi[0];
        c[27] = x[0] ? 0u : kb::ONE;
        c[28] = xi[1];
        c[29] = x[1] ? 0u : kb::ONE;
        // generate_dependencies (global.rs:102-110)
        uint32_t* s = s_lk + threadIdx.x * GLK * LK_WORDS;
        for (int k = 0; k < 4; k++) put_lookup(s + LK_WORDS * k, OP_RANGE, limb(e.value, k), 16, 0, 1);
        for (int k = 0; k < 3; k++) put_lookup(s + LK_WORDS * (4 + k), OP_RANGE, limb(prev, k), 16, 0, 1);
        for (int k = 0; k < 3; k++) put_lookup(s + LK_WORDS * (7 + k), OP_RANGE, limb(addr, k), 16, 0, 1);
        put_lookup(s + LK_WORDS * 10, OP_U8RANGE, 0, lower, upper, 1);
        put_lookup(s + LK_WORDS * 11, OP_RANGE, (pk - ak) & 0xFFFFu, 16, 0, comp ? 1u : 0u);   // U16CompareOperation::populate
        if (is_finalize)
            put_global(s_ge + threadIdx.x * GE_WORDS, (uint32_t)(e.timestamp >> 24), (uint32_t)(e.timestamp & 0xFFFFFF), addr, e.value, 1);
        else
            put_global(s_ge + threadIdx.x * GE_WORDS, 0, 0, addr, e.value, 0);
    }
    if (r < h)
        for (uint32_t k = 0; k < GCOLS; k++) out[k * h + r] = c[k];
    __syncthreads();
    if (row0 < n) {
        const uint32_t real = (uint32_t)min((uint64_t)ROWS, n - row0);
        flush(s_lk, lookups, row0, real, GLK * LK_WORDS);
        flush(s_ge, globals, row0, real, GE_WORDS);
    }
}

// MemoryLocalChip rows in input order: thread r < h writes row r of the [LCOLS x h] trace; r < n also writes its LLK lookups and its
// two global events.  An address or either timestamp >= 2^48 leaves r in flags[F_ADDR] / flags[F_TS].
__global__ void __launch_bounds__(ROWS) memory_local_rows_kernel(const sp1b200_memory_local_event* __restrict__ ev, uint64_t n, uint64_t h,
                                                                 uint32_t* __restrict__ out, uint32_t* __restrict__ lookups,
                                                                 uint32_t* __restrict__ globals, unsigned long long* flags) {
    __shared__ uint32_t s_lk[ROWS * LLK * LK_WORDS];
    __shared__ uint32_t s_ge[ROWS * 2 * GE_WORDS];
    const uint64_t row0 = (uint64_t)blockIdx.x * ROWS;
    const uint64_t r = row0 + threadIdx.x;
    uint32_t c[LCOLS];
    for (uint32_t k = 0; k < LCOLS; k++) c[k] = 0;
    if (r < n) {
        const sp1b200_memory_local_event e = ev[r];
        if (e.addr >= ADDR_LIMIT) atomicMin(flags + F_ADDR, (unsigned long long)r);
        if (e.initial_timestamp >= TS_LIMIT || e.final_timestamp >= TS_LIMIT) atomicMin(flags + F_TS, (unsigned long long)r);
        for (int k = 0; k < 3; k++) c[k] = mont(limb(e.addr, k));
        c[3] = mont((uint32_t)(e.initial_timestamp >> 24));
        c[4] = mont((uint32_t)(e.final_timestamp >> 24));
        c[5] = mont((uint32_t)(e.initial_timestamp & 0xFFFFFF));
        c[6] = mont((uint32_t)(e.final_timestamp & 0xFFFFFF));
        for (int k = 0; k < 4; k++) {
            c[7 + k] = mont(limb(e.initial_value, k));
            c[11 + k] = mont(limb(e.final_value, k));
        }
        c[15] = mont((uint32_t)(e.initial_value >> 32) & 0xFF);
        c[16] = mont((uint32_t)(e.initial_value >> 40) & 0xFF);
        c[17] = mont((uint32_t)(e.final_value >> 32) & 0xFF);
        c[18] = mont((uint32_t)(e.final_value >> 40) & 0xFF);
        c[19] = kb::ONE;
        // generate_dependencies (local.rs:108-153): per access U8Range of bytes 4, 5, then Range(16) of the four limbs
        uint32_t* s = s_lk + threadIdx.x * LLK * LK_WORDS;
        for (int a = 0; a < 2; a++) {
            const uint64_t v = a ? e.final_value : e.initial_value;
            put_lookup(s + LK_WORDS * 5 * a, OP_U8RANGE, 0, (uint32_t)(v >> 32) & 0xFF, (uint32_t)(v >> 40) & 0xFF, 1);
            for (int k = 0; k < 4; k++) put_lookup(s + LK_WORDS * (5 * a + 1 + k), OP_RANGE, limb(v, k), 16, 0, 1);
        }
        uint32_t* g = s_ge + threadIdx.x * 2 * GE_WORDS;
        put_global(g, (uint32_t)(e.initial_timestamp >> 24), (uint32_t)(e.initial_timestamp & 0xFFFFFF), e.addr, e.initial_value, 1);
        put_global(g + GE_WORDS, (uint32_t)(e.final_timestamp >> 24), (uint32_t)(e.final_timestamp & 0xFFFFFF), e.addr, e.final_value, 0);
    }
    if (r < h)
        for (uint32_t k = 0; k < LCOLS; k++) out[k * h + r] = c[k];
    __syncthreads();
    if (row0 < n) {
        const uint32_t real = (uint32_t)min((uint64_t)ROWS, n - row0);
        flush(s_lk, lookups, row0, real, LLK * LK_WORDS);
        flush(s_ge, globals, row0, real, 2 * GE_WORDS);
    }
}

// next_multiple_of_32(n, None) (hypercube/src/util.rs:50-59) of an included chip; a chip without events is not included: height 0
uint64_t chip_height(uint64_t n) { return n ? (n + 31) / 32 * 32 : 0; }

const char* const SECTION[3] = {"init", "finalize", "local"};

}  // namespace

extern "C" sp1b200_err sp1b200_memory_traces(sp1b200_ctx* ctx, const sp1b200_memory_event* init_any, uint64_t n_init,
                                             const sp1b200_memory_event* finalize_any, uint64_t n_finalize, uint64_t previous_init_addr,
                                             uint64_t previous_finalize_addr, const sp1b200_memory_local_event* local_any, uint64_t n_local,
                                             uint32_t* init_out_any, uint32_t* finalize_out_any, uint32_t* local_out_any,
                                             sp1b200_byte_lookup* lookups_out_any, sp1b200_global_event* globals_out_any, uint64_t* h_rows3,
                                             uint64_t* h_n_lookups, uint64_t* h_n_globals) {
    SP1_DEVICE_GUARD(ctx);
    const char* what = "memory_traces";
    if (!ctx) return sp1b200_set_error("%s: NULL context", what);
    const void* in_any[3] = {init_any, finalize_any, local_any};
    const uint64_t n[3] = {n_init, n_finalize, n_local};
    const uint64_t previous[2] = {previous_init_addr, previous_finalize_addr};
    for (int s = 0; s < 3; s++) {
        if (n[s] && !in_any[s]) return sp1b200_set_error("%s: NULL %s event array with %llu events", what, SECTION[s], (unsigned long long)n[s]);
        if (n[s] >= MAX_EVENTS)
            return sp1b200_set_error("%s: %llu %s events; at most 2^31 - 1", what, (unsigned long long)n[s], SECTION[s]);
    }
    for (int s = 0; s < 2; s++)
        if (previous[s] >= ADDR_LIMIT)
            return sp1b200_set_error("%s: previous_%s_addr 0x%llx >= 2^48", what, SECTION[s], (unsigned long long)previous[s]);
    const uint64_t h[3] = {chip_height(n[0]), chip_height(n[1]), chip_height(n[2])};
    const uint64_t cols[3] = {GCOLS, GCOLS, LCOLS};
    const uint64_t lk_off[4] = {0, GLK * n[0], GLK * (n[0] + n[1]), GLK * (n[0] + n[1]) + LLK * n[2]};
    const uint64_t ge_off[4] = {0, n[0], n[0] + n[1], n[0] + n[1] + 2 * n[2]};
    if (h_rows3) for (int s = 0; s < 3; s++) h_rows3[s] = h[s];
    if (h_n_lookups) *h_n_lookups = lk_off[3];
    if (h_n_globals) *h_n_globals = ge_off[3];
    uint32_t* trace_any[3] = {init_out_any, finalize_out_any, local_out_any};
    if (!init_out_any && !finalize_out_any && !local_out_any && !lookups_out_any && !globals_out_any) return nullptr;   // a size query
    for (int s = 0; s < 3; s++)
        if (h[s] && !trace_any[s]) return sp1b200_set_error("%s: NULL %s trace output for %llu rows (all outputs NULL is a size query)", what,
                                                            SECTION[s], (unsigned long long)h[s]);
    if (lk_off[3] && !lookups_out_any) return sp1b200_set_error("%s: NULL lookup output for %llu records", what, (unsigned long long)lk_off[3]);
    if (ge_off[3] && !globals_out_any) return sp1b200_set_error("%s: NULL global event output for %llu records", what, (unsigned long long)ge_off[3]);

    cudaStream_t st = ctx->stream;
    PhaseTimer t_all(ctx, "memory_traces");
    DevFree mem(ctx);
    unsigned long long* d_flags;
    SP1_TRY(mem.alloc((void**)&d_flags, 3 * F_PER * 8));
    SP1_CUDA(cudaMemsetAsync(d_flags, 0xff, 3 * F_PER * 8, st));
    DevBuf in[3], trace[3], lookups, globals;
    SP1_TRY(in[0].in(ctx, init_any, n[0] * sizeof(sp1b200_memory_event)));
    SP1_TRY(in[1].in(ctx, finalize_any, n[1] * sizeof(sp1b200_memory_event)));
    SP1_TRY(in[2].in(ctx, local_any, n[2] * sizeof(sp1b200_memory_local_event)));
    for (int s = 0; s < 3; s++) SP1_TRY(trace[s].out(ctx, trace_any[s], cols[s] * h[s] * 4));
    SP1_TRY(lookups.out(ctx, lookups_out_any, lk_off[3] * sizeof(sp1b200_byte_lookup)));
    SP1_TRY(globals.out(ctx, globals_out_any, ge_off[3] * sizeof(sp1b200_global_event)));
    uint64_t* keys[2] = {nullptr, nullptr};
    uint32_t* idx[2] = {nullptr, nullptr};
    {
        PhaseTimer t(ctx, "memory_traces.sort");
        for (int s = 0; s < 2; s++) {
            if (!n[s]) continue;
            uint64_t* k_in;
            uint32_t* i_in;
            SP1_TRY(mem.alloc((void**)&k_in, n[s] * 8));
            SP1_TRY(mem.alloc((void**)&keys[s], n[s] * 8));
            SP1_TRY(mem.alloc((void**)&i_in, n[s] * 4));
            SP1_TRY(mem.alloc((void**)&idx[s], n[s] * 4));
            SP1_LAUNCH(ctx, memory_keys_kernel, blocks_for(n[s]), 256, 0, (const sp1b200_memory_event*)in[s].d, n[s], k_in, i_in,
                       d_flags + F_PER * s);
            SP1_TRY(radix_sort::pairs(ctx, mem, k_in, keys[s], i_in, idx[s], n[s], 48));
        }
        t.stop();
    }
    {
        PhaseTimer t(ctx, "memory_traces.rows");
        for (int s = 0; s < 2; s++)
            if (h[s])
                SP1_LAUNCH(ctx, memory_global_rows_kernel, blocks_for(h[s], ROWS), ROWS, 0, (const sp1b200_memory_event*)in[s].d, keys[s],
                           idx[s], n[s], h[s], previous[s], (uint32_t)s, (uint32_t*)trace[s].d,
                           (uint32_t*)lookups.d + lk_off[s] * LK_WORDS, (uint32_t*)globals.d + ge_off[s] * GE_WORDS,
                           d_flags + F_PER * s + F_ORDER);
        if (h[2])
            SP1_LAUNCH(ctx, memory_local_rows_kernel, blocks_for(h[2], ROWS), ROWS, 0, (const sp1b200_memory_local_event*)in[2].d, n[2], h[2],
                       (uint32_t*)trace[2].d, (uint32_t*)lookups.d + lk_off[2] * LK_WORDS, (uint32_t*)globals.d + ge_off[2] * GE_WORDS,
                       d_flags + F_PER * 2);
        t.stop();
    }
    unsigned long long flags[3 * F_PER];
    SP1_CUDA(cudaMemcpyAsync(flags, d_flags, sizeof(flags), cudaMemcpyDeviceToHost, st));
    SP1_CUDA(cudaStreamSynchronize(st));
    for (int s = 0; s < 3; s++) {
        const unsigned long long* f = flags + F_PER * s;
        if (f[F_ADDR] == NONE && f[F_TS] == NONE && f[F_ORDER] == NONE) continue;
        if (s == 2) {
            sp1b200_memory_local_event e;
            const uint64_t i = f[F_ADDR] != NONE ? f[F_ADDR] : f[F_TS];
            SP1_CUDA(cudaMemcpy(&e, (const sp1b200_memory_local_event*)in[2].d + i, sizeof(e), cudaMemcpyDeviceToHost));
            if (f[F_ADDR] != NONE)
                return sp1b200_set_error("%s: local event %llu has address 0x%llx >= 2^48", what, (unsigned long long)i, (unsigned long long)e.addr);
            const bool init_bad = e.initial_timestamp >= TS_LIMIT;
            return sp1b200_set_error("%s: local event %llu has %s timestamp 0x%llx >= 2^48 (clk_high would not fit 24 bits)", what,
                                     (unsigned long long)i, init_bad ? "initial" : "final",
                                     (unsigned long long)(init_bad ? e.initial_timestamp : e.final_timestamp));
        }
        if (f[F_ADDR] != NONE || f[F_TS] != NONE) {
            sp1b200_memory_event e;
            const uint64_t i = f[F_ADDR] != NONE ? f[F_ADDR] : f[F_TS];
            SP1_CUDA(cudaMemcpy(&e, (const sp1b200_memory_event*)in[s].d + i, sizeof(e), cudaMemcpyDeviceToHost));
            if (f[F_ADDR] != NONE)
                return sp1b200_set_error("%s: %s event %llu has address 0x%llx >= 2^48", what, SECTION[s], (unsigned long long)i,
                                         (unsigned long long)e.addr);
            return sp1b200_set_error("%s: %s event %llu has timestamp 0x%llx >= 2^48 (clk_high would not fit 24 bits)", what, SECTION[s],
                                     (unsigned long long)i, (unsigned long long)e.timestamp);
        }
        // row r's address is not above the one before it (sorted), or not above previous_*_addr at row 0
        const uint64_t r = f[F_ORDER];
        uint64_t addr, prev = previous[s];
        uint32_t i;
        SP1_CUDA(cudaMemcpy(&addr, keys[s] + r, 8, cudaMemcpyDeviceToHost));
        if (r) SP1_CUDA(cudaMemcpy(&prev, keys[s] + r - 1, 8, cudaMemcpyDeviceToHost));
        SP1_CUDA(cudaMemcpy(&i, idx[s] + r, 4, cudaMemcpyDeviceToHost));
        if (r && addr == prev)
            return sp1b200_set_error("%s: duplicate %s address 0x%llx (event %u)", what, SECTION[s], (unsigned long long)addr, i);
        return sp1b200_set_error("%s: %s event %u has address 0x%llx, not above previous_%s_addr 0x%llx", what, SECTION[s], i,
                                 (unsigned long long)addr, SECTION[s], (unsigned long long)prev);
    }
    for (int s = 0; s < 3; s++) SP1_TRY(trace[s].finish());
    SP1_TRY(lookups.finish());
    SP1_TRY(globals.finish());
    t_all.stop();
    return nullptr;
}
