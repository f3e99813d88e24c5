// Program setup: the verifying key's words after the preprocessed commitment, computed from the program's memory image
// (MachineProgram::pc_start / initial_global_cumulative_sum / untrusted_config, crates/core/executor/src/program.rs:161-229).
// One thread lifts one image entry onto the septic curve (septic.cuh), a tree of per-thread chunk sums adds the points under the
// complete law, and a radix sort of the keys finds duplicate addresses and page indices.
#include "ctx.cuh"
#include "radix_sort.cuh"
#include "septic.cuh"
#include "sumcheck.cuh"

namespace {

constexpr uint32_t SUM_CHUNK = 16;   // points per thread and tree level
constexpr uint64_t NONE = ~0ull;

// entry i < n_mem: memory entry i; n_mem <= i < n: page entry i - n_mem; i = n: SepticDigest::zero().  pts[i] = -lift_x(message);
// an entry without a point leaves infinity and records its index in *failed (lowest wins).
__global__ void __launch_bounds__(128) setup_lift_kernel(const uint64_t* __restrict__ addrs, const uint64_t* __restrict__ words,
                                                         uint64_t n_mem, const uint64_t* __restrict__ pages, const uint8_t* __restrict__ prots,
                                                         uint64_t n, uint32_t* __restrict__ pts, unsigned long long* failed) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    if (i == n) { s7::store_point(s7::digest_zero(), pts + 14 * i); return; }
    uint32_t m[8];
    if (i < n_mem) s7::memory_message(addrs[i], words[i], m);
    else s7::page_message(pages[i - n_mem], prots[i - n_mem], m);
    s7::Pt p;
    if (s7::lift_x(m, p) < 0) {
        atomicMin(failed, (unsigned long long)i);
        p = s7::infinity();
    } else {
        p = s7::neg(p);
    }
    s7::store_point(p, pts + 14 * i);
}

// out[t] = in[t * SUM_CHUNK] + ... + in[min(n, (t + 1) * SUM_CHUNK) - 1] under the complete law
__global__ void __launch_bounds__(128) setup_sum_kernel(const uint32_t* __restrict__ in, uint64_t n, uint32_t* __restrict__ out) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t b = t * SUM_CHUNK;
    if (b >= n) return;
    const uint64_t e = b + SUM_CHUNK < n ? b + SUM_CHUNK : n;
    s7::Pt acc = s7::load_point(in + 14 * b);
    for (uint64_t k = b + 1; k < e; k++) acc = s7::add_complete(acc, s7::load_point(in + 14 * k));
    s7::store_point(acc, out + 14 * t);
}

// sorted keys: the lowest key that occurs twice
__global__ void setup_dup_kernel(const uint64_t* __restrict__ keys, uint64_t n, unsigned long long* dup) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i + 1 < n && keys[i] == keys[i + 1]) atomicMin(dup, (unsigned long long)keys[i]);
}

sp1b200_err find_duplicate(sp1b200_ctx* ctx, DevFree& mem, const uint64_t* d_keys, uint64_t n, unsigned long long* d_dup) {
    if (n < 2) return nullptr;
    uint64_t* d_sorted;
    SP1_TRY(mem.alloc((void**)&d_sorted, n * 8));
    SP1_TRY(radix_sort::keys(ctx, mem, d_keys, d_sorted, n, 64));
    SP1_LAUNCH(ctx, setup_dup_kernel, blocks_for(n), 256, 0, d_sorted, n, d_dup);
    return nullptr;
}

}  // namespace

extern "C" sp1b200_err sp1b200_program_vk_tail(sp1b200_ctx* ctx, uint64_t pc_start_abs, const uint64_t* mem_addrs_any,
                                               const uint64_t* mem_words_any, uint64_t n_mem, const uint64_t* page_idx_any,
                                               const uint8_t* page_prot_any, uint64_t n_pages, int enable_untrusted_programs,
                                               uint32_t* h_vk_tail24) {
    SP1_DEVICE_GUARD(ctx);
    if (!ctx || !h_vk_tail24) return sp1b200_set_error("program_vk_tail: NULL argument");
    if (n_mem && (!mem_addrs_any || !mem_words_any)) return sp1b200_set_error("program_vk_tail: NULL memory image with %llu entries", (unsigned long long)n_mem);
    if (n_pages && (!page_idx_any || !page_prot_any)) return sp1b200_set_error("program_vk_tail: NULL page image with %llu entries", (unsigned long long)n_pages);
    if (enable_untrusted_programs != 0 && enable_untrusted_programs != 1)
        return sp1b200_set_error("program_vk_tail: enable_untrusted_programs is %d, not 0 or 1", enable_untrusted_programs);
    const uint64_t n_pg = enable_untrusted_programs ? n_pages : 0;   // without untrusted programs the page image is not read
    const uint64_t n = n_mem + n_pg;
    if (n_mem >= (1ull << 31) || n_pg >= (1ull << 31) || n >= (1ull << 31) - 1)
        return sp1b200_set_error("program_vk_tail: %llu image entries (at most 2^31 - 2)", (unsigned long long)n);
    cudaStream_t st = ctx->stream;
    DevFree mem(ctx);
    DevBuf addrs, words, pages, prots;
    SP1_TRY(addrs.in(ctx, mem_addrs_any, n_mem * 8));
    SP1_TRY(words.in(ctx, mem_words_any, n_mem * 8));
    SP1_TRY(pages.in(ctx, page_idx_any, n_pg * 8));
    SP1_TRY(prots.in(ctx, page_prot_any, n_pg));
    // flags: [0] lowest duplicate address, [1] lowest duplicate page index, [2] lowest entry without a point
    unsigned long long* d_flags;
    SP1_TRY(mem.alloc((void**)&d_flags, 3 * 8));
    SP1_CUDA(cudaMemsetAsync(d_flags, 0xff, 3 * 8, st));
    uint32_t *d_a, *d_b;
    SP1_TRY(mem.alloc((void**)&d_a, (n + 1) * 14 * 4));
    SP1_TRY(mem.alloc((void**)&d_b, (n / SUM_CHUNK + 1) * 14 * 4));
    PhaseTimer t_all(ctx, "program_vk_tail");
    SP1_TRY(find_duplicate(ctx, mem, (const uint64_t*)addrs.d, n_mem, d_flags));
    SP1_TRY(find_duplicate(ctx, mem, (const uint64_t*)pages.d, n_pg, d_flags + 1));
    {
        PhaseTimer t(ctx, "program_vk_tail.lift");
        SP1_LAUNCH(ctx, setup_lift_kernel, blocks_for(n + 1, 128), 128, 0, (const uint64_t*)addrs.d, (const uint64_t*)words.d, n_mem,
                   (const uint64_t*)pages.d, (const uint8_t*)prots.d, n, d_a, d_flags + 2);
        t.stop();
    }
    uint64_t m = n + 1;
    {
        PhaseTimer t(ctx, "program_vk_tail.sum");
        while (m > 1) {
            const uint64_t threads = (m + SUM_CHUNK - 1) / SUM_CHUNK;
            SP1_LAUNCH(ctx, setup_sum_kernel, blocks_for(threads, 128), 128, 0, d_a, m, d_b);
            std::swap(d_a, d_b);
            m = threads;
        }
        t.stop();
    }
    t_all.stop();
    unsigned long long flags[3];
    uint32_t sum[14];
    SP1_CUDA(cudaMemcpyAsync(flags, d_flags, sizeof(flags), cudaMemcpyDeviceToHost, st));
    SP1_CUDA(cudaMemcpyAsync(sum, d_a, sizeof(sum), cudaMemcpyDeviceToHost, st));
    SP1_CUDA(cudaStreamSynchronize(st));
    if (flags[0] != NONE) return sp1b200_set_error("program_vk_tail: duplicate memory address 0x%llx in the memory image", flags[0]);
    if (flags[1] != NONE) return sp1b200_set_error("program_vk_tail: duplicate page index 0x%llx in the page image", flags[1]);
    if (flags[2] != NONE) {
        const uint64_t i = flags[2];
        uint64_t key = 0;
        const uint64_t* src = i < n_mem ? (const uint64_t*)addrs.d + i : (const uint64_t*)pages.d + (i - n_mem);
        SP1_CUDA(cudaMemcpy(&key, src, 8, cudaMemcpyDeviceToHost));
        return sp1b200_set_error("program_vk_tail: no curve point for the %s 0x%llx after 256 offsets", i < n_mem ? "memory address" : "page index",
                                 (unsigned long long)key);
    }
    bool inf = true;
    for (uint32_t w : sum) inf = inf && w == 0;
    if (inf) return sp1b200_set_error("program_vk_tail: the initial global cumulative sum is the point at infinity");
    h_vk_tail24[0] = kb::to_monty_c(pc_start_abs & 0xFFFF);
    h_vk_tail24[1] = kb::to_monty_c((pc_start_abs >> 16) & 0xFFFF);
    h_vk_tail24[2] = kb::to_monty_c((pc_start_abs >> 32) & 0xFFFF);
    for (int i = 0; i < 14; i++) h_vk_tail24[3 + i] = sum[i];
    h_vk_tail24[17] = enable_untrusted_programs ? kb::ONE : 0;
    for (int i = 18; i < 24; i++) h_vk_tail24[i] = 0;
    SP1_TRY(addrs.finish()); SP1_TRY(words.finish()); SP1_TRY(pages.finish());
    return prots.finish();
}
