// Plumbing shared by the sumcheck and PCS drivers (gkr.cu, zerocheck.cu, jagged.cu, pcs.cu; ntt.cu for root_pow): pool scope,
// launch geometry, the eq table, the block reduction that posts to the mailbox and the host sums of its per-block partials.
// Everything here is inline or a template (an unused internal-linkage function would be compiled and warned about in every
// including translation unit); the table kernels live once, in sumcheck.cu.
#pragma once
#include "ctx.cuh"
#include "hostfield.hpp"
#include "kb31.cuh"
#include <vector>

// stream-ordered pool allocations, freed at scope exit
struct DevFree {
    sp1b200_ctx* ctx;
    std::vector<void*> ptrs;
    explicit DevFree(sp1b200_ctx* c) : ctx(c) {}
    ~DevFree() { for (void* p : ptrs) cudaFreeAsync(p, ctx->stream); }
    sp1b200_err alloc(void** p, size_t bytes) {
        SP1_CUDA(cudaMallocFromPoolAsync(p, bytes ? bytes : 4, ctx->pool, ctx->stream));
        ptrs.push_back(*p);
        return nullptr;
    }
};
inline unsigned blocks_for(uint64_t n, unsigned bs = 256) { return (unsigned)((n + bs - 1) / bs); }

// w^e for the two-adic generator w of order 2^24, from the context's tables: TH[e >> 12] * TL[e & 4095]
__device__ __forceinline__ uint32_t root_pow(const uint32_t* __restrict__ TH, const uint32_t* __restrict__ TL, uint32_t e) {
    uint32_t hi = __ldg(TH + (e >> 12));
    uint32_t lo = e & 4095u;
    return lo ? kb::mul(hi, __ldg(TL + lo)) : hi;
}

// One layer of the jagged branching program (slop/crates/jagged/src/poly.rs:136-175, 384-470), for the prover's kernels
// (jagged.cu) and the verifier's host evaluation (verify.cu).  state = carry + 2 * comparison_so_far; returns -1 on failure.
__host__ __device__ __forceinline__ int bp_transition(int row_bit, int index_bit, int cur_bit, int next_bit, int state) {
    int carry = state & 1, cmp = state >> 1;
    int new_cmp = (index_bit == next_bit) ? cmp : next_bit;
    int s = row_bit + carry + cur_bit;
    if (index_bit != (s & 1)) return -1;
    return (s >> 1) + 2 * new_cmp;
}

// E[j] = prod_t (bit (k-1-t) of j ? x_t : 1 - x_t) for j < 2^k, point[0] <-> most significant bit of j (sumcheck.cu)
sp1b200_err launch_eq_table(sp1b200_ctx* ctx, const uint32_t* d_point, int k, uint32_t* d_out);
// E'[j] = E[2j] + E[2j+1], j < n_out: drops the last coordinate of the eq point (sumcheck.cu)
sp1b200_err launch_halve_eq(sp1b200_ctx* ctx, const uint32_t* d_E, uint64_t n_out, uint32_t* d_out);

// `width` base-field columns of `height` rows each, column-major at `cols`; their evaluations go to out[first_out ..]
struct EvalTable { const uint32_t* cols; uint64_t height; uint32_t width, first_out; };
// out[t.first_out + c] = sum_{r < t.height} eq[r] * t.cols[c * t.height + r] for every table t, in two launches (sumcheck.cu).
// d_out holds n_out EF values; the ones no table writes are zero.  Tables with no rows or no columns are skipped.
sp1b200_err launch_table_evals(sp1b200_ctx* ctx, const std::vector<EvalTable>& tables, const uint32_t* d_eq, uint32_t* d_out, size_t n_out);

// NE extension sums per block -> partial[block][4 NE] (the mailbox payload: the host transcript polls the flag, ctx.cuh); a null
// mail flag makes it a plain reduction.  Warp shuffles + one barrier (the late sumcheck rounds are latency-bound: a shared-memory
// tree costs 8 barriers).  Every thread of the block calls it; blocks have at most 8 warps.
template <int NE>
__device__ __forceinline__ void block_reduce(const kb::Ext (&v)[NE], uint32_t* __restrict__ partial, const Mail& mail) {
    __shared__ uint32_t red[4 * NE][8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 4 * NE; k++) {
        uint32_t x = v[k / 4].c[k % 4];
#pragma unroll
        for (int sft = 16; sft > 0; sft >>= 1) x = kb::add(x, __shfl_down_sync(0xffffffffu, x, sft));
        if (lane == 0) red[k][warp] = x;
    }
    __syncthreads();
    if (threadIdx.x < 4 * NE) {
        uint32_t x = 0;
        for (int q = 0; q < (int)(blockDim.x >> 5); q++) x = kb::add(x, red[threadIdx.x][q]);
        partial[blockIdx.x * 4 * NE + threadIdx.x] = x;
    }
    sp1_mail_done(mail);
}

// host sums of the per-block partials of block_reduce<NE>: s[q] = sum_k h[k][q]
template <int NE>
void sum_partials(const uint32_t* h, unsigned nblk, hf::E4 (&s)[NE]) {
    for (auto& x : s) x = hf::E4();
    for (unsigned k = 0; k < nblk; k++)
        for (int q = 0; q < NE; q++) s[q] = s[q] + hf::E4::load(&h[4 * (NE * k + q)]);
}
// ... posted to the mailbox by the launch with sequence number `seq`
template <int NE>
sp1b200_err sum_mail_partials(sp1b200_ctx* ctx, uint32_t seq, unsigned nblk, hf::E4 (&s)[NE]) {
    SP1_TRY(sp1b200_mail_wait(ctx, seq));
    sum_partials<NE>(sp1b200_mail_host(ctx), nblk, s);
    return nullptr;
}
// ... left in device memory (copy + synchronise)
template <int NE>
sp1b200_err sum_device_partials(sp1b200_ctx* ctx, const uint32_t* d_partial, unsigned nblk, hf::E4 (&s)[NE]) {
    std::vector<uint32_t> h((size_t)nblk * 4 * NE);
    SP1_CUDA(cudaMemcpyAsync(h.data(), d_partial, h.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
    SP1_CUDA(cudaStreamSynchronize(ctx->stream));
    sum_partials<NE>(h.data(), nblk, s);
    return nullptr;
}
