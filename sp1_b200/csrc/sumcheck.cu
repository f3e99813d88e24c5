// The eq-table and per-column evaluation kernels the sumcheck and PCS drivers share (declared in sumcheck.cuh).
#include "sumcheck.cuh"

namespace {

using kb::Ext;

// The EQ_LOW_BITS low bits of j vary inside a block, the others do not: their product is formed once per block, so a thread
// does EQ_LOW_BITS products instead of k.  Launched with 2^EQ_LOW_BITS threads.
constexpr int EQ_LOW_BITS = 8;
__global__ void __launch_bounds__(1 << EQ_LOW_BITS) eq_table_kernel(const uint32_t* __restrict__ point, int k, uint32_t* __restrict__ E) {
    const int lo = k < EQ_LOW_BITS ? k : EQ_LOW_BITS;
    const uint64_t j0 = (uint64_t)blockIdx.x << EQ_LOW_BITS, j = j0 + threadIdx.x;
    auto factor = [&](uint64_t idx, int t) {
        const Ext x = kb::ext_load(point + 4 * t);
        return ((idx >> (k - 1 - t)) & 1) ? x : kb::ext_sub(kb::ext_one(), x);
    };
    __shared__ Ext high;
    if (threadIdx.x == 0) {
        Ext acc = kb::ext_one();
        for (int t = 0; t < k - lo; t++) acc = kb::ext_mul(acc, factor(j0, t));
        high = acc;
    }
    __syncthreads();
    if (j >= ((uint64_t)1 << k)) return;
    Ext acc = high;
    for (int t = k - lo; t < k; t++) acc = kb::ext_mul(acc, factor(j, t));
    kb::ext_store(E + 4 * j, acc);
}

__global__ void halve_eq_kernel(const uint32_t* __restrict__ E, uint64_t n_out, uint32_t* __restrict__ Eo) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_out) return;
    kb::ext_store(Eo + 4 * j, kb::ext_add(kb::ext_load(E + 8 * j), kb::ext_load(E + 8 * j + 4)));
}

// per-column evaluations of many tables in two launches: out[c] = sum_{r < rows} eq[r] * col[r].
// A block takes one chunk of EVAL_ROWS rows of one table, keeps its eq values in registers and walks all the table's columns
// (coalesced column-major reads, 4 products per 64-bit accumulator and reduction); per-column block sums go to
// partial[(blk_of_table)][col], a second launch adds the chunks.
constexpr int EVAL_ROWS_PER_THREAD = 16;
constexpr int EVAL_ROWS = 256 * EVAL_ROWS_PER_THREAD;
struct EvalJob { const uint32_t* cols; uint64_t h; uint32_t w, blk_start, nblk, out_col; uint64_t part_off; };

template <class J>
__device__ __forceinline__ int eval_find_job(const J* __restrict__ jobs, int n, uint32_t blk) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (jobs[mid].blk_start <= blk) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(256) table_evals_partial_kernel(const EvalJob* __restrict__ jobs, int n_jobs, const uint32_t* __restrict__ eq,
                                                                  uint32_t* __restrict__ partial) {
    const EvalJob job = jobs[eval_find_job(jobs, n_jobs, blockIdx.x)];
    const uint32_t chunk = blockIdx.x - job.blk_start;
    const uint64_t row0 = (uint64_t)chunk * EVAL_ROWS + threadIdx.x;
    uint4 e[EVAL_ROWS_PER_THREAD];
#pragma unroll
    for (int k = 0; k < EVAL_ROWS_PER_THREAD; k++) {
        const uint64_t r = row0 + (uint64_t)k * 256;
        e[k] = r < job.h ? __ldg(reinterpret_cast<const uint4*>(eq + 4 * r)) : make_uint4(0, 0, 0, 0);
    }
    __shared__ uint32_t red[8][4];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* outp = partial + (job.part_off + (uint64_t)chunk * job.w) * 4;
    for (uint32_t c = 0; c < job.w; c++) {
        const uint32_t* col = job.cols + (uint64_t)c * job.h;
        uint32_t a0 = 0, a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
        for (int k4 = 0; k4 < EVAL_ROWS_PER_THREAD; k4 += 4) {
            uint64_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
#pragma unroll
            for (int k = k4; k < k4 + 4; k++) {
                const uint64_t r = row0 + (uint64_t)k * 256;
                const uint32_t x = r < job.h ? __ldg(col + r) : 0u;
                s0 = kb::mac(x, e[k].x, s0); s1 = kb::mac(x, e[k].y, s1); s2 = kb::mac(x, e[k].z, s2); s3 = kb::mac(x, e[k].w, s3);
            }
            a0 = kb::add(a0, kb::monty_reduce2(s0)); a1 = kb::add(a1, kb::monty_reduce2(s1));
            a2 = kb::add(a2, kb::monty_reduce2(s2)); a3 = kb::add(a3, kb::monty_reduce2(s3));
        }
        for (int sft = 16; sft > 0; sft >>= 1) {
            a0 = kb::add(a0, __shfl_down_sync(0xffffffffu, a0, sft)); a1 = kb::add(a1, __shfl_down_sync(0xffffffffu, a1, sft));
            a2 = kb::add(a2, __shfl_down_sync(0xffffffffu, a2, sft)); a3 = kb::add(a3, __shfl_down_sync(0xffffffffu, a3, sft));
        }
        __syncthreads();  // previous column's red[] has been consumed
        if (lane == 0) { red[warp][0] = a0; red[warp][1] = a1; red[warp][2] = a2; red[warp][3] = a3; }
        __syncthreads();
        if (threadIdx.x < 4) {
            uint32_t v = 0;
            for (int w = 0; w < 8; w++) v = kb::add(v, red[w][threadIdx.x]);
            outp[4 * c + threadIdx.x] = v;
        }
    }
}
// out[(job.out_col + c)] = sum over the table's chunks; one block per table, thread -> (column, limb)
__global__ void __launch_bounds__(256) table_evals_reduce_kernel(const EvalJob* __restrict__ jobs, const uint32_t* __restrict__ partial,
                                                                 uint32_t* __restrict__ out) {
    const EvalJob job = jobs[blockIdx.x];
    for (uint32_t t = threadIdx.x; t < job.w * 4; t += blockDim.x) {
        uint32_t v = 0;
        for (uint32_t b = 0; b < job.nblk; b++) v = kb::add(v, partial[(job.part_off + (uint64_t)b * job.w) * 4 + t]);
        out[(uint64_t)job.out_col * 4 + t] = v;
    }
}

}  // namespace

sp1b200_err launch_eq_table(sp1b200_ctx* ctx, const uint32_t* d_point, int k, uint32_t* d_out) {
    SP1_LAUNCH(ctx, eq_table_kernel, blocks_for((uint64_t)1 << k, 1u << EQ_LOW_BITS), 1u << EQ_LOW_BITS, 0, d_point, k, d_out);
    return nullptr;
}

sp1b200_err launch_halve_eq(sp1b200_ctx* ctx, const uint32_t* d_E, uint64_t n_out, uint32_t* d_out) {
    SP1_LAUNCH(ctx, halve_eq_kernel, blocks_for(n_out), 256, 0, d_E, n_out, d_out);
    return nullptr;
}

sp1b200_err launch_table_evals(sp1b200_ctx* ctx, const std::vector<EvalTable>& tables, const uint32_t* d_eq, uint32_t* d_out, size_t n_out) {
    std::vector<EvalJob> jobs;
    uint32_t blk = 0; uint64_t part = 0;
    for (const EvalTable& t : tables) {
        if (!t.height || !t.width) continue;
        const uint32_t nb = (uint32_t)((t.height + EVAL_ROWS - 1) / EVAL_ROWS);
        jobs.push_back(EvalJob{t.cols, t.height, t.width, blk, nb, t.first_out, part});
        blk += nb; part += (uint64_t)nb * t.width;
    }
    SP1_CUDA(cudaMemsetAsync(d_out, 0, n_out * 16, ctx->stream));
    if (jobs.empty()) return nullptr;
    DevFree mem(ctx);  // freed in stream order, after the launches below
    EvalJob* d_jobs; uint32_t* d_part;
    SP1_TRY(mem.alloc((void**)&d_jobs, jobs.size() * sizeof(EvalJob)));
    SP1_TRY(mem.alloc((void**)&d_part, part * 16));
    SP1_CUDA(cudaMemcpyAsync(d_jobs, jobs.data(), jobs.size() * sizeof(EvalJob), cudaMemcpyHostToDevice, ctx->stream));
    SP1_LAUNCH(ctx, table_evals_partial_kernel, blk, 256, 0, d_jobs, (int)jobs.size(), d_eq, d_part);
    SP1_LAUNCH(ctx, table_evals_reduce_kernel, (unsigned)jobs.size(), 256, 0, d_jobs, d_part, d_out);
    return nullptr;
}
