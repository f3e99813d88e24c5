// The eq-table kernels every sumcheck and PCS driver shares (declared in sumcheck.cuh).
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

}  // namespace

sp1b200_err launch_eq_table(sp1b200_ctx* ctx, const uint32_t* d_point, int k, uint32_t* d_out) {
    SP1_LAUNCH(ctx, eq_table_kernel, blocks_for((uint64_t)1 << k, 1u << EQ_LOW_BITS), 1u << EQ_LOW_BITS, 0, d_point, k, d_out);
    return nullptr;
}

sp1b200_err launch_halve_eq(sp1b200_ctx* ctx, const uint32_t* d_E, uint64_t n_out, uint32_t* d_out) {
    SP1_LAUNCH(ctx, halve_eq_kernel, blocks_for(n_out), 256, 0, d_E, n_out, d_out);
    return nullptr;
}
