// Radix sorts of 64-bit keys on the context's stream, their temporary storage taken from the context's pool (returned when `mem`
// goes): the duplicate-key check of program setup (setup.cu) and the address order of the memory chips (memory_traces.cu).
#pragma once
#include "ctx.cuh"
#include "sumcheck.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace radix_sort {

// d_out[0 .. n) = d_in sorted ascending on key bits [0, end_bit); n < 2^31
inline sp1b200_err keys(sp1b200_ctx* ctx, DevFree& mem, const uint64_t* d_in, uint64_t* d_out, uint64_t n, int end_bit) {
    size_t tb = 0;
    void* d_tmp = nullptr;
    SP1_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, d_in, d_out, (int)n, 0, end_bit, ctx->stream));
    SP1_TRY(mem.alloc(&d_tmp, tb));
    SP1_CUDA(cub::DeviceRadixSort::SortKeys(d_tmp, tb, d_in, d_out, (int)n, 0, end_bit, ctx->stream));
    ctx->launches++;
    return nullptr;
}

// the same with a 32-bit payload carried along; the sort is stable, so equal keys keep their payloads' input order
inline sp1b200_err pairs(sp1b200_ctx* ctx, DevFree& mem, const uint64_t* d_keys_in, uint64_t* d_keys_out, const uint32_t* d_vals_in,
                         uint32_t* d_vals_out, uint64_t n, int end_bit) {
    size_t tb = 0;
    void* d_tmp = nullptr;
    SP1_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, d_keys_in, d_keys_out, d_vals_in, d_vals_out, (int)n, 0, end_bit, ctx->stream));
    SP1_TRY(mem.alloc(&d_tmp, tb));
    SP1_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, d_keys_in, d_keys_out, d_vals_in, d_vals_out, (int)n, 0, end_bit, ctx->stream));
    ctx->launches++;
    return nullptr;
}

}  // namespace radix_sort
