// oracle/ref_launcher.cu — TEST INFRASTRUCTURE ONLY ("the checker").  Never linked into sp1_b200/libsp1b200.so.
//
// The reference's own CUDA kernels (sp1-gpu/crates/sys/lib/**, compiled UNMODIFIED from the reference sources by
// oracle/Makefile into oracle/_ref/) are launched from Rust by kernel pointer (sys/src/runtime.rs:151-158,
// `cuda_launch_kernel(ptr, grid, block, args, smem, stream)`).  This file is the C launcher that stands in for that
// Rust host code so that the `-m gpu` tests can compare libsp1b200 and the CPU oracle with reference-held code, and so
// that bench.py can time the reference kernels head to head ("vs_ref_kernels").  Grid / block sizes are the ones the
// reference host code uses (cited per function).  Only thin `__global__` wrappers that call the reference's device
// classes (kb31_t, kb31_extension_t, poseidon2::KoalaBearHasher, DuplexChallenger) are defined here; no algorithm is.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "fields/kb31_t.cuh"
#include "fields/kb31_extension_t.cuh"
#include "poseidon2/poseidon2.cuh"
#include "merkle_tree/merkle_tree.cuh"
#include "challenger/challenger.cuh"
#include "basefold/basefold.cuh"
#include "mle/mle.cuh"
#include "logup_gkr/tracegen.cuh"
#include "logup_gkr/execution.cuh"
#include "logup_gkr/first_layer.cuh"
#include "logup_gkr/lookahead.cuh"
#include "logup_gkr/round.cuh"
#include "zerocheck/sequential.cuh"
#include "zerocheck/aggregate.cuh"
#include "zerocheck/geq_corrections.cuh"
#include "zerocheck/gkr_sweep.cuh"
#include "zerocheck/jagged_mle.cuh"
#include "zerocheck/pad_adj.cuh"
#include "jagged_assist/chip_layouts.cuh"
#include "jagged_sumcheck/jagged_sumcheck.cuh"
#include "tracegen/jagged_tracegen/jagged.cuh"
#include "runtime/exception.cuh"

// sys/include/ntt/sppark.cuh (definitions live in lib/ntt/sppark.cu; prototypes restated: sys/src/dft.rs:5-50)
extern "C" rustCudaError_t sppark_init(const cudaStream_t stream);
extern "C" rustCudaError_t batch_coset_dft(kb31_t* d_out, kb31_t* d_in, uint32_t lg_domain_size, uint32_t lg_blowup, kb31_t shift,
                                           uint32_t poly_count, bool bit_rev_output, const cudaStream_t stream);

static thread_local char g_err[512];
#define RCHK(expr)                                                                                         \
    do {                                                                                                   \
        cudaError_t e_ = (expr);                                                                           \
        if (e_ != cudaSuccess) {                                                                           \
            snprintf(g_err, sizeof g_err, "%s:%d %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e_)); \
            return g_err;                                                                                  \
        }                                                                                                  \
    } while (0)

struct Timer {
    cudaEvent_t a, b;
    Timer() { cudaEventCreate(&a); cudaEventCreate(&b); }
    ~Timer() { cudaEventDestroy(a); cudaEventDestroy(b); }
    void start(cudaStream_t s) { cudaEventRecord(a, s); }
    float stop(cudaStream_t s) {
        cudaEventRecord(b, s);
        cudaEventSynchronize(b);
        float ms = 0;
        cudaEventElapsedTime(&ms, a, b);
        return ms;
    }
};

// ---- thin wrappers over the reference device classes ------------------------------------------------------------------

// op: 0 add, 1 sub, 2 mul, 3 reciprocal(a), 4 a^3 (operator^= int), 5 neg
__global__ void ref_field_op_kernel(int op, const kb31_t* a, const kb31_t* b, kb31_t* out, size_t n) {
    for (size_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)blockDim.x * gridDim.x) {
        kb31_t x = a[i], y = b[i], r;
        switch (op) {
        case 0: r = x + y; break;
        case 1: r = x - y; break;
        case 2: r = x * y; break;
        case 3: r = x.reciprocal(); break;
        case 4: r = x; r ^= 3; break;
        default: r = -x; break;
        }
        out[i] = r;
    }
}

// op: 0 add, 1 sub, 2 mul, 3 reciprocal(a), 4 ext*base (b.value[0]), 5 interpolateLinear: a.interpolateLinear(one=b, zero=c)
__global__ void ref_ext_op_kernel(int op, const kb31_extension_t* a, const kb31_extension_t* b, const kb31_extension_t* c,
                                  kb31_extension_t* out, size_t n) {
    for (size_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)blockDim.x * gridDim.x) {
        kb31_extension_t x = a[i], y = b[i], r;
        switch (op) {
        case 0: r = x + y; break;
        case 1: r = x - y; break;
        case 2: r = x * y; break;
        case 3: r = x.reciprocal(); break;
        case 4: r = x * y.value[0]; break;
        default: r = x.interpolateLinear(y, c[i]); break;
        }
        out[i] = r;
    }
}

__global__ void ref_permute_kernel(kb31_t* states, size_t n) {
    for (size_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)blockDim.x * gridDim.x) {
        kb31_t s[16];
        for (int k = 0; k < 16; k++) s[k] = states[i * 16 + k];
        poseidon2::KoalaBearHasher::permute(s, s);
        for (int k = 0; k < 16; k++) states[i * 16 + k] = s[k];
    }
}

// hash of n_in elements per item (sponge, poseidon2.cuh:103-122) and compress(l, r) (poseidon2.cuh:82-101)
__global__ void ref_hash_kernel(kb31_t* in, size_t n_in, kb31_t* out, size_t n_items) {
    for (size_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += (size_t)blockDim.x * gridDim.x) {
        __align__(16) kb31_t d[8];
        poseidon2::KoalaBearHasher::hash(in + i * n_in, n_in, d);
        for (int k = 0; k < 8; k++) out[i * 8 + k] = d[k];
    }
}
__global__ void ref_compress_kernel(kb31_t* l, kb31_t* r, kb31_t* out, size_t n_items) {
    for (size_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += (size_t)blockDim.x * gridDim.x) {
        __align__(16) kb31_t a[8], b[8], d[8];
        for (int k = 0; k < 8; k++) { a[k] = l[i * 8 + k]; b[k] = r[i * 8 + k]; }
        poseidon2::KoalaBearHasher::compress(a, b, d);
        for (int k = 0; k < 8; k++) out[i * 8 + k] = d[k];
    }
}

// Transcript script on the reference's device DuplexChallenger (challenger.cuh:22-112).
// ops[i]: 0 observe(vals[i]) | 1 sample -> out | 2 sample_bits(vals[i]) -> out | 3 check_witness(bits = vals[i] >> 32 ... )
__global__ void ref_challenger_script_kernel(DuplexChallenger ch, const uint32_t* ops, const uint32_t* vals, uint32_t* out, size_t n) {
    if (blockIdx.x || threadIdx.x) return;
    for (size_t i = 0; i < n; i++) {
        uint32_t op = ops[i];
        if (op == 0) {
            kb31_t v;
            v.val = vals[i];
            ch.observe(&v);
            out[i] = 0;
        } else if (op == 1) {
            out[i] = ch.sample().val;
        } else {
            out[i] = (uint32_t)ch.sample_bits(vals[i]);
        }
    }
}

// POD with the layout of DuplexChallenger's (private) members: sponge_state, input_buffer, buffer_sizes, output_buffer
struct ChallengerRaw {
    kb31_t* sponge_state;
    kb31_t* input_buffer;
    size_t* buffer_sizes;
    kb31_t* output_buffer;
};
static_assert(sizeof(ChallengerRaw) == sizeof(DuplexChallenger), "DuplexChallenger layout changed");

// kernel-argument image of a kb31_extension_t (its default constructor is __device__-only): 4 words, 4-byte aligned
struct Ext4Raw {
    uint32_t v[4];
};
static_assert(sizeof(Ext4Raw) == sizeof(kb31_extension_t) && alignof(Ext4Raw) == alignof(kb31_extension_t), "ext layout");

// device buffers owned by one launcher call: freed when it returns, on the error paths too
struct DevScope {
    std::vector<void*> bufs;
    cudaError_t alloc(void** d, size_t bytes) {
        cudaError_t e = cudaMalloc(d, bytes ? bytes : 8);
        if (e == cudaSuccess) bufs.push_back(*d);
        return e;
    }
    void release(void* p) {
        for (auto& b : bufs)
            if (b == p) { cudaFree(b); b = nullptr; }
    }
    ~DevScope() { for (void* b : bufs) if (b) cudaFree(b); }
};

struct DevChallenger {
    uint32_t* d_words = nullptr;  // 16 + 8 + 16 (the device duplexing writes WIDTH words into output_buffer)
    size_t* d_sizes = nullptr;
    ChallengerRaw raw{};
    const char* init(const uint32_t* st34) {
        RCHK(cudaMalloc(&d_words, 40 * 4));
        RCHK(cudaMalloc(&d_sizes, 2 * sizeof(size_t)));
        uint32_t w[40] = {0};
        memcpy(w, st34, 16 * 4);
        memcpy(w + 16, st34 + 16, 8 * 4);
        memcpy(w + 24, st34 + 24, 8 * 4);
        size_t sz[2] = {st34[32], st34[33]};
        RCHK(cudaMemcpy(d_words, w, sizeof w, cudaMemcpyHostToDevice));
        RCHK(cudaMemcpy(d_sizes, sz, sizeof sz, cudaMemcpyHostToDevice));
        raw.sponge_state = (kb31_t*)d_words;
        raw.input_buffer = (kb31_t*)d_words + 16;
        raw.output_buffer = (kb31_t*)d_words + 24;
        raw.buffer_sizes = d_sizes;
        return nullptr;
    }
    const char* read(uint32_t* st34) {
        uint32_t w[40];
        size_t sz[2];
        RCHK(cudaMemcpy(w, d_words, sizeof w, cudaMemcpyDeviceToHost));
        RCHK(cudaMemcpy(sz, d_sizes, sizeof sz, cudaMemcpyDeviceToHost));
        memcpy(st34, w, 32 * 4);
        st34[32] = (uint32_t)sz[0];
        st34[33] = (uint32_t)sz[1];
        return nullptr;
    }
    ~DevChallenger() { cudaFree(d_words); cudaFree(d_sizes); }
};

extern "C" {

const char* ref_init() {
    rustCudaError_t e = sppark_init(0);
    if (e.message != CUDA_SUCCESS_CSL.message) return e.message;   // success is the "no error" string (lib/runtime/exception.cu:9-10)
    RCHK(cudaDeviceSynchronize());
    return nullptr;
}

const char* ref_malloc(size_t bytes, void** out) { RCHK(cudaMalloc(out, bytes)); return nullptr; }
const char* ref_free(void* p) { RCHK(cudaFree(p)); return nullptr; }
const char* ref_h2d(void* d, const void* h, size_t bytes) { RCHK(cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice)); return nullptr; }
const char* ref_d2h(void* h, const void* d, size_t bytes) { RCHK(cudaMemcpy(h, d, bytes, cudaMemcpyDeviceToHost)); return nullptr; }

// host-buffer conveniences for the element-wise checks
const char* ref_field_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n) {
    kb31_t *da, *db, *dout;
    RCHK(cudaMalloc(&da, n * 4)); RCHK(cudaMalloc(&db, n * 4)); RCHK(cudaMalloc(&dout, n * 4));
    RCHK(cudaMemcpy(da, a, n * 4, cudaMemcpyHostToDevice));
    RCHK(cudaMemcpy(db, b, n * 4, cudaMemcpyHostToDevice));
    ref_field_op_kernel<<<256, 256>>>(op, da, db, dout, n);
    RCHK(cudaGetLastError());
    RCHK(cudaMemcpy(out, dout, n * 4, cudaMemcpyDeviceToHost));
    cudaFree(da); cudaFree(db); cudaFree(dout);
    return nullptr;
}

const char* ref_ext_op(int op, const uint32_t* a, const uint32_t* b, const uint32_t* c, uint32_t* out, size_t n) {
    kb31_extension_t *da, *db, *dc, *dout;
    RCHK(cudaMalloc(&da, n * 16)); RCHK(cudaMalloc(&db, n * 16)); RCHK(cudaMalloc(&dc, n * 16)); RCHK(cudaMalloc(&dout, n * 16));
    RCHK(cudaMemcpy(da, a, n * 16, cudaMemcpyHostToDevice));
    RCHK(cudaMemcpy(db, b, n * 16, cudaMemcpyHostToDevice));
    RCHK(cudaMemcpy(dc, c, n * 16, cudaMemcpyHostToDevice));
    ref_ext_op_kernel<<<256, 256>>>(op, da, db, dc, dout, n);
    RCHK(cudaGetLastError());
    RCHK(cudaMemcpy(out, dout, n * 16, cudaMemcpyDeviceToHost));
    cudaFree(da); cudaFree(db); cudaFree(dc); cudaFree(dout);
    return nullptr;
}

const char* ref_permute(uint32_t* states, size_t n) {
    kb31_t* d;
    RCHK(cudaMalloc(&d, n * 64));
    RCHK(cudaMemcpy(d, states, n * 64, cudaMemcpyHostToDevice));
    ref_permute_kernel<<<(unsigned)((n + 127) / 128), 128>>>(d, n);
    RCHK(cudaGetLastError());
    RCHK(cudaMemcpy(states, d, n * 64, cudaMemcpyDeviceToHost));
    cudaFree(d);
    return nullptr;
}

const char* ref_hash(const uint32_t* in, size_t n_in, uint32_t* out8, size_t n_items) {
    kb31_t *d, *o;
    RCHK(cudaMalloc(&d, (n_items * n_in + 1) * 4)); RCHK(cudaMalloc(&o, n_items * 32));
    RCHK(cudaMemcpy(d, in, n_items * n_in * 4, cudaMemcpyHostToDevice));
    ref_hash_kernel<<<(unsigned)((n_items + 127) / 128), 128>>>(d, n_in, o, n_items);
    RCHK(cudaGetLastError());
    RCHK(cudaMemcpy(out8, o, n_items * 32, cudaMemcpyDeviceToHost));
    cudaFree(d); cudaFree(o);
    return nullptr;
}

const char* ref_compress(const uint32_t* l, const uint32_t* r, uint32_t* out8, size_t n_items) {
    kb31_t *dl, *dr, *o;
    RCHK(cudaMalloc(&dl, n_items * 32)); RCHK(cudaMalloc(&dr, n_items * 32)); RCHK(cudaMalloc(&o, n_items * 32));
    RCHK(cudaMemcpy(dl, l, n_items * 32, cudaMemcpyHostToDevice));
    RCHK(cudaMemcpy(dr, r, n_items * 32, cudaMemcpyHostToDevice));
    ref_compress_kernel<<<(unsigned)((n_items + 127) / 128), 128>>>(dl, dr, o, n_items);
    RCHK(cudaGetLastError());
    RCHK(cudaMemcpy(out8, o, n_items * 32, cudaMemcpyDeviceToHost));
    cudaFree(dl); cudaFree(dr); cudaFree(o);
    return nullptr;
}

// MerkleTreeSingleLayerProver::commit_tensors (sp1-gpu/crates/merkle_tree/src/single_layer.rs:109-150): leafHashPacked with
// block 256 / grid ceil(2^h / 256), then one `compress` launch per layer k = h-1 .. 0 with block 512.
// d_mat: [width x 2^height] column-major; d_digests: (2^(height+1) - 1) x 8 words in HEAP order (root at 0, leaves at 2^h - 1 + i).
// ms_out[0] = leaf hash, ms_out[1] = all compress layers (CUDA events, device time).
const char* ref_merkle_tree(const uint32_t* d_mat, uint32_t* d_digests, size_t width, size_t height, float* ms_out) {
    poseidon2::KoalaBearHasher hasher;
    cudaStream_t s = 0;
    Timer t;
    {
        const kb31_t* in = (const kb31_t*)d_mat;
        void* dg = d_digests;
        void* args[] = {&hasher, &in, &dg, &width, &height};
        size_t block = 256, grid = (((size_t)1 << height) + block - 1) / block;
        t.start(s);
        RCHK(cudaLaunchKernel(leaf_hash_merkle_tree_koala_bear_16_kernel(), dim3((unsigned)grid), dim3((unsigned)block), args, 0, s));
        float ms = t.stop(s);
        if (ms_out) ms_out[0] = ms;
    }
    t.start(s);
    for (size_t k = height; k-- > 0;) {
        void* dg = d_digests;
        size_t kk = k;
        void* args[] = {&hasher, &dg, &kk};
        unsigned block = 512, grid = (unsigned)((((size_t)1 << k) + block - 1) / block);
        RCHK(cudaLaunchKernel(compress_merkle_tree_koala_bear_16_kernel(), dim3(grid), dim3(block), args, 0, s));
    }
    float ms = t.stop(s);
    if (ms_out) ms_out[1] = ms;
    RCHK(cudaGetLastError());
    return nullptr;
}

// SpparkDft::coset_dft_into (sp1-gpu/crates/basefold/src/encoder.rs:66-118) -> batch_coset_dft (sys/include/ntt/sppark.cuh:49-107).
// shift_monty is the word the Rust side passes (`shift / generator`, encoder.rs:80; encode_batch uses shift = 1).
const char* ref_batch_coset_dft(uint32_t* d_out, uint32_t* d_in, uint32_t lg_n, uint32_t lg_blowup, uint32_t shift_monty, uint32_t count,
                                int bit_rev_output, float* ms_out) {
    kb31_t shift;
    memcpy(&shift, &shift_monty, 4);
    Timer t;
    t.start(0);
    rustCudaError_t e = batch_coset_dft((kb31_t*)d_out, (kb31_t*)d_in, lg_n, lg_blowup, shift, count, bit_rev_output != 0, 0);
    float ms = t.stop(0);
    if (e.message != CUDA_SUCCESS_CSL.message) return e.message;
    RCHK(cudaGetLastError());
    if (ms_out) *ms_out = ms;
    return nullptr;
}

// batchKernel (sys/lib/basefold/basefold.cu:7-19); launch shape of sp1-gpu/crates/basefold: block 256, grid ceil(height/256)
const char* ref_batch(const uint32_t* d_in, uint32_t* d_out_ext, const uint32_t* d_beta_powers, size_t height, size_t width, float* ms_out) {
    void* args[] = {&d_in, &d_out_ext, &d_beta_powers, &height, &width};
    Timer t;
    t.start(0);
    RCHK(cudaLaunchKernel(batch_koala_bear_base_ext_kernel(), dim3((unsigned)((height + 255) / 256)), dim3(256), args, 0, 0));
    float ms = t.stop(0);
    RCHK(cudaGetLastError());
    if (ms_out) *ms_out = ms;
    return nullptr;
}

// foldMle<ext, ext> (sys/lib/mle/mle.cu:222-238): out[i] = beta * in[2i+1] + in[2i]
const char* ref_fold_mle_ext(const uint32_t* d_in, uint32_t* d_out, const uint32_t* h_beta4, size_t out_height, size_t width, float* ms_out) {
    Ext4Raw beta;
    memcpy(&beta, h_beta4, 16);
    void* args[] = {&d_in, &d_out, &beta, &out_height, &width};
    Timer t;
    t.start(0);
    RCHK(cudaLaunchKernel(mle_fold_koala_bear_ext_ext(), dim3((unsigned)((out_height + 255) / 256), (unsigned)width), dim3(256, 1), args, 0, 0));
    float ms = t.stop(0);
    RCHK(cudaGetLastError());
    if (ms_out) *ms_out = ms;
    return nullptr;
}

// fixLastVariableInPlace<ext> (sys/lib/mle/mle.cu:196-212): value = zero * (1 - alpha) + one * alpha; NOT in place safe across
// threads for width > 1 in general, the reference calls it per MLE; used here on a copy.
const char* ref_fix_last_variable_ext(uint32_t* d_inout, const uint32_t* h_alpha4, size_t out_height, size_t width) {
    Ext4Raw alpha;
    memcpy(&alpha, h_alpha4, 16);
    void* args[] = {&d_inout, &alpha, &out_height, &width};
    RCHK(cudaLaunchKernel(mle_fix_last_variable_in_place_koala_bear_extension(), dim3((unsigned)((out_height + 255) / 256), 1), dim3(256, 1), args, 0, 0));
    RCHK(cudaDeviceSynchronize());
    return nullptr;
}

// partial_lagrange_naive<ext> (sys/lib/mle/mle.cu:112-126): the eq table, first coordinate = most significant bit
const char* ref_partial_lagrange_ext(uint32_t* d_out, const uint32_t* d_point, size_t num_vars) {
    void* args[] = {&d_out, &d_point, &num_vars};
    size_t n = (size_t)1 << num_vars;
    RCHK(cudaLaunchKernel(partial_lagrange_koala_bear_extension(), dim3((unsigned)((n + 255) / 256)), dim3(256), args, 0, 0));
    RCHK(cudaDeviceSynchronize());
    return nullptr;
}

// grind_duplex_challenger_on_device (sp1-gpu/crates/challenger/src/grinding_challenger.rs:31-76): block 512,
// grid max(512, 2^(bits - 16)), n = field order.  The kernel returns ANY valid witness (racing found_flag).
const char* ref_grind(const uint32_t* st34, uint32_t bits, uint32_t* witness_out, float* ms_out) {
    DevChallenger ch;
    if (const char* e = ch.init(st34)) return e;
    kb31_t* d_result;
    bool* d_found;
    RCHK(cudaMalloc(&d_result, 4));
    RCHK(cudaMalloc(&d_found, 4));
    RCHK(cudaMemset(d_found, 0, 4));
    size_t b = bits, n = 0x7f000001ull;
    void* args[] = {&ch.raw, &d_result, &b, &n, &d_found};
    size_t grid = bits > 16 ? ((size_t)1 << (bits - 16)) : 1;
    if (grid < 512) grid = 512;
    Timer t;
    t.start(0);
    RCHK(cudaLaunchKernel(grind_koala_bear(), dim3((unsigned)grid), dim3(512), args, 0, 0));
    float ms = t.stop(0);
    RCHK(cudaGetLastError());
    RCHK(cudaMemcpy(witness_out, d_result, 4, cudaMemcpyDeviceToHost));
    cudaFree(d_result); cudaFree(d_found);
    if (ms_out) *ms_out = ms;
    return nullptr;
}

// run a transcript script on the reference's device challenger; st34 is updated to the final state
const char* ref_challenger_script(uint32_t* st34, const uint32_t* ops, const uint32_t* vals, uint32_t* out, size_t n) {
    DevChallenger ch;
    if (const char* e = ch.init(st34)) return e;
    uint32_t *d_ops, *d_vals, *d_out;
    RCHK(cudaMalloc(&d_ops, n * 4 + 4)); RCHK(cudaMalloc(&d_vals, n * 4 + 4)); RCHK(cudaMalloc(&d_out, n * 4 + 4));
    RCHK(cudaMemcpy(d_ops, ops, n * 4, cudaMemcpyHostToDevice));
    RCHK(cudaMemcpy(d_vals, vals, n * 4, cudaMemcpyHostToDevice));
    const uint32_t *co = d_ops, *cv = d_vals;
    void* args[] = {&ch.raw, &co, &cv, &d_out, &n};
    RCHK(cudaLaunchKernel((void*)ref_challenger_script_kernel, dim3(1), dim3(32), args, 0, 0));
    RCHK(cudaDeviceSynchronize());
    RCHK(cudaMemcpy(out, d_out, n * 4, cudaMemcpyDeviceToHost));
    cudaFree(d_ops); cudaFree(d_vals); cudaFree(d_out);
    return ch.read(st34);
}


// ---- LogUp-GKR first layer: the reference's interaction evaluation ------------------------------------------------------------------
static cudaError_t dev_upload(DevScope& mem, const void* h, size_t bytes, void** d) {
    cudaError_t e = mem.alloc(d, bytes);
    if (e == cudaSuccess && bytes) e = cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice);
    return e;
}

// The interactions of ONE chip in the flattened CSR form of `Interactions<F>` (sys/include/logup_gkr/tracegen.cuh:20-36; host twin
// sp1-gpu/crates/logup_gkr/src/interactions.rs), every index local to the chip: values_ptr / mult_ptr have n_inter + 1 entries, vcw_ptr
// n_values + 1, the column-weight lists n_vcw and n_mcw entries.
struct InteractionsCsr {
    const uint64_t *values_ptr, *mult_ptr, *vcw_ptr, *vcw_col, *mcw_col;
    const uint8_t *vcw_is_prep, *mcw_is_prep, *is_send;
    const uint32_t *vcw_weight, *values_constants, *mcw_weight, *mult_constants, *arg_indices;
    uint32_t n_inter;
    uint64_t n_values, n_vcw, n_mcw;
};

static cudaError_t upload_interactions(DevScope& mem, const InteractionsCsr& c, Interactions<felt_t>* I) {
    std::vector<PairCol<felt_t>> vcw(c.n_vcw), mcw(c.n_mcw);
    for (uint64_t i = 0; i < c.n_vcw; i++) { vcw[i].column_idx = c.vcw_col[i]; vcw[i].is_preprocessed = c.vcw_is_prep[i]; memcpy(&vcw[i].weight, &c.vcw_weight[i], 4); }
    for (uint64_t i = 0; i < c.n_mcw; i++) { mcw[i].column_idx = c.mcw_col[i]; mcw[i].is_preprocessed = c.mcw_is_prep[i]; memcpy(&mcw[i].weight, &c.mcw_weight[i], 4); }
    std::vector<uint8_t> send(c.is_send, c.is_send + c.n_inter);   // bool on the device side
    cudaError_t e;
    if ((e = dev_upload(mem, c.values_ptr, (c.n_inter + 1) * 8, (void**)&I->values_ptr)) != cudaSuccess) return e;
    if ((e = dev_upload(mem, c.mult_ptr, (c.n_inter + 1) * 8, (void**)&I->multiplicities_ptr)) != cudaSuccess) return e;
    if ((e = dev_upload(mem, c.vcw_ptr, (c.n_values + 1) * 8, (void**)&I->values_col_weights_ptr)) != cudaSuccess) return e;
    if ((e = dev_upload(mem, vcw.data(), c.n_vcw * sizeof(PairCol<felt_t>), (void**)&I->values_col_weights)) != cudaSuccess) return e;
    if ((e = dev_upload(mem, c.values_constants, c.n_values * 4, (void**)&I->values_constants)) != cudaSuccess) return e;
    if ((e = dev_upload(mem, mcw.data(), c.n_mcw * sizeof(PairCol<felt_t>), (void**)&I->mult_col_weights)) != cudaSuccess) return e;
    if ((e = dev_upload(mem, c.mult_constants, c.n_inter * 4, (void**)&I->mult_constants)) != cudaSuccess) return e;
    if ((e = dev_upload(mem, c.arg_indices, c.n_inter * 4, (void**)&I->arg_indices)) != cudaSuccess) return e;
    if ((e = dev_upload(mem, send.data(), c.n_inter, (void**)&I->is_send)) != cudaSuccess) return e;
    I->num_interactions = c.n_inter;
    return cudaSuccess;
}

// Chip by chip over CSR arrays that lie back to back: csr_enter reads the current chip's counts, csr_leave steps past its arrays.
static void csr_enter(InteractionsCsr& c, uint32_t n_inter) {
    c.n_inter = n_inter;
    c.n_values = c.values_ptr[n_inter];
    c.n_vcw = c.vcw_ptr[c.n_values];
    c.n_mcw = c.mult_ptr[n_inter];
}
static void csr_leave(InteractionsCsr& c) {
    c.values_ptr += c.n_inter + 1; c.mult_ptr += c.n_inter + 1; c.vcw_ptr += c.n_values + 1;
    c.vcw_col += c.n_vcw; c.vcw_is_prep += c.n_vcw; c.vcw_weight += c.n_vcw; c.values_constants += c.n_values;
    c.mcw_col += c.n_mcw; c.mcw_is_prep += c.n_mcw; c.mcw_weight += c.n_mcw;
    c.mult_constants += c.n_inter; c.arg_indices += c.n_inter; c.is_send += c.n_inter;
}

// What interactionValue (sys/lib/logup_gkr/tracegen.cu:20-66) reads unchecked for one chip of `height` rows: column c of a source is
// words [c * height, (c + 1) * height) of the chip's main (prep) table, of which main_avail (prep_avail) words exist; message k reads
// betas[0 .. values + 1).  nullptr when every read is in bounds.
static const char* check_interaction_reads(const InteractionsCsr& c, uint64_t height, uint64_t main_avail, uint64_t prep_avail, uint32_t n_betas) {
    if (c.n_inter && n_betas < 1) return "ref_logup_gkr: no beta powers";
    for (uint32_t j = 0; j < c.n_inter; j++)
        if (c.values_ptr[j + 1] - c.values_ptr[j] + 1 > n_betas) return "ref_logup_gkr: a message longer than the beta table";
    if (!height) return nullptr;   // an empty chip is padding: populateLastCircuitLayer reads no trace word
    auto in_bounds = [&](uint64_t col, bool prep) { return (col + 1) * height <= (prep ? prep_avail : main_avail); };
    for (uint64_t i = 0; i < c.n_vcw; i++)
        if (!in_bounds(c.vcw_col[i], c.vcw_is_prep[i])) return "ref_logup_gkr: an interaction value reads past its chip's trace";
    for (uint64_t i = 0; i < c.n_mcw; i++)
        if (!in_bounds(c.mcw_col[i], c.mcw_is_prep[i])) return "ref_logup_gkr: a multiplicity reads past its chip's trace";
    return nullptr;
}

// One populateLastCircuitLayer launch for one chip, as generate_first_layer issues it (sp1-gpu/crates/logup_gkr/src/tracegen.rs:94-139):
// block 256, grid (ceil(max(h, 2).div_ceil(2) / (256 * 8)), ceil(n_inter / 4)), is_padding = (h == 0).  out_height is the layer's total
// pair count: slot i of a chip's interaction holds row 2i at [i] and row 2i+1 at [i + 2 out_height].
static cudaError_t launch_populate(Interactions<felt_t> I, const uint32_t* d_start, uint32_t* d_col, felt_t* d_num, ext_t* d_den,
                                   felt_t* d_prep, felt_t* d_main, Ext4Raw alpha, ext_t* d_betas, size_t interaction_offset, size_t height,
                                   size_t out_height) {
    bool is_padding = height == 0;
    const size_t half = (std::max<size_t>(height, 2) + 1) / 2;
    void* args[] = {&I, &d_start, &d_col, &d_num, &d_den, &d_prep, &d_main, &alpha, &d_betas, &interaction_offset, &height, &out_height, &is_padding};
    return cudaLaunchKernel(logup_gkr_populate_last_circuit_layer(), dim3((unsigned)((half + 2047) / 2048), (I.num_interactions + 3) / 4), dim3(256),
                            args, 0, 0);
}

// populateLastCircuitLayer for ONE chip of height > 0 on its own.  Output layout as the kernel writes it: with q = ceil(ceil(height/2)/2), interaction j
// owns the row-pair slots [2 q j, 2 q j + ceil(height/2)); slot i holds (numerator at row 2i, denominator at row 2i) and, 2 * output_height
// further, the same for row 2i+1; output_height = 2 q n.
const char* ref_gkr_populate(const uint32_t* h_prep, uint64_t prep_words, const uint32_t* h_main, uint64_t main_words, uint64_t height, uint32_t n_inter,
                             const uint64_t* values_ptr, const uint64_t* mult_ptr, const uint64_t* vcw_ptr, uint64_t n_values, const uint64_t* vcw_col,
                             const uint8_t* vcw_is_prep, const uint32_t* vcw_weight, uint64_t n_vcw, const uint32_t* values_constants,
                             const uint64_t* mcw_col, const uint8_t* mcw_is_prep, const uint32_t* mcw_weight, uint64_t n_mcw,
                             const uint32_t* mult_constants, const uint32_t* arg_indices, const uint8_t* is_send, const uint32_t* alpha4,
                             const uint32_t* betas, uint32_t n_betas, uint32_t* out_num, uint32_t* out_den, uint64_t* out_height) {
    // an empty chip (is_padding) writes four slots per interaction, more than the 2 q = 2 this layout gives it: ref_logup_gkr covers that case
    if (height == 0) return "ref_gkr_populate: height 0 is not supported (the padding path writes past an interaction's slots)";
    const uint64_t half = (height + 1) / 2, q = (half + 1) / 2, outH = 2 * q * n_inter;
    DevScope mem;   // every device buffer below is freed on every return
    InteractionsCsr csr{values_ptr, mult_ptr, vcw_ptr, vcw_col, mcw_col, vcw_is_prep, mcw_is_prep, is_send, vcw_weight, values_constants,
                        mcw_weight, mult_constants, arg_indices, n_inter, n_values, n_vcw, n_mcw};
    Interactions<felt_t> I{};
    RCHK(upload_interactions(mem, csr, &I));
    std::vector<uint32_t> start(n_inter + 1);
    for (uint32_t j = 0; j <= n_inter; j++) start[j] = (uint32_t)(q * j);
    void *d_prep, *d_main, *d_start, *d_col, *d_num, *d_den, *d_betas;
    RCHK(dev_upload(mem, h_prep, prep_words * 4, &d_prep));
    RCHK(dev_upload(mem, h_main, main_words * 4, &d_main));
    RCHK(dev_upload(mem, start.data(), start.size() * 4, &d_start));
    RCHK(dev_upload(mem, betas, (size_t)n_betas * 16, &d_betas));
    RCHK(mem.alloc(&d_col, (2 * outH + 8) * 4));
    RCHK(mem.alloc(&d_num, 4 * outH * 4 + 16));
    RCHK(mem.alloc(&d_den, 4 * outH * 16 + 16));
    RCHK(cudaMemset(d_num, 0, 4 * outH * 4 + 16));
    RCHK(cudaMemset(d_den, 0, 4 * outH * 16 + 16));
    Ext4Raw alpha;
    memcpy(&alpha, alpha4, 16);
    RCHK(launch_populate(I, (const uint32_t*)d_start, (uint32_t*)d_col, (felt_t*)d_num, (ext_t*)d_den, (felt_t*)d_prep, (felt_t*)d_main, alpha,
                         (ext_t*)d_betas, 0, height, outH));
    RCHK(cudaDeviceSynchronize());
    RCHK(cudaMemcpy(out_num, d_num, 4 * outH * 4, cudaMemcpyDeviceToHost));
    RCHK(cudaMemcpy(out_den, d_den, 4 * outH * 16, cudaMemcpyDeviceToHost));
    *out_height = outH;
    return nullptr;
}

// ---- zerocheck: the reference's constraint-bytecode interpreter ----------------------------------------------------------------------
// zerocheck_fused_sequential<felt_t, 1024> (sys/lib/zerocheck/sequential.cu:110-190) over ONE chip = one chunk: per block the sum over its
// row pairs of eq[pair] * sum_k powers_of_alpha[alpha_idx_k] * reg_k at the node blockIdx.z of {0, 2, 4}, times powers_of_lambda[chip].
// trace = main columns then preprocessed columns (column-major, even height).  out12 = the three node sums (ext each); the per-block
// partials are added on the device with the reference's own kb31_extension_t addition (thin kernel below).
__global__ void ref_sum_partials_kernel(const kb31_extension_t* partials, uint32_t n_blocks, kb31_extension_t* out3) {
    if (blockIdx.x || threadIdx.x >= 3) return;
    kb31_extension_t acc = kb31_extension_t::zero();
    for (uint32_t b = 0; b < n_blocks; b++) acc += partials[b * 3 + threadIdx.x];
    out3[threadIdx.x] = acc;
}
const char* ref_zerocheck_node_sums(const uint32_t* h_instrs, uint32_t n_instrs, const uint32_t* h_leaves, uint32_t n_leaves, const uint32_t* h_consts,
                                    uint32_t n_consts, const uint32_t* h_publics, uint32_t n_publics, const uint32_t* h_assert_regs,
                                    const uint32_t* h_assert_alphas, uint32_t n_asserts, const uint32_t* h_main, uint32_t main_w,
                                    const uint32_t* h_prep, uint32_t prep_w, uint32_t height, const uint32_t* h_pv, uint32_t n_pv,
                                    const uint32_t* h_alpha_pows, uint32_t n_alpha, const uint32_t* h_E, uint32_t log_pairs, uint32_t* out12) {
    if (height & 1) return "ref_zerocheck_node_sums: even heights only (the kernel reads rows 2i and 2i+1)";
    auto up = [](const void* h, size_t bytes, void** d) -> cudaError_t {
        cudaError_t e = cudaMalloc(d, bytes ? bytes : 8);
        if (e == cudaSuccess && bytes) e = cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice);
        return e;
    };
    std::vector<uint16_t> regs16(n_asserts);
    for (uint32_t i = 0; i < n_asserts; i++) regs16[i] = (uint16_t)h_assert_regs[i];
    ChunkStatic st{};
    void *d_trace, *d_pv, *d_ap, *d_E, *d_lambda, *d_gkr, *d_disp, *d_st, *d_lay, *d_part, *d_out;
    RCHK(up(h_instrs, (size_t)n_instrs * 8, (void**)&st.instrs));
    RCHK(up(h_leaves, (size_t)n_leaves * 8, (void**)&st.leaves));
    RCHK(up(h_consts, (size_t)n_consts * 4, (void**)&st.consts));
    RCHK(up(h_publics, (size_t)n_publics * 4, (void**)&st.publics));
    RCHK(up(regs16.data(), (size_t)n_asserts * 2, (void**)&st.assert_regs));
    RCHK(up(h_assert_alphas, (size_t)n_asserts * 4, (void**)&st.assert_alphas));
    st.n_instrs = n_instrs; st.n_asserts = n_asserts; st.chip_idx = 0; st.gkr_main_width = 0; st.gkr_prep_width = 0; st.chip_alpha_offset = 0;
    std::vector<uint32_t> trace((size_t)(main_w + prep_w) * height);
    memcpy(trace.data(), h_main, (size_t)main_w * height * 4);
    if (prep_w) memcpy(trace.data() + (size_t)main_w * height, h_prep, (size_t)prep_w * height * 4);
    ChipLayout lay{0, (uint64_t)main_w * height, height, 0};
    const uint32_t pairs = height / 2, tile = 1024, n_blocks = (pairs + tile - 1) / tile;
    std::vector<BlockDispatch> disp(n_blocks ? n_blocks : 1);
    for (uint32_t b = 0; b < n_blocks; b++) disp[b] = BlockDispatch{0, b * tile, (b + 1) * tile <= pairs ? tile : pairs - b * tile};
    const uint32_t one[4] = {0x01fffffeu, 0, 0, 0};
    RCHK(up(trace.data(), trace.size() * 4, &d_trace));
    RCHK(up(h_pv, (size_t)n_pv * 4, &d_pv));
    RCHK(up(h_alpha_pows, (size_t)n_alpha * 16, &d_ap));
    RCHK(up(h_E, ((size_t)16) << log_pairs, &d_E));
    RCHK(up(one, 16, &d_lambda));
    RCHK(up(one, 16, &d_gkr));
    RCHK(up(disp.data(), disp.size() * sizeof(BlockDispatch), &d_disp));
    RCHK(up(&st, sizeof st, &d_st));
    RCHK(up(&lay, sizeof lay, &d_lay));
    RCHK(cudaMalloc(&d_part, (size_t)(n_blocks ? n_blocks : 1) * 3 * 16));
    RCHK(cudaMalloc(&d_out, 3 * 16));
    uint32_t dim = log_pairs;
    void* args[] = {&d_disp, &d_st, &d_lay, &d_trace, &d_pv, &d_ap, &d_E, &d_lambda, &d_gkr, &dim, &d_part};
    if (n_blocks) RCHK(cudaLaunchKernel(zerocheck_fused_sequential_kb_1024_kernel(), dim3(n_blocks, 1, 3), dim3(256), args, (256 / 32) * 16, 0));
    ref_sum_partials_kernel<<<1, 32>>>((const kb31_extension_t*)d_part, n_blocks, (kb31_extension_t*)d_out);
    RCHK(cudaGetLastError());
    RCHK(cudaMemcpy(out12, d_out, 48, cudaMemcpyDeviceToHost));
    for (void* p : {(void*)st.instrs, (void*)st.leaves, (void*)st.consts, (void*)st.publics, (void*)st.assert_regs, (void*)st.assert_alphas, d_trace, d_pv, d_ap,
                    d_E, d_lambda, d_gkr, d_disp, d_st, d_lay, d_part, d_out})
        cudaFree(p);
    return nullptr;
}

// ---- jagged Hadamard sumcheck: the reference's round kernels -------------------------------------------------------------------------
// DeviceTensor::sum_dim(1) over a [rows x n_blocks] tensor of per-block partials, with the reference's kb31_extension_t addition
__global__ void ref_sum_rows_kernel(const kb31_extension_t* partials, uint32_t rows, uint32_t n_blocks, kb31_extension_t* out) {
    if (blockIdx.x || threadIdx.x >= rows) return;
    kb31_extension_t acc = kb31_extension_t::zero();
    for (uint32_t b = 0; b < n_blocks; b++) acc += partials[(size_t)threadIdx.x * n_blocks + b];
    out[threadIdx.x] = acc;
}

extern "C" void* padded_hadamard_fix_and_sum();
extern "C" void* mle_fix_last_variable_koala_bear_ext_ext_zero_padding();

// jagged_sumcheck (sp1-gpu/crates/jagged_sumcheck/src/sumcheck.rs:233-355) with the challenges supplied instead of sampled: challenges[r]
// is the challenge of round r, counted from 0 (alpha_1 = challenges[0], alpha_2 = challenges[1]).  The JaggedMle<JaggedSumcheckData>
// argument is built as JaggedTraceMle::from_chip_layout builds it (sp1-gpu/crates/utils/src/traces.rs:294-350): startIndices[c] = the first
// dense PAIR of column c (n_cols + 1 entries), colIndex[j] = the column of dense pair j; col_heights are element counts.
// Raw outputs, ext (4 words) each:
//   grid8    jaggedTwoRoundSumAsPoly (sumcheck.rs:103-136), block 256, grid ceil(height / (256 * 32 * 2)), height = dense_len / 2:
//            h(0,0) h(0,1) 4h(0,1/2) h(1,0) 4h(1,1/2) 4h(1/2,0) 4h(1/2,1) 16h(1/2,1/2)
//   r2       jaggedTwoRoundFixAndSum(alpha_1, alpha_2) (sumcheck.rs:141-209), grid ceil(height / (256 * 32 * 4)): eval_0, 4 eval_1/2 of round 2
//   rounds   paddedHadamardFixAndSum for r = 3 .. log_m - 1 with alpha = challenges[r - 1] (sumcheck.rs:313-336 -> hadamard.rs:131-177),
//            grid ceil(output_height / 256): eval_0, 4 eval_1/2 of round r
//   pq       mle_fix_last_variable_koala_bear_ext_ext_zero_padding of p, then of q, with challenges[log_m - 1] (sumcheck.rs:338-352 ->
//            hadamard.rs:82-128): p_eval, q_eval
//   stacked  p right after the fold of round log_stacking_height (sumcheck.rs:326-328): dense_len >> log_stacking_height entries
const char* ref_jagged_sumcheck(const uint32_t* h_dense, uint64_t dense_len, const uint64_t* col_heights, uint32_t n_cols, const uint32_t* h_eq_row,
                                uint64_t eq_row_len, const uint32_t* h_eq_col, uint64_t eq_col_len, const uint32_t* challenges, uint32_t log_m,
                                uint32_t log_stacking_height, uint32_t* out_grid8, uint32_t* out_r2, uint32_t* out_rounds, uint32_t* out_pq,
                                uint32_t* out_stacked) {
    // the kernels' preconditions (sumcheck.rs:107, 150, 247-248; jagged_sumcheck.cu:32-34, 106-107).  The kernels read eqZRow[2 rowIdx + 1] and
    // eqZCol[colIdx] unchecked, and the stacked snapshot exists only when log_stacking_height < log_m and holds whole stacked columns.
    if (log_m < 3 || log_stacking_height < 3 || log_stacking_height >= log_m)
        return "ref_jagged_sumcheck: need 3 <= log_stacking_height < log_m";
    if (dense_len % 8 || dense_len > (1ull << log_m) || dense_len <= (1ull << (log_m - 1))) return "ref_jagged_sumcheck: dense_len";
    if (dense_len % (1ull << log_stacking_height)) return "ref_jagged_sumcheck: dense_len must be a multiple of 2^log_stacking_height";
    if (n_cols > eq_col_len) return "ref_jagged_sumcheck: more columns than eq_z_col entries";
    std::vector<uint32_t> col_index(dense_len / 2), start(n_cols + 1, 0);
    size_t cnt = 0;
    for (uint32_t c = 0; c < n_cols; c++) {
        const size_t half = col_heights[c] / 2;
        if (col_heights[c] % 16) return "ref_jagged_sumcheck: column heights must be multiples of 16";
        if (col_heights[c] > eq_row_len) return "ref_jagged_sumcheck: a column is taller than eq_z_row";
        if (cnt + half > col_index.size()) return "ref_jagged_sumcheck: the columns overrun the dense data";
        std::fill(col_index.begin() + cnt, col_index.begin() + cnt + half, c);
        cnt += half;
        start[c + 1] = start[c] + (uint32_t)half;
    }
    if (cnt != col_index.size()) return "ref_jagged_sumcheck: the columns do not cover the dense data";
    DevScope mem;   // every device buffer below is freed on every return
    auto up = [&](const void* h, size_t bytes, void** d) -> cudaError_t {
        cudaError_t e = mem.alloc(d, bytes);
        if (e == cudaSuccess && bytes) e = cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice);
        return e;
    };
    auto ext = [&](uint32_t r) { Ext4Raw a; memcpy(&a, challenges + 4 * r, 16); return a; };
    const size_t E = sizeof(kb31_extension_t), BLOCK = 256, STRIDE = 32, smem = (BLOCK / STRIDE) * E, height = dense_len / 2;
    void *d_dense, *d_col, *d_start, *d_eq_row, *d_eq_col, *d_part, *d_sum, *d_p, *d_q;
    RCHK(up(h_dense, dense_len * 4, &d_dense));
    RCHK(up(col_index.data(), col_index.size() * 4, &d_col));
    RCHK(up(start.data(), start.size() * 4, &d_start));
    RCHK(up(h_eq_row, eq_row_len * E, &d_eq_row));
    RCHK(up(h_eq_col, eq_col_len * E, &d_eq_col));
    const size_t g1 = (height + BLOCK * STRIDE * 2 - 1) / (BLOCK * STRIDE * 2), g2 = (height + BLOCK * STRIDE * 4 - 1) / (BLOCK * STRIDE * 4);
    const size_t max_blocks = std::max(8 * g1, (height / 2 + BLOCK - 1) / BLOCK * 2);
    RCHK(mem.alloc(&d_part, max_blocks * E));
    RCHK(mem.alloc(&d_sum, 8 * E));
    RCHK(mem.alloc(&d_p, (height / 2 + 1) * E));
    RCHK(mem.alloc(&d_q, (height / 2 + 1) * E));
    JaggedMle<JaggedSumcheckData> mle;
    mle.colIndex = (uint32_t*)d_col;
    mle.startIndices = (uint32_t*)d_start;
    mle.denseData.base = (felt_t*)d_dense;
    mle.denseData.eqZCol = (ext_t*)d_eq_col;
    mle.denseData.eqZRow = (ext_t*)d_eq_row;
    mle.denseData.height = height;
    auto sum_rows = [&](uint32_t rows, size_t n_blocks, uint32_t* out) -> cudaError_t {
        ref_sum_rows_kernel<<<1, 32>>>((const kb31_extension_t*)d_part, rows, (uint32_t)n_blocks, (kb31_extension_t*)d_sum);
        cudaError_t e = cudaGetLastError();
        return e == cudaSuccess ? cudaMemcpy(out, d_sum, rows * E, cudaMemcpyDeviceToHost) : e;
    };
    {
        void* args[] = {&d_part, &mle};
        RCHK(cudaLaunchKernel(jagged_two_round_sum_as_poly(), dim3((unsigned)g1), dim3((unsigned)BLOCK), args, smem, 0));
        RCHK(sum_rows(8, g1, out_grid8));
    }
    {
        Ext4Raw a1 = ext(0), a2 = ext(1);
        void* args[] = {&d_part, &mle, &d_p, &d_q, &a1, &a2};
        RCHK(cudaLaunchKernel(jagged_two_round_fix_and_sum(), dim3((unsigned)g2), dim3((unsigned)BLOCK), args, smem, 0));
        RCHK(sum_rows(2, g2, out_r2));
    }
    size_t len = height / 2;
    for (uint32_t r = 3; r < log_m; r++) {
        // paddedHadamardFixAndSum stores output pairs (2i, 2i + 1) for i < ceil(out_len / 2): one entry of slack for an odd out_len
        const size_t out_len = (len + 1) / 2, g = (out_len + BLOCK - 1) / BLOCK, hsmem = (BLOCK / 32) * E;
        void *d_p2, *d_q2;
        RCHK(mem.alloc(&d_p2, (out_len + 1) * E));
        RCHK(mem.alloc(&d_q2, (out_len + 1) * E));
        Ext4Raw a = ext(r - 1);
        void* args[] = {&d_p, &d_q, &d_p2, &d_q2, &a, &d_part, &len};
        RCHK(cudaLaunchKernel(padded_hadamard_fix_and_sum(), dim3((unsigned)g), dim3((unsigned)BLOCK), args, hsmem, 0));
        RCHK(sum_rows(2, g, out_rounds + 8 * (r - 3)));
        if (r == log_stacking_height) RCHK(cudaMemcpy(out_stacked, d_p2, out_len * E, cudaMemcpyDeviceToHost));
        mem.release(d_p);
        mem.release(d_q);
        d_p = d_p2;
        d_q = d_q2;
        len = out_len;
    }
    {
        Ext4Raw a = ext(log_m - 1);
        size_t width = 1;
        const unsigned g = (unsigned)(((len + 1) / 2 + BLOCK - 1) / BLOCK);
        for (int k = 0; k < 2; k++) {
            void* in = k ? d_q : d_p;
            void* args[] = {&in, &d_sum, &a, &len, &width};
            RCHK(cudaLaunchKernel(mle_fix_last_variable_koala_bear_ext_ext_zero_padding(), dim3(g, 1), dim3((unsigned)BLOCK, 1), args, 0, 0));
            RCHK(cudaMemcpy(out_pq + 4 * k, d_sum, E, cudaMemcpyDeviceToHost));
        }
    }
    return nullptr;
}

// ---- jagged evaluation (branching-program) sumcheck: the reference's jagged_assist kernels ------------------------------------------
extern "C" void* branching_program_kernel();
extern "C" void* transition_kernel();
extern "C" void* interpolateAndObserve_kernel_duplex();
extern "C" void* fixLastVariable_kernel();

// the device constants JaggedAssistSumAsPolyGPUImpl::new and new_jagged_eval_sumcheck_poly_sync upload (sumcheck_sum_as_poly.rs:74-78,
// sync_eval_sumcheck.rs:121-124): lambdas = [0, EF::two().inverse()], intermediate_eq_full_evals = [1; n]
__global__ void ref_jagged_eval_init_kernel(kb31_extension_t* lambdas, kb31_extension_t* inter, uint32_t n) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        lambdas[0] = kb31_extension_t::zero();
        lambdas[1] = kb31_extension_t::two().reciprocal();
    }
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += blockDim.x * gridDim.x) inter[i] = kb31_extension_t::one();
}

// challenger.observe_ext_element(expected_sum) (sync_eval_sumcheck.rs:277), on the device challenger the Rust builds right after it
__global__ void ref_observe_ext_kernel(DuplexChallenger ch, kb31_extension_t* v) {
    if (blockIdx.x || threadIdx.x) return;
    ch.observe_ext(v);
}

// The 16 x 5 TRANSITIONS table of jagged_assist/branching_program.cuh as transition_kernel writes it (branching_program.rs:254-279: one
// thread): out[bit_state * 5 + input memory state] = output memory state, FAIL = 4.
const char* ref_bp_transitions(uint64_t* out80) {
    DevScope mem;
    void* d_out;
    RCHK(mem.alloc(&d_out, 80 * sizeof(size_t)));
    void* args[] = {&d_out};
    RCHK(cudaLaunchKernel(transition_kernel(), dim3(1), dim3(1), args, 0, 0));
    RCHK(cudaMemcpy(out80, d_out, 80 * sizeof(size_t), cudaMemcpyDeviceToHost));
    return nullptr;
}

// prove_jagged_eval_sumcheck_sync (jagged_assist/src/sync_eval_sumcheck.rs:141-239) with the device state that
// new_jagged_eval_sumcheck_poly_sync (:36-137) and JaggedAssistSumAsPolyGPUImpl::new (sumcheck_sum_as_poly.rs:34-90) build, each round
// one sum_as_poly_and_sample_into_point (sumcheck_sum_as_poly.rs:93-162 -> branching_program.rs:89-195) and one fix_last_variable_kernel
// (sumcheck_sum_as_poly.rs:164-201).  Inputs, as the Rust has them after condensing (sync_eval_sumcheck.rs:77-87):
//   merged   [nk][2 (log_m + 1)] field words: merged prefix sum k = (bits of t_k || bits of t_{k+1}), most significant bit first
//   zc       [nk] ext: the condensed z_col eq values;  z_row [z_row_len], z_index [z_index_len] ext (z_index = the Hadamard sumcheck point)
//   claim4   the claimed sum;  st34: the challenger before the claim is observed (prove_jagged_evaluation_sync, :277-280), updated in place
// Outputs: out_bp [2][nk] ext: one branchingProgram launch with round_num = -1 (no substitution: the program at the boolean prefix
// sums, both rows); out_sum_values [2 (log_m + 1)][3] ext: (y_0, y_1/2, y_1) per round as interpolateAndObserve stores them;
// out_point [2 (log_m + 1)] ext: the sampled point, most recent first (branching_program.rs:192 prepends every new sample).
const char* ref_jagged_eval(const uint32_t* merged, uint32_t nk, uint32_t log_m, const uint32_t* zc, const uint32_t* z_row, uint32_t z_row_len,
                            const uint32_t* z_index, uint32_t z_index_len, const uint32_t* claim4, uint32_t* st34, uint32_t* out_bp,
                            uint32_t* out_sum_values, uint32_t* out_point) {
    // round_num is an int8_t kernel argument (branching_program.cu:320), so the last round, 2 (log_m + 1) - 1, must fit in it
    if (nk == 0) return "ref_jagged_eval: need at least one merged prefix sum";
    if (2 * ((uint64_t)log_m + 1) > 127) return "ref_jagged_eval: 2 (log_m + 1) rounds do not fit the kernels' int8_t round_num";
    const size_t psl = log_m + 1, dim = 2 * psl, E = sizeof(kb31_extension_t);
    // JaggedAssistSumAsPolyGPUImpl::new: split each merged prefix sum into current | next and transpose each [nk, psl] tensor to [psl, nk]
    std::vector<uint32_t> cur_t(psl * nk), next_t(psl * nk);
    for (size_t k = 0; k < nk; k++)
        for (size_t i = 0; i < psl; i++) {
            cur_t[i * nk + k] = merged[k * dim + i];
            next_t[i * nk + k] = merged[k * dim + psl + i];
        }
    DevScope mem;
    void *d_cur, *d_next, *d_merged, *d_zc, *d_zrow, *d_zindex, *d_claim, *d_lambdas, *d_inter, *d_bp, *d_results, *d_sum_values, *d_rho, *d_new;
    RCHK(dev_upload(mem, cur_t.data(), cur_t.size() * 4, &d_cur));
    RCHK(dev_upload(mem, next_t.data(), next_t.size() * 4, &d_next));
    RCHK(dev_upload(mem, merged, (size_t)nk * dim * 4, &d_merged));
    RCHK(dev_upload(mem, zc, (size_t)nk * E, &d_zc));
    RCHK(dev_upload(mem, z_row, (size_t)z_row_len * E, &d_zrow));
    RCHK(dev_upload(mem, z_index, (size_t)z_index_len * E, &d_zindex));
    RCHK(dev_upload(mem, claim4, E, &d_claim));
    RCHK(mem.alloc(&d_lambdas, 2 * E));
    RCHK(mem.alloc(&d_inter, (size_t)nk * E));
    RCHK(mem.alloc(&d_bp, 2 * (size_t)nk * E));
    RCHK(mem.alloc(&d_results, 2 * E));
    RCHK(mem.alloc(&d_sum_values, 3 * dim * E));
    RCHK(cudaMemset(d_sum_values, 0, 3 * dim * E));   // Tensor::zeros_in([3, 2 (log_m + 1)]) (sync_eval_sumcheck.rs:275)
    RCHK(mem.alloc(&d_rho, dim * E));
    RCHK(mem.alloc(&d_new, dim * E));
    ref_jagged_eval_init_kernel<<<(nk + 255) / 256, 256>>>((kb31_extension_t*)d_lambdas, (kb31_extension_t*)d_inter, nk);
    RCHK(cudaGetLastError());
    const size_t BLOCK = 256;   // branching_program.rs:119-122: block 256, grid (ceil(nk / 256), 2)
    const dim3 bp_grid((unsigned)((nk + BLOCK - 1) / BLOCK), 2);
    size_t z_row_n = z_row_len, z_index_n = z_index_len, n_cols = nk, psl_arg = psl;
    auto launch_bp = [&](int8_t round_num, void* cur_rho, size_t cur_rho_len, void* next_rho, size_t next_rho_len) -> cudaError_t {
        void* args[] = {&d_cur, &d_next, &psl_arg, &d_zrow, &z_row_n, &d_zindex, &z_index_n, &cur_rho, &cur_rho_len, &next_rho,
                        &next_rho_len, &n_cols, &round_num, &d_lambdas, &d_zc, &d_inter, &d_bp};
        return cudaLaunchKernel(branching_program_kernel(), bp_grid, dim3((unsigned)BLOCK), args, 0, 0);
    };
    // round_num = -1: the per-column program values at the boolean prefix sums, which the claimed sum is made of
    RCHK(launch_bp(-1, d_rho, 0, d_rho, 0));
    RCHK(cudaMemcpy(out_bp, d_bp, 2 * (size_t)nk * E, cudaMemcpyDeviceToHost));
    DevChallenger ch;
    if (const char* e = ch.init(st34)) return e;
    {
        void* args[] = {&ch.raw, &d_claim};
        RCHK(cudaLaunchKernel((void*)ref_observe_ext_kernel, dim3(1), dim3(1), args, 0, 0));
    }
    Ext4Raw claim;
    memcpy(&claim, claim4, 16);
    for (size_t r = 0; r < dim; r++) {
        // sumcheck_sum_as_poly.rs:106-135: rounds < psl bind next-prefix-sum bits (current rho empty, next rho = the whole point);
        // later rounds split the point after its first r - psl entries
        void *cur_rho = d_rho, *next_rho = d_rho;
        size_t cur_len = 0, next_len = r;
        if (r >= psl) {
            cur_len = r - psl;
            next_rho = (char*)d_rho + cur_len * E;
            next_len = r - cur_len;
        }
        int8_t round_num = (int8_t)r;
        RCHK(launch_bp(round_num, cur_rho, cur_len, next_rho, next_len));
        ref_sum_rows_kernel<<<1, 32>>>((const kb31_extension_t*)d_bp, 2, nk, (kb31_extension_t*)d_results);   // sum_dim(1)
        RCHK(cudaGetLastError());
        {
            void* args[] = {&d_results, &ch.raw, &d_new, &round_num, &d_sum_values, &claim};
            RCHK(cudaLaunchKernel(interpolateAndObserve_kernel_duplex(), dim3(1), dim3((unsigned)BLOCK), args, 0, 0));
        }
        // the new point = [alpha] ++ the old point (branching_program.rs:163-192)
        if (r) RCHK(cudaMemcpy((char*)d_new + E, d_rho, r * E, cudaMemcpyDeviceToDevice));
        std::swap(d_rho, d_new);
        // the next round's claim: bp_results[0], read back to the host (sumcheck_sum_as_poly.rs:156-161)
        RCHK(cudaMemcpy(&claim, d_results, E, cudaMemcpyDeviceToHost));
        {
            // fix_last_variable_kernel: block 512, grid ceil(merged_prefix_sums.len() / 512) over the flat nk x dim words
            size_t mdim = dim, rn = r, rho_len = r + 1;
            void* args[] = {&d_merged, &d_inter, &d_rho, &mdim, &n_cols, &rn, &rho_len};
            RCHK(cudaLaunchKernel(fixLastVariable_kernel(), dim3((unsigned)((nk * dim + 511) / 512)), dim3(512), args, 0, 0));
        }
    }
    RCHK(cudaDeviceSynchronize());
    RCHK(cudaMemcpy(out_sum_values, d_sum_values, 3 * dim * E, cudaMemcpyDeviceToHost));
    RCHK(cudaMemcpy(out_point, d_rho, dim * E, cudaMemcpyDeviceToHost));
    return ch.read(st34);
}

// ---- LogUp-GKR: the reference's circuit and round kernels -----------------------------------------------------------------------------
extern "C" void* logup_gkr_first_sum_as_poly_circuit_layer();
extern "C" void* logup_gkr_fix_and_sum_circuit_layer();
extern "C" void* logup_gkr_fix_and_sum_last_circuit_layer();
extern "C" void* logup_gkr_fix_and_sum_interactions_layer();
extern "C" void* logup_gkr_fix_and_sum_first_layer();
extern "C" void* jagged_fold_metadata_kernel();
extern "C" uint32_t jagged_fold_metadata_block_dim();
extern "C" uint32_t jagged_fold_metadata_section_size();
extern "C" void* mle_fix_last_variable_koala_bear_ext_ext_constant_padding();

#define CECHK(expr)                          \
    do {                                     \
        cudaError_t e_ = (expr);             \
        if (e_ != cudaSuccess) return e_;    \
    } while (0)

// fold_jagged_metadata_dev (sp1-gpu/crates/utils/src/jagged.rs:207-279, zerocheck/src/primitives.rs:53-112): from the n_cols column
// heights d_h (row pairs), the folded heights h.div_ceil(4) * 2 and their exclusive prefix sums (n_cols + 1 entries, the last = *total)
static cudaError_t fold_metadata(DevScope& mem, const uint32_t* d_h, uint32_t n_cols, uint32_t** new_h, uint32_t** new_start, uint32_t* total) {
    const uint32_t sec = jagged_fold_metadata_section_size(), bd = jagged_fold_metadata_block_dim();
    const uint32_t nb = std::max<uint32_t>((n_cols + sec - 1) / sec, 1);
    void *bc, *fl, *sv;
    CECHK(mem.alloc((void**)new_h, n_cols * 4));
    CECHK(mem.alloc((void**)new_start, (n_cols + 1) * 4));
    CECHK(mem.alloc(&bc, 4));
    CECHK(mem.alloc(&fl, (nb + 1) * 4));
    CECHK(mem.alloc(&sv, (nb + 1) * 4));
    CECHK(cudaMemset(bc, 0, 4));
    CECHK(cudaMemset(fl, 0, (nb + 1) * 4));
    CECHK(cudaMemset(fl, 1, 4));   // flags[0] != 0: the first block does not wait
    CECHK(cudaMemset(sv, 0, (nb + 1) * 4));
    uint32_t n = n_cols;
    void* args[] = {&d_h, &n, new_h, new_start, &bc, &fl, &sv};
    CECHK(cudaLaunchKernel(jagged_fold_metadata_kernel(), dim3(nb), dim3(bd), args, 0, 0));
    return cudaMemcpy(total, *new_start + n_cols, 4, cudaMemcpyDeviceToHost);
}

// one circuit layer on the device: the JaggedMle kernel argument and its column heights (row-pair counts), from which the reference's
// fold-metadata kernel derives the next layer's
struct GkrCircuitDev {
    JaggedMle<JaggedGkrLayer> mle;
    uint32_t* heights;
};

// prove_logup_gkr's device work (sp1-gpu/crates/logup_gkr/src/lib.rs:177-253) with the challenges supplied instead of sampled, for chips
// taken in the order given (the proof's chip order, which is the reference's chip-name order).
//   chips      chip c: height chip_heights[c], chip_n_inter[c] interactions whose InteractionsCsr arrays lie back to back after chip c - 1's;
//              its main (prep) columns start at h_main + main_off[c] (h_prep + prep_off[c]), column-major
//   lambdas    per GKR layer in proof order (the top layer, one row variable, first; the leaf last): lambda
//   points     per layer p: its evaluation point, v + p + 1 coordinates (interaction variables first), v = log2 of the padded interaction count
//   challenges per layer p: its v + p + 1 sumcheck challenges in round order
// Raw outputs, ext (4 words) each, in this order:
//   the output numerators, then the output denominators: 2^(v+1) each (extractOutput, tracegen.rs:191-248 -> execution.rs:139-169)
//   per layer p in proof order, n = v + p + 1 rounds:
//     lookahead layer (p + 1 > 2 row variables, sumcheck.rs:941 / 1043): the 10-value grid of two_round_sum_* (sumcheck.rs:109-142),
//       then (eval_0, eval_1/2 unscaled, eq_sum) of rounds 2 .. n - 1
//     otherwise: (eval_0, eval_1/2 unscaled, eq_sum) of rounds 0 .. n - 1
//     then n_0, n_1, d_0, d_1 of fixLastVariableInteractionsLayer (sumcheck.rs:467-517, 48-56)
const char* ref_logup_gkr(uint32_t n_chips, const uint64_t* chip_heights, const uint32_t* chip_n_inter, const uint32_t* h_main, const uint64_t* main_off,
                          uint64_t main_words, const uint32_t* h_prep, const uint64_t* prep_off, uint64_t prep_words, const uint64_t* values_ptr,
                          const uint64_t* mult_ptr, const uint64_t* vcw_ptr, const uint64_t* vcw_col, const uint8_t* vcw_is_prep, const uint32_t* vcw_weight,
                          const uint32_t* values_constants, const uint64_t* mcw_col, const uint8_t* mcw_is_prep, const uint32_t* mcw_weight,
                          const uint32_t* mult_constants, const uint32_t* arg_indices, const uint8_t* is_send, const uint32_t* alpha4,
                          const uint32_t* betas, uint32_t n_betas, uint32_t mlr, const uint32_t* lambdas, const uint32_t* points,
                          const uint32_t* challenges, uint64_t point_words, uint32_t* out, uint64_t out_cap) {
    // ---- host-side rejection of every input that would make an unchecked reference kernel fault or read unwritten memory
    if (mlr < 3) return "ref_logup_gkr: max_log_row_count < 3 (tracegen.rs:229 underflows)";
    uint64_t n_int = 0;
    for (uint32_t c = 0; c < n_chips; c++) n_int += chip_n_inter[c];
    if (n_int < 2) return "ref_logup_gkr: fewer than two interactions (v = 0: sumcheck.rs:534 launches the 4-parameter fixLastVariableLastCircuitLayer with 2 arguments)";
    uint32_t v = 0;
    while ((1ull << v) < n_int) v++;
    const bool leaf_lookahead = mlr - 1 > 2;
    std::vector<uint32_t> counts;   // interaction_row_counts (tracegen.rs:43-59): max(h, 8).div_ceil(4) row pairs per interaction
    for (uint32_t c = 0; c < n_chips; c++) {
        const uint64_t h = chip_heights[c];
        if (h & 1) return "ref_logup_gkr: odd chip height (tracegen.rs:98 asserts)";
        if (h > (1ull << mlr)) return "ref_logup_gkr: a chip taller than 2^max_log_row_count";
        if (h && (h < 8 || h % 4)) return "ref_logup_gkr: a non-empty chip shorter than 8 rows or not a multiple of 4 (populateLastCircuitLayer leaves row pairs unwritten)";
        const uint32_t cnt = (uint32_t)((std::max<uint64_t>(h, 8) + 3) / 4);
        if (leaf_lookahead && (cnt & 1)) return "ref_logup_gkr: odd leaf pair height on a lookahead leaf (fixLastTwoVariablesTwoPadding traps, jagged.cuh:113-117)";
        counts.insert(counts.end(), chip_n_inter[c], cnt);
    }
    const uint64_t n_out = 2ull << v;
    uint64_t need = 8 * n_out;
    for (uint32_t p = 0; p + 1 < mlr; p++) {
        const uint64_t n = v + p + 1;
        need += 4 * ((p + 1 > 2 ? 10 + 3 * (n - 2) : 3 * n) + 4);
    }
    if (out_cap < need) return "ref_logup_gkr: output buffer too small";
    uint64_t layer_words = 0;
    for (uint32_t p = 0; p + 1 < mlr; p++) layer_words += 4ull * (v + p + 1);
    if (point_words != layer_words) return "ref_logup_gkr: the points / challenges do not have v + p + 1 coordinates per layer p";
    {
        InteractionsCsr c{values_ptr, mult_ptr, vcw_ptr, vcw_col, mcw_col, vcw_is_prep, mcw_is_prep, is_send, vcw_weight, values_constants,
                          mcw_weight, mult_constants, arg_indices, 0, 0, 0, 0};
        for (uint32_t k = 0; k < n_chips; k++) {
            if (main_off[k] > main_words || prep_off[k] > prep_words) return "ref_logup_gkr: a chip's trace starts past the trace words";
            csr_enter(c, chip_n_inter[k]);
            if (const char* e = check_interaction_reads(c, chip_heights[k], main_words - main_off[k], prep_words - prep_off[k], n_betas)) return e;
            csr_leave(c);
        }
    }

    DevScope mem;   // every device buffer below is freed on every return
    const size_t E = sizeof(kb31_extension_t), BLOCK = 256, smem = (BLOCK / 32) * E;
    const uint32_t n_cols = (uint32_t)n_int;
    auto ext = [](const uint32_t* w) { Ext4Raw a; memcpy(&a, w, 16); return a; };
    void* d_sum;
    RCHK(mem.alloc(&d_sum, 10 * E));
    // DeviceTensor::sum_dim(1) of a [rows, n_blocks] tensor of per-block partials, appended to the raw outputs
    uint32_t* o = out;
    auto sum_rows = [&](void* part, uint32_t rows, size_t n_blocks) -> cudaError_t {
        ref_sum_rows_kernel<<<1, 32>>>((const kb31_extension_t*)part, rows, (uint32_t)n_blocks, (kb31_extension_t*)d_sum);
        CECHK(cudaGetLastError());
        CECHK(cudaMemcpy(o, d_sum, rows * E, cudaMemcpyDeviceToHost));
        o += 4 * rows;
        return cudaSuccess;
    };
    // launch a summing kernel whose first argument is its [rows, grid] partials, then sum them
    auto run_sum = [&](void* kernel, size_t grid, uint32_t rows, void** part, void** args) -> cudaError_t {
        CECHK(mem.alloc(part, rows * grid * E));
        CECHK(cudaLaunchKernel(kernel, dim3((unsigned)grid), dim3((unsigned)BLOCK), args, smem, 0));
        return sum_rows(*part, rows, grid);
    };
    auto fold = [&](const uint32_t* d_h, uint32_t** new_h, uint32_t** new_start, uint32_t* total) {
        return fold_metadata(mem, d_h, n_cols, new_h, new_start, total);
    };
    // the next circuit layer's buffers, its metadata advanced `folds` folds from the column heights d_h; Tensor [4, 1, 2 * height] and a
    // colIndex of `height` entries, zeroed (the reference leaves them uninitialised; every entry read is written by the kernels)
    auto new_circuit = [&](const uint32_t* d_h, int folds, GkrCircuitDev* next) -> cudaError_t {
        uint32_t *h1, *s1, total;
        CECHK(fold(d_h, &h1, &s1, &total));
        if (folds == 2) CECHK(fold(h1, &h1, &s1, &total));
        void *layer, *col;
        CECHK(mem.alloc(&layer, 8 * (size_t)total * E));
        CECHK(mem.alloc(&col, (size_t)total * 4));
        CECHK(cudaMemset(layer, 0, 8 * (size_t)total * E));
        CECHK(cudaMemset(col, 0, (size_t)total * 4));
        next->mle.colIndex = (uint32_t*)col;
        next->mle.startIndices = s1;
        next->mle.denseData.layer = (ext_t*)layer;
        next->mle.denseData.height = total;
        next->heights = h1;
        return cudaSuccess;
    };
    // DevicePoint::partial_lagrange (sp1-gpu/crates/cuda/src/mle/eval.rs:66-90): block 256, grid ceil(2^dim / 256)
    auto eq_table = [&](const uint32_t* h_point, uint32_t dim, void** d_out) -> cudaError_t {
        void* d_pt;
        CECHK(dev_upload(mem, h_point, (size_t)dim * E, &d_pt));
        CECHK(mem.alloc(d_out, (E << dim)));
        size_t nv = dim;
        void* args[] = {d_out, &d_pt, &nv};
        return cudaLaunchKernel(partial_lagrange_koala_bear_extension(), dim3((unsigned)(((1ull << dim) + 255) / 256)), dim3(256), args, 0, 0);
    };
    // DeviceMle::fix_last_variable_constant_padding(alpha, zero) (sp1-gpu/crates/cuda/src/mle/restrict.rs:77-110): block 256,
    // grid (ceil(out / (256 * 128)), 1)
    auto eq_fix = [&](void** d_eq, size_t* len, Ext4Raw a) -> cudaError_t {
        const size_t out_len = (*len + 1) / 2;
        void* d_out;
        CECHK(mem.alloc(&d_out, out_len * E));
        Ext4Raw zero{};
        size_t in_len = *len, width = 1;
        void* args[] = {d_eq, &d_out, &zero, &a, &in_len, &width};
        CECHK(cudaLaunchKernel(mle_fix_last_variable_koala_bear_ext_ext_constant_padding(), dim3((unsigned)((out_len + BLOCK * 128 - 1) / (BLOCK * 128)), 1),
                               dim3((unsigned)BLOCK), args, 0, 0));
        *d_eq = d_out;
        *len = out_len;
        return cudaSuccess;
    };

    // ---- first layer (generate_first_layer, tracegen.rs:36-166)
    std::vector<uint32_t> start(n_cols + 1, 0);
    for (uint32_t j = 0; j < n_cols; j++) start[j + 1] = start[j] + counts[j];
    const size_t H0 = start[n_cols];
    void *d_main, *d_prep, *d_betas, *d_start, *d_counts, *d_col, *d_num, *d_den;
    RCHK(dev_upload(mem, h_main, main_words * 4, &d_main));
    RCHK(dev_upload(mem, h_prep, prep_words * 4, &d_prep));
    RCHK(dev_upload(mem, betas, (size_t)n_betas * E, &d_betas));
    RCHK(dev_upload(mem, start.data(), start.size() * 4, &d_start));
    RCHK(dev_upload(mem, counts.data(), counts.size() * 4, &d_counts));
    RCHK(mem.alloc(&d_col, H0 * 4));
    RCHK(mem.alloc(&d_num, 4 * H0 * 4));
    RCHK(mem.alloc(&d_den, 4 * H0 * E));
    RCHK(cudaMemset(d_col, 0, H0 * 4));
    RCHK(cudaMemset(d_num, 0, 4 * H0 * 4));
    RCHK(cudaMemset(d_den, 0, 4 * H0 * E));
    {
        const Ext4Raw alpha = ext(alpha4);
        InteractionsCsr c{values_ptr, mult_ptr, vcw_ptr, vcw_col, mcw_col, vcw_is_prep, mcw_is_prep, is_send, vcw_weight, values_constants,
                          mcw_weight, mult_constants, arg_indices, 0, 0, 0, 0};
        size_t offset = 0;
        for (uint32_t k = 0; k < n_chips; k++) {
            csr_enter(c, chip_n_inter[k]);
            if (c.n_inter) {   // a chip without interactions owns no column (a launch with grid.y = 0 would be an error)
                Interactions<felt_t> I{};
                RCHK(upload_interactions(mem, c, &I));
                RCHK(launch_populate(I, (const uint32_t*)d_start, (uint32_t*)d_col, (felt_t*)d_num, (ext_t*)d_den, (felt_t*)d_prep + prep_off[k],
                                     (felt_t*)d_main + main_off[k], alpha, (ext_t*)d_betas, offset, chip_heights[k], H0));
            }
            offset += c.n_inter;
            csr_leave(c);
        }
    }
    JaggedMle<JaggedFirstGkrLayer> leaf;
    leaf.colIndex = (uint32_t*)d_col;
    leaf.startIndices = (uint32_t*)d_start;
    leaf.denseData.numeratorValues = (felt_t*)d_num;
    leaf.denseData.denominatorValues = (ext_t*)d_den;
    leaf.denseData.height = H0;

    // ---- forward circuit (generate_gkr_circuit, tracegen.rs:211-244; execution.rs:26-115): block 256, grid ceil(height / (256 * 32))
    std::vector<GkrCircuitDev> circ(mlr - 1);   // circ[k]: mlr - 1 - k row variables, k >= 1
    RCHK(new_circuit((const uint32_t*)d_counts, 1, &circ[1]));
    {
        void* args[] = {&leaf, &circ[1].mle};
        RCHK(cudaLaunchKernel(logup_gkr_first_layer_transition(), dim3((unsigned)((H0 + 8191) / 8192)), dim3(256), args, 0, 0));
    }
    for (uint32_t k = 2; k + 1 < mlr; k++) {
        RCHK(new_circuit(circ[k - 1].heights, 1, &circ[k]));
        void* args[] = {&circ[k - 1].mle, &circ[k].mle};
        RCHK(cudaLaunchKernel(logup_gkr_circuit_transition(), dim3((unsigned)((circ[k - 1].mle.denseData.height + 8191) / 8192)), dim3(256), args, 0, 0));
    }
    {   // extract_outputs (execution.rs:139-169): block 256, grid ceil(2^v / (256 * 4))
        void *d_on, *d_od;
        RCHK(mem.alloc(&d_on, n_out * E));
        RCHK(mem.alloc(&d_od, n_out * E));
        size_t grid_height = n_out / 2;
        void* args[] = {&circ[mlr - 2].mle, &d_on, &d_od, &grid_height};
        RCHK(cudaLaunchKernel(logup_gkr_extract_output(), dim3((unsigned)((grid_height + 1023) / 1024)), dim3(256), args, 0, 0));
        RCHK(cudaMemcpy(o, d_on, n_out * E, cudaMemcpyDeviceToHost));
        RCHK(cudaMemcpy(o + 4 * n_out, d_od, n_out * E, cudaMemcpyDeviceToHost));
        o += 8 * n_out;
    }

    // ---- per GKR layer, top down (prove_gkr_circuit, lib.rs:133-174 -> prove_round)
    for (uint32_t p = 0; p + 1 < mlr; p++) {
        const uint32_t k = mlr - 2 - p, R = p + 1, n = v + R;
        Ext4Raw lambda = ext(lambdas + 4 * p);
        auto ch = [&](uint32_t r) { return ext(challenges + 4 * r); };
        void *eq_int, *eq_row, *part;
        size_t eq_int_len = (size_t)1 << v, eq_row_len = (size_t)1 << R;
        RCHK(eq_table(points, v, &eq_int));              // prove_first_round / prove_materialized_round (lib.rs:53-61, 89-97)
        RCHK(eq_table(points + 4 * v, R, &eq_row));
        GkrCircuitDev cur{}, next{};
        uint32_t cur_r = R, r0;
        void* guts = nullptr;   // the interactions layer, Tensor [4, ih]
        size_t ih = 0;
        if (R > 2) {   // two-round lookahead: sumcheck.rs:943-973 (leaf), 1050-1082 (circuit layer)
            size_t H = k ? circ[k].mle.denseData.height : H0;
            void* lm = k ? (void*)&circ[k].mle : (void*)&leaf;
            {
                void* args[] = {&part, lm, &eq_row, &eq_int, &lambda};
                RCHK(run_sum(k ? logup_gkr_two_round_sum_circuit_layer() : logup_gkr_two_round_sum_first_layer(), (H + BLOCK * 64 - 1) / (BLOCK * 64), 10,
                             &part, args));
            }
            RCHK(eq_fix(&eq_row, &eq_row_len, ch(0)));   // sumcheck.rs:312-313, 362-363
            RCHK(eq_fix(&eq_row, &eq_row_len, ch(1)));
            RCHK(new_circuit(k ? circ[k].heights : (const uint32_t*)d_counts, 2, &next));   // sumcheck.rs:221-282
            Ext4Raw a1 = ch(0), a2 = ch(1);
            void* args[] = {&part, lm, &next.mle, &a1, &a2, &eq_row, &eq_int, &lambda};
            RCHK(run_sum(k ? logup_gkr_two_round_fix_and_sum_circuit_layer() : logup_gkr_two_round_fix_and_sum_first_layer(), (H + BLOCK * 32 - 1) / (BLOCK * 32),
                         3, &part, args));
            cur = next;
            cur_r = R - 2;
            r0 = 3;
        } else if (k == 0) {   // leaf, one round at a time: sum_as_poly_first_layer (sumcheck.rs:396-465), fix_and_sum_first_layer (:563-650)
            {
                const size_t h = H0 >> 1;
                void* args[] = {&part, &leaf, &eq_row, &eq_int, &lambda};
                RCHK(run_sum(logup_gkr_sum_as_poly_first_layer(), ((h + BLOCK - 1) / BLOCK + 31) / 32, 3, &part, args));
            }
            Ext4Raw a = ch(0);
            RCHK(new_circuit((const uint32_t*)d_counts, 1, &next));
            RCHK(eq_fix(&eq_row, &eq_row_len, a));
            const size_t h = H0 >> 1;
            void* args[] = {&part, &leaf, &next.mle, &eq_row, &eq_int, &lambda, &a};
            RCHK(run_sum(logup_gkr_fix_and_sum_first_layer(), (h + BLOCK * 32 - 1) / (BLOCK * 32), 3, &part, args));
            cur = next;
            cur_r = R - 1;
            r0 = 2;
        } else {   // circuit layer, first round: sum_as_poly_materialized_round (sumcheck.rs:652-691)
            cur = circ[k];
            const size_t H = cur.mle.denseData.height;
            void* args[] = {&part, &cur.mle, &eq_row, &eq_int, &lambda};
            RCHK(run_sum(eq_row_len == 2 ? logup_gkr_first_sum_as_poly_circuit_layer() : logup_gkr_sum_as_poly_circuit_layer(),
                         ((H + BLOCK - 1) / BLOCK + 31) / 32, 3, &part, args));
            r0 = 1;
        }
        // remaining rounds: fix_and_sum_materialized_round (sumcheck.rs:694-896) with the previous round's challenge
        for (uint32_t r = r0; r < n; r++) {
            Ext4Raw a = ch(r - 1);
            if (guts) {   // interactions layer (:705-761): eq_interaction is folded first
                RCHK(eq_fix(&eq_int, &eq_int_len, a));
                size_t out_h = (ih + 1) / 2, in_h = ih;
                void* d_out;
                RCHK(mem.alloc(&d_out, 4 * out_h * E));
                void* args[] = {&part, &guts, &d_out, &a, &in_h, &out_h, &eq_int, &lambda};
                RCHK(run_sum(logup_gkr_fix_and_sum_interactions_layer(), ((ih + BLOCK - 1) / BLOCK + 31) / 32, 3, &part, args));
                guts = d_out;
                ih = out_h;
            } else if (cur_r == 1) {   // last row variable (:767-814): the layer becomes the interactions layer
                const size_t h = cur.mle.denseData.height >> 1;
                void* d_out;
                RCHK(mem.alloc(&d_out, 4 * h * E));
                RCHK(eq_fix(&eq_row, &eq_row_len, a));
                JaggedGkrLayer dense = cur.mle.denseData;
                void* args[] = {&part, &dense, &a, &d_out, &eq_int, &lambda};
                RCHK(run_sum(logup_gkr_fix_and_sum_last_circuit_layer(), ((h + BLOCK - 1) / BLOCK + 31) / 32, 3, &part, args));
                guts = d_out;
                ih = h;
            } else {   // circuit layer (:815-893)
                RCHK(eq_fix(&eq_row, &eq_row_len, a));
                RCHK(new_circuit(cur.heights, 1, &next));
                const size_t H = cur.mle.denseData.height;
                void* args[] = {&part, &cur.mle, &next.mle, &a, &eq_row, &eq_int, &lambda};
                RCHK(run_sum(logup_gkr_fix_and_sum_circuit_layer(), ((H + BLOCK - 1) / BLOCK + 31) / 32, 3, &part, args));
                cur = next;
                cur_r--;
            }
        }
        if (!guts) return "ref_logup_gkr: the rounds did not reach the interaction variables";
        {   // fix_last_variable_materialized_round on the interactions layer (:476-517): block 256, grid ceil(height / (256 * 32))
            Ext4Raw a = ch(n - 1);
            size_t out_h = (ih + 1) / 2, in_h = ih;
            if (out_h != 1) return "ref_logup_gkr: the interactions layer did not fold to one entry";
            void* d_out;
            RCHK(mem.alloc(&d_out, 4 * E));
            void* args[] = {&guts, &d_out, &a, &in_h, &out_h};
            RCHK(cudaLaunchKernel(logup_gkr_fix_last_variable_interactions_layer(), dim3((unsigned)((ih + BLOCK * 32 - 1) / (BLOCK * 32))), dim3((unsigned)BLOCK),
                                  args, 0, 0));
            RCHK(cudaMemcpy(o, d_out, 4 * E, cudaMemcpyDeviceToHost));
            o += 16;
        }
        points += 4 * n;
        challenges += 4 * n;
    }
    RCHK(cudaDeviceSynchronize());
    return nullptr;
}

}  // extern "C"

// ---- zerocheck: the reference's zerocheck prover kernels ------------------------------------------------------------------------------
// One chip's constraint program as the machine blob stores it (include/sp1b200.h): the chunk the reference's lowering would emit for it.
struct ZcBlobChip {
    uint32_t main_w, prep_w, n_constraints, ni, nl, nc, npub, na, max_reg;
    const uint32_t *instrs, *leaves, *consts, *publics, *assert_regs, *assert_alphas;
};

// Every read the interpreter (sequential.cu:50-108, pad_adj.cu) makes without a check: an opcode it knows (others __trap), a leaf, constant
// and public-value index inside its table, a leaf column inside the chip's trace, a register written before it is read (an unwritten one
// holds the previous row's value) and an alpha index below the chip's constraint count.  max_reg = the highest register used + 1, as
// sp1-gpu/crates/air/src/ir/bytecode.rs:208-209 computes it.
static const char* zc_check_program(ZcBlobChip& c, uint32_t n_pv) {
    std::vector<uint8_t> written(1024, 0);
    uint32_t top = 0;
    auto ok = [&](uint32_t r) { return r < 1024 && written[r]; };
    for (uint32_t i = 0; i < c.ni; i++) {
        const uint32_t op = c.instrs[2 * i] & 0xff, o = c.instrs[2 * i] >> 16, a = c.instrs[2 * i + 1] & 0xffff, b = c.instrs[2 * i + 1] >> 16;
        switch (op) {
        case BC_LOAD_LEAF: {
            if (a >= c.nl) return "ref_zerocheck: a leaf index past the chip's leaf table";
            const uint32_t src = c.leaves[2 * a] & 0xff, col = c.leaves[2 * a + 1];
            if (src == LEAF_SOURCE_MAIN_LOCAL ? col >= c.main_w : (src != LEAF_SOURCE_PREPROCESSED_LOCAL || col >= c.prep_w))
                return "ref_zerocheck: a leaf outside the chip's columns";
            break;
        }
        case BC_LOAD_CONST: if (a >= c.nc) return "ref_zerocheck: a constant index past the chip's constants"; break;
        case BC_LOAD_PUBLIC: if (a >= c.npub || c.publics[a] >= n_pv) return "ref_zerocheck: a public-value index out of range"; break;
        case BC_ADD_F: case BC_SUB_F: case BC_MUL_F: if (!ok(a) || !ok(b)) return "ref_zerocheck: a register read before it is written"; break;
        case BC_NEG_F: if (!ok(a)) return "ref_zerocheck: a register read before it is written"; break;
        default: return "ref_zerocheck: an unknown opcode (the interpreter traps)";
        }
        if (o >= 1024) return "ref_zerocheck: a program above 1024 registers (the largest MAX_REGS template)";
        written[o] = 1;
        top = std::max(top, o + 1);
    }
    for (uint32_t i = 0; i < c.na; i++) {
        if (!ok(c.assert_regs[i])) return "ref_zerocheck: an assert on a register that is never written";
        if (c.assert_alphas[i] >= c.n_constraints) return "ref_zerocheck: an assert's alpha index past the chip's constraint count";
    }
    c.max_reg = top;
    return nullptr;
}

// the MAX_REGS template that covers max_reg (prover.rs:828-852, 1180-1196, 1877-1893)
static void* zc_tier_kernel(uint32_t max_reg, void* (*const k[6])()) {
    return k[max_reg <= 32 ? 0 : max_reg <= 64 ? 1 : max_reg <= 128 ? 2 : max_reg <= 256 ? 3 : max_reg <= 512 ? 4 : 5]();
}

extern "C" {

// zerocheck() (sp1-gpu/crates/zerocheck/src/prover.rs:2412-2741) on the fused first-two-rounds path, with lambda and the round challenges
// supplied instead of sampled and the host-side tables computed by the caller.  One chunk per chip: the blob's program (no ColumnTile).
//   blob         the machine blob; chip k has heights[k] rows, main (prep) columns at h_main + main_off[k] (h_prep + prep_off[k]), column-major
//   prep_pad_rows  the rows of the one preprocessed padding column between the preprocessed and the main columns (zero data)
//   alpha_pows   powers_of_alpha: alpha^0 .. alpha^(max_constraints - 1) reversed;  gkr_pows: gamma^1 .. gamma^n_gkr;
//   lambda_pows  lambda^0 .. lambda^(n_chips - 1) reversed;  zeta: the mlr coordinates of the GKR point;  challenges: mlr, in round order
// The jagged trace is built as the reference's own zerocheck harness builds it (zerocheck/src/lib.rs:1240-1330): every chip's preprocessed
// columns, the padding column, every chip's main columns.  Raw outputs, ext (4 words) each:
//   the padded-row adjustment of every chip (zerocheck_pad_adj, prover.rs:1207-1259)
//   the 16 totals of evaluate_zerocheck_bivariate (prover.rs:1908-2160): 12 node totals, then the corners c = 2x + y
//   per later round r = 2 .. mlr - 1: the 3 totals of evaluate_zerocheck (prover.rs:1434-1772) at the nodes {0, 2, 4}
//   per column, in column order (padding column included): the folded value zerocheck() demultiplexes (prover.rs:2692-2702), 0 for an
//   empty column
// Chips of height 0 are supported: the dispatch builders skip them, the chip-layouts kernel gives them height 0 and the geq kernel sums
// over no rows.  Rejected before any launch: max_log_row_count < 2 (no fused path), a height that is not a multiple of 4 (odd heights break
// the row-pair loads; heights = 2 mod 4 trap in fixLastTwoVariablesTwoPadding, jagged.cuh:113-117), a height above 2^mlr, a chip with rows
// but no columns, and every program fault zc_check_program lists.
const char* ref_zerocheck(const uint32_t* blob, const uint64_t* heights, const uint32_t* h_main, const uint64_t* main_off, uint64_t main_words,
                          const uint32_t* h_prep, const uint64_t* prep_off, uint64_t prep_words, uint32_t prep_pad_rows, const uint32_t* pv,
                          uint32_t n_pv, const uint32_t* alpha_pows, uint32_t n_alpha, const uint32_t* gkr_pows, uint32_t n_gkr,
                          const uint32_t* lambda_pows, uint32_t mlr, const uint32_t* zeta, const uint32_t* challenges, uint32_t* out,
                          uint64_t out_cap) {
    // ---- host-side rejection of every input that would make an unchecked reference kernel fault or read unwritten memory
    if (mlr < 2 || mlr > 24) return "ref_zerocheck: need 2 <= max_log_row_count <= 24 (the fused first two rounds need two variables)";
    const uint32_t n = blob[0];
    if (n == 0) return "ref_zerocheck: no chips";
    std::vector<ZcBlobChip> chips(n);
    {
        const uint32_t* b = blob + 1;
        for (auto& c : chips) {
            c.main_w = b[0]; c.prep_w = b[1]; c.n_constraints = b[2];
            c.ni = b[4]; c.nl = b[5]; c.nc = b[6]; c.npub = b[7]; c.na = b[8];
            b += 9;
            c.instrs = b; b += 2 * c.ni;
            c.leaves = b; b += 2 * c.nl;
            c.consts = b; b += c.nc;
            c.publics = b; b += c.npub;
            c.assert_regs = b; b += c.na;
            c.assert_alphas = b; b += c.na;
        }
    }
    uint32_t max_nc = 0, max_cols = 0, total_prep_w = 0, total_main_w = 0;
    for (uint32_t k = 0; k < n; k++) {
        ZcBlobChip& c = chips[k];
        const uint64_t h = heights[k];
        if (h % 4) return "ref_zerocheck: a height that is not a multiple of 4 (fixLastTwoVariablesTwoPadding traps on odd pair heights)";
        if (h > (1ull << mlr)) return "ref_zerocheck: a chip taller than 2^max_log_row_count";
        if (h && c.main_w + c.prep_w == 0) return "ref_zerocheck: a chip with rows but no columns (the chip-layouts kernel gives it height 0)";
        if (main_off[k] + c.main_w * h > main_words || prep_off[k] + c.prep_w * h > prep_words) return "ref_zerocheck: a chip's trace runs past the trace words";
        if (const char* e = zc_check_program(c, n_pv)) return e;
        max_nc = std::max(max_nc, c.n_constraints);
        max_cols = std::max(max_cols, c.main_w + c.prep_w);
        total_prep_w += c.prep_w;
        total_main_w += c.main_w;
    }
    if (n_alpha < max_nc) return "ref_zerocheck: fewer alpha powers than the largest constraint count";
    if (n_gkr < max_cols) return "ref_zerocheck: fewer gkr powers than the widest chip's columns";
    if (prep_pad_rows == 0 || prep_pad_rows % 4 || prep_pad_rows > (1u << mlr))
        return "ref_zerocheck: the padding column needs a non-zero multiple of 4 rows, at most 2^max_log_row_count";
    const uint32_t n_cols = total_prep_w + 1 + total_main_w;
    if (out_cap < 4ull * (n + 16 + 3 * (mlr - 2) + n_cols)) return "ref_zerocheck: output buffer too small";

    // ---- the jagged trace (build_chip_column_layouts, prover.rs:1271-1294; the layout of zerocheck/src/lib.rs:1240-1330)
    std::vector<uint32_t> colh;                 // column heights in row pairs
    std::vector<ChipColumnLayoutEntry> entries(n);
    std::vector<uint32_t> dense;
    uint64_t total_pairs = 0;
    for (uint32_t k = 0; k < n; k++) total_pairs += (uint64_t)(chips[k].prep_w + chips[k].main_w) * heights[k] / 2;
    total_pairs += prep_pad_rows / 2;
    if (total_pairs >= (1ull << 31)) return "ref_zerocheck: the trace is too long for the kernels' 32-bit lengths";
    dense.reserve(2 * total_pairs);
    for (uint32_t k = 0, cp = 0; k < n; k++) {
        entries[k].prep_col_idx = cp;
        entries[k].prep_width = chips[k].prep_w;
        const uint64_t h = heights[k];
        for (uint32_t j = 0; j < chips[k].prep_w; j++) {
            colh.push_back((uint32_t)(h / 2));
            dense.insert(dense.end(), h_prep + prep_off[k] + j * h, h_prep + prep_off[k] + (j + 1) * h);
        }
        cp += chips[k].prep_w;
    }
    colh.push_back(prep_pad_rows / 2);
    dense.insert(dense.end(), prep_pad_rows, 0u);
    for (uint32_t k = 0, cm = total_prep_w + 1; k < n; k++) {
        entries[k].main_col_idx = cm;
        entries[k].main_width = chips[k].main_w;
        const uint64_t h = heights[k];
        for (uint32_t j = 0; j < chips[k].main_w; j++) {
            colh.push_back((uint32_t)(h / 2));
            dense.insert(dense.end(), h_main + main_off[k] + j * h, h_main + main_off[k] + (j + 1) * h);
        }
        cm += chips[k].main_w;
    }
    std::vector<uint32_t> start(n_cols + 1, 0), col_index(total_pairs);
    for (uint32_t c = 0; c < n_cols; c++) {
        std::fill(col_index.begin() + start[c], col_index.begin() + start[c] + colh[c], c);
        start[c + 1] = start[c] + colh[c];
    }
    const std::vector<uint32_t> input_colh = colh;
    // the layout tracker's chip height in elements (ShardLayoutTracker::chip_height_elements): the chip's main height, else its prep height
    auto chip_height = [&](uint32_t k) {
        return chips[k].main_w ? 2 * colh[entries[k].main_col_idx] : chips[k].prep_w ? 2 * colh[entries[k].prep_col_idx] : 0u;
    };
    auto fold_host = [&]() { for (auto& h : colh) h = (h + 3) / 4 * 2; };

    DevScope mem;   // every device buffer below is freed on every return
    const size_t E = sizeof(kb31_extension_t);
    auto ext = [](const uint32_t* w) { Ext4Raw a; memcpy(&a, w, 16); return a; };
    void *d_dense, *d_col, *d_start, *d_colh, *d_entries, *d_layouts, *d_pv, *d_alpha, *d_gkr, *d_lambda, *d_geq, *d_pad_adj, *d_gkr_info;
    RCHK(dev_upload(mem, dense.data(), dense.size() * 4, &d_dense));
    RCHK(dev_upload(mem, col_index.data(), col_index.size() * 4, &d_col));
    RCHK(dev_upload(mem, start.data(), start.size() * 4, &d_start));
    RCHK(dev_upload(mem, colh.data(), colh.size() * 4, &d_colh));
    RCHK(dev_upload(mem, entries.data(), entries.size() * sizeof(ChipColumnLayoutEntry), &d_entries));
    RCHK(mem.alloc(&d_layouts, n * sizeof(ChipLayout)));
    RCHK(dev_upload(mem, pv, (size_t)n_pv * 4, &d_pv));
    RCHK(dev_upload(mem, alpha_pows, (size_t)n_alpha * E, &d_alpha));
    RCHK(dev_upload(mem, gkr_pows, (size_t)n_gkr * E, &d_gkr));
    RCHK(dev_upload(mem, lambda_pows, (size_t)n * E, &d_lambda));
    // launch_chip_layouts_kernel (prover.rs:1299-1331): block 128
    auto chip_layouts = [&]() {
        void* args[] = {&d_start, &d_colh, &d_entries, (void*)&n, &d_layouts};
        return cudaLaunchKernel(jagged_chip_layouts_kernel(), dim3((n + 127) / 128), dim3(128), args, 0, 0);
    };
    RCHK(chip_layouts());

    // ---- the chunk statics and the sequential tiers (build_seq_tiers, prover.rs:1086-1152; WIDE_GKR_THRESHOLD = 256, :1077)
    std::vector<ChunkStatic> statics(n);
    for (uint32_t k = 0; k < n; k++) {
        const ZcBlobChip& c = chips[k];
        std::vector<uint16_t> regs16(c.assert_regs, c.assert_regs + c.na);
        ChunkStatic& s = statics[k];
        RCHK(dev_upload(mem, c.instrs, (size_t)c.ni * 8, (void**)&s.instrs));
        RCHK(dev_upload(mem, c.leaves, (size_t)c.nl * 8, (void**)&s.leaves));
        RCHK(dev_upload(mem, c.consts, (size_t)c.nc * 4, (void**)&s.consts));
        RCHK(dev_upload(mem, c.publics, (size_t)c.npub * 4, (void**)&s.publics));
        RCHK(dev_upload(mem, regs16.data(), (size_t)c.na * 2, (void**)&s.assert_regs));
        RCHK(dev_upload(mem, c.assert_alphas, (size_t)c.na * 4, (void**)&s.assert_alphas));
        s.n_instrs = c.ni;
        s.n_asserts = c.na;
        s.chip_idx = k;
        const bool decoupled = c.main_w + c.prep_w > 256;
        s.gkr_main_width = decoupled ? 0 : c.main_w;    // the carrier chunk's inline GKR widths
        s.gkr_prep_width = decoupled ? 0 : c.prep_w;
        s.chip_alpha_offset = std::max(max_nc, 1u) - c.n_constraints;
    }
    uint32_t n_high = 0;
    for (auto& c : chips) n_high += c.max_reg > 256;
    const bool split = n_high > 0 && n_high * 10 <= n;
    struct Tier { std::vector<ChunkStatic> st; std::vector<uint32_t> chip; uint32_t max_reg = 0; void* d_st = nullptr; };
    Tier tiers[2];
    for (uint32_t k = 0; k < n; k++) {
        Tier& t = tiers[split && chips[k].max_reg > 256 ? 1 : 0];
        t.st.push_back(statics[k]);
        t.chip.push_back(k);
        t.max_reg = std::max(t.max_reg, chips[k].max_reg);
    }
    for (auto& t : tiers)
        if (!t.st.empty()) RCHK(dev_upload(mem, t.st.data(), t.st.size() * sizeof(ChunkStatic), &t.d_st));
    auto block_size = [](const Tier& t) { return t.max_reg > 128 ? 64u : 256u; };   // prover.rs:1451-1472

    // ---- padded-row adjustment (compute_padded_row_adjustment, prover.rs:1207-1259): block 64, one chunk per thread
    std::vector<uint32_t> pad_adj(4 * n, 0);
    {
        static void* (*const K[6])() = {zerocheck_pad_adj_32_kernel, zerocheck_pad_adj_64_kernel, zerocheck_pad_adj_128_kernel,
                                        zerocheck_pad_adj_256_kernel, zerocheck_pad_adj_512_kernel, zerocheck_pad_adj_1024_kernel};
        for (auto& t : tiers) {
            if (t.st.empty()) continue;
            uint32_t nch = (uint32_t)t.st.size();
            void* d_o;
            RCHK(mem.alloc(&d_o, nch * E));
            void* args[] = {&t.d_st, &nch, &d_pv, &d_alpha, &d_o};
            RCHK(cudaLaunchKernel(zc_tier_kernel(t.max_reg, K), dim3((nch + 63) / 64), dim3(64), args, 0, 0));
            std::vector<uint32_t> o(4 * nch);
            RCHK(cudaMemcpy(o.data(), d_o, nch * E, cudaMemcpyDeviceToHost));
            for (uint32_t i = 0; i < nch; i++) memcpy(&pad_adj[4 * t.chip[i]], &o[4 * i], 16);
        }
    }
    memcpy(out, pad_adj.data(), pad_adj.size() * 4);
    uint32_t* o = out + 4 * n;
    RCHK(dev_upload(mem, pad_adj.data(), pad_adj.size() * 4, &d_pad_adj));
    // the geq chips: a Sequential carrier and a non-zero padded-row adjustment (prover.rs:989-1005)
    std::vector<uint32_t> geq_chips;
    for (uint32_t k = 0; k < n; k++)
        if (pad_adj[4 * k] | pad_adj[4 * k + 1] | pad_adj[4 * k + 2] | pad_adj[4 * k + 3]) geq_chips.push_back(k);
    uint32_t n_geq = (uint32_t)geq_chips.size();
    void* d_geq_chips;
    RCHK(dev_upload(mem, geq_chips.data(), geq_chips.size() * 4, &d_geq_chips));
    {   // VirtualGeq::new(height, 1, 0, num_vars) per chip (prover.rs:958-969)
        std::vector<VirtualGeqState> g(n);
        const uint32_t one[4] = {0x01fffffeu, 0, 0, 0};   // 1 in Montgomery form
        for (uint32_t k = 0; k < n; k++) {
            g[k].threshold = (uint32_t)heights[k];
            g[k].num_vars = mlr;
            memcpy(&g[k].geq_coefficient, one, 16);
            memset(&g[k].eq_coefficient, 0, 16);
        }
        RCHK(dev_upload(mem, g.data(), g.size() * sizeof(VirtualGeqState), &d_geq));
    }
    std::vector<ChipGkrInfo> gkr_info(n);
    std::vector<uint32_t> gkr_active;   // the decoupled-GKR chips (prover.rs:942-951): wider than 256 columns
    for (uint32_t k = 0; k < n; k++) {
        gkr_info[k] = {chips[k].main_w, chips[k].prep_w};
        if (chips[k].main_w + chips[k].prep_w > 256) gkr_active.push_back(k);
    }
    RCHK(dev_upload(mem, gkr_info.data(), gkr_info.size() * sizeof(ChipGkrInfo), &d_gkr_info));
    // zerocheck_fix_geq_state (prover.rs:2229-2246, 2334-2353): block 128, one thread per chip
    auto fix_geq = [&](const uint32_t* a4) {
        Ext4Raw a = ext(a4);
        void* args[] = {&d_geq, (void*)&n, &a};
        return cudaLaunchKernel(zerocheck_fix_geq_state_kernel(), dim3((n + 127) / 128), dim3(128), args, 0, 0);
    };
    // DevicePoint::partial_lagrange of zeta's first dim coordinates: block 256
    auto eq_table = [&](uint32_t dim, void** d_out) -> cudaError_t {
        void* d_pt;
        CECHK(dev_upload(mem, zeta, (size_t)dim * E, &d_pt));
        CECHK(mem.alloc(d_out, E << dim));
        size_t nv = dim;
        void* args[] = {d_out, &d_pt, &nv};
        return cudaLaunchKernel(partial_lagrange_koala_bear_extension(), dim3((unsigned)(((1ull << dim) + 255) / 256)), dim3(256), args, 0, 0);
    };
    // row tiles of `rows` rows (pairs or quadruples): one BlockDispatch per tile (prover.rs:1518-1537, 1942-1962)
    auto tiles = [](std::vector<BlockDispatch>& d, uint32_t id, uint32_t rows, uint32_t tile) {
        for (uint32_t r = 0; r < rows; r += tile) d.push_back(BlockDispatch{id, r, std::min(rows - r, tile)});
    };
    const unsigned SMEM = 8 * E;   // (256 / 32) ext_t for every 256-thread reduction

    // ---- rounds 0 and 1: evaluate_zerocheck_bivariate (prover.rs:1908-2160)
    {
        const uint32_t dim = mlr - 2;
        void *d_eq, *d_nodes, *d_corners, *d_tot;
        RCHK(eq_table(dim, &d_eq));
        std::vector<BlockDispatch> disp[2], corner;
        for (int t = 0; t < 2; t++)
            for (uint32_t i = 0; i < tiers[t].chip.size(); i++) tiles(disp[t], i, (chip_height(tiers[t].chip[i]) + 3) / 4, block_size(tiers[t]));
        for (uint32_t k = 0; k < n; k++)
            if (chips[k].main_w + chips[k].prep_w) tiles(corner, k, (chip_height(k) + 3) / 4, 256);
        const size_t node_slots = (disp[0].size() + disp[1].size() + n_geq) * 12, corner_slots = corner.size() * 4;
        RCHK(mem.alloc(&d_nodes, std::max<size_t>(node_slots, 1) * E));
        RCHK(mem.alloc(&d_corners, std::max<size_t>(corner_slots, 1) * E));
        RCHK(mem.alloc(&d_tot, 16 * E));
        static void* (*const K[6])() = {zerocheck_fused_sequential_bivariate_kb_32_kernel, zerocheck_fused_sequential_bivariate_kb_64_kernel,
                                        zerocheck_fused_sequential_bivariate_kb_128_kernel, zerocheck_fused_sequential_bivariate_kb_256_kernel,
                                        zerocheck_fused_sequential_bivariate_kb_512_kernel, zerocheck_fused_sequential_bivariate_kb_1024_kernel};
        size_t slot = 0;
        for (int t = 0; t < 2; t++) {
            if (disp[t].empty()) continue;
            void *d_disp, *part = (char*)d_nodes + slot * E;
            RCHK(dev_upload(mem, disp[t].data(), disp[t].size() * sizeof(BlockDispatch), &d_disp));
            const unsigned bs = block_size(tiers[t]);
            void* args[] = {&d_disp, &tiers[t].d_st, &d_layouts, &d_dense, &d_pv, &d_alpha, &d_eq, &d_lambda, (void*)&dim, &part};
            RCHK(cudaLaunchKernel(zc_tier_kernel(tiers[t].max_reg, K), dim3((unsigned)disp[t].size()), dim3(bs), args, (bs / 32) * E, 0));
            slot += disp[t].size() * 12;
        }
        if (n_geq) {
            void* part = (char*)d_nodes + slot * E;
            void* args[] = {&d_geq_chips, &n_geq, &d_geq, &d_pad_adj, &d_lambda, &d_layouts, &d_eq, (void*)&dim, &part};
            RCHK(cudaLaunchKernel(zerocheck_geq_corrections_bivariate_kernel(), dim3(n_geq), dim3(256), args, SMEM, 0));
        }
        if (!corner.empty()) {
            void* d_disp;
            RCHK(dev_upload(mem, corner.data(), corner.size() * sizeof(BlockDispatch), &d_disp));
            void* args[] = {&d_disp, &d_layouts, &d_gkr_info, &d_dense, &d_gkr, &d_eq, &d_lambda, (void*)&dim, &d_corners};
            RCHK(cudaLaunchKernel(zerocheck_gkr_corner_sweep_kb_kernel(), dim3((unsigned)corner.size()), dim3(256), args, SMEM, 0));
        }
        {   // zerocheck_aggregate_partials_strided: grid = stride, block 256
            uint32_t ns = (uint32_t)node_slots, cs = (uint32_t)corner_slots, s12 = 12, s4 = 4;
            void* t4 = (char*)d_tot + 12 * E;
            void* a1[] = {&d_nodes, &ns, &s12, &d_tot};
            void* a2[] = {&d_corners, &cs, &s4, &t4};
            RCHK(cudaLaunchKernel(zerocheck_aggregate_partials_strided_kernel(), dim3(12), dim3(256), a1, SMEM, 0));
            RCHK(cudaLaunchKernel(zerocheck_aggregate_partials_strided_kernel(), dim3(4), dim3(256), a2, SMEM, 0));
        }
        RCHK(cudaMemcpy(o, d_tot, 16 * E, cudaMemcpyDeviceToHost));
        o += 64;
    }

    // ---- zerocheck_fix_last_two_variables (prover.rs:2295-2387 -> primitives.rs:238-335)
    uint32_t length = (uint32_t)total_pairs;   // the input's pair count
    {
        fold_host(); fold_host();
        uint64_t want = 0;
        for (auto h : colh) want += h;
        uint32_t *h1, *s1, *h2, *s2, total;
        RCHK(fold_metadata(mem, (const uint32_t*)d_colh, n_cols, &h1, &s1, &total));
        RCHK(fold_metadata(mem, h1, n_cols, &h2, &s2, &total));
        if (total != want) return "ref_zerocheck: the fold metadata disagrees with the h.div_ceil(4) * 2 recurrence";
        void *d_out, *d_ocol;
        RCHK(mem.alloc(&d_out, 2ull * total * E));
        RCHK(mem.alloc(&d_ocol, (size_t)total * 4));
        JaggedMle<DenseBuffer<felt_t>> in;
        in.colIndex = (uint32_t*)d_col; in.startIndices = (uint32_t*)d_start; in.denseData.data = (felt_t*)d_dense;
        JaggedMle<DenseBuffer<ext_t>> nx;
        nx.colIndex = (uint32_t*)d_ocol; nx.startIndices = s2; nx.denseData.data = (ext_t*)d_out;
        uint32_t n_quads = length / 2;
        Ext4Raw a1 = ext(challenges), a2 = ext(challenges + 4);
        void* args[] = {&in, &nx, &n_quads, &a1, &a2};
        RCHK(cudaLaunchKernel(fix_last_two_variables_jagged_felt(), dim3(std::max<uint32_t>((n_quads + 65535) / 65536, 256)), dim3(256), args, 0, 0));
        RCHK(fix_geq(challenges));
        RCHK(fix_geq(challenges + 4));
        d_dense = d_out; d_col = d_ocol; d_start = s2; d_colh = h2;
        length = total;
        RCHK(chip_layouts());
    }

    // ---- rounds 2 .. mlr - 1: evaluate_zerocheck (prover.rs:1434-1796) then zerocheck_fix_last_variable (prover.rs:2189-2285)
    for (uint32_t r = 2; r < mlr; r++) {
        const uint32_t dim = mlr - r - 1;
        void *d_eq, *d_part, *d_tot;
        RCHK(eq_table(dim, &d_eq));
        std::vector<BlockDispatch> disp[2], gkr;
        for (int t = 0; t < 2; t++)
            for (uint32_t i = 0; i < tiers[t].chip.size(); i++) tiles(disp[t], i, chip_height(tiers[t].chip[i]) / 2, block_size(tiers[t]) * 4);
        for (uint32_t k : gkr_active) tiles(gkr, k, chip_height(k) / 2, 256 * 4);
        const size_t slots = (disp[0].size() + disp[1].size() + n_geq + gkr.size()) * 3;
        RCHK(mem.alloc(&d_part, std::max<size_t>(slots, 1) * E));
        RCHK(mem.alloc(&d_tot, 3 * E));
        static void* (*const K[6])() = {zerocheck_fused_sequential_ext_32_kernel, zerocheck_fused_sequential_ext_64_kernel,
                                        zerocheck_fused_sequential_ext_128_kernel, zerocheck_fused_sequential_ext_256_kernel,
                                        zerocheck_fused_sequential_ext_512_kernel, zerocheck_fused_sequential_ext_1024_kernel};
        size_t slot = 0;
        for (int t = 0; t < 2; t++) {
            if (disp[t].empty()) continue;
            void *d_disp, *part = (char*)d_part + slot * E;
            RCHK(dev_upload(mem, disp[t].data(), disp[t].size() * sizeof(BlockDispatch), &d_disp));
            const unsigned bs = block_size(tiers[t]);
            void* args[] = {&d_disp, &tiers[t].d_st, &d_layouts, &d_dense, &d_pv, &d_alpha, &d_eq, &d_lambda, &d_gkr, (void*)&dim, &part};
            RCHK(cudaLaunchKernel(zc_tier_kernel(tiers[t].max_reg, K), dim3((unsigned)disp[t].size(), 1, 3), dim3(bs), args, (bs / 32) * E, 0));
            slot += disp[t].size() * 3;
        }
        if (n_geq) {
            void* part = (char*)d_part + slot * E;
            void* args[] = {&d_geq_chips, &n_geq, &d_geq, &d_pad_adj, &d_lambda, &d_layouts, &d_eq, (void*)&dim, &part};
            RCHK(cudaLaunchKernel(zerocheck_geq_corrections_kernel(), dim3(n_geq), dim3(256), args, SMEM, 0));
            slot += n_geq * 3;
        }
        if (!gkr.empty()) {
            void *d_disp, *part = (char*)d_part + slot * E;
            RCHK(dev_upload(mem, gkr.data(), gkr.size() * sizeof(BlockDispatch), &d_disp));
            void* args[] = {&d_disp, &d_layouts, &d_gkr_info, &d_dense, &d_gkr, &d_eq, &d_lambda, (void*)&dim, &part};
            RCHK(cudaLaunchKernel(zerocheck_gkr_sweep_ext_kernel(), dim3((unsigned)gkr.size(), 1, 3), dim3(256), args, SMEM, 0));
        }
        {   // zerocheck_aggregate_partials: one block of 256
            uint32_t ns = (uint32_t)slots;
            void* args[] = {&d_part, &ns, &d_tot};
            RCHK(cudaLaunchKernel(zerocheck_aggregate_partials_kernel(), dim3(1), dim3(256), args, SMEM, 0));
        }
        RCHK(cudaMemcpy(o, d_tot, 3 * E, cudaMemcpyDeviceToHost));
        o += 12;
        // evaluate_jagged_fix_last_variable (primitives.rs:127-225): block 256, grid max(ceil(length / 2^16), 256)
        fold_host();
        uint32_t *h1, *s1, total;
        RCHK(fold_metadata(mem, (const uint32_t*)d_colh, n_cols, &h1, &s1, &total));
        void *d_out, *d_ocol;
        RCHK(mem.alloc(&d_out, 2ull * total * E));
        RCHK(mem.alloc(&d_ocol, (size_t)total * 4));
        JaggedMle<DenseBuffer<ext_t>> in, nx;
        in.colIndex = (uint32_t*)d_col; in.startIndices = (uint32_t*)d_start; in.denseData.data = (ext_t*)d_dense;
        nx.colIndex = (uint32_t*)d_ocol; nx.startIndices = s1; nx.denseData.data = (ext_t*)d_out;
        Ext4Raw a = ext(challenges + 4 * r);
        void* args[] = {&in, &nx, &length, &a};
        RCHK(cudaLaunchKernel(fix_last_variable_jagged_ext(), dim3(std::max<uint32_t>((length + 65535) / 65536, 256)), dim3(256), args, 0, 0));
        RCHK(fix_geq(challenges + 4 * r));
        mem.release(d_dense);
        d_dense = d_out; d_col = d_ocol; d_start = s1; d_colh = h1;
        length = total;
        RCHK(chip_layouts());
    }

    // ---- the folded values zerocheck() demultiplexes (prover.rs:2692-2702): 4 entries per non-empty column after the last fold
    size_t nonempty = 0;
    for (uint32_t h : input_colh) nonempty += h != 0;
    if (2ull * length != 4 * nonempty) return "ref_zerocheck: the folded trace does not hold 4 entries per non-empty column";
    std::vector<uint32_t> fin(8ull * length);   // 2 * length ext elements
    RCHK(cudaMemcpy(fin.data(), d_dense, fin.size() * 4, cudaMemcpyDeviceToHost));
    for (uint32_t c = 0, idx = 0; c < n_cols; c++) {
        if (input_colh[c]) {
            memcpy(o + 4 * c, &fin[4 * idx], 16);
            idx += 4;
        } else {
            memset(o + 4 * c, 0, 16);
        }
    }
    return nullptr;
}

}  // extern "C"

