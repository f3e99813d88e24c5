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
#include "zerocheck/sequential.cuh"
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
// populateLastCircuitLayer (sys/lib/logup_gkr/tracegen.cu:77-160) for ONE chip.  The interactions arrive in the flattened CSR form of
// `Interactions<F>` (sys/include/logup_gkr/tracegen.cuh:20-36; host twin sp1-gpu/crates/logup_gkr/src/interactions.rs).  Output layout as
// the kernel writes it: with q = ceil(ceil(height/2)/2), interaction j owns the row-pair slots [2 q j, 2 q j + ceil(height/2)); slot i
// holds (numerator at row 2i, denominator at row 2i) and, 2 * output_height further, the same for row 2i+1; output_height = 2 q n.
extern "C" void* logup_gkr_populate_last_circuit_layer();
const char* ref_gkr_populate(const uint32_t* h_prep, uint64_t prep_words, const uint32_t* h_main, uint64_t main_words, uint64_t height, uint32_t n_inter,
                             const uint64_t* values_ptr, const uint64_t* mult_ptr, const uint64_t* vcw_ptr, uint64_t n_values, const uint64_t* vcw_col,
                             const uint8_t* vcw_is_prep, const uint32_t* vcw_weight, uint64_t n_vcw, const uint32_t* values_constants,
                             const uint64_t* mcw_col, const uint8_t* mcw_is_prep, const uint32_t* mcw_weight, uint64_t n_mcw,
                             const uint32_t* mult_constants, const uint32_t* arg_indices, const uint8_t* is_send, const uint32_t* alpha4,
                             const uint32_t* betas, uint32_t n_betas, uint32_t* out_num, uint32_t* out_den, uint64_t* out_height) {
    const uint64_t half = height ? (height + 1) / 2 : 1, q = (half + 1) / 2, outH = 2 * q * n_inter;
    auto up = [](const void* h, size_t bytes, void** d) -> cudaError_t {
        cudaError_t e = cudaMalloc(d, bytes ? bytes : 8);
        if (e == cudaSuccess && bytes) e = cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice);
        return e;
    };
    std::vector<PairCol<felt_t>> vcw(n_vcw), mcw(n_mcw);
    for (uint64_t i = 0; i < n_vcw; i++) { vcw[i].column_idx = vcw_col[i]; vcw[i].is_preprocessed = vcw_is_prep[i]; memcpy(&vcw[i].weight, &vcw_weight[i], 4); }
    for (uint64_t i = 0; i < n_mcw; i++) { mcw[i].column_idx = mcw_col[i]; mcw[i].is_preprocessed = mcw_is_prep[i]; memcpy(&mcw[i].weight, &mcw_weight[i], 4); }
    std::vector<uint8_t> send(is_send, is_send + n_inter);   // bool on the device side
    std::vector<uint32_t> start(n_inter + 1);
    for (uint32_t j = 0; j <= n_inter; j++) start[j] = (uint32_t)(q * j);
    Interactions<felt_t> I{};
    void *d_prep, *d_main, *d_start, *d_col, *d_num, *d_den, *d_betas;
    RCHK(up(values_ptr, (n_inter + 1) * 8, (void**)&I.values_ptr));
    RCHK(up(mult_ptr, (n_inter + 1) * 8, (void**)&I.multiplicities_ptr));
    RCHK(up(vcw_ptr, (n_values + 1) * 8, (void**)&I.values_col_weights_ptr));
    RCHK(up(vcw.data(), n_vcw * sizeof(PairCol<felt_t>), (void**)&I.values_col_weights));
    RCHK(up(values_constants, n_values * 4, (void**)&I.values_constants));
    RCHK(up(mcw.data(), n_mcw * sizeof(PairCol<felt_t>), (void**)&I.mult_col_weights));
    RCHK(up(mult_constants, n_inter * 4, (void**)&I.mult_constants));
    RCHK(up(arg_indices, n_inter * 4, (void**)&I.arg_indices));
    RCHK(up(send.data(), n_inter, (void**)&I.is_send));
    I.num_interactions = n_inter;
    RCHK(up(h_prep, prep_words * 4, &d_prep));
    RCHK(up(h_main, main_words * 4, &d_main));
    RCHK(up(start.data(), start.size() * 4, &d_start));
    RCHK(up(betas, (size_t)n_betas * 16, &d_betas));
    RCHK(cudaMalloc(&d_col, (2 * outH + 8) * 4));
    RCHK(cudaMalloc(&d_num, 4 * outH * 4 + 16));
    RCHK(cudaMalloc(&d_den, 4 * outH * 16 + 16));
    RCHK(cudaMemset(d_num, 0, 4 * outH * 4 + 16));
    RCHK(cudaMemset(d_den, 0, 4 * outH * 16 + 16));
    Ext4Raw alpha;
    memcpy(&alpha, alpha4, 16);
    size_t offset = 0, th = height, oh = outH;
    bool is_padding = false;
    void* args[] = {&I, &d_start, &d_col, &d_num, &d_den, &d_prep, &d_main, &alpha, &d_betas, &offset, &th, &oh, &is_padding};
    dim3 block(64, 4), grid((unsigned)((half + 63) / 64), (n_inter + 3) / 4);
    RCHK(cudaLaunchKernel(logup_gkr_populate_last_circuit_layer(), grid, block, args, 0, 0));
    RCHK(cudaDeviceSynchronize());
    RCHK(cudaMemcpy(out_num, d_num, 4 * outH * 4, cudaMemcpyDeviceToHost));
    RCHK(cudaMemcpy(out_den, d_den, 4 * outH * 16, cudaMemcpyDeviceToHost));
    *out_height = outH;
    for (void* p : {(void*)I.values_ptr, (void*)I.multiplicities_ptr, (void*)I.values_col_weights_ptr, (void*)I.values_col_weights, (void*)I.values_constants,
                    (void*)I.mult_col_weights, (void*)I.mult_constants, (void*)I.arg_indices, (void*)I.is_send, d_prep, d_main, d_start, d_col, d_num, d_den, d_betas})
        cudaFree(p);
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

}  // extern "C"

