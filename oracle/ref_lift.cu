// ORACLE — TEST INFRASTRUCTURE ONLY.  Launches the reference's own hash-to-curve primitives, compiled unmodified from where they lie:
// kb31_septic_extension_t::curve_formula / pow_r / sqrt / is_exception / is_receive and bb31_septic_curve_t::operator+= of
// sp1-gpu/crates/sys/include/fields/kb31_septic_extension_t.cuh, and poseidon2::KoalaBearHasher::permute of
// sp1-gpu/crates/sys/include/poseidon2/poseidon2.cuh.  The trial loop of SepticCurve::lift_x (crates/hypercube/src/septic_curve.rs:
// 124-164) is written here over those primitives: the reference's own GPU loop sits in a translation unit that needs a generated
// header.  Built by oracle/ref_lift.mk into oracle/_ref/libsp1ref_lift.so for tests/test_ref_lift.py, which stores the outputs in
// tests/golden/ref_lift.json.  Words are Montgomery words (kb31_t's representation).
#include "fields/kb31_septic_extension_t.cuh"
#include "poseidon2/poseidon2.cuh"
#include <cuda_runtime.h>
#include <cstdint>

using E7 = kb31_septic_extension_t;
using Pt = bb31_septic_curve_t;

__device__ E7 ld7(const uint32_t* p) { E7 r; for (int i = 0; i < 7; i++) r.value[i] = kb31_t((uint32_t)p[i]); return r; }
__device__ void st7(const E7& a, uint32_t* p) { for (int i = 0; i < 7; i++) p[i] = *reinterpret_cast<const uint32_t*>(&a.value[i]); }
__device__ Pt ldp(const uint32_t* p) { return Pt(ld7(p), ld7(p + 7)); }
__device__ void stp(const Pt& a, uint32_t* p) { st7(a.x, p); st7(a.y, p + 7); }

// the square test of lift_x: the norm pow_r is a square of the base field
__device__ bool norm_is_square(kb31_t n) { return (n ^ (uint32_t)((kb31_t::MOD - 1) >> 1)) == kb31_t::one(); }

// lift_x of msgs[i] (8 words): offsets[i] = the offset (-1: none of 256), pts[i] = (x, y) with y a receive
__global__ void ref_lift_kernel(const uint32_t* msgs, int32_t* offsets, uint32_t* pts, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    offsets[i] = -1;
    for (uint32_t off = 0; off < 256; off++) {
        kb31_t s[16];
        for (int k = 0; k < 8; k++) s[k] = kb31_t((uint32_t)msgs[8 * i + k]);
        s[7] += kb31_t::from_canonical_u32(off << 16);
        for (int k = 8; k < 16; k++) s[k] = kb31_t::zero();
        poseidon2::KoalaBearHasher::permute(s, s);
        E7 x;
        for (int k = 0; k < 7; k++) x.value[k] = s[k];
        const E7 y2 = x.curve_formula();
        const kb31_t nrm = y2.pow_r();
        if (!norm_is_square(nrm)) continue;
        E7 y = y2.sqrt(nrm);
        if (y.is_exception()) continue;
        if (!y.is_receive()) y = E7::zero() - y;
        offsets[i] = (int32_t)off;
        stp(Pt(x, y), pts + 14 * i);
        return;
    }
}
// sqrt of squares: ok[i] = whether the norm is a square, out[i] = sqrt(pow_r) where it is
__global__ void ref_sqrt_kernel(const uint32_t* a, uint32_t* out, uint32_t* ok, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const E7 x = ld7(a + 7 * i);
    const kb31_t nrm = x.pow_r();
    ok[i] = norm_is_square(nrm);
    if (ok[i]) st7(x.sqrt(nrm), out + 7 * i);
}
// p + q under operator+= (infinity = 14 zero words)
__global__ void ref_add_kernel(const uint32_t* p, const uint32_t* q, uint32_t* out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Pt r = ldp(p + 14 * i);
    r += ldp(q + 14 * i);
    stp(r, out + 14 * i);
}

namespace {
const char* err(cudaError_t e) { return e == cudaSuccess ? nullptr : cudaGetErrorString(e); }
#define RL_TRY(x) do { if (const char* msg_ = err(x)) return msg_; } while (0)
struct Buf {
    void* d = nullptr;
    ~Buf() { if (d) cudaFree(d); }
};
}  // namespace

extern "C" {
// n_lift messages -> offsets + points; n_sqrt elements -> roots + flags; n_add point pairs -> sums.  Returns NULL or a CUDA error string.
const char* ref_lift(const uint32_t* h_msgs, uint32_t n_lift, int32_t* h_offsets, uint32_t* h_pts, const uint32_t* h_sq, uint32_t n_sqrt,
                     uint32_t* h_roots, uint32_t* h_ok, const uint32_t* h_p, const uint32_t* h_q, uint32_t n_add, uint32_t* h_sum) {
    Buf msgs, offs, pts, sq, roots, ok, p, q, sum;
    RL_TRY(cudaMalloc(&msgs.d, 32 * n_lift + 4)); RL_TRY(cudaMalloc(&offs.d, 4 * n_lift + 4)); RL_TRY(cudaMalloc(&pts.d, 56 * n_lift + 4));
    RL_TRY(cudaMalloc(&sq.d, 28 * n_sqrt + 4)); RL_TRY(cudaMalloc(&roots.d, 28 * n_sqrt + 4)); RL_TRY(cudaMalloc(&ok.d, 4 * n_sqrt + 4));
    RL_TRY(cudaMalloc(&p.d, 56 * n_add + 4)); RL_TRY(cudaMalloc(&q.d, 56 * n_add + 4)); RL_TRY(cudaMalloc(&sum.d, 56 * n_add + 4));
    RL_TRY(cudaMemcpy(msgs.d, h_msgs, 32 * n_lift, cudaMemcpyHostToDevice));
    RL_TRY(cudaMemset(pts.d, 0, 56 * n_lift + 4)); RL_TRY(cudaMemset(roots.d, 0, 28 * n_sqrt + 4));
    RL_TRY(cudaMemcpy(sq.d, h_sq, 28 * n_sqrt, cudaMemcpyHostToDevice));
    RL_TRY(cudaMemcpy(p.d, h_p, 56 * n_add, cudaMemcpyHostToDevice)); RL_TRY(cudaMemcpy(q.d, h_q, 56 * n_add, cudaMemcpyHostToDevice));
    ref_lift_kernel<<<(n_lift + 63) / 64 + 1, 64>>>((const uint32_t*)msgs.d, (int32_t*)offs.d, (uint32_t*)pts.d, n_lift);
    ref_sqrt_kernel<<<(n_sqrt + 63) / 64 + 1, 64>>>((const uint32_t*)sq.d, (uint32_t*)roots.d, (uint32_t*)ok.d, n_sqrt);
    ref_add_kernel<<<(n_add + 63) / 64 + 1, 64>>>((const uint32_t*)p.d, (const uint32_t*)q.d, (uint32_t*)sum.d, n_add);
    RL_TRY(cudaGetLastError());
    RL_TRY(cudaDeviceSynchronize());
    RL_TRY(cudaMemcpy(h_offsets, offs.d, 4 * n_lift, cudaMemcpyDeviceToHost)); RL_TRY(cudaMemcpy(h_pts, pts.d, 56 * n_lift, cudaMemcpyDeviceToHost));
    RL_TRY(cudaMemcpy(h_roots, roots.d, 28 * n_sqrt, cudaMemcpyDeviceToHost)); RL_TRY(cudaMemcpy(h_ok, ok.d, 4 * n_sqrt, cudaMemcpyDeviceToHost));
    RL_TRY(cudaMemcpy(h_sum, sum.d, 56 * n_add, cudaMemcpyDeviceToHost));
    return nullptr;
}
}
