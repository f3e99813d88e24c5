// ORACLE — TEST INFRASTRUCTURE ONLY.  Launches the reference's own septic arithmetic, sp1-gpu/crates/sys/include/fields/
// kb31_septic_extension_t.cuh (kb31_septic_extension_t, bb31_septic_curve_t), compiled unmodified from where it lies, on given inputs:
// products and reciprocals of septic elements, curve additions, the chains k·P of dummy_point() and start_point() built by repeated
// `+`, and a digest sum.  Built by oracle/ref_septic.mk into oracle/_ref/libsp1ref_septic.so for tests/test_ref_septic.py, which
// stores the outputs in tests/golden/ref_septic.json.  Words are Montgomery words (kb31_t's representation).
#include "fields/kb31_septic_extension_t.cuh"
#include <cuda_runtime.h>
#include <cstdint>

using E7 = kb31_septic_extension_t;
using Pt = bb31_septic_curve_t;

__device__ E7 ld7(const uint32_t* p) { E7 r; for (int i = 0; i < 7; i++) r.value[i] = kb31_t((uint32_t)p[i]); return r; }
__device__ void st7(const E7& a, uint32_t* p) { for (int i = 0; i < 7; i++) p[i] = *reinterpret_cast<const uint32_t*>(&a.value[i]); }   // kb31_t holds its Montgomery word only
__device__ Pt ldp(const uint32_t* p) { return Pt(ld7(p), ld7(p + 7)); }
__device__ void stp(const Pt& a, uint32_t* p) { st7(a.x, p); st7(a.y, p + 7); }

__global__ void ref_septic_ops_kernel(const uint32_t* a, const uint32_t* b, uint32_t* mul, uint32_t* inv, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const E7 x = ld7(a + 7 * i), y = ld7(b + 7 * i);
    st7(x * y, mul + 7 * i);
    st7(x.reciprocal(), inv + 7 * i);
}
__global__ void ref_curve_add_kernel(const uint32_t* p, const uint32_t* q, uint32_t* out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    stp(ldp(p + 14 * i) + ldp(q + 14 * i), out + 14 * i);
}
// out[0..k): P, 2P, ..., kP of dummy_point() (which = 0) or start_point() (which = 1)
__global__ void ref_curve_chain_kernel(uint32_t which, uint32_t k, uint32_t* out) {
    const Pt base = which ? Pt::start_point() : Pt::dummy_point();
    Pt acc = base;
    for (uint32_t i = 0; i < k; i++) {
        stp(acc, out + 14 * i);
        acc = acc + base;
    }
}
// digest sum of pts[0..m): pts[0] + Σ_{i>0} (pts[i] - start_point()) - the group value of SepticDigest additions starting at pts[0]
__global__ void ref_digest_sum_kernel(const uint32_t* pts, uint32_t m, uint32_t* out) {
    const Pt zero = Pt::start_point();
    const Pt neg_zero(zero.x, E7::zero() - zero.y);
    Pt acc = ldp(pts);
    for (uint32_t i = 1; i < m; i++) acc = acc + ldp(pts + 14 * i) + neg_zero;
    stp(acc, out);
}

namespace {
const char* err(cudaError_t e) { return e == cudaSuccess ? nullptr : cudaGetErrorString(e); }
#define RS_TRY(x) do { if (const char* msg_ = err(x)) return msg_; } while (0)
struct Buf {
    uint32_t* d = nullptr;
    ~Buf() { if (d) cudaFree(d); }
};
}  // namespace

extern "C" {
// n septic pairs (a, b) -> a * b and a.reciprocal(); np point pairs -> p + q; the chains of k multiples of dummy_point() and
// start_point(); the digest sum of m points.  Returns NULL or a CUDA error string.
const char* ref_septic(const uint32_t* h_a, const uint32_t* h_b, uint32_t n, uint32_t* h_mul, uint32_t* h_inv, const uint32_t* h_p,
                       const uint32_t* h_q, uint32_t np, uint32_t* h_add, uint32_t k, uint32_t* h_chain_dummy, uint32_t* h_chain_start,
                       const uint32_t* h_pts, uint32_t m, uint32_t* h_sum) {
    Buf a, b, mul, inv, p, q, add, cd, cs, pts, sum;
    RS_TRY(cudaMalloc(&a.d, 28 * n + 4)); RS_TRY(cudaMalloc(&b.d, 28 * n + 4));
    RS_TRY(cudaMalloc(&mul.d, 28 * n + 4)); RS_TRY(cudaMalloc(&inv.d, 28 * n + 4));
    RS_TRY(cudaMalloc(&p.d, 56 * np + 4)); RS_TRY(cudaMalloc(&q.d, 56 * np + 4)); RS_TRY(cudaMalloc(&add.d, 56 * np + 4));
    RS_TRY(cudaMalloc(&cd.d, 56 * k + 4)); RS_TRY(cudaMalloc(&cs.d, 56 * k + 4));
    RS_TRY(cudaMalloc(&pts.d, 56 * m + 4)); RS_TRY(cudaMalloc(&sum.d, 56));
    RS_TRY(cudaMemcpy(a.d, h_a, 28 * n, cudaMemcpyHostToDevice)); RS_TRY(cudaMemcpy(b.d, h_b, 28 * n, cudaMemcpyHostToDevice));
    RS_TRY(cudaMemcpy(p.d, h_p, 56 * np, cudaMemcpyHostToDevice)); RS_TRY(cudaMemcpy(q.d, h_q, 56 * np, cudaMemcpyHostToDevice));
    RS_TRY(cudaMemcpy(pts.d, h_pts, 56 * m, cudaMemcpyHostToDevice));
    ref_septic_ops_kernel<<<(n + 127) / 128 + 1, 128>>>(a.d, b.d, mul.d, inv.d, n);
    ref_curve_add_kernel<<<(np + 127) / 128 + 1, 128>>>(p.d, q.d, add.d, np);
    ref_curve_chain_kernel<<<1, 1>>>(0, k, cd.d);
    ref_curve_chain_kernel<<<1, 1>>>(1, k, cs.d);
    ref_digest_sum_kernel<<<1, 1>>>(pts.d, m, sum.d);
    RS_TRY(cudaGetLastError());
    RS_TRY(cudaDeviceSynchronize());
    RS_TRY(cudaMemcpy(h_mul, mul.d, 28 * n, cudaMemcpyDeviceToHost)); RS_TRY(cudaMemcpy(h_inv, inv.d, 28 * n, cudaMemcpyDeviceToHost));
    RS_TRY(cudaMemcpy(h_add, add.d, 56 * np, cudaMemcpyDeviceToHost));
    RS_TRY(cudaMemcpy(h_chain_dummy, cd.d, 56 * k, cudaMemcpyDeviceToHost)); RS_TRY(cudaMemcpy(h_chain_start, cs.d, 56 * k, cudaMemcpyDeviceToHost));
    RS_TRY(cudaMemcpy(h_sum, sum.d, 56, cudaMemcpyDeviceToHost));
    return nullptr;
}
}
