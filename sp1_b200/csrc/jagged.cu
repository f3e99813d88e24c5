// Jagged PCS on the device: commit of a round of chip tables and the evaluation proof
// (Hadamard sumcheck of the dense trace against the jagged "little polynomial", the branching-program
// evaluation sumcheck, then the stacked/BaseFold proof of pcs.cu).
// Reference behaviour: slop/crates/jagged/src/prover.rs:106-328, hadamard.rs:93-151, poly.rs:136-296,384-470,
// jagged_eval/{sumcheck_poly.rs,sumcheck_sum_as_poly.rs,eval_sumcheck_prover.rs}; the GPU twins it replaces:
// sp1-gpu/crates/{jagged_sumcheck,jagged_assist} + sys/lib/{jagged_sumcheck,jagged_assist}/*.cu.
// HOW (results identical): the dense buffers of all rounds form one virtual long vector (no restacking copy);
// the first K <= 5 rounds are summed straight from the base-field trace, then each round runs as ONE fused kernel (fix the
// previous variable + accumulate the next round's sums) so the folded vectors are written once and read once; the
// branching-program sumcheck evaluates all (column, node) pairs of a round in one launch.
#include "ctx.cuh"
#include "challenger.cuh"
#include "hostfield.hpp"
#include "kb31.cuh"
#include "sumcheck.cuh"
#include <algorithm>
#include <memory>
#include <vector>

#include "pcs.cuh"

namespace {

using kb::Ext;
using hf::E4;

struct SegTable {  // the virtual long base vector = concatenation of the rounds' dense buffers, then zeros
    const uint32_t* ptr[8];
    uint64_t end[8];
    int n;
};

// ---- rounds 0 .. K-1 summed straight from the base-field trace, then one fold pass to level K ----------------------------------
// The jagged little polynomial is ext[i] = col_eq[c(i)] * row_eq[i - prefix[c(i)]] for i < prefix[ncols], else 0.
// c(i) = the last column with prefix[c] <= i (zero-height columns share a prefix value: the last one has the non-empty range).
// start[i >> JP_SHIFT] (built on the host from the same prefix sums) is a column at or before c(i), so the search is a short
// forward walk instead of a binary search per element.
// When 2^K divides every column prefix sum (the reference pads trace heights to
// multiples of 32, crates/hypercube/src/util.rs:57), every aligned block of 2^(r+1) <= 2^K entries lies in one column, and after
// r folds by alpha_0 .. alpha_{r-1} both sides of the sumcheck stay in closed form over the base-field trace b:
//   dense_r[o] = sum_{t < 2^r} w_r[t] b[o 2^r + t],            w_r[t] = prod_{s < r} (bit s of t ? alpha_s : 1 - alpha_s)
//   ext_r[o]   = col_eq[c] * row_eq_r[(o 2^r - prefix[c]) >> r],  row_eq_r[k] = sum_t w_r[t] row_eq[k 2^r + t].
// row_eq = eq(z_row high bits) (x) eq(z_row low JK_LOW bits), so row_eq_r = eq_hi (x) L_r with L_r[u] = sum_t w_r[t] eq_lo[u 2^r + t]
// a table of at most 2^JK_LOW entries that each block builds in shared memory.  A round r < K is then one read-only pass over the
// trace: per block of 2^(r+1) words, two EF x F weighted sums (lazy 64-bit accumulation) and two products with the L_r table; the
// factor col_eq[c] * eq_hi[h] is applied once per (column, high row bits) run of a lane.  After round K-1 one pass writes the
// level-K dense and eq arrays (2^(log_m - K) EF entries each) and sums round K; hadamard_fold_kernel takes it from there.
// K = 0 (some column starts at an odd index) has no trace rounds: the fold pass to level 0 (w_0 = {1}, L_0 = eq_lo) lifts the trace
// to EF, writes the eq array and sums round 0.
constexpr int JP_SHIFT = 12;
constexpr int JK_MAX = 5;   // rounds summed from the trace at most (K = 4 measured slower on S2c, DESIGN.md §3.5)
constexpr int JK_LOW = 10;  // low row bits of the eq_lo factor (the shared tables: 2 x 2^9 EF for round 0)
struct JWeights { Ext w[1 << JK_MAX]; };  // w_r[t], t < 2^r

__device__ __forceinline__ uint32_t jp_column(const uint64_t* __restrict__ prefix, uint32_t ncols, uint32_t c, uint64_t i) {
    while (c + 1 < ncols && prefix[c + 1] <= i) c++;
    return c;
}
// pointer to word i of the virtual vector (i < the last segment end); the caller's aligned block lies inside one segment
__device__ __forceinline__ const uint32_t* seg_ptr(const SegTable& t, uint64_t i) {
    int s = 0;
    uint64_t start = 0;
    while (s + 1 < t.n && i >= t.end[s]) { start = t.end[s]; s++; }
    return t.ptr[s] + (i - start);
}
template <int NW>
__device__ __forceinline__ void load_words(const uint32_t* p, uint32_t* b) {  // p aligned to 4 * min(NW, 4) bytes
    if constexpr (NW == 1) {
        b[0] = __ldg(p);
    } else if constexpr (NW == 2) {
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(p)); b[0] = v.x; b[1] = v.y;
    } else {
#pragma unroll
        for (int k = 0; k < NW / 4; k++) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(p) + k);
            b[4 * k] = v.x; b[4 * k + 1] = v.y; b[4 * k + 2] = v.z; b[4 * k + 3] = v.w;
        }
    }
}
// sum_{t < NW} w[t] b[t]: up to four products (< 4 (p-1)^2 < 2 p 2^32) per 64-bit limb accumulator before one reduction
template <int NW>
__device__ __forceinline__ Ext wdot(const Ext* w, const uint32_t* b) {
    Ext r = kb::ext_zero();
#pragma unroll
    for (int t0 = 0; t0 < NW; t0 += 4) {
        uint64_t a[4] = {0, 0, 0, 0};
#pragma unroll
        for (int t = t0; t < t0 + 4 && t < NW; t++)
#pragma unroll
            for (int l = 0; l < 4; l++) a[l] += (uint64_t)b[t] * w[t].c[l];
#pragma unroll
        for (int l = 0; l < 4; l++) r.c[l] = kb::add(r.c[l], kb::monty_reduce2(a[l]));
    }
    return r;
}
// L_r[u] = sum_{t < 2^r} w[t] eq_lo[u 2^r + t]
template <int R>
__device__ __forceinline__ Ext folded_eq_lo(const JWeights& W, const uint32_t* __restrict__ eq_lo, uint32_t u) {
    Ext acc = kb::ext_zero();
#pragma unroll
    for (int t = 0; t < (1 << R); t++) acc = kb::ext_add(acc, kb::ext_mul(W.w[t], kb::ext_load(eq_lo + 4 * ((u << R) + t))));
    return acc;
}

// round R < K: s0 = sum_j ext_R[2j] dense_R[2j], sh = sum_j (ext_R[2j] + ext_R[2j+1]) (dense_R[2j] + dense_R[2j+1]) over the
// nblk blocks of 2^(R+1) words of the real area; each warp walks a contiguous span of blocks (a multiple of 32)
template <int R>
__global__ void __launch_bounds__(256) jagged_round_kernel(SegTable base, const uint64_t* __restrict__ prefix, uint32_t ncols,
                                                           const uint32_t* __restrict__ start, const uint32_t* __restrict__ col_eq,
                                                           const uint32_t* __restrict__ eq_hi, const uint32_t* __restrict__ eq_lo, int lb,
                                                           JWeights W, uint64_t nblk, uint64_t span, uint32_t* __restrict__ partial, Mail mail) {
    constexpr int NB = 2 << R;  // words per block
    __shared__ Ext tA[1 << (JK_LOW - 1)], tB[1 << (JK_LOW - 1)];  // tA[q] = L_R[2q], tB[q] = L_R[2q] + L_R[2q+1]
    for (uint32_t q = threadIdx.x; q < (1u << (lb - R - 1)); q += blockDim.x) {
        const Ext l0 = folded_eq_lo<R>(W, eq_lo, 2 * q), l1 = folded_eq_lo<R>(W, eq_lo, 2 * q + 1);
        tA[q] = l0; tB[q] = kb::ext_add(l0, l1);
    }
    __syncthreads();
    Ext s0 = kb::ext_zero(), sh = kb::ext_zero();
    Ext t0 = kb::ext_zero(), th = kb::ext_zero();
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t j_begin = warp * span, j_end = min(j_begin + span, nblk);
    const uint64_t lomask = (1ull << lb) - 1;
    uint32_t c = 0xffffffffu;
    uint64_t h = 0;
    auto flush = [&]() {
        const Ext f = kb::ext_mul(kb::ext_load(col_eq + 4 * c), kb::ext_load(eq_hi + 4 * h));
        s0 = kb::ext_add(s0, kb::ext_mul(f, t0)); sh = kb::ext_add(sh, kb::ext_mul(f, th));
        t0 = kb::ext_zero(); th = kb::ext_zero();
    };
    for (uint64_t j = j_begin + lane; j < j_end; j += 32) {
        const uint64_t i = j * NB;
        const uint32_t cn = jp_column(prefix, ncols, c == 0xffffffffu ? start[i >> JP_SHIFT] : c, i);
        const uint64_t rho = i - prefix[cn], hn = rho >> lb;
        if (cn != c || hn != h) {
            if (c != 0xffffffffu) flush();
            c = cn; h = hn;
        }
        uint32_t b[NB];
        load_words<NB>(seg_ptr(base, i), b);
        const uint32_t q = (uint32_t)((rho & lomask) >> (R + 1));
        if constexpr (R == 0) {
            t0 = kb::ext_add(t0, kb::ext_mul_base(tA[q], b[0]));
            th = kb::ext_add(th, kb::ext_mul_base(tB[q], kb::add(b[0], b[1])));
        } else {
            const Ext d0 = wdot<(1 << R)>(W.w, b), d1 = wdot<(1 << R)>(W.w, b + (1 << R));
            t0 = kb::ext_add(t0, kb::ext_mul(tA[q], d0));
            th = kb::ext_add(th, kb::ext_mul(tB[q], kb::ext_add(d0, d1)));
        }
    }
    if (c != 0xffffffffu) flush();
    block_reduce<2>({s0, sh}, partial, mail);
}

// fix alpha_{K-1}: write level K (dense_K, ext_K: nout = 2^(log_m - K) EF entries each, zero beyond the real area) and sum round K
template <int K>
__global__ void __launch_bounds__(256) jagged_fold_to_kernel(SegTable base, const uint64_t* __restrict__ prefix, uint32_t ncols,
                                                             const uint32_t* __restrict__ start, const uint32_t* __restrict__ col_eq,
                                                             const uint32_t* __restrict__ eq_hi, const uint32_t* __restrict__ eq_lo, int lb,
                                                             JWeights W, uint64_t area, uint64_t nout_pairs, uint32_t* __restrict__ base_out,
                                                             uint32_t* __restrict__ ext_out, uint32_t* __restrict__ partial, uint64_t nout, Mail mail) {
    constexpr int NW = 1 << K;  // words per level-K entry
    __shared__ Ext tL[1 << (JK_LOW - (K > 0))];  // L_K[u], u < 2^(lb - K)
    for (uint32_t u = threadIdx.x; u < (1u << (lb - K)); u += blockDim.x) tL[u] = folded_eq_lo<K>(W, eq_lo, u);
    __syncthreads();
    const uint64_t lomask = (1ull << lb) - 1;
    Ext s0 = kb::ext_zero(), sh = kb::ext_zero();
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nout_pairs; j += (uint64_t)gridDim.x * blockDim.x) {
        Ext nb[2], ne[2];
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
            const uint64_t o = 2 * j + hh, i = o * NW;
            nb[hh] = kb::ext_zero(); ne[hh] = kb::ext_zero();
            if (o < nout) {
                if (i < area) {
                    uint32_t b[NW];
                    load_words<NW>(seg_ptr(base, i), b);
                    nb[hh] = wdot<NW>(W.w, b);
                    const uint32_t c = jp_column(prefix, ncols, start[i >> JP_SHIFT], i);
                    const uint64_t rho = i - prefix[c];
                    ne[hh] = kb::ext_mul(kb::ext_mul(kb::ext_load(col_eq + 4 * c), kb::ext_load(eq_hi + 4 * (rho >> lb))),
                                         tL[(rho & lomask) >> K]);
                }
                kb::ext_store(base_out + 4 * o, nb[hh]);
                kb::ext_store(ext_out + 4 * o, ne[hh]);
            }
        }
        s0 = kb::ext_add(s0, kb::ext_mul(ne[0], nb[0]));
        sh = kb::ext_add(sh, kb::ext_mul(kb::ext_add(ne[0], ne[1]), kb::ext_add(nb[0], nb[1])));
    }
    block_reduce<2>({s0, sh}, partial, mail);
}

// rounds >= 1: fix the last variable (EF -> EF) and accumulate the next round's sums
__global__ void __launch_bounds__(256) hadamard_fold_kernel(const uint32_t* __restrict__ base, const uint32_t* __restrict__ ext,
                                                            uint64_t nout_pairs, Ext alpha, uint32_t* __restrict__ base_out,
                                                            uint32_t* __restrict__ ext_out, uint32_t* __restrict__ partial, uint64_t nout, Mail mail) {
    Ext s0 = kb::ext_zero(), sh = kb::ext_zero();
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nout_pairs; j += (uint64_t)gridDim.x * blockDim.x) {
        Ext nb[2], ne[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            uint64_t o = 2 * j + h;
            if (o < nout) {
                Ext b0 = kb::ext_load(base + 8 * o), b1 = kb::ext_load(base + 8 * o + 4);
                Ext e0 = kb::ext_load(ext + 8 * o), e1 = kb::ext_load(ext + 8 * o + 4);
                nb[h] = kb::ext_add(b0, kb::ext_mul(alpha, kb::ext_sub(b1, b0)));
                ne[h] = kb::ext_add(e0, kb::ext_mul(alpha, kb::ext_sub(e1, e0)));
                kb::ext_store(base_out + 4 * o, nb[h]);
                kb::ext_store(ext_out + 4 * o, ne[h]);
                if (nout == 1) kb::ext_store(partial + 8, nb[h]);  // last round: the dense component evaluation rides along
            } else { nb[h] = kb::ext_zero(); ne[h] = kb::ext_zero(); }
        }
        s0 = kb::ext_add(s0, kb::ext_mul(ne[0], nb[0]));
        sh = kb::ext_add(sh, kb::ext_mul(kb::ext_add(ne[0], ne[1]), kb::ext_add(nb[0], nb[1])));
    }
    block_reduce<2>({s0, sh}, partial, mail);
}

// ---- branching program (one layer: bp_transition, sumcheck.cuh), in prefix / suffix form ----------------------------
// The evaluation is  e0^T M_0 M_1 ... M_hl init  with one 4x4 transfer matrix per layer, M_l = M(cur_l, next_l).  In sumcheck
// round r only ONE layer holds the free variable: layers above it still see the column's boolean prefix-sum bits (and, in
// the second half, next-coordinates that were bound earlier and never change again), layers below it see coordinates that
// were bound in earlier rounds.  So per column k:  value = P_k . M_layer(lambda) . T_k[layer + 1]  with
//   T_k[l] = M_l ... M_hl init   (suffix table, one pass per half: bp_suffix_kernel)
//   P_k    = e0^T M_0 ... M_{layer-1}   (prefix row vector, one vector-matrix product per round: bp_update_kernel)
// i.e. two small products per (column, node) and round instead of hl+1 (the reference keeps the same prefix/suffix states,
// sp1-gpu/crates/sys/lib/jagged_assist).  Every product is exact field arithmetic, so the round polynomials are unchanged.
// ri_eq: per layer the 4 values eq((z_row_l, z_index_l), (a, b)) for (a, b) = 00, 01, 10, 11 (shared by all columns)
struct BpMat { Ext ri[4], cc[4]; };
__device__ __forceinline__ void bp_layer_coeffs(const uint32_t* __restrict__ ri_eq, uint32_t layer, uint32_t hl, const Ext& cur, const Ext& nxt, BpMat& m) {
    if (layer < hl) {
        const uint32_t* e = ri_eq + (size_t)layer * 16;
        m.ri[0] = kb::ext_load(e); m.ri[1] = kb::ext_load(e + 4); m.ri[2] = kb::ext_load(e + 8); m.ri[3] = kb::ext_load(e + 12);
    } else { m.ri[0] = kb::ext_one(); m.ri[1] = m.ri[2] = m.ri[3] = kb::ext_zero(); }
    const Ext cn = kb::ext_mul(cur, nxt);
    m.cc[3] = cn; m.cc[2] = kb::ext_sub(cur, cn); m.cc[1] = kb::ext_sub(nxt, cn);
    m.cc[0] = kb::ext_sub(kb::ext_sub(kb::ext_one(), cur), m.cc[1]);
}
// out = M res   (column form)
__device__ __forceinline__ void bp_apply(const BpMat& m, const Ext res[4], Ext out[4]) {
#pragma unroll
    for (int st = 0; st < 4; st++) {
        Ext acc = kb::ext_zero();
#pragma unroll
        for (int a = 0; a < 4; a++) {
            Ext inner = kb::ext_zero();
            bool any = false;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                int o = bp_transition(a >> 1, a & 1, c >> 1, c & 1, st);
                if (o >= 0) { inner = kb::ext_add(inner, kb::ext_mul(m.cc[c], res[o])); any = true; }
            }
            if (any) acc = kb::ext_add(acc, kb::ext_mul(m.ri[a], inner));
        }
        out[st] = acc;
    }
}
// out = P M   (row form)
__device__ __forceinline__ void bp_apply_row(const BpMat& m, const Ext P[4], Ext out[4]) {
    Ext o4[4] = {kb::ext_zero(), kb::ext_zero(), kb::ext_zero(), kb::ext_zero()};
#pragma unroll
    for (int st = 0; st < 4; st++)
#pragma unroll
        for (int a = 0; a < 4; a++) {
            const Ext q = kb::ext_mul(P[st], m.ri[a]);
#pragma unroll
            for (int c = 0; c < 4; c++) {
                int o = bp_transition(a >> 1, a & 1, c >> 1, c & 1, st);
                if (o >= 0) o4[o] = kb::ext_add(o4[o], kb::ext_mul(q, m.cc[c]));
            }
        }
#pragma unroll
    for (int i = 0; i < 4; i++) out[i] = o4[i];
}
__device__ __forceinline__ Ext bp_bit(const uint8_t* b, uint32_t pos) { return b[pos] ? kb::ext_one() : kb::ext_zero(); }

// T[(l * nk + k) * 4 + s], l = hl+1 .. 0.  second_half: next-coordinates are the bound values rho_by_pos[dim-1-l]
__global__ void __launch_bounds__(128) bp_suffix_kernel(const uint8_t* __restrict__ bits, uint32_t nk, uint32_t dim, int second_half,
                                                        const uint32_t* __restrict__ rho_by_pos, const uint32_t* __restrict__ ri_eq,
                                                        uint32_t* __restrict__ T) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nk) return;
    const uint32_t hl = dim / 2;
    const uint8_t* b = bits + (size_t)k * dim;
    Ext res[4] = {kb::ext_zero(), kb::ext_zero(), kb::ext_one(), kb::ext_zero()};
    for (int s = 0; s < 4; s++) kb::ext_store(T + (((size_t)(hl + 1) * nk + k) * 4 + s) * 4, res[s]);
    for (int layer = (int)hl; layer >= 0; layer--) {
        Ext cur = kb::ext_zero(), nxt = kb::ext_zero();
        if ((uint32_t)layer < hl) {
            cur = bp_bit(b, hl - 1 - layer);
            nxt = second_half ? kb::ext_load(rho_by_pos + 4 * (dim - 1 - layer)) : bp_bit(b, dim - 1 - layer);
        }
        BpMat m;
        bp_layer_coeffs(ri_eq, (uint32_t)layer, hl, cur, nxt, m);
        Ext nres[4];
        bp_apply(m, res, nres);
        for (int s = 0; s < 4; s++) { res[s] = nres[s]; kb::ext_store(T + (((size_t)layer * nk + k) * 4 + s) * 4, res[s]); }
    }
}
// round r: thread (k, node) -> zc[k] * inter[k] * eq(lambda, bit) * P_k . M_layer(lambda_node) . T_k[layer+1]
__global__ void __launch_bounds__(128) bp_round_kernel(const uint8_t* __restrict__ bits, uint32_t nk, uint32_t dim, uint32_t round,
                                                       const uint32_t* __restrict__ rho_by_pos, const uint32_t* __restrict__ ri_eq,
                                                       const uint32_t* __restrict__ zc, const uint32_t* __restrict__ inter,
                                                       const uint32_t* __restrict__ P, const uint32_t* __restrict__ T, Ext half,
                                                       uint32_t* __restrict__ partial, Mail mail) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    Ext v = kb::ext_zero();
    const uint32_t k = t >> 1, node = t & 1;
    const uint32_t hl = dim / 2, split = dim - round - 1;
    if (k < nk) {
        const uint8_t* b = bits + (size_t)k * dim;
        const bool second = round >= hl;
        const uint32_t layer = second ? round - hl : round;
        const Ext lam = node ? half : kb::ext_zero();
        const Ext cur = second ? lam : bp_bit(b, hl - 1 - layer);
        const Ext nxt = second ? kb::ext_load(rho_by_pos + 4 * (dim - 1 - layer)) : lam;
        BpMat m;
        bp_layer_coeffs(ri_eq, layer, hl, cur, nxt, m);
        Ext res[4], w[4];
        for (int s = 0; s < 4; s++) res[s] = kb::ext_load(T + (((size_t)(layer + 1) * nk + k) * 4 + s) * 4);
        bp_apply(m, res, w);
        Ext val = kb::ext_zero();
        if (round == 0 || round == hl) val = w[0];  // P_k = e0^T at the start of either half (bp_update_kernel resets it after this round)
        else
            for (int s = 0; s < 4; s++) val = kb::ext_add(val, kb::ext_mul(kb::ext_load(P + ((size_t)k * 4 + s) * 4), w[s]));
        const Ext eqv = node ? half : (b[split] ? kb::ext_zero() : kb::ext_one());
        v = kb::ext_mul(kb::ext_mul(kb::ext_load(zc + 4 * k), val), kb::ext_mul(kb::ext_load(inter + 4 * k), eqv));
    }
    // node 0 -> y_0, node 1 -> y_half: partial[block] = (y_0 limbs, y_half limbs)
    block_reduce<2>({node ? kb::ext_zero() : v, node ? v : kb::ext_zero()}, partial, mail);
}
// after round r's challenge: bind position split = dim-1-r: rho_by_pos, inter[k] *= eq(alpha, bit), P_k <- P_k M_layer(bound)
// (at the switch to the second half P_k restarts at e0^T: the caller rebuilds T with the bound next-coordinates first)
__global__ void __launch_bounds__(128) bp_update_kernel(const uint8_t* __restrict__ bits, uint32_t nk, uint32_t dim, uint32_t round, Ext alpha,
                                                        uint32_t* __restrict__ rho_by_pos, const uint32_t* __restrict__ ri_eq,
                                                        uint32_t* __restrict__ inter, uint32_t* __restrict__ P) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t hl = dim / 2, split = dim - round - 1;
    if (k == 0) kb::ext_store(rho_by_pos + 4 * split, alpha);
    if (k >= nk) return;
    const uint8_t* b = bits + (size_t)k * dim;
    const Ext f = b[split] ? alpha : kb::ext_sub(kb::ext_one(), alpha);
    kb::ext_store(inter + 4 * k, kb::ext_mul(kb::ext_load(inter + 4 * k), f));
    const bool second = round >= hl;
    const uint32_t layer = second ? round - hl : round;
    Ext Pk[4], out[4];
    for (int s = 0; s < 4; s++) Pk[s] = kb::ext_load(P + ((size_t)k * 4 + s) * 4);
    if (round == hl) { Pk[0] = kb::ext_one(); Pk[1] = Pk[2] = Pk[3] = kb::ext_zero(); }
    const Ext cur = second ? alpha : bp_bit(b, hl - 1 - layer);
    // second half: the next-coordinate of this layer was bound in round `layer` (written before this kernel ran)
    const Ext nxt = second ? kb::ext_load(rho_by_pos + 4 * (dim - 1 - layer)) : alpha;
    BpMat m;
    bp_layer_coeffs(ri_eq, layer, hl, cur, nxt, m);
    bp_apply_row(m, Pk, out);
    for (int s = 0; s < 4; s++) kb::ext_store(P + ((size_t)k * 4 + s) * 4, out[s]);
}

// p(x) through (0, y0), (1, y1), (1/2, yh): coefficients c0, c1, c2
inline void interp_0_1_half(const E4& y0, const E4& y1, const E4& yh, E4 c[3]) {
    const uint32_t two = kb::to_monty_c(2), three = kb::to_monty_c(3), four = kb::to_monty_c(4);
    c[0] = y0;
    c[1] = yh * four - y0 * three - y1;
    c[2] = (y1 + y0) * two - yh * four;
}
inline E4 eval3(const E4 c[3], const E4& x) { return (c[2] * x + c[1]) * x + c[0]; }

}  // namespace

extern "C" {

// Jagged commit of one round of chip tables (slop/crates/jagged/src/prover.rs:106-160).
// dense_any: the tables' real cells back to back, each table column-major [cols x rows] (tables with 0 rows
// contribute nothing), host or device; the library keeps its own zero-padded device copy.
sp1b200_err sp1b200_jagged_commit(sp1b200_ctx* ctx, const uint32_t* dense_any, uint32_t n_tables, const uint64_t* rows, const uint64_t* cols,
                                  int keep_codeword, uint32_t* h_commit8, sp1b200_jagged_round** out) { SP1_DEVICE_GUARD(ctx);
    const uint32_t ls = ctx->params.log_stacking_height, mlr = ctx->params.max_log_row_count;
    auto r = std::make_unique<sp1b200_jagged_round>();
    uint64_t area = 0;
    for (uint32_t t = 0; t < n_tables; t++) {
        if (rows[t] > ((uint64_t)1 << mlr)) return sp1b200_set_error("jagged_commit: table %u has %llu rows > 2^%u", t, (unsigned long long)rows[t], mlr);
        r->tables.emplace_back(rows[t], cols[t]); area += rows[t] * cols[t];
    }
    const uint64_t padded = layout::stacked_columns(area, ls) << ls;
    const uint64_t added = padded - area;
    r->area = area; r->padded_area = padded;
    SP1_CUDA(cudaMallocFromPoolAsync((void**)&r->d_dense, padded * 4, ctx->pool, ctx->stream));
    const int up_slot = sp1b200_upload_acquire(ctx, dense_any);  // dense_any may be an upload slot still being filled
    cudaError_t ce = area ? cudaMemcpyAsync(r->d_dense, dense_any, area * 4, cudaMemcpyDefault, ctx->stream) : cudaSuccess;
    sp1b200_upload_release(ctx, up_slot);                        // the slot is free once this copy has run
    if (ce == cudaSuccess && added) ce = cudaMemsetAsync(r->d_dense + area, 0, added * 4, ctx->stream);
    sp1b200_err e = ce == cudaSuccess ? sp1b200_stacked_commit(ctx, r->d_dense, padded >> ls, keep_codeword, r->original_commit, &r->stacked)
                                      : sp1b200_set_error("jagged_commit: copying the dense trace: %s", cudaGetErrorString(ce));
    if (e) { cudaFreeAsync(r->d_dense, ctx->stream); r->d_dense = nullptr; return e; }
    const layout::Tables pad = layout::padding_tables(area, ls, mlr);
    r->tables.insert(r->tables.end(), pad.begin(), pad.end());
    table_size_commitment(r->original_commit, r->tables, r->commit);
    if (h_commit8) memcpy(h_commit8, r->commit, 32);
    *out = r.release();
    return nullptr;
}

void sp1b200_jagged_round_free(sp1b200_ctx* ctx, sp1b200_jagged_round* r) { SP1_DEVICE_GUARD(ctx);
    if (!r) return;
    sp1b200_commit_free(ctx, r->stacked);
    if (r->d_dense) cudaFreeAsync(r->d_dense, ctx->stream);
    delete r;
}

// Per-column evaluations of every table column of the round at z_row (zero-padded to 2^max_log_row_count rows):
// the claims zerocheck hands to the PCS (crates/hypercube/src/prover/shard.rs:736-767).  h_out: sum(cols) ext elements.
sp1b200_err sp1b200_jagged_column_claims(sp1b200_ctx* ctx, const sp1b200_jagged_round* r, const uint32_t* h_z_row, uint32_t* h_out) { SP1_DEVICE_GUARD(ctx);
    const uint32_t mlr = ctx->params.max_log_row_count;
    DevFree mem(ctx);
    uint32_t *d_z, *d_eq, *d_out;
    std::vector<EvalTable> tabs;  // the round's tables without the two padding tables
    uint64_t off = 0;
    uint32_t nc = 0;
    for (size_t t = 0; t + 2 < r->tables.size(); t++) {
        const auto& [rows, cols] = r->tables[t];
        tabs.push_back(EvalTable{r->d_dense + off, rows, (uint32_t)cols, nc});
        off += rows * cols; nc += (uint32_t)cols;
    }
    if (!nc) return nullptr;
    SP1_TRY(mem.alloc((void**)&d_z, mlr * 16));
    SP1_TRY(mem.alloc((void**)&d_eq, ((size_t)16) << mlr));
    SP1_TRY(mem.alloc((void**)&d_out, (size_t)nc * 16));
    SP1_CUDA(cudaMemcpyAsync(d_z, h_z_row, mlr * 16, cudaMemcpyHostToDevice, ctx->stream));
    SP1_TRY(launch_eq_table(ctx, d_z, (int)mlr, d_eq));
    SP1_TRY(launch_table_evals(ctx, tabs, d_eq, d_out, nc));
    SP1_CUDA(cudaMemcpyAsync(h_out, d_out, (size_t)nc * 16, cudaMemcpyDeviceToHost, ctx->stream));
    SP1_CUDA(cudaStreamSynchronize(ctx->stream));
    return nullptr;
}

// JaggedProver::prove_trusted_evaluations (slop/crates/jagged/src/prover.rs:162-328).
// h_claims: for each round, the evaluations at z_row of that round's table columns (ext each), back to back.
// Proof words: the evaluation proof section of a shard proof (proof_layout.hpp), the stacked proof first
// (field order of JaggedPcsProof, slop/crates/jagged/src/verifier.rs:17-27).
sp1b200_err sp1b200_jagged_prove(sp1b200_ctx* ctx, sp1b200_jagged_round* const* rounds, uint32_t n_rounds, const uint32_t* h_z_row,
                                 const uint32_t* h_claims, const uint32_t* h_replay, uint32_t* h_chal, uint32_t* h_proof, uint64_t cap,
                                 uint64_t* h_words) { SP1_DEVICE_GUARD(ctx);
    if (!n_rounds || n_rounds > 8) return sp1b200_set_error("jagged_prove: 1..8 rounds supported");
    const uint32_t mlr = ctx->params.max_log_row_count, ls = ctx->params.log_stacking_height;
    cudaStream_t st = ctx->stream;
    DevFree mem(ctx);
    HostChallenger ch;
    SP1_TRY(ch.init(ctx, h_chal));
    PhaseTimer t_all(ctx, "jagged.total");

    // column prefix sums over all rounds (padding tables included)
    std::vector<uint64_t> prefix{0};
    for (uint32_t r = 0; r < n_rounds; r++) layout::append_column_prefix(prefix, rounds[r]->tables);
    const uint64_t total_cols = prefix.size() - 1;
    const uint32_t lm = hf::log2_ceil(prefix.back());
    if (lm < ls) return sp1b200_set_error("jagged_prove: internal: log_m < log_stacking_height");
    if (lm < 2) return sp1b200_set_error("jagged_prove: fewer than two sumcheck variables (log_m = %u)", lm);
    const uint64_t N = (uint64_t)1 << lm;
    const uint32_t ncv = hf::log2_ceil(total_cols);
    std::vector<E4> z_col(ncv), z_row(mlr);
    for (auto& x : z_col) ch.sample_ext(x.c);
    for (uint32_t i = 0; i < mlr; i++) z_row[i] = E4::load(h_z_row + 4 * i);

    // column claims with zeros for the padding columns; sumcheck claim = MLE(column_claims)(z_col)
    std::vector<E4> column_claims;
    {
        size_t k = 0;
        for (uint32_t r = 0; r < n_rounds; r++) {
            const layout::Tables& tb = rounds[r]->tables;
            for (size_t t = 0; t < tb.size(); t++)
                for (uint64_t c = 0; c < tb[t].second; c++) column_claims.push_back(t + 2 < tb.size() ? E4::load(h_claims + 4 * (k++)) : E4());
        }
    }
    const E4 claim = hf::mle_eval(column_claims, z_col);
    std::vector<E4> col_eq_full = hf::partial_lagrange(z_col);

    // K = the rounds summed straight from the base-field trace (see jagged_round_kernel): every aligned 2^K block must lie in one
    // column (2^K divides every prefix sum), in one segment (K <= log_stacking_height) and in one run of 2^lb rows (K <= lb); round
    // K must still exist (K <= log_m - 1).  K = 0 (odd column starts): no trace rounds, round 0 comes from the fold pass.
    const int lb = (int)std::min<uint32_t>(JK_LOW, mlr);
    uint32_t K = std::min<uint32_t>({(uint32_t)JK_MAX, ls, lm - 1, (uint32_t)lb});
    for (uint64_t p : prefix)
        if (p) K = std::min<uint32_t>(K, (uint32_t)__builtin_ctzll(p));
    const uint64_t area = prefix.back();

    // device tables: col_eq (over last log2_ceil(ncols) coords of z_col == all of z_col), the row eq factors, prefix sums
    uint32_t *d_coleq, *d_zrow, *d_eqhi, *d_eqlo, *d_ext, *d_ext2, *d_b, *d_b2, *d_partial;
    uint64_t* d_prefix;
    SP1_TRY(mem.alloc((void**)&d_coleq, col_eq_full.size() * 16));
    SP1_CUDA(cudaMemcpyAsync(d_coleq, col_eq_full.data(), col_eq_full.size() * 16, cudaMemcpyHostToDevice, st));
    SP1_TRY(mem.alloc((void**)&d_zrow, mlr * 16));
    SP1_CUDA(cudaMemcpyAsync(d_zrow, h_z_row, mlr * 16, cudaMemcpyHostToDevice, st));
    // row_eq = eq_hi (x) eq_lo: z_row[0 .. mlr-lb) is the high (most significant) part
    SP1_TRY(mem.alloc((void**)&d_eqhi, ((size_t)16) << (mlr - lb)));
    SP1_TRY(mem.alloc((void**)&d_eqlo, ((size_t)16) << lb));
    SP1_TRY(launch_eq_table(ctx, d_zrow, (int)(mlr - lb), d_eqhi));
    SP1_TRY(launch_eq_table(ctx, d_zrow + 4 * (mlr - lb), lb, d_eqlo));
    SP1_TRY(mem.alloc((void**)&d_prefix, prefix.size() * 8));
    SP1_CUDA(cudaMemcpyAsync(d_prefix, prefix.data(), prefix.size() * 8, cudaMemcpyHostToDevice, st));
    // start[b] = last column with prefix <= b << JP_SHIFT (two-pointer walk over the blocks of the real area)
    std::vector<uint32_t> jp_start((size_t)((area >> JP_SHIFT) + 1));
    {
        uint32_t c = 0;
        for (size_t b = 0; b < jp_start.size(); b++) {
            const uint64_t i0 = (uint64_t)b << JP_SHIFT;
            while (c + 1 < total_cols && prefix[c + 1] <= i0) c++;
            jp_start[b] = c;
        }
    }
    uint32_t* d_jp_start;
    SP1_TRY(mem.alloc((void**)&d_jp_start, jp_start.size() * 4));
    SP1_CUDA(cudaMemcpyAsync(d_jp_start, jp_start.data(), jp_start.size() * 4, cudaMemcpyHostToDevice, st));
    // working arrays: level K (written by the fold pass to level K) and level K+1; later levels reuse them in turn
    SP1_TRY(mem.alloc((void**)&d_b, (N >> K) * 16));
    SP1_TRY(mem.alloc((void**)&d_ext, (N >> K) * 16));
    SP1_TRY(mem.alloc((void**)&d_b2, ((N >> (K + 1)) + 1) * 16));
    SP1_TRY(mem.alloc((void**)&d_ext2, ((N >> (K + 1)) + 1) * 16));
    const unsigned MAXB = 132 * 8;  // eight blocks per SM of an H100
    static_assert(132 * 8 * 8 + 16 <= SP1_MAIL_WORDS, "round partials must fit the mailbox payload");
    d_partial = sp1b200_mail_dev(ctx);  // the round kernels post their block partials straight into the mailbox
    SegTable seg{};
    seg.n = (int)n_rounds;
    { uint64_t e = 0; for (uint32_t r = 0; r < n_rounds; r++) { seg.ptr[r] = rounds[r]->d_dense; e += rounds[r]->padded_area; seg.end[r] = e; } }

    // ---- Hadamard sumcheck (lambda = 1, t = 1) ---------------------------------------------------------------------
    layout::SumcheckWriter sc;
    std::vector<E4> point;              // most recent challenge first
    E4 round_claim = claim;
    PhaseTimer t_sc(ctx, "jagged.sumcheck");
    auto grid_for = [&](uint64_t n) { unsigned g = blocks_for(n); return g > MAXB ? MAXB : (g ? g : 1u); };
    std::vector<E4> w{E4::one()};  // w_r (see jagged_round_kernel): the weights of the 2^r trace words behind one level-r entry
    JWeights dw{};
    auto load_weights = [&]() { for (size_t t = 0; t < w.size(); t++) for (int l = 0; l < 4; l++) dw.w[t].c[l] = w[t].c[l]; };
    // the sums of round r come from jagged_round_kernel<r> when r < K, from jagged_fold_to_kernel<K> (which writes level K) when
    // r == K, and from hadamard_fold_kernel fixing alpha_{r-1} when r > K (r = log_m: the last fold, for the dense evaluation)
    uint32_t *cur_b = d_b, *cur_e = d_ext, *nxt_b = d_b2, *nxt_e = d_ext2;
    auto launch_sums = [&](uint32_t r, const Ext& alpha, const Mail& mail, unsigned& g) -> sp1b200_err {
        if (r < K) {  // contiguous span of blocks per warp (multiple of 32), over the real area only
            const uint64_t nblk = area >> (r + 1);
            g = grid_for(nblk);
            const uint64_t warps = (uint64_t)g * 8, span = std::max<uint64_t>((((nblk + warps - 1) / warps) + 31) / 32 * 32, 32);
#define SP1_JROUND(k) case k: SP1_LAUNCH(ctx, jagged_round_kernel<k>, g, 256, 0, seg, d_prefix, (uint32_t)total_cols, d_jp_start, d_coleq, \
                                         d_eqhi, d_eqlo, lb, dw, nblk, span, d_partial, mail); break;
            switch (r) { SP1_JROUND(0) SP1_JROUND(1) SP1_JROUND(2) SP1_JROUND(3) SP1_JROUND(4)
                         default: return sp1b200_set_error("jagged_prove: internal: trace round %u", r); }
#undef SP1_JROUND
            static_assert(JK_MAX == 5, "one jagged_round_kernel instance per round below JK_MAX");
        } else if (r == K) {
            const uint64_t nout = N >> K, nout_pairs = nout / 2;
            g = grid_for(nout_pairs);
#define SP1_JFOLD(k) case k: SP1_LAUNCH(ctx, jagged_fold_to_kernel<k>, g, 256, 0, seg, d_prefix, (uint32_t)total_cols, d_jp_start, d_coleq, \
                                        d_eqhi, d_eqlo, lb, dw, area, nout_pairs, cur_b, cur_e, d_partial, nout, mail); break;
            switch (K) { SP1_JFOLD(0) SP1_JFOLD(1) SP1_JFOLD(2) SP1_JFOLD(3) SP1_JFOLD(4) SP1_JFOLD(5)
                         default: return sp1b200_set_error("jagged_prove: internal: fold to level %u", K); }
#undef SP1_JFOLD
        } else {
            const uint64_t nout = N >> r;
            g = grid_for((nout + 1) / 2);
            SP1_LAUNCH(ctx, hadamard_fold_kernel, g, 256, 0, cur_b, cur_e, (nout + 1) / 2, alpha, nxt_b, nxt_e, d_partial, nout, mail);
            std::swap(cur_b, nxt_b); std::swap(cur_e, nxt_e);
        }
        return nullptr;
    };
    unsigned prev_g;
    const Mail first = sp1b200_mail_next(ctx);
    uint32_t prev_seq = first.seq;
    load_weights();
    SP1_TRY(launch_sums(0, Ext{}, first, prev_g));
    for (uint32_t rd = 0; rd < lm; rd++) {
        E4 s2[2];  // eval_0, eval_half, accumulated by the previous launch
        E4 &e0 = s2[0], &eh = s2[1];
        SP1_TRY(sum_mail_partials(ctx, prev_seq, prev_g, s2));
        E4 e1 = round_claim - e0;
        E4 c[3];
        interp_0_1_half(e0, e1, eh * kb::inv(kb::to_monty_c(4)), c);
        for (int i = 0; i < 3; i++) ch.observe_n(c[i].c, 4);
        sc.poly(c, 3);
        E4 alpha; ch.sample_ext(alpha.c);
        point.insert(point.begin(), alpha);
        round_claim = eval3(c, alpha);
        // fix the variable; the same launch accumulates the next round's sums (unless this was the last round)
        const Mail mail = sp1b200_mail_next(ctx); prev_seq = mail.seq;
        if (rd < K) {  // w_{rd+1}[t] = w_rd[t mod 2^rd] * (bit rd of t ? alpha : 1 - alpha)
            const size_t m = w.size();
            w.resize(2 * m);
            for (size_t t = 0; t < m; t++) { w[m + t] = w[t] * alpha; w[t] = w[t] * (E4::one() - alpha); }
            load_weights();
        }
        SP1_TRY(launch_sums(rd + 1, alpha, mail, prev_g));
    }
    // component evaluations: base[0] (the dense trace at the sumcheck point), ext[0]
    // (posted by the last fold launch next to its, unused, partial sums: payload EF slot 2)
    SP1_TRY(sp1b200_mail_wait(ctx, prev_seq));
    const E4 base_eval = E4::load(sp1b200_mail_host(ctx) + 8);
    t_sc.stop();

    // ---- jagged evaluation (branching program) sumcheck --------------------------------------------------------------
    layout::SumcheckWriter je;
    std::vector<E4> rhos;
    E4 je_claimed, je_eval;
    {
        PhaseTimer t(ctx, "jagged.eval_sumcheck");
        const uint32_t dim = 2 * (lm + 1);
        // merged prefix sums (bits), condensed over equal consecutive entries; z_col eq values summed per group
        std::vector<uint8_t> bits;
        std::vector<E4> zc;
        uint32_t nk = 0;
        for (size_t c = 0; c + 1 < prefix.size(); c++) {
            std::vector<uint8_t> b(dim);
            for (uint32_t i = 0; i <= lm; i++) { b[i] = (prefix[c] >> (lm - i)) & 1; b[lm + 1 + i] = (prefix[c + 1] >> (lm - i)) & 1; }
            if (nk && std::equal(b.begin(), b.end(), bits.end() - dim)) zc.back() = zc.back() + col_eq_full[c];
            else { bits.insert(bits.end(), b.begin(), b.end()); zc.push_back(col_eq_full[c]); nk++; }
        }
        // per-layer eq((z_row_l, z_index_l), .) ; z_index = the sumcheck point (lm coords), num_vars = max(mlr, lm) -> lm+1 layers used
        const uint32_t hl = lm + 1;
        std::vector<uint32_t> ri((size_t)hl * 16);
        auto lsb = [](const std::vector<E4>& p, uint32_t i) { return p.size() <= i ? E4() : p[p.size() - 1 - i]; };
        if (mlr > hl) return sp1b200_set_error("jagged_prove: max_log_row_count %u exceeds log_m+1 = %u (unsupported shape)", mlr, hl);
        for (uint32_t l = 0; l < hl; l++) {
            E4 zr = lsb(z_row, l), zi = lsb(point, l), one = E4::one();
            E4 p = zr * zi;
            E4 e11 = p, e10 = zr - p, e01 = zi - p, e00 = one - zr - e01;
            e00.store(&ri[l * 16]); e01.store(&ri[l * 16 + 4]); e10.store(&ri[l * 16 + 8]); e11.store(&ri[l * 16 + 12]);
        }
        uint8_t* d_bits; uint32_t *d_ri, *d_zc, *d_inter, *d_part;
        SP1_TRY(mem.alloc((void**)&d_bits, bits.size()));
        SP1_TRY(mem.alloc((void**)&d_ri, ri.size() * 4));
        SP1_TRY(mem.alloc((void**)&d_zc, (size_t)nk * 16));
        SP1_TRY(mem.alloc((void**)&d_inter, (size_t)nk * 16));
        const unsigned nblk = (2 * nk + 127) / 128;
        SP1_TRY(mem.alloc((void**)&d_part, (size_t)nblk * 32));
        SP1_CUDA(cudaMemcpyAsync(d_bits, bits.data(), bits.size(), cudaMemcpyHostToDevice, st));
        SP1_CUDA(cudaMemcpyAsync(d_ri, ri.data(), ri.size() * 4, cudaMemcpyHostToDevice, st));
        SP1_CUDA(cudaMemcpyAsync(d_zc, zc.data(), (size_t)nk * 16, cudaMemcpyHostToDevice, st));
        std::vector<E4> ones(nk, E4::one());
        SP1_CUDA(cudaMemcpyAsync(d_inter, ones.data(), (size_t)nk * 16, cudaMemcpyHostToDevice, st));
        const Ext dhalf = kb::ext_from_base(kb::inv(kb::to_monty_c(2)));
        // prefix / suffix states (see bp_suffix_kernel): T for the first half now, rebuilt once when the second half starts
        uint32_t *d_T, *d_P, *d_rho_pos;
        SP1_TRY(mem.alloc((void**)&d_T, (size_t)(hl + 2) * nk * 64));
        SP1_TRY(mem.alloc((void**)&d_P, (size_t)nk * 64));
        SP1_TRY(mem.alloc((void**)&d_rho_pos, (size_t)dim * 16));
        {
            std::vector<E4> p0((size_t)nk * 4);
            for (uint32_t k = 0; k < nk; k++) p0[4 * k] = E4::one();
            SP1_CUDA(cudaMemcpyAsync(d_P, p0.data(), p0.size() * 16, cudaMemcpyHostToDevice, st));
            SP1_CUDA(cudaMemsetAsync(d_rho_pos, 0, (size_t)dim * 16, st));
        }
        SP1_LAUNCH(ctx, bp_suffix_kernel, blocks_for(nk, 128), 128, 0, d_bits, nk, dim, 0, d_rho_pos, d_ri, d_T);
        // claimed sum = full evaluation at the boolean prefix sums (full_jagged_little_polynomial_evaluation, poly.rs:183-232):
        // the first-half suffix table at layer 0 holds it per column, je_claimed = sum_k zc[k] T_k[0][state 0]
        {
            std::vector<E4> t0((size_t)nk * 4);  // layer 0 of T: [nk][4 states]
            SP1_CUDA(cudaMemcpyAsync(t0.data(), d_T, t0.size() * 16, cudaMemcpyDeviceToHost, st));
            SP1_CUDA(cudaStreamSynchronize(st));
            for (uint32_t k = 0; k < nk; k++) je_claimed = je_claimed + zc[k] * t0[4 * k];
        }
        ch.observe_n(je_claimed.c, 4);
        E4 cl = je_claimed;
        const bool bp_mail = (size_t)nblk * 8 <= SP1_MAIL_WORDS;  // otherwise fall back to copy + synchronise
        for (uint32_t round = 0; round < dim; round++) {
            if (round == hl) SP1_LAUNCH(ctx, bp_suffix_kernel, blocks_for(nk, 128), 128, 0, d_bits, nk, dim, 1, d_rho_pos, d_ri, d_T);
            const Mail mail = sp1b200_mail_next(ctx);
            SP1_LAUNCH(ctx, bp_round_kernel, nblk, 128, 0, d_bits, nk, dim, round, d_rho_pos, d_ri, d_zc, d_inter, d_P, d_T, dhalf,
                       bp_mail ? sp1b200_mail_dev(ctx) : d_part, bp_mail ? mail : Mail{nullptr, nullptr, 0});
            E4 y[2];
            if (bp_mail) SP1_TRY(sum_mail_partials(ctx, mail.seq, nblk, y));
            else SP1_TRY(sum_device_partials(ctx, d_part, nblk, y));
            const E4 &y0 = y[0], &yh = y[1];
            E4 y1 = cl - y0;
            E4 c[3];
            interp_0_1_half(y0, y1, yh, c);
            for (int i = 0; i < 3; i++) ch.observe_n(c[i].c, 4);
            je.poly(c, 3);
            E4 alpha; ch.sample_ext(alpha.c);
            rhos.insert(rhos.begin(), alpha);
            cl = eval3(c, alpha);
            SP1_LAUNCH(ctx, bp_update_kernel, blocks_for(nk, 128), 128, 0, d_bits, nk, dim, round, alpha, d_rho_pos, d_ri, d_inter, d_P);
        }
        je_eval = cl;
        t.stop();
    }

    // ---- dense PCS: prove_untrusted_evaluation(point, base_eval) ---------------------------------------------------
    ch.observe_n(base_eval.c, 4);
    uint32_t chal[34];
    ch.store(chal);
    std::vector<sp1b200_commit*> handles;
    for (uint32_t r = 0; r < n_rounds; r++) handles.push_back(rounds[r]->stacked);
    std::vector<uint32_t> pt(point.size() * 4);
    for (size_t i = 0; i < point.size(); i++) point[i].store(&pt[4 * i]);
    // the stacked proof is written straight into the caller's buffer; the jagged sections are appended after it
    uint64_t nw = 0;
    SP1_TRY(sp1b200_stacked_prove(ctx, handles.data(), n_rounds, pt.data(), (uint32_t)point.size(), h_replay, chal, h_proof, cap, &nw));
    layout::FlatWriter proof;
    sc.write(proof, claim, point.data(), round_claim);
    je.write(proof, je_claimed, rhos.data(), je_eval);
    for (uint32_t r = 0; r < n_rounds; r++) layout::write_tables(proof, rounds[r]->tables);
    for (uint32_t r = 0; r < n_rounds; r++) proof.put(rounds[r]->original_commit, 8);
    proof.ext(base_eval);
    proof.u(mlr);
    proof.u(lm);
    t_all.stop();
    memcpy(h_chal, chal, sizeof(chal));
    return layout::deliver("jagged_prove", "proof", proof.words, h_proof, cap, h_words, nw);
}

}  // extern "C"
