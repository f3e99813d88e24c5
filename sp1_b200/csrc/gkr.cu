// LogUp-GKR on the device.
// Reference behaviour: crates/hypercube/src/logup_gkr/{prover.rs:70-215, execution.rs:13-382, logup_poly.rs:71-552, cpu.rs:76-226};
// GPU twin it replaces: sp1-gpu/crates/logup_gkr + sys/lib/logup_gkr/{first_layer,execution,round,lookahead}.cu.
// HOW (results identical):
//  * the circuit is kept as ONE fraction sequence per (chip, interaction) and level, F_l[j] (numerator EF, denominator EF;
//    level 0 keeps its numerators, the multiplicities, in the base field: 20 B per entry instead of 32),
//    F_{l+1}[j] = F_l[2j] (+) F_l[2j+1]; the reference's four arrays of a layer are the parity classes of F_l
//    (numerator_0 = even entries, numerator_1 = odd entries), so no transposition or re-layout is needed between levels;
//    levels 0, 1 and 2 come out of one pass over the trace;
//  * every sumcheck round of a layer is one launch over ALL chips (work items are looked up in a small prefix table);
//    rounds 0 and 1 are summed in one pass over the fraction sequence and fixed together in a second one, the later row
//    rounds are fused as "fix the previous variable + accumulate the next round's three sums";
//  * once a layer's row variables are exhausted the remaining (interaction) variables range over <= 2^v <= a few
//    thousand values, which the host transcript driver folds directly.
#include "ctx.cuh"
#include "challenger.cuh"
#include "debug_fp.cuh"
#include "hostfield.hpp"
#include "kb31.cuh"
#include "proof_layout.hpp"
#include "sumcheck.cuh"
#include <algorithm>
#include <map>
#include <memory>
#include <vector>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/discard_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "machine.cuh"

namespace {

using kb::Ext;
using hf::E4;

struct ChipJob {           // one chip inside a batched launch
    uint64_t work_start;   // prefix of work items
    uint64_t in_off, out_off;  // element offsets of the chip's arrays in the in / out arenas
    uint32_t rows_in;      // rows (or sequence length) of the input arrays
    uint32_t I;            // interactions of the chip
    uint32_t int_off;      // offset into eq_interaction
    uint32_t pad;
};
constexpr int MAX_JOBS = 96;  // 96 * 40 B + 16 B < 4 KB of kernel parameters
struct JobTable { ChipJob j[MAX_JOBS]; uint32_t n; uint64_t total; };

__device__ __forceinline__ int find_job(const JobTable& t, uint64_t w) {
    int lo = 0, hi = (int)t.n;  // j[lo].work_start <= w < j[hi].work_start (hi = n: total)
    while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (t.j[mid].work_start <= w) lo = mid; else hi = mid; }
    return lo;
}

__device__ __forceinline__ Ext ldE(const uint32_t* p, uint64_t i) { return kb::ext_load(p + 4 * i); }
__device__ __forceinline__ void stE(uint32_t* p, uint64_t i, const Ext& e) { kb::ext_store(p + 4 * i, e); }

// ---- levels 0 and 1: per (chip, interaction k, row r) fraction from the trace (execution.rs:13-36, 114-252) -----------------
// q = a / b for work indices that almost always fit 32 bits: the 64-bit division (~60 instructions) only when needed
__device__ __forceinline__ uint32_t div_small(uint64_t a, uint64_t b) {
    return ((a | b) >> 32) ? (uint32_t)(a / b) : (uint32_t)a / (uint32_t)b;
}

struct FirstSrc { const uint32_t* main; const uint32_t* prep; uint64_t off2; };  // a job's trace columns, its offset at level 2

__device__ __forceinline__ void frac_add(const Ext& n0, const Ext& d0, const Ext& n1, const Ext& d1, Ext& n, Ext& d) {
    n = kb::ext_add(kb::ext_mul(d1, n0), kb::ext_mul(d0, n1));
    d = kb::ext_mul(d0, d1);
}

// Level 0 keeps its numerators (the multiplicities) in the base field: num0 = u32 words, den0 = EF.  A thread computes the
// entries 4j .. 4j+3 of one (chip, k) sequence and stores them, which the layer-0 sumcheck reads, together with entries 2j, 2j+1
// of level 1 and entry j of level 2 (num2 = nullptr: the tree has two levels).  A missing odd entry is the padding (0,1): the
// even entry passes up unchanged.  work item = (chip, k, j), all chips in one launch; job.int_off doubles as the chip's first
// entry in `inter`.
__global__ void __launch_bounds__(256) gkr_first_level_kernel(JobTable jobs, const FirstSrc* __restrict__ src, const InterDev* __restrict__ inter,
                                                              const VColDev* __restrict__ vcols, const TermDev* __restrict__ terms, Ext alpha,
                                                              const uint32_t* __restrict__ betas, uint32_t* __restrict__ num0, uint32_t* __restrict__ den0,
                                                              uint32_t* __restrict__ num1, uint32_t* __restrict__ den1, uint32_t* __restrict__ num2,
                                                              uint32_t* __restrict__ den2) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= jobs.total) return;
    const int jx = find_job(jobs, w);
    const ChipJob& c = jobs.j[jx];
    const uint64_t lw = w - c.work_start, h = c.rows_in;
    const uint32_t len1 = (c.rows_in + 1) / 2, len2 = (len1 + 1) / 2;
    const uint32_t k = div_small(lw, len2), j = (uint32_t)(lw - (uint64_t)k * len2);
    const InterDev in = inter[c.int_off + k];
    const FirstSrc s = src[jx];
    const uint64_t r0 = 4ull * j;
    const uint32_t nv = (uint32_t)(h - r0 < 4 ? h - r0 : 4);  // entries of level 0 this thread holds (1..4)
    auto apply = [&](const VColDev& v, uint32_t (&a)[4]) {  // the virtual column at rows r0 .. r0 + nv - 1
#pragma unroll
        for (int t = 0; t < 4; t++) a[t] = v.constant;
        for (uint32_t q = 0; q < v.n_terms; q++) {
            const TermDev tm = terms[v.term_start + q];
            const uint32_t* col = (tm.source == 4 ? s.main : s.prep) + (uint64_t)tm.col * h + r0;
#pragma unroll
            for (int t = 0; t < 4; t++)
                if (t < nv) a[t] = kb::add(a[t], kb::mul(__ldg(col + t), tm.weight));
        }
    };
    Ext d[4];
    d[0] = kb::ext_add(alpha, kb::ext_mul_base(ldE(betas, 0), kb::from_canonical(in.arg_index)));
#pragma unroll
    for (int t = 1; t < 4; t++) d[t] = d[0];
    uint32_t x[4];
    for (uint32_t q = 0; q < in.n_values; q++) {
        apply(vcols[in.vcol_start + 1 + q], x);
        const Ext b = ldE(betas, q + 1);
#pragma unroll
        for (int t = 0; t < 4; t++) d[t] = kb::ext_add(d[t], kb::ext_mul_base(b, x[t]));
    }
    uint32_t m[4];
    apply(vcols[in.vcol_start], m);
    if (!in.is_send) {
#pragma unroll
        for (int t = 0; t < 4; t++) m[t] = kb::neg(m[t]);
    }
    const uint64_t o0 = c.in_off + (uint64_t)k * h + r0, o1 = c.out_off + (uint64_t)k * len1 + 2 * j;
#pragma unroll
    for (int t = 0; t < 4; t++)
        if (t < nv) { num0[o0 + t] = m[t]; stE(den0, o0 + t, d[t]); }
    Ext n1[2], d1[2];  // level 1 entries 2j, 2j+1 (the second one exists when nv > 2)
#pragma unroll
    for (int e = 0; e < 2; e++) {
        if (2 * e + 1 < nv) {
            n1[e] = kb::ext_add(kb::ext_mul_base(d[2 * e + 1], m[2 * e]), kb::ext_mul_base(d[2 * e], m[2 * e + 1]));
            d1[e] = kb::ext_mul(d[2 * e], d[2 * e + 1]);
        } else {
            n1[e] = kb::ext_from_base(m[2 * e]); d1[e] = d[2 * e];
        }
    }
    stE(num1, o1, n1[0]); stE(den1, o1, d1[0]);
    if (nv > 2) { stE(num1, o1 + 1, n1[1]); stE(den1, o1 + 1, d1[1]); }
    if (num2) {
        Ext n2 = n1[0], d2 = d1[0];
        if (nv > 2) frac_add(n1[0], d1[0], n1[1], d1[1], n2, d2);
        const uint64_t o2 = s.off2 + (uint64_t)k * len2 + j;
        stE(num2, o2, n2); stE(den2, o2, d2);
    }
}

// ---- level l -> l+1 (l >= 2): F'[j] = F[2j] (+) F[2j+1]  (missing odd entry = padding (0,1): identity) ---------------------
__global__ void __launch_bounds__(256) gkr_level_kernel(JobTable jobs, const uint32_t* __restrict__ num, const uint32_t* __restrict__ den,
                                                        uint32_t* __restrict__ num_o, uint32_t* __restrict__ den_o) {
    uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= jobs.total) return;
    const ChipJob& c = jobs.j[find_job(jobs, w)];
    const uint64_t lw = w - c.work_start;
    const uint32_t len_o = (c.rows_in + 1) / 2;
    const uint32_t k = div_small(lw, len_o);
    const uint32_t j = (uint32_t)(lw - (uint64_t)k * len_o);
    const uint64_t base = c.in_off + (uint64_t)k * c.rows_in;
    Ext n0 = ldE(num, base + 2 * j), d0 = ldE(den, base + 2 * j);
    Ext n = n0, d = d0;
    if (2 * j + 1 < c.rows_in) frac_add(n0, d0, ldE(num, base + 2 * j + 1), ldE(den, base + 2 * j + 1), n, d);
    stE(num_o, c.out_off + (uint64_t)k * len_o + j, n);
    stE(den_o, c.out_off + (uint64_t)k * len_o + j, d);
}

// The four layer arrays seen through a fraction sequence F (length len): row i -> (n0,d0) = F[2i], (n1,d1) = F[2i+1].
// N = numerator type: uint32_t (level 0, base field) or Ext; the overloads below keep one source for both.
template <class N> struct RowT { N n0, n1; Ext d0, d1; };
using Row4 = RowT<Ext>;
__device__ __forceinline__ void ld_num(const uint32_t* p, uint64_t i, uint32_t& x) { x = p[i]; }
__device__ __forceinline__ void ld_num(const uint32_t* p, uint64_t i, Ext& x) { x = ldE(p, i); }
__device__ __forceinline__ uint32_t nadd(uint32_t a, uint32_t b) { return kb::add(a, b); }
__device__ __forceinline__ Ext nadd(const Ext& a, const Ext& b) { return kb::ext_add(a, b); }
__device__ __forceinline__ uint32_t nsub(uint32_t a, uint32_t b) { return kb::sub(a, b); }
__device__ __forceinline__ Ext nsub(const Ext& a, const Ext& b) { return kb::ext_sub(a, b); }
__device__ __forceinline__ Ext nmul(const Ext& d, uint32_t n) { return kb::ext_mul_base(d, n); }  // 4 products
__device__ __forceinline__ Ext nmul(const Ext& d, const Ext& n) { return kb::ext_mul(d, n); }     // 16 products
__device__ __forceinline__ Ext nfix(uint32_t x, uint32_t y, const Ext& a) { return kb::ext_add(kb::ext_from_base(x), kb::ext_mul_base(a, kb::sub(y, x))); }
__device__ __forceinline__ Ext nfix(const Ext& x, const Ext& y, const Ext& a) { return kb::ext_add(x, kb::ext_mul(a, kb::ext_sub(y, x))); }

template <class N>
__device__ __forceinline__ RowT<N> row_from_seq(const uint32_t* num, const uint32_t* den, uint64_t base, uint32_t len, uint32_t i) {
    RowT<N> r;
    r.n0 = N{}; r.n1 = N{}; r.d0 = kb::ext_one(); r.d1 = kb::ext_one();
    if (2 * i < len) { ld_num(num, base + 2 * i, r.n0); r.d0 = ldE(den, base + 2 * i); }
    if (2 * i + 1 < len) { ld_num(num, base + 2 * i + 1, r.n1); r.d1 = ldE(den, base + 2 * i + 1); }
    return r;
}
template <class N> __device__ __forceinline__ RowT<N> row_add(const RowT<N>& x, const RowT<N>& y) {
    return RowT<N>{nadd(x.n0, y.n0), nadd(x.n1, y.n1), kb::ext_add(x.d0, y.d0), kb::ext_add(x.d1, y.d1)};
}
template <class N> __device__ __forceinline__ RowT<N> row_sub(const RowT<N>& x, const RowT<N>& y) {
    return RowT<N>{nsub(x.n0, y.n0), nsub(x.n1, y.n1), kb::ext_sub(x.d0, y.d0), kb::ext_sub(x.d1, y.d1)};
}
// the layer's summand lambda (n0 d1 + n1 d0) + d0 d1: a quadratic form in the row
template <class N> __device__ __forceinline__ Ext row_poly(const RowT<N>& x, const Ext& lambda) {
    return kb::ext_add(kb::ext_mul(lambda, kb::ext_add(nmul(x.d1, x.n0), nmul(x.d0, x.n1))), kb::ext_mul(x.d0, x.d1));
}
// working layout of a chip (after the first fix): [4][I][rows] EF = n0 | d0 | n1 | d1
__device__ __forceinline__ Row4 row_from_work(const uint32_t* a, uint64_t base, uint32_t I, uint32_t rows, uint32_t k, uint32_t i) {
    Row4 r;
    r.n0 = kb::ext_zero(); r.n1 = kb::ext_zero(); r.d0 = kb::ext_one(); r.d1 = kb::ext_one();
    if (i < rows) {
        const uint64_t s = (uint64_t)I * rows, o = base + (uint64_t)k * rows + i;
        r.n0 = ldE(a, o); r.d0 = ldE(a, o + s); r.n1 = ldE(a, o + 2 * s); r.d1 = ldE(a, o + 3 * s);
    }
    return r;
}
template <class N> __device__ __forceinline__ Row4 fix_rows(const RowT<N>& x, const RowT<N>& y, const Ext& a) {
    Row4 r;
    r.n0 = nfix(x.n0, y.n0, a);
    r.d0 = kb::ext_add(x.d0, kb::ext_mul(a, kb::ext_sub(y.d0, x.d0)));
    r.n1 = nfix(x.n1, y.n1, a);
    r.d1 = kb::ext_add(x.d1, kb::ext_mul(a, kb::ext_sub(y.d1, x.d1)));
    return r;
}
// contributions of the row pair (x = row 2i, y = row 2i+1) to (eval_0, eval_half, eq_sum)   logup_poly.rs:330-505
__device__ __forceinline__ void pair_sums(const Row4& x, const Row4& y, const Ext& e, const Ext& er0, const Ext& er1, const Ext& lambda,
                                          Ext& s0, Ext& sh, Ext& se) {
    const Ext t0 = row_poly(x, lambda), th = row_poly(row_add(x, y), lambda);
    const Ext ee0 = kb::ext_mul(e, er0), ees = kb::ext_mul(e, kb::ext_add(er0, er1));  // shared by the three sums
    s0 = kb::ext_add(s0, kb::ext_mul(ee0, t0));
    sh = kb::ext_add(sh, kb::ext_mul(ees, th));
    se = kb::ext_add(se, ees);
}

// Rounds 0 and 1 of a layer in one pass over its fraction sequence.  work item = (chip, k, row quad i): rows x0..x3 = 4i..4i+3.
// The eq table is a product, E[2j + b] = P[j] (b ? last : 1 - last) with P[j] = E[2j] + E[2j+1], `last` = round 0's point
// coordinate: round 0's eval_0 is (1 - last) sum_pairs e P q(x_even), the host applies the factor.  Binding round 0 to a, the
// round-1 rows are x0 + a (x1 - x0), x2 + a (x3 - x2) and the eq table becomes c(a) P.  The summand q is a quadratic form, so
// q(x + a (y - x)) = (1-a) q(x) + a q(y) + (a^2 - a) q(y - x): round 1's sums are c(a) times a quadratic in a whose
// coefficients per sum are accumulated here; the host evaluates them at the sampled a.  With w = e P0 (first pair), v = e P1
// (second pair), X = x0 + x2, Y = x1 + x3, the sums (EF) are
//   0: v q(x2)   1: v q(x2 + x3)   2: w + v   3: w q(x0)   4: w q(x1)   5: w q(x0 + x1)   6..8: (w + v) q(X), q(Y), q(Y - X)
// two = 0 (a layer with one row variable: no second pair, no round 1): sums 2, 3, 5 with w only.
constexpr int SUM2_WORDS = 36;
constexpr int SUM2_THREADS = 128;  // ~160 registers per thread: three 128-thread blocks per SM instead of one 256-thread block
template <class N>
__global__ void __launch_bounds__(SUM2_THREADS) gkr_sum2_kernel(JobTable jobs, const uint32_t* __restrict__ num, const uint32_t* __restrict__ den,
                                                                const uint32_t* __restrict__ eq_int, const uint32_t* __restrict__ eq_row, Ext lambda,
                                                                int two, uint32_t* __restrict__ partial, Mail mail) {
    Ext acc[9];
#pragma unroll
    for (int q = 0; q < 9; q++) acc[q] = kb::ext_zero();
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < jobs.total; w += (uint64_t)gridDim.x * blockDim.x) {
        const ChipJob& c = jobs.j[find_job(jobs, w)];
        const uint64_t lw = w - c.work_start;
        const uint32_t rows = (c.rows_in + 1) / 2, quads = (rows + 3) / 4;
        const uint32_t k = div_small(lw, quads), i4 = 4 * (uint32_t)(lw - (uint64_t)k * quads);
        const uint64_t base = c.in_off + (uint64_t)k * c.rows_in;
        const Ext e = ldE(eq_int, c.int_off + k);
        const RowT<N> x0 = row_from_seq<N>(num, den, base, c.rows_in, i4), x1 = row_from_seq<N>(num, den, base, c.rows_in, i4 + 1);
        const Ext wt = kb::ext_mul(e, kb::ext_add(ldE(eq_row, i4), ldE(eq_row, i4 + 1)));
        acc[2] = kb::ext_add(acc[2], wt);
        acc[3] = kb::ext_add(acc[3], kb::ext_mul(wt, row_poly(x0, lambda)));
        acc[5] = kb::ext_add(acc[5], kb::ext_mul(wt, row_poly(row_add(x0, x1), lambda)));
        if (two) {  // rows <= 2^r with r >= 2: the second pair is inside the eq table (all padding past the chip's rows)
            const RowT<N> x2 = row_from_seq<N>(num, den, base, c.rows_in, i4 + 2), x3 = row_from_seq<N>(num, den, base, c.rows_in, i4 + 3);
            const Ext vt = kb::ext_mul(e, kb::ext_add(ldE(eq_row, i4 + 2), ldE(eq_row, i4 + 3))), wv = kb::ext_add(wt, vt);
            acc[0] = kb::ext_add(acc[0], kb::ext_mul(vt, row_poly(x2, lambda)));
            acc[1] = kb::ext_add(acc[1], kb::ext_mul(vt, row_poly(row_add(x2, x3), lambda)));
            acc[2] = kb::ext_add(acc[2], vt);
            acc[4] = kb::ext_add(acc[4], kb::ext_mul(wt, row_poly(x1, lambda)));
            const RowT<N> X = row_add(x0, x2), Y = row_add(x1, x3);
            acc[6] = kb::ext_add(acc[6], kb::ext_mul(wv, row_poly(X, lambda)));
            acc[7] = kb::ext_add(acc[7], kb::ext_mul(wv, row_poly(Y, lambda)));
            acc[8] = kb::ext_add(acc[8], kb::ext_mul(wv, row_poly(row_sub(Y, X), lambda)));
        }
    }
    block_reduce<9>(acc, partial, mail);
}

// The first fix of a layer: bind round 0's variable with a0 (and, TWO, round 1's with a1) straight from the fraction sequence,
// write the working arrays of the next round and accumulate that round's sums.  work item = (chip, k, NEW row pair i).
template <class N, bool TWO>
__global__ void __launch_bounds__(256) gkr_fix2_kernel(JobTable jobs, const uint32_t* __restrict__ num, const uint32_t* __restrict__ den,
                                                       uint32_t* __restrict__ out, const uint32_t* __restrict__ eq_int,
                                                       const uint32_t* __restrict__ eq_row_new, Ext a0, Ext a1, Ext lambda,
                                                       uint32_t* __restrict__ partial, Mail mail) {
    Ext s[3] = {kb::ext_zero(), kb::ext_zero(), kb::ext_zero()};
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < jobs.total; w += (uint64_t)gridDim.x * blockDim.x) {
        const ChipJob& c = jobs.j[find_job(jobs, w)];
        const uint64_t lw = w - c.work_start;
        const uint32_t rows = (c.rows_in + 1) / 2;
        const uint32_t rows_new = TWO ? (rows + 3) / 4 : (rows + 1) / 2, pairs = (rows_new + 1) / 2;
        const uint32_t k = div_small(lw, pairs), i = (uint32_t)(lw - (uint64_t)k * pairs);
        const uint64_t base = c.in_off + (uint64_t)k * c.rows_in;
        Row4 nr[2];
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
            const uint32_t o = 2 * i + hh;  // new row index
            if (o < rows_new) {
                if (TWO) {  // old rows 4o .. 4o+3
                    const Row4 lo = fix_rows(row_from_seq<N>(num, den, base, c.rows_in, 4 * o), row_from_seq<N>(num, den, base, c.rows_in, 4 * o + 1), a0);
                    const Row4 hi = fix_rows(row_from_seq<N>(num, den, base, c.rows_in, 4 * o + 2), row_from_seq<N>(num, den, base, c.rows_in, 4 * o + 3), a0);
                    nr[hh] = fix_rows(lo, hi, a1);
                } else {
                    nr[hh] = fix_rows(row_from_seq<N>(num, den, base, c.rows_in, 2 * o), row_from_seq<N>(num, den, base, c.rows_in, 2 * o + 1), a0);
                }
                const uint64_t st = (uint64_t)c.I * rows_new, q = c.out_off + (uint64_t)k * rows_new + o;
                stE(out, q, nr[hh].n0); stE(out, q + st, nr[hh].d0); stE(out, q + 2 * st, nr[hh].n1); stE(out, q + 3 * st, nr[hh].d1);
            } else {  // beyond the real rows: padding values for the sums below
                nr[hh].n0 = kb::ext_zero(); nr[hh].n1 = kb::ext_zero(); nr[hh].d0 = kb::ext_one(); nr[hh].d1 = kb::ext_one();
            }
        }
        pair_sums(nr[0], nr[1], ldE(eq_int, c.int_off + k), ldE(eq_row_new, 2 * i), ldE(eq_row_new, 2 * i + 1), lambda, s[0], s[1], s[2]);
    }
    block_reduce<3>(s, partial, mail);
}

// the later row rounds: fix the last row variable of the working arrays, write the halved arrays and accumulate the next
// round's sums.  work item = (chip, k, NEW row pair i): new rows 2i, 2i+1 come from old rows 4i .. 4i+3.
__global__ void __launch_bounds__(256) gkr_fix_sum_kernel(JobTable jobs, const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                                                          const uint32_t* __restrict__ eq_int, const uint32_t* __restrict__ eq_row_new, Ext alpha,
                                                          Ext lambda, uint32_t* __restrict__ partial, Mail mail) {
    Ext s[3] = {kb::ext_zero(), kb::ext_zero(), kb::ext_zero()};
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < jobs.total; w += (uint64_t)gridDim.x * blockDim.x) {
        const ChipJob& c = jobs.j[find_job(jobs, w)];
        const uint64_t lw = w - c.work_start;
        const uint32_t rows_old = c.rows_in;
        const uint32_t rows_new = (rows_old + 1) / 2, pairs = (rows_new + 1) / 2;
        const uint32_t k = div_small(lw, pairs), i = (uint32_t)(lw - (uint64_t)k * pairs);
        Row4 nr[2];
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
            const uint32_t o = 2 * i + hh;  // new row index; old rows 2o, 2o+1
            const Row4 x = row_from_work(in, c.in_off, c.I, rows_old, k, 2 * o), y = row_from_work(in, c.in_off, c.I, rows_old, k, 2 * o + 1);
            nr[hh] = fix_rows(x, y, alpha);
            if (o < rows_new) {
                const uint64_t st = (uint64_t)c.I * rows_new, q = c.out_off + (uint64_t)k * rows_new + o;
                stE(out, q, nr[hh].n0); stE(out, q + st, nr[hh].d0); stE(out, q + 2 * st, nr[hh].n1); stE(out, q + 3 * st, nr[hh].d1);
            } else {  // beyond the real rows: padding values for the sums below
                nr[hh].n0 = kb::ext_zero(); nr[hh].n1 = kb::ext_zero(); nr[hh].d0 = kb::ext_one(); nr[hh].d1 = kb::ext_one();
            }
        }
        pair_sums(nr[0], nr[1], ldE(eq_int, c.int_off + k), ldE(eq_row_new, 2 * i), ldE(eq_row_new, 2 * i + 1), lambda, s[0], s[1], s[2]);
    }
    block_reduce<3>(s, partial, mail);
}

// ---- interaction variables (logup_poly.rs:118-176 + the generic round of sumcheck/src/prover.rs) -------------------------------
// After the last row variable every (chip, interaction) holds one row; the layer becomes four arrays over the padded
// interaction index (numerator 0 / denominator 1 beyond the machine's interactions), plus the eq table over that index.
// arr = [5][n] EF: n0 | n1 | d0 | d1 | eq.
__global__ void __launch_bounds__(256) gkr_flatten_kernel(JobTable jobs, const uint32_t* __restrict__ work, const uint32_t* __restrict__ eq_int,
                                                          uint32_t n, uint32_t* __restrict__ arr, uint32_t* __restrict__ payload, Mail mail) {
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        Ext n0 = kb::ext_zero(), n1 = kb::ext_zero(), d0 = kb::ext_one(), d1 = kb::ext_one();
        for (int q = 0; q < jobs.n; q++) {
            const ChipJob& c = jobs.j[q];
            if (t >= c.int_off && t < c.int_off + c.I) {
                const uint64_t o = c.in_off + (t - c.int_off), sI = c.I;  // one row per interaction: [4][I][1]
                n0 = ldE(work, o); d0 = ldE(work, o + sI); n1 = ldE(work, o + 2 * sI); d1 = ldE(work, o + 3 * sI);
            }
        }
        stE(arr, t, n0); stE(arr, (uint64_t)n + t, n1); stE(arr, 2ull * n + t, d0); stE(arr, 3ull * n + t, d1);
        stE(arr, 4ull * n + t, ldE(eq_int, t));
        if (n == 1) { stE(payload, 3, n0); stE(payload, 5, n1); stE(payload, 7, d0); stE(payload, 9, d1); }
    }
    if (mail.flag) sp1_mail_done(mail);
}
// One interaction round in one block: (optionally) bind the previous variable with alpha, store the halved arrays, and post
// (eval_0, eval_half, eq_sum) of the next variable.  When two entries remain they are posted too (payload EF slots 3..10:
// n0[0] n0[1] n1[0] n1[1] d0[0] d0[1] d1[0] d1[1]) so that the host can finish the layer without another launch.
__global__ void __launch_bounds__(256) gkr_inter_round_kernel(const uint32_t* __restrict__ in, uint32_t n_in, int fold, Ext alpha, Ext lambda,
                                                              uint32_t* __restrict__ out, uint32_t* __restrict__ payload, Mail mail) {
    const uint32_t n_cur = fold ? n_in / 2 : n_in;
    Ext s0 = kb::ext_zero(), sh = kb::ext_zero(), se = kb::ext_zero();
    for (uint32_t j = threadIdx.x; j < n_cur / 2; j += blockDim.x) {
        Ext v[5][2];
#pragma unroll
        for (int a = 0; a < 5; a++)
#pragma unroll
            for (int hh = 0; hh < 2; hh++) {
                const uint32_t x = 2 * j + hh;
                if (fold) {
                    const Ext lo = ldE(in, (uint64_t)a * n_in + 2 * x), hi = ldE(in, (uint64_t)a * n_in + 2 * x + 1);
                    v[a][hh] = kb::ext_add(lo, kb::ext_mul(alpha, kb::ext_sub(hi, lo)));
                    stE(out, (uint64_t)a * n_cur + x, v[a][hh]);
                } else v[a][hh] = ldE(in, (uint64_t)a * n_in + x);
            }
        const Ext &n0a = v[0][0], &n1a = v[1][0], &d0a = v[2][0], &d1a = v[3][0], &ea = v[4][0], &eb = v[4][1];
        s0 = kb::ext_add(s0, kb::ext_mul(ea, kb::ext_add(kb::ext_mul(lambda, kb::ext_add(kb::ext_mul(d0a, n1a), kb::ext_mul(d1a, n0a))), kb::ext_mul(d0a, d1a))));
        const Ext N0 = kb::ext_add(v[0][0], v[0][1]), N1 = kb::ext_add(v[1][0], v[1][1]), D0 = kb::ext_add(v[2][0], v[2][1]), D1 = kb::ext_add(v[3][0], v[3][1]);
        const Ext es = kb::ext_add(ea, eb);
        sh = kb::ext_add(sh, kb::ext_mul(es, kb::ext_add(kb::ext_mul(lambda, kb::ext_add(kb::ext_mul(D0, N1), kb::ext_mul(D1, N0))), kb::ext_mul(D0, D1))));
        se = kb::ext_add(se, es);
        if (n_cur == 2) {
#pragma unroll
            for (int a = 0; a < 4; a++) { stE(payload, 3 + 2 * a, v[a][0]); stE(payload, 4 + 2 * a, v[a][1]); }
        }
    }
    const Ext sums[3] = {s0, sh, se};
    block_reduce<3>(sums, payload, mail);
}

// E'[j] = E[2j] + alpha (E[2j+1] - E[2j])
__global__ void gkr_fix_eq_kernel(const uint32_t* __restrict__ E, uint64_t n_out, Ext alpha, uint32_t* __restrict__ Eo) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_out) return;
    Ext a = ldE(E, 2 * j), b = ldE(E, 2 * j + 1);
    stE(Eo, j, kb::ext_add(a, kb::ext_mul(alpha, kb::ext_sub(b, a))));
}
// E''[j] = E'[2j] + a1 (E'[2j+1] - E'[2j]) with E' = E folded by a0: two variables in one launch
__global__ void gkr_fix_eq2_kernel(const uint32_t* __restrict__ E, uint64_t n_out, Ext a0, Ext a1, uint32_t* __restrict__ Eo) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_out) return;
    const Ext e0 = ldE(E, 4 * j), e1 = ldE(E, 4 * j + 1), e2 = ldE(E, 4 * j + 2), e3 = ldE(E, 4 * j + 3);
    const Ext lo = kb::ext_add(e0, kb::ext_mul(a0, kb::ext_sub(e1, e0))), hi = kb::ext_add(e2, kb::ext_mul(a0, kb::ext_sub(e3, e2)));
    stE(Eo, j, kb::ext_add(lo, kb::ext_mul(a1, kb::ext_sub(hi, lo))));
}
// every read is bounds-checked against the end of the blob and every column against the chip's widths: a blob exported for another
// chip set must become an error, not an out-of-bounds read on host or device
const uint32_t* parse_vcol(const uint32_t* b, const uint32_t* end, HostInteractions& H, uint32_t main_w, uint32_t prep_w) {
    if (end - b < 2) return nullptr;
    VColDev v; v.n_terms = *b++; v.constant = *b++; v.term_start = (uint32_t)H.terms.size();
    if ((uint64_t)v.n_terms * 3 > (uint64_t)(end - b)) return nullptr;
    for (uint32_t i = 0; i < v.n_terms; i++) {
        if ((b[0] != LEAF_MAIN && b[0] != LEAF_PREP) || b[1] >= (b[0] == LEAF_MAIN ? main_w : prep_w)) return nullptr;
        H.terms.push_back(TermDev{b[0], b[1], b[2]}); b += 3;
    }
    H.vcols.push_back(v);
    return b;
}

// ---- interaction check (debug_interactions_with_all_chips, crates/hypercube/src/lookup/debug.rs:48-200) ------------------------
// A record is one (chip, row, interaction) with its signed multiplicity (sends +, receives -); its rank (chip, row, interaction
// index) is its position in the reference's iteration order.  Records are sorted by the fingerprint of their key (debug_fp.cuh),
// each run of equal fingerprints is summed, and every record of a run is compared with its predecessor by FULL key: a run that
// mixes keys is flagged and resolved on the host.
struct DbgChip { const uint32_t* main; const uint32_t* prep; uint64_t h; uint32_t rank0, I, inter0, chip; };  // chips with records

__device__ __forceinline__ uint32_t dbg_vcol(const VColDev& v, const TermDev* __restrict__ terms, const DbgChip& c, uint64_t row) {
    uint32_t a = v.constant;
    for (uint32_t q = 0; q < v.n_terms; q++) {
        const TermDev tm = terms[v.term_start + q];
        a = kb::add(a, kb::mul(__ldg((tm.source == LEAF_MAIN ? c.main : c.prep) + (uint64_t)tm.col * c.h + row), tm.weight));
    }
    return a;
}
struct DbgRec { DbgChip c; InterDev in; uint32_t row, t; };  // t = index into the chip table
__device__ __forceinline__ DbgRec dbg_decode(const DbgChip* __restrict__ chips, int n, const InterDev* __restrict__ inter, uint32_t rank) {
    int lo = 0, hi = n - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (chips[mid].rank0 <= rank) lo = mid; else hi = mid - 1; }
    DbgRec r;
    r.t = (uint32_t)lo; r.c = chips[lo];
    const uint32_t local = rank - r.c.rank0;
    r.row = local / r.c.I;
    r.in = inter[r.c.inter0 + (local - r.row * r.c.I)];
    return r;
}
__device__ __forceinline__ uint32_t dbg_signed_mult(const DbgRec& r, const VColDev* __restrict__ vcols, const TermDev* __restrict__ terms) {
    const uint32_t x = dbg_vcol(vcols[r.in.vcol_start], terms, r.c, r.row);
    return r.in.is_send ? x : kb::neg(x);
}

// per rank: sort key = fingerprint of the record's key (dbgfp::NONE when its multiplicity is zero), value = the rank; counts[0] += live
__global__ void __launch_bounds__(256) gkr_dbg_records_kernel(const DbgChip* __restrict__ chips, int n_chips, const InterDev* __restrict__ inter,
                                                              const VColDev* __restrict__ vcols, const TermDev* __restrict__ terms, uint32_t n,
                                                              uint64_t* __restrict__ keys, uint32_t* __restrict__ ranks, uint32_t* __restrict__ counts) {
    const uint32_t rank = blockIdx.x * blockDim.x + threadIdx.x;
    bool live = false;
    if (rank < n) {
        const DbgRec r = dbg_decode(chips, n_chips, inter, rank);
        uint64_t key = dbgfp::NONE;
        if (dbg_signed_mult(r, vcols, terms)) {
            live = true;
            dbgfp::Acc f;
            f.head(r.in.arg_index, r.in.n_values);
            for (uint32_t q = 0; q < r.in.n_values; q++) f.value(q, dbg_vcol(vcols[r.in.vcol_start + 1 + q], terms, r.c, r.row));
            key = f.get();
        }
        keys[rank] = key; ranks[rank] = rank;
    }
    const uint32_t bits = __ballot_sync(0xffffffffu, live);
    if ((threadIdx.x & 31) == 0 && bits) atomicAdd(counts, (uint32_t)__popc(bits));
}

// per sorted position i < n_live: the signed multiplicity, bit 31 set when the record's key differs from its predecessor's although
// their fingerprints are equal
__global__ void __launch_bounds__(256) gkr_dbg_eval_kernel(const DbgChip* __restrict__ chips, int n_chips, const InterDev* __restrict__ inter,
                                                           const VColDev* __restrict__ vcols, const TermDev* __restrict__ terms,
                                                           const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ranks, uint32_t n_live,
                                                           uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_live) return;
    const DbgRec r = dbg_decode(chips, n_chips, inter, ranks[i]);
    uint32_t bad = 0;
    if (i > 0 && keys[i] == keys[i - 1]) {
        const DbgRec p = dbg_decode(chips, n_chips, inter, ranks[i - 1]);
        if (p.in.arg_index != r.in.arg_index || p.in.n_values != r.in.n_values) bad = 1;
        for (uint32_t q = 0; !bad && q < r.in.n_values; q++)
            bad = dbg_vcol(vcols[r.in.vcol_start + 1 + q], terms, r.c, r.row) != dbg_vcol(vcols[p.in.vcol_start + 1 + q], terms, p.c, p.row);
    }
    out[i] = dbg_signed_mult(r, vcols, terms) | bad << 31;
}

// run aggregate = (first position << 32) | (mixed-key bit << 31) | net multiplicity
struct DbgRunOp {
    __device__ __forceinline__ uint64_t operator()(uint64_t x, uint64_t y) const {
        const uint32_t a = (uint32_t)x, b = (uint32_t)y;
        const uint32_t lo = kb::add(a & 0x7fffffffu, b & 0x7fffffffu) | ((a | b) & 0x80000000u);
        return ((uint64_t)min((uint32_t)(x >> 32), (uint32_t)(y >> 32)) << 32) | lo;
    }
};
struct DbgPosValue {
    const uint32_t* v;
    __device__ __forceinline__ uint64_t operator()(uint32_t i) const { return ((uint64_t)i << 32) | v[i]; }
};
struct DbgNonZero {
    __device__ __forceinline__ bool operator()(uint32_t x) const { return x != 0; }
};

// per run: a mixed run goes to `mixed` (counts[1]); an unbalanced one is flagged at its first record's rank with run index + 1 (counts[0])
__global__ void __launch_bounds__(256) gkr_dbg_flag_kernel(const uint64_t* __restrict__ agg, uint32_t n_runs, const uint32_t* __restrict__ ranks,
                                                           uint32_t* __restrict__ flags, uint32_t* __restrict__ counts, uint32_t* __restrict__ mixed,
                                                           uint32_t mixed_cap) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_runs) return;
    const uint64_t a = agg[r];
    const uint32_t lo = (uint32_t)a;
    if (lo >> 31) {
        const uint32_t j = atomicAdd(counts + 1, 1u);
        if (j < mixed_cap) mixed[j] = r;
    } else if (lo) {
        flags[ranks[a >> 32]] = r + 1;
        atomicAdd(counts, 1u);
    }
}

__device__ __forceinline__ void dbg_run_extent(const uint64_t* agg, uint32_t n_runs, uint32_t n_live, uint32_t r, uint32_t& s, uint32_t& e) {
    s = (uint32_t)(agg[r] >> 32);
    e = r + 1 < n_runs ? (uint32_t)(agg[r + 1] >> 32) : n_live;
}

// one block per listed run (runs1[b] = run index + 1): out[b * stride ..] = kind, n_values, values[255], first rank, then per chip-table
// entry (net, number of records)
__global__ void __launch_bounds__(256) gkr_dbg_key_kernel(const DbgChip* __restrict__ chips, int n_chips, const InterDev* __restrict__ inter,
                                                          const VColDev* __restrict__ vcols, const TermDev* __restrict__ terms,
                                                          const uint64_t* __restrict__ agg, uint32_t n_runs, uint32_t n_live,
                                                          const uint32_t* __restrict__ ranks, const uint32_t* __restrict__ runs1,
                                                          uint32_t* __restrict__ out, uint32_t stride) {
    extern __shared__ __align__(16) unsigned char dbg_smem[];
    unsigned long long* sums = reinterpret_cast<unsigned long long*>(dbg_smem);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(sums + n_chips);
    for (int c = threadIdx.x; c < n_chips; c += blockDim.x) { sums[c] = 0; cnt[c] = 0; }
    __syncthreads();
    uint32_t s, e;
    dbg_run_extent(agg, n_runs, n_live, runs1[blockIdx.x] - 1, s, e);
    for (uint32_t pos = s + threadIdx.x; pos < e; pos += blockDim.x) {
        const DbgRec r = dbg_decode(chips, n_chips, inter, ranks[pos]);
        atomicAdd(&sums[r.t], (unsigned long long)dbg_signed_mult(r, vcols, terms));
        atomicAdd(&cnt[r.t], 1u);
    }
    __syncthreads();
    uint32_t* o = out + (uint64_t)blockIdx.x * stride;
    if (threadIdx.x == 0) {
        const DbgRec r = dbg_decode(chips, n_chips, inter, ranks[s]);
        o[0] = r.in.arg_index; o[1] = r.in.n_values;
        for (uint32_t q = 0; q < r.in.n_values; q++) o[2 + q] = dbg_vcol(vcols[r.in.vcol_start + 1 + q], terms, r.c, r.row);
        o[257] = ranks[s];
    }
    for (int c = threadIdx.x; c < n_chips; c += blockDim.x) { o[258 + 2 * c] = (uint32_t)(sums[c] % kb::P); o[259 + 2 * c] = cnt[c]; }
}

// every record of the mixed runs (one block per run) as words {rank, signed multiplicity, kind, n_values, values}; used[0] = words needed
__global__ void __launch_bounds__(256) gkr_dbg_collect_kernel(const DbgChip* __restrict__ chips, int n_chips, const InterDev* __restrict__ inter,
                                                              const VColDev* __restrict__ vcols, const TermDev* __restrict__ terms,
                                                              const uint64_t* __restrict__ agg, uint32_t n_runs, uint32_t n_live,
                                                              const uint32_t* __restrict__ ranks, const uint32_t* __restrict__ mixed,
                                                              uint32_t* __restrict__ out, uint32_t* __restrict__ used, uint32_t cap) {
    uint32_t s, e;
    dbg_run_extent(agg, n_runs, n_live, mixed[blockIdx.x], s, e);
    for (uint32_t pos = s + threadIdx.x; pos < e; pos += blockDim.x) {
        const DbgRec r = dbg_decode(chips, n_chips, inter, ranks[pos]);
        const uint32_t nw = 4 + r.in.n_values, at = atomicAdd(used, nw);
        if ((uint64_t)at + nw > cap) continue;
        out[at] = ranks[pos]; out[at + 1] = dbg_signed_mult(r, vcols, terms); out[at + 2] = r.in.arg_index; out[at + 3] = r.in.n_values;
        for (uint32_t q = 0; q < r.in.n_values; q++) out[at + 4 + q] = dbg_vcol(vcols[r.in.vcol_start + 1 + q], terms, r.c, r.row);
    }
}

}  // namespace

// parses the interaction section that follows the AIR records in the machine blob (called by sp1b200_machine_create);
// widths[2k], widths[2k+1] = main / preprocessed width of chip k.  Returns nullptr (with the error set) on a malformed section.
void* sp1b200_parse_interactions(const uint32_t* b, const uint32_t* end, size_t n_chips, const uint32_t* widths) {
    auto H = std::make_unique<HostInteractions>();
    H->per_chip.resize(n_chips);
    if (b >= end) return H.release();  // machine without interactions (zerocheck-only tests)
    size_t k = 0;
    for (auto& chip : H->per_chip) {
        const uint32_t mw = widths[2 * k], pw = widths[2 * k + 1];
        if (end - b < 1) { sp1b200_set_error("machine_create: truncated interaction section (chip %zu)", k); return nullptr; }
        uint32_t n = *b++;
        for (uint32_t i = 0; i < n; i++) {
            if (end - b < 3) { sp1b200_set_error("machine_create: truncated interaction section (chip %zu)", k); return nullptr; }
            InterDev in; in.is_send = *b++; in.arg_index = *b++; in.n_values = *b++; in.vcol_start = (uint32_t)H->vcols.size();
            if (in.n_values > 255) { sp1b200_set_error("machine_create: chip %zu interaction %u has %u values", k, i, in.n_values); return nullptr; }
            for (uint32_t v = 0; v <= in.n_values; v++) {   // multiplicity, then the values
                b = parse_vcol(b, end, *H, mw, pw);
                if (!b) { sp1b200_set_error("machine_create: chip %zu interaction %u: malformed or out-of-range virtual column", k, i); return nullptr; }
            }
            chip.push_back(in);
        }
        k++;
    }
    return H.release();
}
void sp1b200_free_interactions(void* p) { delete static_cast<HostInteractions*>(p); }

extern "C" {

// GkrProverImpl::prove_logup_gkr (crates/hypercube/src/logup_gkr/prover.rs:70-215).
// d_main[k]/d_prep[k]: chip columns (column-major [w x h_heights[k]]), interactions from the machine blob.
// h_replay_witness: the GKR grinding witness when params.grind_mode == 1.
// Output words: the LogUp-GKR section of a shard proof (proof_layout.hpp).
sp1b200_err sp1b200_logup_gkr(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint64_t* h_heights, const uint32_t* const* d_main,
                              const uint32_t* const* d_prep, const uint32_t* h_replay_witness, uint32_t* h_chal, uint32_t* h_out, uint64_t cap,
                              uint64_t* h_words);

}

#include "gkr_driver.inc"

// debug_interactions_with_all_chips (crates/hypercube/src/lookup/debug.rs:48-200) on the device; report words as
// sp1b200_debug_interactions (include/sp1b200.h).  Device memory: 24 B per (row, interaction) of the shard (two 8-byte sort-key and
// two 4-byte rank buffers, reused for the run sums and flags) plus the sort's temporary storage.
sp1b200_err sp1b200_debug_interactions_device(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint64_t* h_heights, const uint32_t* const* d_main,
                                              const uint32_t* const* d_prep, uint32_t max_keys, std::vector<uint32_t>& words) {
    const HostInteractions& H = *static_cast<const HostInteractions*>(m->interactions);
    const size_t nch = m->chips.size();
    cudaStream_t st = ctx->stream;
    std::vector<DbgChip> tab;
    std::vector<InterDev> flat;
    uint64_t n_total = 0;
    for (size_t c = 0; c < nch; c++) {
        const uint32_t I = (uint32_t)H.per_chip[c].size();
        if (h_heights[c] && I)
            tab.push_back(DbgChip{d_main[c], m->chips[c].prep_w ? d_prep[c] : nullptr, h_heights[c], (uint32_t)n_total, I, (uint32_t)flat.size(), (uint32_t)c});
        flat.insert(flat.end(), H.per_chip[c].begin(), H.per_chip[c].end());
        n_total += h_heights[c] * I;
        if (n_total > 0x7fffffffu) return sp1b200_set_error("debug_interactions: more than 2^31 - 1 (row, interaction) pairs in the shard");
    }
    struct Key { uint32_t first_rank; std::vector<uint32_t> w; };   // w: kind .. the per-chip list, without the first-occurrence words
    std::vector<Key> keys;
    uint64_t n_unbalanced = 0;
    auto emit = [&]() {
        // merge the two sources in first-occurrence order; first occurrence = (chip, interaction, row) words from the rank
        std::sort(keys.begin(), keys.end(), [](const Key& a, const Key& b) { return a.first_rank < b.first_rank; });
        const size_t n_listed = std::min<uint64_t>(keys.size(), max_keys);
        words = {(uint32_t)n_unbalanced, (uint32_t)(n_unbalanced >> 32), (uint32_t)n_listed};
        for (size_t j = 0; j < n_listed; j++) {
            const Key& k = keys[j];
            size_t t = 0;
            while (t + 1 < tab.size() && tab[t + 1].rank0 <= k.first_rank) t++;
            const uint32_t local = k.first_rank - tab[t].rank0, row = local / tab[t].I;
            const uint32_t nv = k.w[1];
            words.insert(words.end(), k.w.begin(), k.w.begin() + 3 + nv);            // kind, n_values, values, net
            words.push_back(tab[t].chip); words.push_back(local - row * tab[t].I); words.push_back(row);
            words.insert(words.end(), k.w.begin() + 3 + nv, k.w.end());              // n_chips, per chip (chip, net)
        }
    };
    if (!n_total) { emit(); return nullptr; }
    DevFree mem(ctx);
    PhaseTimer t_all(ctx, "debug_interactions.total");
    const uint32_t n = (uint32_t)n_total;
    DbgChip* d_tab; InterDev* d_inter; VColDev* d_vcols; TermDev* d_terms; uint32_t* d_counts;
    SP1_TRY(mem.alloc((void**)&d_tab, tab.size() * sizeof(DbgChip)));
    SP1_TRY(mem.alloc((void**)&d_inter, flat.size() * sizeof(InterDev)));
    SP1_TRY(mem.alloc((void**)&d_vcols, H.vcols.size() * sizeof(VColDev)));
    SP1_TRY(mem.alloc((void**)&d_terms, (H.terms.size() + 1) * sizeof(TermDev)));
    SP1_TRY(mem.alloc((void**)&d_counts, 8 * 4));
    SP1_CUDA(cudaMemcpyAsync(d_tab, tab.data(), tab.size() * sizeof(DbgChip), cudaMemcpyHostToDevice, st));
    SP1_CUDA(cudaMemcpyAsync(d_inter, flat.data(), flat.size() * sizeof(InterDev), cudaMemcpyHostToDevice, st));
    SP1_CUDA(cudaMemcpyAsync(d_vcols, H.vcols.data(), H.vcols.size() * sizeof(VColDev), cudaMemcpyHostToDevice, st));
    if (!H.terms.empty()) SP1_CUDA(cudaMemcpyAsync(d_terms, H.terms.data(), H.terms.size() * sizeof(TermDev), cudaMemcpyHostToDevice, st));
    SP1_CUDA(cudaMemsetAsync(d_counts, 0, 8 * 4, st));
    const int nt = (int)tab.size();
    // counts: [0] unbalanced runs, [1] mixed runs, [2] live records, [3] runs, [4] words of the mixed-run records
    uint64_t *d_k0, *d_k1; uint32_t *d_v0, *d_v1;
    SP1_TRY(mem.alloc((void**)&d_k0, (size_t)n * 8)); SP1_TRY(mem.alloc((void**)&d_k1, (size_t)n * 8));
    SP1_TRY(mem.alloc((void**)&d_v0, (size_t)n * 4)); SP1_TRY(mem.alloc((void**)&d_v1, (size_t)n * 4));
    SP1_LAUNCH(ctx, gkr_dbg_records_kernel, blocks_for(n), 256, 0, d_tab, nt, d_inter, d_vcols, d_terms, n, d_k0, d_v0, d_counts + 2);
    cub::DoubleBuffer<uint64_t> kb_(d_k0, d_k1);
    cub::DoubleBuffer<uint32_t> vb_(d_v0, d_v1);
    {
        size_t tb = 0; void* d_tmp = nullptr;
        SP1_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, kb_, vb_, (int)n, 0, 63, st));
        SP1_TRY(mem.alloc(&d_tmp, tb));
        SP1_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, kb_, vb_, (int)n, 0, 63, st));
        ctx->launches++;
    }
    uint32_t cnt[8];
    SP1_CUDA(cudaMemcpyAsync(cnt, d_counts, sizeof(cnt), cudaMemcpyDeviceToHost, st));
    SP1_CUDA(cudaStreamSynchronize(st));
    const uint32_t n_live = cnt[2];
    if (!n_live) { t_all.stop(); emit(); return nullptr; }
    const uint64_t* d_keys = kb_.Current();
    uint64_t* d_agg = kb_.Alternate();
    const uint32_t* d_ranks = vb_.Current();
    uint32_t* d_scratch = vb_.Alternate();   // signed multiplicities by position, then unbalanced-run flags by rank
    SP1_LAUNCH(ctx, gkr_dbg_eval_kernel, blocks_for(n_live), 256, 0, d_tab, nt, d_inter, d_vcols, d_terms, d_keys, d_ranks, n_live, d_scratch);
    {
        auto vals = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), DbgPosValue{d_scratch});
        size_t tb = 0; void* d_tmp = nullptr;
        SP1_CUDA(cub::DeviceReduce::ReduceByKey(nullptr, tb, d_keys, thrust::make_discard_iterator(), vals, d_agg, d_counts + 3, DbgRunOp{}, (int)n_live, st));
        SP1_TRY(mem.alloc(&d_tmp, tb));
        SP1_CUDA(cub::DeviceReduce::ReduceByKey(d_tmp, tb, d_keys, thrust::make_discard_iterator(), vals, d_agg, d_counts + 3, DbgRunOp{}, (int)n_live, st));
        ctx->launches++;
    }
    SP1_CUDA(cudaMemcpyAsync(cnt, d_counts, sizeof(cnt), cudaMemcpyDeviceToHost, st));
    SP1_CUDA(cudaStreamSynchronize(st));
    const uint32_t n_runs = cnt[3];
    constexpr uint32_t MIXED_CAP = 4096, MIXED_WORDS = 1u << 24;
    uint32_t* d_mixed;
    SP1_TRY(mem.alloc((void**)&d_mixed, MIXED_CAP * 4));
    SP1_CUDA(cudaMemsetAsync(d_scratch, 0, (size_t)n * 4, st));
    SP1_LAUNCH(ctx, gkr_dbg_flag_kernel, blocks_for(n_runs), 256, 0, d_agg, n_runs, d_ranks, d_scratch, d_counts, d_mixed, MIXED_CAP);
    SP1_CUDA(cudaMemcpyAsync(cnt, d_counts, sizeof(cnt), cudaMemcpyDeviceToHost, st));
    SP1_CUDA(cudaStreamSynchronize(st));
    const uint32_t n_unb = cnt[0], n_mixed = cnt[1];
    if (n_mixed > MIXED_CAP) return sp1b200_set_error("debug_interactions: %u runs of equal fingerprints mix different keys (at most %u are resolved)", n_mixed, MIXED_CAP);
    n_unbalanced = n_unb;
    // the first max_keys unbalanced runs in rank order: compaction of the flags (run index + 1) into the sort-key buffer, no longer needed
    const uint32_t n_dev = std::min(n_unb, max_keys);
    if (n_dev) {
        uint32_t* d_sel = reinterpret_cast<uint32_t*>(kb_.Current());
        size_t tb = 0; void* d_tmp = nullptr;
        SP1_CUDA(cub::DeviceSelect::If(nullptr, tb, d_scratch, d_sel, d_counts + 5, (int)n, DbgNonZero{}, st));
        SP1_TRY(mem.alloc(&d_tmp, tb));
        SP1_CUDA(cub::DeviceSelect::If(d_tmp, tb, d_scratch, d_sel, d_counts + 5, (int)n, DbgNonZero{}, st));
        ctx->launches++;
        const uint32_t stride = 258 + 2 * (uint32_t)nt, batch = 1024;
        const size_t smem = (size_t)nt * 12;
        if (smem > 48 * 1024) return sp1b200_set_error("debug_interactions: %d chips with interactions exceed the per-key table", nt);
        uint32_t* d_out;
        SP1_TRY(mem.alloc((void**)&d_out, (size_t)std::min(n_dev, batch) * stride * 4));
        std::vector<uint32_t> h((size_t)std::min(n_dev, batch) * stride);
        for (uint32_t b0 = 0; b0 < n_dev; b0 += batch) {
            const uint32_t nb = std::min(batch, n_dev - b0);
            SP1_LAUNCH(ctx, gkr_dbg_key_kernel, nb, 256, smem, d_tab, nt, d_inter, d_vcols, d_terms, d_agg, n_runs, n_live, d_ranks, d_sel + b0, d_out, stride);
            SP1_CUDA(cudaMemcpyAsync(h.data(), d_out, (size_t)nb * stride * 4, cudaMemcpyDeviceToHost, st));
            SP1_CUDA(cudaStreamSynchronize(st));
            for (uint32_t j = 0; j < nb; j++) {
                const uint32_t* o = &h[(size_t)j * stride];
                Key k; k.first_rank = o[257];
                k.w.assign(o, o + 2 + o[1]);
                uint64_t net = 0; uint32_t n_chips = 0;
                for (int t = 0; t < nt; t++) if (o[259 + 2 * t]) { net += o[258 + 2 * t]; n_chips++; }
                k.w.push_back((uint32_t)(net % kb::P)); k.w.push_back(n_chips);
                for (int t = 0; t < nt; t++) if (o[259 + 2 * t]) { k.w.push_back(tab[t].chip); k.w.push_back(o[258 + 2 * t]); }
                keys.push_back(std::move(k));
            }
        }
    }
    // runs whose records do not all share one key: every record back to the host, grouped by full key
    if (n_mixed) {
        uint32_t* d_rec;
        SP1_TRY(mem.alloc((void**)&d_rec, (size_t)MIXED_WORDS * 4));
        SP1_LAUNCH(ctx, gkr_dbg_collect_kernel, n_mixed, 256, 0, d_tab, nt, d_inter, d_vcols, d_terms, d_agg, n_runs, n_live, d_ranks, d_mixed, d_rec,
                   d_counts + 4, MIXED_WORDS);
        SP1_CUDA(cudaMemcpyAsync(cnt, d_counts, sizeof(cnt), cudaMemcpyDeviceToHost, st));
        SP1_CUDA(cudaStreamSynchronize(st));
        if (cnt[4] > MIXED_WORDS) return sp1b200_set_error("debug_interactions: the runs of colliding fingerprints hold %u words of records (at most %u)", cnt[4], MIXED_WORDS);
        std::vector<uint32_t> rec(cnt[4]);
        SP1_CUDA(cudaMemcpyAsync(rec.data(), d_rec, (size_t)cnt[4] * 4, cudaMemcpyDeviceToHost, st));
        SP1_CUDA(cudaStreamSynchronize(st));
        std::vector<const uint32_t*> recs;
        for (size_t o = 0; o < rec.size(); o += 4 + rec[o + 3]) recs.push_back(&rec[o]);
        std::sort(recs.begin(), recs.end(), [](const uint32_t* a, const uint32_t* b) { return a[0] < b[0]; });
        struct Group { uint32_t first_rank; uint64_t net = 0; std::map<uint32_t, uint64_t> chips; };
        std::map<std::vector<uint32_t>, Group> groups;
        for (const uint32_t* r : recs) {
            size_t t = 0;
            while (t + 1 < tab.size() && tab[t + 1].rank0 <= r[0]) t++;
            auto it = groups.emplace(std::vector<uint32_t>(r + 2, r + 4 + r[3]), Group{r[0]}).first;
            it->second.net += r[1];
            it->second.chips[tab[t].chip] += r[1];
        }
        for (auto& [key, g] : groups) {
            if (g.net % kb::P == 0) continue;
            n_unbalanced++;
            Key k; k.first_rank = g.first_rank; k.w = key;
            k.w.push_back((uint32_t)(g.net % kb::P)); k.w.push_back((uint32_t)g.chips.size());
            for (auto& [c, x] : g.chips) { k.w.push_back(c); k.w.push_back((uint32_t)(x % kb::P)); }
            keys.push_back(std::move(k));
        }
    }
    t_all.stop();
    emit();
    return nullptr;
}
