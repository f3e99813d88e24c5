// Septic extension F_p^7 = F_p[z]/(z^7 - 3z - 5) over KoalaBear and the curve y^2 = x^3 + 45x + 41z^3 over it, on the device, for
// the program setup (setup.cu): the hash-to-curve SepticCurve::lift_x and the complete addition law of SepticCurveComplete
// (crates/hypercube/src/septic_extension.rs, septic_curve.rs).  Every lift takes a square test and usually a square root, so the
// Frobenius maps are table-driven (49 products each) and the reciprocal goes through the norm; the host-only septic.hpp serves the
// verifier's few hundred operations with a Fermat-power inverse instead.  Montgomery words, like kb31.cuh; __host__ __device__ so
// that the CPU suite runs the same source through libsp1b200_hostcheck.so.
#pragma once
#include "kb31.cuh"
#include "poseidon2.cuh"

namespace s7 {

struct E7 { uint32_t c[7]; };
struct Pt { E7 x, y; };   // (0, 0) is not on the curve (41 z^3 != 0): it stands for the point at infinity

// ---- Frobenius tables, derived at compile time in canonical integers -------------------------------------------------------------
// FROB[i] = z^(i p), DFROB[i] = z^(i p^2), i = 0..6, so that a^p = sum a_i FROB[i] and a^(p^2) = sum a_i DFROB[i].
struct C7 { uint64_t c[7]; };
__host__ __device__ constexpr C7 c7_mul(const C7& a, const C7& b) {
    uint64_t t[13] = {};
    for (int i = 0; i < 7; i++)
        for (int j = 0; j < 7; j++) t[i + j] = (t[i + j] + a.c[i] * b.c[j]) % kb::P;
    for (int k = 12; k >= 7; k--) {   // z^k = z^(k-7) (3z + 5)
        t[k - 6] = (t[k - 6] + 3 * t[k]) % kb::P;
        t[k - 7] = (t[k - 7] + 5 * t[k]) % kb::P;
    }
    C7 r{};
    for (int i = 0; i < 7; i++) r.c[i] = t[i];
    return r;
}
__host__ __device__ constexpr C7 c7_pow(C7 b, uint64_t e) {
    C7 r{{1, 0, 0, 0, 0, 0, 0}};
    while (e) { if (e & 1) r = c7_mul(r, b); b = c7_mul(b, b); e >>= 1; }
    return r;
}
struct FrobTable { uint32_t v[7][7]; };
__host__ __device__ constexpr FrobTable make_frob(int k) {   // k = 1: z^(i p); k = 2: z^(i p^2)
    C7 zq{{0, 1, 0, 0, 0, 0, 0}};
    for (int t = 0; t < k; t++) zq = c7_pow(zq, kb::P);
    FrobTable f{};
    C7 cur{{1, 0, 0, 0, 0, 0, 0}};
    for (int i = 0; i < 7; i++) {
        for (int j = 0; j < 7; j++) f.v[i][j] = kb::to_monty_c(cur.c[j]);
        cur = c7_mul(cur, zq);
    }
    return f;
}
static __constant__ FrobTable FROB = make_frob(1);
static __constant__ FrobTable DFROB = make_frob(2);
constexpr FrobTable FROB_HOST = make_frob(1);
constexpr FrobTable DFROB_HOST = make_frob(2);
#ifdef __CUDA_ARCH__
#define S7_FROB s7::FROB
#define S7_DFROB s7::DFROB
#else
#define S7_FROB s7::FROB_HOST
#define S7_DFROB s7::DFROB_HOST
#endif

// ---- field -----------------------------------------------------------------------------------------------------------------------
KB_HD E7 zero() { return E7{{0, 0, 0, 0, 0, 0, 0}}; }
KB_HD E7 add(const E7& a, const E7& b) { E7 r; for (int i = 0; i < 7; i++) r.c[i] = kb::add(a.c[i], b.c[i]); return r; }
KB_HD E7 sub(const E7& a, const E7& b) { E7 r; for (int i = 0; i < 7; i++) r.c[i] = kb::sub(a.c[i], b.c[i]); return r; }
KB_HD E7 neg(const E7& a) { E7 r; for (int i = 0; i < 7; i++) r.c[i] = kb::neg(a.c[i]); return r; }
KB_HD E7 scale(const E7& a, uint32_t s) { E7 r; for (int i = 0; i < 7; i++) r.c[i] = kb::mul(a.c[i], s); return r; }
KB_HD bool is_zero(const E7& a) { uint32_t o = 0; for (int i = 0; i < 7; i++) o |= a.c[i]; return o == 0; }
KB_HD bool eq(const E7& a, const E7& b) { uint32_t o = 0; for (int i = 0; i < 7; i++) o |= a.c[i] ^ b.c[i]; return o == 0; }

// Every coefficient is a sum of up to seven products of canonical words: accumulated four at a time in 64 bits (4 (p-1)^2 < 2p 2^32)
// and reduced once per group (monty_reduce2).  z^(7+k) = 5 z^k + 3 z^(k+1) folds the top six coefficients with additions only.
KB_HD E7 mul(const E7& a, const E7& b) {
    uint32_t t[13];
#pragma unroll
    for (int k = 0; k < 13; k++) {
        uint64_t acc = 0;
        uint32_t r = 0;
        int n = 0;
#pragma unroll
        for (int i = 0; i < 7; i++) {
            const int j = k - i;
            if (j < 0 || j > 6) continue;
            acc += (uint64_t)a.c[i] * b.c[j];
            if (++n == 4) { r = kb::monty_reduce2(acc); acc = 0; }
        }
        t[k] = n > 4 ? kb::add(r, kb::monty_reduce2(acc)) : n == 4 ? r : kb::monty_reduce2(acc);
    }
    E7 o;
#pragma unroll
    for (int i = 0; i < 7; i++) o.c[i] = t[i];
#pragma unroll
    for (int k = 7; k < 13; k++) {
        const uint32_t x = t[k], x2 = kb::dbl(x);
        o.c[k - 7] = kb::add(o.c[k - 7], kb::add(kb::dbl(x2), x));
        o.c[k - 6] = kb::add(o.c[k - 6], kb::add(x2, x));
    }
    return o;
}
KB_HD E7 sqr(const E7& a) { return mul(a, a); }

// sum_i a_i T[i]
KB_HD E7 lin(const E7& a, const FrobTable& T) {
    E7 r;
#pragma unroll
    for (int j = 0; j < 7; j++) {
        uint64_t lo = 0, hi = 0;
#pragma unroll
        for (int i = 0; i < 4; i++) lo += (uint64_t)a.c[i] * T.v[i][j];
#pragma unroll
        for (int i = 4; i < 7; i++) hi += (uint64_t)a.c[i] * T.v[i][j];
        r.c[j] = kb::add(kb::monty_reduce2(lo), kb::monty_reduce2(hi));
    }
    return r;
}
KB_HD E7 frobenius(const E7& a) { return lin(a, S7_FROB); }
KB_HD E7 double_frobenius(const E7& a) { return lin(a, S7_DFROB); }

// a^(r - 1), r = 1 + p + ... + p^6: (a^p a^(p^2)) (a^p a^(p^2))^(p^2) (a^p a^(p^2))^(p^4)
KB_HD E7 pow_r_1(const E7& a) {
    const E7 base = mul(frobenius(a), double_frobenius(a));
    const E7 b2 = double_frobenius(base), b4 = double_frobenius(b2);
    return mul(mul(base, b2), b4);
}
// the norm a^r, an element of the base field
KB_HD uint32_t pow_r(const E7& a) { return mul(pow_r_1(a), a).c[0]; }
// a^-1 = a^(r-1) / a^r; the zero element maps to zero
KB_HD E7 inv(const E7& a) {
    const E7 q = pow_r_1(a);
    return scale(q, kb::inv(mul(q, a).c[0]));
}

KB_HD bool base_is_square(uint32_t n) { return kb::pow(n, (kb::P - 1) >> 1) == kb::ONE; }

// A square root of a, given its norm n = a^r (a square: n is a square of F_p).  With a^((p+1)/2)^(p + p^3 + p^5) a squared =
// a^(p + ... + p^6) a^2 = n a, the root is a^((p+1)/2 (p + p^3 + p^5)) a / sqrt(n), and sqrt(1/n) comes from Cipolla's method in
// F_p[sqrt(c^2 - 1/n)] with the first c = 3^k whose c^2 - 1/n is not a square (septic_extension.rs:634-681).
KB_HD E7 sqrt(const E7& a, uint32_t n) {
    if (is_zero(a)) return a;
    E7 it = a, pw = a;
    for (int i = 1; i < 30; i++) {   // pw = a^(1 + 2^23 + ... + 2^29) = a^((p+1)/2)
        it = sqr(it);
        if (i >= 23) pw = mul(pw, it);
    }
    E7 f = frobenius(pw), den = f;
    f = double_frobenius(f); den = mul(den, f);
    f = double_frobenius(f); den = mul(den, f);
    den = mul(den, a);
    const uint32_t base = kb::inv(n), g = kb::to_monty_c(3);
    uint32_t c = kb::ONE, nr = kb::sub(kb::ONE, base);
    while (kb::pow(nr, (kb::P - 1) >> 1) == kb::ONE) {
        c = kb::mul(c, g);
        nr = kb::sub(kb::sqr(c), base);
    }
    // (c + w)^((p+1)/2) with w^2 = nr
    uint32_t rr = kb::ONE, ri = 0, br = c, bi = kb::ONE;
    for (uint32_t e = (kb::P + 1) >> 1; e; e >>= 1) {
        if (e & 1) {
            const uint32_t t = kb::add(kb::mul(rr, br), kb::mul(nr, kb::mul(ri, bi)));
            ri = kb::add(kb::mul(rr, bi), kb::mul(ri, br));
            rr = t;
        }
        const uint32_t t = kb::add(kb::sqr(br), kb::mul(nr, kb::sqr(bi)));
        bi = kb::dbl(kb::mul(br, bi));
        br = t;
    }
    return scale(den, rr);
}

// x^3 + 45 x + 41 z^3
KB_HD E7 curve_formula(const E7& x) {
    E7 r = add(mul(sqr(x), x), scale(x, kb::to_monty_c(45)));
    r.c[3] = kb::add(r.c[3], kb::to_monty_c(41));
    return r;
}
// the y-coordinate's limb 6 (canonical) classifies a digest: receive [1, 63 2^24], send [p - 63 2^24, p - 1], anything else cannot
// represent an interaction (septic_extension.rs:686-705)
constexpr uint32_t LIMB6_RANGE = 63u << 24;
KB_HD bool is_send(const E7& y) { return kb::to_canonical(y.c[6]) >= kb::P - LIMB6_RANGE; }
KB_HD bool is_exception(const E7& y) {
    const uint32_t l = kb::to_canonical(y.c[6]);
    return l == 0 || (l > LIMB6_RANGE && l < kb::P - LIMB6_RANGE);
}

// ---- curve -----------------------------------------------------------------------------------------------------------------------
// SepticCurve::lift_x (septic_curve.rs:124-164): for offset = 0, 1, ...: x = the first seven words of the Poseidon2 permutation of
// [m_0 .. m_6, m_7 + offset 2^16, 0^8]; the first x with a square x^3 + 45x + 41z^3 whose root y is not an exception gives the point
// (x, y) with y normalised not to be a send.  m: Montgomery words.  Returns the offset, or -1 when none of the 256 has a point.
KB_HD int lift_x(const uint32_t (&m)[8], Pt& out) {
    for (int off = 0; off < 256; off++) {
        uint32_t s[16];
#pragma unroll
        for (int i = 0; i < 7; i++) s[i] = m[i];
        s[7] = kb::add(m[7], kb::from_canonical((uint32_t)off << 16));
#pragma unroll
        for (int i = 8; i < 16; i++) s[i] = 0;
        p2::permute(s);
        E7 x;
#pragma unroll
        for (int i = 0; i < 7; i++) x.c[i] = s[i];
        const E7 y2 = curve_formula(x);
        const uint32_t n = pow_r(y2);
        if (!base_is_square(n)) continue;   // also y2 = 0, whose root would be an exception
        E7 y = sqrt(y2, n);
        if (is_exception(y)) continue;
        if (is_send(y)) y = neg(y);
        out = Pt{x, y};
        return off;
    }
    return -1;
}

KB_HD Pt infinity() { return Pt{zero(), zero()}; }
KB_HD bool is_infinity(const Pt& p) { return is_zero(p.x) && is_zero(p.y); }
KB_HD Pt neg(const Pt& p) { return Pt{p.x, neg(p.y)}; }

// SepticCurveComplete + SepticCurveComplete (septic_curve.rs:212-231): infinity is the identity, the chord for distinct x, the
// tangent for p = q, infinity for p = -q
KB_HD Pt add_complete(const Pt& p, const Pt& q) {
    if (is_infinity(p)) return q;
    if (is_infinity(q)) return p;
    const E7 dx = sub(q.x, p.x);
    E7 slope;
    if (is_zero(dx)) {
        if (!eq(p.y, q.y)) return infinity();
        const E7 x2 = sqr(p.x);
        E7 num = add(add(x2, x2), x2);
        num.c[0] = kb::add(num.c[0], kb::to_monty_c(45));
        slope = mul(num, inv(add(p.y, p.y)));
    } else {
        slope = mul(sub(q.y, p.y), inv(dx));
    }
    Pt r;
    r.x = sub(sub(sqr(slope), p.x), q.x);
    r.y = sub(mul(slope, sub(p.x, r.x)), p.y);
    return r;
}

// SepticDigest::zero() (CURVE_CUMULATIVE_SUM_START), Montgomery words
KB_HD Pt digest_zero() {
    constexpr uint32_t x[7] = {0x1414213, 0x5623730, 0x9504880, 0x1688724, 0x2096980, 0x7856967, 0x1875376};
    constexpr uint32_t y[7] = {2020310104, 1513506566, 1843922297, 2003644209, 805967281, 1882435203, 1623804682};
    Pt p;
    for (int i = 0; i < 7; i++) { p.x.c[i] = kb::to_monty_c(x[i]); p.y.c[i] = kb::to_monty_c(y[i]); }
    return p;
}

// the lift_x messages of Program::initial_global_cumulative_sum (crates/core/executor/src/program.rs:175-221), Montgomery words.
// Memory (InteractionKind 1): [1 << 24, 0, addr limbs 0..16 / 16..32 / 32..48, word bytes as two 16+8-bit limbs, word bits 48..64]
KB_HD void memory_message(uint64_t addr, uint64_t w, uint32_t (&m)[8]) {
    const uint32_t v[8] = {1u << 24, 0, (uint32_t)(addr & 0xFFFF), (uint32_t)((addr >> 16) & 0xFFFF), (uint32_t)((addr >> 32) & 0xFFFF),
                           (uint32_t)(w & 0xFFFF) + (1u << 16) * (uint32_t)((w >> 32) & 0xFF),
                           (uint32_t)((w >> 16) & 0xFFFF) + (1u << 16) * (uint32_t)((w >> 40) & 0xFF), (uint32_t)((w >> 48) & 0xFFFF)};
    for (int i = 0; i < 8; i++) m[i] = kb::from_canonical(v[i]);
}
// PageProtAccess (InteractionKind 19): [19 << 24, 0, split_page_idx(idx) (4 / 16 / 16 bits, crates/primitives/src/consts.rs:218-220),
// prot, 0, 0]
KB_HD void page_message(uint64_t idx, uint8_t prot, uint32_t (&m)[8]) {
    const uint32_t v[8] = {19u << 24, 0, (uint32_t)(idx & 0xF), (uint32_t)((idx >> 4) & 0xFFFF), (uint32_t)((idx >> 20) & 0xFFFF), prot, 0, 0};
    for (int i = 0; i < 8; i++) m[i] = kb::from_canonical(v[i]);
}

}  // namespace s7
