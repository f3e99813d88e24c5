// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header).  Restates, for the tests of sp1b200_program_vk_tail, on the septic
// extension and curve of core.hpp:
//   crates/hypercube/src/septic_extension.rs:583-705   frobenius / double_frobenius, pow_r_1, inv, is_square, sqrt, is_send / is_exception
//   crates/hypercube/src/septic_curve.rs:100-164       curve_formula, lift_x;  :75-81 double;  :212-231 SepticCurveComplete + (complete law)
//   crates/core/executor/src/program.rs:170-229        Program::initial_global_cumulative_sum (its messages; split_page_idx from
//                                                      crates/primitives/src/consts.rs:218-220)
#pragma once
#include "core.hpp"
#include "poseidon2.hpp"
#include <vector>

namespace orc {

// ---- lift_x and the initial global cumulative sum ---------------------------------------------------------------------------------
// z_pow_p(i) = z^(i p) and z_pow_p2(i) = z^(i p^2) (septic_extension.rs tables), computed here from their definition
inline S7 s7_pow(S7 b, uint64_t e) {
    S7 r = S7::base(F::one());
    while (e) { if (e & 1) r = r * b; b = b * b; e >>= 1; }
    return r;
}
struct FrobConsts {
    S7 p1[7], p2[7];
    FrobConsts() {
        S7 z; z.c[1] = F::one();
        const S7 zp = s7_pow(z, KB_P), zp2 = s7_pow(zp, KB_P);
        p1[0] = p2[0] = S7::base(F::one());
        for (int i = 1; i < 7; i++) { p1[i] = p1[i - 1] * zp; p2[i] = p2[i - 1] * zp2; }
    }
};
inline const FrobConsts& frob_consts() { static const FrobConsts c; return c; }
inline S7 s7_scale(const S7& a, F s) { S7 r; for (int i = 0; i < 7; i++) r.c[i] = a.c[i] * s; return r; }
inline S7 frobenius(const S7& a) {            // :583-593
    S7 r = S7::base(a.c[0]);
    for (int i = 1; i < 7; i++) r = r + s7_scale(frob_consts().p1[i], a.c[i]);
    return r;
}
inline S7 double_frobenius(const S7& a) {     // :596-606
    S7 r = S7::base(a.c[0]);
    for (int i = 1; i < 7; i++) r = r + s7_scale(frob_consts().p2[i], a.c[i]);
    return r;
}
inline S7 pow_r_1(const S7& a) {              // :609-614
    const S7 base = frobenius(a) * double_frobenius(a);
    const S7 b2 = double_frobenius(base), b4 = double_frobenius(b2);
    return base * b2 * b4;
}
inline S7 s7_inv_norm(const S7& a) {          // :617-621 (a != 0)
    const S7 q = pow_r_1(a);
    return s7_scale(q, (q * a).c[0].inv());
}
inline bool is_square(const S7& a, F& norm) { // :623-630
    norm = (pow_r_1(a) * a).c[0];
    return norm.pow((KB_P - 1) / 2) == F::one();
}
// :634-681; F::generator() of KoalaBear is 3
inline bool s7_sqrt(const S7& n, S7& out) {
    if (n.is_zero() || n == S7::base(F::one())) { out = n; return true; }
    F numerator;
    if (!is_square(n, numerator)) return false;
    S7 it = n, pw = n;
    for (int i = 1; i < 30; i++) { it = it * it; if (i >= 23) pw = pw * it; }
    S7 f = frobenius(pw), den = f;
    f = double_frobenius(f); den = den * f;
    f = double_frobenius(f); den = den * f;
    den = den * n;
    const F base = numerator.inv(), g = F::from_canonical(3);
    F a = F::one(), nr = F::one() - base;
    while (nr.pow((KB_P - 1) / 2) == F::one()) { a = a * g; nr = a * a - base; }
    F rr = F::one(), ri = F::zero(), br = a, bi = F::one();   // CipollaExtension::pow, :731-743
    for (uint64_t e = ((uint64_t)KB_P + 1) / 2; e; e >>= 1) {
        if (e & 1) { const F t = rr * br + nr * ri * bi; ri = rr * bi + ri * br; rr = t; }
        const F t = br * br + nr * bi * bi; bi = br * bi + bi * br; br = t;
    }
    out = s7_scale(den, rr);
    return true;
}
inline S7 curve_formula(const S7& x) {        // septic_curve.rs:100-112
    S7 b; b.c[3] = F::from_canonical(41);
    return x * x * x + s7_scale(x, F::from_canonical(45)) + b;
}
inline uint32_t limb6(const S7& y) { return y.c[6].canonical(); }
inline bool is_send(const S7& y) { return limb6(y) >= KB_P - 63u * (1u << 24); }   // :694-697
inline bool is_exception(const S7& y) {                                             // :701-705
    const uint32_t l = limb6(y);
    return l == 0 || (63u * (1u << 24) < l && l < KB_P - 63u * (1u << 24));
}
// septic_curve.rs:124-164: -> the offset, or -1 where the reference panics
inline int lift_x(const F (&m)[8], SPoint& out) {
    for (int off = 0; off < 256; off++) {
        F s[16];
        for (int i = 0; i < 8; i++) s[i] = m[i];
        s[7] = m[7] + F::from_canonical(1u << 16) * F::from_canonical((uint32_t)off);
        poseidon2_permute(s);
        S7 x;
        for (int i = 0; i < 7; i++) x.c[i] = s[i];
        S7 y;
        if (!s7_sqrt(curve_formula(x), y)) continue;
        if (is_exception(y)) continue;
        out = SPoint{x, is_send(y) ? -y : y};
        return off;
    }
    return -1;
}
// SepticCurveComplete<F>
struct CPoint { bool inf = true; SPoint p; };
inline CPoint c_add(const CPoint& a, const CPoint& b) {   // septic_curve.rs:212-231
    if (a.inf) return b;
    if (b.inf) return a;
    const SPoint &p = a.p, &q = b.p;
    CPoint r; r.inf = false;
    if (!(p.x == q.x)) {                                   // add_incomplete, :58-63
        const S7 l = (q.y - p.y) * s7_inv_norm(q.x - p.x);
        r.p.x = l * l - p.x - q.x;
        r.p.y = l * (p.x - r.p.x) - p.y;
        return r;
    }
    if (!(p.y == q.y)) return CPoint{};
    const S7 l = (s7_scale(p.x * p.x, F::from_canonical(3)) + S7::base(F::from_canonical(45))) * s7_inv_norm(s7_scale(p.y, F::two()));   // double, :75-81
    r.p.x = l * l - s7_scale(p.x, F::two());
    r.p.y = l * (p.x - r.p.x) - p.y;
    return r;
}
// program.rs:175-221 messages
inline void memory_message(uint64_t addr, uint64_t w, F (&m)[8]) {
    const uint32_t limb1 = (uint32_t)(w & 0xFFFF) + (1u << 16) * (uint32_t)((w >> 32) & 0xFF);
    const uint32_t limb2 = (uint32_t)((w >> 16) & 0xFFFF) + (1u << 16) * (uint32_t)((w >> 40) & 0xFF);
    const uint32_t v[8] = {1u << 24, 0, (uint32_t)(addr & 0xFFFF), (uint32_t)((addr >> 16) & 0xFFFF), (uint32_t)((addr >> 32) & 0xFFFF), limb1,
                           limb2, (uint32_t)((w >> 48) & 0xFFFF)};
    for (int i = 0; i < 8; i++) m[i] = F::from_canonical(v[i]);
}
inline void page_message(uint64_t idx, uint8_t prot, F (&m)[8]) {
    const uint32_t v[8] = {19u << 24, 0, (uint32_t)(idx & 0xF), (uint32_t)((idx >> 4) & 0xFFFF), (uint32_t)((idx >> 20) & 0xFFFF), prot, 0, 0};
    for (int i = 0; i < 8; i++) m[i] = F::from_canonical(v[i]);
}
// program.rs:170-229: -> 0 and the sum, 1 when an entry has no point (*bad = its index), 2 when the sum is at infinity.  The lifts and
// the sum run on all OpenMP threads (any order of the group sum gives the same point).
inline int initial_global_cumulative_sum(const uint64_t* addrs, const uint64_t* words, uint64_t n_mem, const uint64_t* pages, const uint8_t* prots,
                                         uint64_t n_pages, bool untrusted, SPoint& out, uint64_t* bad) {
    const uint64_t n = n_mem + (untrusted ? n_pages : 0);
    std::vector<CPoint> pts(n + 1);
    int64_t first_bad = -1;
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        F m[8];
        if ((uint64_t)i < n_mem) memory_message(addrs[i], words[i], m);
        else page_message(pages[i - n_mem], prots[i - n_mem], m);
        SPoint p;
        if (lift_x(m, p) < 0) {
#pragma omp critical
            if (first_bad < 0 || i < first_bad) first_bad = i;
            continue;
        }
        pts[i].inf = false;
        pts[i].p = SPoint{p.x, -p.y};
    }
    if (first_bad >= 0) { *bad = (uint64_t)first_bad; return 1; }
    pts[n].inf = false;
    pts[n].p = digest_zero();
    std::vector<CPoint> part;
#pragma omp parallel
    {
        CPoint acc;
#pragma omp for schedule(static) nowait
        for (int64_t i = 0; i <= (int64_t)n; i++) acc = c_add(acc, pts[i]);
#pragma omp critical
        part.push_back(acc);
    }
    CPoint sum;
    for (const CPoint& c : part) sum = c_add(sum, c);
    if (sum.inf) return 2;
    out = sum.p;
    return 0;
}

}  // namespace orc
