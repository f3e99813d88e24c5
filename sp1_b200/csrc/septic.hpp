// Septic extension F_p^7 = F_p[z]/(z^7 - 3z - 5) over KoalaBear and the curve y^2 = x^3 + 45x + 41z^3 over it
// (crates/hypercube/src/septic_extension.rs, septic_curve.rs, septic_digest.rs).  The core-proof verifier sums the shards' global
// cumulative sums with it: a few hundred field operations per shard, host only.  Montgomery words, like hostfield.hpp.
#pragma once
#include "hostfield.hpp"

namespace sep {

struct E7 {
    uint32_t c[7] = {0, 0, 0, 0, 0, 0, 0};
    static E7 from_base(uint32_t a) { E7 r; r.c[0] = a; return r; }
    static E7 one() { return from_base(hf::ONE); }
    static E7 load(const uint32_t* p) { E7 r; for (int i = 0; i < 7; i++) r.c[i] = p[i]; return r; }
    void store(uint32_t* p) const { for (int i = 0; i < 7; i++) p[i] = c[i]; }
    bool operator==(const E7& o) const { for (int i = 0; i < 7; i++) if (c[i] != o.c[i]) return false; return true; }
    bool is_zero() const { for (int i = 0; i < 7; i++) if (c[i]) return false; return true; }
};
inline E7 operator+(const E7& a, const E7& b) { E7 r; for (int i = 0; i < 7; i++) r.c[i] = hf::add(a.c[i], b.c[i]); return r; }
inline E7 operator-(const E7& a, const E7& b) { E7 r; for (int i = 0; i < 7; i++) r.c[i] = hf::sub(a.c[i], b.c[i]); return r; }
inline E7 operator-(const E7& a) { E7 r; for (int i = 0; i < 7; i++) r.c[i] = hf::neg(a.c[i]); return r; }
inline E7 operator*(const E7& a, uint32_t s) { E7 r; for (int i = 0; i < 7; i++) r.c[i] = hf::mul(a.c[i], s); return r; }
inline E7 operator*(const E7& a, const E7& b) {
    uint32_t t[13] = {0};
    for (int i = 0; i < 7; i++)
        for (int j = 0; j < 7; j++) t[i + j] = hf::add(t[i + j], hf::mul(a.c[i], b.c[j]));
    // z^(7+k) = 5 z^k + 3 z^(k+1), k + 1 <= 6
    constexpr uint32_t three = hf::to_monty(3), five = hf::to_monty(5);
    E7 r;
    for (int i = 0; i < 7; i++) r.c[i] = t[i];
    for (int i = 7; i < 13; i++) {
        r.c[i - 7] = hf::add(r.c[i - 7], hf::mul(t[i], five));
        r.c[i - 6] = hf::add(r.c[i - 6], hf::mul(t[i], three));
    }
    return r;
}
inline E7 pow(E7 b, uint64_t e) {
    E7 r = E7::one();
    while (e) { if (e & 1) r = r * b; b = b * b; e >>= 1; }
    return r;
}
// a^-1 = a^(r-1) / N(a), r = 1 + p + ... + p^6: a^(r-1) is the product of the six Frobenius conjugates a^(p^i), and the norm
// N(a) = a^r lies in the base field.  The zero element has no inverse; inv(0) returns 0.
inline E7 inv(const E7& a) {
    E7 conj = E7::one(), f = a;
    for (int i = 1; i < 7; i++) { f = pow(f, hf::P); conj = conj * f; }
    const E7 n = a * conj;
    return conj * (n.c[0] ? hf::inv(n.c[0]) : 0u);
}

struct Point { E7 x, y; };

// y^2 - (x^3 + 45 x + 41 z^3): zero on the curve
inline E7 curve_residual(const Point& p) {
    E7 b; b.c[3] = hf::to_monty(41);
    return p.y * p.y - (p.x * p.x * p.x + p.x * hf::to_monty(45) + b);
}

// SepticCurve::add_incomplete: the chord through p and q.  Returns false (and leaves r alone) on the exceptional case x_p == x_q,
// where the reference divides by zero and panics.
inline bool add_incomplete(const Point& p, const Point& q, Point& r) {
    const E7 dx = q.x - p.x;
    if (dx.is_zero()) return false;
    const E7 slope = (q.y - p.y) * inv(dx);
    Point o;
    o.x = slope * slope - p.x - q.x;
    o.y = slope * (p.x - o.x) - p.y;
    r = o;
    return true;
}
inline bool sub_incomplete(const Point& p, const Point& q, Point& r) { return add_incomplete(p, Point{q.x, -q.y}, r); }

inline Point point_from_canonical(const uint32_t (&x)[7], const uint32_t (&y)[7]) {
    Point p;
    for (int i = 0; i < 7; i++) { p.x.c[i] = hf::to_monty(x[i]); p.y.c[i] = hf::to_monty(y[i]); }
    return p;
}
// CURVE_CUMULATIVE_SUM_START (from sqrt 2): SepticDigest::zero()
inline Point digest_zero() {
    static const uint32_t x[7] = {0x1414213, 0x5623730, 0x9504880, 0x1688724, 0x2096980, 0x7856967, 0x1875376};
    static const uint32_t y[7] = {2020310104, 1513506566, 1843922297, 2003644209, 805967281, 1882435203, 1623804682};
    return point_from_canonical(x, y);
}
// DIGEST_SUM_START (from sqrt 3): SepticDigest::starting_digest()
inline Point digest_start() {
    static const uint32_t x[7] = {0x1732050, 0x8075688, 0x7729352, 0x7446341, 0x5058723, 0x6694280, 0x5253810};
    static const uint32_t y[7] = {1095433104, 7540207, 1124564165, 2035506693, 11121645, 102781365, 398772161};
    return point_from_canonical(x, y);
}
// CURVE_WITNESS_DUMMY_POINT (from e): SepticCurve::dummy()
inline Point dummy_point() {
    static const uint32_t x[7] = {0x2718281 + (1 << 24), 0x8284590, 0x4523536, 0x0287471, 0x3526624, 0x9775724, 0x7093699};
    static const uint32_t y[7] = {1250555984, 1592495468, 656721246, 420301347, 2125819749, 819876460, 17687681};
    return point_from_canonical(x, y);
}
inline bool is_zero_digest(const Point& p) { const Point z = digest_zero(); return p.x == z.x && p.y == z.y; }

// SepticDigest + SepticDigest (septic_digest.rs:67-83): start + (a - zero) + (b - zero) + zero - start, one incomplete addition at a
// time.  Returns false when one of them meets the exceptional case.
inline bool digest_add(const Point& a, const Point& b, Point& r) {
    const Point start = digest_start(), zero = digest_zero();
    Point s;
    return add_incomplete(start, a, s) && sub_incomplete(s, zero, s) && add_incomplete(s, b, s) && sub_incomplete(s, zero, s) &&
           add_incomplete(s, zero, s) && sub_incomplete(s, start, s) && (r = s, true);
}

}  // namespace sep
