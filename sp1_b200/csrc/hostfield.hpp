// Host-side KoalaBear / ext4 scalar arithmetic used by the library's transcript driver (a few hundred
// operations per proof: batching coefficients, claimed sums, round-polynomial bookkeeping).  Product code,
// independent of oracle/.  Same representation as the device code (Montgomery words).
#pragma once
#include <cstdint>
#include <vector>

namespace hf {

constexpr uint32_t P = 0x7f000001u;
constexpr uint32_t MPRIME = 0x7effffffu;
constexpr uint32_t ONE = 0x01fffffeu;

inline uint32_t reduce(uint64_t x) {
    uint32_t m = (uint32_t)x * MPRIME;
    uint64_t u = x + (uint64_t)m * P;
    uint32_t r = (uint32_t)(u >> 32);
    return r >= P ? r - P : r;
}
inline uint32_t add(uint32_t a, uint32_t b) { uint32_t s = a + b; return s >= P ? s - P : s; }
inline uint32_t sub(uint32_t a, uint32_t b) { return a >= b ? a - b : a + P - b; }
inline uint32_t neg(uint32_t a) { return a ? P - a : 0; }
inline uint32_t mul(uint32_t a, uint32_t b) { return reduce((uint64_t)a * b); }
constexpr uint32_t to_monty(uint64_t c) { return (uint32_t)(((c % P) << 32) % P); }
inline uint32_t from_monty(uint32_t m) { return reduce(m); }
inline uint32_t pow(uint32_t b, uint64_t e) {
    uint32_t r = ONE;
    while (e) { if (e & 1) r = mul(r, b); b = mul(b, b); e >>= 1; }
    return r;
}
inline uint32_t inv(uint32_t a) { return pow(a, P - 2); }

struct E4 {
    uint32_t c[4] = {0, 0, 0, 0};
    static E4 one() { E4 r; r.c[0] = ONE; return r; }
    static E4 from_base(uint32_t a) { E4 r; r.c[0] = a; return r; }
    static E4 load(const uint32_t* p) { E4 r; for (int i = 0; i < 4; i++) r.c[i] = p[i]; return r; }
    void store(uint32_t* p) const { for (int i = 0; i < 4; i++) p[i] = c[i]; }
    bool operator==(const E4& o) const { return c[0] == o.c[0] && c[1] == o.c[1] && c[2] == o.c[2] && c[3] == o.c[3]; }
    bool is_zero() const { return !(c[0] | c[1] | c[2] | c[3]); }
};
inline E4 operator+(const E4& a, const E4& b) { E4 r; for (int i = 0; i < 4; i++) r.c[i] = add(a.c[i], b.c[i]); return r; }
inline E4 operator-(const E4& a, const E4& b) { E4 r; for (int i = 0; i < 4; i++) r.c[i] = sub(a.c[i], b.c[i]); return r; }
inline E4 operator*(const E4& a, uint32_t s) { E4 r; for (int i = 0; i < 4; i++) r.c[i] = mul(a.c[i], s); return r; }
// x < 2 p 2^32 (a sum of up to four products of canonical values) -> canonical x 2^-32 mod p; subtractive Montgomery form
inline uint32_t reduce4(uint64_t x) {
    uint32_t hi = (uint32_t)(x >> 32);
    if (hi >= P) hi -= P;
    const uint32_t m = (uint32_t)x * 0x81000001u;  // lo(x) * p^-1 mod 2^32
    const uint32_t q = (uint32_t)(((uint64_t)m * P) >> 32);
    return hi >= q ? hi - q : hi + P - q;
}
inline E4 operator*(const E4& a, const E4& b) {
    // x^4 = 3 folded into b: every coefficient is one sum of four 62-bit products and one reduction (same form as kb::ext_mul)
    auto tri = [](uint32_t v) { return add(add(v, v), v); };
    const uint64_t a0 = a.c[0], a1 = a.c[1], a2 = a.c[2], a3 = a.c[3];
    const uint64_t b0 = b.c[0], b1 = b.c[1], b2 = b.c[2], b3 = b.c[3];
    const uint64_t t1 = tri(b.c[1]), t2 = tri(b.c[2]), t3 = tri(b.c[3]);
    E4 r;
    r.c[0] = reduce4(a0 * b0 + a1 * t3 + a2 * t2 + a3 * t1);
    r.c[1] = reduce4(a0 * b1 + a1 * b0 + a2 * t3 + a3 * t2);
    r.c[2] = reduce4(a0 * b2 + a1 * b1 + a2 * b0 + a3 * t3);
    r.c[3] = reduce4(a0 * b3 + a1 * b2 + a2 * b1 + a3 * b0);
    return r;
}
// the base-field names for E4, so that code templated on the value type (the constraint interpreter, machine.cuh) takes either
inline E4 add(const E4& a, const E4& b) { return a + b; }
inline E4 sub(const E4& a, const E4& b) { return a - b; }
inline E4 mul(const E4& a, const E4& b) { return a * b; }
inline E4 neg(const E4& a) { return E4() - a; }
inline E4 inv(const E4& a) {
    // Frobenius-free inverse via the tower F[y]/(y^2-3) (y = x^2)
    const uint32_t three = to_monty(3);
    uint32_t A0 = a.c[0], A1 = a.c[2], B0 = a.c[1], B1 = a.c[3];
    uint32_t n0 = sub(add(mul(A0, A0), mul(three, mul(A1, A1))), mul(three, add(mul(B0, B1), mul(B0, B1))));
    uint32_t n1 = sub(add(mul(A0, A1), mul(A0, A1)), add(mul(B0, B0), mul(three, mul(B1, B1))));
    uint32_t d = inv(sub(mul(n0, n0), mul(three, mul(n1, n1))));
    uint32_t i0 = mul(n0, d), i1 = neg(mul(n1, d));
    E4 conj; conj.c[0] = A0; conj.c[1] = neg(B0); conj.c[2] = A1; conj.c[3] = neg(B1);
    E4 s; s.c[0] = i0; s.c[2] = i1;
    return conj * s;
}

// eq(point, i), point[0] <-> MSB of i  (slop/crates/multilinear/src/lagrange.rs:19-45)
inline std::vector<E4> partial_lagrange(const std::vector<E4>& point) {
    std::vector<E4> ev{E4::one()};
    for (const E4& x : point) {
        std::vector<E4> nx(ev.size() * 2);
        for (size_t i = 0; i < ev.size(); i++) {
            E4 pr = ev[i] * x;
            nx[2 * i] = ev[i] - pr;
            nx[2 * i + 1] = pr;
        }
        ev.swap(nx);
    }
    return ev;
}

// Σ_i eq(point, i) · vals[i] over the first min(|vals|, 2^|point|) values: the multilinear extension of vals at point
inline E4 mle_eval(const std::vector<E4>& vals, const std::vector<E4>& point) {
    const std::vector<E4> eq = partial_lagrange(point);
    E4 acc;
    for (size_t i = 0; i < vals.size() && i < eq.size(); i++) acc = acc + eq[i] * vals[i];
    return acc;
}

// Lagrange basis over N distinct nodes, L[i][k] = coefficient of X^k in L_i(X) (degree N-1), with ONE field inversion
// (Montgomery's trick) and no allocation: the transcript drivers call this once per sumcheck round.
template <int N> inline void lagrange_basis(const E4 (&x)[N], E4 (&L)[N][N]) {
    // P(X) = prod_j (X - x_j), monic of degree N
    E4 p[N + 1];
    p[0] = E4::one();
    for (int j = 0; j < N; j++) {           // multiply by (X - x_j)
        p[j + 1] = p[j];
        for (int k = j; k >= 1; k--) p[k] = p[k - 1] - p[k] * x[j];
        p[0] = E4() - p[0] * x[j];
    }
    // den_i = prod_{j != i} (x_i - x_j), all inverted with one inversion
    E4 den[N], pre[N];
    for (int i = 0; i < N; i++) {
        E4 d = E4::one();
        for (int j = 0; j < N; j++) if (j != i) d = d * (x[i] - x[j]);
        den[i] = d;
    }
    pre[0] = den[0];
    for (int i = 1; i < N; i++) pre[i] = pre[i - 1] * den[i];
    E4 acc = inv(pre[N - 1]);
    for (int i = N - 1; i >= 0; i--) {
        const E4 di = i ? acc * pre[i - 1] : acc;  // 1 / den_i
        acc = acc * den[i];
        // Q_i(X) = P(X) / (X - x_i) by synthetic division, scaled by 1/den_i
        E4 q = E4::one();                    // coefficient of X^(N-1)
        L[i][N - 1] = di;
        for (int k = N - 1; k >= 1; k--) { q = p[k] + x[i] * q; L[i][k - 1] = q * di; }
    }
}
template <int N> inline E4 eval_poly(const E4 (&c)[N], const E4& x) { E4 r; for (int i = N; i-- > 0;) r = r * x + c[i]; return r; }

inline unsigned log2_ceil(uint64_t n) { unsigned k = 0; while (((uint64_t)1 << k) < n) k++; return k; }

}  // namespace hf
