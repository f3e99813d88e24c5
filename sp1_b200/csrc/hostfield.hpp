// Host-side extension-field helpers for the library's transcript drivers (a few hundred operations per proof: batching coefficients,
// claimed sums, round-polynomial bookkeeping).  The arithmetic itself is the device code's (kb31.cuh, __host__ __device__); this adds
// host conveniences on top of it.  Product code, independent of oracle/.
#pragma once
#include "kb31.cuh"
#include <cstddef>
#include <cstdint>
#include <vector>

namespace hf {

// kb::Ext with value semantics for host code: default-constructed to zero, and operators.  Passes wherever a kernel takes a kb::Ext.
struct E4 : kb::Ext {
    E4() : kb::Ext{{0, 0, 0, 0}} {}
    E4(const kb::Ext& e) : kb::Ext(e) {}
    static E4 one() { return kb::ext_one(); }
    static E4 from_base(uint32_t a) { return kb::ext_from_base(a); }
    // word by word: host buffers (caller arrays, proof words at odd offsets) are only 4-byte aligned, and kb::ext_load reads a uint4
    static E4 load(const uint32_t* p) { E4 r; for (int i = 0; i < 4; i++) r.c[i] = p[i]; return r; }
    void store(uint32_t* p) const { for (int i = 0; i < 4; i++) p[i] = c[i]; }
    bool operator==(const E4& o) const { return kb::ext_eq(*this, o); }
    bool is_zero() const { return !(c[0] | c[1] | c[2] | c[3]); }
};
inline E4 operator+(const E4& a, const E4& b) { return kb::ext_add(a, b); }
inline E4 operator-(const E4& a, const E4& b) { return kb::ext_sub(a, b); }
inline E4 operator-(const E4& a) { return kb::ext_neg(a); }
inline E4 operator*(const E4& a, const E4& b) { return kb::ext_mul(a, b); }
inline E4 operator*(const E4& a, uint32_t s) { return kb::ext_mul_base(a, s); }

// every word is a canonical Montgomery word (< p)
inline bool canonical(const uint32_t* w, size_t n) { for (size_t i = 0; i < n; i++) if (w[i] >= kb::P) return false; return true; }

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
    E4 acc = kb::ext_inv(pre[N - 1]);
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
