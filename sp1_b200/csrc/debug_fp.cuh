// Fingerprint of a LogUp message key (kind = arg_index, n_values, values...) used by the interaction check (gkr.cu) to group
// equal keys with one radix sort.  It is two fixed linear forms over F, L_j(key) = sum_t c_j(t) x_t with x_0 = kind,
// x_1 = n_values, x_(2+i) = value i, packed into 62 bits.  Linearity makes collisions constructible from the coefficients (the
// test suite builds colliding keys through libsp1b200_hostcheck.so); grouping therefore never trusts the fingerprint alone and
// compares full keys inside every run of equal fingerprints.
#pragma once
#include "kb31.cuh"

namespace dbgfp {

// every fingerprint is < 2^62: the sort key of a record with zero multiplicity (dropped from the check) sorts after all of them
constexpr uint64_t NONE = (uint64_t)1 << 62;

// c_j(t): a fixed pseudo-random field element (Montgomery word in [1, p)) for form j in {0, 1} and word position t
KB_HD uint32_t coef(uint32_t j, uint32_t t) {
    uint32_t x = t * 0x9e3779b9u + (j + 1) * 0x85ebca6bu;
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    x %= kb::P;
    return x ? x : 1u;
}

struct Acc {
    uint32_t a = 0, b = 0;
    KB_HD void add(uint32_t t, uint32_t x) {
        a = kb::add(a, kb::mul(coef(0, t), x));
        b = kb::add(b, kb::mul(coef(1, t), x));
    }
    KB_HD void head(uint32_t kind, uint32_t n_values) { add(0, kb::from_canonical(kind)); add(1, kb::from_canonical(n_values)); }
    KB_HD void value(uint32_t i, uint32_t x) { add(2 + i, x); }
    KB_HD uint64_t get() const { return ((uint64_t)a << 31) | b; }
};

KB_HD uint64_t fingerprint(uint32_t kind, uint32_t n_values, const uint32_t* values) {
    Acc f;
    f.head(kind, n_values);
    for (uint32_t i = 0; i < n_values; i++) f.value(i, values[i]);
    return f.get();
}

}  // namespace dbgfp
