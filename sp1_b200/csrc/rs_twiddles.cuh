// Per-pass twiddle table of the radix-8 RS-encode passes (ntt.cu), built once per context next to TH / TL.
// A radix-8 DIF pass whose top stage has 2^s points and whose elements sit 2^(s-3) apart needs, at offset `low` of its block,
//   wA[j] = w^((j 2^(s-3) + low) 2^(24-s))  j < 4,   wB[j] = w^((j 2^(s-3) + low) 2^(25-s))  j < 2,   wC = w^(low 2^(26-s))
// (w = generator of the 2^24-th roots).  Entry (s, low) holds these seven words and a zero in 8 consecutive words at entry index
// 2^(s-3) + low, so that a thread reads its pass's twiddles as two 16-byte loads with no index arithmetic beyond `low`.
// Passes with 4 <= s <= 11 have entries (512 x 32 B = 16 KiB).  __host__ __device__: the CPU suite checks the builder.
#pragma once
#include "kb31.cuh"

namespace rs_tw {

constexpr int MIN_S = 4, MAX_S = 11;
constexpr uint32_t ENTRIES = 1u << (MAX_S - 2);   // index 2^(s-3) + low < 2^(MAX_S-2)
constexpr uint32_t WORDS = 8 * ENTRIES;

// exponent of w in word k of table entry i (0 for the padding word and the unused entries 0 and 1)
KB_HD uint32_t exponent(uint32_t i, int k) {
    if (i < 2 || k == 7) return 0;
    int s = 3;
    while ((i >> (s - 2)) != 0) s++;          // i in [2^(s-3), 2^(s-2))
    const uint32_t stride = 1u << (s - 3), low = i - stride;
    if (k < 4) return (k * stride + low) << (24 - s);
    if (k < 6) return ((k - 4) * stride + low) << (25 - s);
    return low << (26 - s);
}

// word k of entry i in Montgomery form
KB_HD uint32_t word(uint32_t i, int k) {
    if (i < 2 || k == 7) return 0;
    const uint32_t w = kb::pow(kb::to_monty_c(3), 127);
    return kb::pow(w, exponent(i, k));
}

}  // namespace rs_tw
