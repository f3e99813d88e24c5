// Host execution of the DEVICE arithmetic sources (kb31.cuh / poseidon2.cuh are __host__ __device__): lets the CPU
// test-suite check the exact code the kernels run (lazy-reduction bounds, half-product Montgomery forms) against the
// oracle before any GPU time is spent.  Test support only; not part of include/sp1b200.h.
#include "poseidon2.cuh"
#include "rs_twiddles.cuh"
#include "debug_fp.cuh"
#include "hostfield.hpp"
#include "septic.cuh"
#include "sumcheck.cuh"
#include "zc_lower.hpp"
#include <cstring>
#include <type_traits>

extern "C" {
void sp1b200_hostcheck_permute(uint32_t* states, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        uint32_t s[16];
        for (int k = 0; k < 16; k++) s[k] = states[i * 16 + k];
        p2::permute(s);
        for (int k = 0; k < 16; k++) states[i * 16 + k] = s[k];
    }
}
// every instruction-selection mode of the permutation (poseidon2.cuh, permute_m<MODE>); returns 0 for an unknown mode
int sp1b200_hostcheck_permute_mode(uint32_t* states, uint64_t n, int mode) {
    for (uint64_t i = 0; i < n; i++) {
        uint32_t s[16];
        for (int k = 0; k < 16; k++) s[k] = states[i * 16 + k];
        switch (mode) {
#define P2_CASE(M) case M: p2::permute_m<M>(s); break;
            P2_CASE(0) P2_CASE(1) P2_CASE(2) P2_CASE(3) P2_CASE(4) P2_CASE(5) P2_CASE(6) P2_CASE(7)
            P2_CASE(8) P2_CASE(9) P2_CASE(10) P2_CASE(11) P2_CASE(12) P2_CASE(13) P2_CASE(14) P2_CASE(15)
            P2_CASE(19) P2_CASE(21) P2_CASE(23)
#undef P2_CASE
            case -1: p2::permute_r1(s); break;
            default: return 0;
        }
        for (int k = 0; k < 16; k++) states[i * 16 + k] = s[k];
    }
    return 1;
}
void sp1b200_hostcheck_ext_mul(const uint32_t* a, const uint32_t* b, uint32_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        kb::Ext x{{a[4 * i], a[4 * i + 1], a[4 * i + 2], a[4 * i + 3]}}, y{{b[4 * i], b[4 * i + 1], b[4 * i + 2], b[4 * i + 3]}};
        kb::Ext r = kb::ext_mul(x, y);
        for (int k = 0; k < 4; k++) out[4 * i + k] = r.c[k];
    }
}
void sp1b200_hostcheck_ext_inv(const uint32_t* a, uint32_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        kb::Ext x{{a[4 * i], a[4 * i + 1], a[4 * i + 2], a[4 * i + 3]}};
        kb::Ext r = kb::ext_inv(x);
        for (int k = 0; k < 4; k++) out[4 * i + k] = r.c[k];
    }
}
// the RS-encode kernels' per-pass twiddle table (rs_twiddles.cuh), rs_tw::WORDS words, built by the same code as on the device
uint32_t sp1b200_hostcheck_rs_tw8(uint32_t* out) {
    for (uint32_t i = 0; i < rs_tw::WORDS; i++) out[i] = rs_tw::word(i / 8, (int)(i % 8));
    return rs_tw::WORDS;
}
void sp1b200_hostcheck_field(const uint32_t* a, const uint32_t* b, uint32_t* add, uint32_t* sub, uint32_t* mul, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) { add[i] = kb::add(a[i], b[i]); sub[i] = kb::sub(a[i], b[i]); mul[i] = kb::mul(a[i], b[i]); }
}
// The three Montgomery reductions of kb31.cuh on n 64-bit inputs: monty_reduce, monty_reduce2 and monty_reduce_lazy of each x[i]
// (the caller judges each result only inside that reduction's domain)
void sp1b200_hostcheck_reduce(const uint64_t* x, uint32_t* r, uint32_t* r2, uint32_t* r_lazy, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) { r[i] = kb::monty_reduce(x[i]); r2[i] = kb::monty_reduce2(x[i]); r_lazy[i] = kb::monty_reduce_lazy(x[i]); }
}
// The Poseidon2 s-box's products (poseidon2.cuh): mont_lazy(a, b), mont_wide_lazy(a, b) and sbox(a, b) (b as the round constant)
void sp1b200_hostcheck_p2_products(const uint32_t* a, const uint32_t* b, uint32_t* lazy, uint32_t* wide_lazy, uint32_t* sbox, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        lazy[i] = p2::mont_lazy(a[i], b[i]); wide_lazy[i] = p2::mont_wide_lazy(a[i], b[i]); sbox[i] = p2::sbox(a[i], b[i]);
    }
}

// Evaluate ONE chip's constraint program on one row (base-field values) two ways: the bytecode as given, and the stream
// produced by zc_lower (what the zerocheck kernels interpret).  chip = the per-chip words of the machine blob
// (sp1b200_machine_create).  out[0..4) = sum_k alpha_pows[assert_alphas[k]] * value_k (original), out[4..8) = lowered;
// out[8..12) = the sum over the self-contained pieces; returns the lowered register pressure, or -1 on a lowering error.
int sp1b200_hostcheck_zc_lower(const uint32_t* chip, const uint32_t* main_row, const uint32_t* prep_row, const uint32_t* pv,
                               const uint32_t* alpha_pows, uint32_t window, uint32_t* out, uint32_t* n_lowered) {
    using hf::E4;
    const uint32_t* b = chip;
    HostProg hp;
    b += 3;  // main_w prep_w n_constraints
    const uint32_t n_regs = *b++;
    const uint32_t ni = *b++, nl = *b++, nc = *b++, np = *b++, na = *b++;
    hp.instrs.resize(ni); memcpy(hp.instrs.data(), b, ni * 8); b += 2 * ni;
    hp.leaves.resize(nl); memcpy(hp.leaves.data(), b, nl * 8); b += 2 * nl;
    hp.consts.assign(b, b + nc); b += nc;
    hp.publics.assign(b, b + np); b += np;
    hp.assert_regs.assign(b, b + na); b += na;
    hp.assert_alphas.assign(b, b + na); b += na;
    auto leaf = [&](const LeafRef& l) { return l.source == LEAF_MAIN ? main_row[l.col] : prep_row[l.col]; };
    {
        std::vector<uint32_t> regs(n_regs ? n_regs : 1, 0);
        for (const DagInstr& in : hp.instrs) {
            switch (in.opcode) {
                case BC_LOAD_LEAF: regs[in.out] = leaf(hp.leaves[in.a]); break;
                case BC_LOAD_CONST: regs[in.out] = hp.consts[in.a]; break;
                case BC_LOAD_PUBLIC: regs[in.out] = pv[hp.publics[in.a]]; break;
                case BC_ADD_F: regs[in.out] = kb::add(regs[in.a], regs[in.b]); break;
                case BC_SUB_F: regs[in.out] = kb::sub(regs[in.a], regs[in.b]); break;
                case BC_MUL_F: regs[in.out] = kb::mul(regs[in.a], regs[in.b]); break;
                case BC_NEG_F: regs[in.out] = kb::neg(regs[in.a]); break;
            }
        }
        E4 acc;
        for (size_t k = 0; k < hp.assert_regs.size(); k++) acc = acc + E4::load(alpha_pows + 4 * hp.assert_alphas[k]) * regs[hp.assert_regs[k]];
        acc.store(out);
    }
    auto run = [&](const ZcLowered& Lw) {
        std::vector<uint32_t> rf(Lw.n_regs, 0);
        E4 a;
        for (const ZcInstr& in : Lw.instrs) {
            switch (in.op) {
                case ZC_LOAD_MAIN: rf[in.out] = main_row[(uint32_t)in.a | ((uint32_t)in.b << 16)]; break;
                case ZC_LOAD_PREP: rf[in.out] = prep_row[(uint32_t)in.a | ((uint32_t)in.b << 16)]; break;
                case ZC_CONST: rf[in.out] = hp.consts[in.a]; break;
                case ZC_PUBLIC: rf[in.out] = pv[hp.publics[in.a]]; break;
                case ZC_ADD: { uint32_t x = rf[in.a], y = rf[in.b]; rf[in.out] = kb::add(x, y); break; }
                case ZC_SUB: { uint32_t x = rf[in.a], y = rf[in.b]; rf[in.out] = kb::sub(x, y); break; }
                case ZC_MUL: { uint32_t x = rf[in.a], y = rf[in.b]; rf[in.out] = kb::mul(x, y); break; }
                case ZC_NEG: rf[in.out] = kb::neg(rf[in.a]); break;
                case ZC_ASSERT: a = a + E4::load(alpha_pows + 4 * in.b) * rf[in.a]; break;
            }
        }
        return a;
    };
    ZcLowered L = zc_lower(hp, window);
    if (!L.error.empty()) return -1;
    if (n_lowered) *n_lowered = (uint32_t)L.instrs.size();
    E4 acc = run(L);
    // the same polynomial as a sum of self-contained pieces (the partition machine_create uses for the short rounds)
    {
        const size_t na = hp.assert_regs.size();
        const size_t np_ = std::max<size_t>(1, std::min<size_t>(16, na / 4));
        E4 sum;
        for (size_t q = 0; q < np_; q++) {
            ZcLowered P = zc_lower(hp, window, na * q / np_, na * (q + 1) / np_);
            if (!P.error.empty() || P.n_regs > L.n_regs + 8) return -1;
            sum = sum + run(P);
        }
        sum.store(out + 8);
    }
    acc.store(out + 4);
    return (int)L.n_regs;
}

// The interaction check's key fingerprint (debug_fp.cuh): 62 bits, two linear forms over F of (kind, n_values, values)
uint64_t sp1b200_hostcheck_fingerprint(uint32_t kind, uint32_t n_values, const uint32_t* values) {
    return dbgfp::fingerprint(kind, n_values, values);
}

// Host transcript arithmetic (hostfield.hpp, kb31.cuh): product, inverse, and the batched-inversion Lagrange interpolation through 4 / 5 nodes
// that the sumcheck drivers use.  coeffs_out: n ext elements = coefficients of the polynomial through (x_i, y_i).
void sp1b200_hostcheck_e4(const uint32_t* a, const uint32_t* b, uint32_t* mul_out, uint32_t* inv_out, uint64_t n) {
    using hf::E4;
    for (uint64_t i = 0; i < n; i++) {
        (E4::load(a + 4 * i) * E4::load(b + 4 * i)).store(mul_out + 4 * i);
        E4(kb::ext_inv(E4::load(a + 4 * i))).store(inv_out + 4 * i);
    }
}
int sp1b200_hostcheck_interpolate(const uint32_t* xs, const uint32_t* ys, uint32_t n, uint32_t* coeffs_out) {
    using hf::E4;
    auto go = [&](auto tag) {
        constexpr int N = decltype(tag)::value;
        E4 x[N], L[N][N], c[N];
        for (int i = 0; i < N; i++) x[i] = E4::load(xs + 4 * i);
        hf::lagrange_basis<N>(x, L);
        for (int k = 0; k < N; k++) for (int i = 0; i < N; i++) c[k] = c[k] + L[i][k] * E4::load(ys + 4 * i);
        for (int k = 0; k < N; k++) c[k].store(coeffs_out + 4 * k);
    };
    if (n == 3) go(std::integral_constant<int, 3>{});
    else if (n == 4) go(std::integral_constant<int, 4>{});
    else if (n == 5) go(std::integral_constant<int, 5>{});
    else return -1;
    return 0;
}

// The core-proof verifier's septic arithmetic (septic.cuh), Montgomery words: n products and inverses of septic elements (7 words
// each); n curve additions add_incomplete(p, q) of points (14 words: x then y), ok[i] = 0 on the exceptional case; SepticDigest
// addition; and the three constant points zero, starting digest, dummy (42 words).
void sp1b200_hostcheck_septic(const uint32_t* a, const uint32_t* b, uint32_t* mul_out, uint32_t* inv_out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        s7::E7 x, y;
        for (int k = 0; k < 7; k++) { x.c[k] = a[7 * i + k]; y.c[k] = b[7 * i + k]; }
        const s7::E7 m = s7::mul(x, y), v = s7::inv(x);
        for (int k = 0; k < 7; k++) { mul_out[7 * i + k] = m.c[k]; inv_out[7 * i + k] = v.c[k]; }
    }
}
// frobenius and double_frobenius of n septic elements (septic.cuh, the lazily reduced table products of `lin`)
void sp1b200_hostcheck_septic_frobenius(const uint32_t* a, uint32_t* frob_out, uint32_t* dfrob_out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        s7::E7 x;
        for (int k = 0; k < 7; k++) x.c[k] = a[7 * i + k];
        const s7::E7 f = s7::frobenius(x), d = s7::double_frobenius(x);
        for (int k = 0; k < 7; k++) { frob_out[7 * i + k] = f.c[k]; dfrob_out[7 * i + k] = d.c[k]; }
    }
}
void sp1b200_hostcheck_septic_curve_add(const uint32_t* p, const uint32_t* q, uint32_t* out, uint32_t* ok, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        s7::Pt r = s7::infinity();
        ok[i] = s7::add_incomplete(s7::load_point(p + 14 * i), s7::load_point(q + 14 * i), r);
        s7::store_point(r, out + 14 * i);
    }
}
int sp1b200_hostcheck_septic_digest_add(const uint32_t* a, const uint32_t* b, uint32_t* out) {
    s7::Pt r;
    if (!s7::digest_add(s7::load_point(a), s7::load_point(b), r)) return 0;
    s7::store_point(r, out);
    return 1;
}
void sp1b200_hostcheck_septic_constants(uint32_t* out42) {
    s7::store_point(s7::digest_zero(), out42);
    s7::store_point(s7::digest_start(), out42 + 14);
    s7::store_point(s7::dummy_point(), out42 + 28);
}
// The program setup's device septic code (septic.cuh), Montgomery words: lift_x of n messages (8 words each) -> offsets[i] (-1 when
// none of the 256 offsets gives a point) and points (x then y, 14 words); square roots of n septic elements (ok[i] = 0 for a
// non-square, out left zero); n complete additions of points (infinity = 14 zero words).
void sp1b200_hostcheck_lift_x(const uint32_t* msgs, int32_t* offsets, uint32_t* pts, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        uint32_t m[8];
        for (int k = 0; k < 8; k++) m[k] = msgs[8 * i + k];
        s7::Pt p = s7::infinity();
        offsets[i] = s7::lift_x(m, p);
        s7::store_point(p, pts + 14 * i);
    }
}
void sp1b200_hostcheck_septic_sqrt(const uint32_t* a, uint32_t* out, uint32_t* ok, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        s7::E7 x;
        for (int k = 0; k < 7; k++) x.c[k] = a[7 * i + k];
        const uint32_t nrm = s7::pow_r(x);
        ok[i] = s7::is_zero(x) || s7::base_is_square(nrm);
        const s7::E7 r = ok[i] ? s7::sqrt(x, nrm) : s7::zero();
        for (int k = 0; k < 7; k++) out[7 * i + k] = r.c[k];
    }
}
// the jagged branching program's one-layer transition (bp_transition, shared by the prover's kernels and the verifier) on every
// (bit state, memory state) pair: out[bit_state * 4 + state], bit_state = row * 8 + index * 4 + current bit * 2 + next bit,
// state = carry + 2 * comparison_so_far; -1 on failure
void sp1b200_hostcheck_bp_transitions(int32_t* out64) {
    for (int b = 0; b < 16; b++)
        for (int st = 0; st < 4; st++) out64[b * 4 + st] = bp_transition(b >> 3, (b >> 2) & 1, (b >> 1) & 1, b & 1, st);
}
void sp1b200_hostcheck_curve_add_complete(const uint32_t* p, const uint32_t* q, uint32_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) {
        s7::store_point(s7::add_complete(s7::load_point(p + 14 * i), s7::load_point(q + 14 * i)), out + 14 * i);
    }
}
}
