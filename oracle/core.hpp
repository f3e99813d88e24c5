// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header).  Restates, for the tests of sp1b200_verify_core_proof:
//   crates/hypercube/src/septic_extension.rs   F_p^7 = F_p[z]/(z^7 - 3z - 5): product, inverse (here by Fermat, a^(p^7 - 2))
//   crates/hypercube/src/septic_curve.rs       y^2 = x^3 + 45x + 41z^3: add_incomplete / sub_incomplete
//   crates/hypercube/src/septic_digest.rs      SepticDigest::zero / starting_digest, SepticDigest + SepticDigest
//   crates/prover/src/verify.rs:116-510        the public-value checks of SP1Prover::verify across the shards of a core proof
#pragma once
#include "field.hpp"
#include <cstring>
#include <vector>

namespace orc {

struct S7 {
    F c[7];
    static S7 base(F a) { S7 r; r.c[0] = a; return r; }
    bool operator==(const S7& o) const { for (int i = 0; i < 7; i++) if (c[i] != o.c[i]) return false; return true; }
    bool is_zero() const { for (int i = 0; i < 7; i++) if (!c[i].is_zero()) return false; return true; }
    S7 operator+(const S7& o) const { S7 r; for (int i = 0; i < 7; i++) r.c[i] = c[i] + o.c[i]; return r; }
    S7 operator-(const S7& o) const { S7 r; for (int i = 0; i < 7; i++) r.c[i] = c[i] - o.c[i]; return r; }
    S7 operator-() const { S7 r; for (int i = 0; i < 7; i++) r.c[i] = -c[i]; return r; }
    S7 operator*(const S7& o) const {
        F t[13];
        for (int i = 0; i < 7; i++) for (int j = 0; j < 7; j++) t[i + j] += c[i] * o.c[j];
        for (int i = 12; i >= 7; i--) {   // z^i = z^(i-7) (3z + 5)
            t[i - 6] += t[i] * F::from_canonical(3);
            t[i - 7] += t[i] * F::from_canonical(5);
        }
        S7 r;
        for (int i = 0; i < 7; i++) r.c[i] = t[i];
        return r;
    }
};

// a^(p^7 - 2): the exponent in base 2^32 limbs, square-and-multiply from the top bit
inline S7 s7_inv(const S7& a) {
    uint32_t e[8] = {1, 0, 0, 0, 0, 0, 0, 0};   // p^7, little-endian 32-bit limbs
    for (int k = 0; k < 7; k++) {
        uint64_t carry = 0;
        for (int i = 0; i < 8; i++) { const uint64_t x = (uint64_t)e[i] * KB_P + carry; e[i] = (uint32_t)x; carry = x >> 32; }
    }
    uint64_t borrow = 2;   // p^7 - 2
    for (int i = 0; i < 8 && borrow; i++) {
        const uint64_t x = e[i];
        e[i] = (uint32_t)(x + ((uint64_t)1 << 32) - borrow);
        borrow = x < borrow ? 1 : 0;
    }
    S7 r = S7::base(F::one());
    for (int i = 7; i >= 0; i--)
        for (int b = 31; b >= 0; b--) { r = r * r; if ((e[i] >> b) & 1) r = r * a; }
    return r;
}

struct SPoint { S7 x, y; };

inline bool s_add(const SPoint& p, const SPoint& q, SPoint& out) {
    const S7 dx = q.x - p.x;
    if (dx.is_zero()) return false;
    const S7 l = (q.y - p.y) * s7_inv(dx);
    SPoint r;
    r.x = l * l - p.x - q.x;
    r.y = l * (p.x - r.x) - p.y;
    out = r;
    return true;
}
inline bool s_sub(const SPoint& p, const SPoint& q, SPoint& out) { return s_add(p, SPoint{q.x, -q.y}, out); }

inline SPoint s_point(const uint32_t (&x)[7], const uint32_t (&y)[7]) {
    SPoint p;
    for (int i = 0; i < 7; i++) { p.x.c[i] = F::from_canonical(x[i]); p.y.c[i] = F::from_canonical(y[i]); }
    return p;
}
inline SPoint digest_zero() {
    static const uint32_t x[7] = {0x1414213, 0x5623730, 0x9504880, 0x1688724, 0x2096980, 0x7856967, 0x1875376};
    static const uint32_t y[7] = {2020310104, 1513506566, 1843922297, 2003644209, 805967281, 1882435203, 1623804682};
    return s_point(x, y);
}
inline SPoint digest_start() {
    static const uint32_t x[7] = {0x1732050, 0x8075688, 0x7729352, 0x7446341, 0x5058723, 0x6694280, 0x5253810};
    static const uint32_t y[7] = {1095433104, 7540207, 1124564165, 2035506693, 11121645, 102781365, 398772161};
    return s_point(x, y);
}
// SepticDigest + SepticDigest: start + (a - zero) + (b - zero) + zero - start
inline bool digest_add(const SPoint& a, const SPoint& b, SPoint& out) {
    const SPoint st = digest_start(), z = digest_zero();
    SPoint s;
    if (!s_add(st, a, s) || !s_sub(s, z, s) || !s_add(s, b, s) || !s_sub(s, z, s) || !s_add(s, z, s) || !s_sub(s, st, s)) return false;
    out = s;
    return true;
}

// verdict codes of include/sp1b200.h
enum : int64_t {
    CORE_EMPTY_PROOF = 43, CORE_TOO_MANY_SHARDS, CORE_INVALID_SHARD_PROOF, PV_LENGTH, PV_FIRST_MULTIPLE, PV_FIRST_NOT_BOOLEAN,
    PV_FIRST_NOT_SET, PV_INITIAL_TIMESTAMP, PV_TS_UNCHANGED, PV_TS_CHANGED, PV_PC_START_VK, PV_PC_START_PREV, PV_PC_NON_EXEC,
    PV_NOT_HALTED, PV_PREV_EXIT, PV_EXIT_NON_EXEC, PV_EXIT_CHANGED, PV_NONCE, PV_INIT_ADDR, PV_FIN_ADDR, PV_INIT_PAGE, PV_FIN_PAGE,
    PV_UNTRUSTED, PV_NEVER_INIT, PV_NEVER_FIN, PV_CVD, PV_DPD, PV_COMMIT, PV_COMMIT_DEF, PV_COMMIT_NEVER, PV_COMMIT_DEF_NEVER,
    PV_CUMULATIVE_SUM, PV_EXCEPTIONAL
};

// the public values of one shard, field by field (PublicValues<[F;4],[F;3],[F;4],F> without mprotect, in declaration order)
struct PvView {
    const uint32_t* w;
    std::vector<F> get(uint32_t at, uint32_t n) const { std::vector<F> v(n); for (uint32_t i = 0; i < n; i++) v[i] = F::raw(w[at + i]); return v; }
    F one(uint32_t at) const { return F::raw(w[at]); }
};
struct PvLayout {   // offsets computed from the field sizes, not written out
    uint32_t prev_cvd, cvd, prev_dpd, dpd, pc_start, next_pc, prev_exit, exit, is_exec, prev_init_addr, last_init_addr, prev_fin_addr,
        last_fin_addr, prev_init_page, last_init_page, prev_fin_page, last_fin_page, init_ts, last_ts, gcs, prev_commit, commit,
        prev_commit_def, commit_def, is_first, untrusted, nonce, total;
    PvLayout() {
        uint32_t at = 0;
        auto f = [&](uint32_t n) { const uint32_t r = at; at += n; return r; };
        prev_cvd = f(32); cvd = f(32); prev_dpd = f(8); dpd = f(8); pc_start = f(3); next_pc = f(3); prev_exit = f(1); exit = f(1);
        is_exec = f(1); prev_init_addr = f(3); last_init_addr = f(3); prev_fin_addr = f(3); last_fin_addr = f(3); prev_init_page = f(3);
        last_init_page = f(3); prev_fin_page = f(3); last_fin_page = f(3); init_ts = f(4); last_ts = f(4);
        f(1); f(1); f(1); f(1);                 // is_timestamp_high_eq, inv_timestamp_high, is_timestamp_low_eq, inv_timestamp_low
        f(1); f(1); f(1); f(1); f(1);           // global init / finalize / page-prot init / page-prot finalize / interaction counts
        gcs = f(14); prev_commit = f(1); commit = f(1); prev_commit_def = f(1); commit_def = f(1);
        f(1); f(1);                             // initial_timestamp_inv, last_timestamp_inv
        is_first = f(1); untrusted = f(1); nonce = f(4); f(4);
        total = at;
    }
};

// verify.rs:116-510 on the shards' public values (Montgomery words); vk_tail: pc_start[3] | initial sum x[7] y[7] | untrusted | 6 zeros.
// Returns 0 or the verdict, *shard = the shard at which the check stops (n for the end-of-chain checks).
inline int64_t core_public_value_checks(const std::vector<const uint32_t*>& pvw, const std::vector<uint64_t>& npv, const uint32_t* vk_tail,
                                        uint32_t* shard) {
    const PvLayout L;
    const size_t n = pvw.size();
    *shard = 0;
    if (n == 0) return CORE_EMPTY_PROOF;
    auto fail = [&](int64_t code, size_t s) { *shard = (uint32_t)s; return code; };
    for (size_t s = 0; s < n; s++) if (npv[s] != 187) return fail(PV_LENGTH, s);
    std::vector<PvView> pv;
    for (auto w : pvw) pv.push_back(PvView{w});
    bool first = false;
    for (size_t s = 0; s < n; s++) {
        const F f = pv[s].one(L.is_first);
        if (f == F::one()) { if (first) return fail(PV_FIRST_MULTIPLE, s); first = true; }
        else if (!f.is_zero()) return fail(PV_FIRST_NOT_BOOLEAN, s);
    }
    if (!first) return fail(PV_FIRST_NOT_SET, n);
    std::vector<F> ts{F::zero(), F::zero(), F::zero(), F::one()};
    for (size_t s = 0; s < n; s++) {
        const auto a = pv[s].get(L.init_ts, 4), b = pv[s].get(L.last_ts, 4);
        const F ex = pv[s].one(L.is_exec);
        if (a != ts) return fail(PV_INITIAL_TIMESTAMP, s);
        if (!ex.is_zero() && a == b) return fail(PV_TS_UNCHANGED, s);
        if (ex != F::one() && a != b) return fail(PV_TS_CHANGED, s);
        ts = b;
    }
    std::vector<F> pc{F::raw(vk_tail[0]), F::raw(vk_tail[1]), F::raw(vk_tail[2])};
    for (size_t s = 0; s < n; s++) {
        const auto a = pv[s].get(L.pc_start, 3), b = pv[s].get(L.next_pc, 3);
        if (a != pc) return fail(s == 0 ? PV_PC_START_VK : PV_PC_START_PREV, s);
        if (pv[s].one(L.is_exec) != F::one() && a != b) return fail(PV_PC_NON_EXEC, s);
        pc = b;
    }
    if (pc != std::vector<F>{F::one(), F::zero(), F::zero()}) return fail(PV_NOT_HALTED, n);
    F ec = F::zero();
    for (size_t s = 0; s < n; s++) {
        const F pe = pv[s].one(L.prev_exit), e = pv[s].one(L.exit);
        if (pe != ec) return fail(PV_PREV_EXIT, s);
        if (pv[s].one(L.is_exec) != F::one() && pe != e) return fail(PV_EXIT_NON_EXEC, s);
        if (!pe.is_zero() && pe != e) return fail(PV_EXIT_CHANGED, s);
        ec = e;
    }
    for (size_t s = 1; s < n; s++) if (pv[s].get(L.nonce, 4) != pv[0].get(L.nonce, 4)) return fail(PV_NONCE, s);
    const std::vector<F> z3(3);
    std::vector<F> ia = z3, fa = z3, ip = z3, fp = z3;
    for (size_t s = 0; s < n; s++) {
        if (pv[s].get(L.prev_init_addr, 3) != ia) return fail(PV_INIT_ADDR, s);
        if (pv[s].get(L.prev_fin_addr, 3) != fa) return fail(PV_FIN_ADDR, s);
        if (pv[s].get(L.prev_init_page, 3) != ip) return fail(PV_INIT_PAGE, s);
        if (pv[s].get(L.prev_fin_page, 3) != fp) return fail(PV_FIN_PAGE, s);
        if (pv[s].one(L.untrusted) != F::raw(vk_tail[17])) return fail(PV_UNTRUSTED, s);
        ia = pv[s].get(L.last_init_addr, 3); fa = pv[s].get(L.last_fin_addr, 3);
        ip = pv[s].get(L.last_init_page, 3); fp = pv[s].get(L.last_fin_page, 3);
    }
    if (ia == z3) return fail(PV_NEVER_INIT, n);
    if (fa == z3) return fail(PV_NEVER_FIN, n);
    std::vector<F> cvd(32), dpd(8);
    F cm = F::zero(), cd = F::zero();
    for (size_t s = 0; s < n; s++) {
        if (pv[s].get(L.prev_cvd, 32) != cvd) return fail(PV_CVD, s);
        if (pv[s].get(L.prev_dpd, 8) != dpd) return fail(PV_DPD, s);
        if (pv[s].one(L.prev_commit) != cm) return fail(PV_COMMIT, s);
        if (pv[s].one(L.prev_commit_def) != cd) return fail(PV_COMMIT_DEF, s);
        cvd = pv[s].get(L.cvd, 32); dpd = pv[s].get(L.dpd, 8); cm = pv[s].one(L.commit); cd = pv[s].one(L.commit_def);
    }
    if (cm != F::one()) return fail(PV_COMMIT_NEVER, n);
    if (cd != F::one()) return fail(PV_COMMIT_DEF_NEVER, n);
    if (n >= ((size_t)1 << 24)) return fail(CORE_TOO_MANY_SHARDS, n);
    SPoint sum;
    for (int i = 0; i < 7; i++) { sum.x.c[i] = F::raw(vk_tail[3 + i]); sum.y.c[i] = F::raw(vk_tail[10 + i]); }
    for (size_t s = 0; s < n; s++) {
        SPoint d;
        const auto g = pv[s].get(L.gcs, 14);
        for (int i = 0; i < 7; i++) { d.x.c[i] = g[i]; d.y.c[i] = g[7 + i]; }
        if (!digest_add(sum, d, sum)) return fail(PV_EXCEPTIONAL, s);
    }
    const SPoint z = digest_zero();
    if (!(sum.x == z.x && sum.y == z.y)) return fail(PV_CUMULATIVE_SUM, n);
    return 0;
}

}  // namespace orc
