// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header).  PARITY UNPINNED BY STORED FIXTURES.
//
// Zerocheck: constraint bytecode interpreter, per-chip round polynomials, the multi-chip sumcheck and the restated
// verifier check.  Restates
//   crates/hypercube/src/prover/shard.rs:474-646                 (ShardProver::zerocheck)
//   crates/hypercube/src/prover/zerocheck/sum_as_poly.rs:49-440  (round polynomial, nodes {0,1,2,4,b}, corrections)
//   crates/hypercube/src/prover/zerocheck/fix_last_variable.rs:8-62
//   crates/hypercube/src/folder.rs:276-344                       (ConstraintSumcheckFolder: acc += powers[idx] * c)
//   slop/crates/multilinear/src/virtual_geq.rs:13-87, mle.rs:398-407 (VirtualGeq, full_geq)
//   slop/crates/sumcheck/src/prover.rs:13-96                     (multi-polynomial driver, RLC by lambda)
//   crates/hypercube/src/verifier/shard.rs:288-434               (verify_zerocheck)
// AIR constraints enter as bytecode in the reference GPU prover's own format
//   sp1-gpu/crates/sys/include/zerocheck/sequential.cuh:13-49 (DagInstr, LeafRef, BcOp) and
//   sp1-gpu/crates/sys/lib/zerocheck/sequential.cu:52-110 (interpreter semantics),
// because the Rust AIRs cannot be lowered in this image (SURVEY.md §7 "hard parts").
#pragma once
#include "jagged.hpp"
#include <string>

namespace orc {

struct DagInstr { uint8_t opcode, pad; uint16_t out, a, b; };
struct LeafRef { uint8_t source, pad; uint16_t pad2; uint32_t col; };
enum : uint8_t { BC_LOAD_LEAF = 0, BC_LOAD_CONST = 1, BC_LOAD_PUBLIC = 2, BC_ADD_F = 3, BC_SUB_F = 4, BC_MUL_F = 5, BC_NEG_F = 6 };
enum : uint8_t { LEAF_PREP = 2, LEAF_MAIN = 4 };

struct AirProgram {
    std::vector<DagInstr> instrs;
    std::vector<LeafRef> leaves;
    std::vector<F> consts;
    std::vector<uint32_t> publics;
    std::vector<uint16_t> assert_regs;
    std::vector<uint32_t> assert_alphas;  // chip-relative index into the reversed alpha powers
    uint32_t n_regs = 0, n_constraints = 0;
};

template <class K> static inline K to_K(F x);
template <> inline F to_K<F>(F x) { return x; }
template <> inline EF to_K<EF>(F x) { return EF(x); }

// Σ_k powers[alpha_idx_k] * reg_k  (powers = [α^(n-1), ..., α^0])
template <class K>
static inline EF eval_air(const AirProgram& a, const K* prep_row, const K* main_row, const F* pv, const EF* powers, std::vector<K>& regs) {
    regs.resize(a.n_regs);
    for (const DagInstr& in : a.instrs) {
        switch (in.opcode) {
            case BC_LOAD_LEAF: { const LeafRef& l = a.leaves[in.a]; regs[in.out] = (l.source == LEAF_MAIN ? main_row : prep_row)[l.col]; break; }
            case BC_LOAD_CONST: regs[in.out] = to_K<K>(a.consts[in.a]); break;
            case BC_LOAD_PUBLIC: regs[in.out] = to_K<K>(pv[a.publics[in.a]]); break;
            case BC_ADD_F: regs[in.out] = regs[in.a] + regs[in.b]; break;
            case BC_SUB_F: regs[in.out] = regs[in.a] - regs[in.b]; break;
            case BC_MUL_F: regs[in.out] = regs[in.a] * regs[in.b]; break;
            case BC_NEG_F: regs[in.out] = K() - regs[in.a]; break;
            default: assert(false && "bad opcode");
        }
    }
    EF acc;
    for (size_t i = 0; i < a.assert_regs.size(); i++) acc += powers[a.assert_alphas[i]] * regs[a.assert_regs[i]];
    return acc;
}

struct VirtualGeq {
    uint32_t threshold = 0, num_vars = 0;
    EF geq_c, eq_c;
    VirtualGeq fix_last(const EF& alpha) const {
        VirtualGeq r;
        r.threshold = threshold >> 1; r.num_vars = num_vars ? num_vars - 1 : 0; r.geq_c = geq_c;
        r.eq_c = (threshold & 1) == 0 ? (EF::one() - alpha) * eq_c : alpha * (eq_c + geq_c) - geq_c;
        return r;
    }
    EF eval_at_usize(size_t idx) const { return idx < threshold ? EF() : (idx == threshold ? eq_c + geq_c : geq_c); }
};

static inline EF full_geq(const std::vector<EF>& threshold, const std::vector<EF>& point) {
    EF acc = EF::one();
    for (size_t i = threshold.size(); i-- > 0;) {
        const EF &x = threshold[i], &y = point[i];
        acc = ((EF::one() - y) * (EF::one() - x) + y * x) * acc + y * (EF::one() - x);
    }
    return acc;
}

struct ZcChip {
    std::string name;
    const AirProgram* air = nullptr;
    size_t height = 0, main_w = 0, prep_w = 0;
    const F* main = nullptr;  // column-major [main_w x height]
    const F* prep = nullptr;  // column-major [prep_w x height] (same height) or null
};

struct ChipOpened { std::vector<EF> prep, main; std::vector<EF> degree; };

struct ZerocheckResult {
    PartialSumcheckProof proof;
    std::vector<ChipOpened> opened;  // in chip order
};

// tests only: the inputs of this thread's last zerocheck_prove (tests/test_ref_zerocheck.py replays them through the reference's
// kernels): the constraint batching challenge alpha, the opening batching challenge gamma, lambda, the claimed sum and the round
// challenges in round order
struct ZerocheckProveInputs { EF alpha, gamma, lambda, claimed_sum; std::vector<EF> challenges; };
static inline ZerocheckProveInputs& zerocheck_last_inputs() { static thread_local ZerocheckProveInputs v; return v; }

namespace zc_detail {
struct State {
    size_t h, mw, pw;
    std::vector<F> mF, pF;    // round 0: row-major [h x w] copies
    std::vector<EF> mE, pE;   // later rounds
    std::vector<EF> zeta;
    EF eq_adj = EF::one(), geq_value, pra;
    VirtualGeq vg;
    std::vector<EF> alpha_pows, gkr_pows;
    const AirProgram* air;
};

// E = partial_lagrange(zeta without its last coordinate): every chip with rows carries the same zeta in a given round, so the
// caller builds the table once per round
template <class K>
static Uni sum_as_poly(const State& s, const std::vector<K>& M, const std::vector<K>& Pp, const F* pv, bool first, const EF& claim,
                       const std::vector<EF>& E) {
    Uni out;
    if (s.h == 0) { out.c.assign(5, EF()); return out; }
    EF last = s.zeta.back();
    size_t terms = (s.h + 1) / 2;
    EF y0, y2, y4;
#pragma omp parallel
    {
        EF l0, l2, l4;
        std::vector<K> m0(s.mw), m2(s.mw), m4(s.mw), p0(s.pw), p2(s.pw), p4(s.pw), regs;
#pragma omp for schedule(static) nowait
        for (size_t i = 0; i < terms; i++) {
            for (size_t c = 0; c < s.mw; c++) {
                K a = M[(2 * i) * s.mw + c], b = (2 * i + 1 < s.h) ? M[(2 * i + 1) * s.mw + c] : K();
                K sl = b - a, sl2 = sl + sl;
                m0[c] = a; m2[c] = sl2 + a; m4[c] = sl2 + sl2 + a;
            }
            for (size_t c = 0; c < s.pw; c++) {
                K a = Pp[(2 * i) * s.pw + c], b = (2 * i + 1 < s.h) ? Pp[(2 * i + 1) * s.pw + c] : K();
                K sl = b - a, sl2 = sl + sl;
                p0[c] = a; p2[c] = sl2 + a; p4[c] = sl2 + sl2 + a;
            }
            auto gkr = [&](const std::vector<K>& m, const std::vector<K>& p) {
                EF g; size_t k = 0;
                for (size_t c = 0; c < s.mw; c++) g += s.gkr_pows[k++] * m[c];
                for (size_t c = 0; c < s.pw; c++) g += s.gkr_pows[k++] * p[c];
                return g;
            };
            EF g0 = gkr(m0, p0), g2 = gkr(m2, p2);
            EF a0 = g0;
            if (!first) a0 += eval_air<K>(*s.air, p0.data(), m0.data(), pv, s.alpha_pows.data(), regs);
            EF a2 = eval_air<K>(*s.air, p2.data(), m2.data(), pv, s.alpha_pows.data(), regs) + g2;
            EF a4 = eval_air<K>(*s.air, p4.data(), m4.data(), pv, s.alpha_pows.data(), regs) + (g2 + g2 - g0);
            l0 += a0 * E[i]; l2 += a2 * E[i]; l4 += a4 * E[i];
        }
#pragma omp critical
        { y0 += l0; y2 += l2; y4 += l4; }
    }
    size_t th = terms - 1;
    EF msb = s.eq_adj * (th < E.size() ? E[th] : EF());
    EF v0 = s.vg.fix_last(EF()).eval_at_usize(th);
    EF v2 = s.vg.fix_last(EF(F::from_canonical(2))).eval_at_usize(th);
    EF v4 = s.vg.fix_last(EF(F::from_canonical(4))).eval_at_usize(th);
    EF f0 = EF::one() - last;
    y0 = y0 * (f0 * s.eq_adj) - s.pra * v0 * msb * f0;
    EF y1 = claim - y0;
    EF f2 = last * F::from_canonical(3) - EF::one();
    y2 = y2 * (f2 * s.eq_adj) - s.pra * v2 * msb * f2;
    EF f4 = last * F::from_canonical(7) - EF(F::from_canonical(3));
    y4 = y4 * (f4 * s.eq_adj) - s.pra * v4 * msb * f4;
    EF b = (EF::one() - last) / (EF::one() - (last + last));
    return interpolate({EF(), EF::one(), EF(F::from_canonical(2)), EF(F::from_canonical(4)), b}, {y0, y1, y2, y4, EF()});
}

template <class K>
static void fix_cols(const std::vector<K>& in, size_t h, size_t w, const EF& alpha, std::vector<EF>& out) {
    size_t nh = (h + 1) / 2;
    out.assign(nh * w, EF());
#pragma omp parallel for schedule(static) if (nh * w >= 4096)
    for (size_t i = 0; i < nh; i++)
        for (size_t c = 0; c < w; c++) {
            EF a = EF(in[(2 * i) * w + c]);
            EF b = (2 * i + 1 < h) ? EF(in[(2 * i + 1) * w + c]) : EF();
            out[i * w + c] = a + alpha * (b - a);
        }
}
}  // namespace zc_detail

// claims[c] = Σ_j gkr_challenge^(j+1) * opening_j(gkr_point)   (main openings first, then preprocessed)
static inline ZerocheckResult zerocheck_prove(const std::vector<ZcChip>& chips, const EF& batching_challenge, const EF& gkr_challenge,
                                              const std::vector<EF>& gkr_point, const std::vector<EF>& claims, const std::vector<F>& pv,
                                              unsigned max_log_rows, Challenger& ch) {
    using namespace zc_detail;
    size_t maxc = 0;
    for (auto& c : chips) maxc = std::max<size_t>(maxc, c.air->n_constraints);
    std::vector<EF> pw(maxc ? maxc : 1); pw[0] = EF::one();
    for (size_t i = 1; i < pw.size(); i++) pw[i] = pw[i - 1] * batching_challenge;
    std::vector<State> st(chips.size());
    for (size_t k = 0; k < chips.size(); k++) {
        const ZcChip& c = chips[k]; State& s = st[k];
        s.h = c.height; s.mw = c.main_w; s.pw = c.prep_w; s.air = c.air; s.zeta = gkr_point;
        s.alpha_pows.assign(pw.begin(), pw.begin() + c.air->n_constraints);
        std::reverse(s.alpha_pows.begin(), s.alpha_pows.end());
        EF g = gkr_challenge;
        for (size_t j = 0; j < c.main_w + c.prep_w; j++) { s.gkr_pows.push_back(g); g *= gkr_challenge; }
        s.mF.resize(c.height * c.main_w); s.pF.resize(c.height * c.prep_w);
#pragma omp parallel for schedule(static) if (c.height >= 1024)
        for (size_t r = 0; r < c.height; r++) {
            for (size_t j = 0; j < c.main_w; j++) s.mF[r * c.main_w + j] = c.main[j * c.height + r];
            for (size_t j = 0; j < c.prep_w; j++) s.pF[r * c.prep_w + j] = c.prep[j * c.height + r];
        }
        std::vector<F> zm(c.main_w), zp(c.prep_w), regs;
        s.pra = eval_air<F>(*c.air, zp.data(), zm.data(), pv.data(), s.alpha_pows.data(), regs);
        s.geq_value = c.height > 0 ? EF() : EF::one();
        s.vg.threshold = (uint32_t)c.height; s.vg.geq_c = EF::one(); s.vg.eq_c = EF(); s.vg.num_vars = max_log_rows;
    }
    EF lambda = ch.sample_ext();
    ZerocheckResult res;
    PartialSumcheckProof& pf = res.proof;
    for (const EF& c : claims) pf.claimed_sum = pf.claimed_sum * lambda + c;
    ZerocheckProveInputs& rec = zerocheck_last_inputs();
    rec = {batching_challenge, gkr_challenge, lambda, pf.claimed_sum, {}};
    std::vector<EF> round_claims = claims;
    std::vector<Uni> unis(chips.size());
    for (unsigned rd = 0; rd < max_log_rows; rd++) {
        std::vector<EF> E = partial_lagrange(std::vector<EF>(gkr_point.begin(), gkr_point.end() - rd - 1));
        for (size_t k = 0; k < chips.size(); k++)
            unis[k] = rd == 0 ? sum_as_poly<F>(st[k], st[k].mF, st[k].pF, pv.data(), true, round_claims[k], E)
                              : sum_as_poly<EF>(st[k], st[k].mE, st[k].pE, pv.data(), false, round_claims[k], E);
        Uni rlc; rlc.c.assign(1, EF());
        for (auto& u : unis) {
            size_t n = std::max(rlc.c.size(), u.c.size());
            std::vector<EF> nc(n);
            for (size_t i = 0; i < n; i++) nc[i] = (i < rlc.c.size() ? rlc.c[i] * lambda : EF()) + (i < u.c.size() ? u.c[i] : EF());
            rlc.c.swap(nc);
        }
        ch.observe_ext_slice(rlc.c.data(), rlc.c.size());
        pf.polys.push_back(rlc);
        EF alpha = ch.sample_ext();
        rec.challenges.push_back(alpha);
        pf.point.insert(pf.point.begin(), alpha);
        for (size_t k = 0; k < chips.size(); k++) {
            State& s = st[k];
            round_claims[k] = unis[k].eval(alpha);
            std::vector<EF> nm, np;
            if (rd == 0) { fix_cols<F>(s.mF, s.h, s.mw, alpha, nm); fix_cols<F>(s.pF, s.h, s.pw, alpha, np); }
            else { fix_cols<EF>(s.mE, s.h, s.mw, alpha, nm); fix_cols<EF>(s.pE, s.h, s.pw, alpha, np); }
            s.mE.swap(nm); s.pE.swap(np);
            s.vg = s.vg.fix_last(alpha);
            if (s.h != 0) {
                EF last = s.zeta.back();
                s.eq_adj = s.eq_adj * (alpha * last + (EF::one() - alpha) * (EF::one() - last));
                s.geq_value = s.h > 1 ? EF() : (EF::one() - s.geq_value) * alpha + s.geq_value;
                s.zeta.pop_back();
            }
            s.h = (s.h + 1) / 2;
        }
    }
    for (auto& c : round_claims) pf.eval = pf.eval * lambda + c;
    ch.observe(F::from_canonical(chips.size()));
    for (size_t k = 0; k < chips.size(); k++) {
        ChipOpened o;
        o.prep.assign(st[k].pE.begin(), st[k].pE.end());
        if (st[k].h) o.main.assign(st[k].mE.begin(), st[k].mE.end()); else o.main.assign(chips[k].main_w, EF());
        if (o.prep.size() != chips[k].prep_w) o.prep.assign(chips[k].prep_w, EF());
        o.degree = point_from_usize(chips[k].height, max_log_rows + 1);
        ch.observe_variable_length_ext_slice(o.prep.data(), o.prep.size());
        ch.observe_variable_length_ext_slice(o.main.data(), o.main.size());
        res.opened.push_back(o);
    }
    return res;
}

// ShardVerifier::verify_zerocheck (crates/hypercube/src/verifier/shard.rs:288-434); the caller has sampled nothing:
// alpha, the gkr batching challenge and lambda are sampled here in the reference's order.
static inline const char* zerocheck_verify(const std::vector<ZcChip>& chips, const std::vector<ChipOpened>& opened,
                                           const std::vector<EF>& gkr_point, const std::vector<std::vector<EF>>& gkr_main_openings,
                                           const std::vector<std::vector<EF>>& gkr_prep_openings, const PartialSumcheckProof& pf,
                                           const std::vector<F>& pv, unsigned max_log_rows, Challenger& ch) {
    EF alpha = ch.sample_ext(), gkr_c = ch.sample_ext(), lambda = ch.sample_ext();
    if (gkr_point.size() != max_log_rows || pf.point.size() != max_log_rows) return "InvalidShape";
    EF eqv = EF::one();
    for (size_t i = 0; i < gkr_point.size(); i++) eqv *= gkr_point[i] * pf.point[i] + (EF::one() - gkr_point[i]) * (EF::one() - pf.point[i]);
    EF rlc;
    for (size_t k = 0; k < chips.size(); k++) {
        const ZcChip& c = chips[k]; const ChipOpened& o = opened[k];
        if (o.prep.size() != c.prep_w || o.main.size() != c.main_w) return "OpeningShape";
        std::vector<EF> pt = pf.point; pt.insert(pt.begin(), EF());
        for (auto& x : o.degree) if (x * (x - EF::one()) != EF()) return "InvalidHeightBitDecomposition";
        for (size_t i = 1; i < o.degree.size(); i++) if (o.degree[i] * o.degree[0] != EF()) return "HeightTooLarge";
        EF geq = full_geq(o.degree, pt);
        // Horner folder == Σ α^(n-1-i) C_i
        std::vector<EF> pws(c.air->n_constraints ? c.air->n_constraints : 1); pws[0] = EF::one();
        for (size_t i = 1; i < pws.size(); i++) pws[i] = pws[i - 1] * alpha;
        std::vector<EF> rev(pws.begin(), pws.begin() + c.air->n_constraints); std::reverse(rev.begin(), rev.end());
        std::vector<EF> zm(c.main_w), zp(c.prep_w), regs;
        EF pra = eval_air<EF>(*c.air, zp.data(), zm.data(), pv.data(), rev.data(), regs);
        EF ce = eval_air<EF>(*c.air, o.prep.data(), o.main.data(), pv.data(), rev.data(), regs) - pra * geq;
        EF ob, g = gkr_c;
        for (auto& v : o.main) { ob += v * g; g *= gkr_c; }
        for (auto& v : o.prep) { ob += v * g; g *= gkr_c; }
        rlc = rlc * lambda + eqv * (ce + ob);
    }
    if (pf.eval != rlc) return "ConstraintsCheckFailed(InconsistencyWithEval)";
    EF mod;
    for (size_t k = 0; k < chips.size(); k++) {
        EF m, g = gkr_c;
        for (auto& v : gkr_main_openings[k]) { m += v * g; g *= gkr_c; }
        for (auto& v : gkr_prep_openings[k]) { m += v * g; g *= gkr_c; }
        mod = lambda * mod + m;
    }
    if (pf.claimed_sum != mod) return "ConstraintsCheckFailed(InconsistencyWithClaimedSum)";
    if (const char* e = sumcheck_partial_verify(pf, ch, max_log_rows, 4)) return e;
    ch.observe(F::from_canonical(chips.size()));
    for (auto& o : opened) { ch.observe_variable_length_ext_slice(o.prep.data(), o.prep.size()); ch.observe_variable_length_ext_slice(o.main.data(), o.main.size()); }
    return nullptr;
}

}  // namespace orc
