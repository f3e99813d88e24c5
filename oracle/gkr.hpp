// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header).  PARITY UNPINNED BY STORED FIXTURES.
//
// LogUp-GKR: interaction fractions, the fraction-sum circuit over the row variables, the per-layer sumcheck
// (LogupRoundPolynomial) and the restated verifier.  Restates
//   crates/hypercube/src/lookup/interaction.rs:11-22, logup_gkr/execution.rs:13-36   (interaction values)
//   crates/hypercube/src/logup_gkr/execution.rs:38-252 (first layer, outputs), :254-382 (layer transition)
//   crates/hypercube/src/logup_gkr/logup_poly.rs:71-228 (fix), :230-552 (round polynomial, nodes {0,1,1/2,b})
//   crates/hypercube/src/logup_gkr/cpu.rs:76-226 (circuit, prove_gkr_round), prover.rs:33-215 (protocol)
//   crates/hypercube/src/logup_gkr/verifier.rs:60-330 (verify_logup_gkr)
// The machine-specific public-values interactions (Record::eval_public_values, verifier.rs:60-82) are outside the
// synthetic machines used here: the expected cumulative sum is 0.
#pragma once
#include "zerocheck.hpp"

namespace orc {

struct VTerm { uint8_t source; uint32_t col; F weight; };   // source: LEAF_PREP / LEAF_MAIN
struct VCol { F constant; std::vector<VTerm> terms; };      // slop_air::VirtualPairCol: Σ w·col + constant
struct Interaction { bool is_send = true; uint32_t arg_index = 0; VCol mult; std::vector<VCol> values; };

template <class K> static inline K vcol_apply(const VCol& v, const K* prep, const K* main) {
    K r = to_K<K>(v.constant);
    for (auto& t : v.terms) r += (t.source == LEAF_MAIN ? main : prep)[t.col] * t.weight;
    return r;
}
// (multiplicity (negated for receives), denominator)   execution.rs:13-36
template <class K> static inline std::pair<K, EF> interaction_vals(const Interaction& in, const K* prep, const K* main, const EF& alpha, const std::vector<EF>& betas) {
    EF den = alpha + betas[0] * F::from_canonical(in.arg_index);
    for (size_t k = 0; k < in.values.size(); k++) den += betas[k + 1] * vcol_apply<K>(in.values[k], prep, main);
    K m = vcol_apply<K>(in.mult, prep, main);
    if (!in.is_send) m = K() - m;
    return {m, den};
}

struct GkrChip {
    size_t height = 0, main_w = 0, prep_w = 0;
    const F* main = nullptr; const F* prep = nullptr;  // column-major
    std::vector<Interaction> inter;                    // sends then receives
};

// one layer of the circuit for one chip: four [rows x I] row-major EF arrays (n padded with 0, d with 1)
struct ChipLayer { size_t rows = 0, I = 0; std::vector<EF> n0, d0, n1, d1; };
struct Layer { std::vector<ChipLayer> chips; unsigned num_row_vars = 0, num_int_vars = 0; };

struct GkrRoundProof { EF n0, n1, d0, d1; PartialSumcheckProof sc; };
struct GkrProof {
    std::vector<EF> out_num, out_den;
    std::vector<GkrRoundProof> rounds;
    std::vector<EF> point;                                   // logup_evaluations.point (max_log_rows)
    std::vector<std::vector<EF>> main_open, prep_open;       // per chip
    F witness;
};

// tests only: the inputs of this thread's last gkr_prove that are not in the proof (tests/test_ref_gkr.py replays them through the
// reference's kernels): alpha, the beta seed and, per GKR layer in proof order, lambda, the evaluation point and the claim
struct GkrLayerInputs { EF lambda, claim; std::vector<EF> point; };
struct GkrProveInputs { EF alpha; std::vector<EF> beta_seed; std::vector<GkrLayerInputs> layers; };
static inline GkrProveInputs& gkr_last_inputs() { static thread_local GkrProveInputs v; return v; }

namespace gkr_detail {

static inline Layer first_layer(const std::vector<GkrChip>& chips, const EF& alpha, const std::vector<EF>& betas, unsigned mlr) {
    Layer L; L.num_row_vars = mlr - 1;
    size_t total = 0;
    for (auto& c : chips) {
        ChipLayer cl; cl.I = c.inter.size(); cl.rows = (c.height + 1) / 2; total += cl.I;
        cl.n0.assign(cl.rows * cl.I, EF()); cl.n1 = cl.n0;
        cl.d0.assign(cl.rows * cl.I, EF::one()); cl.d1 = cl.d0;
#pragma omp parallel if (c.height * cl.I >= 4096)
        {
            std::vector<F> mr(c.main_w), pr(c.prep_w);
#pragma omp for schedule(static)
            for (size_t r = 0; r < c.height; r++) {   // every (row, interaction) writes its own slot
                for (size_t j = 0; j < c.main_w; j++) mr[j] = c.main[j * c.height + r];
                for (size_t j = 0; j < c.prep_w; j++) pr[j] = c.prep[j * c.height + r];
                for (size_t k = 0; k < cl.I; k++) {
                    auto [m, d] = interaction_vals<F>(c.inter[k], pr.data(), mr.data(), alpha, betas);
                    size_t idx = (r / 2) * cl.I + k;
                    if (r & 1) { cl.n1[idx] = EF(m); cl.d1[idx] = d; } else { cl.n0[idx] = EF(m); cl.d0[idx] = d; }
                }
            }
        }
        L.chips.push_back(std::move(cl));
    }
    L.num_int_vars = log2_ceil(total);
    return L;
}

static inline Layer transition(const Layer& L) {
    Layer N; N.num_row_vars = L.num_row_vars - 1; N.num_int_vars = L.num_int_vars;
    for (auto& c : L.chips) {
        ChipLayer cl; cl.I = c.I; cl.rows = (c.rows + 1) / 2;
        cl.n0.assign(cl.rows * cl.I, EF()); cl.n1 = cl.n0;
        cl.d0.assign(cl.rows * cl.I, EF::one()); cl.d1 = cl.d0;
#pragma omp parallel for schedule(static) if (cl.rows * cl.I >= 4096)
        for (size_t i = 0; i < cl.rows; i++)
            for (size_t k = 0; k < c.I; k++) {
                size_t e = (2 * i) * c.I + k, o = (2 * i + 1) * c.I + k, t = i * c.I + k;
                cl.n0[t] = c.d1[e] * c.n0[e] + c.d0[e] * c.n1[e];
                cl.d0[t] = c.d0[e] * c.d1[e];
                if (2 * i + 1 < c.rows) { cl.n1[t] = c.d1[o] * c.n0[o] + c.d0[o] * c.n1[o]; cl.d1[t] = c.d0[o] * c.d1[o]; }
            }
        N.chips.push_back(std::move(cl));
    }
    return N;
}

// extract_outputs (execution.rs:38-112): last layer has one row variable
static inline void outputs(const Layer& L, std::vector<EF>& num, std::vector<EF>& den) {
    size_t n = (size_t)1 << (L.num_int_vars + 1);
    std::vector<EF> n0, n1, d0, d1;
    for (auto& c : L.chips)
        for (size_t k = 0; k < c.I; k++)
            for (int b = 0; b < 2; b++) {  // fix_last_variable(0/1) of a 2-row padded MLE = row b (padding if absent)
                bool have = (size_t)b < c.rows;
                n0.push_back(have ? c.n0[b * c.I + k] : EF()); n1.push_back(have ? c.n1[b * c.I + k] : EF());
                d0.push_back(have ? c.d0[b * c.I + k] : EF::one()); d1.push_back(have ? c.d1[b * c.I + k] : EF::one());
            }
    n0.resize(n, EF()); n1.resize(n, EF()); d0.resize(n, EF::one()); d1.resize(n, EF::one());
    num.resize(n); den.resize(n);
    for (size_t i = 0; i < n; i++) { num[i] = n0[i] * d1[i] + n1[i] * d0[i]; den[i] = d0[i] * d1[i]; }
}

// one GKR round: sumcheck of  eq(point, .) * (lambda (n0 d1 + n1 d0) + d0 d1)  over (interaction vars || row vars)
static inline GkrRoundProof prove_round(Layer L, const std::vector<EF>& eval_point, const EF& num_eval, const EF& den_eval, Challenger& ch) {
    GkrRoundProof rp;
    EF lambda = ch.sample_ext();
    unsigned v = L.num_int_vars;
    std::vector<EF> ipt(eval_point.begin(), eval_point.begin() + v), rpt(eval_point.begin() + v, eval_point.end());
    std::vector<EF> eq_int = partial_lagrange(ipt), eq_row = partial_lagrange(rpt);
    std::vector<EF> point = eval_point;
    EF eq_adj = EF::one(), pad_adj = EF::one();
    EF claim = num_eval * lambda + den_eval;
    gkr_last_inputs().layers.push_back({lambda, claim, eval_point});
    PartialSumcheckProof& pf = rp.sc;
    pf.claimed_sum = claim;
    EF round_claim = claim;
    const EF half = EF(F::two().inv()), eighth = EF(F::from_canonical(8).inv()), four = EF(F::from_canonical(4));
    bool interaction_mode = false;
    std::vector<EF> in0, in1, id0, id1;  // interaction-layer vectors
    size_t nvars = v + L.num_row_vars;
    for (size_t rd = 0; rd < nvars; rd++) {
        EF e0, eh, eqs;
        if (!interaction_mode) {
            size_t off = 0;
            for (auto& c : L.chips) {
                const size_t half_rows = (c.rows + 1) / 2;
#pragma omp parallel if (half_rows * c.I >= 2048)
                {
                EF le0, leh, leqs;   // exact field arithmetic: any summation order gives the same words
#pragma omp for schedule(static) nowait
                for (size_t i = 0; i < half_rows; i++) {
                    EF er0 = eq_row[2 * i], er1 = eq_row[2 * i + 1];
                    bool full = 2 * i + 1 < c.rows;
                    EF a0, ah, es;
                    for (size_t k = 0; k < c.I; k++) {
                        const EF& e = eq_int[off + k];
                        size_t x = (2 * i) * c.I + k, y = (2 * i + 1) * c.I + k;
                        EF n0 = c.n0[x], n1 = c.n1[x], d0 = c.d0[x], d1 = c.d1[x];
                        EF n0b = full ? c.n0[y] : EF(), n1b = full ? c.n1[y] : EF(), d0b = full ? c.d0[y] : EF::one(), d1b = full ? c.d1[y] : EF::one();
                        a0 += e * (lambda * (d0 * n1 + d1 * n0) + d0 * d1);
                        ah += e * (lambda * ((d0 + d0b) * (n1 + n1b) + (d1 + d1b) * (n0 + n0b)) + (d0 + d0b) * (d1 + d1b));
                        es += e * (er0 + er1);
                    }
                    le0 += a0 * er0; leh += ah * (er0 + er1); leqs += es;
                }
#pragma omp critical
                { e0 += le0; eh += leh; eqs += leqs; }
                }
                off += c.I;
            }
        } else {
            for (size_t j = 0; j < in0.size() / 2; j++) {
                const EF &ea = eq_int[2 * j], &eb = eq_int[2 * j + 1];
                e0 += ea * (lambda * (id0[2 * j] * in1[2 * j] + id1[2 * j] * in0[2 * j]) + id0[2 * j] * id1[2 * j]);
                EF n0h = in0[2 * j] + in0[2 * j + 1], n1h = in1[2 * j] + in1[2 * j + 1], d0h = id0[2 * j] + id0[2 * j + 1], d1h = id1[2 * j] + id1[2 * j + 1];
                eh += (ea + eb) * (lambda * (d0h * n1h + d1h * n0h) + d0h * d1h);
                eqs += ea + eb;
            }
        }
        EF last = point.back();
        EF corr = pad_adj - eqs;
        e0 += corr * (EF::one() - last);
        eh += corr * four;
        eh = eh * eighth;
        e0 = e0 * eq_adj; eh = eh * eq_adj;
        EF b = (EF::one() - last) / (EF::one() - (last + last));
        EF e1 = round_claim - e0;
        Uni poly = interpolate({EF(), EF::one(), half, b}, {e0, e1, eh, EF()});
        ch.observe_ext_slice(poly.c.data(), poly.c.size());
        pf.polys.push_back(poly);
        EF a = ch.sample_ext();
        pf.point.insert(pf.point.begin(), a);
        round_claim = poly.eval(a);
        // fix_t_variables
        point.pop_back();
        pad_adj = pad_adj * (last * a + (EF::one() - last) * (EF::one() - a));
        auto fix = [&](const EF& x, const EF& y) { return x + a * (y - x); };
        if (!interaction_mode) {
            for (auto& c : L.chips) {
                size_t nr = (c.rows + 1) / 2;
                std::vector<EF> n0(nr * c.I), n1(nr * c.I), d0(nr * c.I), d1(nr * c.I);
#pragma omp parallel for schedule(static) if (nr * c.I >= 2048)
                for (size_t i = 0; i < nr; i++)
                    for (size_t k = 0; k < c.I; k++) {
                        size_t x = (2 * i) * c.I + k, y = (2 * i + 1) * c.I + k, t = i * c.I + k;
                        bool full = 2 * i + 1 < c.rows;
                        n0[t] = fix(c.n0[x], full ? c.n0[y] : EF()); n1[t] = fix(c.n1[x], full ? c.n1[y] : EF());
                        d0[t] = fix(c.d0[x], full ? c.d0[y] : EF::one()); d1[t] = fix(c.d1[x], full ? c.d1[y] : EF::one());
                    }
                c.n0.swap(n0); c.n1.swap(n1); c.d0.swap(d0); c.d1.swap(d1); c.rows = nr;
            }
            std::vector<EF> ne(eq_row.size() / 2);
#pragma omp parallel for schedule(static) if (ne.size() >= 4096)
            for (size_t i = 0; i < ne.size(); i++) ne[i] = fix(eq_row[2 * i], eq_row[2 * i + 1]);
            eq_row.swap(ne);
            if (L.num_row_vars == 1) {
                // every chip is now a single (possibly virtual) row: flatten over interactions, pad to 2^v
                for (auto& c : L.chips)
                    for (size_t k = 0; k < c.I; k++) {
                        bool have = c.rows > 0;
                        in0.push_back(have ? c.n0[k] : EF()); in1.push_back(have ? c.n1[k] : EF());
                        id0.push_back(have ? c.d0[k] : EF::one()); id1.push_back(have ? c.d1[k] : EF::one());
                    }
                size_t n = (size_t)1 << v;
                in0.resize(n, EF()); in1.resize(n, EF()); id0.resize(n, EF::one()); id1.resize(n, EF::one());
                interaction_mode = true;
                eq_adj = pad_adj; pad_adj = EF::one();
            } else L.num_row_vars--;
        } else {
            size_t n = in0.size() / 2;
            std::vector<EF> a0(n), a1(n), b0(n), b1(n), ne(n);
            for (size_t j = 0; j < n; j++) {
                a0[j] = fix(in0[2 * j], in0[2 * j + 1]); a1[j] = fix(in1[2 * j], in1[2 * j + 1]);
                b0[j] = fix(id0[2 * j], id0[2 * j + 1]); b1[j] = fix(id1[2 * j], id1[2 * j + 1]);
                ne[j] = fix(eq_int[2 * j], eq_int[2 * j + 1]);
            }
            in0.swap(a0); in1.swap(a1); id0.swap(b0); id1.swap(b1); eq_int.swap(ne);
        }
    }
    pf.eval = round_claim;
    rp.n0 = in0[0]; rp.d0 = id0[0]; rp.n1 = in1[0]; rp.d1 = id1[0];
    return rp;
}
}  // namespace gkr_detail

static inline unsigned gkr_beta_dim(const std::vector<GkrChip>& chips) {
    size_t ar = 1;
    for (auto& c : chips) for (auto& i : c.inter) ar = std::max(ar, i.values.size() + 1);
    return log2_ceil(ar);
}

// GkrProverImpl::prove_logup_gkr (logup_gkr/prover.rs:70-215)
static inline GkrProof gkr_prove(const std::vector<GkrChip>& chips, unsigned mlr, unsigned gkr_pow_bits, Challenger& ch, const F* replay_witness = nullptr) {
    using namespace gkr_detail;
    GkrProof pf;
    unsigned bdim = gkr_beta_dim(chips);
    if (replay_witness) { pf.witness = *replay_witness; bool ok = ch.check_witness(gkr_pow_bits, *replay_witness); assert(ok); (void)ok; }
    else pf.witness = ch.grind(gkr_pow_bits);
    EF alpha = ch.sample_ext();
    std::vector<EF> beta_seed = ch.sample_point(bdim);
    (void)ch.sample_ext();  // _pv_challenge
    std::vector<EF> betas = partial_lagrange(beta_seed);
    GkrProveInputs& rec = gkr_last_inputs();
    rec = {alpha, beta_seed, {}};
    std::vector<Layer> layers;
    { OrcTrace t("gkr.first_layer"); layers.push_back(first_layer(chips, alpha, betas, mlr)); }
    { OrcTrace t("gkr.transitions"); while (layers.back().num_row_vars > 1) layers.push_back(transition(layers.back())); }
    outputs(layers.back(), pf.out_num, pf.out_den);
    ch.observe_variable_length_ext_slice(pf.out_num.data(), pf.out_num.size());
    ch.observe_variable_length_ext_slice(pf.out_den.data(), pf.out_den.size());
    unsigned v = layers.back().num_int_vars;
    std::vector<EF> eval_point = ch.sample_point(v + 1);
    EF num_eval = mle_eval(pf.out_num.data(), pf.out_num.size(), eval_point);
    EF den_eval = mle_eval(pf.out_den.data(), pf.out_den.size(), eval_point);
    OrcTrace* t_r = new OrcTrace("gkr.rounds");
    while (!layers.empty()) {
        GkrRoundProof rp = prove_round(std::move(layers.back()), eval_point, num_eval, den_eval, ch);
        layers.pop_back();
        ch.observe_ext(rp.n0); ch.observe_ext(rp.n1); ch.observe_ext(rp.d0); ch.observe_ext(rp.d1);
        eval_point = rp.sc.point;
        EF lc = ch.sample_ext();
        num_eval = rp.n0 + (rp.n1 - rp.n0) * lc;
        den_eval = rp.d0 + (rp.d1 - rp.d0) * lc;
        eval_point.push_back(lc);
        pf.rounds.push_back(std::move(rp));
    }
    delete t_r;
    OrcTrace t_o("gkr.openings");
    pf.point = last_k(eval_point, mlr);
    std::vector<EF> eq = partial_lagrange(pf.point);
    ch.observe(F::from_canonical(chips.size()));
    for (auto& c : chips) {
        std::vector<EF> mo(c.main_w), po(c.prep_w);
#pragma omp parallel for schedule(dynamic, 1)
        for (size_t j = 0; j < c.main_w + c.prep_w; j++) {
            const F* col = j < c.main_w ? c.main + j * c.height : c.prep + (j - c.main_w) * c.height;
            EF a;
            for (size_t r = 0; r < c.height; r++) a += eq[r] * col[r];
            (j < c.main_w ? mo[j] : po[j - c.main_w]) = a;
        }
        if (c.prep_w) ch.observe_variable_length_ext_slice(po.data(), po.size());
        ch.observe_variable_length_ext_slice(mo.data(), mo.size());
        pf.main_open.push_back(mo); pf.prep_open.push_back(po);
    }
    return pf;
}

// LogUpGkrVerifier::verify_logup_gkr (logup_gkr/verifier.rs:84-330), expected cumulative sum 0 (see header)
static inline const char* gkr_verify(const std::vector<GkrChip>& chips, unsigned mlr, unsigned gkr_pow_bits, const GkrProof& pf, Challenger& ch) {
    unsigned bdim = gkr_beta_dim(chips);
    if (!ch.check_witness(gkr_pow_bits, pf.witness)) return "Pow";
    EF alpha = ch.sample_ext();
    std::vector<EF> beta_seed = ch.sample_point(bdim);
    (void)ch.sample_ext();
    size_t ni = 0;
    for (auto& c : chips) ni += c.inter.size();
    unsigned v = log2_ceil(ni);
    size_t expected = (size_t)1 << (v + 1);
    if (pf.out_num.size() != expected || pf.out_den.size() != expected) return "InvalidShape";
    ch.observe_variable_length_ext_slice(pf.out_num.data(), pf.out_num.size());
    ch.observe_variable_length_ext_slice(pf.out_den.data(), pf.out_den.size());
    EF cum;
    for (size_t i = 0; i < expected; i++) { if (pf.out_den[i].is_zero()) return "ZeroDenominator"; cum += pf.out_num[i] / pf.out_den[i]; }
    if (!cum.is_zero()) return "CumulativeSumMismatch";
    std::vector<EF> eval_point = ch.sample_point(v + 1);
    EF num_eval = mle_eval(pf.out_num.data(), expected, eval_point), den_eval = mle_eval(pf.out_den.data(), expected, eval_point);
    if (pf.rounds.size() + 1 != mlr) return "InvalidShape(rounds)";
    for (size_t i = 0; i < pf.rounds.size(); i++) {
        const GkrRoundProof& r = pf.rounds[i];
        EF lambda = ch.sample_ext();
        if (r.sc.claimed_sum != num_eval * lambda + den_eval) return "InconsistentSumcheckClaim";
        if (const char* e = sumcheck_partial_verify(r.sc, ch, i + v + 1, 3)) return e;
        EF eqv = EF::one();
        for (size_t k = 0; k < eval_point.size(); k++) eqv *= r.sc.point[k] * eval_point[k] + (EF::one() - r.sc.point[k]) * (EF::one() - eval_point[k]);
        EF expect = eqv * ((r.n0 * r.d1 + r.n1 * r.d0) * lambda + r.d0 * r.d1);
        if (r.sc.eval != expect) return "InconsistentEvaluation";
        ch.observe_ext(r.n0); ch.observe_ext(r.n1); ch.observe_ext(r.d0); ch.observe_ext(r.d1);
        eval_point = r.sc.point;
        EF lc = ch.sample_ext();
        eval_point.push_back(lc);
        num_eval = r.n0 + (r.n1 - r.n0) * lc;
        den_eval = r.d0 + (r.d1 - r.d0) * lc;
    }
    std::vector<EF> ipt(eval_point.begin(), eval_point.begin() + v), tpt(eval_point.begin() + v, eval_point.end());
    if (tpt.size() != mlr) return "InvalidLastLayerDimension";
    if (tpt != pf.point) return "TracePointMismatch";
    std::vector<EF> betas = partial_lagrange(beta_seed);
    std::vector<EF> pe = pf.point; pe.insert(pe.begin(), EF());
    std::vector<EF> nv, dv;
    ch.observe(F::from_canonical(chips.size()));
    for (size_t k = 0; k < chips.size(); k++) {
        const GkrChip& c = chips[k];
        if (c.prep_w) ch.observe_variable_length_ext_slice(pf.prep_open[k].data(), pf.prep_open[k].size());
        ch.observe_variable_length_ext_slice(pf.main_open[k].data(), pf.main_open[k].size());
        if (pf.main_open[k].size() != c.main_w || pf.prep_open[k].size() != c.prep_w) return "InvalidShape(openings)";
        EF geq = full_geq(point_from_usize(c.height, mlr + 1), pe);
        std::vector<EF> zm(c.main_w), zp(c.prep_w);
        for (auto& in : c.inter) {
            Interaction pos = in; pos.is_send = true;  // sign applied below, as the reference does
            auto [rn, rd] = interaction_vals<EF>(pos, pf.prep_open[k].data(), pf.main_open[k].data(), alpha, betas);
            auto [pn, pd] = interaction_vals<EF>(pos, zp.data(), zm.data(), alpha, betas);
            EF ne = rn - pn * geq, de = rd + (EF::one() - pd) * geq;
            nv.push_back(in.is_send ? ne : -ne); dv.push_back(de);
        }
    }
    nv.resize((size_t)1 << v, EF()); dv.resize((size_t)1 << v, EF::one());
    if (num_eval != mle_eval(nv.data(), nv.size(), ipt)) return "NumeratorEvaluationMismatch";
    if (den_eval != mle_eval(dv.data(), dv.size(), ipt)) return "DenominatorEvaluationMismatch";
    return nullptr;
}

}  // namespace orc
