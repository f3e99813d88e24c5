// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header).  PARITY UNPINNED BY STORED FIXTURES.
//
// Generic sumcheck driver + verifier, the jagged PCS (commit / prove / verify), the Hadamard sumcheck of the
// dense trace against the jagged "little polynomial", and the branching-program evaluation sumcheck.  Restates
//   slop/crates/algebra/src/univariate.rs:85-108            (interpolation -> coefficient vectors, RLC)
//   slop/crates/sumcheck/src/prover.rs:13-96, verifier.rs:21-107
//   slop/crates/jagged/src/prover.rs:106-328                (commit_multilinears, prove_trusted_evaluations)
//   slop/crates/jagged/src/hadamard.rs:93-151, sumcheck.rs:13-39
//   slop/crates/jagged/src/poly.rs:136-296 (transition function, prover params, partial jagged poly),
//                              :384-470 (BranchingProgram::eval)
//   slop/crates/jagged/src/jagged_eval/{sumcheck_poly.rs:81-165, sumcheck_sum_as_poly.rs:67-247,
//                              eval_sumcheck_prover.rs:17-79, sumcheck_eval.rs:45-243}
//   slop/crates/jagged/src/verifier.rs:113-384
#pragma once
#include "basefold.hpp"
#include <algorithm>

namespace orc {

// ---- univariate polynomials as coefficient vectors ---------------------------------------------------------------
struct Uni {
    std::vector<EF> c;
    EF eval(const EF& x) const { EF r; for (size_t i = c.size(); i-- > 0;) r = r * x + c[i]; return r; }
    EF eval_one_plus_eval_zero() const { EF s = c.empty() ? EF() : c[0]; for (auto& v : c) s += v; return s; }
};

// Lagrange interpolation, coefficient form; result has exactly xs.size() coefficients
static inline Uni interpolate(const std::vector<EF>& xs, const std::vector<EF>& ys) {
    size_t n = xs.size();
    Uni res; res.c.assign(n, EF());
    for (size_t i = 0; i < n; i++) {
        std::vector<EF> num{ys[i]};
        EF den = EF::one();
        for (size_t j = 0; j < n; j++) {
            if (j == i) continue;
            den *= xs[i] - xs[j];
            std::vector<EF> nx(num.size() + 1);
            for (size_t k = 0; k < num.size(); k++) { nx[k + 1] += num[k]; nx[k] -= num[k] * xs[j]; }
            num.swap(nx);
        }
        EF dinv = den.inv();
        for (size_t k = 0; k < num.size(); k++) res.c[k] += num[k] * dinv;
    }
    return res;
}

struct PartialSumcheckProof {
    std::vector<Uni> polys;
    EF claimed_sum;
    std::vector<EF> point;
    EF eval;
};

// partially_verify_sumcheck_proof (sumcheck/src/verifier.rs:21-107)
static inline const char* sumcheck_partial_verify(const PartialSumcheckProof& p, Challenger& ch, size_t nvars, size_t degree) {
    if (p.polys.size() != p.point.size() || p.polys.size() != nvars || nvars == 0) return "InvalidProofShape";
    if (p.polys[0].eval_one_plus_eval_zero() != p.claimed_sum) return "InconsistencyWithClaimedSum";
    if (p.polys[0].c.size() != degree + 1) return "InvalidProofShape";
    ch.observe_ext_slice(p.polys[0].c.data(), p.polys[0].c.size());
    std::vector<EF> alphas;
    const Uni* prev = &p.polys[0];
    for (size_t i = 1; i < p.polys.size(); i++) {
        if (p.polys[i].c.size() != degree + 1) return "InvalidProofShape";
        EF a = ch.sample_ext();
        alphas.insert(alphas.begin(), a);
        if (prev->eval(a) != p.polys[i].eval_one_plus_eval_zero()) return "SumcheckRoundInconsistency";
        ch.observe_ext_slice(p.polys[i].c.data(), p.polys[i].c.size());
        prev = &p.polys[i];
    }
    EF a = ch.sample_ext();
    alphas.insert(alphas.begin(), a);
    if (alphas != p.point) return "InvalidProofShape(point)";
    if (prev->eval(a) != p.eval) return "InconsistencyWithEval";
    return nullptr;
}

// ---- jagged little polynomial ---------------------------------------------------------------------------------------
struct JaggedParams {
    std::vector<size_t> prefix;  // col_prefix_sums_usize: L+1 entries
    unsigned max_log_rows = 0;
    unsigned log_m() const { return log2_ceil(prefix.back()); }
};
static inline JaggedParams jagged_params(const std::vector<size_t>& col_heights, unsigned max_log_rows) {
    JaggedParams p; p.max_log_rows = max_log_rows;
    size_t s = 0;
    for (size_t h : col_heights) { p.prefix.push_back(s); s += h; }
    p.prefix.push_back(p.prefix.back() + col_heights.back());
    return p;
}

static inline std::vector<EF> last_k(const std::vector<EF>& p, size_t k) { return std::vector<EF>(p.end() - k, p.end()); }

// partial_jagged_little_polynomial_evaluation (poly.rs:251-296): value at long-vector index i
static inline std::vector<EF> jagged_little_poly(const JaggedParams& jp, const std::vector<EF>& z_row, const std::vector<EF>& z_col) {
    size_t total = (size_t)1 << jp.log_m();
    size_t ncols = jp.prefix.size() - 1;
    std::vector<EF> col_eq = partial_lagrange(last_k(z_col, log2_ceil(ncols)));
    std::vector<EF> row_eq = partial_lagrange(last_k(z_row, jp.max_log_rows));
    std::vector<EF> out(total);
#pragma omp parallel for schedule(dynamic, 1)
    for (size_t c = 0; c < ncols; c++)
        for (size_t i = jp.prefix[c]; i < jp.prefix[c + 1]; i++) out[i] = col_eq[c] * row_eq[i - jp.prefix[c]];
    return out;
}

// branching program (poly.rs:136-175 transition, :384-470 eval).  Points are big-endian.
struct BranchingProgram {
    std::vector<EF> z_row, z_index;
    size_t num_vars;
    BranchingProgram(const std::vector<EF>& r, const std::vector<EF>& i) : z_row(r), z_index(i), num_vars(std::max(r.size(), i.size())) {}
    static EF lsb(const std::vector<EF>& p, size_t i) { return p.size() <= i ? EF() : p[p.size() - 1 - i]; }
    // memory state index = carry + 2*comparison_so_far; returns -1 on fail
    static int transition(int row_bit, int index_bit, int cur_bit, int next_bit, int state) {
        int carry = state & 1, cmp = state >> 1;
        int new_cmp = (index_bit == next_bit) ? cmp : next_bit;
        int s = row_bit + carry + cur_bit;
        if (index_bit != (s & 1)) return -1;
        return (s >> 1) + 2 * new_cmp;
    }
    EF eval(const std::vector<EF>& prefix_sum, const std::vector<EF>& next_prefix_sum) const {
        EF res[4]; res[2] = EF::one();  // success = carry 0, comparison 1
        for (size_t layer = num_vars + 1; layer-- > 0;) {
            std::vector<EF> pt{lsb(z_row, layer), lsb(z_index, layer), lsb(prefix_sum, layer), lsb(next_prefix_sum, layer)};
            std::vector<EF> eq = partial_lagrange(pt);  // index = row*8 + index*4 + cur*2 + next
            EF nres[4];
            for (int st = 0; st < 4; st++) {
                EF acc[4];
                for (int i = 0; i < 16; i++) {
                    int o = transition((i >> 3) & 1, (i >> 2) & 1, (i >> 1) & 1, i & 1, st);
                    if (o >= 0) acc[o] += eq[i];
                }
                EF a;
                for (int k = 0; k < 4; k++) a += acc[k] * res[k];
                nres[st] = a;
            }
            for (int k = 0; k < 4; k++) res[k] = nres[k];
        }
        return res[0];  // initial state: carry 0, comparison 0
    }
};

static inline std::vector<EF> point_from_usize(size_t x, unsigned dim) {
    std::vector<EF> p(dim);
    for (unsigned i = 0; i < dim; i++) p[i] = EF(F::from_canonical((x >> (dim - 1 - i)) & 1));
    return p;
}

// full_jagged_little_polynomial_evaluation (poly.rs:183-232)
static inline EF jagged_full_eval(const JaggedParams& jp, const std::vector<EF>& z_row, const std::vector<EF>& z_col, const std::vector<EF>& z_index) {
    unsigned lm = jp.log_m();
    std::vector<EF> col_eq = partial_lagrange(z_col);
    BranchingProgram bp(z_row, z_index);
    EF res;
    for (size_t c = 0; c + 1 < jp.prefix.size(); c++)
        res += col_eq[c] * bp.eval(point_from_usize(jp.prefix[c], lm + 1), point_from_usize(jp.prefix[c + 1], lm + 1));
    return res;
}

// jagged evaluation sumcheck prover (jagged_eval/*): returns the PartialSumcheckProof, drives the challenger
static inline PartialSumcheckProof jagged_eval_prove(const JaggedParams& jp, const std::vector<EF>& z_row, const std::vector<EF>& z_col,
                                                     const std::vector<EF>& z_trace, Challenger& ch) {
    unsigned lm = jp.log_m();
    size_t dim = 2 * (lm + 1);
    std::vector<EF> col_eq = partial_lagrange(z_col);
    // merged prefix sums (bits, big-endian, t_c || t_{c+1}), condensed over equal consecutive entries
    std::vector<std::vector<int>> merged; std::vector<EF> zc;
    for (size_t c = 0; c + 1 < jp.prefix.size(); c++) {
        std::vector<int> bits(dim);
        for (unsigned i = 0; i < lm + 1; i++) {
            bits[i] = (jp.prefix[c] >> (lm - i)) & 1;
            bits[lm + 1 + i] = (jp.prefix[c + 1] >> (lm - i)) & 1;
        }
        if (!merged.empty() && merged.back() == bits) zc.back() += col_eq[c];
        else { merged.push_back(bits); zc.push_back(col_eq[c]); }
    }
    EF expected_sum = jagged_full_eval(jp, z_row, z_col, z_trace);
    ch.observe_ext(expected_sum);
    BranchingProgram bp(z_row, z_trace);
    EF half = EF(F::two().inv());
    std::vector<EF> inter(merged.size(), EF::one());
    std::vector<EF> rhos;  // most recent challenge first
    PartialSumcheckProof pf; pf.claimed_sum = expected_sum;
    EF claim = expected_sum;
    for (size_t round = 0; round < dim; round++) {
        EF y0, yh;
#pragma omp parallel
        {
        EF ly0, lyh;
#pragma omp for schedule(dynamic, 8) nowait
        for (size_t k = 0; k < merged.size(); k++) {
            for (int which = 0; which < 2; which++) {
                EF lambda = which ? half : EF();
                size_t split = dim - round - 1;
                EF eq_val = which ? half : (EF::one() - EF(F::from_canonical(merged[k][split])));
                EF eq_eval = inter[k] * eq_val;
                std::vector<EF> hp(split);
                for (size_t i = 0; i < split; i++) hp[i] = EF(F::from_canonical(merged[k][i]));
                hp.push_back(lambda);
                hp.insert(hp.end(), rhos.begin(), rhos.end());
                std::vector<EF> left(hp.begin(), hp.begin() + hp.size() / 2), right(hp.begin() + hp.size() / 2, hp.end());
                EF v = zc[k] * bp.eval(left, right) * eq_eval;
                if (which) lyh += v; else ly0 += v;
            }
        }
#pragma omp critical
        { y0 += ly0; yh += lyh; }
        }
        EF y1 = claim - y0;
        Uni poly = interpolate({EF(), half, EF::one()}, {y0, yh, y1});
        ch.observe_ext_slice(poly.c.data(), poly.c.size());
        EF alpha = ch.sample_ext();
        rhos.insert(rhos.begin(), alpha);
        claim = poly.eval(alpha);
        pf.polys.push_back(poly);
        // fix_last_variable: fold the eq factor of this round's bit
        for (size_t k = 0; k < merged.size(); k++) {
            EF xi = EF(F::from_canonical(merged[k][dim - 1 - round]));
            inter[k] = inter[k] * (alpha * xi + (EF::one() - alpha) * (EF::one() - xi));
        }
    }
    pf.point = rhos;
    pf.eval = pf.polys.back().eval(rhos[0]);
    return pf;
}

// JaggedEvalSumcheckConfig::jagged_evaluation (sumcheck_eval.rs:45-155)
static inline const char* jagged_eval_verify(const JaggedParams& jp, const std::vector<EF>& z_row, const std::vector<EF>& z_col,
                                             const std::vector<EF>& z_trace, const PartialSumcheckProof& pf, Challenger& ch, EF* out) {
    unsigned lm = jp.log_m();
    std::vector<EF> col_eq = partial_lagrange(z_col);
    ch.observe_ext(pf.claimed_sum);
    if (const char* e = sumcheck_partial_verify(pf, ch, 2 * (lm + 1), 2)) return e;
    std::vector<EF> first(pf.point.begin(), pf.point.begin() + pf.point.size() / 2), second(pf.point.begin() + pf.point.size() / 2, pf.point.end());
    if (jp.prefix.size() - 1 > col_eq.size()) return "IncorrectShape";
    EF acc;
    for (size_t c = 0; c + 1 < jp.prefix.size(); c++) {
        std::vector<EF> m = point_from_usize(jp.prefix[c], lm + 1), n = point_from_usize(jp.prefix[c + 1], lm + 1);
        m.insert(m.end(), n.begin(), n.end());
        EF full = EF::one();  // full_lagrange_eval(merged, point)
        for (size_t i = 0; i < m.size(); i++) full *= m[i] * pf.point[i] + (EF::one() - m[i]) * (EF::one() - pf.point[i]);
        acc += col_eq[c] * full;
    }
    acc *= BranchingProgram(z_row, z_trace).eval(first, second);
    if (acc != pf.eval) return "JaggedEvaluationFailed";
    *out = pf.claimed_sum;
    return nullptr;
}

// ---- jagged PCS ----------------------------------------------------------------------------------------------------
struct Table {
    size_t rows = 0, cols = 0;   // real rows (<= 2^max_log_rows), columns
    const F* data = nullptr;     // column-major [cols x rows]; ignored when rows == 0
};

struct JaggedRound {
    std::shared_ptr<StackedRound> stacked;
    std::vector<size_t> row_counts, col_counts;  // including the two dummy tables
    size_t padding_cols = 0;
    Digest original_commit, commit;
};

// JaggedProver::commit_multilinears (jagged/src/prover.rs:106-160)
static inline JaggedRound jagged_commit(const std::vector<Table>& tables, unsigned log_stack, unsigned max_log_rows, const FriParams& fp) {
    JaggedRound r;
    size_t area = 0;
    for (auto& t : tables) { r.row_counts.push_back(t.rows); r.col_counts.push_back(t.cols); area += t.rows * t.cols; }
    size_t S = (size_t)1 << log_stack;
    size_t padded = std::max(((area + S - 1) / S) * S, S);
    size_t added = padded - area;
    std::vector<F> dense(padded);
    size_t off = 0;
    for (auto& t : tables) if (t.rows) { std::copy(t.data, t.data + t.rows * t.cols, dense.begin() + off); off += t.rows * t.cols; }
    r.stacked = stacked_commit(dense.data(), padded / S, log_stack, fp);
    r.original_commit = r.stacked->tree.commitment;
    size_t R = (size_t)1 << max_log_rows;
    size_t added_cols = std::max<size_t>((added + R - 1) / R, 1);
    r.row_counts.push_back(R); r.row_counts.push_back(added - (added_cols - 1) * R);
    r.col_counts.push_back(added_cols - 1); r.col_counts.push_back(1);
    r.padding_cols = added_cols;
    std::vector<F> meta{F::from_canonical(r.row_counts.size())};
    for (size_t x : r.row_counts) meta.push_back(F::from_canonical(x));
    for (size_t x : r.col_counts) meta.push_back(F::from_canonical(x));
    r.commit = p2_compress(r.original_commit, p2_hash(meta));
    return r;
}

struct JaggedProof {
    StackedProof pcs;
    PartialSumcheckProof sumcheck, jagged_eval;
    std::vector<std::vector<std::pair<size_t, size_t>>> rc_cc;
    std::vector<Digest> merkle_commits;
    EF expected_eval;
    unsigned max_log_rows = 0, log_m = 0;
};

// The transcript-derived inputs of the last jagged_prove on this thread: z_col and the Hadamard sumcheck's claim.  Tests read them to
// rerun the sumcheck rounds on the reference's own kernels.
struct JaggedProveInputs { std::vector<EF> z_col; EF claim; };
static inline JaggedProveInputs& jagged_last_inputs() { static thread_local JaggedProveInputs v; return v; }

// JaggedProver::prove_trusted_evaluations (jagged/src/prover.rs:162-328).  claims[r] = per-column evaluations at
// z_row of every (real or empty) table column of round r, in table order.
static inline JaggedProof jagged_prove(const std::vector<EF>& z_row, const std::vector<std::vector<EF>>& claims,
                                       const std::vector<JaggedRound>& rounds, unsigned max_log_rows, Challenger& ch,
                                       const FriParams& fp, const F* replay_witnesses = nullptr) {
    OrcTrace* t_pre = new OrcTrace("jagged.setup");
    size_t total_cols = 0;
    for (auto& r : rounds) for (size_t c : r.col_counts) total_cols += c;
    std::vector<EF> z_col = ch.sample_point(log2_ceil(total_cols));
    std::vector<EF> column_claims;
    std::vector<size_t> heights;
    for (size_t ri = 0; ri < rounds.size(); ri++) {
        column_claims.insert(column_claims.end(), claims[ri].begin(), claims[ri].end());
        column_claims.insert(column_claims.end(), rounds[ri].padding_cols, EF());
        for (size_t t = 0; t < rounds[ri].row_counts.size(); t++)
            for (size_t c = 0; c < rounds[ri].col_counts[t]; c++) heights.push_back(rounds[ri].row_counts[t]);
    }
    JaggedParams jp = jagged_params(heights, max_log_rows);
    unsigned lm = jp.log_m();
    size_t N = (size_t)1 << lm;
    delete t_pre;
    // Round 0 reads the committed base-field words and the jagged little polynomial (partial_jagged_little_polynomial_evaluation,
    // poly.rs:251-296: value at long-vector index i = col_eq[c] * row_eq[i - prefix[c]]) in place: neither the 2^log_m EF lift of the
    // trace nor the 2^log_m little polynomial is materialised (same field values, a quarter of the memory).
    const size_t ncols_j = jp.prefix.size() - 1;
    const std::vector<EF> col_eq = partial_lagrange(last_k(z_col, log2_ceil(ncols_j)));
    const std::vector<EF> row_eq = partial_lagrange(last_k(z_row, jp.max_log_rows));
    std::vector<std::pair<size_t, const F*>> segs;   // (first index, words) of each round's stacked buffer in the long vector
    { size_t off = 0; for (auto& r : rounds) { segs.push_back({off, r.stacked->mles.data()}); off += r.stacked->mles.size(); } segs.push_back({off, nullptr}); }
    auto base_at = [&](size_t idx) -> F {
        size_t k = 0;
        while (k + 2 < segs.size() && segs[k + 1].first <= idx) k++;
        return idx < segs.back().first ? segs[k].second[idx - segs[k].first] : F();
    };
    auto col_of = [&](size_t idx) { return (size_t)(std::upper_bound(jp.prefix.begin(), jp.prefix.end(), idx) - jp.prefix.begin()) - 1; };
    auto ext_at = [&](size_t idx, size_t& c) -> EF {   // c: cursor, never ahead of idx's column
        if (idx >= jp.prefix.back()) return EF();
        while (jp.prefix[c + 1] <= idx) c++;
        return col_eq[c] * row_eq[idx - jp.prefix[c]];
    };
    EF claim = mle_eval(column_claims.data(), column_claims.size(), z_col);
    jagged_last_inputs() = {z_col, claim};
    JaggedProof pf;
    pf.sumcheck.claimed_sum = claim;
    EF half = EF(F::two().inv()), quarter = EF(F::from_canonical(4).inv());
    std::vector<EF> point;
    EF round_claim = claim;
    OrcTrace* t_sc = new OrcTrace("jagged.hadamard_sumcheck");
    std::vector<EF> base, ext;
    {
        EF e0, eh;
#pragma omp parallel
        {
            EF l0, lh;
            size_t c = 0; bool init = false;
#pragma omp for schedule(static) nowait
            for (size_t i = 0; i < N / 2; i++) {
                if (!init) { c = std::min(col_of(2 * i), ncols_j - 1); init = true; }
                const EF x0 = ext_at(2 * i, c), x1 = ext_at(2 * i + 1, c);
                const F b0 = base_at(2 * i), b1 = base_at(2 * i + 1);
                l0 += x0 * b0;
                lh += (x0 + x1) * (b0 + b1);
            }
#pragma omp critical
            { e0 += l0; eh += lh; }
        }
        EF e1 = round_claim - e0;
        Uni poly = interpolate({EF(), EF::one(), half}, {e0, e1, eh * quarter});
        ch.observe_ext_slice(poly.c.data(), poly.c.size());
        pf.sumcheck.polys.push_back(poly);
        EF alpha = ch.sample_ext();
        point.insert(point.begin(), alpha);
        base.resize(N / 2); ext.resize(N / 2);
#pragma omp parallel
        {
            size_t c = 0; bool init = false;
#pragma omp for schedule(static)
            for (size_t i = 0; i < N / 2; i++) {
                if (!init) { c = std::min(col_of(2 * i), ncols_j - 1); init = true; }
                const EF x0 = ext_at(2 * i, c), x1 = ext_at(2 * i + 1, c);
                const F b0 = base_at(2 * i), b1 = base_at(2 * i + 1);
                base[i] = EF(b0) + alpha * (b1 - b0);
                ext[i] = x0 + alpha * (x1 - x0);
            }
        }
        round_claim = poly.eval(alpha);
    }
    for (unsigned rd = 1; rd < lm; rd++) {
        size_t n = base.size();
        EF e0, eh;
#pragma omp parallel
        {
            EF l0, lh;
#pragma omp for schedule(static) nowait
            for (size_t i = 0; i < n / 2; i++) {
                l0 += ext[2 * i] * base[2 * i];
                lh += (ext[2 * i] + ext[2 * i + 1]) * (base[2 * i] + base[2 * i + 1]);
            }
#pragma omp critical
            { e0 += l0; eh += lh; }
        }
        EF e1 = round_claim - e0;
        Uni poly = interpolate({EF(), EF::one(), half}, {e0, e1, eh * quarter});
        ch.observe_ext_slice(poly.c.data(), poly.c.size());
        pf.sumcheck.polys.push_back(poly);
        EF alpha = ch.sample_ext();
        point.insert(point.begin(), alpha);
        std::vector<EF> nb(n / 2), ne(n / 2);
#pragma omp parallel for schedule(static)
        for (size_t i = 0; i < n / 2; i++) {
            nb[i] = base[2 * i] + alpha * (base[2 * i + 1] - base[2 * i]);
            ne[i] = ext[2 * i] + alpha * (ext[2 * i + 1] - ext[2 * i]);
        }
        base.swap(nb); ext.swap(ne);
        round_claim = poly.eval(alpha);
    }
    pf.sumcheck.point = point;
    pf.sumcheck.eval = round_claim;
    delete t_sc;
    EF base_eval = base[0];
    { OrcTrace t("jagged.eval_sumcheck"); pf.jagged_eval = jagged_eval_prove(jp, z_row, z_col, point, ch); }
    std::vector<std::shared_ptr<StackedRound>> srounds;
    for (auto& r : rounds) {
        srounds.push_back(r.stacked);
        std::vector<std::pair<size_t, size_t>> v;
        for (size_t t = 0; t < r.row_counts.size(); t++) v.push_back({r.row_counts[t], r.col_counts[t]});
        pf.rc_cc.push_back(v);
        pf.merkle_commits.push_back(r.original_commit);
    }
    // prove_untrusted_evaluation: observe the claim, then the stacked proof
    ch.observe_ext(base_eval);
    { OrcTrace t("jagged.stacked_prove"); pf.pcs = stacked_prove(point, srounds, ch, fp, replay_witnesses); }
    pf.expected_eval = base_eval;
    pf.max_log_rows = max_log_rows;
    pf.log_m = lm;
    return pf;
}

// JaggedPcsVerifier::verify_trusted_evaluations (jagged/src/verifier.rs:113-384)
static inline const char* jagged_verify(const std::vector<Digest>& commitments, const std::vector<EF>& point,
                                        const std::vector<std::vector<EF>>& evaluation_claims, const JaggedProof& pf, Challenger& ch,
                                        unsigned log_stack, unsigned max_log_rows, const FriParams& fp) {
    for (auto& v : pf.rc_cc) if (v.empty()) return "IncorrectShape";
    std::vector<size_t> heights;
    for (auto& v : pf.rc_cc) for (auto& rc : v) for (size_t c = 0; c < rc.second; c++) heights.push_back(rc.first);
    if (heights.empty()) return "IncorrectShape";
    JaggedParams jp = jagged_params(heights, max_log_rows);
    if (pf.max_log_rows != max_log_rows || pf.log_m != jp.log_m()) return "IncorrectShape";
    std::vector<EF> z_col = ch.sample_point(log2_ceil(jp.prefix.size() - 1));
    if (point.size() != max_log_rows) return "IncorrectShape";
    size_t nr = commitments.size();
    if (evaluation_claims.size() != nr || pf.rc_cc.size() != nr || pf.merkle_commits.size() != nr) return "IncorrectShape";
    std::vector<size_t> round_areas, added_vals, added_cols;
    size_t R = (size_t)1 << max_log_rows, S = (size_t)1 << log_stack;
    for (size_t r = 0; r < nr; r++) {
        auto& v = pf.rc_cc[r];
        if (v.size() < 2) return "IncorrectShape";
        size_t expect = 0, area = 0;
        for (size_t t = 0; t + 2 < v.size(); t++) { expect += v[t].second; area += v[t].first * v[t].second; }
        if (evaluation_claims[r].size() != expect) return "IncorrectShape";
        std::vector<F> meta{F::from_canonical(v.size())};
        for (auto& rc : v) meta.push_back(F::from_canonical(rc.first));
        for (auto& rc : v) meta.push_back(F::from_canonical(rc.second));
        if (p2_compress(pf.merkle_commits[r], p2_hash(meta)) != commitments[r]) return "IncorrectTableSizes";
        if (area == 0 || area >= ((size_t)1 << 30)) return "AreaOutOfBounds";
        size_t next = ((area + S - 1) / S) * S;
        size_t av = next - area, ac = std::max<size_t>((av + R - 1) / R, 1);
        if (v[v.size() - 2].second + 1 != ac || v.back().second != 1 || v[v.size() - 2].first != R ||
            v.back().first != av - (ac - 1) * R)
            return "IncorrectShape(dummy tables)";
        for (auto& rc : v) if (rc.first > R) return "IncorrectShape";
        round_areas.push_back(area); added_vals.push_back(av); added_cols.push_back(ac);
    }
    if (pf.log_m >= 30) return "AreaOutOfBounds";
    std::vector<EF> column_claims;
    for (size_t r = 0; r < nr; r++) {
        column_claims.insert(column_claims.end(), evaluation_claims[r].begin(), evaluation_claims[r].end());
        column_claims.insert(column_claims.end(), added_cols[r], EF());
    }
    if (jp.prefix.size() != column_claims.size() + 1) return "IncorrectShape";
    if (mle_eval(column_claims.data(), column_claims.size(), z_col) != pf.sumcheck.claimed_sum) return "SumcheckClaimMismatch";
    if (const char* e = sumcheck_partial_verify(pf.sumcheck, ch, jp.log_m(), 2)) return e;
    for (size_t c = 0; c + 1 < jp.prefix.size(); c++) if (jp.prefix[c] > jp.prefix[c + 1]) return "MonotonicityCheckFailed";
    EF jagged_eval;
    if (const char* e = jagged_eval_verify(jp, point, z_col, pf.sumcheck.point, pf.jagged_eval, ch, &jagged_eval)) return e;
    if (pf.expected_eval * jagged_eval != pf.sumcheck.eval) return "JaggedEvalProofVerificationFailed";
    std::vector<size_t> total_areas;
    for (size_t r = 0; r < nr; r++) total_areas.push_back(round_areas[r] + added_vals[r]);
    ch.observe_ext(pf.expected_eval);
    return stacked_verify(pf.merkle_commits, total_areas, pf.sumcheck.point, pf.pcs, pf.expected_eval, ch, log_stack, fp);
}

}  // namespace orc
