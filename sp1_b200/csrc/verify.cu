// ShardVerifier::verify_shard (crates/hypercube/src/verifier/shard.rs:437-750) on the flat proof words of sp1b200_prove_shard, for one
// shard (sp1b200_verify_shard), for every shard of a core proof (sp1b200_verify_core_proof, verify_core.cu) or for a list of recursion
// proofs (sp1b200_verify_compressed, recursion_vks.cu).
// A shard is verified in two phases.  The host phase - the transcript, the PoW checks, the GKR / zerocheck / jagged sumcheck rounds, the
// branching program and every chip's constraints at the zerocheck point (a few thousand extension-field operations) - touches no CUDA
// API: it records the device work the queries need (ShardWork), so the host phases of many shards can run on as many threads.  The
// device phase then runs the recorded work of a batch of shards in three kernels on the context's stream with memory from its pool:
//   verify_merkle_kernel   every Merkle opening of every shard (all commitment rounds and all FRI fold rounds, every query): leaf hash,
//                          path walk, root comparison; and each opening's tensor commitment compress(root, hash([log_h, width]))
//   verify_fold_kernel     per (shard, query): the batched codeword value, the fold chain through the log_stacking_height rounds,
//                          final_poly
//   verify_jagged_kernel   per shard, sum_c col_eq[c] * eq(prefix_c || prefix_{c+1}, point) over every jagged column
// Their flags and partial sums are copied back once per batch.  Checks are reported in verify_shard's order: a check whose inputs come
// from the device is recorded when the transcript reaches it and resolved after the copy, so the verdict names the first failing check,
// as the reference's verifier (and the oracle's restatement of it) would.
#include "ctx.cuh"
#include "challenger.cuh"
#include "hostfield.hpp"
#include "machine.cuh"
#include "poseidon2.cuh"
#include "proof_layout.hpp"
#include "sumcheck.cuh"
#include "verify.cuh"
#include <atomic>
#include <chrono>
#include <cstring>
#include <iterator>
#include <memory>
#include <thread>
#include <vector>

namespace {

using hf::E4;
using hf::canonical;
using kb::Ext;

// ---- device part ----------------------------------------------------------------------------------------------------------------

// one opening: `width` values per query at values_off, log_h sibling digests per query at paths_off (word offsets into the evaluation
// sections on the device); the leaf index of query q is idx[idx_off + q] >> shift (idx_off: the shard's first query index)
struct OpenJob { uint32_t values_off, width, paths_off, root_off, commit_off, log_h, shift, idx_off; };

__device__ __forceinline__ void hash_row(const uint32_t* __restrict__ v, uint32_t n, uint32_t (&d)[8]) {
    uint32_t s[16];
#pragma unroll
    for (int i = 0; i < 16; i++) s[i] = 0;
    uint32_t fill = 0;
    for (uint32_t i = 0; i < n; i++) {   // PaddingFreeSponge<16, 8, 8>: overwrite mode, permute after every chunk
        const uint32_t x = __ldg(v + i);
#pragma unroll
        for (int k = 0; k < 8; k++) if (k == (int)fill) s[k] = x;
        if (++fill == 8) { p2::permute(s); fill = 0; }
    }
    if (fill) p2::permute(s);
#pragma unroll
    for (int i = 0; i < 8; i++) d[i] = s[i];
}
// four words at any word offset (kb::ext_load needs 16-byte alignment; offsets into the proof words have none)
__device__ __forceinline__ Ext ld4(const uint32_t* __restrict__ p) { return Ext{{__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3)}}; }
__device__ __forceinline__ bool digest_eq(const uint32_t (&a)[8], const uint32_t* __restrict__ b) {
    bool eq = true;
#pragma unroll
    for (int i = 0; i < 8; i++) eq &= a[i] == __ldg(b + i);
    return eq;
}

// threads [0, n_jobs * nq): opening (job, query); threads [n_jobs * nq, n_jobs * (nq + 1)): the job's tensor commitment.
// flags[t] = 1 when the check fails.
__global__ void __launch_bounds__(128) verify_merkle_kernel(const OpenJob* __restrict__ jobs, uint32_t n_jobs, uint32_t nq,
                                                            const uint32_t* __restrict__ ev, const uint32_t* __restrict__ idx,
                                                            uint32_t* __restrict__ flags) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n_open = n_jobs * nq;
    if (t >= n_open + n_jobs) return;
    uint32_t d[8];
    if (t < n_open) {
        const OpenJob j = jobs[t / nq];
        const uint32_t q = t % nq;
        hash_row(ev + j.values_off + (uint64_t)q * j.width, j.width, d);
        uint32_t index = __ldg(idx + j.idx_off + q) >> j.shift;
        const uint32_t* sib = ev + j.paths_off + (uint64_t)q * j.log_h * 8;
        for (uint32_t k = 0; k < j.log_h; k++, sib += 8) {
            uint32_t s[8], o[8];
#pragma unroll
            for (int i = 0; i < 8; i++) s[i] = __ldg(sib + i);
            if (index & 1) p2::compress(s, d, o); else p2::compress(d, s, o);
#pragma unroll
            for (int i = 0; i < 8; i++) d[i] = o[i];
            index >>= 1;
        }
        flags[t] = !digest_eq(d, ev + j.root_off);
    } else {
        const OpenJob j = jobs[t - n_open];
        uint32_t s[16];
#pragma unroll
        for (int i = 0; i < 16; i++) s[i] = 0;
        s[0] = kb::from_canonical(j.log_h); s[1] = kb::from_canonical(j.width);
        p2::permute(s);
        uint32_t r[8], h[8], o[8];
#pragma unroll
        for (int i = 0; i < 8; i++) { r[i] = __ldg(ev + j.root_off + i); h[i] = s[i]; }
        p2::compress(r, h, o);
        flags[t] = !digest_eq(o, ev + j.commit_off);
    }
}

// per shard (blockIdx.y) and query q: Σ_c coeff_c · v_c over the component columns of every round, then the fold chain.
// out[q] = first round whose opened pair does not hold the running value (len if none), out[nq + q] = 1 when the chain ends away from
// final_poly.  The *_off / *_at words place the shard's inputs and outputs: ev offsets into the evaluation sections, aux offsets into
// the auxiliary words, out_at into the output words.
struct FoldArgs {
    uint32_t nq, len, n_comp;
    uint32_t comp_off[2], comp_w[2];
    uint32_t g;        // generator of order 2^(len + log_blowup), Montgomery
    uint32_t log_n;    // len + log_blowup
    uint32_t minus1;
    uint32_t final_off;
    uint32_t idx_at, coeff_at, beta_at, fold_off_at, out_at;
};
__global__ void __launch_bounds__(128) verify_fold_kernel(const FoldArgs* __restrict__ args, const uint32_t* __restrict__ ev,
                                                          const uint32_t* __restrict__ aux, uint32_t* __restrict__ out_all) {
    const FoldArgs a = args[blockIdx.y];
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= a.nq) return;
    const uint32_t *idx = aux + a.idx_at, *coeffs = aux + a.coeff_at, *betas = aux + a.beta_at, *fold_off = aux + a.fold_off_at;
    uint32_t* out = out_all + a.out_at;
    Ext folded = kb::ext_zero();
    uint32_t k = 0;
    for (uint32_t r = 0; r < a.n_comp; r++) {
        const uint32_t* v = ev + a.comp_off[r] + (uint64_t)q * a.comp_w[r];
        for (uint32_t c = 0; c < a.comp_w[r]; c++, k++) folded = kb::ext_add(folded, kb::ext_mul_base(ld4(coeffs + 4 * k), __ldg(v + c)));
    }
    uint32_t index = __ldg(idx + q);
    const uint32_t rev = __brev(index) >> (32 - a.log_n);
    uint32_t xi = kb::pow(a.g, rev);
    uint32_t first_bad = a.len;
    for (uint32_t r = 0; r < a.len; r++) {
        const uint32_t* v = ev + __ldg(fold_off + r) + (uint64_t)q * 8;
        const Ext e0 = ld4(v), e1 = ld4(v + 4);
        if (!kb::ext_eq((index & 1) ? e1 : e0, folded)) { first_bad = r; break; }
        const uint32_t x0 = (index & 1) ? kb::mul(xi, a.minus1) : xi, x1 = (index & 1) ? xi : kb::mul(xi, a.minus1);
        const Ext bx = kb::ext_sub(ld4(betas + 4 * r), kb::ext_from_base(x0));
        folded = kb::ext_add(e0, kb::ext_mul_base(kb::ext_mul(bx, kb::ext_sub(e1, e0)), kb::inv(kb::sub(x1, x0))));
        index >>= 1;
        xi = kb::mul(xi, xi);
    }
    out[q] = first_bad;
    out[a.nq + q] = first_bad == a.len && !kb::ext_eq(folded, ld4(ev + a.final_off));
}

// per shard (blockIdx.y): sum_c col_eq[c] * prod_i eq(bit_i, point_i) over the 2 (log_m + 1) bits of prefix[c] || prefix[c+1] (most
// significant first), one column per thread; per-block sums to partial[block] of the shard's own partial range
struct JagArgs { uint32_t prefix_at, n_cols, col_eq_at, point_at, nb, partial_at; };   // aux offsets (prefix_at in 64-bit words)
__global__ void __launch_bounds__(256) verify_jagged_kernel(const JagArgs* __restrict__ args, const uint32_t* __restrict__ aux,
                                                            uint32_t* __restrict__ out_all) {
    const JagArgs ja = args[blockIdx.y];
    const uint64_t* prefix = reinterpret_cast<const uint64_t*>(aux) + ja.prefix_at;
    const uint32_t *col_eq = aux + ja.col_eq_at, *point = aux + ja.point_at;
    const uint32_t n_cols = ja.n_cols, nb = ja.nb;
    uint32_t* partial = out_all + ja.partial_at;
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    Ext acc[1] = {kb::ext_zero()};
    if (c < n_cols) {
        const uint64_t a = prefix[c], b = prefix[c + 1];
        Ext f = ld4(col_eq + 4 * (uint64_t)c);
        for (uint32_t i = 0; i < 2 * nb; i++) {
            const uint64_t x = i < nb ? a : b;
            const uint32_t bit = (uint32_t)(x >> (nb - 1 - (i < nb ? i : i - nb))) & 1u;
            const Ext p = ld4(point + 4 * i);
            f = kb::ext_mul(f, bit ? p : kb::ext_sub(kb::ext_one(), p));
        }
        acc[0] = f;
    }
    block_reduce<1>(acc, partial, Mail{nullptr, nullptr, 0});
}

// ---- host part ------------------------------------------------------------------------------------------------------------------

const char* const VERDICT_NAMES[] = {
    "Accepted", "Pow", "InvalidShape", "ZeroDenominator", "CumulativeSumMismatch", "InvalidShape(rounds)", "InconsistentSumcheckClaim",
    "InvalidProofShape", "InconsistencyWithClaimedSum", "SumcheckRoundInconsistency", "InvalidProofShape(point)", "InconsistencyWithEval",
    "InconsistentEvaluation", "InvalidLastLayerDimension", "TracePointMismatch", "InvalidShape(openings)", "NumeratorEvaluationMismatch",
    "DenominatorEvaluationMismatch", "OpeningShape", "InvalidHeightBitDecomposition", "HeightTooLarge",
    "ConstraintsCheckFailed(InconsistencyWithEval)", "ConstraintsCheckFailed(InconsistencyWithClaimedSum)", "IncorrectShape",
    "IncorrectTableSizes", "AreaOutOfBounds", "IncorrectShape(dummy tables)", "SumcheckClaimMismatch", "MonotonicityCheckFailed",
    "JaggedEvaluationFailed", "JaggedEvalProofVerificationFailed", "StackingError", "BatchPow", "SumcheckFriLengthMismatch", "Sumcheck",
    "TwoAdicityOverflow", "TcsError(component)", "QueryValueMismatch", "TcsError(query)", "QueryFinalPolyMismatch",
    "SumcheckFinalPolyMismatch", "InvalidShape(preprocessed widths)", "InvalidShape(chip tables)"};
// indexed by the shard verdict codes of include/sp1b200.h; the core-proof verdicts follow them (verify_core.cu)
static_assert(std::size(VERDICT_NAMES) == SP1B200_VERDICT_EMPTY_PROOF, "one name per shard verdict code of include/sp1b200.h");

inline bool neq(const E4& a, const E4& b) { return !(a == b); }
inline E4 ld(const uint32_t* p) { return E4::load(p); }
inline E4 eqf(const E4& a, const E4& b) { return a * b + (E4::one() - a) * (E4::one() - b); }
inline E4 base(uint64_t canonical) { return E4::from_base(kb::to_monty_c(canonical)); }

std::vector<E4> ext_vec(const uint32_t* p, size_t n) { std::vector<E4> v(n); for (size_t i = 0; i < n; i++) v[i] = ld(p + 4 * i); return v; }
std::vector<E4> point_from_usize(uint64_t x, unsigned dim) {
    std::vector<E4> p(dim);
    for (unsigned i = 0; i < dim; i++) p[i] = base((x >> (dim - 1 - i)) & 1);
    return p;
}
E4 full_geq(const std::vector<E4>& threshold, const std::vector<E4>& point) {
    E4 acc = E4::one();
    for (size_t i = threshold.size(); i-- > 0;) {
        const E4 &x = threshold[i], &y = point[i];
        acc = ((E4::one() - y) * (E4::one() - x) + y * x) * acc + y * (E4::one() - x);
    }
    return acc;
}

// BranchingProgram::eval (slop/crates/jagged/src/poly.rs:136-175, :384-470); points are big-endian
struct BranchingProgram {
    const std::vector<E4>& z_row; const std::vector<E4>& z_index; size_t num_vars;
    static E4 lsb(const std::vector<E4>& p, size_t i) { return p.size() <= i ? E4() : p[p.size() - 1 - i]; }
    E4 eval(const std::vector<E4>& prefix, const std::vector<E4>& next) const {
        E4 res[4]; res[2] = E4::one();
        for (size_t layer = num_vars + 1; layer-- > 0;) {
            const std::vector<E4> eq = hf::partial_lagrange({lsb(z_row, layer), lsb(z_index, layer), lsb(prefix, layer), lsb(next, layer)});
            E4 nres[4];
            for (int st = 0; st < 4; st++) {
                E4 acc[4];
                for (int i = 0; i < 16; i++) {
                    const int o = bp_transition((i >> 3) & 1, (i >> 2) & 1, (i >> 1) & 1, i & 1, st);
                    if (o >= 0) acc[o] = acc[o] + eq[i];
                }
                for (int k = 0; k < 4; k++) nres[st] = nres[st] + acc[k] * res[k];
            }
            for (int k = 0; k < 4; k++) res[k] = nres[k];
        }
        return res[0];
    }
};

// a check whose inputs the device computes, resolved after the final copy; job: the opening job (local index) of a TcsError check
struct Deferred { uint32_t code; uint32_t job; };
constexpr uint32_t NO_JOB = ~0u;

// one shard's verifier: the host phase (run) records the device work, resolve() reads the device results back in verify_shard's order
struct Verifier {
    const sp1b200_params& prm;
    const sp1b200_machine* m;
    const HostInteractions& H;
    const layout::ShardProof& p;
    const uint64_t* heights;
    const char* const* names;
    const std::vector<size_t>& ncols;
    const uint32_t* prep_commit8;
    const uint32_t* ev_base;   // host start of the evaluation section (device offsets are relative to it)
    uint64_t ev_words;
    HostChallenger ch;
    uint32_t mlr, ls, lb, nq;

    // outcome of the host phase: `verdict` is a failure found before any device check; otherwise the deferred checks, then host_fail,
    // then tail_fail (the chip-table check) decide
    uint32_t verdict = SP1B200_VERDICT_ACCEPT, host_fail = SP1B200_VERDICT_ACCEPT, tail_fail = SP1B200_VERDICT_ACCEPT;
    std::vector<Deferred> deferred;
    // recorded device work.  Jagged column sum: the column prefix sums, eq(z_col, c) and the jagged-eval point; acc * jag_bp ==
    // jag_expect is checked after the copy
    bool jag = false;
    std::vector<uint64_t> prefix;
    std::vector<uint32_t> col_eq, jag_point;
    uint32_t jag_nb = 0, jag_cols = 0;
    E4 jag_bp, jag_expect;
    // BaseFold queries: openings (offsets into the evaluation section), query indices, batching coefficients, fold betas, the fold
    // rounds' value offsets, and the fold arguments (offsets relative to this shard)
    bool fold = false;
    std::vector<OpenJob> jobs;
    std::vector<uint32_t> idx, coeff_words, beta_words, fold_offs;
    FoldArgs fa{};

    Verifier(const sp1b200_params& pr, const sp1b200_machine* mm, const layout::ShardProof& pp, const uint64_t* h, const char* const* nm,
             const std::vector<size_t>& nc, const uint32_t* pc8)
        : prm(pr), m(mm), H(*static_cast<const HostInteractions*>(mm->interactions)), p(pp), heights(h), names(nm), ncols(nc),
          prep_commit8(pc8), ev_base(pp.univariate), ev_words((uint64_t)(pp.pv - pp.univariate)) {
        mlr = pr.max_log_row_count; ls = pr.log_stacking_height; lb = pr.log_blowup; nq = pr.num_queries;
    }

    uint32_t off(const uint32_t* ptr) const { return (uint32_t)(ptr - ev_base); }
    void observe_ext(const E4& e) { ch.observe_n(e.c, 4); }
    void observe_var_ext(const uint32_t* w, size_t n) { ch.observe(kb::to_monty_c(n)); ch.observe_n(w, 4 * n); }
    E4 sample_ext() { E4 e; ch.sample_ext(e.c); return e; }
    std::vector<E4> sample_point(size_t n) { std::vector<E4> v(n); for (auto& x : v) x = sample_ext(); return v; }

    // partially_verify_sumcheck_proof (slop/crates/sumcheck/src/verifier.rs:21-107)
    uint32_t sumcheck(const layout::Sumcheck& s, size_t nvars, size_t degree) {
        const size_t n = s.polys.size();
        if (n != nvars || nvars == 0) return SP1B200_VERDICT_SUMCHECK_PROOF_SHAPE;
        auto eval = [&](size_t i, const E4& x) { E4 r; for (size_t k = s.n_coeffs[i]; k-- > 0;) r = r * x + ld(s.polys[i] + 4 * k); return r; };
        auto sum01 = [&](size_t i) { E4 r = s.n_coeffs[i] ? ld(s.polys[i]) : E4(); for (size_t k = 0; k < s.n_coeffs[i]; k++) r = r + ld(s.polys[i] + 4 * k); return r; };
        if (neq(sum01(0), ld(s.claimed_sum))) return SP1B200_VERDICT_SUMCHECK_CLAIMED_SUM;
        if (s.n_coeffs[0] != degree + 1) return SP1B200_VERDICT_SUMCHECK_PROOF_SHAPE;
        ch.observe_n(s.polys[0], 4 * (size_t)s.n_coeffs[0]);
        std::vector<E4> alphas;   // most recent first
        for (size_t i = 1; i < n; i++) {
            if (s.n_coeffs[i] != degree + 1) return SP1B200_VERDICT_SUMCHECK_PROOF_SHAPE;
            const E4 a = sample_ext();
            alphas.insert(alphas.begin(), a);
            if (neq(eval(i - 1, a), sum01(i))) return SP1B200_VERDICT_SUMCHECK_ROUND;
            ch.observe_n(s.polys[i], 4 * (size_t)s.n_coeffs[i]);
        }
        const E4 a = sample_ext();
        alphas.insert(alphas.begin(), a);
        for (size_t i = 0; i < n; i++) if (neq(alphas[i], ld(s.point + 4 * i))) return SP1B200_VERDICT_SUMCHECK_POINT;
        if (neq(eval(n - 1, a), ld(s.eval))) return SP1B200_VERDICT_SUMCHECK_EVAL;
        return SP1B200_VERDICT_ACCEPT;
    }

    E4 vcol(const VColDev& v, const E4* prep, const E4* main) const {
        E4 r = E4::from_base(v.constant);
        if (!main) return r;
        for (uint32_t t = 0; t < v.n_terms; t++) {
            const TermDev& tm = H.terms[v.term_start + t];
            r = r + (tm.source == LEAF_MAIN ? main : prep)[tm.col] * tm.weight;
        }
        return r;
    }

    // LogUpGkrVerifier::verify_logup_gkr (crates/hypercube/src/logup_gkr/verifier.rs:84-330), expected cumulative sum 0
    uint32_t gkr() {
        const size_t nch = m->chips.size();
        size_t arity = 1, ni = 0;
        for (auto& c : H.per_chip) { ni += c.size(); for (auto& in : c) arity = std::max<size_t>(arity, in.n_values + 1); }
        const unsigned bdim = hf::log2_ceil(arity);
        if (!ch.check_witness(prm.gkr_pow_bits, p.gkr_witness[0])) return SP1B200_VERDICT_POW;
        const E4 alpha = sample_ext();
        const std::vector<E4> beta_seed = sample_point(bdim);
        (void)sample_ext();
        const unsigned v = hf::log2_ceil(ni);
        const size_t expected = (size_t)1 << (v + 1);
        if (p.n_out != expected) return SP1B200_VERDICT_INVALID_SHAPE;
        observe_var_ext(p.out_num, p.n_out);
        observe_var_ext(p.out_den, p.n_out);
        const std::vector<E4> num = ext_vec(p.out_num, expected), den = ext_vec(p.out_den, expected);
        E4 cum;
        for (size_t i = 0; i < expected; i++) { if (den[i].is_zero()) return SP1B200_VERDICT_ZERO_DENOMINATOR; cum = cum + num[i] * kb::ext_inv(den[i]); }
        if (!cum.is_zero()) return SP1B200_VERDICT_CUMULATIVE_SUM_MISMATCH;
        std::vector<E4> point = sample_point(v + 1);
        E4 num_eval = hf::mle_eval(num, point), den_eval = hf::mle_eval(den, point);
        if (p.rounds.size() + 1 != mlr) return SP1B200_VERDICT_INVALID_SHAPE_ROUNDS;
        for (size_t i = 0; i < p.rounds.size(); i++) {
            const layout::GkrRound& r = p.rounds[i];
            const E4 lambda = sample_ext();
            if (neq(ld(r.sc.claimed_sum), num_eval * lambda + den_eval)) return SP1B200_VERDICT_INCONSISTENT_SUMCHECK_CLAIM;
            if (uint32_t e = sumcheck(r.sc, i + v + 1, 3)) return e;
            const E4 n0 = ld(r.nd), n1 = ld(r.nd + 4), d0 = ld(r.nd + 8), d1 = ld(r.nd + 12);
            E4 eqv = E4::one();
            for (size_t k = 0; k < point.size(); k++) eqv = eqv * eqf(ld(r.sc.point + 4 * k), point[k]);
            if (neq(ld(r.sc.eval), eqv * ((n0 * d1 + n1 * d0) * lambda + d0 * d1))) return SP1B200_VERDICT_INCONSISTENT_EVALUATION;
            ch.observe_n(r.nd, 16);
            point = ext_vec(r.sc.point, r.sc.polys.size());
            const E4 lc = sample_ext();
            point.push_back(lc);
            num_eval = n0 + (n1 - n0) * lc;
            den_eval = d0 + (d1 - d0) * lc;
        }
        const std::vector<E4> ipt(point.begin(), point.begin() + v), tpt(point.begin() + v, point.end());
        if (tpt.size() != mlr) return SP1B200_VERDICT_LAST_LAYER_DIMENSION;
        for (uint32_t k = 0; k < mlr; k++) if (neq(tpt[k], ld(p.gkr_point + 4 * k))) return SP1B200_VERDICT_TRACE_POINT_MISMATCH;
        const std::vector<E4> betas = hf::partial_lagrange(beta_seed);
        std::vector<E4> pe{E4()};
        pe.insert(pe.end(), tpt.begin(), tpt.end());
        std::vector<E4> nv, dv;
        ch.observe(kb::to_monty_c(nch));
        for (size_t k = 0; k < nch; k++) {
            const ChipProg& c = m->chips[k];
            if (c.prep_w) observe_var_ext(p.gkr_prep[k], c.prep_w);
            observe_var_ext(p.gkr_main[k], c.main_w);
            const E4 geq = full_geq(point_from_usize(heights[k], mlr + 1), pe);
            const std::vector<E4> mo = ext_vec(p.gkr_main[k], c.main_w), po = ext_vec(p.gkr_prep[k], c.prep_w);
            for (const InterDev& in : H.per_chip[k]) {
                auto fraction = [&](const E4* prep, const E4* main, E4& n, E4& d) {
                    d = alpha + betas[0] * kb::to_monty_c(in.arg_index);
                    for (uint32_t q = 0; q < in.n_values; q++) d = d + betas[q + 1] * vcol(H.vcols[in.vcol_start + 1 + q], prep, main);
                    n = vcol(H.vcols[in.vcol_start], prep, main);
                };
                E4 rn, rd, pn, pd;
                fraction(po.data(), mo.data(), rn, rd);
                fraction(nullptr, nullptr, pn, pd);   // the all-zero row: constants only
                const E4 ne = rn - pn * geq, de = rd + (E4::one() - pd) * geq;
                nv.push_back(in.is_send ? ne : E4() - ne);
                dv.push_back(de);
            }
        }
        nv.resize((size_t)1 << v, E4()); dv.resize((size_t)1 << v, E4::one());
        if (neq(num_eval, hf::mle_eval(nv, ipt))) return SP1B200_VERDICT_NUMERATOR_EVALUATION;
        if (neq(den_eval, hf::mle_eval(dv, ipt))) return SP1B200_VERDICT_DENOMINATOR_EVALUATION;
        return SP1B200_VERDICT_ACCEPT;
    }

    // the chip's constraints folded with the reversed α powers (the verifier folder's Horner order) at one row of extension values;
    // null columns: the all-zero row
    E4 eval_air(size_t k, const E4* prep, const E4* main, const std::vector<E4>& powers) const {
        return host_eval_constraints(m->host[k], m->chips[k].n_regs, p.pv, powers,
                                     [&](const LeafRef& l) { return main ? (l.source == LEAF_MAIN ? main : prep)[l.col] : E4(); });
    }

    // ShardVerifier::verify_zerocheck (crates/hypercube/src/verifier/shard.rs:288-434)
    uint32_t zerocheck() {
        const size_t nch = m->chips.size();
        const E4 alpha = sample_ext(), gkr_c = sample_ext(), lambda = sample_ext();
        if (p.zc.polys.size() != mlr) return SP1B200_VERDICT_INVALID_SHAPE;
        const std::vector<E4> zp = ext_vec(p.zc.point, mlr);
        E4 eqv = E4::one();
        for (uint32_t i = 0; i < mlr; i++) eqv = eqv * eqf(ld(p.gkr_point + 4 * i), zp[i]);
        std::vector<E4> pt{E4()};
        pt.insert(pt.end(), zp.begin(), zp.end());
        E4 rlc;
        for (size_t k = 0; k < nch; k++) {
            const ChipProg& c = m->chips[k];
            const std::vector<E4> degree = point_from_usize(heights[k], mlr + 1);
            for (size_t i = 1; i < degree.size(); i++) if (!(degree[i] * degree[0]).is_zero()) return SP1B200_VERDICT_HEIGHT_TOO_LARGE;
            const E4 geq = full_geq(degree, pt);
            std::vector<E4> rev(c.n_constraints);
            E4 pw = E4::one();
            for (uint32_t i = 0; i < c.n_constraints; i++) { rev[c.n_constraints - 1 - i] = pw; pw = pw * alpha; }
            const std::vector<E4> mo = ext_vec(p.zc_main[k], c.main_w), po = ext_vec(p.zc_prep[k], c.prep_w);
            const E4 pra = eval_air(k, nullptr, nullptr, rev);
            const E4 ce = eval_air(k, po.data(), mo.data(), rev) - pra * geq;
            const E4 ob = batched_opening_claim(p.zc_main[k], c.main_w, p.zc_prep[k], c.prep_w, gkr_c);
            rlc = rlc * lambda + eqv * (ce + ob);
        }
        if (neq(ld(p.zc.eval), rlc)) return SP1B200_VERDICT_CONSTRAINTS_EVAL;
        E4 mod;
        for (size_t k = 0; k < nch; k++)
            mod = lambda * mod + batched_opening_claim(p.gkr_main[k], m->chips[k].main_w, p.gkr_prep[k], m->chips[k].prep_w, gkr_c);
        if (neq(ld(p.zc.claimed_sum), mod)) return SP1B200_VERDICT_CONSTRAINTS_CLAIMED_SUM;
        if (uint32_t e = sumcheck(p.zc, mlr, 4)) return e;
        ch.observe(kb::to_monty_c(nch));
        for (size_t k = 0; k < nch; k++) { observe_var_ext(p.zc_prep[k], m->chips[k].prep_w); observe_var_ext(p.zc_main[k], m->chips[k].main_w); }
        return SP1B200_VERDICT_ACCEPT;
    }

    // JaggedPcsVerifier::verify_trusted_evaluations (slop/crates/jagged/src/verifier.rs:113-384) with the stacked and BaseFold verifiers
    // behind it; commitments = {preprocessed,} main
    void jagged(const std::vector<const uint32_t*>& commitments) {
        const size_t nr = commitments.size();
        for (auto& v : p.rc_cc) if (v.empty()) { verdict = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
        // column heights as (rows, cols) runs; totals in 128 bits so that no count in the words can wrap them
        unsigned __int128 total_cols = 0, total_area = 0;
        for (auto& v : p.rc_cc) for (auto& rc : v) { total_cols += rc.second; total_area += (unsigned __int128)rc.first * rc.second; }
        if (total_cols == 0) { verdict = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
        const uint64_t area64 = total_area >> 63 ? ~(uint64_t)0 : (uint64_t)total_area;
        if (p.max_log_rows != mlr || p.log_m != hf::log2_ceil(area64) || total_area >> 63) { verdict = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
        // log_m matches the area, so the columns with rows are few; a column count that is absurd only through empty tables cannot be
        // laid out
        if (total_cols > ((uint64_t)1 << 24)) { verdict = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
        const size_t n_cols = (size_t)total_cols;
        std::vector<uint64_t> prefix{0};
        prefix.reserve(n_cols + 1);
        for (auto& v : p.rc_cc) layout::append_column_prefix(prefix, v);
        const std::vector<E4> z_col = sample_point(hf::log2_ceil(n_cols));
        const uint64_t R = (uint64_t)1 << mlr;
        std::vector<uint64_t> padded_area(nr), added_cols(nr);
        std::vector<std::vector<E4>> claims(nr);
        for (size_t r = 0; r < nr; r++) {
            const auto& v = p.rc_cc[r];
            if (v.size() < 2) { verdict = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
            uint64_t expect = 0, area = 0;
            for (size_t t = 0; t + 2 < v.size(); t++) { expect += v[t].second; area += (uint64_t)v[t].first * v[t].second; }
            // the claims of round r are the zerocheck's opened values of that round's columns, in chip order
            size_t have = 0;
            for (size_t k = 0; k < m->chips.size(); k++) have += (nr == 2 && r == 0) ? m->chips[k].prep_w : m->chips[k].main_w;
            if (have != expect) { verdict = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
            for (size_t k = 0; k < m->chips.size(); k++) {
                const bool prep = nr == 2 && r == 0;
                const uint32_t w = prep ? m->chips[k].prep_w : m->chips[k].main_w;
                const uint32_t* o = prep ? p.zc_prep[k] : p.zc_main[k];
                for (uint32_t j = 0; j < w; j++) claims[r].push_back(ld(o + 4 * j));
            }
            uint32_t cm[8];
            table_size_commitment(p.merkle_commits + 8 * r, v, cm);
            if (memcmp(cm, commitments[r], 32)) { verdict = SP1B200_VERDICT_INCORRECT_TABLE_SIZES; return; }
            if (area == 0 || area >= ((uint64_t)1 << 30)) { verdict = SP1B200_VERDICT_AREA_OUT_OF_BOUNDS; return; }
            const layout::Tables pad = layout::padding_tables(area, ls, mlr);
            if (!std::equal(pad.begin(), pad.end(), v.end() - 2)) { verdict = SP1B200_VERDICT_DUMMY_TABLES; return; }
            for (auto& rc : v) if (rc.first > R) { verdict = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
            padded_area[r] = layout::stacked_columns(area, ls) << ls; added_cols[r] = pad[0].second + pad[1].second;
        }
        if (p.log_m >= 30) { verdict = SP1B200_VERDICT_AREA_OUT_OF_BOUNDS; return; }
        std::vector<E4> column_claims;
        for (size_t r = 0; r < nr; r++) { column_claims.insert(column_claims.end(), claims[r].begin(), claims[r].end()); column_claims.resize(column_claims.size() + added_cols[r]); }
        if (prefix.size() != column_claims.size() + 1) { verdict = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
        if (neq(hf::mle_eval(column_claims, z_col), ld(p.jagged_sc.claimed_sum))) { verdict = SP1B200_VERDICT_SUMCHECK_CLAIM_MISMATCH; return; }
        if ((verdict = sumcheck(p.jagged_sc, p.log_m, 2))) return;
        for (size_t c = 0; c + 1 < prefix.size(); c++) if (prefix[c] > prefix[c + 1]) { verdict = SP1B200_VERDICT_MONOTONICITY; return; }
        // JaggedEvalSumcheckConfig::jagged_evaluation (slop/crates/jagged/src/jagged_eval/sumcheck_eval.rs:45-155)
        const uint32_t lm = p.log_m;
        observe_ext(ld(p.jagged_eval.claimed_sum));
        if ((verdict = sumcheck(p.jagged_eval, 2 * (lm + 1), 2))) return;
        {
            const std::vector<E4> jp = ext_vec(p.jagged_eval.point, 2 * (lm + 1));
            const std::vector<E4> first(jp.begin(), jp.begin() + lm + 1), second(jp.begin() + lm + 1, jp.end());
            const std::vector<E4> z_row = ext_vec(p.zc.point, mlr), z_trace = ext_vec(p.jagged_sc.point, p.jagged_sc.polys.size());
            jag_bp = BranchingProgram{z_row, z_trace, std::max(z_row.size(), z_trace.size())}.eval(first, second);
            jag_expect = ld(p.jagged_eval.eval);
            // the column sum on the device, one thread per column; eq(z_col, c) is tabled here
            const std::vector<E4> eq = hf::partial_lagrange(z_col);
            col_eq.resize(4 * eq.size());
            for (size_t c = 0; c < eq.size(); c++) eq[c].store(&col_eq[4 * c]);
            jag_point.assign(p.jagged_eval.point, p.jagged_eval.point + 8 * (size_t)(lm + 1));
            jag_nb = lm + 1;
            jag_cols = (uint32_t)n_cols;
            this->prefix = std::move(prefix);
            jag = true;
        }
        const E4 jagged_eval = ld(p.jagged_eval.claimed_sum);
        // (the check acc == eval of the jagged-eval sumcheck is resolved with the device flags; nothing below reads acc)
        deferred.push_back(Deferred{SP1B200_VERDICT_JAGGED_EVALUATION, NO_JOB});
        if (neq(ld(p.expected_eval) * jagged_eval, ld(p.jagged_sc.eval))) { host_fail = SP1B200_VERDICT_JAGGED_EVAL_PROOF; return; }
        observe_ext(ld(p.expected_eval));
        stacked(padded_area);
    }

    // StackedPcsVerifier::verify_trusted_evaluation (slop/crates/stacked/src/verifier.rs:39-99)
    void stacked(const std::vector<uint64_t>& areas) {
        const size_t npt = p.jagged_sc.polys.size();
        if (npt < ls) { host_fail = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
        const std::vector<E4> pt = ext_vec(p.jagged_sc.point, npt);
        const std::vector<E4> batch_point(pt.begin(), pt.end() - ls), stack_point(pt.end() - ls, pt.end());
        std::vector<E4> flat;
        for (size_t r = 0; r < areas.size(); r++) {
            if (areas[r] % ((uint64_t)1 << ls) || (areas[r] >> ls) != ncols[r]) { host_fail = SP1B200_VERDICT_INCORRECT_SHAPE; return; }
            const std::vector<E4> e = ext_vec(p.batch_evals[r], ncols[r]);
            flat.insert(flat.end(), e.begin(), e.end());
        }
        if (neq(ld(p.expected_eval), hf::mle_eval(flat, batch_point))) { host_fail = SP1B200_VERDICT_STACKING; return; }
        for (size_t r = 0; r < areas.size(); r++) ch.observe_n(p.batch_evals[r], 4 * ncols[r]);
        basefold(stack_point, flat);
    }

    // BasefoldVerifier::verify_mle_evaluations (slop/crates/basefold/src/verifier.rs:122-420)
    void basefold(const std::vector<E4>& point, const std::vector<E4>& claims) {
        if (!ch.check_witness(prm.batch_pow_bits, p.batch_witness[0])) { host_fail = SP1B200_VERDICT_BATCH_POW; return; }
        const std::vector<E4> coeffs = hf::partial_lagrange(sample_point(hf::log2_ceil(claims.size())));
        E4 claim;
        for (size_t k = 0; k < claims.size(); k++) claim = claim + claims[k] * coeffs[k];
        const size_t len = ls;
        if (point.size() != len || len == 0) { host_fail = SP1B200_VERDICT_FRI_LENGTH; return; }
        ch.observe(kb::to_monty_c(len));
        std::vector<E4> betas;
        for (size_t i = 0; i < len; i++) {
            ch.observe_n(p.univariate + 8 * i, 8);
            ch.observe_n(p.fri_commits + 8 * i, 8);
            betas.push_back(sample_ext());
        }
        E4 expected = claim;
        for (size_t i = 0; i < len; i++) {
            const E4 p0 = ld(p.univariate + 8 * i), p1 = ld(p.univariate + 8 * i + 4), x = point[len - 1 - i];
            if (neq(expected, (E4::one() - x) * p0 + x * p1)) { host_fail = SP1B200_VERDICT_BASEFOLD_SUMCHECK; return; }
            expected = p0 + betas[i] * p1;
        }
        ch.observe_n(p.final_poly, 4);
        if (!ch.check_witness(prm.pow_bits, p.pow_witness[0])) { host_fail = SP1B200_VERDICT_POW; return; }
        const uint32_t log_n = (uint32_t)len + lb;
        if (log_n > 24) { host_fail = SP1B200_VERDICT_TWO_ADICITY; return; }
        idx.resize(nq);
        for (auto& q : idx) q = ch.sample_bits(log_n);
        // device: every opening, and the fold chain of every query
        const size_t ncomp = ncols.size();
        for (size_t r = 0; r < ncomp; r++) {   // component openings are checked against the jagged round's original commitments
            const layout::Opening& o = p.component[r];
            jobs.push_back(OpenJob{off(o.values), o.width, off(o.paths), off(o.root), off(p.merkle_commits + 8 * r), o.log_height, 0, 0});
        }
        for (size_t r = 0; r < len; r++) {
            const layout::Opening& o = p.query[r];
            jobs.push_back(OpenJob{off(o.values), o.width, off(o.paths), off(o.root), off(p.fri_commits + 8 * r), o.log_height, (uint32_t)r + 1, 0});
        }
        for (size_t k = 0; k < claims.size(); k++) for (int i = 0; i < 4; i++) coeff_words.push_back(coeffs[k].c[i]);
        for (auto& b : betas) for (int i = 0; i < 4; i++) beta_words.push_back(b.c[i]);
        for (size_t r = 0; r < len; r++) fold_offs.push_back(off(p.query[r].values));
        fa.nq = nq; fa.len = (uint32_t)len; fa.n_comp = (uint32_t)ncomp;
        for (size_t r = 0; r < ncomp; r++) { fa.comp_off[r] = off(p.component[r].values); fa.comp_w[r] = p.component[r].width; }
        fa.log_n = log_n;
        fa.g = kb::pow(kb::to_monty_c(3), (uint64_t)127 << (24 - log_n));
        fa.minus1 = kb::pow(kb::to_monty_c(3), (uint64_t)127 << 23);
        fa.final_off = off(p.final_poly);
        fold = true;
        // the device checks in verify_mle_evaluations' order: component openings round by round, then per fold round the opened value
        // and that round's openings, then final_poly
        for (size_t r = 0; r < ncomp; r++) deferred.push_back(Deferred{SP1B200_VERDICT_TCS_COMPONENT, (uint32_t)r});
        for (size_t r = 0; r < len; r++) {
            deferred.push_back(Deferred{SP1B200_VERDICT_QUERY_VALUE, (uint32_t)r});
            deferred.push_back(Deferred{SP1B200_VERDICT_TCS_QUERY, (uint32_t)(ncomp + r)});
        }
        deferred.push_back(Deferred{SP1B200_VERDICT_QUERY_FINAL_POLY, NO_JOB});
        const E4 f = ld(p.final_poly);
        if (neq(f, ld(p.univariate + 8 * (len - 1)) + betas.back() * ld(p.univariate + 8 * (len - 1) + 4)))
            host_fail = SP1B200_VERDICT_SUMCHECK_FINAL_POLY;
    }


    // the last checks of verify_shard (shard.rs:662-742): without its two dummy tables, each round lists one table per chip (per chip
    // with preprocessed columns in the preprocessed round), in chip order, with that chip's height as its row count and its width as
    // its column count.  The table-size hash only binds these counts to the prover's own commitment, so without this check a proof
    // could commit a jagged layout other than the heights the LogUp-GKR and zerocheck corrections use.
    uint32_t chip_tables() const {
        const size_t nr = p.rc_cc.size();
        for (size_t r = 0; r < nr; r++) {
            const bool prep = nr == 2 && r == 0;
            std::vector<std::pair<uint64_t, uint64_t>> want;
            for (size_t k = 0; k < m->chips.size(); k++) {
                const uint32_t w = prep ? m->chips[k].prep_w : m->chips[k].main_w;
                if (!prep || w) want.emplace_back(heights[k], w);
            }
            const auto& v = p.rc_cc[r];
            if (v.size() != want.size() + 2) return SP1B200_VERDICT_CHIP_TABLES;
            for (size_t t = 0; t < want.size(); t++)
                if (v[t].first != want[t].first || v[t].second != want[t].second) return SP1B200_VERDICT_CHIP_TABLES;
        }
        return SP1B200_VERDICT_ACCEPT;
    }

    // the host phase: the shard's own words enter the transcript started from `start` - public values, main commitment, chip shapes
    // (shard.rs:437-470) - then every host check in verify_shard's order, recording the device work.  No CUDA call.
    void run(const uint32_t* start) {
        const size_t nch = m->chips.size();
        ch.load(start);
        ch.observe_n(p.pv, p.n_pv);
        ch.observe_n(p.commit, 8);
        observe_chip_shapes(ch, nch, heights, names);
        if (nch && mlr + 1 >= 30) verdict = SP1B200_VERDICT_INVALID_SHAPE;   // a degree point of 30 or more bits (shard.rs:477)
        // the preprocessed round's leading column counts are the preprocessed widths (shard.rs:506-523)
        const bool has_prep = ncols.size() == 2;
        if (!verdict && has_prep) {
            size_t t = 0;
            for (size_t k = 0; k < nch && !verdict; k++) {
                if (!m->chips[k].prep_w) continue;
                if (t >= p.rc_cc[0].size() || p.rc_cc[0][t].second != m->chips[k].prep_w) verdict = SP1B200_VERDICT_PREPROCESSED_WIDTHS;
                t++;
            }
        }
        if (!verdict) verdict = gkr();
        if (!verdict) verdict = zerocheck();
        if (!verdict) {
            std::vector<const uint32_t*> commits;
            if (has_prep) commits.push_back(prep_commit8);
            commits.push_back(p.commit);
            jagged(commits);
        }
        if (!verdict) tail_fail = chip_tables();
    }

    // where the device phase put this shard's results: its first opening job, its fold words, its jagged partials
    uint32_t job0 = 0, fold_at = 0, jag_at = 0;

    // the checks in order after the device phase: an immediate verdict, then the deferred checks, then host_fail, then tail_fail.
    // out: the batch's output words; n_jobs: the batch's opening jobs
    uint32_t resolve(const std::vector<uint32_t>& out, uint32_t n_jobs) const {
        if (verdict) return verdict;
        uint32_t min_bad = ~0u, final_bad = 0;
        if (fold)
            for (uint32_t q = 0; q < nq; q++) { min_bad = std::min(min_bad, out[fold_at + q]); final_bad |= out[fold_at + nq + q]; }
        for (const Deferred& d : deferred) {
            bool bad = false;
            if (d.code == SP1B200_VERDICT_JAGGED_EVALUATION) {
                hf::E4 acc[1];
                sum_partials<1>(out.data() + jag_at, blocks_for(jag_cols), acc);
                bad = neq(acc[0] * jag_bp, jag_expect);
            } else if (d.code == SP1B200_VERDICT_QUERY_VALUE) {
                bad = min_bad == d.job;
            } else if (d.code == SP1B200_VERDICT_QUERY_FINAL_POLY) {
                bad = final_bad != 0;
            } else {   // an opening job: its nq path checks and its tensor commitment
                const size_t j = (size_t)job0 + d.job;
                for (uint32_t q = 0; q < nq; q++) bad |= out[j * nq + q] != 0;
                bad |= out[(size_t)n_jobs * nq + j] != 0;
            }
            if (bad) return d.code;
        }
        return host_fail ? host_fail : tail_fail;
    }
};

// every field word of the proof is a canonical Montgomery word
bool canonical_sumcheck(const layout::Sumcheck& s) {
    for (size_t i = 0; i < s.polys.size(); i++) if (!canonical(s.polys[i], 4 * (size_t)s.n_coeffs[i])) return false;
    return canonical(s.claimed_sum, 4) && canonical(s.point, 4 * s.polys.size()) && canonical(s.eval, 4);
}
bool canonical_proof(const layout::ShardProof& p, const sp1b200_machine* m, uint32_t mlr, uint32_t ls, uint32_t nq) {
    bool ok = canonical(p.commit, 8) && canonical(p.pv, p.n_pv) && canonical(p.out_num, 4 * (size_t)p.n_out) && canonical(p.out_den, 4 * (size_t)p.n_out);
    for (auto& r : p.rounds) ok = ok && canonical(r.nd, 16) && canonical_sumcheck(r.sc);
    ok = ok && canonical(p.gkr_point, 4 * (size_t)mlr) && canonical(p.gkr_witness, 1) && canonical_sumcheck(p.zc);
    for (size_t k = 0; k < m->chips.size(); k++) {
        const size_t mw = m->chips[k].main_w, pw = m->chips[k].prep_w;
        ok = ok && canonical(p.gkr_main[k], 4 * mw) && canonical(p.gkr_prep[k], 4 * pw) && canonical(p.zc_main[k], 4 * mw) && canonical(p.zc_prep[k], 4 * pw);
    }
    ok = ok && canonical(p.univariate, 8 * (size_t)ls) && canonical(p.fri_commits, 8 * (size_t)ls);
    for (auto* v : {&p.component, &p.query})
        for (auto& o : *v) ok = ok && canonical(o.values, (size_t)nq * o.width) && canonical(o.root, 8) && canonical(o.paths, (size_t)nq * o.log_height * 8);
    ok = ok && canonical(p.final_poly, 4) && canonical(p.pow_witness, 1) && canonical(p.batch_witness, 1);
    for (size_t r = 0; r < p.batch_evals.size(); r++) ok = ok && canonical(p.batch_evals[r], 4 * (r < p.component.size() ? p.component[r].width : 0));
    ok = ok && canonical_sumcheck(p.jagged_sc) && canonical_sumcheck(p.jagged_eval);
    return ok && canonical(p.merkle_commits, 8 * p.rc_cc.size()) && canonical(p.expected_eval, 4);
}

// the device phase of a batch: every shard's evaluation section in one buffer, every recorded input in one auxiliary buffer, one
// launch per kernel, one copy back; then each shard's checks in order
sp1b200_err run_device(sp1b200_ctx* ctx, const std::vector<Verifier*>& vs, uint32_t* verdicts, VerifyTimes& t) {
    const uint32_t nq = ctx->params.num_queries;
    std::vector<uint64_t> ev_at(vs.size());
    uint64_t ev_words = 0;
    std::vector<uint32_t> aux;
    auto align = [&](size_t a) { while (aux.size() % a) aux.push_back(0); };
    auto put = [&](const std::vector<uint32_t>& v) { const uint32_t at = (uint32_t)aux.size(); aux.insert(aux.end(), v.begin(), v.end()); return at; };
    std::vector<OpenJob> jobs;
    std::vector<FoldArgs> folds;
    std::vector<JagArgs> jags;
    unsigned jag_blocks = 0;
    for (Verifier* v : vs) if (v->jag) jag_blocks = std::max(jag_blocks, blocks_for(v->jag_cols));
    size_t n_fold = 0, n_jag = 0;
    for (Verifier* v : vs) { n_fold += v->fold; n_jag += v->jag; }
    uint64_t n_jobs = 0;
    for (Verifier* v : vs) if (v->fold) n_jobs += v->jobs.size();
    const size_t fold_base = (size_t)n_jobs * (nq + 1), jag_base = fold_base + 2 * (size_t)nq * n_fold;
    const size_t out_words = jag_base + 4 * (size_t)jag_blocks * n_jag;
    if (out_words >> 32) return sp1b200_set_error("verify: %zu device result words in one batch do not fit 32-bit offsets", out_words);
    for (size_t s = 0; s < vs.size(); s++) {
        Verifier& v = *vs[s];
        if (!v.fold && !v.jag) continue;
        ev_at[s] = ev_words;
        const uint32_t base = (uint32_t)ev_words;
        ev_words += v.ev_words;
        if (v.fold) {
            v.job0 = (uint32_t)jobs.size();
            v.fold_at = (uint32_t)(fold_base + 2 * (size_t)nq * folds.size());
            FoldArgs a = v.fa;
            a.idx_at = put(v.idx);
            for (OpenJob j : v.jobs) {
                j.values_off += base; j.paths_off += base; j.root_off += base; j.commit_off += base; j.idx_off = a.idx_at;
                jobs.push_back(j);
            }
            a.coeff_at = put(v.coeff_words);
            a.beta_at = put(v.beta_words);
            std::vector<uint32_t> fo(v.fold_offs);
            for (auto& o : fo) o += base;
            a.fold_off_at = put(fo);
            for (uint32_t r = 0; r < a.n_comp; r++) a.comp_off[r] += base;
            a.final_off += base;
            a.out_at = v.fold_at;
            folds.push_back(a);
        }
        if (v.jag) {
            v.jag_at = (uint32_t)(jag_base + 4 * (size_t)jag_blocks * jags.size());
            JagArgs j{};
            j.n_cols = v.jag_cols; j.nb = v.jag_nb; j.partial_at = v.jag_at;
            j.col_eq_at = put(v.col_eq);
            j.point_at = put(v.jag_point);
            align(2);
            j.prefix_at = (uint32_t)(aux.size() / 2);
            const size_t at = aux.size();
            aux.resize(at + 2 * v.prefix.size());
            memcpy(&aux[at], v.prefix.data(), v.prefix.size() * 8);
            jags.push_back(j);
        }
    }
    if (ev_words >> 32 || aux.size() >> 31) return sp1b200_set_error("verify: a batch of %zu shards does not fit 32-bit offsets", vs.size());
    std::vector<uint32_t> out(out_words);
    if (out_words) {
        align(4);
        const size_t jobs_at = aux.size();
        aux.resize(jobs_at + jobs.size() * sizeof(OpenJob) / 4);
        memcpy(aux.data() + jobs_at, jobs.data(), jobs.size() * sizeof(OpenJob));
        const size_t folds_at = aux.size();
        aux.resize(folds_at + folds.size() * sizeof(FoldArgs) / 4);
        memcpy(aux.data() + folds_at, folds.data(), folds.size() * sizeof(FoldArgs));
        const size_t jags_at = aux.size();
        aux.resize(jags_at + jags.size() * sizeof(JagArgs) / 4);
        memcpy(aux.data() + jags_at, jags.data(), jags.size() * sizeof(JagArgs));
        DevFree mem(ctx);
        uint32_t *d_ev, *d_aux, *d_out;
        SP1_TRY(mem.alloc((void**)&d_ev, std::max<uint64_t>(ev_words, 1) * 4));
        SP1_TRY(mem.alloc((void**)&d_aux, aux.size() * 4));
        SP1_TRY(mem.alloc((void**)&d_out, out_words * 4));
        for (size_t s = 0; s < vs.size(); s++)
            if (vs[s]->fold || vs[s]->jag)
                SP1_CUDA(cudaMemcpyAsync(d_ev + ev_at[s], vs[s]->ev_base, vs[s]->ev_words * 4, cudaMemcpyHostToDevice, ctx->stream));
        SP1_CUDA(cudaMemcpyAsync(d_aux, aux.data(), aux.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
        SP1_CUDA(cudaMemsetAsync(d_out, 0, out_words * 4, ctx->stream));
        cudaEvent_t ev[4] = {};
        struct Events { cudaEvent_t* e; ~Events() { for (int i = 0; i < 4; i++) if (e[i]) cudaEventDestroy(e[i]); } } guard{ev};
        for (auto& e : ev) SP1_CUDA(cudaEventCreate(&e));
        SP1_CUDA(cudaEventRecord(ev[0], ctx->stream));
        if (!jobs.empty())
            SP1_LAUNCH(ctx, verify_merkle_kernel, blocks_for(n_jobs * (nq + 1), 128), 128, 0, reinterpret_cast<const OpenJob*>(d_aux + jobs_at),
                       (uint32_t)n_jobs, nq, d_ev, d_aux, d_out);
        SP1_CUDA(cudaEventRecord(ev[1], ctx->stream));
        if (!folds.empty())
            SP1_LAUNCH(ctx, verify_fold_kernel, dim3(blocks_for(nq, 128), (unsigned)folds.size()), 128, 0,
                       reinterpret_cast<const FoldArgs*>(d_aux + folds_at), d_ev, d_aux, d_out);
        SP1_CUDA(cudaEventRecord(ev[2], ctx->stream));
        if (!jags.empty())
            SP1_LAUNCH(ctx, verify_jagged_kernel, dim3(jag_blocks, (unsigned)jags.size()), 256, 0, reinterpret_cast<const JagArgs*>(d_aux + jags_at),
                       d_aux, d_out);
        SP1_CUDA(cudaEventRecord(ev[3], ctx->stream));
        SP1_CUDA(cudaMemcpyAsync(out.data(), d_out, out_words * 4, cudaMemcpyDeviceToHost, ctx->stream));
        SP1_CUDA(cudaStreamSynchronize(ctx->stream));
        float ms = 0;
        if (!folds.empty()) {
            t.fold_ran = true;
            if (cudaEventElapsedTime(&ms, ev[0], ev[1]) == cudaSuccess) t.merkle += ms;
            if (cudaEventElapsedTime(&ms, ev[1], ev[2]) == cudaSuccess) t.fold += ms;
        }
        if (!jags.empty()) {
            t.jagged_ran = true;
            if (cudaEventElapsedTime(&ms, ev[2], ev[3]) == cudaSuccess) t.jagged += ms;
        }
    }
    for (size_t s = 0; s < vs.size(); s++) verdicts[s] = vs[s]->resolve(out, (uint32_t)n_jobs);
    return nullptr;
}

}  // namespace

sp1b200_err verify_parse_shard(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint32_t* h_prep_commit8, const uint64_t* h_heights,
                               const char* const* chip_names, const uint32_t* h_proof, uint64_t n_words, const std::string& who_s,
                               VerifyShardIn& out) {
    const char* who = who_s.c_str();
    const sp1b200_params& prm = ctx->params;
    const uint32_t mlr = prm.max_log_row_count, ls = prm.log_stacking_height, nq = prm.num_queries;
    if (mlr > 30 || ls > 30 || prm.log_blowup > 24 || nq == 0 || nq > (1u << 16))
        return sp1b200_set_error("%s: context parameters out of range (max_log_row_count %u, log_stacking_height %u, num_queries %u)", who, mlr, ls, nq);
    const size_t nch = m->chips.size();
    out.mw.resize(nch); out.pw.resize(nch);
    bool has_prep = false;
    for (size_t k = 0; k < nch; k++) {
        out.mw[k] = m->chips[k].main_w; out.pw[k] = m->chips[k].prep_w;
        has_prep |= out.pw[k] != 0;
        if (!chip_names[k]) return sp1b200_set_error("%s: chip %zu has no name", who, k);
        if (h_heights[k] >> (mlr + 1)) return sp1b200_set_error("%s: chip %zu: height %llu does not fit %u bits", who, k, (unsigned long long)h_heights[k], mlr + 1);
    }
    if (!m->interactions || m->host.size() != nch) return sp1b200_set_error("%s: machine is not initialised", who);
    if (has_prep && !h_prep_commit8) return sp1b200_set_error("%s: the machine has preprocessed columns but h_prep_commit8 is NULL", who);
    out.heights = h_heights;
    out.prep_commit8 = h_prep_commit8;
    layout::Shape& shape = out.shape;
    shape.n_chips = nch; shape.main_w = out.mw.data(); shape.prep_w = out.pw.data();
    shape.max_log_row_count = mlr; shape.log_stacking_height = ls; shape.num_queries = nq;
    shape.ncols = layout::round_columns(nch, h_heights, out.mw.data(), out.pw.data(), ls);
    layout::ShardProof& p = out.p;
    if (const char* why = layout::parse_shard_proof(h_proof, n_words, shape, p)) return sp1b200_set_error("%s: %s", who, why);
    // the oracle's reader and BasefoldProof's shape: every opening has the height of its round's tree
    for (size_t r = 0; r < p.component.size(); r++)
        if (p.component[r].log_height != ls + prm.log_blowup) return sp1b200_set_error("%s: evaluation proof: commitment round %zu opening has log_height %u, the layout needs %u", who, r, p.component[r].log_height, ls + prm.log_blowup);
    for (uint32_t r = 0; r < ls; r++)
        if (p.query[r].log_height != ls + prm.log_blowup - r - 1) return sp1b200_set_error("%s: evaluation proof: fold round %u opening has log_height %u, the layout needs %u", who, r, p.query[r].log_height, ls + prm.log_blowup - r - 1);
    if (!canonical_proof(p, m, mlr, ls, nq)) return sp1b200_set_error("%s: a field word of the proof is not canonical (>= p)", who);
    for (size_t k = 0; k < nch; k++)
        for (uint32_t pi : m->host[k].publics)
            if (pi >= p.n_pv) return sp1b200_set_error("%s: chip %zu reads public value %u but the proof carries %u", who, k, pi, p.n_pv);
    // the verifier reads no more GKR outputs or tables per round than a shard of this library can have (the layout reader admits
    // more, for the wire format's sake)
    if (p.n_out > (1u << 20)) return sp1b200_set_error("%s: LogUp-GKR section: %u outputs, more than 2^20", who, p.n_out);
    for (auto& t : p.rc_cc)
        if (t.size() > 4096) return sp1b200_set_error("%s: evaluation proof: %zu tables in a round, more than 4096", who, t.size());
    return nullptr;
}

sp1b200_err verify_shards(sp1b200_ctx* ctx, const sp1b200_machine* m, const char* const* chip_names,
                          const std::vector<const VerifyShardIn*>& shards, const std::vector<const uint32_t*>& starts, uint32_t host_threads,
                          uint32_t* verdicts, uint32_t* finals, VerifyTimes& t) {
    const size_t n = shards.size();
    std::vector<std::unique_ptr<Verifier>> vs;
    std::vector<Verifier*> vp;
    for (const VerifyShardIn* in : shards) {
        vs.emplace_back(new Verifier(ctx->params, m, in->p, in->heights, chip_names, in->shape.ncols, in->prep_commit8));
        vp.push_back(vs.back().get());
    }
    const auto h0 = std::chrono::steady_clock::now();
    const size_t nt = std::min<size_t>(std::max<uint32_t>(host_threads, 1), n);
    if (nt <= 1) {
        for (size_t s = 0; s < n; s++) vs[s]->run(starts[s]);
    } else {   // the host phases share nothing but the read-only machine; each thread takes the next shard
        std::atomic<size_t> next{0};
        std::vector<std::thread> pool;
        for (size_t i = 0; i < nt; i++)
            pool.emplace_back([&] { for (size_t s; (s = next.fetch_add(1)) < n;) vs[s]->run(starts[s]); });
        for (auto& th : pool) th.join();
    }
    t.host_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - h0).count();
    SP1_TRY(run_device(ctx, vp, verdicts, t));
    if (finals)
        for (size_t s = 0; s < n; s++) if (!verdicts[s]) vs[s]->ch.store(finals + 34 * s);
    return nullptr;
}

extern "C" {

const char* sp1b200_verdict_name(uint32_t verdict) {
    if (verdict < std::size(VERDICT_NAMES)) return VERDICT_NAMES[verdict];
    const char* core = verify_core_verdict_name(verdict);
    if (!core) core = verify_compressed_verdict_name(verdict);
    return core ? core : "Unknown";
}

sp1b200_err sp1b200_verify_shard(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint32_t* h_prep_commit8, const uint64_t* h_heights,
                                 const char* const* chip_names, const uint32_t* h_proof, uint64_t n_words, uint32_t* h_chal, uint32_t* h_verdict) {
    SP1_DEVICE_GUARD(ctx);
    if (!ctx || !m || !h_heights || !chip_names || !h_proof || !h_chal || !h_verdict) return sp1b200_set_error("verify_shard: NULL argument");
    const auto t0 = std::chrono::steady_clock::now();
    VerifyShardIn in;
    SP1_TRY(verify_parse_shard(ctx, m, h_prep_commit8, h_heights, chip_names, h_proof, n_words, "verify_shard", in));
    uint32_t verdict = SP1B200_VERDICT_ACCEPT, fin[34];
    VerifyTimes t;
    SP1_TRY(verify_shards(ctx, m, chip_names, {&in}, {h_chal}, 1, &verdict, fin, t));
    float kernel_ms = 0;
    if (t.fold_ran) { ctx->phase_ms["verify.merkle"] = t.merkle; ctx->phase_ms["verify.fold"] = t.fold; kernel_ms += t.merkle + t.fold; }
    if (t.jagged_ran) { ctx->phase_ms["verify.jagged_eval"] = t.jagged; kernel_ms += t.jagged; }
    ctx->phase_ms["verify.kernels"] = kernel_ms;
    ctx->phase_ms["verify.total"] = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *h_verdict = verdict;
    if (!verdict) memcpy(h_chal, fin, sizeof(fin));
    return nullptr;
}

}  // extern "C"
