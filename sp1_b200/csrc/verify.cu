// ShardVerifier::verify_shard (crates/hypercube/src/verifier/shard.rs:437-750) on the flat proof words of sp1b200_prove_shard.
// The transcript, the PoW checks, the GKR / zerocheck / jagged sumcheck rounds, the branching program and every chip's constraints at
// the zerocheck point run on the host (a few thousand extension-field operations).  The work that grows with the number of queries runs
// on the device, in three kernels on the context's stream with memory from its pool:
//   verify_merkle_kernel   every Merkle opening of the proof (all commitment rounds and all FRI fold rounds, every query): leaf hash,
//                          path walk, root comparison; and each opening's tensor commitment compress(root, hash([log_h, width]))
//   verify_fold_kernel     per query: the batched codeword value, the fold chain through the log_stacking_height rounds, final_poly
//   verify_jagged_kernel   sum_c col_eq[c] * eq(prefix_c || prefix_{c+1}, point) over every jagged column
// Their flags and partial sums are copied back once, at the end of the call.  Checks are reported in verify_shard's order: a check
// whose inputs come from the device is recorded when the transcript reaches it and resolved after the copy, so the verdict names
// the first failing check, as the reference's verifier (and the oracle's restatement of it) would.
#include "ctx.cuh"
#include "challenger.cuh"
#include "hostfield.hpp"
#include "machine.cuh"
#include "poseidon2.cuh"
#include "proof_layout.hpp"
#include "sumcheck.cuh"
#include <chrono>
#include <cstring>
#include <vector>

// Poseidon2 sponge / 2-to-1 compression on the host (the transcript's permutation), for the verifier's few table-size hashes
static void host_hash(const uint32_t* in, size_t n, uint32_t* out8) {
    uint32_t s[16] = {0};
    size_t fill = 0;
    for (size_t i = 0; i < n; i++) { s[fill++] = in[i]; if (fill == 8) { host_poseidon2_permute(s); fill = 0; } }
    if (fill) host_poseidon2_permute(s);
    memcpy(out8, s, 32);
}
static void host_compress(const uint32_t* l8, const uint32_t* r8, uint32_t* out8) {
    uint32_t s[16];
    memcpy(s, l8, 32); memcpy(s + 8, r8, 32);
    host_poseidon2_permute(s);
    memcpy(out8, s, 32);
}

namespace {

using hf::E4;
using kb::Ext;

// ---- device part ----------------------------------------------------------------------------------------------------------------

// one opening: `width` values per query at values_off, log_h sibling digests per query at paths_off (word offsets into the evaluation
// section on the device); the leaf index of query q is idx[q] >> shift
struct OpenJob { uint32_t values_off, width, paths_off, root_off, commit_off, log_h, shift, pad; };

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
        uint32_t index = __ldg(idx + q) >> j.shift;
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

// per query q: Σ_c coeff_c · v_c over the component columns of every round, then the fold chain.  out[q] = first round whose opened
// pair does not hold the running value (len if none), out[nq + q] = 1 when the chain ends away from final_poly.
struct FoldArgs {
    uint32_t nq, len, n_comp;
    uint32_t comp_off[2], comp_w[2];
    uint32_t g;        // generator of order 2^(len + log_blowup), Montgomery
    uint32_t log_n;    // len + log_blowup
    uint32_t minus1;
    uint32_t final_off;
};
__global__ void __launch_bounds__(128) verify_fold_kernel(FoldArgs a, const uint32_t* __restrict__ ev, const uint32_t* __restrict__ fold_off,
                                                          const uint32_t* __restrict__ idx, const uint32_t* __restrict__ coeffs,
                                                          const uint32_t* __restrict__ betas, uint32_t* __restrict__ out) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= a.nq) return;
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

// sum_c col_eq[c] * prod_i eq(bit_i, point_i) over the 2 (log_m + 1) bits of prefix[c] || prefix[c+1] (most significant first), one
// column per thread; per-block sums to partial[block]
__global__ void __launch_bounds__(256) verify_jagged_kernel(const uint64_t* __restrict__ prefix, uint32_t n_cols, const uint32_t* __restrict__ col_eq,
                                                            const uint32_t* __restrict__ point, uint32_t nb, uint32_t* __restrict__ partial) {
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

enum : uint32_t {
    V_ACCEPT = 0, V_POW, V_INVALID_SHAPE, V_ZERO_DENOMINATOR, V_CUMULATIVE_SUM, V_INVALID_SHAPE_ROUNDS, V_INCONSISTENT_SUMCHECK_CLAIM,
    V_SC_PROOF_SHAPE, V_SC_CLAIMED_SUM, V_SC_ROUND, V_SC_POINT, V_SC_EVAL, V_INCONSISTENT_EVALUATION, V_LAST_LAYER_DIMENSION,
    V_TRACE_POINT, V_INVALID_SHAPE_OPENINGS, V_NUMERATOR_EVAL, V_DENOMINATOR_EVAL, V_OPENING_SHAPE, V_HEIGHT_BITS, V_HEIGHT_TOO_LARGE,
    V_CONSTRAINTS_EVAL, V_CONSTRAINTS_CLAIMED_SUM, V_INCORRECT_SHAPE, V_INCORRECT_TABLE_SIZES, V_AREA_OUT_OF_BOUNDS, V_DUMMY_TABLES,
    V_SUMCHECK_CLAIM_MISMATCH, V_MONOTONICITY, V_JAGGED_EVALUATION, V_JAGGED_EVAL_PROOF, V_STACKING, V_BATCH_POW, V_FRI_LENGTH,
    V_BASEFOLD_SUMCHECK, V_TWO_ADICITY, V_TCS_COMPONENT, V_QUERY_VALUE, V_TCS_QUERY, V_QUERY_FINAL_POLY, V_SUMCHECK_FINAL_POLY,
    V_PREP_WIDTHS, V_CHIP_TABLES, V_COUNT
};
// every code is the one include/sp1b200.h documents
static_assert(V_ACCEPT == SP1B200_VERDICT_ACCEPT, "verdict code differs from include/sp1b200.h");
static_assert(V_POW == SP1B200_VERDICT_POW, "verdict code differs from include/sp1b200.h");
static_assert(V_INVALID_SHAPE == SP1B200_VERDICT_INVALID_SHAPE, "verdict code differs from include/sp1b200.h");
static_assert(V_ZERO_DENOMINATOR == SP1B200_VERDICT_ZERO_DENOMINATOR, "verdict code differs from include/sp1b200.h");
static_assert(V_CUMULATIVE_SUM == SP1B200_VERDICT_CUMULATIVE_SUM_MISMATCH, "verdict code differs from include/sp1b200.h");
static_assert(V_INVALID_SHAPE_ROUNDS == SP1B200_VERDICT_INVALID_SHAPE_ROUNDS, "verdict code differs from include/sp1b200.h");
static_assert(V_INCONSISTENT_SUMCHECK_CLAIM == SP1B200_VERDICT_INCONSISTENT_SUMCHECK_CLAIM, "verdict code differs from include/sp1b200.h");
static_assert(V_SC_PROOF_SHAPE == SP1B200_VERDICT_SUMCHECK_PROOF_SHAPE, "verdict code differs from include/sp1b200.h");
static_assert(V_SC_CLAIMED_SUM == SP1B200_VERDICT_SUMCHECK_CLAIMED_SUM, "verdict code differs from include/sp1b200.h");
static_assert(V_SC_ROUND == SP1B200_VERDICT_SUMCHECK_ROUND, "verdict code differs from include/sp1b200.h");
static_assert(V_SC_POINT == SP1B200_VERDICT_SUMCHECK_POINT, "verdict code differs from include/sp1b200.h");
static_assert(V_SC_EVAL == SP1B200_VERDICT_SUMCHECK_EVAL, "verdict code differs from include/sp1b200.h");
static_assert(V_INCONSISTENT_EVALUATION == SP1B200_VERDICT_INCONSISTENT_EVALUATION, "verdict code differs from include/sp1b200.h");
static_assert(V_LAST_LAYER_DIMENSION == SP1B200_VERDICT_LAST_LAYER_DIMENSION, "verdict code differs from include/sp1b200.h");
static_assert(V_TRACE_POINT == SP1B200_VERDICT_TRACE_POINT_MISMATCH, "verdict code differs from include/sp1b200.h");
static_assert(V_INVALID_SHAPE_OPENINGS == SP1B200_VERDICT_INVALID_SHAPE_OPENINGS, "verdict code differs from include/sp1b200.h");
static_assert(V_NUMERATOR_EVAL == SP1B200_VERDICT_NUMERATOR_EVALUATION, "verdict code differs from include/sp1b200.h");
static_assert(V_DENOMINATOR_EVAL == SP1B200_VERDICT_DENOMINATOR_EVALUATION, "verdict code differs from include/sp1b200.h");
static_assert(V_OPENING_SHAPE == SP1B200_VERDICT_OPENING_SHAPE, "verdict code differs from include/sp1b200.h");
static_assert(V_HEIGHT_BITS == SP1B200_VERDICT_HEIGHT_BITS, "verdict code differs from include/sp1b200.h");
static_assert(V_HEIGHT_TOO_LARGE == SP1B200_VERDICT_HEIGHT_TOO_LARGE, "verdict code differs from include/sp1b200.h");
static_assert(V_CONSTRAINTS_EVAL == SP1B200_VERDICT_CONSTRAINTS_EVAL, "verdict code differs from include/sp1b200.h");
static_assert(V_CONSTRAINTS_CLAIMED_SUM == SP1B200_VERDICT_CONSTRAINTS_CLAIMED_SUM, "verdict code differs from include/sp1b200.h");
static_assert(V_INCORRECT_SHAPE == SP1B200_VERDICT_INCORRECT_SHAPE, "verdict code differs from include/sp1b200.h");
static_assert(V_INCORRECT_TABLE_SIZES == SP1B200_VERDICT_INCORRECT_TABLE_SIZES, "verdict code differs from include/sp1b200.h");
static_assert(V_AREA_OUT_OF_BOUNDS == SP1B200_VERDICT_AREA_OUT_OF_BOUNDS, "verdict code differs from include/sp1b200.h");
static_assert(V_DUMMY_TABLES == SP1B200_VERDICT_DUMMY_TABLES, "verdict code differs from include/sp1b200.h");
static_assert(V_SUMCHECK_CLAIM_MISMATCH == SP1B200_VERDICT_SUMCHECK_CLAIM_MISMATCH, "verdict code differs from include/sp1b200.h");
static_assert(V_MONOTONICITY == SP1B200_VERDICT_MONOTONICITY, "verdict code differs from include/sp1b200.h");
static_assert(V_JAGGED_EVALUATION == SP1B200_VERDICT_JAGGED_EVALUATION, "verdict code differs from include/sp1b200.h");
static_assert(V_JAGGED_EVAL_PROOF == SP1B200_VERDICT_JAGGED_EVAL_PROOF, "verdict code differs from include/sp1b200.h");
static_assert(V_STACKING == SP1B200_VERDICT_STACKING, "verdict code differs from include/sp1b200.h");
static_assert(V_BATCH_POW == SP1B200_VERDICT_BATCH_POW, "verdict code differs from include/sp1b200.h");
static_assert(V_FRI_LENGTH == SP1B200_VERDICT_FRI_LENGTH, "verdict code differs from include/sp1b200.h");
static_assert(V_BASEFOLD_SUMCHECK == SP1B200_VERDICT_BASEFOLD_SUMCHECK, "verdict code differs from include/sp1b200.h");
static_assert(V_TWO_ADICITY == SP1B200_VERDICT_TWO_ADICITY, "verdict code differs from include/sp1b200.h");
static_assert(V_TCS_COMPONENT == SP1B200_VERDICT_TCS_COMPONENT, "verdict code differs from include/sp1b200.h");
static_assert(V_QUERY_VALUE == SP1B200_VERDICT_QUERY_VALUE, "verdict code differs from include/sp1b200.h");
static_assert(V_TCS_QUERY == SP1B200_VERDICT_TCS_QUERY, "verdict code differs from include/sp1b200.h");
static_assert(V_QUERY_FINAL_POLY == SP1B200_VERDICT_QUERY_FINAL_POLY, "verdict code differs from include/sp1b200.h");
static_assert(V_SUMCHECK_FINAL_POLY == SP1B200_VERDICT_SUMCHECK_FINAL_POLY, "verdict code differs from include/sp1b200.h");
static_assert(V_PREP_WIDTHS == SP1B200_VERDICT_PREPROCESSED_WIDTHS, "verdict code differs from include/sp1b200.h");
static_assert(V_CHIP_TABLES == SP1B200_VERDICT_CHIP_TABLES, "verdict code differs from include/sp1b200.h");
const char* const VERDICT_NAMES[V_COUNT] = {
    "Accepted", "Pow", "InvalidShape", "ZeroDenominator", "CumulativeSumMismatch", "InvalidShape(rounds)", "InconsistentSumcheckClaim",
    "InvalidProofShape", "InconsistencyWithClaimedSum", "SumcheckRoundInconsistency", "InvalidProofShape(point)", "InconsistencyWithEval",
    "InconsistentEvaluation", "InvalidLastLayerDimension", "TracePointMismatch", "InvalidShape(openings)", "NumeratorEvaluationMismatch",
    "DenominatorEvaluationMismatch", "OpeningShape", "InvalidHeightBitDecomposition", "HeightTooLarge",
    "ConstraintsCheckFailed(InconsistencyWithEval)", "ConstraintsCheckFailed(InconsistencyWithClaimedSum)", "IncorrectShape",
    "IncorrectTableSizes", "AreaOutOfBounds", "IncorrectShape(dummy tables)", "SumcheckClaimMismatch", "MonotonicityCheckFailed",
    "JaggedEvaluationFailed", "JaggedEvalProofVerificationFailed", "StackingError", "BatchPow", "SumcheckFriLengthMismatch", "Sumcheck",
    "TwoAdicityOverflow", "TcsError(component)", "QueryValueMismatch", "TcsError(query)", "QueryFinalPolyMismatch",
    "SumcheckFinalPolyMismatch", "InvalidShape(preprocessed widths)", "InvalidShape(chip tables)"};

inline bool neq(const E4& a, const E4& b) { return !(a == b); }
inline E4 ld(const uint32_t* p) { return E4::load(p); }
inline E4 eqf(const E4& a, const E4& b) { return a * b + (E4::one() - a) * (E4::one() - b); }
inline E4 base(uint64_t canonical) { return E4::from_base(hf::to_monty(canonical)); }

std::vector<E4> ext_vec(const uint32_t* p, size_t n) { std::vector<E4> v(n); for (size_t i = 0; i < n; i++) v[i] = ld(p + 4 * i); return v; }
E4 mle_eval(const std::vector<E4>& vals, const std::vector<E4>& point) {
    const std::vector<E4> eq = hf::partial_lagrange(point);
    E4 acc;
    for (size_t i = 0; i < vals.size() && i < eq.size(); i++) acc = acc + eq[i] * vals[i];
    return acc;
}
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
    static int transition(int row_bit, int index_bit, int cur_bit, int next_bit, int state) {   // state = carry + 2 * comparison
        const int carry = state & 1, cmp = state >> 1;
        const int new_cmp = index_bit == next_bit ? cmp : next_bit;
        const int s = row_bit + carry + cur_bit;
        if (index_bit != (s & 1)) return -1;
        return (s >> 1) + 2 * new_cmp;
    }
    E4 eval(const std::vector<E4>& prefix, const std::vector<E4>& next) const {
        E4 res[4]; res[2] = E4::one();
        for (size_t layer = num_vars + 1; layer-- > 0;) {
            const std::vector<E4> eq = hf::partial_lagrange({lsb(z_row, layer), lsb(z_index, layer), lsb(prefix, layer), lsb(next, layer)});
            E4 nres[4];
            for (int st = 0; st < 4; st++) {
                E4 acc[4];
                for (int i = 0; i < 16; i++) {
                    const int o = transition((i >> 3) & 1, (i >> 2) & 1, (i >> 1) & 1, i & 1, st);
                    if (o >= 0) acc[o] = acc[o] + eq[i];
                }
                for (int k = 0; k < 4; k++) nres[st] = nres[st] + acc[k] * res[k];
            }
            for (int k = 0; k < 4; k++) res[k] = nres[k];
        }
        return res[0];
    }
};

// a check whose inputs the device computes, resolved after the final copy
struct Deferred { uint32_t code; std::vector<uint32_t> flag_ranges; };   // flag_ranges: [begin, end) pairs into the flag words

struct Verifier {
    sp1b200_ctx* ctx;
    const sp1b200_machine* m;
    const HostInteractions& H;
    const layout::ShardProof& p;
    const uint64_t* heights;
    const std::vector<size_t>& ncols;
    const uint32_t* ev_base;   // host start of the evaluation section (device offsets are relative to it)
    uint64_t ev_words;
    HostChallenger ch;
    DevFree mem;
    uint32_t mlr, ls, lb, nq;
    // device outputs: merkle flags | fold words (2 nq) | jagged partials; copied back once
    uint32_t* d_out = nullptr;
    size_t n_merkle_flags = 0, fold_at = 0, jag_at = 0, out_words = 0;
    unsigned jag_blocks = 0;
    bool launched = false, fold_launched = false;
    cudaEvent_t ev[5] = {};   // merkle start / end = fold start, fold end, jagged start, jagged end
    // jagged eval: acc * bp == eval is checked after the copy
    E4 jag_bp, jag_expect;
    bool jag_pending = false;

    Verifier(sp1b200_ctx* c, const sp1b200_machine* mm, const layout::ShardProof& pp, const uint64_t* h, const std::vector<size_t>& nc,
             const uint32_t* evb, uint64_t evw)
        : ctx(c), m(mm), H(*static_cast<const HostInteractions*>(mm->interactions)), p(pp), heights(h), ncols(nc), ev_base(evb), ev_words(evw),
          mem(c) {
        mlr = c->params.max_log_row_count; ls = c->params.log_stacking_height; lb = c->params.log_blowup; nq = c->params.num_queries;
    }
    ~Verifier() { for (auto e : ev) if (e) cudaEventDestroy(e); }

    uint32_t off(const uint32_t* ptr) const { return (uint32_t)(ptr - ev_base); }
    void observe_ext(const E4& e) { ch.observe_n(e.c, 4); }
    void observe_var_ext(const uint32_t* w, size_t n) { ch.observe(hf::to_monty(n)); ch.observe_n(w, 4 * n); }
    E4 sample_ext() { E4 e; ch.sample_ext(e.c); return e; }
    std::vector<E4> sample_point(size_t n) { std::vector<E4> v(n); for (auto& x : v) x = sample_ext(); return v; }

    // partially_verify_sumcheck_proof (slop/crates/sumcheck/src/verifier.rs:21-107)
    uint32_t sumcheck(const layout::Sumcheck& s, size_t nvars, size_t degree) {
        const size_t n = s.polys.size();
        if (n != nvars || nvars == 0) return V_SC_PROOF_SHAPE;
        auto eval = [&](size_t i, const E4& x) { E4 r; for (size_t k = s.n_coeffs[i]; k-- > 0;) r = r * x + ld(s.polys[i] + 4 * k); return r; };
        auto sum01 = [&](size_t i) { E4 r = s.n_coeffs[i] ? ld(s.polys[i]) : E4(); for (size_t k = 0; k < s.n_coeffs[i]; k++) r = r + ld(s.polys[i] + 4 * k); return r; };
        if (neq(sum01(0), ld(s.claimed_sum))) return V_SC_CLAIMED_SUM;
        if (s.n_coeffs[0] != degree + 1) return V_SC_PROOF_SHAPE;
        ch.observe_n(s.polys[0], 4 * (size_t)s.n_coeffs[0]);
        std::vector<E4> alphas;   // most recent first
        for (size_t i = 1; i < n; i++) {
            if (s.n_coeffs[i] != degree + 1) return V_SC_PROOF_SHAPE;
            const E4 a = sample_ext();
            alphas.insert(alphas.begin(), a);
            if (neq(eval(i - 1, a), sum01(i))) return V_SC_ROUND;
            ch.observe_n(s.polys[i], 4 * (size_t)s.n_coeffs[i]);
        }
        const E4 a = sample_ext();
        alphas.insert(alphas.begin(), a);
        for (size_t i = 0; i < n; i++) if (neq(alphas[i], ld(s.point + 4 * i))) return V_SC_POINT;
        if (neq(eval(n - 1, a), ld(s.eval))) return V_SC_EVAL;
        return V_ACCEPT;
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
        if (!ch.check_witness(ctx->params.gkr_pow_bits, p.gkr_witness[0])) return V_POW;
        const E4 alpha = sample_ext();
        const std::vector<E4> beta_seed = sample_point(bdim);
        (void)sample_ext();
        const unsigned v = hf::log2_ceil(ni);
        const size_t expected = (size_t)1 << (v + 1);
        if (p.n_out != expected) return V_INVALID_SHAPE;
        observe_var_ext(p.out_num, p.n_out);
        observe_var_ext(p.out_den, p.n_out);
        const std::vector<E4> num = ext_vec(p.out_num, expected), den = ext_vec(p.out_den, expected);
        E4 cum;
        for (size_t i = 0; i < expected; i++) { if (den[i].is_zero()) return V_ZERO_DENOMINATOR; cum = cum + num[i] * hf::inv(den[i]); }
        if (!cum.is_zero()) return V_CUMULATIVE_SUM;
        std::vector<E4> point = sample_point(v + 1);
        E4 num_eval = mle_eval(num, point), den_eval = mle_eval(den, point);
        if (p.rounds.size() + 1 != mlr) return V_INVALID_SHAPE_ROUNDS;
        for (size_t i = 0; i < p.rounds.size(); i++) {
            const layout::GkrRound& r = p.rounds[i];
            const E4 lambda = sample_ext();
            if (neq(ld(r.sc.claimed_sum), num_eval * lambda + den_eval)) return V_INCONSISTENT_SUMCHECK_CLAIM;
            if (uint32_t e = sumcheck(r.sc, i + v + 1, 3)) return e;
            const E4 n0 = ld(r.nd), n1 = ld(r.nd + 4), d0 = ld(r.nd + 8), d1 = ld(r.nd + 12);
            E4 eqv = E4::one();
            for (size_t k = 0; k < point.size(); k++) eqv = eqv * eqf(ld(r.sc.point + 4 * k), point[k]);
            if (neq(ld(r.sc.eval), eqv * ((n0 * d1 + n1 * d0) * lambda + d0 * d1))) return V_INCONSISTENT_EVALUATION;
            ch.observe_n(r.nd, 16);
            point = ext_vec(r.sc.point, r.sc.polys.size());
            const E4 lc = sample_ext();
            point.push_back(lc);
            num_eval = n0 + (n1 - n0) * lc;
            den_eval = d0 + (d1 - d0) * lc;
        }
        const std::vector<E4> ipt(point.begin(), point.begin() + v), tpt(point.begin() + v, point.end());
        if (tpt.size() != mlr) return V_LAST_LAYER_DIMENSION;
        for (uint32_t k = 0; k < mlr; k++) if (neq(tpt[k], ld(p.gkr_point + 4 * k))) return V_TRACE_POINT;
        const std::vector<E4> betas = hf::partial_lagrange(beta_seed);
        std::vector<E4> pe{E4()};
        pe.insert(pe.end(), tpt.begin(), tpt.end());
        std::vector<E4> nv, dv;
        ch.observe(hf::to_monty(nch));
        for (size_t k = 0; k < nch; k++) {
            const ChipProg& c = m->chips[k];
            if (c.prep_w) observe_var_ext(p.gkr_prep[k], c.prep_w);
            observe_var_ext(p.gkr_main[k], c.main_w);
            const E4 geq = full_geq(point_from_usize(heights[k], mlr + 1), pe);
            const std::vector<E4> mo = ext_vec(p.gkr_main[k], c.main_w), po = ext_vec(p.gkr_prep[k], c.prep_w);
            for (const InterDev& in : H.per_chip[k]) {
                auto fraction = [&](const E4* prep, const E4* main, E4& n, E4& d) {
                    d = alpha + betas[0] * hf::to_monty(in.arg_index);
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
        if (neq(num_eval, mle_eval(nv, ipt))) return V_NUMERATOR_EVAL;
        if (neq(den_eval, mle_eval(dv, ipt))) return V_DENOMINATOR_EVAL;
        return V_ACCEPT;
    }

    // the chip's constraints folded with the reversed α powers (the verifier folder's Horner order) at one row of extension values
    E4 eval_air(size_t k, const E4* prep, const E4* main, const std::vector<E4>& powers) const {
        const HostProg& hp = m->host[k];
        std::vector<E4> regs(std::max<uint32_t>(m->chips[k].n_regs, 1));
        for (const DagInstr& in : hp.instrs) {
            switch (in.opcode) {
                case BC_LOAD_LEAF: { const LeafRef& l = hp.leaves[in.a]; regs[in.out] = main ? (l.source == LEAF_MAIN ? main : prep)[l.col] : E4(); break; }
                case BC_LOAD_CONST: regs[in.out] = E4::from_base(hp.consts[in.a]); break;
                case BC_LOAD_PUBLIC: regs[in.out] = E4::from_base(p.pv[hp.publics[in.a]]); break;
                case BC_ADD_F: regs[in.out] = regs[in.a] + regs[in.b]; break;
                case BC_SUB_F: regs[in.out] = regs[in.a] - regs[in.b]; break;
                case BC_MUL_F: regs[in.out] = regs[in.a] * regs[in.b]; break;
                case BC_NEG_F: regs[in.out] = E4() - regs[in.a]; break;
            }
        }
        E4 acc;
        for (size_t i = 0; i < hp.assert_regs.size(); i++) acc = acc + powers[hp.assert_alphas[i]] * regs[hp.assert_regs[i]];
        return acc;
    }

    // ShardVerifier::verify_zerocheck (crates/hypercube/src/verifier/shard.rs:288-434)
    uint32_t zerocheck() {
        const size_t nch = m->chips.size();
        const E4 alpha = sample_ext(), gkr_c = sample_ext(), lambda = sample_ext();
        if (p.zc.polys.size() != mlr) return V_INVALID_SHAPE;
        const std::vector<E4> zp = ext_vec(p.zc.point, mlr);
        E4 eqv = E4::one();
        for (uint32_t i = 0; i < mlr; i++) eqv = eqv * eqf(ld(p.gkr_point + 4 * i), zp[i]);
        std::vector<E4> pt{E4()};
        pt.insert(pt.end(), zp.begin(), zp.end());
        E4 rlc;
        for (size_t k = 0; k < nch; k++) {
            const ChipProg& c = m->chips[k];
            const std::vector<E4> degree = point_from_usize(heights[k], mlr + 1);
            for (size_t i = 1; i < degree.size(); i++) if (!(degree[i] * degree[0]).is_zero()) return V_HEIGHT_TOO_LARGE;
            const E4 geq = full_geq(degree, pt);
            std::vector<E4> rev(c.n_constraints);
            E4 pw = E4::one();
            for (uint32_t i = 0; i < c.n_constraints; i++) { rev[c.n_constraints - 1 - i] = pw; pw = pw * alpha; }
            const std::vector<E4> mo = ext_vec(p.zc_main[k], c.main_w), po = ext_vec(p.zc_prep[k], c.prep_w);
            const E4 pra = eval_air(k, nullptr, nullptr, rev);
            const E4 ce = eval_air(k, po.data(), mo.data(), rev) - pra * geq;
            E4 ob, g = gkr_c;
            for (auto& x : mo) { ob = ob + x * g; g = g * gkr_c; }
            for (auto& x : po) { ob = ob + x * g; g = g * gkr_c; }
            rlc = rlc * lambda + eqv * (ce + ob);
        }
        if (neq(ld(p.zc.eval), rlc)) return V_CONSTRAINTS_EVAL;
        E4 mod;
        for (size_t k = 0; k < nch; k++) {
            E4 s, g = gkr_c;
            for (uint32_t j = 0; j < m->chips[k].main_w; j++) { s = s + ld(p.gkr_main[k] + 4 * j) * g; g = g * gkr_c; }
            for (uint32_t j = 0; j < m->chips[k].prep_w; j++) { s = s + ld(p.gkr_prep[k] + 4 * j) * g; g = g * gkr_c; }
            mod = lambda * mod + s;
        }
        if (neq(ld(p.zc.claimed_sum), mod)) return V_CONSTRAINTS_CLAIMED_SUM;
        if (uint32_t e = sumcheck(p.zc, mlr, 4)) return e;
        ch.observe(hf::to_monty(nch));
        for (size_t k = 0; k < nch; k++) { observe_var_ext(p.zc_prep[k], m->chips[k].prep_w); observe_var_ext(p.zc_main[k], m->chips[k].main_w); }
        return V_ACCEPT;
    }

    sp1b200_err ensure_out() {
        if (d_out) return nullptr;
        n_merkle_flags = (size_t)(ncols.size() + ls) * (nq + 1);
        fold_at = n_merkle_flags;
        jag_at = fold_at + 2 * (size_t)nq;
        out_words = jag_at + 4 * (size_t)jag_blocks;
        SP1_TRY(mem.alloc((void**)&d_out, out_words * 4));
        SP1_CUDA(cudaMemsetAsync(d_out, 0, out_words * 4, ctx->stream));
        for (auto& e : ev) SP1_CUDA(cudaEventCreate(&e));
        return nullptr;
    }

    // JaggedPcsVerifier::verify_trusted_evaluations (slop/crates/jagged/src/verifier.rs:113-384) with the stacked and BaseFold verifiers
    // behind it; commitments = {preprocessed,} main
    sp1b200_err jagged(const std::vector<const uint32_t*>& commitments, uint32_t* verdict) {
        *verdict = V_ACCEPT;
        const size_t nr = commitments.size();
        for (auto& v : p.rc_cc) if (v.empty()) { *verdict = V_INCORRECT_SHAPE; return nullptr; }
        // column heights as (rows, cols) runs; totals in 128 bits so that no count in the words can wrap them
        unsigned __int128 total_cols = 0, total_area = 0;
        for (auto& v : p.rc_cc) for (auto& rc : v) { total_cols += rc.second; total_area += (unsigned __int128)rc.first * rc.second; }
        if (total_cols == 0) { *verdict = V_INCORRECT_SHAPE; return nullptr; }
        const uint64_t area64 = total_area >> 63 ? ~(uint64_t)0 : (uint64_t)total_area;
        if (p.max_log_rows != mlr || p.log_m != hf::log2_ceil(area64) || total_area >> 63) { *verdict = V_INCORRECT_SHAPE; return nullptr; }
        // log_m matches the area, so the columns with rows are few; a column count that is absurd only through empty tables cannot be
        // laid out
        if (total_cols > ((uint64_t)1 << 24)) { *verdict = V_INCORRECT_SHAPE; return nullptr; }
        const size_t n_cols = (size_t)total_cols;
        std::vector<uint64_t> prefix;
        prefix.reserve(n_cols + 1);
        {
            uint64_t s = 0;
            for (auto& v : p.rc_cc) for (auto& rc : v) for (uint32_t c = 0; c < rc.second; c++) { prefix.push_back(s); s += rc.first; }
            prefix.push_back(s);
        }
        const std::vector<E4> z_col = sample_point(hf::log2_ceil(n_cols));
        const uint64_t R = (uint64_t)1 << mlr, S = (uint64_t)1 << ls;
        std::vector<uint64_t> round_area(nr), added_vals(nr), added_cols(nr);
        std::vector<std::vector<E4>> claims(nr);
        for (size_t r = 0; r < nr; r++) {
            const auto& v = p.rc_cc[r];
            if (v.size() < 2) { *verdict = V_INCORRECT_SHAPE; return nullptr; }
            uint64_t expect = 0, area = 0;
            for (size_t t = 0; t + 2 < v.size(); t++) { expect += v[t].second; area += (uint64_t)v[t].first * v[t].second; }
            // the claims of round r are the zerocheck's opened values of that round's columns, in chip order
            size_t have = 0;
            for (size_t k = 0; k < m->chips.size(); k++) have += (nr == 2 && r == 0) ? m->chips[k].prep_w : m->chips[k].main_w;
            if (have != expect) { *verdict = V_INCORRECT_SHAPE; return nullptr; }
            for (size_t k = 0; k < m->chips.size(); k++) {
                const bool prep = nr == 2 && r == 0;
                const uint32_t w = prep ? m->chips[k].prep_w : m->chips[k].main_w;
                const uint32_t* o = prep ? p.zc_prep[k] : p.zc_main[k];
                for (uint32_t j = 0; j < w; j++) claims[r].push_back(ld(o + 4 * j));
            }
            std::vector<uint32_t> meta{hf::to_monty(v.size())};
            for (auto& rc : v) meta.push_back(hf::to_monty(rc.first));
            for (auto& rc : v) meta.push_back(hf::to_monty(rc.second));
            uint32_t h[8], cm[8];
            host_hash(meta.data(), meta.size(), h);
            host_compress(p.merkle_commits + 8 * r, h, cm);
            if (memcmp(cm, commitments[r], 32)) { *verdict = V_INCORRECT_TABLE_SIZES; return nullptr; }
            if (area == 0 || area >= ((uint64_t)1 << 30)) { *verdict = V_AREA_OUT_OF_BOUNDS; return nullptr; }
            const uint64_t next = ((area + S - 1) / S) * S, av = next - area, ac = std::max<uint64_t>((av + R - 1) / R, 1);
            if (v[v.size() - 2].second + 1 != ac || v.back().second != 1 || v[v.size() - 2].first != R || v.back().first != av - (ac - 1) * R) {
                *verdict = V_DUMMY_TABLES; return nullptr;
            }
            for (auto& rc : v) if (rc.first > R) { *verdict = V_INCORRECT_SHAPE; return nullptr; }
            round_area[r] = area; added_vals[r] = av; added_cols[r] = ac;
        }
        if (p.log_m >= 30) { *verdict = V_AREA_OUT_OF_BOUNDS; return nullptr; }
        std::vector<E4> column_claims;
        for (size_t r = 0; r < nr; r++) { column_claims.insert(column_claims.end(), claims[r].begin(), claims[r].end()); column_claims.resize(column_claims.size() + added_cols[r]); }
        if (prefix.size() != column_claims.size() + 1) { *verdict = V_INCORRECT_SHAPE; return nullptr; }
        if (neq(mle_eval(column_claims, z_col), ld(p.jagged_sc.claimed_sum))) { *verdict = V_SUMCHECK_CLAIM_MISMATCH; return nullptr; }
        if ((*verdict = sumcheck(p.jagged_sc, p.log_m, 2))) return nullptr;
        for (size_t c = 0; c + 1 < prefix.size(); c++) if (prefix[c] > prefix[c + 1]) { *verdict = V_MONOTONICITY; return nullptr; }
        // JaggedEvalSumcheckConfig::jagged_evaluation (slop/crates/jagged/src/jagged_eval/sumcheck_eval.rs:45-155)
        const uint32_t lm = p.log_m;
        observe_ext(ld(p.jagged_eval.claimed_sum));
        if ((*verdict = sumcheck(p.jagged_eval, 2 * (lm + 1), 2))) return nullptr;
        {
            const std::vector<E4> jp = ext_vec(p.jagged_eval.point, 2 * (lm + 1));
            const std::vector<E4> first(jp.begin(), jp.begin() + lm + 1), second(jp.begin() + lm + 1, jp.end());
            const std::vector<E4> z_row = ext_vec(p.zc.point, mlr), z_trace = ext_vec(p.jagged_sc.point, p.jagged_sc.polys.size());
            jag_bp = BranchingProgram{z_row, z_trace, std::max(z_row.size(), z_trace.size())}.eval(first, second);
            jag_expect = ld(p.jagged_eval.eval);
            // the column sum on the device: col_eq from the shared eq-table launcher, one thread per column
            jag_blocks = blocks_for(n_cols);
            SP1_TRY(ensure_out());
            const int kz = (int)z_col.size();
            std::vector<uint32_t> hz(4 * (size_t)kz + 8 * (size_t)(lm + 1));
            for (int i = 0; i < kz; i++) z_col[i].store(&hz[4 * i]);
            memcpy(&hz[4 * (size_t)kz], p.jagged_eval.point, 32 * (size_t)(lm + 1));
            uint32_t *d_pts, *d_col_eq; uint64_t* d_prefix;
            SP1_TRY(mem.alloc((void**)&d_pts, hz.size() * 4));
            SP1_TRY(mem.alloc((void**)&d_col_eq, ((size_t)4 << kz) * 4));
            SP1_TRY(mem.alloc((void**)&d_prefix, prefix.size() * 8));
            SP1_CUDA(cudaMemcpyAsync(d_pts, hz.data(), hz.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
            SP1_CUDA(cudaMemcpyAsync(d_prefix, prefix.data(), prefix.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
            SP1_CUDA(cudaEventRecord(ev[3], ctx->stream));
            SP1_TRY(launch_eq_table(ctx, d_pts, kz, d_col_eq));
            SP1_LAUNCH(ctx, verify_jagged_kernel, jag_blocks, 256, 0, d_prefix, (uint32_t)n_cols, d_col_eq, d_pts + 4 * kz, lm + 1, d_out + jag_at);
            SP1_CUDA(cudaEventRecord(ev[4], ctx->stream));
            jag_pending = true;
            launched = true;
        }
        const E4 jagged_eval = ld(p.jagged_eval.claimed_sum);
        // (the check acc == eval of the jagged-eval sumcheck is resolved with the device flags; nothing below reads acc)
        deferred.push_back(Deferred{V_JAGGED_EVALUATION, {}});
        if (neq(ld(p.expected_eval) * jagged_eval, ld(p.jagged_sc.eval))) { host_fail = V_JAGGED_EVAL_PROOF; return nullptr; }
        std::vector<uint64_t> total(nr);
        for (size_t r = 0; r < nr; r++) total[r] = round_area[r] + added_vals[r];
        observe_ext(ld(p.expected_eval));
        return stacked(total);
    }

    // StackedPcsVerifier::verify_trusted_evaluation (slop/crates/stacked/src/verifier.rs:39-99)
    sp1b200_err stacked(const std::vector<uint64_t>& areas) {
        const size_t npt = p.jagged_sc.polys.size();
        if (npt < ls) { host_fail = V_INCORRECT_SHAPE; return nullptr; }
        const std::vector<E4> pt = ext_vec(p.jagged_sc.point, npt);
        const std::vector<E4> batch_point(pt.begin(), pt.end() - ls), stack_point(pt.end() - ls, pt.end());
        std::vector<E4> flat;
        for (size_t r = 0; r < areas.size(); r++) {
            if (areas[r] % ((uint64_t)1 << ls) || (areas[r] >> ls) != ncols[r]) { host_fail = V_INCORRECT_SHAPE; return nullptr; }
            const std::vector<E4> e = ext_vec(p.batch_evals[r], ncols[r]);
            flat.insert(flat.end(), e.begin(), e.end());
        }
        if (neq(ld(p.expected_eval), mle_eval(flat, batch_point))) { host_fail = V_STACKING; return nullptr; }
        for (size_t r = 0; r < areas.size(); r++) ch.observe_n(p.batch_evals[r], 4 * ncols[r]);
        return basefold(stack_point, flat);
    }

    // BasefoldVerifier::verify_mle_evaluations (slop/crates/basefold/src/verifier.rs:122-420)
    sp1b200_err basefold(const std::vector<E4>& point, const std::vector<E4>& claims) {
        if (!ch.check_witness(ctx->params.batch_pow_bits, p.batch_witness[0])) { host_fail = V_BATCH_POW; return nullptr; }
        const std::vector<E4> coeffs = hf::partial_lagrange(sample_point(hf::log2_ceil(claims.size())));
        E4 claim;
        for (size_t k = 0; k < claims.size(); k++) claim = claim + claims[k] * coeffs[k];
        const size_t len = ls;
        if (point.size() != len || len == 0) { host_fail = V_FRI_LENGTH; return nullptr; }
        ch.observe(hf::to_monty(len));
        std::vector<E4> betas;
        for (size_t i = 0; i < len; i++) {
            ch.observe_n(p.univariate + 8 * i, 8);
            ch.observe_n(p.fri_commits + 8 * i, 8);
            betas.push_back(sample_ext());
        }
        E4 expected = claim;
        for (size_t i = 0; i < len; i++) {
            const E4 p0 = ld(p.univariate + 8 * i), p1 = ld(p.univariate + 8 * i + 4), x = point[len - 1 - i];
            if (neq(expected, (E4::one() - x) * p0 + x * p1)) { host_fail = V_BASEFOLD_SUMCHECK; return nullptr; }
            expected = p0 + betas[i] * p1;
        }
        ch.observe_n(p.final_poly, 4);
        if (!ch.check_witness(ctx->params.pow_bits, p.pow_witness[0])) { host_fail = V_POW; return nullptr; }
        const uint32_t log_n = (uint32_t)len + lb;
        if (log_n > 24) { host_fail = V_TWO_ADICITY; return nullptr; }
        std::vector<uint32_t> idx(nq);
        for (auto& q : idx) q = ch.sample_bits(log_n);
        // device: every opening, and the fold chain of every query
        SP1_TRY(ensure_out());
        const size_t ncomp = ncols.size();
        std::vector<OpenJob> jobs;
        for (size_t r = 0; r < ncomp; r++) {
            const layout::Opening& o = p.component[r];
            jobs.push_back(OpenJob{off(o.values), o.width, off(o.paths), off(o.root), 0, o.log_height, 0, 0});
        }
        for (size_t r = 0; r < len; r++) {
            const layout::Opening& o = p.query[r];
            jobs.push_back(OpenJob{off(o.values), o.width, off(o.paths), off(o.root), off(p.fri_commits + 8 * r), o.log_height, (uint32_t)r + 1, 0});
        }
        // component openings are checked against the jagged round's original commitments; the device reads them from the evaluation section
        for (size_t r = 0; r < ncomp; r++) jobs[r].commit_off = off(p.merkle_commits + 8 * r);
        std::vector<uint32_t> aux;   // idx | coeffs | betas | fold offsets, then the jobs
        aux.insert(aux.end(), idx.begin(), idx.end());
        const size_t coeff_at = aux.size();
        for (size_t k = 0; k < claims.size(); k++) for (int i = 0; i < 4; i++) aux.push_back(coeffs[k].c[i]);
        const size_t beta_at = aux.size();
        for (auto& b : betas) for (int i = 0; i < 4; i++) aux.push_back(b.c[i]);
        const size_t fold_off_at = aux.size();
        for (size_t r = 0; r < len; r++) aux.push_back(off(p.query[r].values));
        while (aux.size() % 4) aux.push_back(0);
        const size_t jobs_at = aux.size();
        aux.resize(aux.size() + jobs.size() * sizeof(OpenJob) / 4);
        memcpy(&aux[jobs_at], jobs.data(), jobs.size() * sizeof(OpenJob));
        uint32_t *d_ev, *d_aux;
        SP1_TRY(mem.alloc((void**)&d_ev, ev_words * 4));
        SP1_TRY(mem.alloc((void**)&d_aux, aux.size() * 4));
        SP1_CUDA(cudaMemcpyAsync(d_ev, ev_base, ev_words * 4, cudaMemcpyHostToDevice, ctx->stream));
        SP1_CUDA(cudaMemcpyAsync(d_aux, aux.data(), aux.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
        const uint32_t n_jobs = (uint32_t)jobs.size();
        SP1_CUDA(cudaEventRecord(ev[0], ctx->stream));
        SP1_LAUNCH(ctx, verify_merkle_kernel, blocks_for((uint64_t)n_jobs * (nq + 1), 128), 128, 0, reinterpret_cast<const OpenJob*>(d_aux + jobs_at),
                   n_jobs, nq, d_ev, d_aux, d_out);
        SP1_CUDA(cudaEventRecord(ev[1], ctx->stream));
        FoldArgs a{};
        a.nq = nq; a.len = (uint32_t)len; a.n_comp = (uint32_t)ncomp;
        for (size_t r = 0; r < ncomp; r++) { a.comp_off[r] = off(p.component[r].values); a.comp_w[r] = p.component[r].width; }
        a.log_n = log_n;
        a.g = hf::pow(hf::to_monty(3), (uint64_t)127 << (24 - log_n));
        a.minus1 = hf::pow(hf::to_monty(3), (uint64_t)127 << 23);
        a.final_off = off(p.final_poly);
        SP1_LAUNCH(ctx, verify_fold_kernel, blocks_for(nq, 128), 128, 0, a, d_ev, d_aux + fold_off_at, d_aux, d_aux + coeff_at, d_aux + beta_at,
                   d_out + fold_at);
        SP1_CUDA(cudaEventRecord(ev[2], ctx->stream));
        launched = fold_launched = true;
        // the device checks in verify_mle_evaluations' order: component openings round by round, then per fold round the opened value
        // and that round's openings, then final_poly
        for (size_t r = 0; r < ncomp; r++) deferred.push_back(Deferred{V_TCS_COMPONENT, {(uint32_t)(r * nq), (uint32_t)((r + 1) * nq),
                                                                                          (uint32_t)(n_jobs * nq + r), (uint32_t)(n_jobs * nq + r + 1)}});
        for (size_t r = 0; r < len; r++) {
            deferred.push_back(Deferred{V_QUERY_VALUE, {(uint32_t)r}});
            const size_t j = ncomp + r;
            deferred.push_back(Deferred{V_TCS_QUERY, {(uint32_t)(j * nq), (uint32_t)((j + 1) * nq), (uint32_t)(n_jobs * nq + j), (uint32_t)(n_jobs * nq + j + 1)}});
        }
        deferred.push_back(Deferred{V_QUERY_FINAL_POLY, {}});
        const E4 f = ld(p.final_poly);
        if (neq(f, ld(p.univariate + 8 * (len - 1)) + betas.back() * ld(p.univariate + 8 * (len - 1) + 4))) host_fail = V_SUMCHECK_FINAL_POLY;
        return nullptr;
    }

    std::vector<Deferred> deferred;
    uint32_t host_fail = V_ACCEPT;

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
            if (v.size() != want.size() + 2) return V_CHIP_TABLES;
            for (size_t t = 0; t < want.size(); t++)
                if (v[t].first != want[t].first || v[t].second != want[t].second) return V_CHIP_TABLES;
        }
        return V_ACCEPT;
    }

    // one copy of every device result, then the checks in order; host_fail (if set) comes after every deferred check
    sp1b200_err resolve(uint32_t* verdict, float* kernel_ms) {
        *kernel_ms = 0;
        std::vector<uint32_t> out(out_words);
        if (launched) {
            SP1_CUDA(cudaMemcpyAsync(out.data(), d_out, out_words * 4, cudaMemcpyDeviceToHost, ctx->stream));
            SP1_CUDA(cudaStreamSynchronize(ctx->stream));
            float ms = 0;
            if (fold_launched && cudaEventElapsedTime(&ms, ev[0], ev[1]) == cudaSuccess) { ctx->phase_ms["verify.merkle"] = ms; *kernel_ms += ms; }
            if (fold_launched && cudaEventElapsedTime(&ms, ev[1], ev[2]) == cudaSuccess) { ctx->phase_ms["verify.fold"] = ms; *kernel_ms += ms; }
            if (jag_pending && cudaEventElapsedTime(&ms, ev[3], ev[4]) == cudaSuccess) { ctx->phase_ms["verify.jagged_eval"] = ms; *kernel_ms += ms; }
        }
        uint32_t min_bad = ~0u, final_bad = 0;
        if (fold_launched)
            for (uint32_t q = 0; q < nq; q++) { min_bad = std::min(min_bad, out[fold_at + q]); final_bad |= out[fold_at + nq + q]; }
        for (const Deferred& d : deferred) {
            bool bad = false;
            if (d.code == V_JAGGED_EVALUATION) {
                hf::E4 acc[1];
                sum_partials<1>(out.data() + jag_at, jag_blocks, acc);
                bad = neq(acc[0] * jag_bp, jag_expect);
            } else if (d.code == V_QUERY_VALUE) {
                bad = min_bad == d.flag_ranges[0];
            } else if (d.code == V_QUERY_FINAL_POLY) {
                bad = final_bad != 0;
            } else {
                for (size_t i = 0; i < d.flag_ranges.size(); i += 2)
                    for (uint32_t t = d.flag_ranges[i]; t < d.flag_ranges[i + 1]; t++) bad |= out[t] != 0;
            }
            if (bad) { *verdict = d.code; return nullptr; }
        }
        *verdict = host_fail;
        return nullptr;
    }
};

// every field word of the proof is a canonical Montgomery word
bool canonical(const uint32_t* w, size_t n) { for (size_t i = 0; i < n; i++) if (w[i] >= hf::P) return false; return true; }
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

}  // namespace

extern "C" {

const char* sp1b200_verdict_name(uint32_t verdict) { return verdict < V_COUNT ? VERDICT_NAMES[verdict] : "Unknown"; }

sp1b200_err sp1b200_verify_shard(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint32_t* h_prep_commit8, const uint64_t* h_heights,
                                 const char* const* chip_names, const uint32_t* h_proof, uint64_t n_words, uint32_t* h_chal, uint32_t* h_verdict) {
    SP1_DEVICE_GUARD(ctx);
    if (!ctx || !m || !h_heights || !chip_names || !h_proof || !h_chal || !h_verdict) return sp1b200_set_error("verify_shard: NULL argument");
    const auto t0 = std::chrono::steady_clock::now();
    const sp1b200_params& prm = ctx->params;
    const uint32_t mlr = prm.max_log_row_count, ls = prm.log_stacking_height, nq = prm.num_queries;
    if (mlr > 30 || ls > 30 || prm.log_blowup > 24 || nq == 0 || nq > (1u << 16))
        return sp1b200_set_error("verify_shard: context parameters out of range (max_log_row_count %u, log_stacking_height %u, num_queries %u)", mlr, ls, nq);
    const size_t nch = m->chips.size();
    std::vector<uint32_t> mw(nch), pw(nch);
    bool has_prep = false;
    for (size_t k = 0; k < nch; k++) {
        mw[k] = m->chips[k].main_w; pw[k] = m->chips[k].prep_w;
        has_prep |= pw[k] != 0;
        if (!chip_names[k]) return sp1b200_set_error("verify_shard: chip %zu has no name", k);
        if (h_heights[k] >> (mlr + 1)) return sp1b200_set_error("verify_shard: chip %zu: height %llu does not fit %u bits", k, (unsigned long long)h_heights[k], mlr + 1);
    }
    if (!m->interactions || m->host.size() != nch) return sp1b200_set_error("verify_shard: machine is not initialised");
    if (has_prep && !h_prep_commit8) return sp1b200_set_error("verify_shard: the machine has preprocessed columns but h_prep_commit8 is NULL");
    layout::Shape shape;
    shape.n_chips = nch; shape.main_w = mw.data(); shape.prep_w = pw.data();
    shape.max_log_row_count = mlr; shape.log_stacking_height = ls; shape.num_queries = nq;
    shape.ncols = layout::round_columns(nch, h_heights, mw.data(), pw.data(), ls);
    layout::ShardProof p;
    if (const char* why = layout::parse_shard_proof(h_proof, n_words, shape, p)) return sp1b200_set_error("verify_shard: %s", why);
    // the oracle's reader and BasefoldProof's shape: every opening has the height of its round's tree
    for (size_t r = 0; r < p.component.size(); r++)
        if (p.component[r].log_height != ls + prm.log_blowup) return sp1b200_set_error("verify_shard: evaluation proof: commitment round %zu opening has log_height %u, the layout needs %u", r, p.component[r].log_height, ls + prm.log_blowup);
    for (uint32_t r = 0; r < ls; r++)
        if (p.query[r].log_height != ls + prm.log_blowup - r - 1) return sp1b200_set_error("verify_shard: evaluation proof: fold round %u opening has log_height %u, the layout needs %u", r, p.query[r].log_height, ls + prm.log_blowup - r - 1);
    if (!canonical_proof(p, m, mlr, ls, nq)) return sp1b200_set_error("verify_shard: a field word of the proof is not canonical (>= p)");
    for (size_t k = 0; k < nch; k++)
        for (uint32_t pi : m->host[k].publics)
            if (pi >= p.n_pv) return sp1b200_set_error("verify_shard: chip %zu reads public value %u but the proof carries %u", k, pi, p.n_pv);
    // the verifier reads no more GKR outputs or tables per round than a shard of this library can have (the layout reader admits
    // more, for the wire format's sake)
    if (p.n_out > (1u << 20)) return sp1b200_set_error("verify_shard: LogUp-GKR section: %u outputs, more than 2^20", p.n_out);
    for (auto& t : p.rc_cc)
        if (t.size() > 4096) return sp1b200_set_error("verify_shard: evaluation proof: %zu tables in a round, more than 4096", t.size());
    const uint32_t* ev_base = p.univariate;
    const uint64_t ev_words = (uint64_t)(p.pv - ev_base);
    Verifier v(ctx, m, p, h_heights, shape.ncols, ev_base, ev_words);
    v.ch.load(h_chal);
    // the shard's own words enter the transcript: public values, main commitment, chip shapes (shard.rs:437-470)
    v.ch.observe_n(p.pv, p.n_pv);
    v.ch.observe_n(p.commit, 8);
    v.ch.observe(hf::to_monty(nch));
    uint32_t verdict = V_ACCEPT;
    if (nch && mlr + 1 >= 30) verdict = V_INVALID_SHAPE;   // a degree point of 30 or more bits (shard.rs:477)
    for (size_t k = 0; k < nch && !verdict; k++) {
        v.ch.observe(hf::to_monty(h_heights[k]));
        const size_t len = strlen(chip_names[k]);
        v.ch.observe(hf::to_monty(len));
        for (size_t i = 0; i < len; i++) v.ch.observe(hf::to_monty((uint8_t)chip_names[k][i]));
    }
    // the preprocessed round's leading column counts are the preprocessed widths (shard.rs:506-523)
    if (!verdict && has_prep) {
        size_t t = 0;
        for (size_t k = 0; k < nch && !verdict; k++) {
            if (!pw[k]) continue;
            if (t >= p.rc_cc[0].size() || p.rc_cc[0][t].second != pw[k]) verdict = V_PREP_WIDTHS;
            t++;
        }
    }
    if (!verdict) verdict = v.gkr();
    if (!verdict) verdict = v.zerocheck();
    if (!verdict) {
        std::vector<const uint32_t*> commits;
        if (has_prep) commits.push_back(h_prep_commit8);
        commits.push_back(p.commit);
        SP1_TRY(v.jagged(commits, &verdict));
    }
    float kernel_ms = 0;
    if (!verdict) SP1_TRY(v.resolve(&verdict, &kernel_ms));
    else SP1_CUDA(cudaStreamSynchronize(ctx->stream));
    if (!verdict) verdict = v.chip_tables();
    ctx->phase_ms["verify.kernels"] = kernel_ms;
    ctx->phase_ms["verify.total"] = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *h_verdict = verdict;
    if (!verdict) v.ch.store(h_chal);
    return nullptr;
}

}  // extern "C"
