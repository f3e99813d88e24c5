// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header: primitives pinned to the reference's own CUDA kernels, protocol glue unpinned).
// C entry points for tests/ (ctypes), __graft_entry__.smoke() and bench.py's cpu_baseline leg.
// All field elements cross this boundary as u32 Montgomery words (the reference's in-memory form).
#include "gkr.hpp"
#include <cstdio>
#include <cstdlib>
#include <chrono>
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

static inline const F* asF(const uint32_t* p) { return reinterpret_cast<const F*>(p); }
static inline F* asF(uint32_t* p) { return reinterpret_cast<F*>(p); }

static void put(std::vector<uint32_t>& o, F x) { o.push_back(x.v); }
static void put(std::vector<uint32_t>& o, const EF& x) { for (int i = 0; i < 4; i++) o.push_back(x.c[i].v); }
static void put(std::vector<uint32_t>& o, const Digest& d) { for (int i = 0; i < 8; i++) o.push_back(d.d[i].v); }
static void put(std::vector<uint32_t>& o, const OpeningAndProof& op) {
    for (F v : op.values) put(o, v);
    put(o, op.proof.merkle_root);
    o.push_back(op.proof.log_tensor_height);
    o.push_back((uint32_t)op.proof.width);
    for (auto& d : op.proof.paths) put(o, d);
}
// flat word order = field order of slop_basefold::BasefoldProof (slop/crates/basefold/src/verifier.rs:97-116)
static void put(std::vector<uint32_t>& o, const BasefoldProof& p) {
    for (auto& m : p.univariate_messages) { put(o, m[0]); put(o, m[1]); }
    for (auto& d : p.fri_commitments) put(o, d);
    for (auto& c : p.component) put(o, c);
    for (auto& c : p.query_phase) put(o, c);
    put(o, p.final_poly);
    put(o, p.pow_witness);
    put(o, p.batch_grinding_witness);
}
static void put(std::vector<uint32_t>& o, const StackedProof& p) {
    put(o, p.basefold);
    for (auto& r : p.batch_evaluations) for (auto& e : r) put(o, e);
}

static void put(std::vector<uint32_t>& o, const PartialSumcheckProof& p) {
    o.push_back((uint32_t)p.polys.size());
    for (auto& u : p.polys) { o.push_back((uint32_t)u.c.size()); for (auto& c : u.c) put(o, c); }
    put(o, p.claimed_sum);
    for (auto& x : p.point) put(o, x);
    put(o, p.eval);
}
// flat word order = field order of slop_jagged::JaggedPcsProof (slop/crates/jagged/src/verifier.rs:17-27)
static void put(std::vector<uint32_t>& o, const JaggedProof& p) {
    put(o, p.pcs);
    put(o, p.sumcheck);
    put(o, p.jagged_eval);
    for (auto& v : p.rc_cc) { o.push_back((uint32_t)v.size()); for (auto& rc : v) { o.push_back((uint32_t)rc.first); o.push_back((uint32_t)rc.second); } }
    for (auto& d : p.merkle_commits) put(o, d);
    put(o, p.expected_eval);
    o.push_back(p.max_log_rows);
    o.push_back(p.log_m);
}

static void chal_load(Challenger& c, const uint32_t* s) {
    for (int i = 0; i < 16; i++) c.sponge[i].v = s[i];
    for (int i = 0; i < 8; i++) c.inbuf[i].v = s[16 + i];
    for (int i = 0; i < 8; i++) c.outbuf[i].v = s[24 + i];
    c.nin = (int)s[32]; c.nout = (int)s[33];
}
static void chal_store(const Challenger& c, uint32_t* s) {
    for (int i = 0; i < 16; i++) s[i] = c.sponge[i].v;
    for (int i = 0; i < 8; i++) s[16 + i] = c.inbuf[i].v;
    for (int i = 0; i < 8; i++) s[24 + i] = c.outbuf[i].v;
    s[32] = (uint32_t)c.nin; s[33] = (uint32_t)c.nout;
}

static int g_skip_verify = 0;
static double g_times[4] = {0, 0, 0, 0};  // seconds: claims, commit (all rounds, last round separately), prove
static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

extern "C" {

// bench.py cpu_baseline support: skip the (restated) verifier and report the phase times of the last jagged run
void orc_set_skip_verify(int v) { g_skip_verify = v; }
// tests only: make every grind return its (skip+1)-th smallest valid witness; the witnesses found are logged in grind order
void orc_set_grind_skip(uint32_t skip) { Challenger::grind_skip() = skip; Challenger::witness_log().clear(); }
uint32_t orc_witness_log(uint32_t* out, uint32_t cap) {
    auto& l = Challenger::witness_log();
    for (uint32_t i = 0; i < l.size() && i < cap; i++) out[i] = l[i];
    return (uint32_t)l.size();
}
void orc_last_times(double* out4) { for (int i = 0; i < 4; i++) out4[i] = g_times[i]; }
static double g_shard_times[5] = {0, 0, 0, 0, 0};  // seconds of the last orc_prove_shard_verify: prep commit, main commit, LogUp-GKR, zerocheck, jagged/BaseFold open
void orc_shard_times(double* out5) { for (int i = 0; i < 5; i++) out5[i] = g_shard_times[i]; }

int orc_num_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
// launchers such as torchrun export OMP_NUM_THREADS=1: the CPU baseline arm asks for the host's cores explicitly
void orc_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

// ---- field -------------------------------------------------------------------------------------
uint32_t orc_to_monty(uint32_t canonical) { return F::from_canonical(canonical).v; }
uint32_t orc_from_monty(uint32_t m) { return F::raw(m).canonical(); }
uint32_t orc_mul(uint32_t a, uint32_t b) { return (F::raw(a) * F::raw(b)).v; }
uint32_t orc_add(uint32_t a, uint32_t b) { return (F::raw(a) + F::raw(b)).v; }
uint32_t orc_sub(uint32_t a, uint32_t b) { return (F::raw(a) - F::raw(b)).v; }
uint32_t orc_inv(uint32_t a) { return F::raw(a).inv().v; }
uint32_t orc_two_adic_generator(uint32_t k) { return two_adic_generator(k).v; }
void orc_ext_mul(const uint32_t* a, const uint32_t* b, uint32_t* out) {
    EF r = EF::from_base_slice(asF(a)) * EF::from_base_slice(asF(b));
    for (int i = 0; i < 4; i++) out[i] = r.c[i].v;
}
void orc_ext_inv(const uint32_t* a, uint32_t* out) {
    EF r = EF::from_base_slice(asF(a)).inv();
    for (int i = 0; i < 4; i++) out[i] = r.c[i].v;
}

// primitives exported so that tests can pin them to the reference's CUDA kernels (oracle/_ref): eq table, batching, folds
void orc_partial_lagrange(const uint32_t* point, uint64_t n_vars, uint32_t* out) {
    std::vector<EF> p(n_vars);
    for (uint64_t i = 0; i < n_vars; i++) p[i] = EF::from_base_slice(asF(point + 4 * i));
    std::vector<EF> eq = partial_lagrange(p);
    for (size_t i = 0; i < eq.size(); i++) for (int k = 0; k < 4; k++) out[4 * i + k] = eq[i].c[k].v;
}
// out[row] = sum_c coeff[c] * mat[c][row]   (the BaseFold batching of columns, basefold-prover/src/prover.rs:140-170)
void orc_batch_columns(const uint32_t* mat, uint64_t width, uint64_t height, const uint32_t* coeffs, uint32_t* out) {
    for (uint64_t r = 0; r < height; r++) {
        EF acc;
        for (uint64_t c = 0; c < width; c++) acc += EF::from_base_slice(asF(coeffs + 4 * c)) * F::raw(mat[c * height + r]);
        for (int k = 0; k < 4; k++) out[4 * r + k] = acc.c[k].v;
    }
}
// out[i] = in[2i] + beta * in[2i+1]   (multilinear/src/fold.rs:12-26)  and  out[i] = in[2i] + alpha (in[2i+1] - in[2i])
void orc_fold_ext(const uint32_t* in, uint64_t m, const uint32_t* beta, int fix_last, uint32_t* out) {
    EF b = EF::from_base_slice(asF(beta));
    for (uint64_t i = 0; i < m; i++) {
        EF e = EF::from_base_slice(asF(in + 8 * i)), o = EF::from_base_slice(asF(in + 8 * i + 4));
        EF r = fix_last ? e + b * (o - e) : e + b * o;
        for (int k = 0; k < 4; k++) out[4 * i + k] = r.c[k].v;
    }
}

// ---- poseidon2 ---------------------------------------------------------------------------------
void orc_poseidon2_permute(uint32_t* state16) { poseidon2_permute(asF(state16)); }
void orc_hash(const uint32_t* in, uint64_t n, uint32_t* out8) {
    Digest d = p2_hash(asF(in), n);
    for (int i = 0; i < 8; i++) out8[i] = d.d[i].v;
}
void orc_compress(const uint32_t* l, const uint32_t* r, uint32_t* out8) {
    Digest a, b;
    for (int i = 0; i < 8; i++) { a.d[i].v = l[i]; b.d[i].v = r[i]; }
    Digest d = p2_compress(a, b);
    for (int i = 0; i < 8; i++) out8[i] = d.d[i].v;
}

// ---- challenger (state = 34 words: sponge[16] input[8] output[8] n_in n_out) --------------------
void orc_challenger_init(uint32_t* st) { Challenger c; chal_store(c, st); }
void orc_challenger_observe(uint32_t* st, const uint32_t* vals, uint64_t n) {
    Challenger c; chal_load(c, st); c.observe_slice(asF(vals), n); chal_store(c, st);
}
void orc_challenger_sample(uint32_t* st, uint32_t* out, uint64_t n) {
    Challenger c; chal_load(c, st); for (uint64_t i = 0; i < n; i++) out[i] = c.sample().v; chal_store(c, st);
}
uint32_t orc_challenger_sample_bits(uint32_t* st, uint32_t bits) {
    Challenger c; chal_load(c, st); uint32_t r = c.sample_bits(bits); chal_store(c, st); return r;
}
uint32_t orc_challenger_grind(uint32_t* st, uint32_t bits) {
    Challenger c; chal_load(c, st); F w = c.grind(bits); chal_store(c, st); return w.v;
}
int orc_challenger_check_witness(uint32_t* st, uint32_t bits, uint32_t w) {
    Challenger c; chal_load(c, st); bool ok = c.check_witness(bits, F::raw(w)); chal_store(c, st); return ok;
}

// ---- RS encode / Merkle ------------------------------------------------------------------------
void orc_rs_encode(const uint32_t* msg, uint64_t ncols, uint32_t log_h, uint32_t log_blowup, uint32_t* out) {
    rs_encode_columns(asF(msg), ncols, log_h, log_blowup, asF(out));
}
void orc_dft_naive(const uint32_t* msg, uint64_t msg_len, uint32_t log_n, uint32_t* out) {
    dft_bitrev_naive(asF(msg), msg_len, asF(out), log_n);
}
// layers_out (optional): all digests bottom-up, layer k at offset sum_{j<k} 2^(log_h-j) digests
void orc_merkle_commit(const uint32_t* mat_colmajor, uint64_t width, uint32_t log_h, uint32_t* layers_out,
                       uint32_t* root8, uint32_t* commit8) {
    MerkleTree t = merkle_commit_columns(asF(mat_colmajor), width, log_h);
    for (int i = 0; i < 8; i++) { root8[i] = t.root.d[i].v; commit8[i] = t.commitment.d[i].v; }
    if (layers_out) {
        size_t off = 0;
        for (auto& L : t.layers) for (auto& d : L) { for (int i = 0; i < 8; i++) layers_out[off + i] = d.d[i].v; off += 8; }
    }
}

// ---- stacked PCS + BaseFold: commit rounds, prove at a point, verify with the restated verifier -----
// dense[r]: column-major [ncols[r] x 2^log_h] for each of n_rounds rounds.  point: (n_extra + log_h) EF
// elements as 4 words each (only the last log_h are used by BaseFold).  challenger_state: in/out.
// proof_out: flat words (see put(BasefoldProof)); returns number of words, or -1 if the restated verifier
// rejects the oracle's own proof.  commits_out: n_rounds x 8 words.
int64_t orc_stacked_prove_verify(const uint32_t* const* dense, const uint64_t* ncols, uint32_t n_rounds, uint32_t log_h,
                                 const uint32_t* point, uint32_t point_len, uint32_t log_blowup, uint32_t num_queries,
                                 uint32_t pow_bits, uint32_t batch_pow_bits, const uint32_t* replay_witnesses,
                                 uint32_t* challenger_state, uint32_t* commits_out, uint32_t* proof_out,
                                 uint64_t proof_cap) {
    FriParams fp; fp.log_blowup = log_blowup; fp.num_queries = num_queries; fp.pow_bits = pow_bits; fp.batch_pow_bits = batch_pow_bits;
    std::vector<std::shared_ptr<StackedRound>> rounds;
    std::vector<Digest> commits;
    std::vector<size_t> areas;
    for (uint32_t r = 0; r < n_rounds; r++) {
        rounds.push_back(stacked_commit(asF(dense[r]), ncols[r], log_h, fp));
        commits.push_back(rounds.back()->tree.commitment);
        areas.push_back(ncols[r] << log_h);
        for (int i = 0; i < 8; i++) commits_out[r * 8 + i] = commits.back().d[i].v;
    }
    std::vector<EF> pt(point_len);
    for (uint32_t i = 0; i < point_len; i++) pt[i] = EF::from_base_slice(asF(point + 4 * i));
    Challenger ch; chal_load(ch, challenger_state);
    Challenger vch = ch;
    F rw[2];
    if (replay_witnesses) { rw[0] = F::raw(replay_witnesses[0]); rw[1] = F::raw(replay_witnesses[1]); }
    StackedProof sp = stacked_prove(pt, rounds, ch, fp, replay_witnesses ? rw : nullptr);
    chal_store(ch, challenger_state);
    // evaluation claim of the stacked polynomial at the full point
    std::vector<EF> flat;
    for (auto& r : sp.batch_evaluations) flat.insert(flat.end(), r.begin(), r.end());
    std::vector<EF> batch_point(pt.begin(), pt.end() - log_h);
    EF claim = mle_eval(flat.data(), flat.size(), batch_point);
    const char* err = stacked_verify(commits, areas, pt, sp, claim, vch, log_h, fp);
    if (err) { std::fprintf(stderr, "oracle verifier rejected oracle proof: %s\n", err); return -1; }
    std::vector<uint32_t> o;
    put(o, sp);
    if (proof_out) { if (o.size() > proof_cap) return -2; std::copy(o.begin(), o.end(), proof_out); }
    return (int64_t)o.size();
}


// ---- jagged PCS: commit rounds of tables, prove evaluations at z_row, verify with the restated verifier -----------
// Round r has n_tables[r] tables; table t of round r: rows[k], cols[k] (k running over all rounds), data at
// dense[r] + offset (column-major [cols x rows] per table, tables with rows == 0 contribute nothing).
// z_row: max_log_rows ext elements.  The per-column evaluation claims at z_row (what zerocheck would hand over)
// are computed here and returned in claims_out (sum over rounds of sum cols, ext each).
// Returns proof words or a negative value on failure; commits_out: n_rounds x 8 (the jagged commitments).
int64_t orc_jagged_prove_verify(const uint32_t* const* dense, uint32_t n_rounds, const uint32_t* n_tables, const uint64_t* rows,
                                const uint64_t* cols, uint32_t log_stack, uint32_t max_log_rows, const uint32_t* z_row_words,
                                uint32_t log_blowup, uint32_t num_queries, uint32_t pow_bits, uint32_t batch_pow_bits,
                                const uint32_t* replay_witnesses, uint32_t* challenger_state, uint32_t* commits_out,
                                uint32_t* claims_out, uint32_t* proof_out, uint64_t proof_cap) {
    FriParams fp; fp.log_blowup = log_blowup; fp.num_queries = num_queries; fp.pow_bits = pow_bits; fp.batch_pow_bits = batch_pow_bits;
    std::vector<EF> z_row(max_log_rows);
    for (uint32_t i = 0; i < max_log_rows; i++) z_row[i] = EF::from_base_slice(asF(z_row_words + 4 * i));
    std::vector<EF> row_eq = partial_lagrange(z_row);
    std::vector<JaggedRound> rounds;
    std::vector<std::vector<EF>> claims;
    std::vector<Digest> commits;
    size_t k = 0, co = 0;
    for (uint32_t r = 0; r < n_rounds; r++) {
        std::vector<Table> tabs;
        const F* p = asF(dense[r]);
        std::vector<EF> cl;
        for (uint32_t t = 0; t < n_tables[r]; t++, k++) {
            Table tb; tb.rows = rows[k]; tb.cols = cols[k]; tb.data = p;
            for (size_t c = 0; c < tb.cols; c++) {
                EF acc;
                for (size_t i = 0; i < tb.rows; i++) acc += row_eq[i] * p[c * tb.rows + i];
                cl.push_back(acc);
            }
            p += tb.rows * tb.cols;
            tabs.push_back(tb);
        }
        double tc0 = now_s();
        rounds.push_back(jagged_commit(tabs, log_stack, max_log_rows, fp));
        g_times[2] = now_s() - tc0;               // commit time of the last (main) round
        g_times[1] = (r == 0 ? 0.0 : g_times[1]) + g_times[2];
        commits.push_back(rounds.back().commit);
        for (int i = 0; i < 8; i++) commits_out[r * 8 + i] = commits.back().d[i].v;
        for (auto& e : cl) for (int i = 0; i < 4; i++) claims_out[co++] = e.c[i].v;
        claims.push_back(cl);
    }
    Challenger ch; chal_load(ch, challenger_state);
    Challenger vch = ch;
    F rw[2];
    if (replay_witnesses) { rw[0] = F::raw(replay_witnesses[0]); rw[1] = F::raw(replay_witnesses[1]); }
    double tp0 = now_s();
    JaggedProof pf = jagged_prove(z_row, claims, rounds, max_log_rows, ch, fp, replay_witnesses ? rw : nullptr);
    g_times[3] = now_s() - tp0;
    chal_store(ch, challenger_state);
    const char* err = g_skip_verify ? nullptr : jagged_verify(commits, z_row, claims, pf, vch, log_stack, max_log_rows, fp);
    if (err) { std::fprintf(stderr, "oracle jagged verifier rejected oracle proof: %s\n", err); return -1; }
    std::vector<uint32_t> o;
    put(o, pf);
    if (proof_out) { if (o.size() > proof_cap) return -2; std::copy(o.begin(), o.end(), proof_out); }
    return (int64_t)o.size();
}

// tests only: z_col (4 words each, written when it fits in cap entries) and the Hadamard sumcheck claim of this thread's last jagged prove.
// Returns the length of z_col.
uint32_t orc_jagged_last_inputs(uint32_t* z_col_out, uint32_t cap, uint32_t* claim4) {
    const JaggedProveInputs& in = jagged_last_inputs();
    if (in.z_col.size() <= cap)
        for (size_t i = 0; i < in.z_col.size(); i++) for (int k = 0; k < 4; k++) z_col_out[4 * i + k] = in.z_col[i].c[k].v;
    for (int k = 0; k < 4; k++) claim4[k] = in.claim.c[k].v;
    return (uint32_t)in.z_col.size();
}

// tests only: the challenger (34 words each) just before the evaluation sumcheck of this thread's last jagged prove observes its claimed
// sum, and just after the sumcheck's last sample
void orc_jagged_eval_states(uint32_t* before34, uint32_t* after34) {
    const JaggedProveInputs& in = jagged_last_inputs();
    chal_store(in.eval_before, before34);
    chal_store(in.eval_after, after34);
}


}  // extern "C"

// ---- machine blob: the AIR bytecode of every chip as u32 words (layout documented in include/sp1b200.h) ------------
// [n_chips] then per chip: main_w prep_w n_constraints n_regs n_instrs n_leaves n_consts n_publics n_asserts,
// instrs (2 words each = the 8-byte DagInstr), leaves (2 words each = LeafRef), consts, publics, assert_regs, assert_alphas
struct MachineChip { AirProgram air; uint32_t main_w, prep_w; };
static std::vector<MachineChip> parse_machine(const uint32_t* b, const uint32_t** end_out = nullptr) {
    uint32_t n = *b++;
    std::vector<MachineChip> out(n);
    for (auto& c : out) {
        c.main_w = *b++; c.prep_w = *b++; c.air.n_constraints = *b++; c.air.n_regs = *b++;
        uint32_t ni = *b++, nl = *b++, nc = *b++, np = *b++, na = *b++;
        for (uint32_t i = 0; i < ni; i++, b += 2) { DagInstr d; std::memcpy(&d, b, 8); c.air.instrs.push_back(d); }
        for (uint32_t i = 0; i < nl; i++, b += 2) { LeafRef l; std::memcpy(&l, b, 8); c.air.leaves.push_back(l); }
        for (uint32_t i = 0; i < nc; i++) c.air.consts.push_back(F::raw(*b++));
        for (uint32_t i = 0; i < np; i++) c.air.publics.push_back(*b++);
        for (uint32_t i = 0; i < na; i++) c.air.assert_regs.push_back((uint16_t)*b++);
        for (uint32_t i = 0; i < na; i++) c.air.assert_alphas.push_back(*b++);
    }
    if (end_out) *end_out = b;
    return out;
}

// interactions section (follows the AIR records): per chip [n_interactions] then per interaction
//   is_send arg_index n_values, multiplicity vcol, value vcols;  vcol = n_terms constant(Montgomery) {source col weight(Montgomery)}*
static const uint32_t* parse_vcol(const uint32_t* b, VCol& v) {
    uint32_t nt = *b++; v.constant = F::raw(*b++);
    for (uint32_t i = 0; i < nt; i++) { VTerm t; t.source = (uint8_t)b[0]; t.col = b[1]; t.weight = F::raw(b[2]); b += 3; v.terms.push_back(t); }
    return b;
}
static std::vector<std::vector<Interaction>> parse_interactions(const uint32_t* b, size_t n_chips) {
    std::vector<std::vector<Interaction>> out(n_chips);
    for (auto& chip : out) {
        uint32_t n = *b++;
        for (uint32_t i = 0; i < n; i++) {
            Interaction in; in.is_send = *b++ != 0; in.arg_index = *b++; uint32_t nv = *b++;
            b = parse_vcol(b, in.mult);
            for (uint32_t k = 0; k < nv; k++) { VCol v; b = parse_vcol(b, v); in.values.push_back(v); }
            chip.push_back(in);
        }
    }
    return out;
}

extern "C" {

// ---- zerocheck stand-alone: sample (alpha, gamma) as prove_shard_with_data does, prove, verify with the restated
// ShardVerifier::verify_zerocheck.  heights[k]; main[k]/prep[k]: column-major [w x height]; gkr_point: max_log_rows ext.
// openings_out: per chip main evals then prep evals AT gkr_point (what LogUp-GKR would hand over).
// out words: sumcheck proof | per chip {prep evals, main evals} at the zerocheck point.
int64_t orc_zerocheck_prove_verify(const uint32_t* machine_blob, const uint64_t* heights, const uint32_t* const* main, const uint32_t* const* prep,
                                   const uint32_t* pv_words, uint32_t n_pv, uint32_t max_log_rows, const uint32_t* gkr_point_words,
                                   uint32_t* challenger_state, uint32_t* openings_out, uint32_t* out, uint64_t cap) {
    std::vector<MachineChip> mc = parse_machine(machine_blob);
    std::vector<F> pv(n_pv);
    for (uint32_t i = 0; i < n_pv; i++) pv[i] = F::raw(pv_words[i]);
    std::vector<EF> gp(max_log_rows);
    for (uint32_t i = 0; i < max_log_rows; i++) gp[i] = EF::from_base_slice(asF(gkr_point_words + 4 * i));
    std::vector<EF> eq = partial_lagrange(gp);
    std::vector<ZcChip> chips(mc.size());
    std::vector<std::vector<EF>> om(mc.size()), op(mc.size());
    size_t oo = 0;
    for (size_t k = 0; k < mc.size(); k++) {
        ZcChip& c = chips[k];
        c.air = &mc[k].air; c.height = heights[k]; c.main_w = mc[k].main_w; c.prep_w = mc[k].prep_w;
        c.main = asF(main[k]); c.prep = c.prep_w ? asF(prep[k]) : nullptr;
        for (size_t j = 0; j < c.main_w; j++) { EF a; for (size_t r = 0; r < c.height; r++) a += eq[r] * c.main[j * c.height + r]; om[k].push_back(a); }
        for (size_t j = 0; j < c.prep_w; j++) { EF a; for (size_t r = 0; r < c.height; r++) a += eq[r] * c.prep[j * c.height + r]; op[k].push_back(a); }
        for (auto& e : om[k]) for (int i = 0; i < 4; i++) openings_out[oo++] = e.c[i].v;
        for (auto& e : op[k]) for (int i = 0; i < 4; i++) openings_out[oo++] = e.c[i].v;
    }
    Challenger ch; chal_load(ch, challenger_state);
    Challenger vch = ch;
    EF alpha = ch.sample_ext(), gamma = ch.sample_ext();
    std::vector<EF> claims(mc.size());
    for (size_t k = 0; k < mc.size(); k++) {
        EF g = gamma, a;
        for (auto& e : om[k]) { a += e * g; g *= gamma; }
        for (auto& e : op[k]) { a += e * g; g *= gamma; }
        claims[k] = a;
    }
    ZerocheckResult r = zerocheck_prove(chips, alpha, gamma, gp, claims, pv, max_log_rows, ch);
    chal_store(ch, challenger_state);
    const char* err = g_skip_verify ? nullptr : zerocheck_verify(chips, r.opened, gp, om, op, r.proof, pv, max_log_rows, vch);
    if (err) { std::fprintf(stderr, "oracle zerocheck verifier rejected oracle proof: %s\n", err); return -1; }
    std::vector<uint32_t> o;
    put(o, r.proof);
    for (auto& c : r.opened) { for (auto& e : c.prep) put(o, e); for (auto& e : c.main) put(o, e); }
    if (out) { if (o.size() > cap) return -2; std::copy(o.begin(), o.end(), out); }
    return (int64_t)o.size();
}

// tests only: the inputs of this thread's last zerocheck prove as words: alpha | gamma | lambda | claimed sum | n | challenges[n] in round
// order (ext = 4 words).  The words are written when they fit in cap; returns their number.
uint64_t orc_zerocheck_last_inputs(uint32_t* out, uint64_t cap) {
    const ZerocheckProveInputs& in = zerocheck_last_inputs();
    std::vector<uint32_t> o;
    put(o, in.alpha); put(o, in.gamma); put(o, in.lambda); put(o, in.claimed_sum);
    o.push_back((uint32_t)in.challenges.size());
    for (auto& e : in.challenges) put(o, e);
    if (out && o.size() <= cap) std::copy(o.begin(), o.end(), out);
    return o.size();
}


static void put(std::vector<uint32_t>& o, const GkrProof& p) {
    o.push_back((uint32_t)p.out_num.size());
    for (auto& e : p.out_num) put(o, e);
    for (auto& e : p.out_den) put(o, e);
    o.push_back((uint32_t)p.rounds.size());
    for (auto& r : p.rounds) { put(o, r.n0); put(o, r.n1); put(o, r.d0); put(o, r.d1); put(o, r.sc); }
    for (auto& e : p.point) put(o, e);
    for (size_t k = 0; k < p.main_open.size(); k++) { for (auto& e : p.main_open[k]) put(o, e); for (auto& e : p.prep_open[k]) put(o, e); }
    put(o, p.witness);
}

// ---- primitives exported so that tests can pin them to the reference's own CUDA kernels (oracle/_ref) ----------------------------------
// First-layer LogUp fractions of ONE chip (execution.rs:13-36; reference kernel: populateLastCircuitLayer / interactionValue,
// sys/lib/logup_gkr/tracegen.cu:20-75): out_num[k * height + r] = multiplicity (negated for receives), out_den[(k * height + r) * 4 ..] =
// alpha + betas[0] * arg_index + sum_j betas[j + 1] * value_j, for interaction k and row r.
int64_t orc_interaction_values(const uint32_t* machine_blob, uint32_t chip, const uint32_t* main, const uint32_t* prep, uint64_t height,
                               const uint32_t* alpha4, const uint32_t* betas, uint32_t n_betas, uint32_t* out_num, uint32_t* out_den) {
    const uint32_t* rest;
    std::vector<MachineChip> mc = parse_machine(machine_blob, &rest);
    auto inter = parse_interactions(rest, mc.size());
    if (chip >= mc.size()) return -1;
    const EF alpha = EF::from_base_slice(asF(alpha4));
    std::vector<EF> bs(n_betas);
    for (uint32_t i = 0; i < n_betas; i++) bs[i] = EF::from_base_slice(asF(betas + 4 * i));
    const auto& I = inter[chip];
    std::vector<F> mr(mc[chip].main_w), pr(mc[chip].prep_w);
    for (uint64_t r = 0; r < height; r++) {
        for (size_t j = 0; j < mr.size(); j++) mr[j] = F::raw(main[j * height + r]);
        for (size_t j = 0; j < pr.size(); j++) pr[j] = F::raw(prep[j * height + r]);
        for (size_t k = 0; k < I.size(); k++) {
            if (I[k].values.size() + 1 > bs.size()) return -2;
            auto [m, d] = interaction_vals<F>(I[k], pr.data(), mr.data(), alpha, bs);
            out_num[k * height + r] = m.v;
            for (int l = 0; l < 4; l++) out_den[(k * height + r) * 4 + l] = d.c[l].v;
        }
    }
    return (int64_t)I.size();
}

// Zerocheck round-0 node sums of ONE chip's constraint program (sum_as_poly.rs:225-286; reference kernel: zerocheck_fused_sequential,
// sys/lib/zerocheck/sequential.cu:110-190): out[t] = sum_i E[i] * sum_k powers[alpha_idx_k] * reg_k evaluated on the row pair
// (2i, 2i+1) interpolated at the nodes {0, 2, 4} - no opening-batching term, no geq / padded-row correction, lambda = 1.
int64_t orc_zerocheck_node_sums(const uint32_t* machine_blob, uint32_t chip, const uint32_t* main, const uint32_t* prep, uint64_t height,
                                const uint32_t* pv_words, uint32_t n_pv, const uint32_t* alpha_pows, const uint32_t* E, uint32_t* out12) {
    std::vector<MachineChip> mc = parse_machine(machine_blob);
    if (chip >= mc.size() || (height & 1)) return -1;
    const AirProgram& air = mc[chip].air;
    const size_t mw = mc[chip].main_w, pw = mc[chip].prep_w;
    std::vector<F> pv(n_pv);
    for (uint32_t i = 0; i < n_pv; i++) pv[i] = F::raw(pv_words[i]);
    std::vector<EF> pw_(air.n_constraints ? air.n_constraints : 1);
    for (size_t i = 0; i < air.n_constraints; i++) pw_[i] = EF::from_base_slice(asF(alpha_pows + 4 * i));
    EF y[3];
    std::vector<F> m0(mw), m2(mw), m4(mw), p0(pw), p2(pw), p4(pw), regs;
    for (uint64_t i = 0; i < height / 2; i++) {
        for (size_t c = 0; c < mw; c++) {
            F a = F::raw(main[c * height + 2 * i]), b = F::raw(main[c * height + 2 * i + 1]);
            F sl = b - a, sl2 = sl + sl;
            m0[c] = a; m2[c] = sl2 + a; m4[c] = sl2 + sl2 + a;
        }
        for (size_t c = 0; c < pw; c++) {
            F a = F::raw(prep[c * height + 2 * i]), b = F::raw(prep[c * height + 2 * i + 1]);
            F sl = b - a, sl2 = sl + sl;
            p0[c] = a; p2[c] = sl2 + a; p4[c] = sl2 + sl2 + a;
        }
        const EF e = EF::from_base_slice(asF(E + 4 * i));
        y[0] += eval_air<F>(air, p0.data(), m0.data(), pv.data(), pw_.data(), regs) * e;
        y[1] += eval_air<F>(air, p2.data(), m2.data(), pv.data(), pw_.data(), regs) * e;
        y[2] += eval_air<F>(air, p4.data(), m4.data(), pv.data(), pw_.data(), regs) * e;
    }
    for (int t = 0; t < 3; t++) for (int l = 0; l < 4; l++) out12[4 * t + l] = y[t].c[l].v;
    return 0;
}

// ---- LogUp-GKR stand-alone: prove + restated verify_logup_gkr.  Words out: n_out | numerator[n_out] | denominator[n_out] |
// n_rounds | per round {numerator_0 numerator_1 denominator_0 denominator_1 sumcheck} | point | per chip {main openings, prep openings} | witness
int64_t orc_gkr_prove_verify(const uint32_t* machine_blob, const uint64_t* heights, const uint32_t* const* main, const uint32_t* const* prep,
                             uint32_t max_log_rows, uint32_t gkr_pow_bits, const uint32_t* replay_witness, uint32_t* challenger_state,
                             uint32_t* out, uint64_t cap) {
    const uint32_t* rest;
    std::vector<MachineChip> mc = parse_machine(machine_blob, &rest);
    auto inter = parse_interactions(rest, mc.size());
    std::vector<GkrChip> chips(mc.size());
    for (size_t k = 0; k < mc.size(); k++) {
        chips[k].height = heights[k]; chips[k].main_w = mc[k].main_w; chips[k].prep_w = mc[k].prep_w;
        chips[k].main = asF(main[k]); chips[k].prep = mc[k].prep_w ? asF(prep[k]) : nullptr; chips[k].inter = inter[k];
    }
    Challenger ch; chal_load(ch, challenger_state);
    Challenger vch = ch;
    F rw; if (replay_witness) rw = F::raw(*replay_witness);
    GkrProof pf = gkr_prove(chips, max_log_rows, gkr_pow_bits, ch, replay_witness ? &rw : nullptr);
    chal_store(ch, challenger_state);
    const char* err = g_skip_verify ? nullptr : gkr_verify(chips, max_log_rows, gkr_pow_bits, pf, vch);
    if (err) { std::fprintf(stderr, "oracle gkr verifier rejected oracle proof: %s\n", err); return -1; }
    std::vector<uint32_t> o;
    put(o, pf);
    if (out) { if (o.size() > cap) return -2; std::copy(o.begin(), o.end(), out); }
    return (int64_t)o.size();
}

// tests only: the inputs of this thread's last LogUp-GKR prove that the proof does not carry, as words: alpha | n_beta | beta_seed[n_beta] |
// n_layers | per layer in proof order {lambda | claim = num_eval * lambda + den_eval | n_point | point[n_point]} (ext = 4 words).  The
// words are written when they fit in cap; returns their number.
uint64_t orc_gkr_last_inputs(uint32_t* out, uint64_t cap) {
    const GkrProveInputs& in = gkr_last_inputs();
    std::vector<uint32_t> o;
    put(o, in.alpha);
    o.push_back((uint32_t)in.beta_seed.size());
    for (auto& e : in.beta_seed) put(o, e);
    o.push_back((uint32_t)in.layers.size());
    for (auto& l : in.layers) {
        put(o, l.lambda); put(o, l.claim);
        o.push_back((uint32_t)l.point.size());
        for (auto& e : l.point) put(o, e);
    }
    if (out && o.size() <= cap) std::copy(o.begin(), o.end(), out);
    return o.size();
}


// ---- whole shard: ShardProver::prove_shard_with_data (crates/hypercube/src/prover/shard.rs:650-792) + the restated
// ShardVerifier::verify_shard (crates/hypercube/src/verifier/shard.rs:437-750; machine-shape / cluster checks that depend on the
// Rust machine definition are out of scope).  prep_dense: preprocessed tables of the chips with prep_w > 0 back to back
// (column-major each); main_dense: main tables of all chips.  names: chip names separated by '\0'.
// Words out: [5][len_0..len_4] | main commitment | gkr | zerocheck (+ opened values) | evaluation proof | public values.
int64_t orc_prove_shard_verify(const uint32_t* machine_blob, const uint64_t* heights, const uint32_t* prep_dense, const uint32_t* main_dense,
                               const char* names, const uint32_t* pv_words, uint32_t n_pv, uint32_t log_stack, uint32_t max_log_rows,
                               uint32_t log_blowup, uint32_t num_queries, uint32_t pow_bits, uint32_t batch_pow_bits, uint32_t gkr_pow_bits,
                               uint32_t* challenger_state, uint32_t* prep_commit_out, uint32_t* out, uint64_t cap) {
    FriParams fp; fp.log_blowup = log_blowup; fp.num_queries = num_queries; fp.pow_bits = pow_bits; fp.batch_pow_bits = batch_pow_bits;
    const uint32_t* rest;
    std::vector<MachineChip> mc = parse_machine(machine_blob, &rest);
    auto inter = parse_interactions(rest, mc.size());
    const size_t n = mc.size();
    std::vector<std::string> nm;
    { const char* p = names; for (size_t k = 0; k < n; k++) { nm.emplace_back(p); p += nm.back().size() + 1; } }
    std::vector<F> pv(n_pv);
    for (uint32_t i = 0; i < n_pv; i++) pv[i] = F::raw(pv_words[i]);
    // tables
    std::vector<Table> ptabs, mtabs;
    std::vector<GkrChip> gchips(n);
    std::vector<ZcChip> zchips(n);
    const F* pp = asF(prep_dense); const F* mp = asF(main_dense);
    for (size_t k = 0; k < n; k++) {
        Table t; t.rows = heights[k]; t.cols = mc[k].main_w; t.data = mp; mtabs.push_back(t);
        gchips[k].height = heights[k]; gchips[k].main_w = mc[k].main_w; gchips[k].prep_w = mc[k].prep_w; gchips[k].main = mp; gchips[k].inter = inter[k];
        zchips[k].air = &mc[k].air; zchips[k].height = heights[k]; zchips[k].main_w = mc[k].main_w; zchips[k].prep_w = mc[k].prep_w; zchips[k].main = mp;
        mp += heights[k] * mc[k].main_w;
        if (mc[k].prep_w) {
            Table p; p.rows = heights[k]; p.cols = mc[k].prep_w; p.data = pp; ptabs.push_back(p);
            gchips[k].prep = pp; zchips[k].prep = pp;
            pp += heights[k] * mc[k].prep_w;
        }
    }
    const bool has_prep = !ptabs.empty();
    // setup: preprocessed commit (AirProver::setup, shard.rs:406-429)
    JaggedRound prep_round;
    double t0 = now_s();
    if (has_prep) { prep_round = jagged_commit(ptabs, log_stack, max_log_rows, fp); for (int i = 0; i < 8; i++) prep_commit_out[i] = prep_round.commit.d[i].v; }
    g_shard_times[0] = now_s() - t0; t0 = now_s();
    Challenger ch; chal_load(ch, challenger_state);
    Challenger vch = ch;
    // ---- prove
    ch.observe_slice(pv.data(), pv.size());
    JaggedRound main_round = jagged_commit(mtabs, log_stack, max_log_rows, fp);
    g_shard_times[1] = now_s() - t0; t0 = now_s();
    ch.observe(main_round.commit);
    ch.observe(F::from_canonical(n));
    for (size_t k = 0; k < n; k++) {
        ch.observe(F::from_canonical(heights[k])); ch.observe(F::from_canonical(nm[k].size()));
        for (unsigned char b : nm[k]) ch.observe(F::from_canonical(b));
    }
    GkrProof gp = gkr_prove(gchips, max_log_rows, gkr_pow_bits, ch);
    g_shard_times[2] = now_s() - t0; t0 = now_s();
    EF alpha = ch.sample_ext(), gamma = ch.sample_ext();
    std::vector<EF> claims(n);
    for (size_t k = 0; k < n; k++) {
        EF g = gamma, a;
        for (auto& e : gp.main_open[k]) { a += e * g; g *= gamma; }
        for (auto& e : gp.prep_open[k]) { a += e * g; g *= gamma; }
        claims[k] = a;
    }
    ZerocheckResult zr = zerocheck_prove(zchips, alpha, gamma, gp.point, claims, pv, max_log_rows, ch);
    g_shard_times[3] = now_s() - t0; t0 = now_s();
    std::vector<JaggedRound> rounds;
    std::vector<std::vector<EF>> jclaims;
    if (has_prep) { rounds.push_back(prep_round); std::vector<EF> c; for (auto& o : zr.opened) c.insert(c.end(), o.prep.begin(), o.prep.end()); jclaims.push_back(c); }
    { rounds.push_back(main_round); std::vector<EF> c; for (auto& o : zr.opened) c.insert(c.end(), o.main.begin(), o.main.end()); jclaims.push_back(c); }
    JaggedProof jp = jagged_prove(zr.proof.point, jclaims, rounds, max_log_rows, ch, fp);
    g_shard_times[4] = now_s() - t0;
    chal_store(ch, challenger_state);
    // ---- verify (verify_shard order)
    if (!g_skip_verify) {
        vch.observe_slice(pv.data(), pv.size());
        vch.observe(main_round.commit);
        vch.observe(F::from_canonical(n));
        for (size_t k = 0; k < n; k++) {
            vch.observe(F::from_canonical(heights[k])); vch.observe(F::from_canonical(nm[k].size()));
            for (unsigned char b : nm[k]) vch.observe(F::from_canonical(b));
        }
        const char* err = gkr_verify(gchips, max_log_rows, gkr_pow_bits, gp, vch);
        if (!err) err = zerocheck_verify(zchips, zr.opened, gp.point, gp.main_open, gp.prep_open, zr.proof, pv, max_log_rows, vch);
        if (!err) {
            std::vector<Digest> commits;
            if (has_prep) commits.push_back(prep_round.commit);
            commits.push_back(main_round.commit);
            err = jagged_verify(commits, zr.proof.point, jclaims, jp, vch, log_stack, max_log_rows, fp);
        }
        if (err) { std::fprintf(stderr, "oracle shard verifier rejected oracle proof: %s\n", err); return -1; }
    }
    std::vector<uint32_t> s0, s1, s2, s3;
    put(s0, main_round.commit);
    put(s1, gp);
    put(s2, zr.proof);
    for (auto& c : zr.opened) { for (auto& e : c.prep) put(s2, e); for (auto& e : c.main) put(s2, e); }
    put(s3, jp);
    std::vector<uint32_t> o{5, (uint32_t)s0.size(), (uint32_t)s1.size(), (uint32_t)s2.size(), (uint32_t)s3.size(), n_pv};
    o.insert(o.end(), s0.begin(), s0.end()); o.insert(o.end(), s1.begin(), s1.end()); o.insert(o.end(), s2.begin(), s2.end());
    o.insert(o.end(), s3.begin(), s3.end()); o.insert(o.end(), pv_words, pv_words + n_pv);
    if (out) { if (o.size() > cap) return -2; std::copy(o.begin(), o.end(), out); }
    return (int64_t)o.size();
}


// ---- verify-only: the restated ShardVerifier::verify_shard (crates/hypercube/src/verifier/shard.rs:437-750) on proof WORDS produced
// elsewhere (the CUDA library).  No trace data is needed: shapes come from the machine blob and the heights.  Returns 0 if the proof
// is accepted, -1 if rejected (reason on stderr), -2 if the words do not parse.  challenger_state: the state the prover started from
// (updated to the verifier's final state, which must equal the prover's).
namespace {
struct WordReader {
    const uint32_t* p; const uint32_t* end; bool ok = true;
    uint32_t u() { if (p >= end) { ok = false; return 0; } return *p++; }
    F f() { return F::raw(u()); }
    EF ef() { EF e; for (int i = 0; i < 4; i++) e.c[i] = f(); return e; }
    Digest dg() { Digest d; for (int i = 0; i < 8; i++) d.d[i] = f(); return d; }
};
PartialSumcheckProof get_sumcheck(WordReader& r) {
    PartialSumcheckProof p;
    const uint32_t n = r.u();
    if (n > 4096) { r.ok = false; return p; }
    p.polys.resize(n);
    for (auto& u : p.polys) { const uint32_t m = r.u(); if (m > 64) { r.ok = false; return p; } u.c.resize(m); for (auto& c : u.c) c = r.ef(); }
    p.claimed_sum = r.ef();
    p.point.resize(n);
    for (auto& x : p.point) x = r.ef();
    p.eval = r.ef();
    return p;
}
OpeningAndProof get_opening(WordReader& r, size_t nq, size_t width, unsigned log_height) {
    OpeningAndProof op;
    op.values.resize(nq * width);
    for (auto& v : op.values) v = r.f();
    op.proof.merkle_root = r.dg();
    op.proof.log_tensor_height = r.u();
    op.proof.width = r.u();
    if (op.proof.log_tensor_height != log_height || op.proof.width != width) r.ok = false;
    op.proof.paths.resize(nq * log_height);
    for (auto& d : op.proof.paths) d = r.dg();
    return op;
}
}  // namespace

int64_t orc_verify_shard(const uint32_t* machine_blob, const uint64_t* heights, const char* names, uint32_t log_stack, uint32_t max_log_rows,
                         uint32_t log_blowup, uint32_t num_queries, uint32_t pow_bits, uint32_t batch_pow_bits, uint32_t gkr_pow_bits,
                         uint32_t* challenger_state, const uint32_t* prep_commit8, const uint32_t* words, uint64_t n_words) {
    FriParams fp; fp.log_blowup = log_blowup; fp.num_queries = num_queries; fp.pow_bits = pow_bits; fp.batch_pow_bits = batch_pow_bits;
    const uint32_t* rest;
    std::vector<MachineChip> mc = parse_machine(machine_blob, &rest);
    auto inter = parse_interactions(rest, mc.size());
    const size_t n = mc.size();
    std::vector<std::string> nm;
    { const char* p = names; for (size_t k = 0; k < n; k++) { nm.emplace_back(p); p += nm.back().size() + 1; } }
    std::vector<GkrChip> gchips(n);
    std::vector<ZcChip> zchips(n);
    uint64_t prep_area = 0, main_area = 0;
    bool has_prep = false;
    for (size_t k = 0; k < n; k++) {
        gchips[k].height = heights[k]; gchips[k].main_w = mc[k].main_w; gchips[k].prep_w = mc[k].prep_w; gchips[k].inter = inter[k];
        zchips[k].air = &mc[k].air; zchips[k].height = heights[k]; zchips[k].main_w = mc[k].main_w; zchips[k].prep_w = mc[k].prep_w;
        main_area += heights[k] * mc[k].main_w;
        if (mc[k].prep_w) { has_prep = true; prep_area += heights[k] * mc[k].prep_w; }
    }
    if (n_words < 6 || words[0] != 5) return -2;
    const uint64_t l0 = words[1], l1 = words[2], l2 = words[3], l3 = words[4], l4 = words[5];
    if (6 + l0 + l1 + l2 + l3 + l4 != n_words || l0 != 8) return -2;
    const uint32_t* s0 = words + 6; const uint32_t* s1 = s0 + l0; const uint32_t* s2 = s1 + l1; const uint32_t* s3 = s2 + l2; const uint32_t* s4 = s3 + l3;
    Digest main_commit; for (int i = 0; i < 8; i++) main_commit.d[i] = F::raw(s0[i]);
    std::vector<F> pv(l4);
    for (uint64_t i = 0; i < l4; i++) pv[i] = F::raw(s4[i]);
    // LogUp-GKR section
    GkrProof gp;
    {
        WordReader r{s1, s2};
        const uint32_t n_out = r.u();
        if (n_out > (1u << 20)) return -2;
        gp.out_num.resize(n_out); gp.out_den.resize(n_out);
        for (auto& e : gp.out_num) e = r.ef();
        for (auto& e : gp.out_den) e = r.ef();
        const uint32_t nr = r.u();
        if (nr > 64) return -2;
        gp.rounds.resize(nr);
        for (auto& q : gp.rounds) { q.n0 = r.ef(); q.n1 = r.ef(); q.d0 = r.ef(); q.d1 = r.ef(); q.sc = get_sumcheck(r); }
        gp.point.resize(max_log_rows);
        for (auto& e : gp.point) e = r.ef();
        gp.main_open.resize(n); gp.prep_open.resize(n);
        for (size_t k = 0; k < n; k++) {
            gp.main_open[k].resize(mc[k].main_w); gp.prep_open[k].resize(mc[k].prep_w);
            for (auto& e : gp.main_open[k]) e = r.ef();
            for (auto& e : gp.prep_open[k]) e = r.ef();
        }
        gp.witness = r.f();
        if (!r.ok || r.p != s2) return -2;
    }
    // zerocheck section
    ZerocheckResult zr;
    {
        WordReader r{s2, s3};
        zr.proof = get_sumcheck(r);
        zr.opened.resize(n);
        for (size_t k = 0; k < n; k++) {
            zr.opened[k].prep.resize(mc[k].prep_w); zr.opened[k].main.resize(mc[k].main_w);
            for (auto& e : zr.opened[k].prep) e = r.ef();
            for (auto& e : zr.opened[k].main) e = r.ef();
            zr.opened[k].degree = point_from_usize(heights[k], max_log_rows + 1);
        }
        if (!r.ok || r.p != s3) return -2;
    }
    // evaluation proof section
    JaggedProof jp;
    const size_t n_rounds = has_prep ? 2 : 1;
    {
        WordReader r{s3, s4};
        const uint64_t S = (uint64_t)1 << log_stack;
        std::vector<size_t> ncols;
        if (has_prep) ncols.push_back((size_t)std::max<uint64_t>((prep_area + S - 1) / S, 1));
        ncols.push_back((size_t)std::max<uint64_t>((main_area + S - 1) / S, 1));
        BasefoldProof& bf = jp.pcs.basefold;
        bf.univariate_messages.resize(log_stack);
        for (auto& m : bf.univariate_messages) { m[0] = r.ef(); m[1] = r.ef(); }
        bf.fri_commitments.resize(log_stack);
        for (auto& d : bf.fri_commitments) d = r.dg();
        for (size_t q = 0; q < n_rounds; q++) bf.component.push_back(get_opening(r, num_queries, ncols[q], log_stack + log_blowup));
        for (uint32_t q = 0; q < log_stack; q++) bf.query_phase.push_back(get_opening(r, num_queries, 8, log_stack + log_blowup - q - 1));
        bf.final_poly = r.ef();
        bf.pow_witness = r.f();
        bf.batch_grinding_witness = r.f();
        jp.pcs.batch_evaluations.resize(n_rounds);
        for (size_t q = 0; q < n_rounds; q++) { jp.pcs.batch_evaluations[q].resize(ncols[q]); for (auto& e : jp.pcs.batch_evaluations[q]) e = r.ef(); }
        jp.sumcheck = get_sumcheck(r);
        jp.jagged_eval = get_sumcheck(r);
        jp.rc_cc.resize(n_rounds);
        for (auto& v : jp.rc_cc) {
            const uint32_t cnt = r.u();
            if (cnt > 4096) return -2;
            v.resize(cnt);
            for (auto& rc : v) { rc.first = r.u(); rc.second = r.u(); }
        }
        jp.merkle_commits.resize(n_rounds);
        for (auto& d : jp.merkle_commits) d = r.dg();
        jp.expected_eval = r.ef();
        jp.max_log_rows = r.u();
        jp.log_m = r.u();
        if (!r.ok || r.p != s4) return -2;
    }
    // ---- verify_shard order (same as the verify block of orc_prove_shard_verify)
    Challenger vch; chal_load(vch, challenger_state);
    vch.observe_slice(pv.data(), pv.size());
    vch.observe(main_commit);
    vch.observe(F::from_canonical(n));
    for (size_t k = 0; k < n; k++) {
        vch.observe(F::from_canonical(heights[k])); vch.observe(F::from_canonical(nm[k].size()));
        for (unsigned char b : nm[k]) vch.observe(F::from_canonical(b));
    }
    const char* err = gkr_verify(gchips, max_log_rows, gkr_pow_bits, gp, vch);
    if (!err) err = zerocheck_verify(zchips, zr.opened, gp.point, gp.main_open, gp.prep_open, zr.proof, pv, max_log_rows, vch);
    if (!err) {
        std::vector<Digest> commits;
        std::vector<std::vector<EF>> jclaims;
        if (has_prep) {
            Digest pc; for (int i = 0; i < 8; i++) pc.d[i] = F::raw(prep_commit8[i]);
            commits.push_back(pc);
            std::vector<EF> c; for (auto& o : zr.opened) c.insert(c.end(), o.prep.begin(), o.prep.end());
            jclaims.push_back(c);
        }
        commits.push_back(main_commit);
        { std::vector<EF> c; for (auto& o : zr.opened) c.insert(c.end(), o.main.begin(), o.main.end()); jclaims.push_back(c); }
        err = jagged_verify(commits, zr.proof.point, jclaims, jp, vch, log_stack, max_log_rows, fp);
    }
    if (err) { std::fprintf(stderr, "restated shard verifier rejected the proof: %s\n", err); return -1; }
    chal_store(vch, challenger_state);
    return 0;
}

}  // extern "C"
