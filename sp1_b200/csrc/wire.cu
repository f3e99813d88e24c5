// ShardProof wire format: the flat proof words of sp1b200_prove_shard <-> bincode(ShardProof<SP1GlobalContext, SP1PcsProofInner>),
// the bytes the reference moves between its prover workers, the recursion tree and the verifier
// (crates/hypercube/src/verifier/proof.rs:47-61; bincode = "1.3.3", default configuration: little endian, fixed-width integers,
// u64 lengths, usize as u64, Option tag u8, tuples / arrays / struct fields back to back).  Host code only.
//
// Nested types, in field order (file:line of every struct this follows):
//   ShardProof { public_values: Vec<F>, main_commitment: [F; 8], logup_gkr_proof, zerocheck_proof, opened_values, evaluation_proof }
//   LogupGkrProof { circuit_output { numerator: Mle, denominator: Mle }, round_proofs: Vec<{n0, n1, d0, d1, sumcheck}>,
//                   logup_evaluations { point: Point, chip_openings: BTreeMap<String, { main: MleEval, preprocessed: Option<MleEval> }> },
//                   witness: F }                                                  crates/hypercube/src/logup_gkr/proof.rs:9-62
//   PartialSumcheckProof { univariate_polys: Vec<{coefficients: Vec<EF>}>, claimed_sum, point_and_eval: (Point, EF) }
//                                                                                 slop/crates/sumcheck/src/proof.rs:9-14
//   ShardOpenedValues { chips: BTreeMap<String, { preprocessed {local: Vec<EF>}, main {local}, degree: Point<F> }> }   proof.rs:66-94
//   JaggedPcsProof { pcs_proof: StackedBasefoldProof { basefold_proof, batch_evaluations: Rounds<MleEval> }, sumcheck_proof,
//                    jagged_eval_proof { partial_sumcheck_proof }, row_counts_and_column_counts: Rounds<Vec<(usize, usize)>>,
//                    merkle_tree_commitments: Rounds<[F; 8]>, expected_eval, max_log_row_count, log_m }
//                                                   slop/crates/jagged/src/verifier.rs:16-26, slop/crates/stacked/src/verifier.rs:27-31
//   BasefoldProof { univariate_messages: Vec<[EF; 2]>, fri_commitments: Vec<[F; 8]>, component_..: Vec<MerkleTreeOpeningAndProof>,
//                   query_phase_..: Vec<MerkleTreeOpeningAndProof>, final_poly, pow_witness: F, batch_grinding_witness: F }
//                                                                                 slop/crates/basefold/src/verifier.rs:94-116
//   MerkleTreeOpeningAndProof { values: Tensor<F> [queries, width], proof { merkle_root, log_tensor_height, width, paths: Tensor<[F;8]>
//                   [queries, log_height] } }                                     slop/crates/merkle-tree/src/tcs.rs:50-57,85-91, p3sync.rs:146-170,222
//   Tensor { storage: Vec<T>, dimensions: Vec<usize> }   slop/crates/tensor/src/inner.rs:670-677, dimensions.rs:159-163;
//   Mle { guts: Tensor [n, 1] }  mle.rs:27-31,364-369;  MleEval { evaluations: Tensor [n] }  mle.rs:410-414;  Point { values: Vec }  point.rs:14-18
//   Rounds { rounds: Vec }                                                        slop/crates/commit/src/rounds.rs:6-9
// Leaf encodings: F = KoalaBear as its CANONICAL u32 (not the Montgomery word): pinned by the reference-held file
// crates/prover/src/vk_map_dummy.bin = bincode(BTreeMap<[F; 8], usize>) whose keys [F::from_canonical_u32(i); 8]
// (crates/prover/src/recursion.rs:72-75) appear as the words i (tests/golden/bincode_pins.json); EF = its 4 base coefficients
// back to back (p3 BinomialExtensionField serialises `value: [F; 4]` as a tuple); [F; 8] = 8 words; String = u64 length + bytes.
#include "ctx.cuh"
#include "hostfield.hpp"
#include "proof_layout.hpp"
#include <cstring>
#include <string>
#include <vector>

namespace {

struct BinWriter {
    std::vector<uint8_t> b;
    void u8(uint8_t v) { b.push_back(v); }
    void u32(uint32_t v) { for (int i = 0; i < 4; i++) b.push_back((uint8_t)(v >> (8 * i))); }
    void u64(uint64_t v) { for (int i = 0; i < 8; i++) b.push_back((uint8_t)(v >> (8 * i))); }
    void f(uint32_t monty) { u32(kb::to_canonical(monty)); }
    void fs(const uint32_t* w, size_t n) { for (size_t i = 0; i < n; i++) f(w[i]); }
    void str(const char* s) { const size_t n = strlen(s); u64(n); b.insert(b.end(), s, s + n); }
    void dims(std::initializer_list<uint64_t> d) { u64(d.size()); for (uint64_t x : d) u64(x); }
};

// PartialSumcheckProof
void put_sumcheck(const layout::Sumcheck& s, BinWriter& w) {
    const size_t n = s.polys.size();
    w.u64(n);
    for (size_t i = 0; i < n; i++) { w.u64(s.n_coeffs[i]); w.fs(s.polys[i], 4 * (size_t)s.n_coeffs[i]); }
    w.fs(s.claimed_sum, 4);
    w.u64(n);
    w.fs(s.point, 4 * n);
    w.fs(s.eval, 4);
}

// MleEval<EF> of n evaluations = Tensor { storage, dimensions [n] }
void put_mle_eval(const uint32_t* e, BinWriter& w, size_t n) {
    w.u64(n);
    w.fs(e, 4 * n);
    w.dims({(uint64_t)n});
}

// MerkleTreeOpeningAndProof
void put_opening(const layout::Opening& o, BinWriter& w, size_t nq) {
    w.u64(nq * o.width);
    w.fs(o.values, nq * o.width);
    w.dims({(uint64_t)nq, (uint64_t)o.width});
    w.fs(o.root, 8);
    w.u64(o.log_height); w.u64(o.width);
    w.u64(nq * (uint64_t)o.log_height);
    w.fs(o.paths, nq * (size_t)o.log_height * 8);
    w.dims({(uint64_t)nq, (uint64_t)o.log_height});
}

struct BinReader {
    const uint8_t* p; const uint8_t* end; bool ok = true; const char* why = "truncated";
    bool need(size_t n) { if ((size_t)(end - p) < n) { ok = false; p = end; return false; } return true; }
    uint8_t u8() { if (!need(1)) return 0; return *p++; }
    uint32_t u32() { if (!need(4)) return 0; uint32_t v = 0; for (int i = 0; i < 4; i++) v |= (uint32_t)p[i] << (8 * i); p += 4; return v; }
    uint64_t u64() { if (!need(8)) return 0; uint64_t v = 0; for (int i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i); p += 8; return v; }
    uint32_t f() { const uint32_t c = u32(); if (c >= kb::P) { ok = false; why = "field element is not canonical (>= p)"; return 0; } return kb::to_monty_c(c); }
    void fail(const char* m) { if (ok) { ok = false; why = m; } }
    // a length that is about to be used to read at least `unit` bytes per element
    uint64_t len(size_t unit) { const uint64_t n = u64(); if (ok && unit && n > (uint64_t)(end - p) / unit) fail("length prefix exceeds the input"); return ok ? n : 0; }
    // a count about to become one flat word
    uint32_t narrow(uint64_t v) { if (v > 0xffffffffull) fail("count does not fit the flat layout"); return (uint32_t)v; }
    // n field elements onto o / as n extension elements (zero after a failure); reading stops at the first failure
    void fs(layout::FlatWriter& o, uint64_t n) { for (uint64_t i = 0; i < n && ok; i++) o.u(f()); }
    std::vector<hf::E4> exts(uint64_t n) { std::vector<hf::E4> v(n); for (auto& x : v) for (int i = 0; i < 4 && ok; i++) x.c[i] = f(); return v; }
};

void get_dims(BinReader& r, std::initializer_list<uint64_t> want) {
    const uint64_t nd = r.len(8);
    if (nd != want.size()) { r.fail("tensor has an unexpected number of dimensions"); return; }
    for (uint64_t x : want) if (r.u64() != x) r.fail("tensor dimensions do not match its storage");
}

void get_sumcheck(BinReader& r, layout::FlatWriter& o) {
    const uint64_t n = r.len(8);
    r.narrow(n);
    layout::SumcheckWriter s;
    for (uint64_t i = 0; i < n && r.ok; i++) { const uint32_t m = r.narrow(r.len(16)); s.poly(r.exts(m).data(), m); }
    const hf::E4 claimed_sum = r.exts(1)[0];
    if (r.len(16) != n) r.fail("sumcheck point dimension differs from the number of round polynomials");
    const std::vector<hf::E4> point = r.exts(n);   // at least n_polys coordinates
    s.write(o, claimed_sum, point.data(), r.exts(1)[0]);
}

// MleEval<EF>; returns the number of evaluations
uint64_t get_mle_eval(BinReader& r, layout::FlatWriter& o) {
    const uint64_t n = r.len(16);
    r.fs(o, 4 * n);
    get_dims(r, {n});
    return n;
}

void get_opening(BinReader& r, layout::FlatWriter& o) {
    const uint64_t nv = r.len(4);
    layout::FlatWriter values, root, paths;
    r.fs(values, nv);
    const uint64_t nd = r.len(8);
    if (nd != 2) { r.fail("opening values are not a 2-D tensor"); return; }
    const uint64_t nq = r.u64(), width = r.u64();
    if (nq * width != nv) r.fail("opening values: dimensions do not match the storage");
    r.fs(root, 8);
    const uint64_t lh = r.u64(), wd = r.u64();
    if (wd != width) r.fail("opening: proof width differs from the width of the values");
    r.narrow(lh); r.narrow(wd);
    const uint64_t np = r.len(32);
    if (np != nq * lh) r.fail("opening: number of path digests is not queries x log_height");
    r.fs(paths, 8 * np);
    get_dims(r, {nq, lh});
    // only an intact opening has the words its dimensions promise
    if (r.ok) layout::write_opening(o, values.words.data(), nq, (uint32_t)wd, root.words.data(), (uint32_t)lh, paths.words.data());
}

bool names_sorted(const char* const* names, size_t n) {
    for (size_t k = 1; k < n; k++) if (strcmp(names[k - 1], names[k]) >= 0) return false;
    return true;
}

}  // namespace

extern "C" {

// flat words of sp1b200_prove_shard -> bincode(ShardProof)
sp1b200_err sp1b200_shard_proof_to_bincode(const sp1b200_params* params, uint32_t n_chips, const char* const* chip_names, const uint64_t* h_heights,
                                           const uint32_t* h_main_w, const uint32_t* h_prep_w, const uint32_t* h_proof, uint64_t n_words,
                                           uint8_t* h_out, uint64_t cap_bytes, uint64_t* h_out_bytes) {
    if (!params || !h_heights || !chip_names || !h_main_w || !h_prep_w || !h_proof) return sp1b200_set_error("shard_proof_to_bincode: NULL argument");
    const size_t nch = n_chips;
    const uint32_t mlr = params->max_log_row_count, ls = params->log_stacking_height, nq = params->num_queries;
    if (mlr > 62 || ls > 62) return sp1b200_set_error("shard_proof_to_bincode: parameters out of range");
    if (!names_sorted(chip_names, nch)) return sp1b200_set_error("shard_proof_to_bincode: chip names must be strictly ascending (BTreeMap order)");
    for (size_t k = 0; k < nch; k++)
        if (h_heights[k] >> (mlr + 1)) return sp1b200_set_error("shard_proof_to_bincode: chip %zu: height does not fit %u bits", k, mlr + 1);
    layout::Shape shape;
    shape.n_chips = nch; shape.main_w = h_main_w; shape.prep_w = h_prep_w;
    shape.max_log_row_count = mlr; shape.log_stacking_height = ls; shape.num_queries = nq;
    shape.ncols = layout::round_columns(nch, h_heights, h_main_w, h_prep_w, ls);
    layout::ShardProof v;
    if (const char* why = layout::parse_shard_proof(h_proof, n_words, shape, v))
        return sp1b200_set_error("shard_proof_to_bincode: %s (%llu words)", why, (unsigned long long)n_words);
    BinWriter w;
    w.b.reserve(n_words * 4 + 4096);
    // public_values, main_commitment
    w.u64(v.n_pv); w.fs(v.pv, v.n_pv);
    w.fs(v.commit, 8);
    // logup_gkr_proof: circuit_output.numerator, .denominator = Mle { Tensor [n_out, 1] }
    for (const uint32_t* side : {v.out_num, v.out_den}) { w.u64(v.n_out); w.fs(side, 4 * (size_t)v.n_out); w.dims({v.n_out, 1}); }
    w.u64(v.rounds.size());
    for (auto& q : v.rounds) { w.fs(q.nd, 16); put_sumcheck(q.sc, w); }
    w.u64(mlr);
    w.fs(v.gkr_point, 4 * (size_t)mlr);
    w.u64(nch);
    for (size_t k = 0; k < nch; k++) {
        w.str(chip_names[k]);
        put_mle_eval(v.gkr_main[k], w, h_main_w[k]);
        if (h_prep_w[k]) { w.u8(1); put_mle_eval(v.gkr_prep[k], w, h_prep_w[k]); }
        else w.u8(0);
    }
    w.fs(v.gkr_witness, 1);
    // zerocheck_proof, opened_values
    put_sumcheck(v.zc, w);
    w.u64(nch);
    for (size_t k = 0; k < nch; k++) {
        w.str(chip_names[k]);
        w.u64(h_prep_w[k]); w.fs(v.zc_prep[k], 4 * (size_t)h_prep_w[k]);
        w.u64(h_main_w[k]); w.fs(v.zc_main[k], 4 * (size_t)h_main_w[k]);
        w.u64(mlr + 1);   // degree: Point::from_usize(height, max_log_row_count + 1), most significant bit first
        for (int i = (int)mlr; i >= 0; i--) w.u32((uint32_t)((h_heights[k] >> i) & 1));
    }
    {   // evaluation_proof
        const size_t n_rounds = shape.ncols.size();
        w.u64(ls); w.fs(v.univariate, 8 * (size_t)ls);   // univariate_messages: Vec<[EF; 2]>
        w.u64(ls); w.fs(v.fri_commits, 8 * (size_t)ls);  // fri_commitments
        w.u64(n_rounds);
        for (auto& o : v.component) put_opening(o, w, nq);
        w.u64(ls);
        for (auto& o : v.query) put_opening(o, w, nq);
        w.fs(v.final_poly, 4); w.fs(v.pow_witness, 1); w.fs(v.batch_witness, 1);
        w.u64(n_rounds);
        for (size_t q = 0; q < n_rounds; q++) put_mle_eval(v.batch_evals[q], w, shape.ncols[q]);
        put_sumcheck(v.jagged_sc, w); put_sumcheck(v.jagged_eval, w);
        w.u64(n_rounds);
        for (auto& t : v.rc_cc) { w.u64(t.size()); for (auto& rc : t) { w.u64(rc.first); w.u64(rc.second); } }
        w.u64(n_rounds);
        w.fs(v.merkle_commits, 8 * n_rounds);
        w.fs(v.expected_eval, 4);
        w.u64(v.max_log_rows); w.u64(v.log_m);
    }
    if (h_out_bytes) *h_out_bytes = w.b.size();
    if (h_out) {
        if (w.b.size() > cap_bytes) return sp1b200_set_error("shard_proof_to_bincode: needs %zu bytes, capacity %llu", w.b.size(), (unsigned long long)cap_bytes);
        memcpy(h_out, w.b.data(), w.b.size());
    }
    return nullptr;
}

// bincode(ShardProof) -> flat words (the form sp1b200's own consumers and the restated verifier read); chip heights are recovered
// from the `degree` points.  Every length, dimension and canonical-range invariant of the byte string is checked.
sp1b200_err sp1b200_shard_proof_from_bincode(const sp1b200_params* params, uint32_t n_chips, const char* const* chip_names, const uint32_t* h_main_w,
                                             const uint32_t* h_prep_w, const uint8_t* h_bytes, uint64_t n_bytes, uint64_t* h_heights_out,
                                             uint32_t* h_proof, uint64_t cap_words, uint64_t* h_words) {
    if (!params || !chip_names || !h_main_w || !h_prep_w || !h_bytes) return sp1b200_set_error("shard_proof_from_bincode: NULL argument");
    const size_t nch = n_chips;
    const uint32_t mlr = params->max_log_row_count;
    if (mlr > 62) return sp1b200_set_error("shard_proof_from_bincode: parameters out of range");
    if (!names_sorted(chip_names, nch)) return sp1b200_set_error("shard_proof_from_bincode: chip names must be strictly ascending (BTreeMap order)");
    BinReader r{h_bytes, h_bytes + n_bytes};
    layout::FlatWriter pv, gkr, zc, ev;
    uint32_t commit[8];
    auto chip_name = [&](size_t k) {
        const uint64_t n = r.len(1);
        if (!r.ok) return;
        if (n != strlen(chip_names[k]) || memcmp(r.p, chip_names[k], n)) r.fail("chip name differs from the machine's");
        r.p += n;
    };
    const uint64_t n_pv = r.len(4);
    r.fs(pv, n_pv);
    for (int i = 0; i < 8; i++) commit[i] = r.f();
    {   // logup_gkr_proof
        uint64_t n_out = 0;
        for (int side = 0; side < 2 && r.ok; side++) {
            const uint64_t n = r.len(16);
            if (side == 0) { n_out = n; gkr.u(r.narrow(n)); } else if (n != n_out) r.fail("circuit output: numerator and denominator lengths differ");
            r.fs(gkr, 4 * n);
            get_dims(r, {n, 1});
        }
        const uint64_t nr = r.len(64);
        gkr.u(r.narrow(nr));
        for (uint64_t i = 0; i < nr && r.ok; i++) { r.fs(gkr, 16); get_sumcheck(r, gkr); }
        if (r.len(16) != mlr) r.fail("LogUp evaluation point is not max_log_row_count long");
        r.fs(gkr, 4 * (size_t)mlr);
        if (r.len(8) != nch) r.fail("chip_openings: number of chips differs from the machine's");
        for (size_t k = 0; k < nch && r.ok; k++) {
            chip_name(k);
            if (get_mle_eval(r, gkr) != h_main_w[k]) r.fail("chip_openings: main width differs from the machine's");
            const uint8_t tag = r.u8();
            if (tag > 1) r.fail("invalid Option tag");
            if ((tag == 1) != (h_prep_w[k] != 0)) r.fail("chip_openings: preprocessed openings present/absent against the machine");
            if (tag == 1 && get_mle_eval(r, gkr) != h_prep_w[k]) r.fail("chip_openings: preprocessed width differs from the machine's");
        }
        r.fs(gkr, 1);
    }
    get_sumcheck(r, zc);
    if (r.len(8) != nch) r.fail("opened_values: number of chips differs from the machine's");
    for (size_t k = 0; k < nch && r.ok; k++) {
        chip_name(k);
        if (r.len(16) != h_prep_w[k]) r.fail("opened_values: preprocessed width differs from the machine's");
        r.fs(zc, 4 * (size_t)h_prep_w[k]);
        if (r.len(16) != h_main_w[k]) r.fail("opened_values: main width differs from the machine's");
        r.fs(zc, 4 * (size_t)h_main_w[k]);
        if (r.len(4) != mlr + 1) r.fail("opened_values: degree is not max_log_row_count + 1 bits");
        uint64_t h = 0;
        for (uint32_t i = 0; i <= mlr && r.ok; i++) { const uint32_t bit = r.u32(); if (bit > 1) r.fail("opened_values: degree coordinate is not a bit"); h = (h << 1) | bit; }
        if (h_heights_out) h_heights_out[k] = h;
    }
    {   // evaluation_proof
        const uint64_t n_um = r.len(32);
        r.fs(ev, 8 * n_um);
        if (r.len(32) != n_um) r.fail("fri_commitments and univariate_messages differ in length");
        r.fs(ev, 8 * n_um);
        if (n_um != params->log_stacking_height) r.fail("BaseFold proof does not have log_stacking_height rounds");
        const uint64_t n_rounds = r.len(64);
        for (uint64_t q = 0; q < n_rounds && r.ok; q++) get_opening(r, ev);
        if (r.len(64) != n_um) r.fail("query phase does not have one opening per fold round");
        for (uint64_t q = 0; q < n_um && r.ok; q++) get_opening(r, ev);
        r.fs(ev, 6);
        if (r.len(24) != n_rounds) r.fail("batch_evaluations: number of rounds differs");
        for (uint64_t q = 0; q < n_rounds && r.ok; q++) get_mle_eval(r, ev);
        get_sumcheck(r, ev); get_sumcheck(r, ev);
        if (r.len(8) != n_rounds) r.fail("row/column counts: number of rounds differs");
        for (uint64_t q = 0; q < n_rounds && r.ok; q++) {
            layout::Tables t(r.narrow(r.len(16)));
            for (auto& rc : t) if (r.ok) { rc.first = r.narrow(r.u64()); rc.second = r.narrow(r.u64()); }
            layout::write_tables(ev, t);
        }
        if (r.len(32) != n_rounds) r.fail("merkle_tree_commitments: number of rounds differs");
        r.fs(ev, 8 * n_rounds);
        r.fs(ev, 4);
        ev.u(r.narrow(r.u64())); ev.u(r.narrow(r.u64()));
    }
    if (r.ok && r.p != r.end) r.fail("trailing bytes");
    if (!r.ok) return sp1b200_set_error("shard_proof_from_bincode: %s (at byte %llu of %llu)", r.why, (unsigned long long)(r.p - h_bytes), (unsigned long long)n_bytes);
    const uint64_t total = layout::shard_proof_words(gkr.words.size(), zc.words.size(), ev.words.size(), pv.words.size());
    if (h_words) *h_words = total;
    if (h_proof) {
        if (total > cap_words) return sp1b200_set_error("shard_proof_from_bincode: needs %llu words, capacity %llu", (unsigned long long)total, (unsigned long long)cap_words);
        layout::write_shard_proof(h_proof, commit, gkr.words.data(), gkr.words.size(), zc.words.data(), zc.words.size(), ev.words.data(),
                                  ev.words.size(), pv.words.data(), pv.words.size());
    }
    return nullptr;
}

}  // extern "C"
