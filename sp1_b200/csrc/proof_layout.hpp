// The flat proof words of sp1b200_prove_shard, read and written in one place.  The wire format (wire.cu) and the shard verifier
// (verify.cu) walk a proof through parse_shard_proof, and the shard prover (shard.cu) reads the LogUp-GKR and zerocheck outputs it
// chains with the same section readers.  The phase provers and the wire format write the sections through the writers next to those
// readers, so no reader or writer can disagree about the layout.  Also the jagged round's shape rules the prover and the verifier
// share, and the copy-out of an entry point's words.  Host code only.
//
// Words: [5][len_0..len_4] then the sections
//   0 main commitment (8)
//   1 LogUp-GKR: n_out | numerator ext[n_out] | denominator ext[n_out] | n_rounds | per round {n0 n1 d0 d1 ext, sumcheck} |
//     point ext[max_log_row_count] | per chip {main openings ext[main_w], preprocessed openings ext[prep_w]} | witness
//   2 zerocheck: sumcheck | per chip {preprocessed evaluations ext[prep_w], main evaluations ext[main_w]}
//   3 evaluation proof: univariate_messages ext[2 log_stacking_height] | fri_commitments digest[log_stacking_height] |
//     per commitment round an opening of width ncols[round] | per fold round an opening of width 8 | final_poly ext |
//     pow_witness | batch_grinding_witness | batch_evaluations ext[ncols[round]] per round | Hadamard sumcheck | jagged-eval sumcheck |
//     per round {n_tables, (rows, cols) per table} | original commitments digest[n_rounds] | expected_eval ext | max_log_row_count | log_m
//   4 public values
// sumcheck = n_polys | per poly {n_coeffs, coeffs ext} | claimed_sum ext | point ext[n_polys] | eval ext
// opening  = values[num_queries][width] | root digest | log_height | width | paths digest[num_queries][log_height]
// Every length read from the words is checked against the words that remain before it is used.
#pragma once
#include "hostfield.hpp"
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <utility>
#include <vector>

const char* sp1b200_set_error(const char* fmt, ...);   // ctx.cu

namespace layout {

// limits on the counts a proof carries (anything larger cannot come from a prover of this library)
constexpr uint32_t MAX_GKR_OUTPUTS = 1u << 24;
constexpr uint32_t MAX_ROUNDS = 64;         // GKR layers
constexpr uint32_t MAX_SUMCHECK_VARS = 4096;
constexpr uint32_t MAX_COEFFS = 64;
constexpr uint32_t MAX_LOG_HEIGHT = 64;
constexpr uint32_t MAX_TABLES = 1u << 20;

struct FlatReader {
    const uint32_t* p; const uint32_t* end; bool ok = true;
    uint32_t u() { if (p >= end) { ok = false; return 0; } return *p++; }
    const uint32_t* take(size_t n) { if ((size_t)(end - p) < n) { ok = false; p = end; return nullptr; } const uint32_t* r = p; p += n; return r; }
};

struct FlatWriter {
    std::vector<uint32_t> words;
    void u(uint32_t x) { words.push_back(x); }
    void put(const uint32_t* p, size_t n) { words.insert(words.end(), p, p + n); }
    void ext(const hf::E4& e) { put(e.c, 4); }
};

struct Sumcheck {
    std::vector<const uint32_t*> polys;   // coefficients, ext each
    std::vector<uint32_t> n_coeffs;
    const uint32_t* claimed_sum = nullptr;
    const uint32_t* point = nullptr;      // ext[polys.size()]
    const uint32_t* eval = nullptr;
};
struct Opening {
    const uint32_t* values = nullptr;     // [num_queries][width]
    const uint32_t* root = nullptr;
    uint32_t log_height = 0, width = 0;
    const uint32_t* paths = nullptr;      // [num_queries][log_height] digests
};
struct GkrRound { const uint32_t* nd = nullptr; Sumcheck sc; };   // nd: n0 n1 d0 d1, ext each

// The machine's side of the layout: chip widths, the protocol parameters and the stacked column count of every commitment round.
struct Shape {
    size_t n_chips = 0;
    const uint32_t* main_w = nullptr; const uint32_t* prep_w = nullptr;
    uint32_t max_log_row_count = 0, log_stacking_height = 0, num_queries = 0;
    std::vector<size_t> ncols;            // per commitment round: {preprocessed,} main
};

// A jagged round's tables as (rows, cols) runs: its chip tables, then its two padding tables.
using Tables = std::vector<std::pair<uint64_t, uint64_t>>;

// n_tables | (rows, cols) per table: one round of the evaluation proof's row and column counts
inline void write_tables(FlatWriter& w, const Tables& tables) {
    w.u((uint32_t)tables.size());
    for (auto& t : tables) { w.u((uint32_t)t.first); w.u((uint32_t)t.second); }
}

// the stacked columns of 2^log_stack cells that hold a round of `area` cells: ceil(area / 2^log_stack), at least 1
inline uint64_t stacked_columns(uint64_t area, uint32_t log_stack) {
    const uint64_t S = (uint64_t)1 << log_stack;
    return std::max<uint64_t>((area + S - 1) / S, 1);
}

// The two padding tables that fill a round of `area` cells up to its stacked columns: (2^max_log_row_count rows, n - 1 columns)
// and (the rest, 1 column), n being the fewest columns of 2^max_log_row_count rows that hold the padding (at least 1).
inline Tables padding_tables(uint64_t area, uint32_t log_stack, uint32_t max_log_row_count) {
    const uint64_t R = (uint64_t)1 << max_log_row_count, added = (stacked_columns(area, log_stack) << log_stack) - area;
    const uint64_t n = std::max<uint64_t>((added + R - 1) / R, 1);
    return {{R, n - 1}, {added - (n - 1) * R, 1}};
}

// Appends the tables' columns to the column prefix sums: prefix[c] = the rows of every column before column c, and the last entry
// is the running total (start from {0}).
inline void append_column_prefix(std::vector<uint64_t>& prefix, const Tables& tables) {
    for (auto& t : tables)
        for (uint64_t c = 0; c < t.second; c++) prefix.push_back(prefix.back() + t.first);
}

// ncols of a shard: stacked_columns per round (a preprocessed round only if a chip has such columns)
inline std::vector<size_t> round_columns(size_t n_chips, const uint64_t* heights, const uint32_t* main_w, const uint32_t* prep_w, uint32_t log_stack) {
    uint64_t prep_area = 0, main_area = 0; bool has_prep = false;
    for (size_t k = 0; k < n_chips; k++) {
        main_area += heights[k] * main_w[k];
        if (prep_w[k]) { has_prep = true; prep_area += heights[k] * prep_w[k]; }
    }
    std::vector<size_t> n;
    if (has_prep) n.push_back((size_t)stacked_columns(prep_area, log_stack));
    n.push_back((size_t)stacked_columns(main_area, log_stack));
    return n;
}

struct ShardProof {
    const uint32_t* commit = nullptr;
    const uint32_t* pv = nullptr; uint32_t n_pv = 0;
    // LogUp-GKR
    uint32_t n_out = 0; const uint32_t* out_num = nullptr; const uint32_t* out_den = nullptr;
    std::vector<GkrRound> rounds;
    const uint32_t* gkr_point = nullptr;
    std::vector<const uint32_t*> gkr_main, gkr_prep;
    const uint32_t* gkr_witness = nullptr;
    // zerocheck
    Sumcheck zc;
    std::vector<const uint32_t*> zc_prep, zc_main;
    // evaluation proof
    const uint32_t* univariate = nullptr;   // ext[2 * log_stacking_height]
    const uint32_t* fri_commits = nullptr;  // digest[log_stacking_height]
    std::vector<Opening> component, query;
    const uint32_t* final_poly = nullptr;
    const uint32_t* pow_witness = nullptr; const uint32_t* batch_witness = nullptr;
    std::vector<const uint32_t*> batch_evals;
    Sumcheck jagged_sc, jagged_eval;
    std::vector<Tables> rc_cc;
    const uint32_t* merkle_commits = nullptr;
    const uint32_t* expected_eval = nullptr;
    uint32_t max_log_rows = 0, log_m = 0;
};

inline bool read_sumcheck(FlatReader& r, Sumcheck& s) {
    const uint32_t n = r.u();
    if (!r.ok || n > MAX_SUMCHECK_VARS) return false;
    s.polys.resize(n); s.n_coeffs.resize(n);
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t m = r.u();
        if (!r.ok || m > MAX_COEFFS) return false;
        s.n_coeffs[i] = m;
        s.polys[i] = r.take(4 * (size_t)m);
    }
    s.claimed_sum = r.take(4);
    s.point = r.take(4 * (size_t)n);
    s.eval = r.take(4);
    return r.ok;
}

// A sumcheck as its prover emits it: poly() once per round polynomial, between transcript steps, then write() once the point and
// the evaluation are known.  The point has one coordinate per round polynomial, the most recent challenge first.
struct SumcheckWriter {
    FlatWriter polys;
    uint32_t n_polys = 0;
    void poly(const hf::E4* coeffs, uint32_t n_coeffs) {
        polys.u(n_coeffs);
        for (uint32_t i = 0; i < n_coeffs; i++) polys.ext(coeffs[i]);
        n_polys++;
    }
    void write(FlatWriter& w, const hf::E4& claimed_sum, const hf::E4* point, const hf::E4& eval) const {
        w.u(n_polys);
        w.put(polys.words.data(), polys.words.size());
        w.ext(claimed_sum);
        for (uint32_t i = 0; i < n_polys; i++) w.ext(point[i]);
        w.ext(eval);
    }
};

// nullptr, or what is wrong with the opening
inline const char* read_opening(FlatReader& r, Opening& o, size_t nq, size_t width) {
    o.values = r.take(nq * width);
    o.root = r.take(8);
    o.log_height = r.u(); o.width = r.u();
    if (r.ok && (o.width != width || o.log_height > MAX_LOG_HEIGHT)) return "evaluation proof section: opening width / height words do not match the layout";
    if (r.ok) o.paths = r.take(nq * (size_t)o.log_height * 8);
    return r.ok ? nullptr : "evaluation proof section: section is shorter than its layout";
}

// values: [nq][width]; paths: [nq][log_height] digests
inline void write_opening(FlatWriter& w, const uint32_t* values, size_t nq, uint32_t width, const uint32_t* root, uint32_t log_height,
                          const uint32_t* paths) {
    w.put(values, nq * width);
    w.put(root, 8);
    w.u(log_height); w.u(width);
    w.put(paths, nq * (size_t)log_height * 8);
}

// The LogUp-GKR section (all of r's words) into v's LogUp-GKR fields.  Returns nullptr on success, else what is wrong.
inline const char* read_gkr(FlatReader& r, const Shape& s, ShardProof& v) {
    const size_t nch = s.n_chips;
    v.n_out = r.u();
    if (!r.ok || v.n_out > MAX_GKR_OUTPUTS) return "LogUp-GKR section: output count out of range";
    v.out_num = r.take(4 * (size_t)v.n_out); v.out_den = r.take(4 * (size_t)v.n_out);
    const uint32_t nr = r.u();
    if (!r.ok || nr > MAX_ROUNDS) return "LogUp-GKR section: round count out of range";
    v.rounds.resize(nr);
    for (auto& q : v.rounds) {
        q.nd = r.take(16);
        if (!read_sumcheck(r, q.sc)) return "LogUp-GKR section: malformed round sumcheck";
    }
    v.gkr_point = r.take(4 * (size_t)s.max_log_row_count);
    v.gkr_main.resize(nch); v.gkr_prep.resize(nch);
    for (size_t k = 0; k < nch; k++) { v.gkr_main[k] = r.take(4 * (size_t)s.main_w[k]); v.gkr_prep[k] = r.take(4 * (size_t)s.prep_w[k]); }
    v.gkr_witness = r.take(1);
    if (!r.ok) return "LogUp-GKR section: section is shorter than its layout";
    if (r.p != r.end) return "LogUp-GKR section: trailing words";
    return nullptr;
}

// The zerocheck section (all of r's words) into v's zerocheck fields and opened values.  Returns nullptr on success, else what is wrong.
inline const char* read_zerocheck(FlatReader& r, const Shape& s, ShardProof& v) {
    const size_t nch = s.n_chips;
    if (!read_sumcheck(r, v.zc)) return "zerocheck section: malformed sumcheck";
    v.zc_prep.resize(nch); v.zc_main.resize(nch);
    for (size_t k = 0; k < nch; k++) { v.zc_prep[k] = r.take(4 * (size_t)s.prep_w[k]); v.zc_main[k] = r.take(4 * (size_t)s.main_w[k]); }
    if (!r.ok) return "zerocheck section: section is shorter than its layout";
    if (r.p != r.end) return "zerocheck section: trailing words";
    return nullptr;
}

// Splits and walks the words.  Returns nullptr on success, else what is wrong (prefixed by the section).
inline const char* parse_shard_proof(const uint32_t* w, uint64_t n_words, const Shape& s, ShardProof& v) {
    if (!w || n_words < 6 || w[0] != 5) return "not a shard proof (header)";
    const uint64_t l0 = w[1], l1 = w[2], l2 = w[3], l3 = w[4], l4 = w[5];
    if (6 + l0 + l1 + l2 + l3 + l4 != n_words || l0 != 8) return "section lengths do not add up";
    const uint32_t* s0 = w + 6; const uint32_t* s1 = s0 + l0; const uint32_t* s2 = s1 + l1; const uint32_t* s3 = s2 + l2; const uint32_t* s4 = s3 + l3;
    v.commit = s0; v.pv = s4; v.n_pv = (uint32_t)l4;
    const size_t nq = s.num_queries;
    const uint32_t ls = s.log_stacking_height;
    FlatReader gkr{s1, s2}, zc{s2, s3};
    if (const char* e = read_gkr(gkr, s, v)) return e;
    if (const char* e = read_zerocheck(zc, s, v)) return e;
    {   // evaluation proof
        FlatReader r{s3, s4};
        const size_t n_rounds = s.ncols.size();
        v.univariate = r.take(8 * (size_t)ls);
        v.fri_commits = r.take(8 * (size_t)ls);
        if (!r.ok) return "evaluation proof section: section is shorter than its layout";
        v.component.resize(n_rounds); v.query.resize(ls);
        for (size_t q = 0; q < n_rounds; q++)
            if (const char* e = read_opening(r, v.component[q], nq, s.ncols[q])) return e;
        for (uint32_t q = 0; q < ls; q++)
            if (const char* e = read_opening(r, v.query[q], nq, 8)) return e;
        v.final_poly = r.take(4); v.pow_witness = r.take(1); v.batch_witness = r.take(1);
        v.batch_evals.resize(n_rounds);
        for (size_t q = 0; q < n_rounds; q++) v.batch_evals[q] = r.take(4 * s.ncols[q]);
        if (!r.ok) return "evaluation proof section: section is shorter than its layout";
        if (!read_sumcheck(r, v.jagged_sc) || !read_sumcheck(r, v.jagged_eval)) return "evaluation proof section: malformed sumcheck";
        v.rc_cc.resize(n_rounds);
        for (auto& t : v.rc_cc) {
            const uint32_t cnt = r.u();
            if (!r.ok || cnt > MAX_TABLES || (uint64_t)cnt * 2 > (uint64_t)(r.end - r.p)) return "evaluation proof section: table count out of range";
            t.resize(cnt);
            for (auto& rc : t) { rc.first = r.u(); rc.second = r.u(); }
        }
        v.merkle_commits = r.take(8 * n_rounds);
        v.expected_eval = r.take(4);
        v.max_log_rows = r.u(); v.log_m = r.u();
        if (!r.ok) return "evaluation proof section: section is shorter than its layout";
        if (r.p != s4) return "evaluation proof section: trailing words";
    }
    return nullptr;
}

// The words of a shard proof whose sections 1..4 have these lengths.
inline uint64_t shard_proof_words(uint64_t n_gkr, uint64_t n_zc, uint64_t n_ev, uint64_t n_pv) { return 6 + 8 + n_gkr + n_zc + n_ev + n_pv; }

// The mirror of parse_shard_proof's split: [5][len_0..len_4] and the five sections into out (shard_proof_words of room).
inline void write_shard_proof(uint32_t* out, const uint32_t* commit, const uint32_t* gkr, uint64_t n_gkr, const uint32_t* zc, uint64_t n_zc,
                              const uint32_t* ev, uint64_t n_ev, const uint32_t* pv, uint64_t n_pv) {
    const uint32_t hdr[6] = {5, 8, (uint32_t)n_gkr, (uint32_t)n_zc, (uint32_t)n_ev, (uint32_t)n_pv};
    const std::pair<const uint32_t*, uint64_t> sections[6] = {{hdr, 6}, {commit, 8}, {gkr, n_gkr}, {zc, n_zc}, {ev, n_ev}, {pv, n_pv}};
    for (auto& s : sections) { memcpy(out, s.first, s.second * 4); out += s.second; }
}

// Copies an entry point's words to h_out (if not NULL) after the `at` words it already wrote there.  *h_words (if not NULL) gets the
// total either way; a total above cap is the error "<who>: <what> needs N words, capacity C" and copies nothing.
inline const char* deliver(const char* who, const char* what, const std::vector<uint32_t>& words, uint32_t* h_out, uint64_t cap,
                           uint64_t* h_words, uint64_t at = 0) {
    const uint64_t total = at + words.size();
    if (h_words) *h_words = total;
    if (total > cap) return sp1b200_set_error("%s: %s needs %llu words, capacity %llu", who, what, (unsigned long long)total, (unsigned long long)cap);
    if (h_out) memcpy(h_out + at, words.data(), words.size() * 4);
    return nullptr;
}

}  // namespace layout
