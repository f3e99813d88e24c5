// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header).  C entry points of the restated shard checks (debug.hpp), built into
// their own library, oracle/libdebugoracle.so (oracle/debug.mk), for tests/debug_oracle_lib.py.  Report words are those of
// sp1b200_debug_constraints / sp1b200_debug_interactions (include/sp1b200.h); field elements cross as u32 Montgomery words.
#include "debug.hpp"
#include <cstring>

using namespace orc;

namespace {

const F* asF(const uint32_t* p) { return reinterpret_cast<const F*>(p); }

// machine blob (layout documented in include/sp1b200.h): [n_chips] then per chip: main_w prep_w n_constraints n_regs n_instrs n_leaves
// n_consts n_publics n_asserts, instrs (2 words each), leaves (2 words each), consts, publics, assert_regs, assert_alphas; then the
// interaction section: per chip [n_interactions] then per interaction is_send arg_index n_values, multiplicity vcol, value vcols;
// vcol = n_terms constant {source col weight}*
struct BlobChip { AirProgram air; uint32_t main_w, prep_w; std::vector<Interaction> inter; };

const uint32_t* parse_vcol(const uint32_t* b, VCol& v) {
    const uint32_t nt = *b++;
    v.constant = F::raw(*b++);
    for (uint32_t i = 0; i < nt; i++, b += 3) v.terms.push_back(VTerm{(uint8_t)b[0], b[1], F::raw(b[2])});
    return b;
}

std::vector<BlobChip> parse_blob(const uint32_t* b, bool with_interactions) {
    std::vector<BlobChip> out(*b++);
    for (BlobChip& c : out) {
        c.main_w = *b++; c.prep_w = *b++; c.air.n_constraints = *b++; c.air.n_regs = *b++;
        const uint32_t ni = *b++, nl = *b++, nc = *b++, np = *b++, na = *b++;
        for (uint32_t i = 0; i < ni; i++, b += 2) { DagInstr d; std::memcpy(&d, b, 8); c.air.instrs.push_back(d); }
        for (uint32_t i = 0; i < nl; i++, b += 2) { LeafRef l; std::memcpy(&l, b, 8); c.air.leaves.push_back(l); }
        for (uint32_t i = 0; i < nc; i++) c.air.consts.push_back(F::raw(*b++));
        for (uint32_t i = 0; i < np; i++) c.air.publics.push_back(*b++);
        for (uint32_t i = 0; i < na; i++) c.air.assert_regs.push_back((uint16_t)*b++);
        for (uint32_t i = 0; i < na; i++) c.air.assert_alphas.push_back(*b++);
    }
    if (!with_interactions) return out;
    for (BlobChip& c : out) {
        const uint32_t n = *b++;
        for (uint32_t i = 0; i < n; i++) {
            Interaction in;
            in.is_send = *b++ != 0; in.arg_index = *b++;
            const uint32_t nv = *b++;
            b = parse_vcol(b, in.mult);
            for (uint32_t k = 0; k < nv; k++) { VCol v; b = parse_vcol(b, v); in.values.push_back(v); }
            c.inter.push_back(in);
        }
    }
    return out;
}

std::vector<DebugChip> debug_chips(const std::vector<BlobChip>& mc, const uint64_t* heights, const uint32_t* const* main, const uint32_t* const* prep) {
    std::vector<DebugChip> chips(mc.size());
    for (size_t k = 0; k < mc.size(); k++) {
        DebugChip& c = chips[k];
        c.air = &mc[k].air; c.inter = &mc[k].inter; c.height = heights[k]; c.main_w = mc[k].main_w; c.prep_w = mc[k].prep_w;
        c.main = c.height ? asF(main[k]) : nullptr;
        c.prep = c.prep_w && c.height ? asF(prep[k]) : nullptr;
    }
    return chips;
}

uint64_t deliver(const std::vector<uint32_t>& w, uint32_t* out, uint64_t cap) {
    if (out && w.size() <= cap) std::copy(w.begin(), w.end(), out);
    return w.size();
}

}  // namespace

extern "C" {

// main[k] / prep[k]: column-major [w x heights[k]].  Both return the number of report words (written when they fit in cap).
uint64_t orc_debug_constraints(const uint32_t* machine_blob, const uint64_t* heights, const uint32_t* const* main, const uint32_t* const* prep,
                               const uint32_t* pv_words, uint32_t n_pv, uint32_t max_rows, uint32_t* out, uint64_t cap) {
    const std::vector<BlobChip> mc = parse_blob(machine_blob, false);
    std::vector<F> pv(n_pv);
    for (uint32_t i = 0; i < n_pv; i++) pv[i] = F::raw(pv_words[i]);
    return deliver(debug_constraints_report(debug_chips(mc, heights, main, prep), pv.data(), max_rows), out, cap);
}

uint64_t orc_debug_interactions(const uint32_t* machine_blob, const uint64_t* heights, const uint32_t* const* main, const uint32_t* const* prep,
                                uint32_t max_keys, uint32_t* out, uint64_t cap) {
    const std::vector<BlobChip> mc = parse_blob(machine_blob, true);
    return deliver(debug_interactions_report(debug_chips(mc, heights, main, prep), max_keys), out, cap);
}

}  // extern "C"
