// ORACLE — TEST INFRASTRUCTURE ONLY (see field.hpp header).  PARITY UNPINNED BY STORED FIXTURES: these restate Rust code
// (the reference's cfg(sp1_debug_constraints) checks), which cannot be compiled in this image, so nothing reference-held pins them.
//
// The two shard checks, as plain CPU loops over the machine blob (the raw DagInstr bytecode, not the product's lowered stream):
//   crates/hypercube/src/debug.rs:27-79  debug_constraints: every row 0 .. height-1 (height 0: nothing, :40-43) through chip.eval
//       with a builder that records the index of every failing constraint (:45-71); failing rows sorted (:75).  The index of a
//       constraint = its position in eval order = its assert's alpha index (alpha index i <-> alpha^(n_constraints-1-i)).
//   crates/hypercube/src/debug.rs:81-130 debug_constraints_all_chips: the chips in order, each chip's failing rows reported.
//   crates/hypercube/src/lookup/debug.rs:48-117  debug_interactions: rows 0 .. height-1 (:60), sends then receives (:66); a record
//       whenever the multiplicity is not zero (:86); key = (kind, values) (:92-94, scope is always local here); count += for sends,
//       -= for receives (:103-108).
//   crates/hypercube/src/lookup/debug.rs:119-200 debug_interactions_with_all_chips: per key the total over chips (final_map) and the
//       per-chip counts (the chip_values map: every chip with a record of the key); a key is unbalanced when its total is not zero.
// Report words are those of sp1b200_debug_constraints / sp1b200_debug_interactions (include/sp1b200.h).
#pragma once
#include "gkr.hpp"
#include <map>
#include <tuple>

namespace orc {

struct DebugChip {
    const AirProgram* air = nullptr;
    const std::vector<Interaction>* inter = nullptr;   // sends then receives
    size_t height = 0, main_w = 0, prep_w = 0;
    const F* main = nullptr; const F* prep = nullptr;  // column-major [w x height]
};

// eval_air (zerocheck.hpp) with every assert checked on its own: the alpha indices of the failing asserts, ascending, each once
static inline std::vector<uint32_t> failing_constraints(const AirProgram& a, const F* prep_row, const F* main_row, const F* pv, std::vector<F>& regs) {
    regs.assign(a.n_regs, F());
    for (const DagInstr& in : a.instrs) {
        switch (in.opcode) {
            case BC_LOAD_LEAF: { const LeafRef& l = a.leaves[in.a]; regs[in.out] = (l.source == LEAF_MAIN ? main_row : prep_row)[l.col]; break; }
            case BC_LOAD_CONST: regs[in.out] = a.consts[in.a]; break;
            case BC_LOAD_PUBLIC: regs[in.out] = pv[a.publics[in.a]]; break;
            case BC_ADD_F: regs[in.out] = regs[in.a] + regs[in.b]; break;
            case BC_SUB_F: regs[in.out] = regs[in.a] - regs[in.b]; break;
            case BC_MUL_F: regs[in.out] = regs[in.a] * regs[in.b]; break;
            case BC_NEG_F: regs[in.out] = F() - regs[in.a]; break;
            default: assert(false && "bad opcode");
        }
    }
    std::vector<uint32_t> out;
    for (size_t k = 0; k < a.assert_regs.size(); k++)
        if (regs[a.assert_regs[k]].v != 0) out.push_back(a.assert_alphas[k]);
    std::sort(out.begin(), out.end());
    out.erase(std::unique(out.begin(), out.end()), out.end());
    return out;
}

static inline std::vector<uint32_t> debug_constraints_report(const std::vector<DebugChip>& chips, const F* pv, uint32_t max_rows) {
    std::vector<uint32_t> w{0};
    for (size_t k = 0; k < chips.size(); k++) {
        const DebugChip& c = chips[k];
        std::vector<std::pair<size_t, std::vector<uint32_t>>> failed;   // (row, constraints), rows ascending
        std::vector<F> mr(c.main_w), pr(c.prep_w), regs;
        for (size_t r = 0; r < c.height; r++) {
            for (size_t j = 0; j < c.main_w; j++) mr[j] = c.main[j * c.height + r];
            for (size_t j = 0; j < c.prep_w; j++) pr[j] = c.prep[j * c.height + r];
            std::vector<uint32_t> f = failing_constraints(*c.air, pr.data(), mr.data(), pv, regs);
            if (!f.empty()) failed.emplace_back(r, std::move(f));
        }
        if (failed.empty()) continue;
        w[0]++;
        const size_t listed = std::min<size_t>(failed.size(), max_rows);
        w.push_back((uint32_t)k); w.push_back((uint32_t)failed.size()); w.push_back((uint32_t)listed);
        for (size_t i = 0; i < listed; i++) {
            w.push_back((uint32_t)failed[i].first); w.push_back((uint32_t)failed[i].second.size());
            w.insert(w.end(), failed[i].second.begin(), failed[i].second.end());
        }
    }
    return w;
}

static inline std::vector<uint32_t> debug_interactions_report(const std::vector<DebugChip>& chips, uint32_t max_keys) {
    struct Entry { std::tuple<size_t, size_t, size_t> first; F net; std::map<size_t, F> per_chip; };   // first: (chip, row, interaction)
    std::map<std::vector<uint32_t>, Entry> keys;                                                         // key words: kind, n_values, values
    for (size_t k = 0; k < chips.size(); k++) {
        const DebugChip& c = chips[k];
        std::vector<F> mr(c.main_w), pr(c.prep_w);
        for (size_t r = 0; r < c.height; r++) {
            for (size_t j = 0; j < c.main_w; j++) mr[j] = c.main[j * c.height + r];
            for (size_t j = 0; j < c.prep_w; j++) pr[j] = c.prep[j * c.height + r];
            for (size_t i = 0; i < c.inter->size(); i++) {
                const Interaction& in = (*c.inter)[i];
                const F m = vcol_apply<F>(in.mult, pr.data(), mr.data());
                if (m.v == 0) continue;
                std::vector<uint32_t> key{in.arg_index, (uint32_t)in.values.size()};
                for (const VCol& v : in.values) key.push_back(vcol_apply<F>(v, pr.data(), mr.data()).v);
                auto it = keys.find(key);
                if (it == keys.end()) it = keys.emplace(key, Entry{{k, r, i}, F(), {}}).first;
                const F s = in.is_send ? m : F() - m;
                it->second.net += s;
                auto pc = it->second.per_chip.find(k);
                if (pc == it->second.per_chip.end()) it->second.per_chip.emplace(k, s); else pc->second += s;
            }
        }
    }
    std::vector<std::pair<const std::vector<uint32_t>*, const Entry*>> bad;
    for (auto& [key, e] : keys) if (e.net.v != 0) bad.emplace_back(&key, &e);
    std::sort(bad.begin(), bad.end(), [](const auto& a, const auto& b) { return a.second->first < b.second->first; });
    const uint64_t n = bad.size();
    const size_t listed = std::min<uint64_t>(n, max_keys);
    std::vector<uint32_t> w{(uint32_t)n, (uint32_t)(n >> 32), (uint32_t)listed};
    for (size_t j = 0; j < listed; j++) {
        const std::vector<uint32_t>& key = *bad[j].first;
        const Entry& e = *bad[j].second;
        w.insert(w.end(), key.begin(), key.end());
        w.push_back(e.net.v);
        w.push_back((uint32_t)std::get<0>(e.first)); w.push_back((uint32_t)std::get<2>(e.first)); w.push_back((uint32_t)std::get<1>(e.first));
        w.push_back((uint32_t)e.per_chip.size());
        for (auto& [c, x] : e.per_chip) { w.push_back((uint32_t)c); w.push_back(x.v); }
    }
    return w;
}

}  // namespace orc
