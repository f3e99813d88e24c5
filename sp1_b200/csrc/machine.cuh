// The machine description shared by zerocheck.cu and gkr.cu: per-chip constraint bytecode (reference layout,
// sp1-gpu/crates/sys/include/zerocheck/sequential.cuh:13-49) and LogUp interactions.
#pragma once
#include "hostfield.hpp"
#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

struct DagInstr { uint8_t opcode, pad; uint16_t out, a, b; };
struct LeafRef { uint8_t source, pad; uint16_t pad2; uint32_t col; };
static_assert(sizeof(DagInstr) == 8 && sizeof(LeafRef) == 8, "bytecode layout must match sequential.cuh");
enum : uint8_t { BC_LOAD_LEAF = 0, BC_LOAD_CONST = 1, BC_LOAD_PUBLIC = 2, BC_ADD_F = 3, BC_SUB_F = 4, BC_MUL_F = 5, BC_NEG_F = 6 };
enum : uint8_t { LEAF_PREP = 2, LEAF_MAIN = 4 };

struct ZcInstr;    // lowered instruction stream (zc_lower.hpp)
struct ChipProg {  // device pointers into the machine arena
    const DagInstr* instrs; const LeafRef* leaves; const uint32_t* consts; const uint32_t* publics;
    const uint32_t* assert_regs; const uint32_t* assert_alphas;
    uint32_t n_instrs, n_asserts, n_regs, main_w, prep_w, n_constraints;
    const ZcInstr* zc; uint32_t n_zc, zc_regs;  // re-scheduled program interpreted by the zerocheck kernels
};
struct HostProg {  // host copy for host_eval_constraints (the prover's all-zero row, the verifier's opened values)
    std::vector<DagInstr> instrs; std::vector<LeafRef> leaves; std::vector<uint32_t> consts, publics, assert_regs, assert_alphas;
    // the same row polynomial as a sum of self-contained pieces (zc_lower.hpp): {offset into the chip's stream arena, length}
    std::vector<std::pair<uint32_t, uint32_t>> zc_pieces;
};

// The host interpreter of a chip's bytecode at one row of extension values: Σ powers[assert_alphas[i]] · regs[assert_regs[i]].
// leaf(l) is the row's value of leaf l (the prover's all-zero row, the verifier's opened values); pv the public values.
template <class Leaf>
hf::E4 host_eval_constraints(const HostProg& p, uint32_t n_regs, const uint32_t* pv, const std::vector<hf::E4>& powers, Leaf leaf) {
    std::vector<hf::E4> regs(std::max<uint32_t>(n_regs, 1));
    for (const DagInstr& in : p.instrs) {
        switch (in.opcode) {
            case BC_LOAD_LEAF: regs[in.out] = leaf(p.leaves[in.a]); break;
            case BC_LOAD_CONST: regs[in.out] = hf::E4::from_base(p.consts[in.a]); break;
            case BC_LOAD_PUBLIC: regs[in.out] = hf::E4::from_base(pv[p.publics[in.a]]); break;
            case BC_ADD_F: regs[in.out] = regs[in.a] + regs[in.b]; break;
            case BC_SUB_F: regs[in.out] = regs[in.a] - regs[in.b]; break;
            case BC_MUL_F: regs[in.out] = regs[in.a] * regs[in.b]; break;
            case BC_NEG_F: regs[in.out] = -regs[in.a]; break;
        }
    }
    hf::E4 acc;
    for (size_t i = 0; i < p.assert_regs.size(); i++) acc = acc + powers[p.assert_alphas[i]] * regs[p.assert_regs[i]];
    return acc;
}

// LogUp interactions (crates/hypercube/src/lookup/interaction.rs:11-22), parsed from the machine blob's interaction section (gkr.cu).
// A virtual column is constant + sum weight * column; an interaction's multiplicity is vcols[vcol_start], its values follow.
struct TermDev { uint32_t source, col, weight; };
struct VColDev { uint32_t term_start, n_terms, constant; };
struct InterDev { uint32_t is_send, arg_index, n_values, vcol_start; };
struct HostInteractions {
    std::vector<std::vector<InterDev>> per_chip;   // sends first, then receives
    std::vector<VColDev> vcols;
    std::vector<TermDev> terms;
};

void sp1b200_free_interactions(void* p);

struct sp1b200_machine {
    sp1b200_machine() = default;
    sp1b200_machine(const sp1b200_machine&) = delete;
    sp1b200_machine& operator=(const sp1b200_machine&) = delete;
    ~sp1b200_machine();  // zerocheck.cu: releases the device arenas and the interaction tables (also on a failed create)
    std::vector<ChipProg> chips;
    std::vector<HostProg> host;
    uint32_t* d_arena = nullptr;
    void* d_zc_arena = nullptr;     // all chips' lowered programs
    ChipProg* d_chips = nullptr;    // device copy of `chips`
    void* interactions = nullptr;  // HostInteractions (gkr.cu)
};

void* sp1b200_parse_interactions(const uint32_t* b, const uint32_t* end, size_t n_chips, const uint32_t* widths);

// the two shard checks behind sp1b200_debug_constraints / sp1b200_debug_interactions (report words as include/sp1b200.h documents):
// zerocheck.cu and gkr.cu.  d_main[k] / d_prep[k]: device pointers to chip k's columns, column-major with stride h_heights[k].
typedef const char* sp1b200_err;
struct sp1b200_ctx;
sp1b200_err sp1b200_debug_constraints_device(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint64_t* h_heights, const uint32_t* const* d_main,
                                             const uint32_t* const* d_prep, const uint32_t* h_pv, uint32_t n_pv, uint32_t max_rows,
                                             std::vector<uint32_t>& words);
sp1b200_err sp1b200_debug_interactions_device(sp1b200_ctx* ctx, const sp1b200_machine* m, const uint64_t* h_heights, const uint32_t* const* d_main,
                                              const uint32_t* const* d_prep, uint32_t max_keys, std::vector<uint32_t>& words);
