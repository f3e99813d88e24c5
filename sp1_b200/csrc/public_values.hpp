// PublicValues<[F; 4], [F; 3], [F; 4], F> (crates/hypercube/src/air/public_values.rs, without the mprotect fields): word offsets of a
// core shard's public values, read by the core-proof verifier (verify_core.cu) and by the public-value lookups of the shard's Byte and
// Range traces (lookup_traces.cu).
#pragma once
#include <cstdint>

namespace pv {
constexpr uint32_t PREV_COMMITTED_VALUE_DIGEST = 0;   // [8][4]
constexpr uint32_t COMMITTED_VALUE_DIGEST = 32;       // [8][4]
constexpr uint32_t PREV_DEFERRED_PROOFS_DIGEST = 64;  // [8]
constexpr uint32_t DEFERRED_PROOFS_DIGEST = 72;       // [8]
constexpr uint32_t PC_START = 80, NEXT_PC = 83;       // [3] each
constexpr uint32_t PREV_EXIT_CODE = 86, EXIT_CODE = 87, IS_EXECUTION_SHARD = 88;
constexpr uint32_t PREVIOUS_INIT_ADDR = 89, LAST_INIT_ADDR = 92, PREVIOUS_FINALIZE_ADDR = 95, LAST_FINALIZE_ADDR = 98;   // [3] each
constexpr uint32_t PREVIOUS_INIT_PAGE_IDX = 101, LAST_INIT_PAGE_IDX = 104, PREVIOUS_FINALIZE_PAGE_IDX = 107, LAST_FINALIZE_PAGE_IDX = 110;
constexpr uint32_t INITIAL_TIMESTAMP = 113, LAST_TIMESTAMP = 117;   // [4] each
constexpr uint32_t GLOBAL_CUMULATIVE_SUM = 130;                     // x[7] then y[7]
constexpr uint32_t PREV_COMMIT_SYSCALL = 144, COMMIT_SYSCALL = 145, PREV_COMMIT_DEFERRED_SYSCALL = 146, COMMIT_DEFERRED_SYSCALL = 147;
constexpr uint32_t IS_FIRST_EXECUTION_SHARD = 150, IS_UNTRUSTED_PROGRAMS_ENABLED = 151;
constexpr uint32_t PROOF_NONCE = 152;                               // [4]
constexpr uint32_t NUM_ELTS = 160;                                  // SP1_PROOF_NUM_PV_ELTS
constexpr uint32_t PROOF_MAX_NUM_PVS = 187;
}  // namespace pv
static_assert(pv::PROOF_NONCE + 4 + 4 == pv::NUM_ELTS, "public values layout");
