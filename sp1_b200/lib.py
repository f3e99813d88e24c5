"""ctypes binding of libsp1b200.so (the C ABI declared in include/sp1b200.h).

Mirrors what the Rust shim of INTEGRATION.md binds.  No compute happens in Python and there is no
fallback path: a missing library or a failing call raises.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "libsp1b200.so")

u32p = C.POINTER(C.c_uint32)


# word offsets of PublicValues<[F; 4], [F; 3], [F; 4], F> (crates/hypercube/src/air/public_values.rs, without mprotect) in a shard's
# public values; (offset, length).  A core proof's shards carry PV_MAX_NUM = PROOF_MAX_NUM_PVS words, the first PV_NUM_ELTS of them used.
PV = dict(prev_committed_value_digest=(0, 32), committed_value_digest=(32, 32), prev_deferred_proofs_digest=(64, 8),
          deferred_proofs_digest=(72, 8), pc_start=(80, 3), next_pc=(83, 3), prev_exit_code=(86, 1), exit_code=(87, 1),
          is_execution_shard=(88, 1), previous_init_addr=(89, 3), last_init_addr=(92, 3), previous_finalize_addr=(95, 3),
          last_finalize_addr=(98, 3), previous_init_page_idx=(101, 3), last_init_page_idx=(104, 3), previous_finalize_page_idx=(107, 3),
          last_finalize_page_idx=(110, 3), initial_timestamp=(113, 4), last_timestamp=(117, 4), is_timestamp_high_eq=(121, 1),
          inv_timestamp_high=(122, 1), is_timestamp_low_eq=(123, 1), inv_timestamp_low=(124, 1), global_init_count=(125, 1),
          global_finalize_count=(126, 1), global_page_prot_init_count=(127, 1), global_page_prot_finalize_count=(128, 1),
          global_count=(129, 1), global_cumulative_sum=(130, 14), prev_commit_syscall=(144, 1), commit_syscall=(145, 1),
          prev_commit_deferred_syscall=(146, 1), commit_deferred_syscall=(147, 1), initial_timestamp_inv=(148, 1),
          last_timestamp_inv=(149, 1), is_first_execution_shard=(150, 1), is_untrusted_programs_enabled=(151, 1), proof_nonce=(152, 4),
          empty=(156, 4))
PV_NUM_ELTS = 160
PV_MAX_NUM = 187
VK_TAIL_WORDS = 24   # pc_start[3] | initial_global_cumulative_sum x[7] y[7] | enable_untrusted_programs | 6 zeros
# word offsets of RecursionPublicValues<F> (crates/recursion/executor/src/public_values.rs:39-143) that verify_compressed reads; the first
# RPV_NUM_TO_HASH words are hashed into `digest`
RPV = dict(sp1_vk_digest=(136, 8), vk_root=(144, 8), is_complete=(168, 1), digest=(175, 8), proof_nonce=(183, 4))
RPV_NUM_TO_HASH = 175
COMPRESSED, SHRINK = 0, 1
# sp1b200_instruction (include/sp1b200.h): Instruction (crates/core/executor/src/instruction.rs:70-83) laid out for C, 24 bytes
INSTRUCTION_DTYPE = np.dtype({"names": ["opcode", "op_a", "imm_b", "imm_c", "pad", "op_b", "op_c"],
                              "formats": [np.uint8, np.uint8, np.uint8, np.uint8, np.uint32, np.uint64, np.uint64],
                              "offsets": [0, 1, 2, 3, 4, 8, 16], "itemsize": 24})
MAX_OPCODE = 52   # Opcode::UNIMP
# preprocessed widths of the core machine's chips with preprocessed columns, in chip-name order
PREP_CHIP_COLS = dict(Byte=7, Program=16, Range=2)
# sp1b200_byte_lookup (include/sp1b200.h): ByteLookupEvent (crates/core/executor/src/events/byte.rs:18-27) with a count, 12 bytes
BYTE_LOOKUP_DTYPE = np.dtype({"names": ["a", "b", "c", "opcode", "pad", "count"],
                              "formats": [np.uint16, np.uint8, np.uint8, np.uint8, (np.uint8, 3), np.uint32],
                              "offsets": [0, 2, 3, 4, 5, 8], "itemsize": 12})
# sp1b200_pc_count: an executed pc with its count, 16 bytes
PC_COUNT_DTYPE = np.dtype({"names": ["pc", "count", "pad"], "formats": [np.uint64, np.uint32, np.uint32], "offsets": [0, 8, 12],
                           "itemsize": 16})
BYTE_OPCODES = dict(AND=0, OR=1, XOR=2, U8Range=3, LTU=4, MSB=5, Range=6)   # ByteOpcode (crates/core/executor/src/opcode.rs:163-178)
# main widths of the same chips: one multiplicity per Byte opcode 0..5, one for Program and one for Range
MAIN_CHIP_COLS = dict(Byte=6, Program=1, Range=1)
# sp1b200_memory_event: MemoryInitializeFinalizeEvent (crates/core/executor/src/events/memory.rs:169-176), 24 bytes
MEMORY_EVENT_DTYPE = np.dtype({"names": ["addr", "value", "timestamp"], "formats": [np.uint64] * 3, "offsets": [0, 8, 16], "itemsize": 24})
# sp1b200_memory_local_event: MemoryLocalEvent (memory.rs:307-314) with its two MemoryRecords inlined, 40 bytes
MEMORY_LOCAL_EVENT_DTYPE = np.dtype({"names": ["addr", "initial_timestamp", "initial_value", "final_timestamp", "final_value"],
                                     "formats": [np.uint64] * 5, "offsets": [0, 8, 16, 24, 32], "itemsize": 40})
# sp1b200_global_event: GlobalInteractionEvent (crates/core/executor/src/events/global.rs), 36 bytes
GLOBAL_EVENT_DTYPE = np.dtype({"names": ["message", "is_receive", "kind", "pad"], "formats": [(np.uint32, 8), np.uint8, np.uint8, (np.uint8, 2)],
                               "offsets": [0, 32, 33, 34], "itemsize": 36})
# main widths of the memory chips, and the byte lookup records sp1b200_memory_traces emits per event
MEMORY_CHIP_COLS = dict(MemoryGlobalInit=30, MemoryGlobalFinalize=30, MemoryLocal=20)
MEMORY_GLOBAL_LOOKUPS, MEMORY_LOCAL_LOOKUPS = 12, 10


def pack_instructions(opcode, op_a, op_b, op_c, imm_b, imm_c):
    """parallel arrays (or scalars) of instruction fields -> a contiguous INSTRUCTION_DTYPE array (the records the library reads)"""
    names = ("opcode", "op_a", "op_b", "op_c", "imm_b", "imm_c")
    cols = [np.atleast_1d(np.asarray(x, dtype=INSTRUCTION_DTYPE[name])) for name, x in zip(names, (opcode, op_a, op_b, op_c, imm_b, imm_c))]
    out = np.zeros(max(c.size for c in cols), INSTRUCTION_DTYPE)
    for name, c in zip(names, cols):
        out[name] = c
    return out


def pack_byte_lookups(opcode, a, b, c, count=1):
    """parallel arrays (or scalars) of byte lookups -> a contiguous BYTE_LOOKUP_DTYPE array (the records the library reads)"""
    names = ("opcode", "a", "b", "c", "count")
    cols = [np.atleast_1d(np.asarray(x, dtype=BYTE_LOOKUP_DTYPE[name])) for name, x in zip(names, (opcode, a, b, c, count))]
    out = np.zeros(max(x.size for x in cols), BYTE_LOOKUP_DTYPE)
    for name, x in zip(names, cols):
        out[name] = x
    return out


def pack_pc_counts(pc, count=1):
    """parallel arrays (or scalars) of executed pcs and their counts -> a contiguous PC_COUNT_DTYPE array"""
    cols = [np.atleast_1d(np.asarray(x, dtype=PC_COUNT_DTYPE[name])) for name, x in (("pc", pc), ("count", count))]
    out = np.zeros(max(x.size for x in cols), PC_COUNT_DTYPE)
    out["pc"], out["count"] = cols
    return out


def pack_memory_events(addr, value, timestamp):
    """parallel arrays (or scalars) of init / finalize events -> a contiguous MEMORY_EVENT_DTYPE array"""
    cols = [x.reshape(-1) for x in np.broadcast_arrays(*[np.asarray(x, dtype=np.uint64) for x in (addr, value, timestamp)])]
    out = np.zeros(cols[0].size, MEMORY_EVENT_DTYPE)
    out["addr"], out["value"], out["timestamp"] = cols
    return out


def pack_memory_local_events(addr, initial_timestamp, initial_value, final_timestamp, final_value):
    """parallel arrays (or scalars) of local memory events -> a contiguous MEMORY_LOCAL_EVENT_DTYPE array"""
    fields = (addr, initial_timestamp, initial_value, final_timestamp, final_value)
    cols = [x.reshape(-1) for x in np.broadcast_arrays(*[np.asarray(x, dtype=np.uint64) for x in fields])]
    out = np.zeros(cols[0].size, MEMORY_LOCAL_EVENT_DTYPE)
    for name, x in zip(MEMORY_LOCAL_EVENT_DTYPE.names, cols):
        out[name] = x
    return out


class Params(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("log_stacking_height", "max_log_row_count", "log_blowup", "num_queries",
                                          "pow_bits", "batch_pow_bits", "gkr_pow_bits", "grind_mode")]


DEFAULT_CORE_PARAMS = dict(log_stacking_height=21, max_log_row_count=22, log_blowup=2, num_queries=124, pow_bits=16,
                           batch_pow_bits=5, gkr_pow_bits=12, grind_mode=0)


class Sp1B200Error(RuntimeError):
    pass


_cdll = None


def load():
    """dlopen the library (no CUDA call is made).  Raises if it has not been built."""
    global _cdll
    if _cdll is None:
        if not os.path.exists(SO_PATH):
            raise Sp1B200Error(f"{SO_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback)")
        L = C.CDLL(SO_PATH)
        L.sp1b200_version.restype = C.c_char_p
        L.sp1b200_ctx_stream.restype = C.c_void_p
        L.sp1b200_launch_count.restype = C.c_uint64
        L.sp1b200_last_phase_ms.restype = C.c_float
        L.sp1b200_challenger_sample_bits.restype = C.c_uint32
        L.sp1b200_challenger_check_witness.restype = C.c_int
        L.sp1b200_machine_num_chips.restype = C.c_uint32
        L.sp1b200_machine_chip_regs.restype = C.c_uint32
        L.sp1b200_verdict_name.restype = C.c_char_p
        L.sp1b200_recursion_vks_num_keys.restype = C.c_uint64
        for name in ERR_FUNCS:
            getattr(L, name).restype = C.c_char_p
        _cdll = L
    return _cdll


# every symbol include/sp1b200.h declares (tests/test_abi.py checks the header against this list and the .so)
ERR_FUNCS = [
    "sp1b200_ctx_create", "sp1b200_ctx_sync", "sp1b200_malloc", "sp1b200_free", "sp1b200_memcpy_h2d",
    "sp1b200_memcpy_d2h", "sp1b200_upload_begin", "sp1b200_pack_row_major", "sp1b200_poseidon2_permute", "sp1b200_rs_encode", "sp1b200_merkle_commit", "sp1b200_grind",
    "sp1b200_stacked_commit", "sp1b200_stacked_prove", "sp1b200_jagged_commit", "sp1b200_jagged_column_claims",
    "sp1b200_jagged_prove", "sp1b200_machine_create", "sp1b200_zerocheck", "sp1b200_logup_gkr", "sp1b200_prove_shard",
    "sp1b200_setup_and_prove_shard", "sp1b200_shard_proof_to_bincode", "sp1b200_shard_proof_from_bincode",
    "sp1b200_debug_constraints", "sp1b200_debug_interactions", "sp1b200_verify_shard", "sp1b200_verify_core_proof",
    "sp1b200_vk_hash", "sp1b200_digest_bytes32", "sp1b200_recursion_pv_digest", "sp1b200_recursion_vks_create", "sp1b200_recursion_vks_open",
    "sp1b200_verify_compressed", "sp1b200_program_vk_tail", "sp1b200_program_preprocessed_traces", "sp1b200_program_setup",
    "sp1b200_lookup_traces", "sp1b200_memory_traces",
]
OTHER_FUNCS = ["sp1b200_challenger_init", "sp1b200_challenger_observe", "sp1b200_challenger_sample",
               "sp1b200_challenger_sample_bits", "sp1b200_challenger_check_witness", "sp1b200_ctx_destroy", "sp1b200_default_core_params", "sp1b200_version", "sp1b200_ctx_stream",
               "sp1b200_launch_count", "sp1b200_last_phase_ms", "sp1b200_commit_free", "sp1b200_jagged_round_free",
               "sp1b200_machine_free", "sp1b200_machine_num_chips", "sp1b200_machine_chip_regs",
               "sp1b200_verdict_name", "sp1b200_recursion_vks_free", "sp1b200_recursion_vks_root", "sp1b200_recursion_vks_num_keys"]


def _ptr(a):
    """numpy uint32 array or torch tensor (cpu or cuda) or int address -> c_void_p"""
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    if isinstance(a, np.ndarray):
        assert a.dtype == np.uint32 and a.flags["C_CONTIGUOUS"], "need contiguous uint32"
        return C.c_void_p(a.ctypes.data)
    if hasattr(a, "data_ptr"):  # torch tensor (int32/uint32 storage)
        assert a.is_contiguous() and a.element_size() == 4
        return C.c_void_p(a.data_ptr())
    raise TypeError(type(a))


def _image_args(mem_addrs, mem_words, page_idx, page_prot):
    """a program's memory image (64-bit addresses and words) and page image (64-bit indices, 8-bit protections) as numpy arrays or torch
    tensors on the host or the device (torch int64 / uint8), None for an absent page image -> (four pointers, n_mem, n_pages, the numpy
    arrays the pointers point into: keep them alive for the call)"""
    ptrs, sizes, keep = [], [], []
    for x, dtype in ((mem_addrs, np.uint64), (mem_words, np.uint64), (page_idx, np.uint64), (page_prot, np.uint8)):
        if x is None:
            ptrs.append(None); sizes.append(0)
        elif hasattr(x, "data_ptr"):
            assert x.is_contiguous() and x.element_size() == np.dtype(dtype).itemsize
            ptrs.append(C.c_void_p(x.data_ptr()) if x.numel() else None); sizes.append(x.numel())
        else:
            x = np.ascontiguousarray(x, dtype=dtype)
            keep.append(x)
            ptrs.append(C.c_void_p(x.ctypes.data) if x.size else None); sizes.append(x.size)
    assert sizes[0] == sizes[1] and sizes[2] == sizes[3], "one word per address and one protection per page index"
    return ptrs, sizes[0], sizes[2], keep


class Lib:
    """One context = one GPU + one stream (reference: one prover process per GPU, crates/cuda/src/server.rs:36-45)."""

    def __init__(self, device=0, **params):
        self.L = load()
        p = dict(DEFAULT_CORE_PARAMS)
        p.update(params)
        self.params = p
        self._p = Params(**p)
        self.ctx = C.c_void_p()
        self._chk(self.L.sp1b200_ctx_create(C.c_int(device), C.byref(self._p), C.byref(self.ctx)))

    def _chk(self, err):
        if err:
            raise Sp1B200Error(err.decode())

    def close(self):
        if self.ctx:
            self.L.sp1b200_ctx_destroy(self.ctx)
            self.ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- runtime ---------------------------------------------------------------------------------------------
    def sync(self):
        self._chk(self.L.sp1b200_ctx_sync(self.ctx))

    def stream(self):
        return self.L.sp1b200_ctx_stream(self.ctx)

    def launch_count(self):
        return int(self.L.sp1b200_launch_count(self.ctx))

    def phase_ms(self, name):
        return float(self.L.sp1b200_last_phase_ms(self.ctx, name.encode()))

    # -- kernel-level ---------------------------------------------------------------------------------------
    def poseidon2_permute(self, states):
        n = states.shape[0] if hasattr(states, "shape") else None
        self._chk(self.L.sp1b200_poseidon2_permute(self.ctx, _ptr(states), C.c_uint64(n)))
        return states

    def rs_encode(self, msg, out, ncols, log_h, log_blowup=None):
        lb = self.params["log_blowup"] if log_blowup is None else log_blowup
        self._chk(self.L.sp1b200_rs_encode(self.ctx, _ptr(msg), C.c_uint64(ncols), C.c_uint32(log_h), C.c_uint32(lb),
                                           _ptr(out)))
        return out

    def merkle_commit(self, mat, width, log_h, d_layers=None):
        root = np.zeros(8, np.uint32)
        commit = np.zeros(8, np.uint32)
        self._chk(self.L.sp1b200_merkle_commit(self.ctx, _ptr(mat), C.c_uint64(width), C.c_uint32(log_h), _ptr(d_layers),
                                               _ptr(root), _ptr(commit)))
        return root, commit

    # -- PCS-level ------------------------------------------------------------------------------------------
    def stacked_commit(self, dense, ncols, keep_codeword=True):
        """dense: [ncols x 2^log_stacking_height] column-major (numpy or cuda tensor). -> (commit[8], handle)"""
        commit = np.zeros(8, np.uint32)
        h = C.c_void_p()
        self._chk(self.L.sp1b200_stacked_commit(self.ctx, _ptr(dense), C.c_uint64(ncols), C.c_int(int(keep_codeword)),
                                                _ptr(commit), C.byref(h)))
        return commit, h

    def commit_free(self, handle):
        self.L.sp1b200_commit_free(self.ctx, handle)

    def stacked_prove(self, handles, point, challenger_state, replay=None, cap_words=1 << 24):
        """point: [k,4] uint32 host array; challenger_state: 34 words (updated in place). -> proof words"""
        n = len(handles)
        arr = (C.c_void_p * n)(*[h.value for h in handles])
        point = np.ascontiguousarray(point, dtype=np.uint32)
        proof = np.empty(cap_words, np.uint32)
        nwords = C.c_uint64()
        rw = None if replay is None else np.ascontiguousarray(replay, dtype=np.uint32)
        self._chk(self.L.sp1b200_stacked_prove(self.ctx, arr, C.c_uint32(n), _ptr(point), C.c_uint32(point.shape[0]),
                                               _ptr(rw), _ptr(challenger_state), _ptr(proof), C.c_uint64(cap_words),
                                               C.byref(nwords)))
        return proof[:nwords.value].copy()

    def jagged_commit(self, tables, keep_codeword=True):
        """tables: list of [cols, rows] uint32 arrays (rows may be 0).  -> (commit[8], handle, shapes)"""
        rows = [int(t.shape[1]) for t in tables]
        cols = [int(t.shape[0]) for t in tables]
        parts = [np.ascontiguousarray(t, dtype=np.uint32).reshape(-1) for t in tables if t.shape[1]]
        dense = np.ascontiguousarray(np.concatenate(parts)) if parts else np.zeros(1, np.uint32)
        return self.jagged_commit_dense(dense, rows, cols, keep_codeword)

    def jagged_commit_dense(self, dense, rows, cols, keep_codeword=True):
        """dense: flat uint32 (numpy or cuda tensor) of all real cells, tables back to back, column-major each"""
        n = len(rows)
        R = (C.c_uint64 * n)(*rows)
        Cc = (C.c_uint64 * n)(*cols)
        commit = np.zeros(8, np.uint32)
        h = C.c_void_p()
        self._chk(self.L.sp1b200_jagged_commit(self.ctx, _ptr(dense), C.c_uint32(n), R, Cc, C.c_int(int(keep_codeword)),
                                               _ptr(commit), C.byref(h)))
        return commit, h

    def jagged_round_free(self, handle):
        self.L.sp1b200_jagged_round_free(self.ctx, handle)

    def jagged_column_claims(self, handle, z_row, ncols_total):
        z = np.ascontiguousarray(z_row, dtype=np.uint32)
        out = np.zeros((ncols_total, 4), np.uint32)
        self._chk(self.L.sp1b200_jagged_column_claims(self.ctx, handle, _ptr(z), _ptr(out)))
        return out

    def jagged_prove(self, handles, z_row, claims, challenger_state, replay=None, cap_words=1 << 24):
        n = len(handles)
        arr = (C.c_void_p * n)(*[h.value for h in handles])
        z = np.ascontiguousarray(z_row, dtype=np.uint32)
        cl = np.ascontiguousarray(claims, dtype=np.uint32)
        proof = np.empty(cap_words, np.uint32)
        nwords = C.c_uint64()
        rw = None if replay is None else np.ascontiguousarray(replay, dtype=np.uint32)
        self._chk(self.L.sp1b200_jagged_prove(self.ctx, arr, C.c_uint32(n), _ptr(z), _ptr(cl), _ptr(rw),
                                              _ptr(challenger_state), _ptr(proof), C.c_uint64(cap_words), C.byref(nwords)))
        return proof[:nwords.value].copy()

    # -- zerocheck --------------------------------------------------------------------------------------------
    def machine_create(self, blob):
        blob = np.ascontiguousarray(blob, dtype=np.uint32)
        h = C.c_void_p()
        self._chk(self.L.sp1b200_machine_create(self.ctx, _ptr(blob), C.c_uint64(blob.size), C.byref(h)))
        return h

    def machine_chip_regs(self, h, chip):
        """peak live registers of a chip's re-scheduled constraint program (register-file tier of the zerocheck kernels)"""
        return int(self.L.sp1b200_machine_chip_regs(h, C.c_uint32(chip)))

    def machine_free(self, h):
        self.L.sp1b200_machine_free(self.ctx, h)

    def zerocheck(self, machine, heights, d_mains, d_preps, pv, gkr_point, alpha, gamma, claims, challenger_state, cap_words=1 << 22):
        """d_mains / d_preps: per chip device tensors (or None).  Returns output words (proof | opened values)."""
        n = len(heights)
        H = (C.c_uint64 * n)(*heights)
        M = (C.c_void_p * n)(*[t.data_ptr() if t is not None and t.numel() else None for t in d_mains])
        Pp = (C.c_void_p * n)(*[t.data_ptr() if t is not None and t.numel() else None for t in d_preps])
        pv = np.ascontiguousarray(pv, dtype=np.uint32)
        out = np.empty(cap_words, np.uint32)
        nw = C.c_uint64()
        self._chk(self.L.sp1b200_zerocheck(self.ctx, machine, H, M, Pp, _ptr(pv), C.c_uint32(pv.size),
                                           _ptr(np.ascontiguousarray(gkr_point, dtype=np.uint32)),
                                           _ptr(np.ascontiguousarray(alpha, dtype=np.uint32)),
                                           _ptr(np.ascontiguousarray(gamma, dtype=np.uint32)),
                                           _ptr(np.ascontiguousarray(claims, dtype=np.uint32)), _ptr(challenger_state), _ptr(out),
                                           C.c_uint64(cap_words), C.byref(nw)))
        return out[:nw.value].copy()

    def logup_gkr(self, machine, heights, d_mains, d_preps, challenger_state, replay=None, cap_words=1 << 22):
        n = len(heights)
        H = (C.c_uint64 * n)(*heights)
        M = (C.c_void_p * n)(*[t.data_ptr() if t is not None and t.numel() else None for t in d_mains])
        Pp = (C.c_void_p * n)(*[t.data_ptr() if t is not None and t.numel() else None for t in d_preps])
        out = np.empty(cap_words, np.uint32)
        nw = C.c_uint64()
        rw = None if replay is None else np.ascontiguousarray([replay], dtype=np.uint32)
        self._chk(self.L.sp1b200_logup_gkr(self.ctx, machine, H, M, Pp, _ptr(rw), _ptr(challenger_state), _ptr(out),
                                           C.c_uint64(cap_words), C.byref(nw)))
        return out[:nw.value].copy()

    def prove_shard(self, machine, prep_round, main_dense, heights, names, pv, challenger_state, replay=None, cap_words=1 << 24):
        n = len(heights)
        H = (C.c_uint64 * n)(*heights)
        NM = (C.c_char_p * n)(*[s.encode() for s in names])
        pv = np.ascontiguousarray(pv, dtype=np.uint32)
        out = np.empty(cap_words, np.uint32)
        nw = C.c_uint64()
        rw = None if replay is None else np.ascontiguousarray(replay, dtype=np.uint32)
        self._chk(self.L.sp1b200_prove_shard(self.ctx, machine, prep_round, _ptr(main_dense), H, NM, _ptr(pv), C.c_uint32(pv.size),
                                             _ptr(rw), _ptr(challenger_state), _ptr(out), C.c_uint64(cap_words), C.byref(nw)))
        return out[:nw.value].copy()

    def verify_shard(self, machine, prep_commit, heights, names, words, challenger_state):
        """ShardVerifier::verify_shard on the flat proof words.  challenger_state: the transcript after the verifying key was observed
        (not modified).  -> (verdict, challenger): verdict 0 accepts, and challenger is then the verifier's final state; otherwise
        verdict names the first failing check (verdict_name) and challenger is the state passed in."""
        n = len(heights)
        H = (C.c_uint64 * max(1, n))(*heights)
        NM = (C.c_char_p * max(1, n))(*[s.encode() for s in names])
        w = np.ascontiguousarray(words, dtype=np.uint32)
        st = np.ascontiguousarray(challenger_state, dtype=np.uint32).copy()
        pc = None if prep_commit is None else np.ascontiguousarray(prep_commit, dtype=np.uint32)
        verdict = C.c_uint32()
        self._chk(self.L.sp1b200_verify_shard(self.ctx, machine, _ptr(pc), H, NM, _ptr(w), C.c_uint64(w.size), _ptr(st), C.byref(verdict)))
        return int(verdict.value), st

    def verify_core_proof(self, machine, prep_commit, vk_tail, heights_per_shard, names, words_per_shard, host_threads=0):
        """SP1Prover::verify on a core proof: the shards' flat proof words (one machine, names and context parameters), chip heights
        per shard, and the verifying key = prep_commit[8] + vk_tail[24].  -> (verdict, shard, shard_verdict, final_challengers):
        verdict 0 accepts and final_challengers is then [n_shards, 34] (each shard verifier's final state), else None; for
        InvalidShardProof, shard_verdict is the failing shard's verify_shard code (verdict_name names both code spaces)."""
        n = len(words_per_shard)
        nch = len(names)
        H = np.ascontiguousarray(np.asarray(heights_per_shard, dtype=np.uint64).reshape(n * nch) if n else np.zeros(1, np.uint64))
        NM = (C.c_char_p * max(1, nch))(*[s.encode() for s in names])
        ws = [None if w is None else np.ascontiguousarray(w, dtype=np.uint32) for w in words_per_shard]
        P = (C.c_void_p * max(1, n))(*[None if w is None else w.ctypes.data for w in ws])
        NW = (C.c_uint64 * max(1, n))(*[0 if w is None else w.size for w in ws])
        pc = np.ascontiguousarray(prep_commit, dtype=np.uint32)
        tail = np.ascontiguousarray(vk_tail, dtype=np.uint32)
        fin = np.zeros((max(1, n), 34), np.uint32)
        verdict, shard, sv = C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._chk(self.L.sp1b200_verify_core_proof(self.ctx, machine, _ptr(pc), _ptr(tail), C.c_uint32(tail.size), C.c_uint32(n),
                                                    C.c_void_p(H.ctypes.data), NM, P, NW, C.c_uint32(host_threads), _ptr(fin),
                                                    C.byref(verdict), C.byref(shard), C.byref(sv)))
        v = int(verdict.value)
        return v, int(shard.value), int(sv.value), (fin[:n].copy() if v == 0 else None)

    def recursion_vks(self, digests, pad_to=0, vk_verification=True):
        """RecursionVks::from_map over the digests ([n, 8] Montgomery words), the tree built on the device -> RecursionVks"""
        d = np.ascontiguousarray(np.asarray(digests, dtype=np.uint32).reshape(-1, 8))
        h = C.c_void_p()
        self._chk(self.L.sp1b200_recursion_vks_create(self.ctx, _ptr(d) if d.size else None, C.c_uint64(d.shape[0]), C.c_uint64(pad_to),
                                                      C.c_int(int(vk_verification)), C.byref(h)))
        return RecursionVks(self.L, h, vk_verification)

    def verify_compressed(self, machine, vks, keys, heights_per_proof, names, words_per_proof, merkle_proofs, sp1_vk_digests,
                          mode=COMPRESSED, shrink_vk=None, host_threads=0):
        """SP1Prover::verify_compressed (mode COMPRESSED) or verify_shrink (mode SHRINK) of n recursion proofs of one machine.
        keys: per proof its verifying key, 32 words (prep_commit[8] | vk_tail[24]); merkle_proofs: per proof (index, path [k, 8]);
        sp1_vk_digests: per proof the expected SP1 program key digest (8 words); shrink_vk: 32 words or None.
        -> (verdicts, shard_verdicts, final_challengers): verdict 0 accepts and final_challengers[s] is then the verifier's final state."""
        n, nch = len(words_per_proof), len(names)
        K = np.ascontiguousarray(np.asarray(keys, dtype=np.uint32).reshape(-1))
        H = np.ascontiguousarray(np.asarray(heights_per_proof, dtype=np.uint64).reshape(-1) if n else np.zeros(1, np.uint64))
        NM = (C.c_char_p * max(1, nch))(*[s.encode() for s in names])
        ws = [None if w is None else np.ascontiguousarray(w, dtype=np.uint32) for w in words_per_proof]
        P = (C.c_void_p * max(1, n))(*[None if w is None else w.ctypes.data for w in ws])
        NW = (C.c_uint64 * max(1, n))(*[0 if w is None else w.size for w in ws])
        paths = [np.ascontiguousarray(np.asarray(p, dtype=np.uint32).reshape(-1)) for _, p in merkle_proofs]
        IDX = (C.c_uint64 * max(1, n))(*[int(i) for i, _ in merkle_proofs])
        PP = (C.c_void_p * max(1, n))(*[p.ctypes.data if p.size else None for p in paths])
        PL = (C.c_uint32 * max(1, n))(*[p.size // 8 for p in paths])
        D = np.ascontiguousarray(np.asarray(sp1_vk_digests, dtype=np.uint32).reshape(-1))
        sv = None if shrink_vk is None else np.ascontiguousarray(shrink_vk, dtype=np.uint32)
        fin = np.zeros((max(1, n), 34), np.uint32)
        verdicts, shard_verdicts = np.zeros(max(1, n), np.uint32), np.zeros(max(1, n), np.uint32)
        self._chk(self.L.sp1b200_verify_compressed(self.ctx, machine, vks.h, C.c_uint32(mode), _ptr(sv), C.c_uint32(n), _ptr(K) if K.size else None,
                                                    C.c_void_p(H.ctypes.data), NM, P, NW, IDX, PP, PL, _ptr(D) if D.size else None,
                                                    C.c_uint32(host_threads), _ptr(fin), _ptr(verdicts), _ptr(shard_verdicts)))
        return [int(v) for v in verdicts[:n]], [int(v) for v in shard_verdicts[:n]], fin[:n].copy()

    def _debug_call(self, fn, args, cap_words):
        out = np.empty(max(1, cap_words), np.uint32)
        nw = C.c_uint64()
        self._chk(fn(self.ctx, *args, _ptr(out), C.c_uint64(cap_words), C.byref(nw)))
        return out[:nw.value].copy()

    def debug_constraints_words(self, machine, prep_round, main_dense, heights, pv, max_rows=3, cap_words=1 << 22):
        """sp1b200_debug_constraints: the report words (include/sp1b200.h)"""
        H = (C.c_uint64 * len(heights))(*heights)
        pv = np.ascontiguousarray(pv, dtype=np.uint32)
        return self._debug_call(self.L.sp1b200_debug_constraints, (machine, prep_round, _ptr(main_dense), H, _ptr(pv), C.c_uint32(pv.size),
                                                                  C.c_uint32(max_rows)), cap_words)

    def debug_interactions_words(self, machine, prep_round, main_dense, heights, max_keys=16, cap_words=1 << 22):
        """sp1b200_debug_interactions: the report words (include/sp1b200.h)"""
        H = (C.c_uint64 * len(heights))(*heights)
        return self._debug_call(self.L.sp1b200_debug_interactions, (machine, prep_round, _ptr(main_dense), H, C.c_uint32(max_keys)), cap_words)

    def debug_constraints(self, machine, prep_round, main_dense, heights, pv, max_rows=3, cap_words=1 << 22):
        """-> {chip: {"n_failing_rows": n, "rows": {row: [failed constraint indices]}}} (empty when every constraint holds)"""
        return parse_constraint_report(self.debug_constraints_words(machine, prep_round, main_dense, heights, pv, max_rows, cap_words))

    def debug_interactions(self, machine, prep_round, main_dense, heights, max_keys=16, cap_words=1 << 22):
        """-> {"n_unbalanced": n, "keys": [{"kind", "values", "net", "first": (chip, interaction, row), "chips": {chip: net}}]}"""
        return parse_interaction_report(self.debug_interactions_words(machine, prep_round, main_dense, heights, max_keys, cap_words))

    def setup_and_prove_shard(self, machine, prep_dense, prep_rows, prep_cols, vk_tail, main_dense, heights, names, pv, challenger_state,
                              replay=None, cap_words=1 << 24):
        """AirProver::setup_and_prove_shard: -> (prep_commit[8], prep_round handle, proof words); challenger_state = the state BEFORE
        the verifying key is observed, updated in place"""
        n = len(heights)
        H = (C.c_uint64 * n)(*heights)
        NM = (C.c_char_p * n)(*[s.encode() for s in names])
        npz = len(prep_rows)
        R = (C.c_uint64 * max(1, npz))(*prep_rows)
        Cc = (C.c_uint64 * max(1, npz))(*prep_cols)
        pv = np.ascontiguousarray(pv, dtype=np.uint32)
        tail = np.ascontiguousarray(vk_tail, dtype=np.uint32)
        out = np.empty(cap_words, np.uint32)
        nw = C.c_uint64()
        pc = np.zeros(8, np.uint32)
        h = C.c_void_p()
        rw = None if replay is None else np.ascontiguousarray(replay, dtype=np.uint32)
        self._chk(self.L.sp1b200_setup_and_prove_shard(self.ctx, machine, _ptr(prep_dense), C.c_uint32(npz), R, Cc, _ptr(tail), C.c_uint32(tail.size),
                                                       _ptr(main_dense), H, NM, _ptr(pv), C.c_uint32(pv.size), _ptr(rw), _ptr(challenger_state),
                                                       _ptr(pc), C.byref(h), _ptr(out), C.c_uint64(cap_words), C.byref(nw)))
        return pc, h, out[:nw.value].copy()

    def program_vk_tail(self, pc_start_abs, mem_addrs, mem_words, page_idx=None, page_prot=None, enable_untrusted_programs=0):
        """MachineProgram::pc_start + initial_global_cumulative_sum + untrusted_config of a program's memory image (and page image) ->
        the 24-word vk_tail (Montgomery words).  Addresses, words and page indices are 64-bit, protections 8-bit: numpy arrays or
        torch tensors on the host or the device (torch int64 / uint8)."""
        (a, w, pi, pp), n_mem, n_pages, _keep = _image_args(mem_addrs, mem_words, page_idx, page_prot)
        out = np.zeros(VK_TAIL_WORDS, np.uint32)
        self._chk(self.L.sp1b200_program_vk_tail(self.ctx, C.c_uint64(pc_start_abs), a, w, C.c_uint64(n_mem), pi, pp,
                                                 C.c_uint64(n_pages), C.c_int(enable_untrusted_programs), _ptr(out)))
        return out

    @staticmethod
    def _instructions(instrs):
        """INSTRUCTION_DTYPE numpy array, or a contiguous torch uint8 tensor of 24-byte records (host or device) -> (pointer, count, the
        array the pointer points into: keep it alive for the call)"""
        if hasattr(instrs, "data_ptr"):
            assert instrs.is_contiguous() and instrs.element_size() == 1 and instrs.numel() % INSTRUCTION_DTYPE.itemsize == 0
            return C.c_void_p(instrs.data_ptr() if instrs.numel() else None), instrs.numel() // INSTRUCTION_DTYPE.itemsize, instrs
        a = np.ascontiguousarray(instrs)
        assert a.dtype == INSTRUCTION_DTYPE, "pack the instructions with pack_instructions"
        return (C.c_void_p(a.ctypes.data) if a.size else None), a.size, a

    def program_preprocessed_traces(self, pc_base, instrs, out=None):
        """the Byte, Program and Range preprocessed tables of a program -> (dense words, shapes [(rows, cols)] x 3).  The words are the
        tables back to back, each column-major (the layout jagged_commit_dense takes).  out: a device tensor (uint32 / int32) to write
        into instead of a new host array; it is returned as the words."""
        p, n, _keep_instrs = self._instructions(instrs)
        R, Cc, nw = (C.c_uint64 * 3)(), (C.c_uint64 * 3)(), C.c_uint64()
        self._chk(self.L.sp1b200_program_preprocessed_traces(self.ctx, C.c_uint64(pc_base), p, C.c_uint64(n), None, C.c_uint64(0), R, Cc,
                                                             C.byref(nw)))
        if out is None:
            out = np.zeros(nw.value, np.uint32)
        cap = out.numel() if hasattr(out, "numel") else out.size
        self._chk(self.L.sp1b200_program_preprocessed_traces(self.ctx, C.c_uint64(pc_base), p, C.c_uint64(n), _ptr(out), C.c_uint64(cap),
                                                             R, Cc, C.byref(nw)))
        return out, [(int(R[t]), int(Cc[t])) for t in range(3)]

    def program_setup(self, pc_base, instrs, pc_start_abs, mem_addrs, mem_words, page_idx=None, page_prot=None, enable_untrusted_programs=0,
                      keep_codeword=True):
        """AirProver::setup(program): the preprocessed tables generated and committed on the device plus the verifying key ->
        dict(prep_rows [3], prep_commit [8], vk_tail [24], vk_digest [8], round = the committed round; free it with jagged_round_free).
        The image arguments are those of program_vk_tail."""
        p, n, _keep_instrs = self._instructions(instrs)
        (a, w, pi, pp), n_mem, n_pages, _keep = _image_args(mem_addrs, mem_words, page_idx, page_prot)
        rows = (C.c_uint64 * 3)()
        commit, tail, digest = np.zeros(8, np.uint32), np.zeros(VK_TAIL_WORDS, np.uint32), np.zeros(8, np.uint32)
        h = C.c_void_p()
        self._chk(self.L.sp1b200_program_setup(self.ctx, C.c_uint64(pc_base), p, C.c_uint64(n), C.c_uint64(pc_start_abs), a, w,
                                               C.c_uint64(n_mem), pi, pp, C.c_uint64(n_pages), C.c_int(enable_untrusted_programs),
                                               C.c_int(int(keep_codeword)), rows, _ptr(commit), _ptr(tail), _ptr(digest), C.byref(h)))
        return dict(prep_rows=[int(rows[t]) for t in range(3)], prep_commit=commit, vk_tail=tail, vk_digest=digest, round=h)

    @staticmethod
    def _records(recs, dtype):
        """a contiguous numpy array of `dtype`, or a contiguous torch uint8 tensor of such records (host or device) -> (pointer, count, the
        object the pointer points into: keep it alive for the call)"""
        if recs is None:
            return None, 0, None
        if hasattr(recs, "data_ptr"):
            assert recs.is_contiguous() and recs.element_size() == 1 and recs.numel() % dtype.itemsize == 0
            return C.c_void_p(recs.data_ptr() if recs.numel() else None), recs.numel() // dtype.itemsize, recs
        a = np.ascontiguousarray(recs)
        assert a.dtype == dtype, f"pack the records as {dtype}"
        return (C.c_void_p(a.ctypes.data) if a.size else None), a.size, a

    def lookup_traces(self, pc_base, n_instrs, lookups, pcs, pv=None, out=None):
        """the Byte, Program and Range main (multiplicity) traces of a shard from its byte lookups (BYTE_LOOKUP_DTYPE, pack_byte_lookups)
        and executed pcs (PC_COUNT_DTYPE, pack_pc_counts), numpy arrays or torch uint8 tensors of the records on the host or the device;
        pv: the shard's 187 public values (Montgomery words) to add the public-value lookups, or None.
        out: None -> three new host arrays [6, 2^16], [1, h], [1, 2^17]; or three uint32 / int32 buffers (numpy arrays or device
        tensors, e.g. views at the chips' offsets of a dense main buffer) written in place and returned.  -> (byte, program, range)"""
        lp, nl, _keep_l = self._records(lookups, BYTE_LOOKUP_DTYPE)
        pp, npc, _keep_p = self._records(pcs, PC_COUNT_DTYPE)
        pvw = None if pv is None else np.ascontiguousarray(pv, dtype=np.uint32)
        rows = (C.c_uint64 * 3)()
        args = (C.c_uint64(pc_base), C.c_uint64(n_instrs), lp, C.c_uint64(nl), pp, C.c_uint64(npc), _ptr(pvw),
                C.c_uint32(0 if pvw is None else pvw.size))
        if out is None:
            self._chk(self.L.sp1b200_lookup_traces(self.ctx, *args, None, None, None, rows))
            out = tuple(np.zeros((c, int(rows[t])), np.uint32) for t, c in enumerate(MAIN_CHIP_COLS.values()))
        self._chk(self.L.sp1b200_lookup_traces(self.ctx, *args, _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), rows))
        return out

    def memory_traces(self, init, finalize, previous_init_addr, previous_finalize_addr, local, out=None):
        """the MemoryGlobalInit, MemoryGlobalFinalize and MemoryLocal main traces of a shard with their byte lookups and global interaction
        events, from its init and finalize events (MEMORY_EVENT_DTYPE, pack_memory_events; any order) and local events
        (MEMORY_LOCAL_EVENT_DTYPE, pack_memory_local_events; record.get_local_mem_events() order): numpy arrays or torch uint8 tensors of
        the records on the host or the device, None for none.
        out: None -> new host arrays; or five buffers written in place and returned: three uint32 / int32 traces (numpy arrays or device
        tensors, e.g. views at the chips' offsets of a dense main buffer), the lookups (BYTE_LOOKUP_DTYPE array or uint8 tensor) and the
        global events (GLOBAL_EVENT_DTYPE array or uint8 tensor).  -> (init [30, h], finalize [30, h], local [20, h], lookups, globals)"""
        ip, ni, _keep_i = self._records(init, MEMORY_EVENT_DTYPE)
        fp, nf, _keep_f = self._records(finalize, MEMORY_EVENT_DTYPE)
        lp, nl, _keep_l = self._records(local, MEMORY_LOCAL_EVENT_DTYPE)
        rows, n_lk, n_ge = (C.c_uint64 * 3)(), C.c_uint64(), C.c_uint64()
        args = (ip, C.c_uint64(ni), fp, C.c_uint64(nf), C.c_uint64(previous_init_addr), C.c_uint64(previous_finalize_addr), lp, C.c_uint64(nl))
        if out is None:
            self._chk(self.L.sp1b200_memory_traces(self.ctx, *args, None, None, None, None, None, rows, C.byref(n_lk), C.byref(n_ge)))
            out = tuple(np.zeros((c, int(rows[t])), np.uint32) for t, c in enumerate(MEMORY_CHIP_COLS.values())) + \
                (np.zeros(n_lk.value, BYTE_LOOKUP_DTYPE), np.zeros(n_ge.value, GLOBAL_EVENT_DTYPE))

        def rec_ptr(x):   # a record array or a uint8 tensor, written in place
            if hasattr(x, "data_ptr"):
                assert x.is_contiguous()
                return C.c_void_p(x.data_ptr() or None)
            assert x.flags["C_CONTIGUOUS"]
            return C.c_void_p(x.ctypes.data)
        self._chk(self.L.sp1b200_memory_traces(self.ctx, *args, _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), rec_ptr(out[3]), rec_ptr(out[4]),
                                               rows, C.byref(n_lk), C.byref(n_ge)))
        return out

    def pack_row_major(self, rows_any, shapes, d_dense_out):
        """tables back to back, each row-major [rows x cols] -> device buffer with each table column-major"""
        n = len(shapes)
        R = (C.c_uint64 * n)(*[int(r) for r, _ in shapes])
        Cc = (C.c_uint64 * n)(*[int(c) for _, c in shapes])
        self._chk(self.L.sp1b200_pack_row_major(self.ctx, _ptr(rows_any), C.c_uint32(n), R, Cc, _ptr(d_dense_out)))

    def upload_begin(self, host_array, slot):
        """async H2D of a (pinned) host array into upload slot 0/1 -> device pointer (int) to pass as main_dense"""
        d = C.c_void_p()
        n = host_array.numel() if hasattr(host_array, "numel") else host_array.size
        self._chk(self.L.sp1b200_upload_begin(self.ctx, _ptr(host_array), C.c_uint64(n), C.c_int(slot), C.byref(d)))
        return d.value

    def grind(self, state34, bits):
        st = np.ascontiguousarray(state34, dtype=np.uint32).copy()
        w = C.c_uint32()
        self._chk(self.L.sp1b200_grind(self.ctx, _ptr(st), C.c_uint32(bits), C.byref(w)))
        return int(w.value), st


def parse_constraint_report(w):
    """report words of sp1b200_debug_constraints -> {chip: {"n_failing_rows": n, "rows": {row: [constraint indices]}}}"""
    w = [int(x) for x in w]
    out, p = {}, 1
    for _ in range(w[0]):
        chip, n_fail, n_listed = w[p:p + 3]; p += 3
        rows = {}
        for _ in range(n_listed):
            row, n = w[p:p + 2]; p += 2
            rows[row] = w[p:p + n]; p += n
        out[chip] = {"n_failing_rows": n_fail, "rows": rows}
    assert p == len(w), "malformed constraint report"
    return out


def parse_interaction_report(w):
    """report words of sp1b200_debug_interactions -> {"n_unbalanced": n, "keys": [...]} (keys in order of first occurrence)"""
    w = [int(x) for x in w]
    keys, p = [], 3
    for _ in range(w[2]):
        kind, nv = w[p:p + 2]; p += 2
        vals = w[p:p + nv]; p += nv
        net, chip, inter, row, n_chips = w[p:p + 5]; p += 5
        chips = {w[p + 2 * i]: w[p + 2 * i + 1] for i in range(n_chips)}; p += 2 * n_chips
        keys.append({"kind": kind, "values": vals, "net": net, "first": (chip, inter, row), "chips": chips})
    assert p == len(w), "malformed interaction report"
    return {"n_unbalanced": w[0] | (w[1] << 32), "keys": keys}


def verdict_name(verdict):
    """the reason a verdict of verify_shard, verify_core_proof or verify_compressed names ("Accepted" for 0)"""
    return load().sp1b200_verdict_name(C.c_uint32(verdict)).decode()


class RecursionVks:
    """the recursion vk map of Lib.recursion_vks: root, key count and openings are host lookups"""

    def __init__(self, L, h, vk_verification):
        self.L, self.h, self.vk_verification = L, h, vk_verification

    def root(self):
        out = np.zeros(8, np.uint32)
        self.L.sp1b200_recursion_vks_root(self.h, _ptr(out))
        return out

    def num_keys(self):
        return int(self.L.sp1b200_recursion_vks_num_keys(self.h))

    def open(self, digest):
        """-> (index, path [height, 8]); a digest outside the map raises"""
        d = np.ascontiguousarray(digest, dtype=np.uint32)
        path = np.zeros((64, 8), np.uint32)
        idx, n = C.c_uint64(), C.c_uint32()
        err = self.L.sp1b200_recursion_vks_open(self.h, _ptr(d), C.byref(idx), _ptr(path), C.c_uint32(64), C.byref(n))
        if err:
            raise Sp1B200Error(err.decode())
        return int(idx.value), path[:n.value].copy()

    def close(self):
        if self.h:
            self.L.sp1b200_recursion_vks_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _host_call(fn, *args):
    err = fn(*args)
    if err:
        raise Sp1B200Error(err.decode())


def vk_hash(prep_commit, vk_tail):
    """MachineVerifyingKey::hash_koalabear (without mprotect) of prep_commit[8] + vk_tail[24] -> 8 words"""
    pc = np.ascontiguousarray(prep_commit, dtype=np.uint32)
    tail = np.ascontiguousarray(vk_tail, dtype=np.uint32)
    out = np.zeros(8, np.uint32)
    _host_call(load().sp1b200_vk_hash, _ptr(pc), _ptr(tail), C.c_uint32(tail.size), _ptr(out))
    return out


def digest_bytes32(digest):
    """koalabears_to_bn254 of a digest as 32 big-endian bytes (vk.bytes32())"""
    d = np.ascontiguousarray(digest, dtype=np.uint32)
    out = np.zeros(32, np.uint8)
    _host_call(load().sp1b200_digest_bytes32, _ptr(d), C.c_void_p(out.ctypes.data))
    return out.tobytes()


def recursion_pv_digest(pv):
    """recursion_public_values_digest of the 187 words of RecursionPublicValues -> 8 words"""
    p = np.ascontiguousarray(pv, dtype=np.uint32)
    assert p.size == PV_MAX_NUM
    out = np.zeros(8, np.uint32)
    _host_call(load().sp1b200_recursion_pv_digest, _ptr(p), _ptr(out))
    return out


class HostChallenger:
    """The library's host transcript object on the 34-word state (no GPU needed)."""

    def __init__(self, state=None):
        self.L = load()
        self.st = np.zeros(34, np.uint32)
        if state is not None:
            self.st[:] = state

    def clone(self):
        return HostChallenger(self.st.copy())

    def observe(self, vals):
        v = np.ascontiguousarray(np.atleast_1d(vals), dtype=np.uint32)
        self.L.sp1b200_challenger_observe(_ptr(self.st), _ptr(v), C.c_uint64(v.size))

    def sample(self, n=1):
        out = np.zeros(n, np.uint32)
        self.L.sp1b200_challenger_sample(_ptr(self.st), _ptr(out), C.c_uint64(n))
        return out

    def sample_bits(self, bits):
        return int(self.L.sp1b200_challenger_sample_bits(_ptr(self.st), C.c_uint32(bits)))

    def check_witness(self, bits, w):
        return bool(self.L.sp1b200_challenger_check_witness(_ptr(self.st), C.c_uint32(bits), C.c_uint32(w)))


# ---- ShardProof wire format (host only, no context): flat proof words <-> bincode(ShardProof) ---------------------------------------
def _wire_args(params, names, main_w, prep_w):
    p = dict(DEFAULT_CORE_PARAMS)
    p.update(params)
    n = len(names)
    return (Params(**p), C.c_uint32(n), (C.c_char_p * n)(*[s.encode() for s in names]), (C.c_uint32 * n)(*[int(x) for x in main_w]),
            (C.c_uint32 * n)(*[int(x) for x in prep_w]))


def shard_proof_to_bincode(words, names, heights, main_w, prep_w, **params):
    """flat words of prove_shard -> bytes of bincode(ShardProof) (crates/hypercube/src/verifier/proof.rs:47-61)"""
    L = load()
    P, n, NM, MW, PW = _wire_args(params, names, main_w, prep_w)
    H = (C.c_uint64 * len(names))(*[int(h) for h in heights])
    w = np.ascontiguousarray(words, dtype=np.uint32)
    nb = C.c_uint64()
    err = L.sp1b200_shard_proof_to_bincode(C.byref(P), n, NM, H, MW, PW, _ptr(w), C.c_uint64(w.size), None, C.c_uint64(0), C.byref(nb))
    if err:
        raise Sp1B200Error(err.decode())
    out = np.empty(nb.value, np.uint8)
    err = L.sp1b200_shard_proof_to_bincode(C.byref(P), n, NM, H, MW, PW, _ptr(w), C.c_uint64(w.size), C.c_void_p(out.ctypes.data),
                                           C.c_uint64(out.size), C.byref(nb))
    if err:
        raise Sp1B200Error(err.decode())
    return out.tobytes()


def shard_proof_from_bincode(data, names, main_w, prep_w, **params):
    """bytes of bincode(ShardProof) -> (flat words, chip heights)"""
    L = load()
    P, n, NM, MW, PW = _wire_args(params, names, main_w, prep_w)
    buf = np.frombuffer(bytes(data), np.uint8)
    H = (C.c_uint64 * max(1, len(names)))()
    nw = C.c_uint64()
    err = L.sp1b200_shard_proof_from_bincode(C.byref(P), n, NM, MW, PW, C.c_void_p(buf.ctypes.data), C.c_uint64(buf.size), H, None,
                                             C.c_uint64(0), C.byref(nw))
    if err:
        raise Sp1B200Error(err.decode())
    out = np.empty(nw.value, np.uint32)
    err = L.sp1b200_shard_proof_from_bincode(C.byref(P), n, NM, MW, PW, C.c_void_p(buf.ctypes.data), C.c_uint64(buf.size), H, _ptr(out),
                                             C.c_uint64(out.size), C.byref(nw))
    if err:
        raise Sp1B200Error(err.decode())
    return out, [int(H[i]) for i in range(len(names))]
