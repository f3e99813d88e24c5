"""GPU tests of the program setup from the instruction list (sp1b200_program_preprocessed_traces, sp1b200_program_setup): the device tables
equal the NumPy restatement (tests/program_ref.py) word for word; the key's commitment is the jagged commitment of the restated tables, its
tail program_vk_tail's and its digest vk_hash's; a core chain proven with the returned round over a machine with the real Byte / Program /
Range preprocessed widths and heights verifies under the returned key and not under the key of a program one bit away; every input bit
moves the digest; malformed programs are errors that name the instruction and leave the context usable; a poisoned pool gives the same
key."""
import ctypes as C

import numpy as np
import pytest

from tests import core_chain as CC
from tests import gpu_prove as GP
from tests import machines as M
from tests import oracle_lib as O
from tests import program_ref as PR
from tests import septic as S
from tests.provers import specs_machine

pytestmark = pytest.mark.gpu

V_INVALID_SHARD_PROOF = 45


def _lib(**params):
    from sp1_b200 import Lib
    return Lib(0, **params)


def _program(n, seed):
    """n random instructions and a pc_base that keeps every pc below 2^48 -> (pc_base, records)"""
    from sp1_b200.lib import MAX_OPCODE, pack_instructions
    rng = np.random.default_rng(seed)
    u64 = lambda: rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
    instrs = pack_instructions(rng.integers(0, MAX_OPCODE + 1, n), rng.integers(0, 32, n), u64(), u64(), rng.integers(0, 2, n),
                               rng.integers(0, 2, n))
    pc_base = int(rng.integers(0, (1 << 48) - 4 * n)) & ~3
    return pc_base, instrs


def _image(n, seed):
    rng = np.random.default_rng(seed)
    return rng.choice(1 << 45, n, replace=False).astype(np.uint64) << np.uint64(3), rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)


def _dev(instrs):
    import torch
    return torch.from_numpy(instrs.view(np.uint8).copy()).cuda()


@pytest.mark.parametrize("n", [1, 15, 16, 17, 31, 32, 33, 1000, 1 << 20])
def test_tables_match_the_restatement(n):
    lib = _lib()
    pc_base, instrs = _program(n, 100 + n)
    want, shapes = PR.dense(pc_base, instrs)
    got, got_shapes = lib.program_preprocessed_traces(pc_base, instrs)
    assert got_shapes == [tuple(s) for s in shapes]
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"first differing words {bad[:8]} of {want.size}"
    got_d, _ = lib.program_preprocessed_traces(pc_base, _dev(instrs))   # instructions in device memory
    assert (got_d == want).all()
    lib.close()


def test_tables_into_device_memory():
    import torch
    lib = _lib()
    pc_base, instrs = _program(1000, 7)
    want, _ = PR.dense(pc_base, instrs)
    out = torch.zeros(want.size, dtype=torch.int32, device="cuda")
    lib.program_preprocessed_traces(pc_base, _dev(instrs), out=out)
    assert (out.cpu().numpy().view(np.uint32) == want).all()
    lib.close()


@pytest.mark.parametrize("n", [1, 33, 1000])
def test_key_is_the_commitment_of_the_restated_tables(n):
    from sp1_b200 import lib as B
    lib = _lib()
    pc_base, instrs = _program(n, 200 + n)
    addrs, words = _image(500, 201)
    key = lib.program_setup(pc_base, instrs, pc_base, addrs, words)
    dense, shapes = PR.dense(pc_base, instrs)
    commit, h = lib.jagged_commit_dense(dense, [s[0] for s in shapes], [s[1] for s in shapes])
    lib.jagged_round_free(h)
    assert key["prep_rows"] == [s[0] for s in shapes]
    assert (key["prep_commit"] == commit).all()
    assert (key["vk_tail"] == lib.program_vk_tail(pc_base, addrs, words)).all()
    assert (key["vk_digest"] == B.vk_hash(commit, key["vk_tail"])).all()
    key_d = lib.program_setup(pc_base, _dev(instrs), pc_base, addrs, words)   # instructions in device memory
    assert (key_d["prep_commit"] == commit).all() and (key_d["vk_digest"] == key["vk_digest"]).all()
    lib.jagged_round_free(key["round"]); lib.jagged_round_free(key_d["round"])
    lib.close()


# the core machine's chips with preprocessed columns at their real widths (Byte 7, Program 16, Range 2) and one chip without
NAMES = ["Byte", "Cpu", "Program", "Range"]


def _chips(program_rows):
    return [M.Chip(1 << 16, 1, True, extra_prep=6), M.Chip(1 << 12, 2, False), M.Chip(program_rows, 1, True, extra_prep=15),
            M.Chip(1 << 17, 1, True, extra_prep=1)]


def _mains(chips, tables, seed, pv0):
    """synthetic main traces whose preprocessed constraint h = g * a reads the real tables' first column as g"""
    mains, _ = M.traces(chips, seed, pv0)
    tabs = iter(tables)
    for c, m in zip(chips, mains):
        if c.wp:
            g = next(tabs)[:, 0].astype(np.uint64)
            a = O.from_monty(m[0]).astype(np.uint64)
            m[6 * c.g] = O.to_monty(g * a % np.uint64(O.P))
    return mains


def test_core_chain_verifies_under_the_key_of_its_program():
    """a 3-shard chain proven with the round program_setup returned verifies under the returned key, with every shard verifier ending in
    its prover's state; under the key of the program with one op_c bit changed the shards do not verify"""
    from sp1_b200 import synth_air as SA
    from sp1_b200.lib import HostChallenger
    n = 1000
    pc_base, instrs = _program(n, 300)
    pvs, tail0 = CC.chain(3, 301)
    pc_abs = tail0[0] | (tail0[1] << 16) | (tail0[2] << 32)
    addrs, words = _image(2000, 302)
    lib = _lib(log_stacking_height=16, max_log_row_count=17, **M.SMALL)
    key = lib.program_setup(pc_base, instrs, pc_abs, addrs, words)
    chips = _chips(key["prep_rows"][1])
    blob, heights, _, _ = specs_machine(chips)
    assert heights == [1 << 16, 1 << 12, key["prep_rows"][1], 1 << 17]
    assert [SA.synth_chip(c.g, c.wp, extra_prep=c.extra_prep)[2] for c in chips] == [7, 0, 16, 2]
    mach = lib.machine_create(blob)
    # the last shard's global cumulative sum absorbs the change of the key's initial sum (as in tests/test_gpu_setup.py)
    initial0, initial = (tail0[3:10], tail0[10:17]), S.words_pt(key["vk_tail"][3:17])
    g = CC.getf(pvs[-1], "global_cumulative_sum")
    d = S.curve_add(S.curve_add((g[:7], g[7:]), initial0), S.curve_neg(initial))
    CC.setf(pvs[-1], "global_cumulative_sum", list(d[0]) + list(d[1]))
    tables = [t for _, t in PR.tables(pc_base, instrs)]
    words_, finals = [], []
    for pv in pvs:
        hc = HostChallenger(); hc.observe(key["prep_commit"]); hc.observe(key["vk_tail"])
        st = hc.st.copy()
        mains = _mains(chips, tables, 303, CC.pv0_of(pv))
        words_.append(GP.prove(lib, mach, key["round"], mains, heights, NAMES, O.to_monty(np.array(pv)), st))
        finals.append(st)
    v, shard, sv, fin = lib.verify_core_proof(mach, key["prep_commit"], key["vk_tail"], [heights] * 3, NAMES, words_)
    assert (v, shard, sv) == (0, 0, 0)
    assert (fin == np.stack(finals)).all()
    changed = instrs.copy(); changed["op_c"][417] ^= np.uint64(1 << 29)
    bad = lib.program_setup(pc_base, changed, pc_abs, addrs, words)
    assert not (bad["prep_commit"] == key["prep_commit"]).all() and (bad["vk_tail"] == key["vk_tail"]).all()
    v, shard, _, _ = lib.verify_core_proof(mach, bad["prep_commit"], bad["vk_tail"], [heights] * 3, NAMES, words_)
    assert (v, shard) == (V_INVALID_SHARD_PROOF, 0)
    for k in (key, bad):
        lib.jagged_round_free(k["round"])
    lib.machine_free(mach)
    lib.close()


def test_every_input_bit_moves_the_digest():
    from sp1_b200.lib import pack_instructions
    lib = _lib()
    pc_base, instrs = _program(32, 400)
    instrs["opcode"][5] = 10
    addrs, words = _image(64, 401)

    def digest(pcb, ins):
        k = lib.program_setup(pcb, ins, 0x1000, addrs, words)
        lib.jagged_round_free(k["round"])
        return tuple(int(v) for v in k["vk_digest"])
    seen = {digest(pc_base, instrs)}
    for field, i, flip in (("opcode", 5, 1), ("op_a", 9, 1 << 4), ("op_b", 0, 1 << 63), ("op_c", 31, 1 << 17), ("imm_b", 12, 1),
                           ("imm_c", 20, 1)):
        ch = instrs.copy()
        ch[field][i] ^= ch.dtype[field].type(flip)
        seen.add(digest(pc_base, ch))
    seen.add(digest(pc_base ^ 4, instrs))
    extra = np.concatenate([instrs, pack_instructions(0, 0, 0, 0, 0, 0)])   # n = 32 -> 33: the Program table grows to 64 rows
    seen.add(digest(pc_base, extra))
    assert len(seen) == 9
    lib.close()


def test_errors_name_the_instruction_and_leave_the_context_usable():
    from sp1_b200.lib import Sp1B200Error
    lib = _lib(max_log_row_count=17)
    pc_base, instrs = _program(100, 500)
    pc_base &= (1 << 40) - 1
    addrs, words = _image(300, 501)
    want = lib.program_setup(pc_base, instrs, 0x2000, addrs, words)
    lib.jagged_round_free(want["round"])

    def same_key():
        k = lib.program_setup(pc_base, instrs, 0x2000, addrs, words)
        lib.jagged_round_free(k["round"])
        assert (k["vk_digest"] == want["vk_digest"]).all() and (k["prep_commit"] == want["prep_commit"]).all()

    def bad(field, i, value):
        ch = instrs.copy(); ch[field][i] = value
        return ch
    dup = addrs.copy(); dup[200] = dup[3]
    cases = [((pc_base, instrs[:0], 0x2000, addrs, words), "empty program"),
             ((pc_base, bad("opcode", 77, 53), 0x2000, addrs, words), "instruction 77 has opcode 53"),
             ((pc_base, bad("imm_b", 41, 2), 0x2000, addrs, words), "instruction 41 has imm_b = 2"),
             ((pc_base, bad("imm_c", 0, 255), 0x2000, addrs, words), "instruction 0 has imm_c = 255"),
             (((1 << 48) - 4 * 60, instrs, 0x2000, addrs, words), "instruction 60 has pc"),
             ((pc_base, np.resize(instrs, (1 << 17) + 1), 0x2000, addrs, words), "rows > 2\\^17"),
             ((pc_base, instrs, 0x2000, dup, words), f"duplicate memory address 0x{int(addrs[3]):x}")]
    for args, msg in cases:
        with pytest.raises(Sp1B200Error, match=msg):
            lib.program_setup(*args)
        same_key()
    with pytest.raises(Sp1B200Error, match="instruction 77 has opcode 53"):
        lib.program_preprocessed_traces(pc_base, bad("opcode", 77, 53))
    same_key()
    nw, R, Cc = C.c_uint64(), (C.c_uint64 * 3)(), (C.c_uint64 * 3)()
    small = np.zeros(16, np.uint32)
    e = lib.L.sp1b200_program_preprocessed_traces(lib.ctx, C.c_uint64(pc_base), C.c_void_p(instrs.ctypes.data), C.c_uint64(100),
                                                  C.c_void_p(small.ctypes.data), C.c_uint64(16), R, Cc, C.byref(nw))
    assert e and b"capacity 16" in e and nw.value == 7 * (1 << 16) + 16 * 128 + 2 * (1 << 17)
    same_key()
    lib.close()


def test_poisoned_pool_gives_the_same_key():
    """every block of the context's pool holds a non-zero pattern before the call (a freed pool keeps its blocks)"""
    lib = _lib()
    pc_base, instrs = _program(5000, 600)
    addrs, words = _image(4096, 601)
    want = lib.program_setup(pc_base, instrs, 0x8000, addrs, words)
    lib.jagged_round_free(want["round"])
    lib.close()
    lib = _lib()
    blocks = []
    for size in [256 << k for k in range(0, 18)] * 2 + [64 << 20, 64 << 20]:
        p = C.c_void_p()
        lib._chk(lib.L.sp1b200_malloc(lib.ctx, C.c_size_t(size), C.byref(p)))
        fill = np.full(size // 4, 0x7effffff, np.uint32)
        lib._chk(lib.L.sp1b200_memcpy_h2d(lib.ctx, p, C.c_void_p(fill.ctypes.data), C.c_size_t(size)))
        lib.sync()
        blocks.append(p)
    for p in blocks:
        lib._chk(lib.L.sp1b200_free(lib.ctx, p))
    lib.sync()
    got = lib.program_setup(pc_base, instrs, 0x8000, addrs, words)
    lib.jagged_round_free(got["round"])
    for k in ("prep_commit", "vk_tail", "vk_digest"):
        assert (got[k] == want[k]).all(), k
    lib.close()
