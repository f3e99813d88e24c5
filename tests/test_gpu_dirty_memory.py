"""Proving and verifying on dirty device memory, word for word against the oracle.

A long-lived context (the benchmark's, the AirProver shim's) hands every call the blocks the previous calls freed: its pool keeps
freed memory with the previous data in it.  A kernel that reads a word of a pooled buffer before writing it, or a driver that forgets
to zero a buffer it accumulates into, gives a right answer on the fresh memory of a new context and a wrong one in production.

1. Poisoned pool: before every entry-point call the context's pool is filled with a known pattern (two random patterns of canonical
   field words and the non-canonical 0xFFFFFFFF), so that every pooled buffer a call allocates starts out dirty.  A canary checks that
   the pattern does reach fresh allocations.
2. One context across changing shapes: large, small, preprocessed-free and 96-chip shards in turn, fed from host memory, device memory
   and an upload slot a larger shard filled first; a verification and a capacity error in between.
3. Guard bands: every device pointer the C ABI takes is a view 256 B into a tensor whose words around the view hold a random pattern;
   those words must be unchanged after the call."""
import ctypes as C

import numpy as np
import pytest

from tests import debug_oracle_lib as DO
from tests import gpu_prove as GP
from tests import machines as M
from tests import oracle_lib as O
from tests import recursion_ref as RR
from tests.machines import ORACLE_LACKS, SMALL, Chip
from tests.provers import Core, Rec, specs_machine

pytestmark = pytest.mark.gpu

P = O.P
PERIOD = 64          # words of one poison pattern: 256 B, the pool's allocation alignment, so a word's value depends on its address only
G = 64               # guard band words on each side of a caller buffer (256 B: a view keeps the alignment of a fresh allocation)


def _patterns():
    rng = np.random.default_rng(7001)
    return {"random-a": O.rand_field(rng, PERIOD), "random-b": O.rand_field(rng, PERIOD),
            "ones": np.full(PERIOD, 0xFFFFFFFF, np.uint32)}


PATTERNS = _patterns()


# ---- the poisoned pool ------------------------------------------------------------------------------------------------------------------
def _ladder(cap):
    """block sizes: every size class below 2 MiB (256 B, 1 KiB, ... 1 MiB) fills 512 KiB in blocks of its size, so that the pool is dirty
    whether or not it splits a freed large block for a small request; then two blocks of each size 2 MiB, 8 MiB, 32 MiB, ... up to cap,
    and one block of cap itself when cap is not one of those sizes"""
    sizes, s = [], 256
    while s < (2 << 20):
        sizes += [s] * max(1, (512 << 10) // s)
        s *= 4
    s = 2 << 20
    while s <= cap:
        sizes += [s, s]
        s *= 4
    if cap not in sizes:
        sizes.append(cap)
    return sizes[::-1]


class _Host:
    """a pinned host buffer holding the pattern repeated, PERIOD words longer than the largest copy so any phase can be copied"""
    CHUNK = 4 << 20

    def __init__(self, pattern):
        import torch
        words = np.resize(pattern, self.CHUNK // 4 + PERIOD)
        self.t = torch.from_numpy(words.view(np.int32)).pin_memory()
        self.addr = self.t.data_ptr()


_hosts = {}
_cuda = []


def _pool_stats(lib, ptr):
    """(reserved bytes, peak used bytes since the last reset) of the pool the block at ptr came from, and reset the peak (driver API:
    the context's pool handle from the pointer, then the pool's attributes)"""
    if not _cuda:
        _cuda.append(C.CDLL("libcuda.so.1"))
    cu = _cuda[0]
    pool = C.c_void_p()
    assert cu.cuPointerGetAttribute(C.byref(pool), C.c_int(17), C.c_uint64(ptr)) == 0 and pool.value    # CU_POINTER_ATTRIBUTE_MEMPOOL_HANDLE
    reserved, peak, zero = C.c_uint64(), C.c_uint64(), C.c_uint64(0)
    assert cu.cuMemPoolGetAttribute(pool, C.c_int(5), C.byref(reserved)) == 0                           # CU_MEMPOOL_ATTR_RESERVED_MEM_CURRENT
    assert cu.cuMemPoolGetAttribute(pool, C.c_int(8), C.byref(peak)) == 0                               # CU_MEMPOOL_ATTR_USED_MEM_HIGH
    assert cu.cuMemPoolSetAttribute(pool, C.c_int(8), C.byref(zero)) == 0
    return reserved.value, peak.value


def _dev_words(lib, ptr, n):
    out = np.empty(n, np.uint32)
    lib._chk(lib.L.sp1b200_memcpy_d2h(lib.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(ptr), C.c_size_t(4 * n)))
    return out


def _malloc(lib, size):
    p = C.c_void_p()
    lib._chk(lib.L.sp1b200_malloc(lib.ctx, C.c_size_t(size), C.byref(p)))
    return p.value


def covered(lib, may_grow=0):
    """the calls since the last poison took every block from memory the pool held at that poison: its reserved size has grown by at most
    may_grow bytes (0: not at all).  -> the peak pooled footprint of those calls"""
    if getattr(lib, "_poisoned", None) is None:
        return None
    lib.sync()
    p = _malloc(lib, 256)
    reserved, peak = _pool_stats(lib, p)
    lib._chk(lib.L.sp1b200_free(lib.ctx, C.c_void_p(p)))
    name, before, cap = lib._poisoned
    lib._poisoned = None
    assert before <= reserved <= before + may_grow, (f"pattern {name}: the pool grew from {before} to {reserved} bytes (peak use {peak} bytes): part of the "
                                f"call ran on memory that was never poisoned; raise the cap of {cap} bytes")
    print(f"pooled peak {peak} bytes inside {before} poisoned bytes")   # shown with pytest -rP
    return peak


def poison(lib, name, cap=32 << 20):
    """fill the context's pool with the pattern `name`: allocate the ladder of blocks, fill each through sp1b200_memcpy_h2d (the word at
    device address a gets pattern[(a / 4) % PERIOD]), free them all, on the context's stream.  Then a canary: blocks of sizes the library
    allocates (a job table, an eq table, a codeword, half the largest block) must come back holding the pattern.  First checks that the
    calls since the previous poison stayed inside the memory it poisoned (covered)."""
    covered(lib)
    pattern = PATTERNS[name]
    if name not in _hosts:
        _hosts[name] = _Host(pattern)
    host = _hosts[name]
    L, ctx = lib.L, lib.ctx
    blocks = []
    for size in _ladder(cap):
        p = _malloc(lib, size)
        blocks.append(p)
        for off in range(0, size, _Host.CHUNK):
            n = min(_Host.CHUNK, size - off)
            phase = ((p + off) // 4) % PERIOD
            lib._chk(L.sp1b200_memcpy_h2d(ctx, C.c_void_p(p + off), C.c_void_p(host.addr + 4 * phase), C.c_size_t(n)))
    for p in blocks:
        lib._chk(L.sp1b200_free(ctx, C.c_void_p(p)))
    canary = [(_malloc(lib, size), size) for size in (37 * 88, (16 << 12) + 64, 4 << 20, cap // 2)]
    for p, size in canary:
        got = _dev_words(lib, p, size // 4)
        want = pattern[(p // 4 + np.arange(size // 4)) % PERIOD]
        assert (got == want).all(), f"pattern {name}: a fresh {size}-byte block does not hold the poison ({(got != want).sum()} words differ)"
    for p, _ in canary:
        lib._chk(L.sp1b200_free(ctx, C.c_void_p(p)))
    lib.sync()
    p = _malloc(lib, 256)
    reserved, _ = _pool_stats(lib, p)
    lib._chk(L.sp1b200_free(ctx, C.c_void_p(p)))
    lib.sync()
    lib._poisoned = (name, reserved, cap)


def poisoned_words(n, name="random-a"):
    """n words of a poison pattern: the starting contents of a caller's output buffer"""
    return np.resize(PATTERNS[name], n)


def _lib(**params):
    from sp1_b200 import Lib
    return Lib(0, **params)


# ---- 1. kernels ---------------------------------------------------------------------------------------------------------------------
RS_SHAPES = [(0, 1, 2), (1, 3, 2), (5, 4, 2), (9, 3, 2), (12, 3, 2), (14, 5, 2), (12, 2, 3), (15, 1, 1),
             (11, 3, 2), (19, 1, 2), (18, 2, 2), (18, 1, 1), (21, 1, 2), (21, 2, 1)]


def test_kernels_on_a_poisoned_pool():
    """rs_encode on generic shapes and both fast step-A / step-B paths, merkle_commit with its layers, poseidon2_permute, grind"""
    import torch
    rng = np.random.default_rng(7100)
    lib = _lib()
    rs = []
    for log_h, ncols, lb in RS_SHAPES:
        msg = O.rand_field(rng, (ncols, 1 << log_h))
        rs.append((msg, lb, O.rs_encode(msg, lb)))
    width, log_h = 13, 9
    mat = O.rand_field(rng, (width, 1 << log_h))
    oroot, ocommit, olayers = O.merkle_commit(mat, want_layers=True)
    states = O.rand_field(rng, (1000, 16))
    operm = np.stack([O.permute(s) for s in states])
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 9)); ch.sample(2)
    och = ch.clone(); ow = och.grind(12)
    for name in PATTERNS:
        for msg, lb, want in rs:
            out = np.zeros(want.shape, np.uint32)
            poison(lib, name, cap=128 << 20)
            lib.rs_encode(msg, out, msg.shape[0], int(np.log2(msg.shape[1])), lb)
            assert (out == want).all(), f"{name}: rs_encode {msg.shape} blowup {lb}"
        layers = torch.from_numpy(poisoned_words(((2 << log_h) - 1) * 8, name).view(np.int32)).cuda()
        torch.cuda.synchronize()
        poison(lib, name)
        root, commit = lib.merkle_commit(mat, width, log_h, d_layers=layers)
        lib.sync()
        assert (root == oroot).all() and (commit == ocommit).all(), f"{name}: merkle_commit"
        assert (layers.cpu().numpy().view(np.uint32).reshape(-1, 8) == olayers).all(), f"{name}: merkle layers"
        poison(lib, name)
        st = states.copy()
        lib.poseidon2_permute(st)
        assert (st == operm).all(), f"{name}: poseidon2_permute"
        poison(lib, name)
        w, gst = lib.grind(ch.st, 12)
        assert w == ow and (gst == och.st).all(), f"{name}: grind"
    covered(lib)
    lib.close()


# ---- 1. jagged PCS ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shapes,log_stack,mlr", [
    ([[(3, 2), (7, 1)], [(16, 2), (0, 4), (9, 3)]], 3, 4),
    ([[(4096, 3), (96, 17), (0, 5)], [(8192, 9), (2048 + 32, 40), (0, 3), (64, 13), (8192, 2)]], 12, 13),
])
def test_jagged_pcs_on_a_poisoned_pool(shapes, log_stack, mlr):
    """the check_jagged flow, the pool poisoned before every commit, the column claims and the proof"""
    for name in PATTERNS:
        GP.check_jagged(shapes, log_stack, mlr, seed=7200 + mlr, between=lambda lib: poison(lib, name))


# ---- 1. LogUp-GKR and zerocheck -------------------------------------------------------------------------------------------------------
PHASE_SPECS = [
    # every register-file tier of the zerocheck kernels next to a flat chip, an absent chip
    ([Chip(512, 6, False, deep=True), Chip(300, 14, True, deep=True), Chip(1024, 28, False, deep=True), Chip(96, 40, False, deep=True),
      (2048, 3, True), (0, 1, False)], 12),
    # the global-memory register file (~1000 registers), heights on both sides of the "pieces" threshold
    ([Chip(192, 250, False, deep=True), Chip(64, 500, True, deep=True), (8192, 3, True), Chip(96, 1000, False, deep=True),
      Chip(6000, 300, False, deep=True)], 13),
]
PHASE_CAPS = [128 << 20, 192 << 20]
# unpoisoned growth the zerocheck call may cause: the second case's global register-file workspace (every global-tier piece job's
# blocks x 1000 registers x 3 nodes x 128 threads x 16 B, ~1.0 GiB) is more than a shared GPU should be asked to poison; every other
# buffer of the call, and every buffer of the LogUp-GKR call, is poisoned
PHASE_ZC_GROWTH = [0, 1152 << 20]


def _to_device(arrays):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda() if a is not None else None for a in arrays]


@pytest.mark.parametrize("case", range(len(PHASE_SPECS)))
def test_logup_gkr_and_zerocheck_on_a_poisoned_pool(case):
    import torch
    spec, mlr = PHASE_SPECS[case]
    rng = np.random.default_rng(7300 + case)
    blob, heights, mains, preps, pv, _ = M.spec_machine(rng, spec)
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 4))
    och = ch.clone()
    ogkr = O.gkr_prove_verify(blob, heights, mains, preps, mlr, och, gkr_pow_bits=4)
    gp, st0, openings, ozc, ozst = M.oracle_zerocheck(rng, blob, heights, mains, preps, pv, mlr)
    lib = _lib(max_log_row_count=mlr, log_stacking_height=min(mlr, 21), gkr_pow_bits=4)
    mach = lib.machine_create(blob)
    d_mains, d_preps = _to_device(mains), _to_device(preps)
    torch.cuda.synchronize()
    for name in PATTERNS:
        poison(lib, name, PHASE_CAPS[case])
        st = ch.st.copy()
        words = lib.logup_gkr(mach, heights, d_mains, d_preps, st)
        assert words.size == ogkr.size and (words == ogkr).all(), M.first_diff(words, ogkr, f"{name}: LogUp-GKR proof")
        assert (st == och.st).all(), f"{name}: LogUp-GKR final challenger"
        poison(lib, name, PHASE_CAPS[case])
        words, st = M.product_zerocheck(lib, mach, heights, mains, preps, pv, gp, st0, openings, device=(d_mains, d_preps))
        covered(lib, PHASE_ZC_GROWTH[case])
        assert words.size == ozc.size and (words == ozc).all(), M.first_diff(words, ozc, f"{name}: zerocheck proof")
        assert (st == ozst).all(), f"{name}: zerocheck final challenger"
    lib.machine_free(mach)
    lib.close()


# ---- 1. whole shards --------------------------------------------------------------------------------------------------------------------
def _shard_case(case):
    """-> ((blob, heights, mains, preps, pv, names), log_stack, mlr, pool cap)"""
    if case.startswith("spec"):
        spec, ls, mlr = M.SHARD_SPECS[int(case[4:])]
        return M.spec_machine(np.random.default_rng(7400 + mlr), spec, names="Chip{:02d}"), ls, mlr, 32 << 20
    if case == "96-chip":
        return M.spec_machine(np.random.default_rng(7410), M.full_table_spec(96, 7411, absent=True)), 5, 5, 32 << 20
    return M.workload_machine(case, seed=7420, max_log_rows=12, scale=0.25), 10, 12, 128 << 20


def _oracle_shard(inp, log_stack, mlr, seed):
    blob, heights, mains, preps, pv, names = inp
    ch = O.Challenger(); ch.observe(O.rand_field(np.random.default_rng(seed), 9))
    och = ch.clone()
    opc, owords = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, och, **SMALL)
    return ch.st.copy(), opc, owords, och.st.copy()


@pytest.mark.parametrize("case", ["spec0", "spec1", "spec2", "tinyc", "tinyr", "96-chip"])
def test_prove_shard_on_a_poisoned_pool(case):
    inp, ls, mlr, cap = _shard_case(case)
    blob, heights, mains, preps, pv, names = inp
    st0, opc, owords, ost = _oracle_shard(inp, ls, mlr, 7430)
    lib = _lib(log_stacking_height=ls, max_log_row_count=mlr, **SMALL)
    mach = lib.machine_create(blob)
    for name in PATTERNS:
        poison(lib, name, cap)
        pc, prep_round = GP.commit_prep(lib, preps)
        assert (pc == opc).all(), f"{name}: preprocessed commitment"
        poison(lib, name, cap)
        st = st0.copy()
        words = GP.prove(lib, mach, prep_round, mains, heights, names, pv, st)
        assert words.size == owords.size and (words == owords).all(), f"{name}: " + M.shard_diff(words, owords)
        assert (st == ost).all(), f"{name}: final challenger"
        covered(lib)
        if prep_round is not None:
            lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()


# ---- 1. shard checks ----------------------------------------------------------------------------------------------------------------
DEBUG_CHIPS = [Chip(300, 14, True, deep=True), Chip(96, 14, False, 120, 0, 0, [12, 4, 9, 5]), Chip(0, 2, True, 18, 1, 2),
               Chip(33, 1, True, 9, 7, 35), Chip(700, 4, False, 36, 5, 0, [9] * 6)]


def test_debug_reports_on_a_poisoned_pool():
    """both reports on a clean trace and on one broken cell"""
    rng = np.random.default_rng(7500)
    blob, heights, mains, preps, pv, _ = M.spec_machine(rng, DEBUG_CHIPS)
    broken = [m.copy() for m in mains]
    broken[1][2, 7] = (int(broken[1][2, 7]) + 3) % P
    want = [(ms, DO.debug_constraints(blob, heights, ms, preps, pv).tolist(), DO.debug_interactions(blob, heights, ms, preps).tolist())
            for ms in (mains, broken)]
    assert want[0][1] == [0] and want[0][2] == [0, 0, 0] and want[1][1:] != want[0][1:]
    lib = _lib(max_log_row_count=10, log_stacking_height=10)
    mach = lib.machine_create(blob)
    for name in PATTERNS:
        poison(lib, name)
        pr = GP.commit_prep(lib, preps)[1]
        for ms, wc, wi in want:
            dense = M.dense_main(ms)
            poison(lib, name)
            assert lib.debug_constraints_words(mach, pr, dense, heights, pv).tolist() == wc, f"{name}: constraint report"
            poison(lib, name)
            assert lib.debug_interactions_words(mach, pr, dense, heights).tolist() == wi, f"{name}: interaction report"
        covered(lib)
        lib.jagged_round_free(pr)
    lib.machine_free(mach)
    lib.close()


# ---- 1. verifiers -------------------------------------------------------------------------------------------------------------------
def _sections(words):
    lens = [int(x) for x in words[1:6]]
    starts = np.cumsum([6] + lens[:-1])
    return [(int(s), int(s) + n) for s, n in zip(starts, lens)]


def _oracle_verdict(capfd, blob, heights, names, ls, mlr, start, pc, words):
    """the oracle's verify_shard -> "accept", "parse" or the name of its first failing check"""
    capfd.readouterr()
    v = O.Challenger(); v.st[:] = start
    r = O.verify_shard(blob, heights, names, ls, mlr, v, pc, words, **SMALL)
    err = capfd.readouterr().err
    return {0: "accept", -2: "parse"}.get(r) or err.strip().rsplit(": ", 1)[-1]


def _library_verdict(lib, mach, pc, heights, names, words, start):
    from sp1_b200.lib import Sp1B200Error, verdict_name
    try:
        v, st = lib.verify_shard(mach, pc, heights, names, words, start)
    except Sp1B200Error:
        return "parse", None
    return ("accept" if v == 0 else verdict_name(v)), st


def test_verify_shard_on_a_poisoned_pool(capfd):
    """acceptance with the prover's final challenger, and one corrupted word in each section plus a wrong preprocessed commitment,
    with the oracle's verdicts"""
    (blob, heights, mains, preps, pv, names), ls, mlr, cap = _shard_case("spec2")
    lib = _lib(log_stacking_height=ls, max_log_row_count=mlr, **SMALL)
    mach = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    start = O.Challenger().st.copy()
    final = start.copy()
    words = GP.prove(lib, mach, prep_round, mains, heights, names, pv, final)
    lib.jagged_round_free(prep_round)
    cases = []
    for s, e in _sections(words):
        for off in (s, (s + e) // 2, e - 1):
            bad = words.copy(); bad[off] = (int(bad[off]) + 1) % P
            cases.append((f"word {off}", pc, bad))
    wrong_pc = pc.copy(); wrong_pc[0] ^= 1
    cases.append(("preprocessed commitment", wrong_pc, words))
    want = [_oracle_verdict(capfd, blob, heights, names, ls, mlr, start, c_pc, w) for _, c_pc, w in cases]
    assert "accept" not in want
    for name in PATTERNS:
        poison(lib, name)
        got, st = _library_verdict(lib, mach, pc, heights, names, words, start)
        assert got == "accept" and (st == final).all(), f"{name}: the library rejects its own proof ({got}) or ends elsewhere"
        for (what, c_pc, w), o in zip(cases, want):
            poison(lib, name)
            got, _ = _library_verdict(lib, mach, c_pc, heights, names, w, start)
            assert got == o or (got in ORACLE_LACKS and o not in ("accept", "parse")), f"{name}, {what}: library {got}, oracle {o}"
    covered(lib)
    lib.machine_free(mach)
    lib.close()


def test_verify_core_proof_on_a_poisoned_pool():
    from tests import core_chain as CC
    c = Core(specs_machine(M.WITH_PREP), 8, 9)
    pvs, tail = CC.chain(3, 7600)
    words, finals, mtail = c.prove(pvs, tail, before_each=lambda: poison(c.lib, "random-a"))
    bad = [w.copy() for w in words]
    at = int(bad[1][1]) + int(bad[1][2]) + 6 + 3   # a word of shard 1's zerocheck section
    bad[1][at] = (int(bad[1][at]) + 1) % P
    for name in PATTERNS:
        poison(c.lib, name)
        v, s, sv, fin = c.verify(words, mtail)
        assert (v, s, sv) == (0, 0, 0), f"{name}: rejected ({v}, {s}, {sv})"
        assert all((fin[k] == finals[k]).all() for k in range(3)), f"{name}: final challengers"
        poison(c.lib, name)
        v, s, sv, fin = c.verify(bad, mtail)
        single, _ = c.lib.verify_shard(c.mach, c.pc, c.heights, c.names, bad[1], c.start(mtail))
        assert (v, s) == (45, 1) and sv == single != 0 and fin is None, f"{name}: ({v}, {s}, {sv}), verify_shard {single}"
    covered(c.lib)
    c.close()


def test_verify_compressed_on_a_poisoned_pool():
    c = Rec(specs_machine(M.NO_PREP), 7, 8, n_keys=2)
    key = c.keys[0]
    poison(c.lib, "random-b")
    words, final = c.prove(key, c.pv())
    poison(c.lib, "ones")
    bad_words, _ = c.prove(c.keys[1], c.pv(vk_root=True))
    good = (key, words, c.merkle(key), c.sp1)
    bad = (c.keys[1], bad_words, c.merkle(c.keys[1]), c.sp1)
    assert c.oracle(*good[:2], 187, *good[2:]) == RR.ACCEPT and c.oracle(*bad[:2], 187, *bad[2:]) == RR.VK_ROOT
    for name in PATTERNS:
        poison(c.lib, name)
        v, sv, fin = c.verify([good])
        assert (v, sv) == ([0], [0]) and (fin[0] == final).all(), f"{name}: {v} {sv}"
        poison(c.lib, name)
        v, sv, _ = c.verify([bad, good])
        assert (v, sv) == ([RR.VK_ROOT, 0], [0, 0]), f"{name}: {v} {sv}"
    covered(c.lib)
    c.close()


@pytest.mark.parametrize("n,pad_to", [(5, 9), (300, 0)])
def test_recursion_vks_on_a_poisoned_pool(n, pad_to):
    rng = np.random.default_rng(7700 + n)
    d = O.rand_field(rng, (n, 8))
    ref = RR.VkMap(d, pad_to=pad_to)
    lib = _lib()
    for name in PATTERNS:
        poison(lib, name)
        vks = lib.recursion_vks(d, pad_to=pad_to)
        assert vks.num_keys() == len(ref.keys) and (vks.root() == ref.root).all(), f"{name}: root"
        for i in range(0, len(ref.keys), max(1, len(ref.keys) // 40)):
            idx, path = vks.open(O.to_monty(np.array(ref.keys[i])))
            assert idx == i and (path == ref.open_index(i)[1]).all(), f"{name}: opening {i}"
        vks.close()
    covered(lib)
    lib.close()


# ---- 2. one context across changing shapes -----------------------------------------------------------------------------------------
def test_one_context_across_changing_shapes():
    """a large shard, a small shard of another machine, a machine without preprocessed columns, the 96-chip table and the large shard
    again on one context; each proved from a host pointer, a device tensor and upload slot 0 (which the larger shard filled first, so the
    smaller one leaves a stale tail); a verification of the large shard right after the small one's proofs; a capacity error right before
    the 96-chip table"""
    import torch
    from sp1_b200.lib import Sp1B200Error
    ls, mlr = 10, 12
    machines = {
        "large": M.workload_machine("tinyc", seed=7800, max_log_rows=mlr, scale=0.25),
        "small": M.spec_machine(np.random.default_rng(7801), [(1024, 2, True), (256 + 32, 3, False), (0, 1, False), (2048, 1, True)],
                                names="Chip{:02d}"),
        "no-prep": M.spec_machine(np.random.default_rng(7802), M.NO_PREP),
        "96-chip": M.spec_machine(np.random.default_rng(7803), M.full_table_spec(96, 7804, absent=True)),
    }
    assert all(max(inp[1]) <= 1 << mlr for inp in machines.values())
    assert M.dense_main(machines["small"][2]).size < M.dense_main(machines["large"][2]).size
    assert all(p is None for p in machines["no-prep"][3])
    oracle = {k: _oracle_shard(inp, ls, mlr, 7810 + i) for i, (k, inp) in enumerate(machines.items())}
    lib = _lib(log_stacking_height=ls, max_log_row_count=mlr, **SMALL)
    machs = {k: lib.machine_create(inp[0]) for k, inp in machines.items()}
    pcs, rounds, proofs = {}, [], {}
    for step, k in enumerate(["large", "small", "no-prep", "96-chip", "large"]):
        blob, heights, mains, preps, pv, names = machines[k]
        st0, opc, owords, ost = oracle[k]
        pc, prep_round = GP.commit_prep(lib, preps)
        assert (pc == opc).all(), f"step {step} ({k}): preprocessed commitment"
        pcs[k] = None if prep_round is None else pc
        rounds.append(prep_round)
        if k == "96-chip":   # a capacity error on another machine's shard first: the transcript is untouched
            big = machines["large"]
            st = oracle["large"][0].copy()
            with pytest.raises(Sp1B200Error, match="capacity"):
                lib.prove_shard(machs["large"], rounds[0], M.dense_main(big[2]), big[1], big[5], big[4], st, cap_words=1000)
            assert (st == oracle["large"][0]).all()
        dense = M.dense_main(mains)
        d_dense = torch.from_numpy(dense.view(np.int32)).cuda()
        pinned = torch.from_numpy(dense.view(np.int32)).pin_memory()
        torch.cuda.synchronize()
        for how in ("host memory", "device memory", "upload slot 0"):
            src = {"host memory": dense, "device memory": d_dense}.get(how)
            if src is None:
                src = lib.upload_begin(pinned, 0)
            st = st0.copy()
            words = lib.prove_shard(machs[k], prep_round, src, heights, names, pv, st)
            assert words.size == owords.size and (words == owords).all(), f"step {step} ({k}) from {how}: " + M.shard_diff(words, owords)
            assert (st == ost).all(), f"step {step} ({k}) from {how}: final challenger"
            proofs[k] = (words, st)
        lib.sync()
        if k == "small":     # the large shard's proof verified right after the small shard's proofs
            big = machines["large"]
            v, st = lib.verify_shard(machs["large"], pcs["large"], big[1], big[5], proofs["large"][0], oracle["large"][0])
            assert v == 0 and (st == proofs["large"][1]).all(), "verifying the large shard after proving the small one"
    for r in rounds:
        if r is not None:
            lib.jagged_round_free(r)
    for m in machs.values():
        lib.machine_free(m)
    lib.close()


# ---- 3. guard-banded caller buffers -----------------------------------------------------------------------------------------------------
class Band:
    """words (uint32) on the device at offset G inside a tensor of n + 2G words; the G words on each side hold a random pattern"""

    def __init__(self, rng, words):
        import torch
        w = np.ascontiguousarray(words, dtype=np.uint32).reshape(-1)
        self.n = w.size
        self.host = rng.integers(0, 1 << 32, self.n + 2 * G, dtype=np.uint64).astype(np.uint32)
        self.host[G:G + self.n] = w
        self.base = torch.from_numpy(self.host.view(np.int32)).cuda()
        self.view = self.base[G:G + self.n]
        torch.cuda.synchronize()    # the library runs on its own non-blocking stream: torch's copy must have finished

    def words(self):
        return self.view.cpu().numpy().view(np.uint32)

    def check(self, lib, what):
        import torch
        lib.sync()
        torch.cuda.synchronize()
        got = self.base.cpu().numpy().view(np.uint32)
        assert (got[:G] == self.host[:G]).all(), f"{what}: the guard words before the buffer changed"
        assert (got[G + self.n:] == self.host[G + self.n:]).all(), f"{what}: the guard words after the buffer changed"


def test_guard_bands_kernels():
    """poseidon2_permute in place, rs_encode input and output (generic and fast paths), merkle_commit matrix and layers, pack_row_major"""
    rng = np.random.default_rng(7900)
    lib = _lib()
    states = O.rand_field(rng, (100, 16))
    b = Band(rng, states)
    lib.poseidon2_permute(b.view.view(100, 16))
    b.check(lib, "poseidon2_permute")
    assert (b.words().reshape(100, 16) == np.stack([O.permute(s) for s in states])).all(), "poseidon2_permute"
    for log_h, ncols, lb in [(9, 3, 2), (11, 3, 2), (19, 1, 2), (18, 1, 1)]:
        msg = O.rand_field(rng, (ncols, 1 << log_h))
        bi, bo = Band(rng, msg), Band(rng, poisoned_words(ncols << (log_h + lb)))
        lib.rs_encode(bi.view, bo.view, ncols, log_h, lb)
        bi.check(lib, "rs_encode input"); bo.check(lib, "rs_encode output")
        assert (bo.words().reshape(ncols, -1) == O.rs_encode(msg, lb)).all(), f"rs_encode {(log_h, ncols, lb)}"
    width, log_h = 13, 9
    mat = O.rand_field(rng, (width, 1 << log_h))
    bm, bl = Band(rng, mat), Band(rng, poisoned_words(((2 << log_h) - 1) * 8))
    root, commit = lib.merkle_commit(bm.view, width, log_h, d_layers=bl.view)
    bm.check(lib, "merkle_commit matrix"); bl.check(lib, "merkle_commit layers")
    oroot, ocommit, olayers = O.merkle_commit(mat, want_layers=True)
    assert (root == oroot).all() and (commit == ocommit).all() and (bl.words().reshape(-1, 8) == olayers).all(), "merkle_commit"
    shapes = [(96, 5), (1, 1), (0, 7), (33, 33), (4099, 70), (64, 246)]
    tabs = [O.rand_field(rng, (r, c)) for r, c in shapes]
    rows = np.concatenate([t.reshape(-1) for t in tabs])
    bi, bo = Band(rng, rows), Band(rng, poisoned_words(rows.size))
    lib.pack_row_major(bi.view, shapes, bo.view)
    bi.check(lib, "pack_row_major input"); bo.check(lib, "pack_row_major output")
    assert (bo.words() == np.concatenate([np.ascontiguousarray(t.T).reshape(-1) for t in tabs])).all(), "pack_row_major"
    lib.close()


def test_guard_bands_stacked_and_jagged_commit():
    """stacked_commit borrows its device input until the commitment is freed: the guards hold after stacked_prove too; jagged_commit_dense
    of a device buffer"""
    rng = np.random.default_rng(7910)
    log_h, nq = 9, 12
    rounds = [O.rand_field(rng, (c, 1 << log_h)) for c in (4, 3)]
    point = O.rand_field(rng, (3 + log_h, 4))      # 3 = log2 of the 7 columns, rounded up
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 5))
    och = ch.clone()
    ocommits, oproof = O.stacked_prove_verify(rounds, log_h, point, och, num_queries=nq, pow_bits=5, batch_pow_bits=2)
    lib = _lib(log_stacking_height=log_h, num_queries=nq, pow_bits=5, batch_pow_bits=2)
    bands, handles = [Band(rng, r) for r in rounds], []
    for i, (b, r) in enumerate(zip(bands, rounds)):
        commit, h = lib.stacked_commit(b.view, r.shape[0])
        assert (commit == ocommits[i]).all(), f"stacked_commit round {i}"
        handles.append(h)
    st = ch.st.copy()
    proof = lib.stacked_prove(handles, point, st)
    for i, b in enumerate(bands):
        b.check(lib, f"stacked_commit / stacked_prove input {i}")
    assert proof.size == oproof.size and (proof == oproof).all() and (st == och.st).all(), "stacked_prove"
    for h in handles:
        lib.commit_free(h)
    lib.close()
    # jagged: the tables' cells back to back on the device
    shapes, ls, mlr = [(4096, 3), (96, 17), (0, 5)], 12, 13
    tabs = O.random_tables(rng, shapes)
    z_row = O.rand_field(rng, (mlr, 4))
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 3))
    och = ch.clone()
    ocommits, oclaims, oproof = O.jagged_prove_verify([tabs], ls, mlr, z_row, och, num_queries=8, pow_bits=4, batch_pow_bits=2)
    lib = _lib(log_stacking_height=ls, max_log_row_count=mlr, num_queries=8, pow_bits=4, batch_pow_bits=2)
    b = Band(rng, np.concatenate([np.ascontiguousarray(t).reshape(-1) for t in tabs if t.shape[1]]))
    commit, h = lib.jagged_commit_dense(b.view, [t.shape[1] for t in tabs], [t.shape[0] for t in tabs])
    b.check(lib, "jagged_commit_dense input")
    assert (commit == ocommits[0]).all(), "jagged_commit_dense"
    claims = lib.jagged_column_claims(h, z_row, sum(t.shape[0] for t in tabs))
    st = ch.st.copy()
    proof = lib.jagged_prove([h], z_row, claims, st)
    assert (claims == oclaims).all() and proof.size == oproof.size and (proof == oproof).all() and (st == och.st).all(), "jagged_prove"
    lib.jagged_round_free(h)
    lib.close()


def test_guard_bands_logup_gkr_and_zerocheck():
    """each chip's main and preprocessed table in a band of its own"""
    spec, mlr = PHASE_SPECS[0]
    rng = np.random.default_rng(7920)
    blob, heights, mains, preps, pv, _ = M.spec_machine(rng, spec)
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 4))
    och = ch.clone()
    ogkr = O.gkr_prove_verify(blob, heights, mains, preps, mlr, och, gkr_pow_bits=4)
    gp, st0, openings, ozc, ozst = M.oracle_zerocheck(rng, blob, heights, mains, preps, pv, mlr)
    lib = _lib(max_log_row_count=mlr, log_stacking_height=mlr, gkr_pow_bits=4)
    mach = lib.machine_create(blob)
    bm = [Band(rng, m) if m.size else None for m in mains]
    bp = [Band(rng, p) if p is not None else None for p in preps]
    d_mains = [b.view if b else None for b in bm]
    d_preps = [b.view if b else None for b in bp]
    st = ch.st.copy()
    words = lib.logup_gkr(mach, heights, d_mains, d_preps, st)
    for b in bm + bp:
        if b:
            b.check(lib, "logup_gkr")
    assert words.size == ogkr.size and (words == ogkr).all() and (st == och.st).all(), M.first_diff(words, ogkr, "LogUp-GKR proof")
    words, st = M.product_zerocheck(lib, mach, heights, mains, preps, pv, gp, st0, openings, device=(d_mains, d_preps))
    for b in bm + bp:
        if b:
            b.check(lib, "zerocheck")
    assert words.size == ozc.size and (words == ozc).all() and (st == ozst).all(), M.first_diff(words, ozc, "zerocheck proof")
    lib.machine_free(mach)
    lib.close()


def test_guard_bands_prove_shard_and_debug_reports():
    """main_dense on the device for prove_shard and both shard checks"""
    rng = np.random.default_rng(7930)
    (blob, heights, mains, preps, pv, names), ls, mlr, _ = _shard_case("spec2")
    st0, opc, owords, ost = _oracle_shard((blob, heights, mains, preps, pv, names), ls, mlr, 7931)
    lib = _lib(log_stacking_height=ls, max_log_row_count=mlr, **SMALL)
    mach = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    b = Band(rng, M.dense_main(mains))
    st = st0.copy()
    words = lib.prove_shard(mach, prep_round, b.view, heights, names, pv, st)
    b.check(lib, "prove_shard")
    assert words.size == owords.size and (words == owords).all() and (st == ost).all(), M.shard_diff(words, owords)
    broken = [m.copy() for m in mains]
    k = int(np.argmax(heights))
    broken[k][1, 3] = (int(broken[k][1, 3]) + 5) % P
    for ms in (mains, broken):
        b = Band(rng, M.dense_main(ms))
        got = lib.debug_constraints_words(mach, prep_round, b.view, heights, pv)
        b.check(lib, "debug_constraints")
        assert got.tolist() == DO.debug_constraints(blob, heights, ms, preps, pv).tolist(), "constraint report"
        got = lib.debug_interactions_words(mach, prep_round, b.view, heights)
        b.check(lib, "debug_interactions")
        assert got.tolist() == DO.debug_interactions(blob, heights, ms, preps).tolist(), "interaction report"
    lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()
