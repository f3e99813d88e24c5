"""GPU tests of a shard's lookup multiplicity traces (sp1b200_lookup_traces): the Byte, Program and Range main tables equal the NumPy
restatement (tests/lookup_ref.py) word for word for random, skewed and Zipf-like streams, from host and device memory into host and device
outputs; a permuted stream and a counted map's expansion into count-1 records give the same words; every malformed input is an error
that names its record and leaves the context usable; a poisoned pool gives the same words.  End to end, the tables written into a
device dense buffer balance the LogUp interactions of a machine whose Byte, Program and Range chips carry the real interactions, and
the shard proven from that buffer verifies under the key program_setup returns."""
import ctypes as C

import numpy as np
import pytest

from tests import lookup_ref as LR
from tests import machines as M
from tests import program_ref as PR

pytestmark = pytest.mark.gpu


def _lib(**params):
    from sp1_b200 import Lib
    return Lib(0, **params)


def _lookups(n, rng, max_count=1):
    """n random valid lookup records: opcode 0..6, Range records with a < 2^b, counts in [1, max_count]"""
    from sp1_b200.lib import pack_byte_lookups
    op = rng.integers(0, 7, n)
    b = rng.integers(0, 256, n)
    c = rng.integers(0, 256, n)
    bits = rng.integers(0, 17, n)
    a_rng = (rng.integers(0, 1 << 16, n) & ((1 << bits) - 1))
    is_range = op == 6
    a = np.where(is_range, a_rng, rng.integers(0, 1 << 16, n))   # a of a byte opcode is not read
    b = np.where(is_range, bits, b)
    return pack_byte_lookups(op, a, b, c, rng.integers(1, max_count + 1, n))


def _pcs(n, pc_base, n_instrs, rng, max_count=1):
    """n pc records: mostly inside the program, some below, above or misaligned"""
    from sp1_b200.lib import pack_pc_counts
    i = rng.integers(0, n_instrs, n).astype(np.uint64)
    pc = np.uint64(pc_base) + np.uint64(4) * i
    kind = rng.integers(0, 16, n)
    pc = np.where(kind == 0, pc + np.uint64(2), pc)                                       # misaligned
    pc = np.where(kind == 1, np.uint64(pc_base) + np.uint64(4 * n_instrs) + np.uint64(4) * i, pc)   # above
    pc = np.where((kind == 2) & (pc_base >= 4), np.uint64(pc_base) - np.uint64(4), pc)    # below
    return pack_pc_counts(pc, rng.integers(1, max_count + 1, n))


def _dev(recs):
    import torch
    return torch.from_numpy(recs.view(np.uint8).reshape(-1).copy()).cuda()


def _check(lib, pc_base, n_instrs, lookups, pcs, pv=None, device=False):
    """the library's words (host or device records and outputs) equal the restatement's"""
    want = LR.main_words(pc_base, n_instrs, lookups, pcs, None if pv is None else _canon(pv))
    if device:
        import torch
        out = tuple(torch.zeros(w.shape, dtype=torch.int32, device="cuda") for w in want)
        lib.lookup_traces(pc_base, n_instrs, _dev(lookups), _dev(pcs), pv, out=out)
        got = tuple(o.cpu().numpy().view(np.uint32) for o in out)
    else:
        got = lib.lookup_traces(pc_base, n_instrs, lookups, pcs, pv)
    for name, g, w in zip(("Byte", "Program", "Range"), got, want):
        assert g.shape == w.shape, (name, g.shape, w.shape)
        bad = np.argwhere(g != w)
        assert bad.size == 0, f"{name}: first differing (column, row) {bad[:4].tolist()}"
    return got


def _canon(pv_monty):
    return [int(x) for x in _from_monty(pv_monty)]


def _from_monty(w):
    from tests import oracle_lib as O
    return O.from_monty(np.asarray(w, np.uint32)).astype(np.int64)


def _pv(rng):
    """187 public values (Montgomery words) whose limbs and bytes are in range, the low timestamp limb of the first timestamp 0"""
    from tests import oracle_lib as O
    pv = rng.integers(0, 1 << 16, 187)
    for at in (LR.INITIAL_TIMESTAMP, LR.LAST_TIMESTAMP):
        pv[at + 1:at + 3] = rng.integers(0, 256, 2)
    pv[LR.INITIAL_TIMESTAMP + 3] = 0
    pv[0:64] = rng.integers(0, 256, 64)
    return O.to_monty(pv.astype(np.uint64))


@pytest.mark.parametrize("n_lookups,n_pcs,n_instrs", [(1, 1, 1), (1000, 1000, 15), (1 << 16, 5000, 16), (12345, 1 << 16, 17),
                                                      (1 << 20, 1 << 20, 32), (3, 1 << 12, 33), (1 << 26, 1 << 22, 1 << 20)])
def test_random_streams_match_the_restatement(n_lookups, n_pcs, n_instrs):
    rng = np.random.default_rng(n_lookups + 7 * n_instrs)
    pc_base = 0x10000 + 4 * int(rng.integers(0, 1 << 20))
    lookups = _lookups(n_lookups, rng, max_count=3)
    pcs = _pcs(n_pcs, pc_base, n_instrs, rng, max_count=3)
    lib = _lib()
    got = _check(lib, pc_base, n_instrs, lookups, pcs)
    _check(lib, pc_base, n_instrs, lookups, pcs, device=True)
    perm_l, perm_p = rng.permutation(n_lookups), rng.permutation(n_pcs)   # a permuted stream gives identical words
    got_p = lib.lookup_traces(pc_base, n_instrs, lookups[perm_l], pcs[perm_p])
    assert all((a == b).all() for a, b in zip(got, got_p))
    lib.close()


def test_skewed_and_zipf_streams():
    from sp1_b200.lib import pack_byte_lookups, pack_pc_counts
    rng = np.random.default_rng(11)
    lib = _lib()
    n = 1 << 24
    hot = pack_byte_lookups(np.full(n, 3), 0, 0, 0, 1)                      # U8Range(0, 0), 2^24 times
    loop = pack_pc_counts(np.full(n, 0x1000 + 4 * 7, np.uint64), 1)         # one pc of a loop
    got = _check(lib, 0x1000, 100, hot, loop, device=True)
    assert got[0][3, 0] == LR.to_monty(n) and got[1][0, 7] == LR.to_monty(n)
    # Zipf-like: key k drawn with weight ~ 1 / k
    base = _lookups(1 << 12, rng)
    keys = np.minimum(rng.zipf(1.3, 1 << 22) - 1, base.size - 1)
    z = base[keys]
    zp = pack_pc_counts(np.uint64(0x1000) + np.uint64(4) * np.minimum(rng.zipf(1.3, 1 << 22) - 1, 4095).astype(np.uint64), 1)
    got = _check(lib, 0x1000, 4096, z, zp)
    perm = rng.permutation(z.size)
    assert all((a == b).all() for a, b in zip(got, lib.lookup_traces(0x1000, 4096, z[perm], zp[perm])))
    lib.close()


def test_counted_map_equals_its_expansion():
    """record.byte_lookups (one record per distinct event with its multiplicity) and the raw events (count 1 each) give identical words"""
    from sp1_b200.lib import pack_byte_lookups, pack_pc_counts
    rng = np.random.default_rng(12)
    raw = _lookups(1 << 18, rng)
    raw = raw[rng.integers(0, 1 << 12, 1 << 20)]              # many repeats
    key = (raw["opcode"].astype(np.int64) << 32) | (raw["a"].astype(np.int64) << 16) | (raw["b"].astype(np.int64) << 8) | raw["c"]
    uniq, n = np.unique(key, return_counts=True)
    counted = pack_byte_lookups(uniq >> 32, (uniq >> 16) & 0xFFFF, (uniq >> 8) & 0xFF, uniq & 0xFF, n)
    raw_pcs = pack_pc_counts(np.uint64(0x4000) + np.uint64(4) * rng.integers(0, 300, 1 << 20).astype(np.uint64), 1)
    pu, pc_count = np.unique(raw_pcs["pc"], return_counts=True)
    counted_pcs = pack_pc_counts(pu, pc_count)
    lib = _lib()
    a = _check(lib, 0x4000, 300, raw, raw_pcs)
    b = _check(lib, 0x4000, 300, counted, counted_pcs)
    assert all((x == y).all() for x, y in zip(a, b))
    lib.close()


@pytest.mark.parametrize("device", [False, True])
def test_public_value_lookups(device):
    rng = np.random.default_rng(13)
    lib = _lib()
    lookups, pcs = _lookups(5000, rng), _pcs(500, 0x2000, 64, rng)
    pv = _pv(rng)
    on = _check(lib, 0x2000, 64, lookups, pcs, pv, device=device)
    off = _check(lib, 0x2000, 64, lookups, pcs, None, device=device)
    assert not (on[0] == off[0]).all() and not (on[2] == off[2]).all() and (on[1] == off[1]).all()
    wrap = LR.RANGE_NUM_ROWS // 16 + 8191                    # the 13-bit check of (0 - 1) / 8 lands on row 2^13 + 8191
    assert int(_from_monty(on[2][0, wrap])) == int(_from_monty(off[2][0, wrap])) + 1
    lib.close()


def test_errors_name_the_record_and_leave_the_context_usable():
    from sp1_b200.lib import Sp1B200Error, pack_byte_lookups, pack_pc_counts
    from tests import oracle_lib as O
    rng = np.random.default_rng(14)
    lib = _lib(max_log_row_count=17)
    lookups, pcs, pv = _lookups(3000, rng), _pcs(800, 0x8000, 200, rng), _pv(rng)

    def fine():
        _check(lib, 0x8000, 200, lookups, pcs, pv)

    def bad(field, i, v):
        x = lookups.copy(); x[field][i] = v
        return x
    big = pack_byte_lookups([3, 3], 0, 1, 1, [0xFFFFFFFF, 0xFFFFFFFF])   # 2^33 - 2 at one key: past 2^32 without wrapping
    near = pack_byte_lookups(6, 5, 4, 0, O.P)
    pv_bad_ts = pv.copy(); pv_bad_ts[LR.INITIAL_TIMESTAMP + 1] = O.to_monty(np.array([256], np.uint64))[0]
    pv_bad_byte = pv.copy(); pv_bad_byte[40] = O.to_monty(np.array([300], np.uint64))[0]
    pv_bad_addr = pv.copy(); pv_bad_addr[LR.NEXT_PC + 2] = O.to_monty(np.array([1 << 16], np.uint64))[0]
    pv_not_field = pv.copy(); pv_not_field[5] = 0x7F000001
    cases = [((0x8000, 200, bad("opcode", 1717, 7), pcs, pv), "lookup 1717 has opcode 7"),
             ((0x8000, 200, _range_b17(lookups, 2999), pcs, pv), "lookup 2999 is a Range check of a = .* with b = 17 bits"),
             ((0x8000, 0, lookups, pcs, pv), "n_instrs = 0"),
             (((1 << 48) - 4 * 60, 200, lookups, pcs, pv), "instruction 60 has pc"),
             ((0x8000, (1 << 17) + 1, lookups, pcs, pv), "rows > 2\\^17"),
             ((0x8000, 200, big, pcs, None), "Byte row 257 column 3 accumulates multiplicity 8589934590 >= p"),
             ((0x8000, 200, near, pcs, None), "Range row 21 column 0 accumulates multiplicity 2130706433 >= p"),
             ((0x8000, 200, lookups, pack_pc_counts([0x8000 + 4 * 9] * 2, [0x7F000000, 1]), None),
              "Program row 9 column 0 accumulates multiplicity 2130706433 >= p"),
             ((0x8000, 200, lookups, pcs, pv[:160]), "160 public values, a core shard has 187"),
             ((0x8000, 200, lookups, pcs, pv_bad_ts), "public value 114 \\(initial_timestamp\\) = 256 does not fit 8 bits"),
             ((0x8000, 200, lookups, pcs, pv_bad_byte), "public value 40 \\(committed_value_digest\\) = 300 does not fit 8 bits"),
             ((0x8000, 200, lookups, pcs, pv_bad_addr), "public value 85 \\(address\\) = 65536 does not fit 16 bits"),
             ((0x8000, 200, lookups, pcs, pv_not_field), "public value 5 is not a field element")]
    for args, msg in cases:
        with pytest.raises(Sp1B200Error, match=msg):
            lib.lookup_traces(*args)
        fine()
    # NULL arrays with a non-zero count, and a partial set of outputs
    out = [np.zeros((6, 1 << 16), np.uint32), np.zeros((1, 224), np.uint32), np.zeros((1, 1 << 17), np.uint32)]
    for n_l, n_p, outs, msg in ((5, 0, out, b"NULL lookup array with 5 records"), (0, 7, out, b"NULL pc array with 7 records"),
                                (0, 0, [out[0], None, out[2]], b"all NULL")):
        e = lib.L.sp1b200_lookup_traces(lib.ctx, C.c_uint64(0x8000), C.c_uint64(200), None, C.c_uint64(n_l), None, C.c_uint64(n_p), None,
                                        C.c_uint32(0), *[None if o is None else C.c_void_p(o.ctypes.data) for o in outs], None)
        assert e and msg in e, e
        fine()
    rows = (C.c_uint64 * 3)()   # NULL outputs only report the heights
    assert not lib.L.sp1b200_lookup_traces(lib.ctx, C.c_uint64(0x8000), C.c_uint64(200), None, C.c_uint64(0), None, C.c_uint64(0), None,
                                           C.c_uint32(0), None, None, None, rows)
    assert list(rows) == [1 << 16, 224, 1 << 17]
    lib.close()


def _range_b17(lookups, i):
    x = lookups.copy(); x["opcode"][i] = 6; x["b"][i] = 17
    return x


def test_poisoned_pool_gives_the_same_words():
    """every block of the context's pool holds a non-zero pattern before the call (a freed pool keeps its blocks)"""
    rng = np.random.default_rng(15)
    lookups, pcs, pv = _lookups(1 << 20, rng, 5), _pcs(1 << 16, 0x1000, 5000, rng), _pv(rng)
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
    _check(lib, 0x1000, 5000, lookups, pcs, pv)
    _check(lib, 0x1000, 5000, lookups, pcs, pv, device=True)
    lib.close()


# ---- end to end: the real Byte / Program / Range interactions balance against a synthetic sender ------------------------------------
NAMES = ["Byte", "Cpu", "Program", "Range"]
KIND_PROGRAM, KIND_BYTE = 2, 5   # InteractionKind (crates/hypercube/src/lookup/interaction.rs)
CPU_W = 1 + 4 + 1 + 16           # byte multiplicity, byte values [4], program multiplicity, program values [16]


def _machine():
    """chips in name order with no constraints; interactions restated from bytes/air.rs, range/air.rs and trusted.rs:311-322 (receives)
    and a Cpu chip that sends one byte lookup and one instruction per row"""
    from sp1_b200 import synth_air as SA
    prep, main = SA.LEAF_PREP, SA.LEAF_MAIN
    col = lambda src, k: SA._vcol([(src, k, 1)])
    const = lambda v: SA._vcol([], constant=v)
    b, c = col(prep, 0), col(prep, 1)
    byte = [(0, KIND_BYTE, col(main, 0), [const(0), col(prep, 2), b, c]),      # AND: and
            (0, KIND_BYTE, col(main, 1), [const(1), col(prep, 3), b, c]),      # OR: or
            (0, KIND_BYTE, col(main, 2), [const(2), col(prep, 4), b, c]),      # XOR: xor
            (0, KIND_BYTE, col(main, 3), [const(3), const(0), b, c]),          # U8Range: zero
            (0, KIND_BYTE, col(main, 4), [const(4), col(prep, 5), b, c]),      # LTU: ltu
            (0, KIND_BYTE, col(main, 5), [const(5), col(prep, 6), b, const(0)])]   # MSB: msb, b, zero
    rng_ = [(0, KIND_BYTE, col(main, 0), [const(6), col(prep, 0), col(prep, 1), const(0)])]
    prog = [(0, KIND_PROGRAM, col(main, 0), [col(prep, k) for k in range(16)])]
    cpu = [(1, KIND_BYTE, col(main, 0), [col(main, k) for k in range(1, 5)]),
           (1, KIND_PROGRAM, col(main, 5), [col(main, k) for k in range(6, 22)])]
    words = [SA.Asm().words(6, 7), SA.Asm().words(CPU_W, 0), SA.Asm().words(1, 16), SA.Asm().words(1, 2)]
    return SA.machine_blob_with_interactions(words, [M._inter_words(x) for x in (byte, cpu, prog, rng_)])


def _lookup_value(op, a, b, c):
    """the values a Byte / Range row receives for a valid event (opcode, a, b, c)"""
    if op == 6:
        return [6, a, b, 0]
    res = [b & c, b | c, b ^ c, 0, int(b < c), b >> 7][op]
    return [op, res, b, 0 if op == 5 else c]


def _cpu_trace(lookups, pcs, pc_base, instrs):
    """one row per distinct lookup key (values, summed count) and one per executed instruction -> canonical [CPU_W, h] and h"""
    sends = {}
    for r in lookups:
        key = tuple(_lookup_value(int(r["opcode"]), int(r["a"]), int(r["b"]), int(r["c"])))
        sends[key] = sends.get(key, 0) + int(r["count"])
    prows = PR.program_trace(pc_base, instrs)
    counts = {}
    for r in pcs:
        off = int(r["pc"]) - pc_base
        if off >= 0 and off % 4 == 0 and off // 4 < len(instrs):
            counts[off // 4] = counts.get(off // 4, 0) + int(r["count"])
    n = max(len(sends), len(counts))
    h = max(32, -(-n // 32) * 32)
    t = np.zeros((CPU_W, h), np.int64)
    for i, (key, m) in enumerate(sends.items()):
        t[0, i] = m
        t[1:5, i] = key
    for i, (row, m) in enumerate(counts.items()):
        t[5, i] = m
        t[6:22, i] = prows[row]
    return t, h


def test_traces_balance_the_real_interactions_and_prove():
    import torch
    from sp1_b200.lib import MAX_OPCODE, HostChallenger, pack_instructions
    from tests import oracle_lib as O
    rng = np.random.default_rng(16)
    n_instrs = 1000
    instrs = pack_instructions(rng.integers(0, MAX_OPCODE + 1, n_instrs), rng.integers(0, 32, n_instrs),
                               rng.integers(0, 1 << 64, n_instrs, dtype=np.uint64, endpoint=False),
                               rng.integers(0, 1 << 64, n_instrs, dtype=np.uint64, endpoint=False), rng.integers(0, 2, n_instrs),
                               rng.integers(0, 2, n_instrs))
    pc_base = 0x20000
    lookups = _lookups(20000, rng, max_count=4)
    pcs = _pcs(30000, pc_base, n_instrs, rng, max_count=3)
    pv = _pv(rng)
    all_lookups = np.concatenate([lookups, LR.dependency_records(_from_monty(pv))])
    lib = _lib(log_stacking_height=16, max_log_row_count=17, **M.SMALL)
    key = lib.program_setup(pc_base, instrs, pc_base, np.zeros(0, np.uint64), np.zeros(0, np.uint64))
    mach = lib.machine_create(_machine())
    cpu, h_cpu = _cpu_trace(all_lookups, pcs, pc_base, instrs)
    heights = [1 << 16, h_cpu, key["prep_rows"][1], 1 << 17]
    widths = [6, CPU_W, 1, 1]
    offs = [0] + [int(x) for x in np.cumsum([w * h for w, h in zip(widths, heights)])]
    dense = torch.zeros(offs[-1], dtype=torch.int32, device="cuda")
    dense[offs[1]:offs[2]] = torch.from_numpy(O.to_monty(cpu.reshape(-1).astype(np.uint64)).view(np.int32)).cuda()
    views = [dense[offs[k]:offs[k + 1]] for k in (0, 2, 3)]

    def write(lk):
        lib.lookup_traces(pc_base, n_instrs, lk, _dev(pcs), pv, out=views)
    write(_dev(lookups))
    rep = lib.debug_interactions(mach, key["round"], dense, heights)
    assert rep["n_unbalanced"] == 0, rep
    # one record's count lowered by one: exactly its key is unbalanced, by one send
    low = lookups.copy()
    i = int(np.nonzero(low["count"] > 1)[0][0])
    low["count"][i] -= 1
    write(_dev(low))
    rep = lib.debug_interactions(mach, key["round"], dense, heights)
    r = low[i]
    want = _lookup_value(int(r["opcode"]), int(r["a"]), int(r["b"]), int(r["c"]))
    assert rep["n_unbalanced"] == 1, rep
    k0 = rep["keys"][0]
    assert k0["kind"] == KIND_BYTE and [int(v) for v in _from_monty(k0["values"])] == want and int(_from_monty([k0["net"]])[0]) == 1
    write(_dev(lookups))
    hc = HostChallenger(); hc.observe(key["prep_commit"]); hc.observe(key["vk_tail"])
    st0 = hc.st.copy()
    st = st0.copy()
    words = lib.prove_shard(mach, key["round"], dense, heights, NAMES, pv, st)
    verdict, fin = lib.verify_shard(mach, key["prep_commit"], heights, NAMES, words, st0)
    assert verdict == 0 and (fin == st).all()
    lib.jagged_round_free(key["round"])
    lib.machine_free(mach)
    lib.close()
