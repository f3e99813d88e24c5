"""GPU tests of a shard's memory chips (sp1b200_memory_traces): the MemoryGlobalInit, MemoryGlobalFinalize and MemoryLocal traces equal
the NumPy restatement (tests/memory_ref.py) word for word, from host and device memory into host and device outputs; a permuted init /
finalize input gives the same words; the emitted byte lookups and global events equal the restatement's, record for record; every
malformed input is an error that names its event and leaves the context usable; a poisoned pool gives the same words.  End to end, the
traces and the Byte / Range tables counted from the emitted lookups satisfy the chips' constraints (hand-lowered from their evals),
balance every Byte, Memory and Global interaction, and give a shard proof that verifies."""
import ctypes as C

import numpy as np
import pytest

from tests import lookup_ref as LR
from tests import machines as M
from tests import memory_ref as MR

pytestmark = pytest.mark.gpu
P = MR.P
A48 = 1 << 48


def _lib(**params):
    from sp1_b200 import Lib
    return Lib(0, **params)


def _addrs(n, rng, lo):
    """n distinct addresses in (lo, 2^48) in random order: a third uniform (differing in limb 2), a third dense above lo (limb 0) and a third
    on a 2^16 stride above lo (limb 1)"""
    k = n + n // 4 + 64
    cand = np.concatenate([rng.integers(lo + 1, A48, k, dtype=np.uint64),
                           np.uint64(lo + 1) + rng.integers(0, 4 * k, k, dtype=np.uint64),
                           np.uint64(lo + 1) + (rng.integers(0, 4 * k, k, dtype=np.uint64) << np.uint64(16))])
    u = np.unique(cand)
    u = u[u < np.uint64(A48)]
    return u[rng.choice(u.size, n, replace=False)]


def _u64(rng, n, bits=64):
    return rng.integers(0, 1 << bits, n, dtype=np.uint64, endpoint=False)


def _global_events(n, rng, previous, with_zero):
    """n init / finalize events after `previous`; with_zero (previous 0): address 0, with value 0, is one of them"""
    from sp1_b200.lib import pack_memory_events
    if n == 0:
        return pack_memory_events(np.zeros(0, np.uint64), 0, 0)
    addrs = _addrs(n - 1, rng, previous) if with_zero else _addrs(n, rng, previous)
    values = _u64(rng, addrs.size)
    if with_zero:
        addrs, values = np.append(addrs, np.uint64(0)), np.append(values, np.uint64(0))
    ev = pack_memory_events(addrs, values, _u64(rng, addrs.size, 48))
    return ev[rng.permutation(ev.size)]


def _local_events(n, rng):
    from sp1_b200.lib import pack_memory_local_events
    return pack_memory_local_events(_u64(rng, n, 48), _u64(rng, n, 48), _u64(rng, n), _u64(rng, n, 48), _u64(rng, n))


def _dev(recs):
    import torch
    return torch.from_numpy(recs.view(np.uint8).reshape(-1).copy()).cuda()


def _shape_out(init, fin, local, device):
    """five zeroed outputs of the sizes the call reports: host arrays or device tensors"""
    import torch
    from sp1_b200.lib import BYTE_LOOKUP_DTYPE, GLOBAL_EVENT_DTYPE
    n = (init.size, fin.size, local.size)
    h = [MR.num_rows(x) for x in n]
    n_lk, n_ge = 12 * (n[0] + n[1]) + 10 * n[2], n[0] + n[1] + 2 * n[2]
    if not device:
        return (np.zeros((30, h[0]), np.uint32), np.zeros((30, h[1]), np.uint32), np.zeros((20, h[2]), np.uint32),
                np.zeros(n_lk, BYTE_LOOKUP_DTYPE), np.zeros(n_ge, GLOBAL_EVENT_DTYPE))
    t = lambda *s: torch.zeros(s, dtype=torch.int32, device="cuda")
    b = lambda nb: torch.zeros(nb, dtype=torch.uint8, device="cuda")
    return (t(30, h[0]), t(30, h[1]), t(20, h[2]), b(n_lk * BYTE_LOOKUP_DTYPE.itemsize), b(n_ge * GLOBAL_EVENT_DTYPE.itemsize))


def _host(out):
    """the five outputs as host arrays (traces uint32, records in their dtypes)"""
    from sp1_b200.lib import BYTE_LOOKUP_DTYPE, GLOBAL_EVENT_DTYPE
    if isinstance(out[0], np.ndarray):
        return out
    tr = tuple(o.cpu().numpy().view(np.uint32) for o in out[:3])
    return tr + (out[3].cpu().numpy().view(BYTE_LOOKUP_DTYPE), out[4].cpu().numpy().view(GLOBAL_EVENT_DTYPE))


def _run(lib, init, fin, pi, pf, local, in_dev=False, out_dev=False):
    args = (_dev(init), _dev(fin), pi, pf, _dev(local)) if in_dev else (init, fin, pi, pf, local)
    out = _shape_out(init, fin, local, out_dev)
    return _host(lib.memory_traces(*args, out=out))


def _lookup_rows(recs):
    """emitted records with a non-zero count -> [(opcode, a, b, c)], in order"""
    keep = recs["count"] != 0
    assert (recs["count"][keep] == 1).all()
    return np.stack([recs[f][keep].astype(np.int64) for f in ("opcode", "a", "b", "c")], axis=1)


def _check(got, init, fin, pi, pf, local, lookups=True):
    want = MR.shard(init, fin, pi, pf, local) if lookups else None
    traces = (MR.global_trace(init, pi), MR.global_trace(fin, pf), MR.local_trace(local)) if want is None else want["traces"]
    for name, g, t in zip(("MemoryGlobalInit", "MemoryGlobalFinalize", "MemoryLocal"), got[:3], traces):
        w = MR.main_words(t)
        assert g.shape == w.shape, (name, g.shape, w.shape)
        bad = np.argwhere(g != w)
        assert bad.size == 0, f"{name}: first differing (column, row) {bad[:4].tolist()}"
    n_i, n_f, n_l = init.size, fin.size, local.size
    assert got[3].size == 12 * (n_i + n_f) + 10 * n_l and got[4].size == n_i + n_f + 2 * n_l
    g = got[4]
    if want is None:
        gi, gf = MR.global_interaction_events(init, False), MR.global_interaction_events(fin, True)
        gl = MR.local_dependencies(local)[1:]
        msg, rcv, kind = (np.concatenate([gi[k], gf[k], gl[k]]) for k in range(3))
    else:
        msg, rcv, kind = want["globals"]
    assert (g["message"] == msg).all() and (g["is_receive"] == rcv).all() and (g["kind"] == kind).all() and not g["pad"].any()
    if want is not None:
        # record for record once the count-0 placeholders (rows that compare nothing) are dropped
        assert (_lookup_rows(got[3]) == want["lookups"]).all()
        zero = got[3][got[3]["count"] == 0]
        assert zero.size == int(pi == 0 and n_i > 0) + int(pf == 0 and n_f > 0)


@pytest.mark.parametrize("n", [1, 15, 16, 17, 31, 32, 33, 1000, 1 << 20])
def test_tables_match_the_restatement(n):
    rng = np.random.default_rng(n)
    zero_init = n % 2 == 1                      # previous address zero (address 0 present) on one chip, non-zero on the other
    pi = 0 if zero_init else int(rng.integers(1, 1 << 47))
    pf = int(rng.integers(1, 1 << 47)) if zero_init else 0
    init, fin = _global_events(n, rng, pi, pi == 0), _global_events(n, rng, pf, pf == 0)
    local = _local_events(n, rng)
    lib = _lib()
    got = _run(lib, init, fin, pi, pf, local)
    _check(got, init, fin, pi, pf, local)
    dev = _run(lib, init, fin, pi, pf, local, in_dev=True, out_dev=True)
    assert all((a == b).all() for a, b in zip(got, dev))
    if n <= 1000:
        mixed = _run(lib, init, fin, pi, pf, local, in_dev=False, out_dev=True)
        assert all((a == b).all() for a, b in zip(got, mixed))
    # a permuted init / finalize input gives identical words, lookups and global events
    perm = _run(lib, init[rng.permutation(n)], fin[rng.permutation(n)], pi, pf, local)
    assert all((a == b).all() for a, b in zip(got, perm))
    lib.close()


def test_large_init_set_and_empty_chips():
    rng = np.random.default_rng(22)
    init = _global_events(1 << 22, rng, 0, True)
    empty = _global_events(0, rng, 0, False)
    none = _local_events(0, rng)
    lib = _lib()
    got = _run(lib, init, empty, 0, 0, none, in_dev=True, out_dev=True)
    assert got[1].shape == (30, 0) and got[2].shape == (20, 0)
    _check(got, init, empty, 0, 0, none, lookups=False)
    # lookups of the large set: the emitted stream counted by sp1b200_lookup_traces gives the restatement's Range and Byte tables
    lk = got[3]
    assert (lk["count"] == 1).sum() == 12 * init.size - 1
    ev = _sorted_rows(init, 0)
    want_range = np.zeros(1 << 17, np.int64)
    want_range[1 << 16:] = sum(np.bincount(limbs, minlength=1 << 16) for limbs in ev["range_limbs"])
    byte, _, rng_t = lib.lookup_traces(0, 1, _dev(lk), None)
    assert (rng_t[0] == LR.to_monty(want_range.astype(np.uint64))).all()
    want_u8 = np.bincount(ev["u8"], minlength=1 << 16)
    assert (byte[3] == LR.to_monty(want_u8.astype(np.uint64))).all() and not np.delete(byte, 3, axis=0).any()
    lib.close()


def _sorted_rows(init, previous):
    """the Range(16) values and U8Range rows of generate_dependencies over a large set, without building the per-record list"""
    ev = init[np.argsort(init["addr"], kind="stable")]
    prev = np.concatenate([np.array([previous], np.uint64), ev["addr"][:-1]])
    v, p, a = MR.u64_to_u16_limbs(ev["value"]), MR.u64_to_u16_limbs(prev), MR.u64_to_u16_limbs(ev["addr"])
    _, _, _, _, range_a = MR.populate_unsigned(prev, ev["addr"])
    comp = (np.arange(ev.size) != 0) | (prev != 0)
    limbs = [v[k] for k in range(4)] + [p[k] for k in range(3)] + [a[k] for k in range(3)] + [range_a[comp]]
    u8 = (((ev["value"] >> np.uint64(32)) & np.uint64(0xFF)) << np.uint64(8)) | ((ev["value"] >> np.uint64(40)) & np.uint64(0xFF))
    return dict(range_limbs=[x.astype(np.int64) for x in limbs], u8=u8.astype(np.int64))


def test_lookups_give_the_restated_byte_and_range_tables():
    """the emitted lookups, as a multiset of keys with counts, give sp1b200_lookup_traces the restatement's Byte and Range tables"""
    from sp1_b200.lib import pack_byte_lookups
    rng = np.random.default_rng(23)
    init, fin = _global_events(5000, rng, 0, True), _global_events(3000, rng, 12345, False)
    local = _local_events(4000, rng)
    lib = _lib()
    got = _run(lib, init, fin, 0, 12345, local, in_dev=True, out_dev=True)
    want = MR.shard(init, fin, 0, 12345, local)["lookups"]
    recs = pack_byte_lookups(want[:, 0], want[:, 1], want[:, 2], want[:, 3], 1)
    w_byte, _, w_range = LR.main_words(0, 1, recs, _no_pcs())
    byte, _, rng_t = lib.lookup_traces(0, 1, got[3], None)
    assert (byte == w_byte).all() and (rng_t == w_range).all()
    lib.close()


def _no_pcs():
    from sp1_b200.lib import pack_pc_counts
    return pack_pc_counts(np.zeros(0, np.uint64), np.zeros(0, np.uint32))


def test_errors_name_the_event_and_leave_the_context_usable():
    from sp1_b200.lib import Sp1B200Error
    rng = np.random.default_rng(24)
    lib = _lib()
    init, fin, local = _global_events(300, rng, 0, True), _global_events(200, rng, 0x5000, False), _local_events(100, rng)

    def fine():
        _check(_run(lib, init, fin, 0, 0x5000, local), init, fin, 0, 0x5000, local)

    def with_(recs, i, **kv):
        x = recs.copy()
        for k, v in kv.items():
            x[k][i] = v
        return x
    dup = with_(fin, 150, addr=fin["addr"][17])
    low = with_(fin, 9, addr=0x5000)
    below = with_(fin, 9, addr=0x4FFF)
    cases = [((with_(init, 17, addr=A48), fin, 0, 0x5000, local), "init event 17 has address 0x1000000000000 >= 2\\^48"),
             ((init, with_(fin, 3, timestamp=A48 + 5), 0, 0x5000, local), "finalize event 3 has timestamp 0x1000000000005 >= 2\\^48"),
             ((init, fin, 0, 0x5000, with_(local, 42, addr=A48 | 7)), "local event 42 has address 0x1000000000007 >= 2\\^48"),
             ((init, fin, 0, 0x5000, with_(local, 7, final_timestamp=A48)), "local event 7 has final timestamp 0x1000000000000"),
             ((init, fin, 0, 0x5000, with_(local, 8, initial_timestamp=1 << 63)), "local event 8 has initial timestamp 0x8000000000000000"),
             ((init, dup, 0, 0x5000, local), f"duplicate finalize address {hex(int(fin['addr'][17]))} \\(event (17|150)\\)"),
             ((init, low, 0, 0x5000, local), "finalize event 9 has address 0x5000, not above previous_finalize_addr 0x5000"),
             ((init, below, 0, 0x5000, local), "finalize event 9 has address 0x4fff, not above previous_finalize_addr 0x5000"),
             ((with_(init, int(np.nonzero(init["addr"])[0][0]), addr=0), fin, 0, 0x5000, local), "duplicate init address 0x0"),
             ((init, fin, A48, 0x5000, local), "previous_init_addr 0x1000000000000 >= 2\\^48")]
    for args, msg in cases:
        with pytest.raises(Sp1B200Error, match=msg):
            lib.memory_traces(*args)
        fine()
    # NULL arrays with a non-zero count, too many events, and a NULL output where one is needed
    a = np.zeros(64, np.uint64)
    p = C.c_void_p(a.ctypes.data)
    u, z = C.c_uint64, C.c_uint64(0)
    rows, nl, ng = (C.c_uint64 * 3)(), C.c_uint64(), C.c_uint64()
    outs = [p, p, p, p, p]
    for ins, outs_, msg in (((None, u(5), None, z, None, z), outs, b"NULL init event array with 5 events"),
                            ((None, z, None, u(2), None, z), outs, b"NULL finalize event array with 2 events"),
                            ((None, z, None, z, None, u(9)), outs, b"NULL local event array with 9 events"),
                            ((p, u(1 << 31), None, z, None, z), outs, b"2147483648 init events; at most 2^31 - 1"),
                            ((None, z, None, z, p, u(1)), [None, None, None, p, p], b"NULL local trace output for 32 rows")):
        e = lib.L.sp1b200_memory_traces(lib.ctx, ins[0], ins[1], ins[2], ins[3], z, z, ins[4], ins[5], *outs_, rows, C.byref(nl), C.byref(ng))
        assert e and msg in e, e
        fine()
    # NULL outputs only report the sizes
    assert not lib.L.sp1b200_memory_traces(lib.ctx, p, u(3), p, u(2), z, z, p, u(40), None, None, None, None, None, rows, C.byref(nl),
                                           C.byref(ng))
    assert list(rows) == [32, 32, 64] and nl.value == 12 * 5 + 400 and ng.value == 5 + 80
    lib.close()


def test_poisoned_pool_gives_the_same_words():
    """every block of the context's pool holds a non-zero pattern before the call (a freed pool keeps its blocks)"""
    rng = np.random.default_rng(25)
    init, fin, local = _global_events(1 << 16, rng, 0, True), _global_events(5000, rng, 77, False), _local_events(20000, rng)
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
    _check(_run(lib, init, fin, 0, 77, local), init, fin, 0, 77, local)
    _check(_run(lib, init, fin, 0, 77, local, in_dev=True, out_dev=True), init, fin, 0, 77, local)
    lib.close()


# ---- end to end: the memory chips' constraints and interactions, hand-lowered from their evals ---------------------------------------
NAMES = ["Byte", "Cpu", "Global", "MemoryGlobalFinalize", "MemoryGlobalInit", "MemoryLocal", "Program", "Range"]
KIND_MEMORY, KIND_PROGRAM, KIND_BYTE, KIND_GLOBAL, KIND_INIT_CONTROL, KIND_FINALIZE_CONTROL = 1, 2, 5, 9, 14, 15   # InteractionKind
CPU_W, GLOBAL_W = 1 + 9 + 9 + 1, 1 + 11


class _Air:
    """a chip's constraints in synth_air.Asm words: each helper returns a register"""

    def __init__(self):
        from sp1_b200 import synth_air as SA
        self.SA, self.a = SA, SA.Asm()

    def col(self, k):
        return self.a.leaf(self.SA.LEAF_MAIN, k)

    def k(self, v):
        return self.a.const(v % P)

    def add(self, *xs):
        r = xs[0]
        for x in xs[1:]:
            r = self.a.op(self.SA.ADD, r, x)
        return r

    def sub(self, x, y):
        return self.a.op(self.SA.SUB, x, y)

    def mul(self, *xs):
        r = xs[0]
        for x in xs[1:]:
            r = self.a.op(self.SA.MUL, r, x)
        return r

    def zero(self, x):
        self.a.assert_zero(x)

    def eq(self, x, y):
        self.zero(self.sub(x, y))

    def bool(self, x):
        self.zero(self.mul(x, self.sub(x, self.k(1))))

    def is_zero(self, a, inv, res, real):
        """IsZeroOperation::eval_is_zero (is_zero.rs:59-83)"""
        self.zero(self.mul(real, self.sub(self.sub(self.k(1), self.mul(inv, a)), res)))
        self.zero(self.mul(real, res, self.sub(res, self.k(1))))
        self.zero(self.mul(real, res, a))


def _global_chip_words():
    """MemoryGlobalChip::eval (global.rs:307-473) with IsZeroOperation, LtOperationUnsigned::eval_lt_unsigned (slt.rs:200-269) and
    U16CompareOperation::eval_compare_u16 (u16_compare.rs:48-72) inlined; interactions are separate"""
    c, A = MR.IC, _Air()
    col = lambda name: A.col(c[name])
    real = col("is_real")
    A.bool(real)
    A.eq(col("value[2]"), A.add(col("value_lower"), A.mul(col("value_upper"), A.k(1 << 8))))
    A.is_zero(A.add(col("prev_addr[0]"), col("prev_addr[1]"), col("prev_addr[2]")), col("is_prev_addr_zero.inverse"),
              col("is_prev_addr_zero.result"), real)
    A.is_zero(col("index"), col("is_index_zero.inverse"), col("is_index_zero.result"), real)
    comp = col("is_comp")
    A.eq(comp, A.mul(real, A.sub(A.k(1), A.mul(col("is_prev_addr_zero.result"), col("is_index_zero.result")))))
    A.bool(comp)
    # LtOperationUnsigned with b = prev_addr, c = addr (limb 3 zero), is_real = is_comp
    A.bool(comp)
    flags = [col(f"lt.u16_flags[{k}]") for k in range(4)]
    for f in flags:
        A.bool(f)
    sum_flags = A.add(*flags)
    A.bool(sum_flags)
    b = [col(f"prev_addr[{k}]") for k in range(3)] + [A.k(0)]
    cc = [col(f"addr[{k}]") for k in range(3)] + [A.k(0)]
    visited = A.k(0)
    b_cmp, c_cmp = A.k(0), A.k(0)
    for k in (3, 2, 1, 0):
        visited = A.add(visited, flags[k])
        A.zero(A.mul(A.sub(comp, visited), A.sub(b[k], cc[k])))
        b_cmp = A.add(b_cmp, A.mul(b[k], flags[k]))
        c_cmp = A.add(c_cmp, A.mul(cc[k], flags[k]))
    bl, cl = col("lt.comparison_limbs[0]"), col("lt.comparison_limbs[1]")
    A.eq(b_cmp, bl)
    A.eq(c_cmp, cl)
    A.zero(A.mul(sum_flags, A.sub(A.mul(col("lt.not_eq_inv"), A.sub(bl, cl)), comp)))
    A.bool(comp)                                                 # U16CompareOperation
    A.bool(col("lt.bit"))
    A.zero(A.mul(comp, A.sub(col("lt.bit"), A.k(1))))           # when(is_comp).assert_one(bit)
    not_comp = A.sub(real, comp)
    A.zero(A.mul(not_comp, A.add(col("addr[0]"), col("addr[1]"), col("addr[2]"))))
    for k in range(4):
        A.zero(A.mul(not_comp, col(f"value[{k}]")))
    return A.a.words(MR.NUM_MEMORY_INIT_COLS, 0)


def _local_chip_words():
    """MemoryLocalChip::eval (local.rs:257-359)"""
    c, A = MR.LC, _Air()
    col = lambda name: A.col(c[name])
    real = col("is_real")
    A.bool(real)
    A.eq(A.mul(real, real, real), A.mul(real, real, real))
    for w in ("initial", "final"):
        A.eq(col(f"{w}_value[2]"), A.add(col(f"{w}_value_lower"), A.mul(col(f"{w}_value_upper"), A.k(1 << 8))))
    return A.a.words(MR.NUM_MEMORY_LOCAL_INIT_COLS, 0)


def _interactions(chains):
    """per chip in NAMES order: [(is_send, kind, mult vcol, [value vcols])].  chains: [(kind, first receive, last send)] of the two control
    chains, which the Cpu closes with multiplicity column 19 (in a real shard the verifier closes them from the public values)"""
    from sp1_b200 import synth_air as SA
    prep, main = SA.LEAF_PREP, SA.LEAF_MAIN
    m = lambda k: SA._vcol([(main, k, 1)])
    pc_ = lambda k: SA._vcol([(prep, k, 1)])
    lin = lambda *terms: SA._vcol([(main, k, w % P) for k, w in terms])
    cst = lambda v: SA._vcol([], constant=v)
    send_byte = lambda mult, op, a, b, c: (1, KIND_BYTE, mult, [op, a, b, c])
    # Byte / Range / Program receives (bytes/air.rs, range/air.rs, trusted.rs:311-322)
    b, c = pc_(0), pc_(1)
    byte = [(0, KIND_BYTE, m(0), [cst(0), pc_(2), b, c]), (0, KIND_BYTE, m(1), [cst(1), pc_(3), b, c]),
            (0, KIND_BYTE, m(2), [cst(2), pc_(4), b, c]), (0, KIND_BYTE, m(3), [cst(3), cst(0), b, c]),
            (0, KIND_BYTE, m(4), [cst(4), pc_(5), b, c]), (0, KIND_BYTE, m(5), [cst(5), pc_(6), b, cst(0)])]
    rng_ = [(0, KIND_BYTE, m(0), [cst(6), pc_(0), pc_(1), cst(0)])]
    prog = [(0, KIND_PROGRAM, m(0), [pc_(k) for k in range(16)])]
    # a Cpu that sends the local events' initial accesses and receives their final ones; a Global that receives every global message
    cpu = [(1, KIND_MEMORY, m(0), [m(k) for k in range(1, 10)]), (0, KIND_MEMORY, m(0), [m(k) for k in range(10, 19)])]
    for kind, first, last in chains:
        cpu += [(1, kind, m(19), [cst(v) for v in first]), (0, kind, m(19), [cst(v) for v in last])]
    glob = [(0, KIND_GLOBAL, m(0), [m(k) for k in range(1, 12)])]

    def memory_global(kind):
        ic = MR.IC
        g = lambda name: m(ic[name])
        real = g("is_real")
        inter = [send_byte(real, cst(6), g(f"value[{k}]"), cst(16), cst(0)) for k in range(4)]
        inter += [send_byte(real, cst(6), g(f"prev_addr[{k}]"), cst(16), cst(0)) for k in range(3)]
        inter += [send_byte(real, cst(6), g(f"addr[{k}]"), cst(16), cst(0)) for k in range(3)]
        inter += [send_byte(real, cst(3), cst(0), g("value_lower"), g("value_upper"))]
        control = KIND_INIT_CONTROL if kind == "init" else KIND_FINALIZE_CONTROL
        inter += [(0, control, real, [g("index")] + [g(f"prev_addr[{k}]") for k in range(3)] + [g("prev_valid")])]
        inter += [(1, control, real, [SA._vcol([(main, ic["index"], 1)], constant=1)] + [g(f"addr[{k}]") for k in range(3)] + [g("is_comp")])]
        clk = [cst(0), cst(0)] if kind == "init" else [g("clk_high"), g("clk_low")]
        flags = [cst(1), cst(0)] if kind == "init" else [cst(0), cst(1)]
        inter += [(1, KIND_GLOBAL, real, clk + [g(f"addr[{k}]") for k in range(3)]
                   + [lin((ic["value[0]"], 1), (ic["value_lower"], 1 << 16)), lin((ic["value[1]"], 1), (ic["value_upper"], 1 << 16)),
                      g("value[3]")] + flags + [cst(KIND_MEMORY)])]
        inter += [send_byte(g("is_comp"), cst(6), lin((ic["lt.comparison_limbs[0]"], 1), (ic["lt.comparison_limbs[1]"], -1),
                                                      (ic["lt.bit"], 1 << 16)), cst(16), cst(0))]
        return inter

    lc = MR.LC
    lo = lambda name: m(lc[name])
    real = lo("is_real")
    local = []
    for w, is_receive in (("initial", 1), ("final", 0)):
        local += [send_byte(real, cst(3), cst(0), lo(f"{w}_value_lower"), lo(f"{w}_value_upper"))]
        local += [send_byte(real, cst(6), lo(f"{w}_value[{k}]"), cst(16), cst(0)) for k in range(4)]
        access = [lo(f"{w}_clk_high"), lo(f"{w}_clk_low")] + [lo(f"addr[{k}]") for k in range(3)] + [lo(f"{w}_value[{k}]") for k in range(4)]
        local += [(1 - is_receive, KIND_MEMORY, real, access)]
        local += [(1, KIND_GLOBAL, real, access[:5] + [lin((lc[f"{w}_value[0]"], 1), (lc[f"{w}_value_lower"], 1 << 16)),
                                                       lin((lc[f"{w}_value[1]"], 1), (lc[f"{w}_value_upper"], 1 << 16)),
                                                       lo(f"{w}_value[3]"), cst(1 - is_receive), cst(is_receive), cst(KIND_MEMORY)])]
    return [byte, cpu, glob, memory_global("finalize"), memory_global("init"), local, prog, rng_]


def _machine(chains):
    from sp1_b200 import synth_air as SA
    g = _global_chip_words()
    words = [SA.Asm().words(6, 7), SA.Asm().words(CPU_W, 0), SA.Asm().words(GLOBAL_W, 0), g, g, _local_chip_words(), SA.Asm().words(1, 16),
             SA.Asm().words(1, 2)]
    return SA.machine_blob_with_interactions(words, [M._inter_words(x) for x in _interactions(chains)])


def test_traces_satisfy_the_chips_and_prove():
    import torch
    from sp1_b200.lib import GLOBAL_EVENT_DTYPE, MAX_OPCODE, HostChallenger, pack_instructions
    from tests import oracle_lib as O
    rng = np.random.default_rng(26)
    n_instrs = 100
    instrs = pack_instructions(rng.integers(0, MAX_OPCODE + 1, n_instrs), rng.integers(0, 32, n_instrs), _u64(rng, n_instrs),
                               _u64(rng, n_instrs), rng.integers(0, 2, n_instrs), rng.integers(0, 2, n_instrs))
    pc_base, pf = 0x20000, int(rng.integers(1, 1 << 40))
    init, fin, local = _global_events(1000, rng, 0, True), _global_events(700, rng, pf, False), _local_events(500, rng)
    lib = _lib(log_stacking_height=16, max_log_row_count=17, **M.SMALL)
    key = lib.program_setup(pc_base, instrs, pc_base, np.zeros(0, np.uint64), np.zeros(0, np.uint64))
    limbs = lambda x: tuple((int(x) >> (16 * k)) & 0xFFFF for k in range(3))
    chains = [(KIND_INIT_CONTROL, (0,) + limbs(0) + (1,), (init.size,) + limbs(np.max(init["addr"])) + (1,)),
              (KIND_FINALIZE_CONTROL, (0,) + limbs(pf) + (1,), (fin.size,) + limbs(np.max(fin["addr"])) + (1,))]
    mach = lib.machine_create(_machine(chains))
    h_mem = [MR.num_rows(x) for x in (init.size, fin.size, local.size)]
    n_globals = init.size + fin.size + 2 * local.size
    heights = [1 << 16, h_mem[2], MR.num_rows(n_globals), h_mem[1], h_mem[0], h_mem[2], key["prep_rows"][1], 1 << 17]
    widths = [6, CPU_W, GLOBAL_W, 30, 30, 20, 1, 1]
    offs = [0] + [int(x) for x in np.cumsum([w * h for w, h in zip(widths, heights)])]
    dense = torch.zeros(offs[-1], dtype=torch.int32, device="cuda")
    view = lambda k: dense[offs[k]:offs[k + 1]].view(widths[k], heights[k])
    lookups, globals_ = _shape_out(init, fin, local, True)[3:]
    lib.memory_traces(_dev(init), _dev(fin), 0, pf, _dev(local), out=(view(4), view(3), view(5), lookups, globals_))
    lib.lookup_traces(pc_base, n_instrs, lookups, None, None, out=(view(0), view(6), view(7)))
    # the synthetic Cpu and Global traces (canonical), from the events and the emitted global records
    cpu = np.zeros((CPU_W, heights[1]), np.uint64)
    cpu[0, :local.size] = 1
    lt = MR.local_trace(local)
    for j, w in enumerate(("initial", "final")):
        names = [f"{w}_clk_high", f"{w}_clk_low"] + [f"addr[{k}]" for k in range(3)] + [f"{w}_value[{k}]" for k in range(4)]
        for k, name in enumerate(names):
            cpu[1 + 9 * j + k, :local.size] = lt[:local.size, MR.LC[name]]
    ge = globals_.cpu().numpy().view(GLOBAL_EVENT_DTYPE)
    glob = np.zeros((GLOBAL_W, heights[2]), np.uint64)
    glob[0, :n_globals] = 1
    glob[1:9, :n_globals] = ge["message"].T
    glob[9, :n_globals] = 1 - ge["is_receive"].astype(np.uint64)
    glob[10, :n_globals] = ge["is_receive"]
    glob[11, :n_globals] = ge["kind"]
    for k, t in ((1, cpu), (2, glob)):
        view(k)[:] = torch.from_numpy(O.to_monty(t.reshape(-1)).view(np.int32).reshape(t.shape)).cuda()
    pv = np.zeros(187, np.uint32)
    assert lib.debug_constraints(mach, key["round"], dense, heights, pv) == {}
    # one changed not_eq_inv word: exactly that chip and row fail
    r, k = 517, MR.IC["lt.not_eq_inv"]
    saved = int(view(4)[k, r])
    changed = int(O.to_monty(np.array([12345], np.uint64))[0])
    assert changed != saved
    view(4)[k, r] = changed
    rep = lib.debug_constraints(mach, key["round"], dense, heights, pv)
    assert list(rep) == [NAMES.index("MemoryGlobalInit")] and list(rep[NAMES.index("MemoryGlobalInit")]["rows"]) == [r], rep
    view(4)[k, r] = saved
    assert lib.debug_constraints(mach, key["round"], dense, heights, pv) == {}
    # with the Cpu's closing column zero, the only unbalanced keys are the ends of the two control chains; nothing of kind Byte, Memory
    # or Global
    rep = lib.debug_interactions(mach, key["round"], dense, heights)
    got = sorted((k["kind"], tuple(int(v) for v in O.from_monty(np.asarray(k["values"], np.uint32))),
                  int(O.from_monty(np.array([k["net"]], np.uint32))[0])) for k in rep["keys"])
    want = sorted([(kind, first, P - 1) for kind, first, _ in chains] + [(kind, last, 1) for kind, _, last in chains])
    assert rep["n_unbalanced"] == 4 and got == want, rep
    view(1)[19, 0] = int(O.to_monty(np.array([1], np.uint64))[0])
    assert lib.debug_interactions(mach, key["round"], dense, heights)["n_unbalanced"] == 0
    hc = HostChallenger(); hc.observe(key["prep_commit"]); hc.observe(key["vk_tail"])
    st0 = hc.st.copy()
    st = st0.copy()
    words = lib.prove_shard(mach, key["round"], dense, heights, NAMES, pv, st)
    verdict, fin_st = lib.verify_shard(mach, key["prep_commit"], heights, NAMES, words, st0)
    assert verdict == 0 and (fin_st == st).all()
    lib.jagged_round_free(key["round"])
    lib.machine_free(mach)
    lib.close()
