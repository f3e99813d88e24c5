"""The program setup's hash-to-curve and curve sum against the reference's own primitives: kb31_septic_extension_t::curve_formula / pow_r /
sqrt / is_exception / is_receive, bb31_septic_curve_t::operator+= and poseidon2::KoalaBearHasher::permute, compiled unmodified
(oracle/ref_lift.mk) under a SepticCurve::lift_x trial loop and run on seeded inputs.  Their outputs are stored in tests/golden/ref_lift.json,
so this runs on the CPU: the library's device code compiled for the host (sp1_b200/csrc/septic.cuh, through libsp1b200_hostcheck.so) and
the oracle's restatement of the Rust (oracle/lift.hpp) must equal them word for word.  Recording needs a GPU and
oracle/_ref/libsp1ref_lift.so: `SP1B200_RECORD_REF=1 python -m pytest tests/test_ref_lift.py`."""
import ctypes as C
import os

import numpy as np

from tests import lift_oracle_lib as LO
from tests import oracle_lib as O
from tests import ref_golden as RG
from tests import septic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STORE = RG.Store("ref_lift", "tests/test_ref_lift.py")
# the message of the Rust test_lift_x (crates/hypercube/src/septic_curve.rs:261-276)
RUST_TEST_MSG = [0x2013, 0x2015, 0x2016, 0x2023, 0x2024, 0x2016, 0x2017, 0]


def _memory_msg(addr, w):
    return [1 << 24, 0, addr & 0xFFFF, (addr >> 16) & 0xFFFF, (addr >> 32) & 0xFFFF, (w & 0xFFFF) + (1 << 16) * ((w >> 32) & 0xFF),
            ((w >> 16) & 0xFFFF) + (1 << 16) * ((w >> 40) & 0xFF), (w >> 48) & 0xFFFF]


def _page_msg(idx, prot):
    return [19 << 24, 0, idx & 0xF, (idx >> 4) & 0xFFFF, (idx >> 20) & 0xFFFF, prot, 0, 0]


def _neg(p):
    return (p[0], [(-v) % S.P for v in p[1]])


def _inputs():
    rng = np.random.default_rng(2027)
    msgs = [RUST_TEST_MSG]
    msgs += [[int(v) for v in rng.integers(0, O.P, 8)] for _ in range(200)]
    msgs += [_memory_msg(int(a), int(w)) for a, w in zip(rng.integers(0, 1 << 48, 80, dtype=np.uint64),
                                                         rng.integers(0, 1 << 63, 80, dtype=np.uint64))]
    msgs += [_page_msg(int(i), int(p)) for i, p in zip(rng.integers(0, 1 << 36, 20, dtype=np.uint64), rng.integers(0, 8, 20))]
    msgs = np.stack([S.mont(m) for m in msgs])
    ys = [[int(v) for v in rng.integers(0, O.P, 7)] for _ in range(48)]
    sq = np.stack([S.mont(S.smul(y, y)) for y in ys[:32]] + [S.mont(y) for y in ys[32:]])   # 32 squares, 16 of either kind
    mult = S.multiples(S.DUMMY, 12)
    pairs = [(mult[i], mult[j]) for i in range(6) for j in range(6, 12)]            # chords
    pairs += [(m, m) for m in mult[:6]] + [(S.ZERO, S.ZERO)]                          # tangents
    pairs += [(m, _neg(m)) for m in mult[:6]]                                         # P + (-P)
    inf = ([0] * 7, [0] * 7)
    pairs += [(inf, m) for m in mult[:3]] + [(m, inf) for m in mult[3:6]] + [(inf, inf)]
    p = np.stack([S.pt_words(a) for a, _ in pairs]); q = np.stack([S.pt_words(b) for _, b in pairs])
    return msgs, sq, p, q


def _run_reference(msgs, sq, p, q):
    L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libsp1ref_lift.so"))
    L.ref_lift.restype = C.c_char_p
    off, pts = np.zeros(msgs.shape[0], np.int32), np.zeros((msgs.shape[0], 14), np.uint32)
    roots, ok = np.zeros_like(sq), np.zeros(sq.shape[0], np.uint32)
    s = np.zeros_like(p)
    P = lambda x: C.c_void_p(x.ctypes.data)
    e = L.ref_lift(P(msgs), C.c_uint32(msgs.shape[0]), P(off), P(pts), P(sq), C.c_uint32(sq.shape[0]), P(roots), P(ok), P(p), P(q),
                   C.c_uint32(p.shape[0]), P(s))
    assert not e, e.decode()
    return dict(offsets=off.view(np.uint32), points=pts, roots=roots, is_square=ok, sums=s)


_REF = None


def ref():
    """name -> reference output words (live while recording, stored otherwise)"""
    global _REF
    if _REF is None:
        live = _run_reference(*_inputs()) if RG.RECORD else {}
        _REF = {k: RG.Ref(k, (lambda k=k: live[k]), keep=True, store=STORE).words for k in ("offsets", "points", "roots", "is_square", "sums")}
        STORE.save()
    return _REF


def _host_lift(msgs):
    off, pts = np.zeros(msgs.shape[0], np.int32), np.zeros((msgs.shape[0], 14), np.uint32)
    S.lib().sp1b200_hostcheck_lift_x(S.ptr(msgs), C.c_void_p(off.ctypes.data), S.ptr(pts), C.c_uint64(msgs.shape[0]))
    return off, pts


def test_lift_matches_the_reference():
    msgs = _inputs()[0]
    R = ref()
    assert (R["offsets"].view(np.int32) >= 0).all()
    off, pts = _host_lift(msgs)
    assert (off.view(np.uint32) == R["offsets"]).all() and (pts.reshape(-1) == R["points"]).all()
    ooff, opts = LO.lift_x(msgs)
    assert (ooff.view(np.uint32) == R["offsets"]).all() and (opts.reshape(-1) == R["points"]).all()


def test_lifted_points_lie_on_the_curve_and_their_negations_are_sends():
    pts = ref()["points"].reshape(-1, 14)
    for w in pts:
        x, y = S.words_pt(w)
        assert S.on_curve((x, y))
        assert 1 <= y[6] <= 63 << 24                       # is_receive
        assert S.P - (63 << 24) <= (-y[6]) % S.P <= S.P - 1  # the negation, which enters the sum, is_send


def test_square_roots_match_the_reference():
    sq = _inputs()[1]
    R = ref()
    n = sq.shape[0]
    assert R["is_square"][:32].all() and 0 < R["is_square"][32:].sum() < 16
    roots, ok = np.zeros_like(sq), np.zeros(n, np.uint32)
    S.lib().sp1b200_hostcheck_septic_sqrt(S.ptr(sq), S.ptr(roots), S.ptr(ok), C.c_uint64(n))
    assert (ok == R["is_square"]).all() and (roots.reshape(-1) == R["roots"]).all()
    oroots, ook = LO.septic_sqrt(sq)
    assert (ook == R["is_square"]).all() and (oroots.reshape(-1) == R["roots"]).all()
    for a, r, k in zip(sq, roots, ok):
        if k:
            assert S.smul(S.canon(r), S.canon(r)) == S.canon(a)


def test_complete_addition_matches_the_reference():
    _, _, p, q = _inputs()
    R = ref()
    out = np.zeros_like(p)
    S.lib().sp1b200_hostcheck_curve_add_complete(S.ptr(p), S.ptr(q), S.ptr(out), C.c_uint64(p.shape[0]))
    assert (out.reshape(-1) == R["sums"]).all()
    assert (LO.curve_add_complete(p, q).reshape(-1) == R["sums"]).all()
    sums = R["sums"].reshape(-1, 14)
    assert not sums[43:49].any() and not sums[-1].any()      # P + (-P) and infinity + infinity are infinity
    assert (sums[49:55] == p[49:55] + q[49:55]).all()         # infinity is the identity (one side is all zeros)
