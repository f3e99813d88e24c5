"""The core-proof verifier's septic arithmetic against the reference's own: kb31_septic_extension_t / bb31_septic_curve_t of
sp1-gpu/crates/sys/include/fields/kb31_septic_extension_t.cuh, compiled unmodified (oracle/ref_septic.mk) and run on seeded inputs.
Their outputs are stored in tests/golden/ref_septic.json, so this runs on the CPU: the library's host code (sp1_b200/csrc/septic.hpp,
through libsp1b200_hostcheck.so) and the oracle's (oracle/core.hpp) must equal them word for word.  Recording needs a GPU and
oracle/_ref/libsp1ref_septic.so: `SP1B200_RECORD_REF=1 python -m pytest tests/test_ref_septic.py`."""
import ctypes as C
import os

import numpy as np

from tests import core_chain as CC
from tests import core_oracle_lib as CO
from tests import oracle_lib as O
from tests import ref_golden as RG
from tests import test_septic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STORE = RG.Store("ref_septic", "tests/test_ref_septic.py")
K = 12   # chain length


def _inputs():
    rng = np.random.default_rng(2026)
    n = 32
    a = np.stack([S.mont([int(x) for x in rng.integers(0, O.P, 7)]) for _ in range(n)])
    b = np.stack([S.mont([int(x) for x in rng.integers(0, O.P, 7)]) for _ in range(n)])
    mult = CC.multiples(S.DUMMY, 40)
    pairs = [(mult[i], mult[j]) for i in range(10) for j in range(10) if i != j and (i + j) % 3 == 0]
    p = np.stack([S.pt_words(x) for x, _ in pairs]); q = np.stack([S.pt_words(y) for _, y in pairs])
    ks = [int(k) for k in rng.integers(1, 8, 5)]
    pts = [S.curve_add(S.ZERO, S.curve_neg(mult[sum(ks) - 1]))] + [S.curve_add(S.ZERO, mult[k - 1]) for k in ks]
    return a, b, p, q, np.stack([S.pt_words(x) for x in pts])


def _run_reference(a, b, p, q, pts):
    so = os.path.join(ROOT, "oracle", "_ref", "libsp1ref_septic.so")
    L = C.CDLL(so)
    L.ref_septic.restype = C.c_char_p
    n, np_, m = a.shape[0], p.shape[0], pts.shape[0]
    mul, inv, add = np.zeros_like(a), np.zeros_like(a), np.zeros_like(p)
    cd, cs, s = np.zeros((K, 14), np.uint32), np.zeros((K, 14), np.uint32), np.zeros(14, np.uint32)
    P = lambda x: C.c_void_p(x.ctypes.data)
    e = L.ref_septic(P(a), P(b), C.c_uint32(n), P(mul), P(inv), P(p), P(q), C.c_uint32(np_), P(add), C.c_uint32(K), P(cd), P(cs),
                     P(pts), C.c_uint32(m), P(s))
    assert not e, e.decode()
    return dict(mul=mul, inv=inv, add=add, chain_dummy=cd, chain_start=cs, digest_sum=s)


_REF = None


def ref():
    """name -> reference output words (live while recording, stored otherwise)"""
    global _REF
    if _REF is None:
        live = _run_reference(*_inputs()) if RG.RECORD else {}
        _REF = {k: RG.Ref(k, (lambda k=k: live[k]), keep=True, store=STORE).words for k in
                ("mul", "inv", "add", "chain_dummy", "chain_start", "digest_sum")}
        STORE.save()
    return _REF


def test_mul_and_reciprocal_match_the_reference():
    a, b, _, _, _ = _inputs()
    n = a.shape[0]
    lm, li = np.zeros(7 * n, np.uint32), np.zeros(7 * n, np.uint32)
    S._lib().sp1b200_hostcheck_septic(S._p(a), S._p(b), S._p(lm), S._p(li), C.c_uint64(n))
    R = ref()
    assert (lm == R["mul"]).all() and (li == R["inv"]).all()
    assert (CO.septic_mul(a, b).reshape(-1) == R["mul"]).all() and (CO.septic_inv(a).reshape(-1) == R["inv"]).all()


def test_curve_addition_matches_the_reference():
    _, _, p, q, _ = _inputs()
    n = p.shape[0]
    out, ok = np.zeros(14 * n, np.uint32), np.zeros(n, np.uint32)
    S._lib().sp1b200_hostcheck_septic_curve_add(S._p(p), S._p(q), S._p(out), S._p(ok), C.c_uint64(n))
    R = ref()
    assert ok.all() and (out == R["add"]).all()
    oo, ook = CO.curve_add(p, q)
    assert ook.all() and (oo.reshape(-1) == R["add"]).all()


def test_constant_points_and_chains_match_the_reference():
    """dummy_point() and start_point() are the library's dummy point and zero digest; every k·P of both chains (from 3P on, where
    the reference's `+` is the chord) is the library's incomplete addition of (k-1)·P and P"""
    R = ref()
    const = np.zeros(42, np.uint32)
    S._lib().sp1b200_hostcheck_septic_constants(S._p(const))
    cd, cs = R["chain_dummy"].reshape(K, 14), R["chain_start"].reshape(K, 14)
    assert (cd[0] == const[28:42]).all() and (cs[0] == const[0:14]).all()
    for chain in (cd, cs):
        n = K - 2
        pw, qw = np.ascontiguousarray(chain[1:K - 1]), np.ascontiguousarray(np.repeat(chain[:1], n, 0))
        out, ok = np.zeros(14 * n, np.uint32), np.zeros(n, np.uint32)
        S._lib().sp1b200_hostcheck_septic_curve_add(S._p(pw), S._p(qw), S._p(out), S._p(ok), C.c_uint64(n))
        assert ok.all() and (out == chain[2:].reshape(-1)).all()
        for w in chain:
            assert S.on_curve(S.words_pt(w))


def test_digest_sum_matches_the_reference():
    """the SepticDigest additions of the core verifier (pairwise, as verify.rs:498-505 adds them) give the reference's group sum"""
    _, _, _, _, pts = _inputs()
    L = S._lib()
    acc, oacc = pts[0].copy(), pts[0].copy()
    for d in pts[1:]:
        out = np.zeros(14, np.uint32)
        assert L.sp1b200_hostcheck_septic_digest_add(S._p(acc), S._p(np.ascontiguousarray(d)), S._p(out)) == 1
        acc = out
        oacc = CO.digest_add(oacc, d)
    R = ref()
    assert (acc == R["digest_sum"]).all() and (oacc == R["digest_sum"]).all()
    assert S.words_pt(acc) == (S.ZERO[0], S.ZERO[1])   # the inputs cancel
