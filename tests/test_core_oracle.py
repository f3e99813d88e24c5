"""CPU tests of the oracle's restated core-proof verifier (oracle/core.hpp, orc_verify_core_proof) and its septic arithmetic: the
septic product, inverse, curve addition and digest addition of the oracle, of the library's host code (libsp1b200_hostcheck.so) and of
the Python restatement agree word for word; the oracle accepts an oracle-proved chain of shards and gives every crafted chain the
verdict and shard the library's verifier is required to give (tests/test_gpu_verify_core.py runs the same cases, core_chain.PV_CASES)."""
import ctypes as C

import numpy as np

from tests import core_chain as CC
from tests import core_oracle_lib as CO
from tests import machines as M
from tests import oracle_lib as O
from tests import septic as S


def test_septic_oracle_library_and_restatement_agree():
    rng = np.random.default_rng(31)
    n = 16
    a = [[int(x) for x in rng.integers(0, O.P, 7)] for _ in range(n)]
    b = [[int(x) for x in rng.integers(0, O.P, 7)] for _ in range(n)]
    A = np.stack([S.mont(x) for x in a]); B = np.stack([S.mont(x) for x in b])
    om, oi = CO.septic_mul(A, B), CO.septic_inv(A)
    lm, li = np.zeros(7 * n, np.uint32), np.zeros(7 * n, np.uint32)
    S.lib().sp1b200_hostcheck_septic(S.ptr(A), S.ptr(B), S.ptr(lm), S.ptr(li), C.c_uint64(n))
    assert (om.reshape(-1) == lm).all() and (oi.reshape(-1) == li).all()
    for i in range(n):
        assert S.canon(om[i]) == S.smul(a[i], b[i])
    pts = S.multiples(S.DUMMY, 6) + S.multiples(S.START, 3)
    pairs = [(p, q) for p in pts for q in pts]
    Pw = np.stack([S.pt_words(p) for p, _ in pairs]); Qw = np.stack([S.pt_words(q) for _, q in pairs])
    out, ok = CO.curve_add(Pw, Qw)
    lout, lok = np.zeros(14 * len(pairs), np.uint32), np.zeros(len(pairs), np.uint32)
    S.lib().sp1b200_hostcheck_septic_curve_add(S.ptr(Pw), S.ptr(Qw), S.ptr(lout), S.ptr(lok), C.c_uint64(len(pairs)))
    assert (ok == lok).all() and (ok == 0).sum() == len(pts)   # exactly the pairs p == q are exceptional
    for i, (p, q) in enumerate(pairs):
        if ok[i]:
            assert (out[i] == lout[14 * i:14 * i + 14]).all()
            assert S.words_pt(out[i]) == S.curve_add(p, q)
    d1, d2 = S.curve_add(S.ZERO, pts[1]), S.curve_add(S.ZERO, pts[4])
    od = CO.digest_add(S.pt_words(d1), S.pt_words(d2))
    assert S.words_pt(od) == S.digest_add(d1, d2)
    assert CO.digest_add(S.pt_words(S.START), S.pt_words(S.ZERO)) is None


class OracleChain:
    def __init__(self, chips, log_stack, mlr):
        self.blob, self.heights, _, _, _, self.names = M.spec_machine(np.random.default_rng(1), chips)
        self.specs, self.log_stack, self.mlr = chips, log_stack, mlr
        mains, preps = M.traces(self.specs, 5, 0)
        self.pc = np.zeros(8, np.uint32)
        if any(p is not None for p in preps):   # the commitment does not depend on the transcript
            self.pc, _ = O.prove_shard_verify(self.blob, self.heights, mains, preps, self.names, O.to_monty(np.zeros(4)), log_stack, mlr,
                                              O.Challenger(), **M.SMALL)

    def prove(self, pvs, tail):
        tail = O.to_monty(np.array(tail))
        words = []
        for pv in pvs:
            mains, preps = M.traces(self.specs, 5, CC.pv0_of(pv))
            ch = O.Challenger(); ch.observe(self.pc); ch.observe(tail)
            pc, w = O.prove_shard_verify(self.blob, self.heights, mains, preps, self.names, O.to_monty(np.array(pv)), self.log_stack,
                                         self.mlr, ch, **M.SMALL)
            assert (pc == self.pc).all()
            words.append(w)
        return words, tail

    def verify(self, words, tail):
        return CO.verify_core_proof(self.blob, [self.heights] * len(words), self.names, self.log_stack, self.mlr, self.pc, tail, words,
                                    **M.SMALL)


def test_oracle_accepts_a_proved_chain_and_rejects_a_corrupted_shard(capfd):
    oc = OracleChain(M.WITH_PREP, 8, 9)
    pvs, tail = CC.chain(3, 300)
    words, mtail = oc.prove(pvs, tail)
    assert oc.verify(words, mtail) == (0, 0, 0)
    bad = [w.copy() for w in words]
    at = 6 + int(bad[1][1]) + int(bad[1][2]) + 3
    bad[1][at] = (int(bad[1][at]) + 1) % O.P
    assert oc.verify(bad, mtail) == (45, 1, -1)
    assert oc.verify([], mtail)[:2] == (43, 0)


def test_oracle_gives_every_public_value_verdict():
    oc = OracleChain(M.NO_PREP, 7, 8)
    seen = set()
    for name, mutate, want, shard in CC.PV_CASES:
        pvs, tail = CC.chain(3, 140, non_execution=1)
        mutate(pvs, tail)
        words, mtail = oc.prove(pvs, tail)
        assert oc.verify(words, mtail) == (want, shard, 0), name
        seen.add(want)
    assert seen == set(range(46, 76))
