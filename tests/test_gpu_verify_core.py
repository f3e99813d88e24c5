"""GPU tests of the core-proof verifier (sp1b200_verify_core_proof, SP1Prover::verify): it accepts N-shard core proofs of the library's
own shards and ends every shard in its prover's challenger state; every public-value check across shards rejects a chain proved with
exactly that fault, at the shard the reference's loop stops at; a corrupted shard is reported as InvalidShardProof with the same inner
verdict sp1b200_verify_shard and the oracle give; thread count and batching never change a result; malformed arguments are errors."""
import os
import threading

import numpy as np
import pytest

from tests import core_chain as CC
from tests import machines as M
from tests import oracle_lib as O
from tests.test_septic import START, curve_add

pytestmark = pytest.mark.gpu

SMALL = dict(num_queries=8, pow_bits=4, batch_pow_bits=2, gkr_pow_bits=3)
WITH_PREP = [M.Chip(256, 2, True), M.Chip(64 + 8, 3, False), M.Chip(0, 1, False), M.Chip(128, 1, True)]
NO_PREP = [M.Chip(128, 2, False), M.Chip(32, 1, False)]

V_INVALID_SHARD_PROOF = 45


def _specs_machine(chips, mlr):
    blob, heights, _, _, _, names = M.spec_machine(np.random.default_rng(1), chips)
    specs = [(c.h, c.g, c.wp, c.extra, c.extra_prep) for c in (M.Chip(*c) for c in chips)]
    return blob, heights, names, specs


def _workload_machine(workload, mlr, scale):
    from sp1_b200 import workload as W
    mach = W.synthetic_machine(workload, seed=42, max_log_rows=mlr, scale=scale)
    specs = [(s.h, s.g, s.wp, s.extra, s.extra_prep) for s in mach["specs"]]
    return mach["blob"], [s.h for s in mach["specs"]], list(mach["names"]), specs


def _traces(specs, seed, pv0):
    """the same traces for every shard (so the preprocessed tables agree), with the shard's own public value 0"""
    from sp1_b200 import synth_air as SA
    rng = np.random.default_rng(seed)
    mains, preps = [], []
    for h, g, wp, extra, extra_prep in specs:
        m, p = SA.synth_trace(rng, h, g, wp, pv0, extra_cols=extra, extra_prep=extra_prep)
        mains.append(m); preps.append(p)
    return mains, preps


class Core:
    """a context + machine proving shards of one program under one verifying key"""

    def __init__(self, machine, log_stack, mlr, prm=SMALL, seed=5, **ctx):
        from sp1_b200 import Lib
        self.blob, self.heights, self.names, self.specs = machine
        self.log_stack, self.mlr, self.prm, self.seed = log_stack, mlr, prm, seed
        self.lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, **prm, **ctx)
        self.mach = self.lib.machine_create(self.blob)
        _, preps = _traces(self.specs, seed, 0)
        tabs = [p for p in preps if p is not None]
        self.pc, self.prep_round = self.lib.jagged_commit(tabs) if tabs else (np.zeros(8, np.uint32), None)

    def start(self, tail):
        from sp1_b200.lib import HostChallenger
        hc = HostChallenger(); hc.observe(self.pc); hc.observe(tail)
        return hc.st.copy()

    def prove(self, pvs, tail):
        """-> (words per shard, final prover state per shard); tail, pvs: canonical"""
        tail = O.to_monty(np.array(tail))
        words, finals = [], []
        for pv in pvs:
            mains, _ = _traces(self.specs, self.seed, CC.pv0_of(pv))
            st = self.start(tail)
            words.append(self.lib.prove_shard(self.mach, self.prep_round, M.dense_main(mains), self.heights, self.names,
                                              O.to_monty(np.array(pv)), st))
            finals.append(st)
        return words, finals, tail

    def verify(self, words, tail, heights=None, threads=0):
        hs = [self.heights] * len(words) if heights is None else heights
        return self.lib.verify_core_proof(self.mach, self.pc, tail, hs, self.names, words, host_threads=threads)

    def close(self):
        if self.prep_round is not None:
            self.lib.jagged_round_free(self.prep_round)
        self.lib.machine_free(self.mach)
        self.lib.close()


def _accept(c, n, seed, **kw):
    from sp1_b200.lib import verdict_name
    pvs, tail = CC.chain(n, seed, **kw)
    words, finals, mtail = c.prove(pvs, tail)
    v, shard, sv, fin = c.verify(words, mtail)
    assert (v, shard, sv) == (0, 0, 0), f"rejected its own core proof: {verdict_name(v)} at {shard} ({verdict_name(sv)})"
    assert fin.shape == (n, 34)
    for s in range(n):
        assert (fin[s] == finals[s]).all(), f"shard {s}: verifier and prover end in different challenger states"
    return words, mtail


@pytest.mark.parametrize("n", [1, 2, 5])
def test_accepts_with_preprocessed_columns(n):
    c = Core(_specs_machine(WITH_PREP, 9), 8, 9)
    _accept(c, n, 100 + n)
    c.close()


@pytest.mark.parametrize("n", [1, 2, 5])
def test_accepts_without_preprocessed_columns(n):
    c = Core(_specs_machine(NO_PREP, 8), 7, 8)
    assert not c.pc.any()
    _accept(c, n, 110 + n, non_execution=1 if n > 2 else None)
    c.close()


@pytest.mark.parametrize("workload,n", [("tinyc", 3), ("tinyr", 2)])
def test_accepts_workload_machines(workload, n):
    c = Core(_workload_machine(workload, 12, 0.25), 10, 12)
    _accept(c, n, 120 + n)
    c.close()


# (name, mutation of the valid 3-shard chain with a non-execution shard 1, expected verdict, expected shard)
def _set(s, name, vals):
    return lambda pvs, tail: CC.setf(pvs[s], name, vals)


def _m_len(pvs, tail):
    pvs[1][:] = pvs[1][:186]


def _m_never(field):
    def f(pvs, tail):
        for pv in pvs:
            CC.setf(pv, "previous_" + field, [0, 0, 0]); CC.setf(pv, "last_" + field, [0, 0, 0])
    return f


def _m_commit(field):
    def f(pvs, tail):
        for pv in pvs:
            CC.setf(pv, "prev_" + field, 0); CC.setf(pv, field, 0)
    return f


def _m_ts_changed(pvs, tail):
    last = CC.getf(pvs[1], "last_timestamp"); last[3] += 1
    CC.setf(pvs[1], "last_timestamp", last); CC.setf(pvs[2], "initial_timestamp", last)


def _m_pc_nonexec(pvs, tail):
    CC.setf(pvs[1], "next_pc", [7, 7, 7]); CC.setf(pvs[2], "pc_start", [7, 7, 7])


def _m_exit_nonexec(pvs, tail):
    CC.setf(pvs[1], "exit_code", 3); CC.setf(pvs[2], "prev_exit_code", 3); CC.setf(pvs[2], "exit_code", 3)


def _m_exit_changed(pvs, tail):
    CC.setf(pvs[0], "exit_code", 3)
    for s in (1, 2):
        CC.setf(pvs[s], "prev_exit_code", 3); CC.setf(pvs[s], "exit_code", 3)
    CC.setf(pvs[2], "exit_code", 4)


def _m_digest(pvs, tail):
    from tests.test_septic import DUMMY
    g = CC.getf(pvs[1], "global_cumulative_sum")
    p = (g[:7], g[7:])
    q = curve_add(p, DUMMY)
    CC.setf(pvs[1], "global_cumulative_sum", list(q[0]) + list(q[1]))


def _m_exceptional(pvs, tail):
    tail[3:17] = list(START[0]) + list(START[1])


def _m_bump(s, name, k=0):
    def f(pvs, tail):
        v = CC.getf(pvs[s], name); v[k] = (v[k] + 1) % O.P
        CC.setf(pvs[s], name, v)
    return f


PV_CASES = [
    ("length", _m_len, 46, 1),
    ("first shard twice", _set(2, "is_first_execution_shard", 1), 47, 2),
    ("first shard not boolean", _set(1, "is_first_execution_shard", 2), 48, 1),
    ("first shard not set", _set(0, "is_first_execution_shard", 0), 49, 3),
    ("initial timestamp", _m_bump(2, "initial_timestamp", 3), 50, 2),
    ("timestamp unchanged on an execution shard", _set(1, "is_execution_shard", 1), 51, 1),
    ("timestamp changed on a non-execution shard", _m_ts_changed, 52, 1),
    ("pc_start != vk.pc_start", _m_bump(0, "pc_start", 1), 53, 0),
    ("pc_start != prev_next_pc", _m_bump(2, "pc_start", 0), 54, 2),
    ("pc changed on a non-execution shard", _m_pc_nonexec, 55, 1),
    ("not halted", _set(2, "next_pc", [5, 0, 0]), 56, 3),
    ("prev_exit_code", _set(0, "prev_exit_code", 1), 57, 0),
    ("exit code changed on a non-execution shard", _m_exit_nonexec, 58, 1),
    ("exit code changed twice", _m_exit_changed, 59, 2),
    ("proof nonce", _m_bump(2, "proof_nonce", 1), 60, 2),
    ("previous_init_addr", _m_bump(1, "previous_init_addr"), 61, 1),
    ("previous_finalize_addr", _m_bump(1, "previous_finalize_addr", 2), 62, 1),
    ("previous_init_page_idx", _m_bump(2, "previous_init_page_idx"), 63, 2),
    ("previous_finalize_page_idx", _m_bump(2, "previous_finalize_page_idx", 1), 64, 2),
    ("untrusted programs flag", _set(0, "is_untrusted_programs_enabled", 1), 65, 0),
    ("zero address never initialized", _m_never("init_addr"), 66, 3),
    ("zero address never finalized", _m_never("finalize_addr"), 67, 3),
    ("committed value digest", _m_bump(1, "prev_committed_value_digest", 5), 68, 1),
    ("deferred proofs digest", _m_bump(2, "prev_deferred_proofs_digest", 7), 69, 2),
    ("commit syscall", _set(0, "prev_commit_syscall", 1), 70, 0),
    ("commit deferred syscall", _set(1, "prev_commit_deferred_syscall", 0), 71, 1),
    ("COMMIT never called", _m_commit("commit_syscall"), 72, 3),
    ("COMMIT_DEFERRED_PROOFS never called", _m_commit("commit_deferred_syscall"), 73, 3),
    ("global cumulative sum", _m_digest, 74, 3),
    ("exceptional point addition", _m_exceptional, 75, 0),
]


def test_every_public_value_check():
    """one chain per reason, proved with the faulty public values (not patched after proving): exactly that verdict at that shard"""
    from sp1_b200.lib import verdict_name
    c = Core(_specs_machine(NO_PREP, 8), 7, 8)
    seen = set()
    for name, mutate, want, shard in PV_CASES:
        pvs, tail = CC.chain(3, 140, non_execution=1)
        mutate(pvs, tail)
        words, _, mtail = c.prove(pvs, tail)
        v, s, sv, fin = c.verify(words, mtail)
        assert (verdict_name(v), s, sv) == (verdict_name(want), shard, 0), name
        assert fin is None
        seen.add(want)
    assert seen == set(range(46, 76))
    v, s, sv, fin = c.verify([], O.to_monty(np.array(CC.chain(1, 141)[1])))
    assert (verdict_name(v), s, sv) == ("EmptyProof", 0, 0)
    c.close()


def _tinyc_chain(n=3, seed=150, **ctx):
    c = Core(_workload_machine("tinyc", 12, 0.25), 10, 12, **ctx)
    pvs, tail = CC.chain(n, seed)
    words, finals, mtail = c.prove(pvs, tail)
    return c, words, finals, mtail


def test_corrupted_shard_matches_verify_shard_and_the_oracle(capfd):
    """a stride sweep over shard 1 of a 3-shard proof, up to its public values (whose changes the checks across shards catch first):
    InvalidShardProof at shard 1 with the inner verdict sp1b200_verify_shard gives on that shard alone (and the oracle's first
    failing check), or a parse error from both calls"""
    from sp1_b200.lib import Sp1B200Error, verdict_name
    from tests.test_gpu_verify import ORACLE_LACKS
    c, words, _, tail = _tinyc_chain()
    start = c.start(tail)
    assert c.verify(words, tail)[0] == 0
    w1 = words[1]
    pv_at = 6 + sum(int(x) for x in w1[1:5])
    stride = max(1, pv_at // 60)
    outcomes = set()
    for i in range(6, pv_at, stride):
        bad = w1.copy(); bad[i] = (int(bad[i]) + 1) % O.P
        ws = [words[0], bad, words[2]]
        try:
            single, _ = c.lib.verify_shard(c.mach, c.pc, c.heights, c.names, bad, start)
        except Sp1B200Error:
            with pytest.raises(Sp1B200Error, match="verify_core_proof: shard 1"):
                c.verify(ws, tail)
            outcomes.add("parse")
            continue
        v, s, sv, _ = c.verify(ws, tail)
        if single == 0:
            assert v == 0, i
            continue
        assert (v, s, sv) == (V_INVALID_SHARD_PROOF, 1, single), (i, verdict_name(v), s, verdict_name(sv), verdict_name(single))
        outcomes.add(verdict_name(single))
        if len(outcomes) <= 6 and verdict_name(single) not in ORACLE_LACKS:
            capfd.readouterr()
            o = O.Challenger(); o.st[:] = start
            r = O.verify_shard(c.blob, c.heights, c.names, c.log_stack, c.mlr, o, c.pc if c.prep_round is not None else None, bad, **c.prm)
            assert r == -1 and capfd.readouterr().err.strip().rsplit(": ", 1)[-1] == verdict_name(single), i
    assert len(outcomes) >= 4, outcomes
    c.close()


def test_two_corrupted_shards_report_the_lower():
    c, words, _, tail = _tinyc_chain()
    bad = [w.copy() for w in words]
    for s in (2, 1):
        sec = int(bad[s][1]) + int(bad[s][2]) + 6 + 3   # a word of the zerocheck section
        bad[s][sec] = (int(bad[s][sec]) + 1) % O.P
    v, s, sv, _ = c.verify(bad, tail)
    assert (v, s) == (V_INVALID_SHARD_PROOF, 1) and sv != 0
    v2, s2, sv2, _ = c.verify([words[0], words[1], bad[2]], tail)
    assert (v2, s2) == (V_INVALID_SHARD_PROOF, 2) and sv2 != 0
    c.close()


def test_threads_and_batching_do_not_change_results():
    c, words, finals, tail = _tinyc_chain(4, 160)
    bad = [w.copy() for w in words]
    sec = int(bad[2][1]) + int(bad[2][2]) + 6 + 3   # a word of the zerocheck section
    bad[2][sec] = (int(bad[2][sec]) + 1) % O.P
    ref_ok = c.verify(words, tail, threads=1)
    ref_bad = c.verify(bad, tail, threads=1)
    assert ref_ok[0] == 0 and ref_bad[:2] == (V_INVALID_SHARD_PROOF, 2)
    cases = [dict(threads=8), dict(threads=8, env=str(min(w.size for w in words))), dict(threads=1, env="1")]
    for case in cases:
        if "env" in case:
            os.environ["SP1B200_VERIFY_BATCH_WORDS"] = case["env"]
        try:
            ok = c.verify(words, tail, threads=case["threads"])
            nb = c.verify(bad, tail, threads=case["threads"])
        finally:
            os.environ.pop("SP1B200_VERIFY_BATCH_WORDS", None)
        assert ok[:3] == ref_ok[:3] and (ok[3] == ref_ok[3]).all(), case
        assert nb[:3] == ref_bad[:3], case
    for s in range(4):
        assert (ref_ok[3][s] == finals[s]).all()
    c.close()


def test_malformed_arguments_are_errors_and_leave_the_context_usable():
    import ctypes as C
    from sp1_b200.lib import Sp1B200Error, _ptr
    c = Core(_specs_machine(NO_PREP, 8), 7, 8)
    pvs, tail = CC.chain(2, 170)
    words, _, mtail = c.prove(pvs, tail)
    with pytest.raises(Sp1B200Error, match="n_vk_tail"):
        c.verify(words, mtail[:23])
    with pytest.raises(Sp1B200Error, match="shard 1: NULL proof"):
        c.verify([words[0], None], mtail)
    with pytest.raises(Sp1B200Error, match="verify_core_proof: shard 0"):
        c.verify([words[0][:-3], words[1]], mtail)
    with pytest.raises(Sp1B200Error, match="NULL argument"):
        v = C.c_uint32()
        c.lib._chk(c.lib.L.sp1b200_verify_core_proof(c.lib.ctx, c.mach, None, _ptr(mtail), C.c_uint32(24), C.c_uint32(0), None, None,
                                                     None, None, C.c_uint32(0), None, C.byref(v), C.byref(v), C.byref(v)))
    assert c.verify(words, mtail)[0] == 0
    c.close()


def test_two_contexts_on_two_threads():
    cores = [Core(_specs_machine(WITH_PREP, 9), 8, 9), Core(_specs_machine(NO_PREP, 8), 7, 8)]
    jobs = []
    for i, c in enumerate(cores):
        pvs, tail = CC.chain(3, 180 + i)
        words, finals, mtail = c.prove(pvs, tail)
        jobs.append((c, words, finals, mtail))
    results = [None, None]

    def run(i):
        c, words, finals, mtail = jobs[i]
        out = []
        for _ in range(3):
            out.append(c.verify(words, mtail, threads=4))
        results[i] = out

    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for i, (c, words, finals, mtail) in enumerate(jobs):
        for v, s, sv, fin in results[i]:
            assert (v, s, sv) == (0, 0, 0)
            assert all((fin[k] == finals[k]).all() for k in range(3))
        c.close()


def test_full_size_s2c_chain():
    """three full-size S2c shards at the core parameters: accepted, every final challenger equal to its prover's; a one-word change in
    the last shard's evaluation proof is InvalidShardProof at that shard"""
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import workload as W
    from tools.verify_core_bench import prove_chain
    lib = Lib(device=0, **W.params_of("S2c"))
    f = prove_chain(lib, "S2c", 3, torch.device("cuda", 0))
    v, s, sv, fin = lib.verify_core_proof(f["machine"], f["pc"], f["tail"], [f["heights"]] * 3, f["names"], f["words"])
    assert (v, s, sv) == (0, 0, 0)
    assert all((fin[k] == f["finals"][k]).all() for k in range(3))
    bad = [w.copy() for w in f["words"]]
    w = bad[2]
    at = 6 + sum(int(x) for x in w[1:4]) + 5   # a univariate-message word of the evaluation proof
    w[at] = (int(w[at]) + 1) % O.P
    v, s, sv, _ = lib.verify_core_proof(f["machine"], f["pc"], f["tail"], [f["heights"]] * 3, f["names"], bad)
    assert (v, s) == (V_INVALID_SHARD_PROOF, 2) and sv != 0
    lib.machine_free(f["machine"])
    lib.close()
