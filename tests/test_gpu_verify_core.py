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
from tests.provers import Core, specs_machine, workload_specs_machine

pytestmark = pytest.mark.gpu

V_INVALID_SHARD_PROOF = 45


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
    c = Core(specs_machine(M.WITH_PREP), 8, 9)
    _accept(c, n, 100 + n)
    c.close()


@pytest.mark.parametrize("n", [1, 2, 5])
def test_accepts_without_preprocessed_columns(n):
    c = Core(specs_machine(M.NO_PREP), 7, 8)
    assert not c.pc.any()
    _accept(c, n, 110 + n, non_execution=1 if n > 2 else None)
    c.close()


@pytest.mark.parametrize("workload,n", [("tinyc", 3), ("tinyr", 2)])
def test_accepts_workload_machines(workload, n):
    c = Core(workload_specs_machine(workload, 12, 0.25), 10, 12)
    _accept(c, n, 120 + n)
    c.close()


def test_every_public_value_check():
    """one chain per reason, proved with the faulty public values (not patched after proving): exactly that verdict at that shard"""
    from sp1_b200.lib import verdict_name
    c = Core(specs_machine(M.NO_PREP), 7, 8)
    seen = set()
    for name, mutate, want, shard in CC.PV_CASES:
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
    c = Core(workload_specs_machine("tinyc", 12, 0.25), 10, 12, **ctx)
    pvs, tail = CC.chain(n, seed)
    words, finals, mtail = c.prove(pvs, tail)
    return c, words, finals, mtail


def test_corrupted_shard_matches_verify_shard_and_the_oracle(capfd):
    """a stride sweep over shard 1 of a 3-shard proof, up to its public values (whose changes the checks across shards catch first):
    InvalidShardProof at shard 1 with the inner verdict sp1b200_verify_shard gives on that shard alone (and the oracle's first
    failing check), or a parse error from both calls"""
    from sp1_b200.lib import Sp1B200Error, verdict_name
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
        if len(outcomes) <= 6 and verdict_name(single) not in M.ORACLE_LACKS:
            capfd.readouterr()
            o = O.Challenger(); o.st[:] = start
            r = O.verify_shard(c.blob, c.heights, c.names, c.log_stack, c.mlr, o, c.pc, bad, **c.prm)
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
    c = Core(specs_machine(M.NO_PREP), 7, 8)
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
    cores = [Core(specs_machine(M.WITH_PREP), 8, 9), Core(specs_machine(M.NO_PREP), 7, 8)]
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
