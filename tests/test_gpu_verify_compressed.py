"""GPU tests of the compressed / shrink proof verifier (sp1b200_verify_compressed, SP1Prover::verify_compressed / verify_shrink) and the
recursion vk map (sp1b200_recursion_vks_*): the tree's root and openings equal the restatement in tests/recursion_ref.py; recursion proofs
of the library's own shards are accepted with the prover's final challengers; every reason is produced by a proof with exactly that fault
and agrees with the restatement on top of the oracle's verify_shard; batching and thread count never change a verdict; malformed inputs
are errors."""
import os

import numpy as np
import pytest

from tests import machines as M
from tests import oracle_lib as O
from tests import recursion_ref as RR
from tests.provers import Rec, specs_machine, workload_specs_machine

pytestmark = pytest.mark.gpu

SHRINK = 1


# ---- the vk tree --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,pad_to", [(2, 0), (3, 0), (5, 0), (5, 9), (4096, 0), (4097, 0), (4097, 5000), (185862, 0)])
def test_vk_tree_matches_the_restatement(n, pad_to):
    from sp1_b200 import Lib
    from sp1_b200.lib import Sp1B200Error
    rng = np.random.default_rng(n + pad_to)
    d = O.rand_field(rng, (n, 8))
    if n > 3:   # duplicates and no order
        d[rng.integers(0, n, n // 10 + 1)] = d[rng.integers(0, n, n // 10 + 1)]
    d = d[rng.permutation(n)]
    lib = Lib(0)
    vks = lib.recursion_vks(d, pad_to=pad_to)
    ref = RR.VkMap(d, pad_to=pad_to)
    assert vks.num_keys() == len(ref.keys)
    assert (vks.root() == ref.root).all()
    stride = 1 if n <= 5000 else 97
    for i in range(0, len(ref.keys), stride):
        key = O.to_monty(np.array(ref.keys[i]))
        idx, path = vks.open(key)
        assert idx == i and (path == ref.open_index(i)[1]).all(), i
        assert RR.merkle_proof_holds(key, idx, path, vks.root())
    with pytest.raises(Sp1B200Error, match="vk not allowed"):
        vks.open(O.rand_field(rng, 8))
    vks.close()
    with pytest.raises(Sp1B200Error, match="at least two"):
        lib.recursion_vks(d[:1])
    with pytest.raises(Sp1B200Error, match="at least two"):
        lib.recursion_vks(np.stack([d[0], d[0]]))
    lib.close()


# ---- acceptance ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["tinyr", "no_prep"])
def test_accepts_recursion_proofs(which):
    m = workload_specs_machine("tinyr", 12, 0.25) if which == "tinyr" else specs_machine(M.NO_PREP)
    c = Rec(m, 10, 12) if which == "tinyr" else Rec(m, 7, 8)
    if which == "no_prep":
        assert not c.pc.any()
    cases, finals = [], []
    for k in c.keys[:3]:
        w, st = c.prove(k, c.pv())
        cases.append((k, w, c.merkle(k), c.sp1)); finals.append(st)
    v, sv, fin = c.verify(cases)
    assert v == [0, 0, 0] and sv == [0, 0, 0]
    for s in range(3):
        assert (fin[s] == finals[s]).all(), f"proof {s}: verifier and prover end in different challenger states"
        assert c.oracle(*cases[s][:2], 187, *cases[s][2:]) == 0
    c.close()


def test_full_size_r1_proof():
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import workload as W
    from tools.verify_compressed_bench import prove_recursion
    lib = Lib(device=0, **W.params_of("R1"))
    f = prove_recursion(lib, "R1", 1, torch.device("cuda", 0))
    v, sv, fin = lib.verify_compressed(f["machine"], f["vks"], f["keys"], [f["heights"]], f["names"], f["words"], f["merkle_proofs"],
                                       [f["sp1_vk_digest"]])
    assert (v, sv) == ([0], [0]) and (fin[0] == f["finals"][0]).all()
    f["vks"].close()
    lib.machine_free(f["machine"])
    lib.close()


# ---- every verdict ------------------------------------------------------------------------------------------------------------------
def _zc_word(w):
    return int(w[1]) + int(w[2]) + 6 + 3   # a word of the zerocheck section


def _faulty_cases(c):
    """(name, case, n_pv, expected verdict) with exactly one fault each, all proved with the faulty values"""
    k = c.keys
    out = []
    w, _ = c.prove(k[0], c.pv()); out.append(("valid", (k[0], w, c.merkle(k[0]), c.sp1), 187, RR.ACCEPT))
    pv = c.pv()
    w, _ = c.prove(k[1], pv[:186]); out.append(("pv length", (k[1], w, c.merkle(k[1]), c.sp1), 186, RR.PV_LENGTH))
    w, _ = c.prove(k[2], c.pv()); w = w.copy(); w[_zc_word(w)] = (int(w[_zc_word(w)]) + 1) % O.P
    out.append(("shard", (k[2], w, c.merkle(k[2]), c.sp1), 187, RR.INVALID_SHARD_PROOF))
    w, _ = c.prove(k[3], c.pv(digest=True)); out.append(("digest", (k[3], w, c.merkle(k[3]), c.sp1), 187, RR.PV_DIGEST))
    w, _ = c.prove(k[4], c.pv(vk_root=True)); out.append(("vk_root", (k[4], w, c.merkle(k[4]), c.sp1), 187, RR.VK_ROOT))
    w, _ = c.prove(c.outsider, c.pv()); out.append(("key outside the map", (c.outsider, w, c.merkle(k[5]), c.sp1), 187, RR.INVALID_VK))
    w, _ = c.prove(k[5], c.pv()); idx, path = c.merkle(k[5]); path = path.copy(); path[1, 4] = (int(path[1, 4]) + 1) % O.P
    out.append(("path word", (k[5], w, (idx, path), c.sp1), 187, RR.INVALID_VK))
    w, _ = c.prove(k[0], c.pv(is_complete=True)); out.append(("is_complete", (k[0], w, c.merkle(k[0]), c.sp1), 187, RR.IS_COMPLETE))
    w, _ = c.prove(k[1], c.pv()); out.append(("sp1 vk", (k[1], w, c.merkle(k[1]), O.rand_field(c.rng, 8)), 187, RR.SP1_VK_DIGEST))
    w, _ = c.prove(k[2], c.pv(vk_root=True, is_complete=True)); out.append(("two faults", (k[2], w, c.merkle(k[2]), c.sp1), 187, RR.VK_ROOT))
    return out


@pytest.fixture(scope="module")
def faulty():
    c = Rec(specs_machine(M.NO_PREP), 7, 8)
    yield c, _faulty_cases(c)
    c.close()


def test_every_verdict_alone_and_in_one_batch(faulty):
    from sp1_b200.lib import verdict_name
    c, cases = faulty
    singles = []
    for name, case, n_pv, want in cases:
        v, sv, _ = c.verify([case])
        assert verdict_name(v[0]) == verdict_name(want), name
        assert c.oracle(*case[:2], n_pv, *case[2:]) == want, name
        if want == RR.INVALID_SHARD_PROOF:
            st = O.Challenger(); st.observe(case[0])
            assert sv[0] == c.lib.verify_shard(c.mach, None, c.heights, c.names, case[1], st.st)[0] != 0
        else:
            assert sv[0] == 0
        singles.append((v[0], sv[0]))
    assert {w for _, _, _, w in cases} == {0, 45, 46, 77, 78, 79, 80, 81}
    v, sv, _ = c.verify([case for _, case, _, _ in cases])
    assert list(zip(v, sv)) == singles


def test_vk_verification_off_accepts_a_key_outside_the_map(faulty):
    c, cases = faulty
    (case,) = [case for name, case, _, _ in cases if name == "key outside the map"]
    assert c.verify([case])[0] == [RR.INVALID_VK]
    assert c.verify([case], vks=c.vks_off)[0] == [0]
    assert c.oracle(*case[:2], 187, *case[2:], vk_verification=False) == 0


def test_shrink_mode(faulty):
    c, cases = faulty
    (name, case, _, _) = cases[0]
    key = case[0]
    assert c.verify([case], mode=SHRINK, shrink_vk=key)[0] == [0]
    assert c.verify([case], mode=SHRINK)[0] == [RR.UNINITIALIZED_VK]
    assert c.oracle(*case[:2], 187, *case[2:], shrink=True) == RR.UNINITIALIZED_VK
    for at in (3, 8 + 5):   # a commitment word, a tail word
        other = key.copy(); other[at] = (int(other[at]) + 1) % O.P
        assert c.verify([case], mode=SHRINK, shrink_vk=other)[0] == [RR.INVALID_VK], at
        assert c.oracle(*case[:2], 187, *case[2:], shrink=True, shrink_vk=other) == RR.INVALID_VK
    # a shrink-mode fault comes before the public values' length
    (pl,) = [case for name, case, _, _ in cases if name == "pv length"]
    assert c.verify([pl], mode=SHRINK)[0] == [RR.UNINITIALIZED_VK]
    assert c.verify([pl], mode=SHRINK, shrink_vk=pl[0])[0] == [RR.PV_LENGTH]


def test_threads_and_batching_do_not_change_results(faulty):
    c, cases = faulty
    five = [cases[i][1] for i in (0, 2, 3, 5, 8)]
    ref = c.verify(five, host_threads=1)
    alone = [c.verify([x], host_threads=1)[:2] for x in five]
    assert [(a[0][0], a[1][0]) for a in alone] == list(zip(ref[0], ref[1]))
    for threads, env in ((8, None), (8, "1"), (1, "1")):
        if env:
            os.environ["SP1B200_VERIFY_BATCH_WORDS"] = env
        try:
            got = c.verify(five, host_threads=threads)
        finally:
            os.environ.pop("SP1B200_VERIFY_BATCH_WORDS", None)
        assert got[0] == ref[0] and got[1] == ref[1], (threads, env)
        assert (got[2][0] == ref[2][0]).all()


def test_corrupted_proof_matches_verify_shard_and_the_oracle(capfd):
    from sp1_b200.lib import HostChallenger, Sp1B200Error, verdict_name
    c = Rec(workload_specs_machine("tinyr", 12, 0.25), 10, 12, n_keys=2)
    key = c.keys[0]
    words, _ = c.prove(key, c.pv())
    hc = HostChallenger(); hc.observe(key)
    start = hc.st.copy()
    merkle = c.merkle(key)
    assert c.verify([(key, words, merkle, c.sp1)])[0] == [0]
    pv_at = 6 + sum(int(x) for x in words[1:5])
    stride = max(1, pv_at // 50)
    outcomes = set()
    for i in range(6, pv_at, stride):
        bad = words.copy(); bad[i] = (int(bad[i]) + 1) % O.P
        try:
            single, _ = c.lib.verify_shard(c.mach, c.pc, c.heights, c.names, bad, start)
        except Sp1B200Error:
            with pytest.raises(Sp1B200Error, match="verify_compressed: proof 0"):
                c.verify([(key, bad, merkle, c.sp1)])
            outcomes.add("parse")
            continue
        v, sv, _ = c.verify([(key, bad, merkle, c.sp1)])
        if single == 0:
            assert v == [0], i
            continue
        assert (v, sv) == ([RR.INVALID_SHARD_PROOF], [single]), (i, verdict_name(single))
        outcomes.add(verdict_name(single))
        if len(outcomes) <= 6 and verdict_name(single) not in M.ORACLE_LACKS:
            capfd.readouterr()
            o = O.Challenger(); o.st[:] = start
            r = O.verify_shard(c.blob, c.heights, c.names, c.log_stack, c.mlr, o, c.pc, bad, **c.prm)
            assert r == -1 and capfd.readouterr().err.strip().rsplit(": ", 1)[-1] == verdict_name(single), i
    assert len(outcomes) >= 4, outcomes
    c.close()


# ---- errors -------------------------------------------------------------------------------------------------------------------------
def test_malformed_inputs_are_errors_and_leave_the_context_usable(faulty):
    import ctypes as C
    from sp1_b200.lib import Sp1B200Error
    c, cases = faulty
    case = cases[0][1]
    key, words, (idx, path), sp1 = case
    with pytest.raises(Sp1B200Error, match="no proofs"):
        c.verify([])
    with pytest.raises(Sp1B200Error, match="more than 64"):
        c.verify([(key, words, (idx, np.zeros((65, 8), np.uint32)), sp1)])
    bad_key = key.copy(); bad_key[9] = O.P
    with pytest.raises(Sp1B200Error, match="verifying-key word is not canonical"):
        c.verify([(bad_key, words, (idx, path), sp1)])
    bad_path = path.copy(); bad_path[0, 0] = 0xFFFFFFFF
    with pytest.raises(Sp1B200Error, match="path word is not canonical"):
        c.verify([(key, words, (idx, bad_path), sp1)])
    with pytest.raises(Sp1B200Error, match="proof 1: NULL proof"):
        c.verify([case, (key, None, (idx, path), sp1)])
    with pytest.raises(Sp1B200Error, match="verify_compressed: proof 0"):
        c.verify([(key, words[:-3], (idx, path), sp1)])
    with pytest.raises(Sp1B200Error, match="shrink key in compressed mode"):
        c.verify([case], shrink_vk=key)
    with pytest.raises(Sp1B200Error, match="NULL argument"):
        v = (C.c_uint32 * 1)()
        c.lib._chk(c.lib.L.sp1b200_verify_compressed(c.lib.ctx, c.mach, None, C.c_uint32(0), None, C.c_uint32(1), None, None, None, None,
                                                     None, None, None, None, None, C.c_uint32(0), None, v, v))
    assert c.verify([case])[0] == [0]
