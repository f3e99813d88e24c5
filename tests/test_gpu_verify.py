"""GPU tests of the library's shard verifier (sp1b200_verify_shard, ShardVerifier::verify_shard): it accepts the library's own proofs and
ends in the prover's challenger state; on every corrupted proof it agrees with the oracle's restated verifier (orc_verify_shard) on
accept / reject / does-not-parse and names the same first failing check; malformed words are errors that leave the context usable."""
import threading

import numpy as np
import pytest

from tests import gpu_prove as GP
from tests import machines as M
from tests import oracle_lib as O
from tests.machines import ORACLE_LACKS, SMALL

pytestmark = pytest.mark.gpu

P = 0x7F000001


def _prove(inp, log_stack, mlr, seed, prm=SMALL, replay=None, **ctx):
    """-> dict with the proof, the inputs the verifier needs, and an open context + machine"""
    from sp1_b200 import Lib
    blob, heights, mains, preps, pv, names = inp
    ch = O.Challenger(); ch.observe(O.rand_field(np.random.default_rng(seed), 9))
    lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, **prm, **ctx)
    mach = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    st = ch.st.copy()
    words = GP.prove(lib, mach, prep_round, mains, heights, names, pv, st, replay=replay)
    if prep_round is not None:
        lib.jagged_round_free(prep_round)
    else:
        pc = None   # the verifier takes no preprocessed commitment for a machine without preprocessed columns
    return dict(lib=lib, mach=mach, blob=blob, heights=list(heights), names=names, pc=pc, words=words, start=ch.st.copy(), final=st,
                log_stack=log_stack, mlr=mlr, prm=prm)


def _close(c):
    c["lib"].machine_free(c["mach"])
    c["lib"].close()


def _spec_inp(spec, seed):
    return M.spec_machine(np.random.default_rng(seed), spec, names="Chip{:02d}")


def _accept(c):
    verdict, st = c["lib"].verify_shard(c["mach"], c["pc"], c["heights"], c["names"], c["words"], c["start"])
    from sp1_b200.lib import verdict_name
    assert verdict == 0, f"the library rejected its own proof: {verdict_name(verdict)}"
    assert (st == c["final"]).all(), "verifier and prover end in different challenger states"


def _oracle(c, words, heights=None, start=None, pc="same"):
    v = O.Challenger(); v.st[:] = c["start"] if start is None else start
    return O.verify_shard(c["blob"], c["heights"] if heights is None else heights, c["names"], c["log_stack"], c["mlr"], v,
                          c["pc"] if isinstance(pc, str) else pc, words, **c["prm"])


def _agree(c, capfd, words, heights=None, start=None, pc="same", what=""):
    """both verifiers on the same (possibly corrupted) inputs: same outcome, same first failing check"""
    from sp1_b200.lib import Sp1B200Error, verdict_name
    capfd.readouterr()
    o = _oracle(c, words, heights, start, pc)
    err = capfd.readouterr().err
    try:
        verdict, _ = c["lib"].verify_shard(c["mach"], c["pc"] if isinstance(pc, str) else pc, c["heights"] if heights is None else heights,
                                           c["names"], words, c["start"] if start is None else start)
    except Sp1B200Error as e:
        assert o == -2, f"{what}: the library fails to parse ({e}) what the oracle parses (oracle {o}: {err.strip()})"
        return "parse"
    assert o != -2, f"{what}: the oracle fails to parse what the library parses (verdict {verdict_name(verdict)})"
    if o == 0:
        assert verdict == 0, f"{what}: the oracle accepts, the library rejects with {verdict_name(verdict)}"
        return "accept"
    reason = err.strip().rsplit(": ", 1)[-1]
    assert verdict != 0, f"{what}: the oracle rejects ({reason}), the library accepts"
    if verdict_name(verdict) in ORACLE_LACKS:
        return verdict_name(verdict)   # a shape check the oracle's restatement does not make; it rejects for a later reason
    assert verdict_name(verdict) == reason, f"{what}: library says {verdict_name(verdict)}, oracle says {reason}"
    return reason


@pytest.mark.parametrize("spec,log_stack,mlr", M.SHARD_SPECS + [M.RANDOM_SHARD_SPEC])
def test_accepts_small_machines(spec, log_stack, mlr):
    """max_log_row_count 3 and 7, machines with and without preprocessed columns, absent chips, random constraint programs (whose
    constraints the verifier evaluates at the opened point with its own interpreter of the bytecode)"""
    c = _prove(_spec_inp(spec, 2100 + mlr), log_stack, mlr, 2101)
    _accept(c)
    assert _oracle(c, c["words"]) == 0, "the oracle's verifier rejects the library's proof"
    _close(c)


def test_accepts_max_log_row_count_2_without_preprocessed_columns():
    c = _prove(_spec_inp([(4, 1, False), (3, 2, False)], 2110), 2, 2, 2111)
    assert c["pc"] is None
    _accept(c)
    _close(c)


@pytest.mark.parametrize("workload", ["tinyc", "tinyr"])
def test_accepts_workload_machines(workload):
    c = _prove(M.workload_machine(workload, seed=2120, max_log_rows=14), 12, 14, 2121)
    _accept(c)
    _close(c)


def test_accepts_the_96_chip_machine():
    c = _prove(M.spec_machine(np.random.default_rng(2130), M.full_table_spec(96, 2131, absent=True)), 5, 5, 2132)
    _accept(c)
    _close(c)


def test_accepts_a_replay_proof_with_non_minimal_witnesses():
    """grind_mode = 1: the proof carries witnesses the oracle ground (the second-smallest valid ones)"""
    import ctypes as C
    inp = _spec_inp([(1024, 2, True), (256 + 32, 3, False), (0, 1, False), (2048, 1, True)], 2140)
    blob, heights, mains, preps, pv, names = inp
    ch = O.Challenger(); ch.observe(O.rand_field(np.random.default_rng(2141), 9))
    L = O.lib()
    L.orc_set_grind_skip(C.c_uint32(1))
    try:
        och = ch.clone()
        O.prove_shard_verify(blob, heights, mains, preps, names, pv, 10, 11, och, **SMALL)
        wl = np.zeros(8, np.uint32)
        n = L.orc_witness_log(O.ptr(wl), C.c_uint32(8))
    finally:
        L.orc_set_grind_skip(C.c_uint32(0))
    assert n == 3
    c = _prove(inp, 10, 11, 2141, replay=wl[:3], grind_mode=1)
    assert (c["final"] == och.st).all()
    _accept(c)
    _close(c)


def _sections(words):
    lens = [int(x) for x in words[1:6]]
    starts = np.cumsum([6] + lens[:-1])
    return [(int(s), int(s) + n) for s, n in zip(starts, lens)]


def test_corruption_sweep_agrees_with_the_oracle(capfd):
    """one word changed in every part of a tinyc proof, plus a wrong preprocessed commitment, a changed height and a challenger that has
    not observed the verifying key: the library and the oracle reach the same outcome and name the same first failing check"""
    c = _prove(M.workload_machine("tinyc", seed=2150, max_log_rows=12, scale=0.25), 10, 12, 2151)
    _accept(c)
    w = c["words"]
    sec = _sections(w)
    positions = {"main commitment": [sec[0][0] + 3]}
    s, e = sec[1]
    n_out = int(w[s])
    positions["GKR output numerator"] = [s + 1]
    positions["GKR output denominator"] = [s + 1 + 4 * n_out + 2]
    positions["GKR sections"] = list(range(s + 1 + 8 * n_out + 1, e, max(1, (e - s) // 40)))
    positions["GKR witness"] = [e - 1]
    s, e = sec[2]
    positions["zerocheck polynomial"] = [s + 2]
    positions["zerocheck sections"] = list(range(s, e, max(1, (e - s) // 30)))
    positions["zerocheck opened value"] = [e - 1]
    s, e = sec[3]
    positions["evaluation proof"] = list(range(s, e, max(1, (e - s) // 150)))
    positions["evaluation proof tail"] = list(range(e - 40, e))
    positions["public value"] = [sec[4][0]]
    outcomes = {}
    for what, offs in positions.items():
        for off in offs:
            bad = w.copy()
            bad[off] = (int(bad[off]) + 1) % P
            r = _agree(c, capfd, bad, what=f"{what} word {off}")
            outcomes[r] = outcomes.get(r, 0) + 1
    assert outcomes.get("accept", 0) == 0, outcomes
    # several distinct checks are exercised, in every part of the protocol
    for name in ("TcsError(component)", "TcsError(query)", "NumeratorEvaluationMismatch", "ConstraintsCheckFailed(InconsistencyWithEval)"):
        assert any(name in k for k in outcomes), (name, outcomes)
    # wrong preprocessed commitment, one height changed, a challenger that has not observed the verifying key
    pc = c["pc"].copy(); pc[0] ^= 1
    assert _agree(c, capfd, w, pc=pc, what="preprocessed commitment") not in ("accept", "parse")
    h = list(c["heights"]); k = max(range(len(h)), key=lambda i: h[i]); h[k] -= 1
    assert _agree(c, capfd, w, heights=h, what="height") != "accept"
    assert _agree(c, capfd, w, start=O.Challenger().st.copy(), what="fresh challenger") not in ("accept", "parse")
    # and the valid proof is still accepted on the same context
    _accept(c)
    _close(c)


def test_malformed_words_are_errors_and_leave_the_context_usable():
    from sp1_b200.lib import Sp1B200Error
    c = _prove(_spec_inp([(32, 2, True), (96, 1, False), (128, 1, False), (0, 1, True)], 2160), 5, 7, 2161)
    w = c["words"]
    huge = w.copy(); huge[2] = 0xFFFFFFFF
    count = w.copy(); count[0] = 4
    gkr_count = w.copy(); gkr_count[_sections(w)[1][0]] = 0x7FFFFFFF
    for what, bad in [("truncated", w[:-1]), ("trailing", np.append(w, np.uint32(0))), ("absurd section length", huge),
                      ("wrong section count", count), ("absurd GKR output count", gkr_count), ("empty", w[:0])]:
        with pytest.raises(Sp1B200Error):
            c["lib"].verify_shard(c["mach"], c["pc"], c["heights"], c["names"], bad, c["start"])
        _accept(c)
    _close(c)


@pytest.mark.parametrize("other", [dict(num_queries=9), dict(log_blowup=1)])
def test_other_context_parameters_reject_or_fail_to_parse(other):
    from sp1_b200 import Lib
    from sp1_b200.lib import Sp1B200Error
    c = _prove(_spec_inp([(32, 2, True), (96, 1, False), (128, 1, False), (0, 1, True)], 2170), 5, 7, 2171)
    prm = dict(SMALL); prm.update({k: v for k, v in other.items() if k in prm})
    lib2 = Lib(0, log_stacking_height=5, max_log_row_count=7, **prm, **{k: v for k, v in other.items() if k not in prm})
    mach2 = lib2.machine_create(c["blob"])
    try:
        verdict, _ = lib2.verify_shard(mach2, c["pc"], c["heights"], c["names"], c["words"], c["start"])
        assert verdict != 0
    except Sp1B200Error:
        pass
    lib2.machine_free(mach2)
    lib2.close()
    _accept(c)
    _close(c)


def test_four_contexts_on_four_threads():
    cases = [_prove(_spec_inp(spec, 2180 + k), ls, mlr, 2190 + k) for k, (spec, ls, mlr) in enumerate(M.SHARD_SPECS + [M.SHARD_SPECS[2]])]
    bad = cases[3]["words"].copy(); bad[_sections(bad)[3][0] + 5] = (int(bad[_sections(bad)[3][0] + 5]) + 1) % P
    inputs = [c["words"] for c in cases[:3]] + [bad]
    results, errors = [None] * 4, []
    go = threading.Barrier(4)

    def run(k):
        try:
            go.wait()
            c = cases[k]
            results[k] = [c["lib"].verify_shard(c["mach"], c["pc"], c["heights"], c["names"], inputs[k], c["start"])[0] for _ in range(3)]
        except Exception as e:  # reported on the main thread
            errors.append((k, e))

    ths = [threading.Thread(target=run, args=(k,)) for k in range(4)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errors, errors
    assert results[:3] == [[0, 0, 0]] * 3 and all(v != 0 for v in results[3]) and len(set(results[3])) == 1, results
    for c in cases:
        _close(c)


@pytest.mark.parametrize("workload", ["S2c", "R1"])
def test_full_size_proofs(workload):
    """full-size GPU proofs at the core (S2c) and recursion (R1) parameters are accepted, and rejected after a one-bit change"""
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import workload as W
    from sp1_b200.lib import HostChallenger, Sp1B200Error
    from tools.verify_bench import full_size_proof
    lib = Lib(device=0, **W.params_of(workload))
    f = full_size_proof(lib, workload, torch.device("cuda", 0))
    verdict, st = lib.verify_shard(f["machine"], f["pc"], f["heights"], f["names"], f["words"], HostChallenger().st)
    assert verdict == 0 and (st == f["final"]).all()
    s, e = _sections(f["words"])[3]
    bad = f["words"].copy(); bad[(s + e) // 2] ^= 1 << 3
    try:
        verdict, _ = lib.verify_shard(f["machine"], f["pc"], f["heights"], f["names"], bad, HostChallenger().st)
    except Sp1B200Error as err:   # the flipped word left the field's canonical range
        assert "canonical" in str(err)
    else:
        assert verdict != 0
    lib.machine_free(f["machine"])
    lib.close()


@pytest.mark.parametrize("case", __import__("tests.golden_util", fromlist=["cases"]).cases(), ids=lambda c: c["name"])
def test_accepts_the_golden_shard_proofs(case):
    """the four committed fixtures, proved again from their seeds: the words match the fixture's SHA-256, the library's verifier accepts
    them and ends in the fixture's final challenger state"""
    from sp1_b200 import Lib
    from tests import golden_util as G
    blob, heights, mains, preps, pv, names, ch = G.inputs_of(case)
    lib = Lib(0, log_stacking_height=case["log_stacking_height"], max_log_row_count=case["max_log_row_count"], num_queries=case["num_queries"],
              pow_bits=case["pow_bits"], batch_pow_bits=case["batch_pow_bits"], gkr_pow_bits=case["gkr_pow_bits"])
    mach = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    st = ch.st.copy()
    words = GP.prove(lib, mach, prep_round, mains, heights, names, pv, st)
    G.check_words(case, pc, words, st)
    verdict, vst = lib.verify_shard(mach, pc, heights, names, words, ch.st.copy())
    assert verdict == 0
    assert [int(x) for x in vst] == case["final_challenger"]
    if prep_round is not None:
        lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()


def _eval_fields(w, c):
    """word offsets of the evaluation proof's fields (layout: sp1_b200/csrc/proof_layout.hpp)"""
    ls, nq = c["log_stack"], c["prm"]["num_queries"]
    wd = M.widths(c["blob"])
    S = 1 << ls
    areas = [sum(h * p for h, (_, p) in zip(c["heights"], wd)), sum(h * m for h, (m, _) in zip(c["heights"], wd))]
    ncols = ([max(1, -(-areas[0] // S))] if any(p for _, p in wd) else []) + [max(1, -(-areas[1] // S))]
    o, f = _sections(w)[3][0], {}
    f["univariate message"] = o; o += 8 * ls
    f["FRI commitment"] = o; o += 8 * ls
    for r, nc in enumerate(ncols):
        f.setdefault("component value", o); o += nq * nc + 8
        lh = int(w[o]); o += 2
        f.setdefault("component path", o); o += nq * lh * 8
    for r in range(ls):
        if r == 0:
            f["fold value, first half"] = o; f["fold value, second half"] = o + 4
        o += nq * 8 + 8
        lh = int(w[o]); o += 2
        if r == 0:
            f["fold path"] = o
        o += nq * lh * 8
    f["final_poly"] = o; o += 4
    f["pow witness"] = o; o += 1
    f["batch grinding witness"] = o; o += 1
    f["batch evaluation"] = o; o += 4 * sum(ncols)
    for name in ("jagged sumcheck", "jagged-eval sumcheck"):
        n = int(w[o]); o += 1
        f[f"{name} polynomial"] = o + 1
        for _ in range(n):
            o += 1 + 4 * int(w[o])
        f[f"{name} claimed sum"] = o; o += 4 + 4 * n
        f[f"{name} eval"] = o; o += 4
    f["row count"] = o + 1; f["column count"] = o + 2
    for _ in ncols:
        o += 1 + 2 * int(w[o])
    f["original commitment"] = o; o += 8 * len(ncols)
    f["expected_eval"] = o; o += 4
    assert o + 2 == _sections(w)[3][1]
    return f


def test_every_evaluation_proof_field_agrees_with_the_oracle(capfd):
    """each field of the evaluation proof changed on purpose (offsets from the layout, not a stride); the PoW witnesses are changed
    until the oracle reports the PoW check itself, so that the checks the library resolves after its device copy are ordered against
    host checks on purpose"""
    c = _prove(_spec_inp([(32, 2, True), (96, 1, False), (128, 1, False), (0, 1, True)], 2200), 5, 7, 2201)
    _accept(c)
    w = c["words"]
    seen = {}
    for what, off in _eval_fields(w, c).items():
        bad = w.copy(); bad[off] = (int(bad[off]) + 1) % P
        seen[what] = _agree(c, capfd, bad, what=what)
    for what, want in (("pow witness", "Pow"), ("batch grinding witness", "BatchPow")):
        off = _eval_fields(w, c)[what]
        for d in range(1, 64):
            bad = w.copy(); bad[off] = (int(bad[off]) + d) % P
            if _agree(c, capfd, bad, what=f"{what} + {d}") == want:
                break
        else:
            raise AssertionError(f"no change of the {what} failed its PoW check")
    assert seen["component path"] == "TcsError(component)", seen
    assert seen["fold path"] == "TcsError(query)", seen
    assert {seen["fold value, first half"], seen["fold value, second half"]} == {"QueryValueMismatch", "TcsError(query)"}, seen
    assert seen["expected_eval"] == "JaggedEvalProofVerificationFailed", seen
    assert seen["row count"] == "IncorrectTableSizes" and seen["original commitment"] == "IncorrectTableSizes", seen
    assert "accept" not in seen.values(), seen
    _accept(c)
    _close(c)


def test_rejects_a_jagged_layout_other_than_the_chip_heights():
    """A proof whose main commitment lays chip 1 out with one more (zero) row than its declared height.  Every column's evaluation is
    unchanged by a zero row, so the LogUp-GKR, zerocheck, jagged and BaseFold checks all pass; only verify_shard's comparison of the
    table row counts with the chip heights (shard.rs:662-742) catches it."""
    import torch
    from sp1_b200.lib import HostChallenger, verdict_name
    from tests.ext_field import EF
    ls, mlr = 7, 8
    inp = _spec_inp([(32, 2, True), (96, 1, False), (100, 1, False)], 2210)
    blob, heights, mains, preps, pv, names = inp
    wd = M.widths(blob)
    area, S = sum(h * m for h, (m, _) in zip(heights, wd)), 1 << ls
    # a chip whose extra row keeps the main round's stacked column count (and so every section length) unchanged
    k = next(i for i in range(len(heights)) if not wd[i][1] and -(-(area + wd[i][0]) // S) == -(-area // S) and heights[i] < 1 << mlr)
    c = _prove(inp, ls, mlr, 2211)
    _accept(c)
    lib, mach = c["lib"], c["mach"]
    tabs = [np.ascontiguousarray(m) for m in mains]
    tabs[k] = np.concatenate([tabs[k], np.zeros((tabs[k].shape[0], 1), np.uint32)], axis=1)   # [cols, rows + 1]
    pc, prep_round = GP.commit_prep(lib, preps)
    commit, main_round = lib.jagged_commit(tabs)
    st = HostChallenger(c["start"])
    st.observe(pv); st.observe(commit); st.observe(O.to_monty(np.array([len(names)])))
    for h, n in zip(heights, names):
        st.observe(O.to_monty(np.array([h, len(n)] + list(n.encode()))))
    d_main = [torch.from_numpy(np.ascontiguousarray(m).view(np.int32)).cuda() for m in mains]
    d_prep = [torch.from_numpy(np.ascontiguousarray(p).view(np.int32)).cuda() if p is not None else None for p in preps]
    gkr = lib.logup_gkr(mach, heights, d_main, d_prep, st.st)
    tw = sum(a + b for a, b in wd)
    openings = gkr[len(gkr) - 1 - 4 * tw:len(gkr) - 1].reshape(-1, 4)
    point = gkr[len(gkr) - 1 - 4 * tw - 4 * mlr:len(gkr) - 1 - 4 * tw].reshape(-1, 4)
    alpha, gamma = st.sample(4), st.sample(4)
    claims, j = [], 0
    for a, b in wd:
        acc, g = EF.of(0), EF(gamma)
        for _ in range(a + b):
            acc = acc + EF(openings[j]) * g; g = g * EF(gamma); j += 1
        claims.append(acc.w)
    zc = lib.zerocheck(mach, heights, d_main, d_prep, pv, point, alpha, gamma, np.array(claims, np.uint32), st.st)
    zpoint = zc[1 + mlr * 21 + 4:1 + mlr * 21 + 4 + 4 * mlr].reshape(-1, 4)
    zopen = zc[1 + mlr * 21 + 4 + 4 * mlr + 4:]
    pcl, mcl, o = [], [], 0
    for a, b in wd:
        pcl.append(zopen[o:o + 4 * b]); o += 4 * b
        mcl.append(zopen[o:o + 4 * a]); o += 4 * a
    jcl = np.concatenate(pcl + mcl)
    ev = lib.jagged_prove([prep_round, main_round], zpoint, jcl, st.st)
    words = np.concatenate([np.array([5, 8, gkr.size, zc.size, ev.size, pv.size], np.uint32), commit, gkr, zc, ev, pv]).astype(np.uint32)
    lib.jagged_round_free(prep_round); lib.jagged_round_free(main_round)
    assert (c["words"][:6] == words[:6]).all() and (words != c["words"]).any(), "same layout sizes, different commitment"
    verdict, _ = lib.verify_shard(mach, pc, heights, names, words, c["start"])
    assert verdict_name(verdict) == "InvalidShape(chip tables)", verdict_name(verdict)
    v = O.Challenger(); v.st[:] = c["start"]
    assert O.verify_shard(blob, heights, names, ls, mlr, v, pc, words, **SMALL) == 0, "the oracle's restatement lacks this check"
    _close(c)
