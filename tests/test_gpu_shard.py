"""GPU parity test of the whole shard proof (A1): sp1b200_prove_shard vs the oracle's prove_shard_with_data restatement
(which runs the restated ShardVerifier::verify_shard on its own proof).  Every proof word and the final challenger state
must be identical."""
import numpy as np
import pytest

from tests import gpu_prove as GP
from tests import machines as M
from tests import oracle_lib as O

pytestmark = pytest.mark.gpu


def _run(spec, log_stack, mlr, seed, nq=8, pow_bits=4, batch_bits=2, gkr_bits=3):
    from sp1_b200 import Lib
    blob, heights, mains, preps, pv, names, ch = M.shard_inputs(spec, seed)
    och = ch.clone()
    opc, owords = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, och, num_queries=nq, pow_bits=pow_bits,
                                       batch_pow_bits=batch_bits, gkr_pow_bits=gkr_bits)
    lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, num_queries=nq, pow_bits=pow_bits, batch_pow_bits=batch_bits,
              gkr_pow_bits=gkr_bits)
    mach = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    assert (pc == opc).all(), "preprocessed commitment differs"
    st = ch.st.copy()
    words = GP.prove(lib, mach, prep_round, mains, heights, names, pv, st)
    assert words.size == owords.size, (words.size, owords.size, words[:6], owords[:6])
    bad = np.nonzero(words != owords)[0]
    assert bad.size == 0, f"first differing words {bad[:8]} of {words.size} (sections {owords[:6]})"
    assert (st == och.st).all()
    # the wire format of the GPU proof: bincode(ShardProof) decoded by the independent reader of the Rust struct definitions gives back
    # the same words, names and heights (tests/test_wire.py covers the format itself on the CPU)
    from sp1_b200 import lib as PL
    from tests import bincode_ref as BR
    w = M.widths(blob)
    prm = dict(log_stacking_height=log_stack, max_log_row_count=mlr, num_queries=nq, pow_bits=pow_bits, batch_pow_bits=batch_bits, gkr_pow_bits=gkr_bits)
    data = PL.shard_proof_to_bincode(words, names, heights, [a for a, _ in w], [b for _, b in w], **prm)
    flat, dn, dh = BR.flatten(BR.decode_shard_proof(data))
    assert dn == names and dh == list(heights) and (np.array(flat, dtype=np.uint64) == words).all()
    if prep_round is not None:
        lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()


@pytest.mark.parametrize("spec,log_stack,mlr", M.SHARD_SPECS + [M.RANDOM_SHARD_SPEC])
def test_prove_shard_matches_oracle(spec, log_stack, mlr):
    _run(spec, log_stack, mlr, seed=1200 + mlr)


def test_prove_shard_medium():
    spec = [(4096, 2, True), (1024 + 32, 3, False), (0, 1, False), (8192, 1, True), (2048, 4, False)]
    _run(spec, 12, 13, seed=99, nq=16, pow_bits=8, batch_bits=5, gkr_bits=6)


def test_prove_shard_from_upload_slots_is_identical():
    """the double-buffered async upload path (sp1b200_upload_begin) feeds the same proof as a plain host pointer"""
    import torch
    from sp1_b200 import Lib
    rng = np.random.default_rng(4242)
    spec = [(2048, 2, True), (512 + 32, 3, False), (4096, 1, False)]
    blob, heights, mains, preps, pv, names = M.spec_machine(rng, spec, names="Chip{:02d}")
    lib = Lib(0, log_stacking_height=11, max_log_row_count=12, **M.SMALL)
    mach = lib.machine_create(blob)
    _, prep_round = GP.commit_prep(lib, preps)
    dense = M.dense_main(mains)
    st0 = O.Challenger().st.copy()
    ref = lib.prove_shard(mach, prep_round, dense, heights, names, pv, st0.copy())
    pinned = torch.from_numpy(dense.view(np.int32)).pin_memory()
    other = torch.from_numpy((dense ^ np.uint32(1)).view(np.int32)).pin_memory()   # a different shard in the other slot
    d0 = lib.upload_begin(pinned, 0)
    d1 = lib.upload_begin(other, 1)
    a = lib.prove_shard(mach, prep_round, d0, heights, names, pv, st0.copy())
    d0b = lib.upload_begin(pinned, 0)          # slot 0 reused while slot 1 is still pending
    b = lib.prove_shard(mach, prep_round, d0b, heights, names, pv, st0.copy())
    assert d0 == d0b and d1 != d0
    assert (a == ref).all() and (b == ref).all()
    lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()


@pytest.mark.parametrize("skip", [1, 3])
def test_prove_shard_replays_non_minimal_witnesses(skip):
    """Whole-shard replay mode (grind_mode = 1) with deliberately NON-minimal witnesses: the oracle grinds the (skip+1)-th smallest
    valid witness at each of the three sites (as a racing reference prover may), the product replays exactly those three witnesses
    and must reproduce every proof word and the final challenger state — the mode used to cross-sign against a Rust-made proof."""
    import ctypes as C
    from sp1_b200 import Lib
    spec = [(1024, 2, True), (256 + 32, 3, False), (0, 1, False), (2048, 1, True)]
    log_stack, mlr, nq, pw, bpw, gpw = 10, 11, 8, 4, 2, 3
    blob, heights, mains, preps, pv, names, ch = M.shard_inputs(spec, 5150 + skip)
    L = O.lib()
    omin = ch.clone()
    _, wmin = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, omin, num_queries=nq, pow_bits=pw,
                                   batch_pow_bits=bpw, gkr_pow_bits=gpw)
    L.orc_set_grind_skip(C.c_uint32(skip))
    try:
        och = ch.clone()
        opc, owords = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, och, num_queries=nq, pow_bits=pw,
                                           batch_pow_bits=bpw, gkr_pow_bits=gpw)
        wl = np.zeros(8, np.uint32)
        n = L.orc_witness_log(O.ptr(wl), C.c_uint32(8))
    finally:
        L.orc_set_grind_skip(C.c_uint32(0))
    assert n == 3, "the shard proof has three grinding sites: LogUp-GKR, BaseFold batching, BaseFold queries"
    assert owords.size == wmin.size and (owords != wmin).any(), "non-minimal witnesses must change the proof"
    lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, num_queries=nq, pow_bits=pw, batch_pow_bits=bpw, gkr_pow_bits=gpw,
              grind_mode=1)
    mach = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    assert (pc == opc).all()
    st = ch.st.copy()
    words = GP.prove(lib, mach, prep_round, mains, heights, names, pv, st, replay=wl[:3])
    assert words.size == owords.size
    bad = np.nonzero(words != owords)[0]
    assert bad.size == 0, f"first differing words {bad[:8]} of {words.size}"
    assert (st == och.st).all()
    lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()


def test_setup_and_prove_shard_equals_setup_then_prove():
    """AirProver::setup_and_prove_shard (shard.rs:56-68): one call = commit the preprocessed traces, observe the verifying key the way
    MachineVerifyingKey::observe_into does (commitment, then the program words), prove.  Must equal the three steps done by hand, and the
    oracle's proof from the same post-vk transcript."""
    from sp1_b200 import Lib
    from sp1_b200.lib import HostChallenger
    spec = [(1024, 2, True), (256 + 32, 3, False), (0, 1, False), (2048, 1, True)]
    log_stack, mlr, nq, pw, bpw, gpw = 10, 11, 8, 4, 2, 3
    rng = np.random.default_rng(8080)
    blob, heights, mains, preps, pv, names = M.spec_machine(rng, spec, names="Chip{:02d}")
    vk_tail = np.concatenate([O.rand_field(rng, 3 + 7 + 7), O.to_monty(np.array([0])), np.zeros(6, np.uint32)])   # pc_start, cumulative sum x, y, flag, padding
    lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, num_queries=nq, pow_bits=pw, batch_pow_bits=bpw, gkr_pow_bits=gpw)
    mach = lib.machine_create(blob)
    prep_tabs = [p for p in preps if p is not None]
    prep_dense = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in prep_tabs]))
    rows, cols = [p.shape[1] for p in prep_tabs], [p.shape[0] for p in prep_tabs]
    dense = M.dense_main(mains)
    st = HostChallenger().st.copy()
    pc, prep_round, words = lib.setup_and_prove_shard(mach, prep_dense, rows, cols, vk_tail, dense, heights, names, pv, st)
    # by hand
    pc2, round2 = lib.jagged_commit(prep_tabs)
    hc = HostChallenger()
    hc.observe(pc2); hc.observe(vk_tail)
    post_vk = hc.st.copy()
    st2 = post_vk.copy()
    words2 = lib.prove_shard(mach, round2, dense, heights, names, pv, st2)
    assert (pc == pc2).all() and (words == words2).all() and (st == st2).all()
    # the returned round is the proving key: a second shard of the same program proves against it
    words3 = lib.prove_shard(mach, prep_round, dense, heights, names, pv, post_vk.copy())
    assert (words3 == words).all()
    och = O.Challenger(); och.st[:] = post_vk
    opc, owords = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, och, num_queries=nq, pow_bits=pw,
                                       batch_pow_bits=bpw, gkr_pow_bits=gpw)
    assert (opc == pc).all() and (owords == words).all() and (och.st == st).all()
    lib.jagged_round_free(prep_round); lib.jagged_round_free(round2)
    lib.machine_free(mach)
    lib.close()


# ---- the benchmark's shapes at reduced size, a full GKR batch table, and several contexts proving at once ------------------------------

def _oracle_shard(inp, log_stack, mlr, seed):
    blob, heights, mains, preps, pv, names = inp
    ch = O.Challenger(); ch.observe(O.rand_field(np.random.default_rng(seed), 9))
    och = ch.clone()
    opc, owords = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, och, **M.SMALL)
    return ch.st.copy(), opc, owords, och.st.copy()


def _prove_and_compare(inp, log_stack, mlr, seed):
    from sp1_b200 import Lib
    blob, heights, mains, preps, pv, names = inp
    st0, opc, owords, ost = _oracle_shard(inp, log_stack, mlr, seed)
    lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, **M.SMALL)
    mach = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    assert (pc == opc).all(), "preprocessed commitment differs from the oracle"
    st = st0.copy()
    words = GP.prove(lib, mach, prep_round, mains, heights, names, pv, st)
    assert words.size == owords.size and (words == owords).all(), M.shard_diff(words, owords)
    assert (st == ost).all(), "final challenger state differs from the oracle"
    lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()


@pytest.mark.parametrize("workload,mlr,log_stack", [("tinyc", 14, 12), ("tinyr", 14, 12)])
def test_prove_shard_workload_machines_match_oracle(workload, mlr, log_stack):
    """the calibrated core machine (36 chips, 640 interactions, a 682-column precompile table, 2.2 M cells) and the compress-shape machine
    (recursion chips with up to 36 preprocessed columns) at full smoke size, word for word"""
    inp = M.workload_machine(workload, seed=1300, max_log_rows=mlr)
    assert max(inp[1]) <= 1 << mlr
    _prove_and_compare(inp, log_stack, mlr, 1301)


def test_prove_shard_full_batch_table():
    """96 chips, the most the LogUp-GKR batch table takes (tests/test_gpu_gkr.py checks that 97 is an error): every phase of the shard
    proof at that chip count, with tiny heights (0 and 1 included)"""
    inp = M.spec_machine(np.random.default_rng(1311), M.full_table_spec(96, 1321, absent=True))
    _prove_and_compare(inp, 5, 5, 1330)


def test_concurrent_contexts_prove_their_own_shards():
    """four contexts on four host threads, as bench.py runs its in-flight provers: each has its own machine and preprocessed commit and
    proves a different shard (own heights and trace seed) twice, so that pooled memory is reused.  Every proof and final challenger
    state must equal the oracle's proof of that context's own input."""
    import threading
    import torch
    from sp1_b200 import Lib
    # (machine, max_log_row_count, log_stacking_height): two compress-shape shards of different heights (machine seeds 42 and 44) and
    # two calibrated core-like shards
    jobs = [(M.workload_machine("tinyr", seed=1400, max_log_rows=12, scale=0.25, machine_seed=42), 12, 10),
            (M.workload_machine("tinyr", seed=1401, max_log_rows=12, scale=0.25, machine_seed=44), 12, 10),
            (M.spec_machine(np.random.default_rng(1402), [M.Chip(1000, 4, False, 30, 3, 0, [12, 4, 9, 5] * 4), M.Chip(0, 2, False, None, 0, 0, [4]),
                                                          M.Chip(700, 3, True, 20, 0, 3, [9] * 10), M.Chip(96, 1, False, None, 0, 0, None)]), 10, 9),
            (M.spec_machine(np.random.default_rng(1403), [M.Chip(512, 4, False, 30, 3, 0, [12, 4, 9, 5] * 4), M.Chip(33, 2, False, None, 0, 0, [4]),
                                                          M.Chip(1024, 3, True, 20, 0, 3, [9] * 10), M.Chip(0, 1, False, None, 0, 0, None)]), 10, 9)]
    inputs = [inp for inp, _, _ in jobs]
    assert len({tuple(x[1]) for x in inputs}) == len(inputs), "every context must prove a shard of its own heights"
    oracle = [_oracle_shard(inp, ls, mlr, 1410 + k) for k, (inp, mlr, ls) in enumerate(jobs)]
    ctxs = []
    for (blob, heights, mains, preps, pv, names), mlr, ls in jobs:
        lib = Lib(0, log_stacking_height=ls, max_log_row_count=mlr, **M.SMALL)
        mach = lib.machine_create(blob)
        pc, prep_round = GP.commit_prep(lib, preps)
        ctxs.append((lib, mach, pc, prep_round))
    # half the contexts read their trace from device memory, half through the double-buffered upload slots from pinned host memory
    dense = [M.dense_main(inp[2]) for inp in inputs]
    d_dense = [torch.from_numpy(d.view(np.int32)).cuda() if k % 2 == 0 else torch.from_numpy(d.view(np.int32)).pin_memory()
               for k, d in enumerate(dense)]
    torch.cuda.synchronize()
    results = [[None, None] for _ in jobs]
    errors = []
    start = threading.Barrier(len(jobs))

    def run(k):
        try:
            lib, mach, _, prep_round = ctxs[k]
            blob, heights, mains, preps, pv, names = inputs[k]
            start.wait()
            for rep in range(2):
                src = d_dense[k] if k % 2 == 0 else lib.upload_begin(d_dense[k], rep)
                st = oracle[k][0].copy()
                words = lib.prove_shard(mach, prep_round, src, heights, names, pv, st)
                results[k][rep] = (words, st)
        except Exception as e:  # reported below, on the main thread
            errors.append((k, e))

    ths = [threading.Thread(target=run, args=(k,)) for k in range(len(jobs))]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errors, errors
    for k, (_, opc, owords, ost) in enumerate(oracle):
        assert (ctxs[k][2] == opc).all(), f"context {k}: preprocessed commitment differs from the oracle"
        for rep, (words, st) in enumerate(results[k]):
            assert words.size == owords.size and (words == owords).all(), f"context {k}, proof {rep}: " + M.shard_diff(words, owords)
            assert (st == ost).all(), f"context {k}, proof {rep}: final challenger state differs from the oracle"
    for lib, mach, _, prep_round in ctxs:
        lib.jagged_round_free(prep_round)
        lib.machine_free(mach)
        lib.close()
