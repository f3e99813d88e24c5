"""GPU parity tests on extreme Montgomery words: every proving phase, word for word against the oracle, on traces, tables and points
whose words are all p - 1, 0, ONE, p - ONE or a mixture of such words with uniform ones (oracle_lib.words), and the RS-encode branches
that uniform tests at the usual sizes do not reach.

The hot kernels sum up to four 32 x 32-bit products in a 64-bit accumulator and reduce once (kb::monty_reduce2, domain x < 2p 2^32).
Uniform operands stay far from that bound: a group of five products overflows it in 3e-7 of accumulations.  With one operand at the word
p - 1 it is 0.7 %, so these inputs make a fifth product in any of those groups fail at the sizes below."""
import os

import numpy as np
import pytest

from tests import gpu_prove as GP
from tests import machines as M
from tests import oracle_lib as O
from tests.machines import Chip, prog_chip

pytestmark = pytest.mark.gpu

KINDS = O.WORD_KINDS
HEAVY = ("max", "mixed")     # the kinds that load the accumulators; the others run where a case is cheap


@pytest.fixture(scope="module")
def lib():
    from sp1_b200 import Lib
    L = Lib(device=0)
    yield L
    L.close()


@pytest.fixture(scope="module")
def lib_generic():
    """a context created under SP1B200_GENERIC_NTT=1: the generic RS-encode kernels at every size (the variable is read when a context
    is created, and restored right after)"""
    from sp1_b200 import Lib
    old = os.environ.get("SP1B200_GENERIC_NTT")
    os.environ["SP1B200_GENERIC_NTT"] = "1"
    try:
        L = Lib(device=0)
    finally:
        if old is None:
            del os.environ["SP1B200_GENERIC_NTT"]
        else:
            os.environ["SP1B200_GENERIC_NTT"] = old
    yield L
    L.close()


def _encode(lib, msg, lb):
    ncols, n = msg.shape
    out = np.zeros((ncols, n << lb), np.uint32)
    lib.rs_encode(msg, out, ncols, n.bit_length() - 1, lb)
    return out


# ---- RS-encode and Merkle commit --------------------------------------------------------------------------------------------------------
# the fast paths: step A at L1 = 7 (log_h 18) and L1 = 10 (log_h 21), the generic step A at L1 = 8 (log_h 19) with the fast step B,
# and the generic kernels throughout (lib_generic)
@pytest.mark.parametrize("kind", HEAVY)
@pytest.mark.parametrize("log_h,ncols,lb", [(18, 2, 2), (19, 1, 2), (21, 1, 1), (14, 3, 2)])
def test_rs_encode_and_merkle_commit_on_extreme_words(lib, lib_generic, kind, log_h, ncols, lb):
    msg = O.words(np.random.default_rng(3000 + log_h), (ncols, 1 << log_h), kind)
    want = O.rs_encode(msg, lb)
    assert (_encode(lib, msg, lb) == want).all(), "fast path"
    assert (_encode(lib_generic, msg, lb) == want).all(), "generic path"
    if log_h + lb <= 16:
        root, commit = lib.merkle_commit(want, ncols, log_h + lb)
        oroot, ocommit = O.merkle_commit(want)
        assert (root == oroot).all() and (commit == ocommit).all()


# the branches no other test reaches: the step-chain twist of the fast step A (L1 = 10 with blowup 3: sh = 24 - L1 - b = 11 < 12),
# three column groups of 64 MiB of output with a ragged last one (log_h 21 with 5 columns, log_h 18 with 33), blowup 4 on every
# path, and the generic kernels at every L1 = log_h - 11 from 1 to 10
RS_BRANCHES = ([(21, 1, 3), (21, 5, 2), (18, 33, 2), (5, 2, 4), (11, 3, 4), (18, 2, 4), (20, 1, 4)]
               + [(11 + l1, 1, 2) for l1 in range(1, 11)])


@pytest.mark.parametrize("log_h,ncols,lb", RS_BRANCHES)
def test_rs_encode_branches_match_oracle_and_the_generic_path(lib, lib_generic, log_h, ncols, lb):
    msg = O.words(np.random.default_rng(3100 + 8 * log_h + lb), (ncols, 1 << log_h), "mixed")
    want = O.rs_encode(msg, lb)
    got = _encode(lib, msg, lb)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, f"columns {bad.tolist()} differ from the oracle"
    assert (_encode(lib_generic, msg, lb) == want).all(), "generic path"


# ---- stacked BaseFold ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("ncols,log_h", [([9, 17], 8), ([33], 10)])
def test_stacked_basefold_on_extreme_words(kind, ncols, log_h):
    """columns and evaluation-point coordinates of the kind: batch_columns_kernel sums two products of a word and a batching
    coefficient per reduction"""
    GP.check_stacked(ncols, log_h, nq=10, pow_bits=6, batch_bits=3, seed=3200 + log_h, kind=kind)


# ---- jagged PCS -------------------------------------------------------------------------------------------------------------------------
def _jagged_shapes(k):
    """two rounds whose column heights are 2^k times odd numbers: the library sums K = k rounds from the base-field trace"""
    u = 1 << k
    return [[(129 * u, 5), (0, 2), (67 * u, 3)], [(33 * u, 7)]]


@pytest.mark.parametrize("k,kind", [(k, kind) for k in range(6) for kind in HEAVY] + [(5, kind) for kind in KINDS if kind not in HEAVY])
def test_jagged_on_extreme_words(k, kind):
    """tables and z_row of the kind, at every trace-round count K: the trace rounds' wdot sums four products per reduction, and the
    column claims go through table_evals_partial_kernel"""
    # the library takes max_log_row_count <= log_m + 1, and the K = 0 tables span 2^11 words
    shapes, log_stack, mlr = _jagged_shapes(k), 10, 13 if k else 11
    assert GP.trace_rounds_k(shapes, log_stack, mlr) == k
    GP.check_jagged(shapes, log_stack, mlr, seed=3300 + k, kind=kind)


@pytest.mark.parametrize("seed", range(24))
def test_lazy_sums_of_words_p_minus_1_under_fresh_challenges(seed):
    """With every word at p - 1, whether a group of five products would overflow depends on the challenges alone: the batching
    coefficients of batch_columns_kernel and the jagged weights of wdot are fixed for a proof, so one proof tries only a few dozen
    accumulator groups.  Fresh transcripts give fresh challenges: a stacked BaseFold proof of 40 columns and a jagged proof that sums
    K = 5 rounds from the trace, each from its own seed"""
    GP.check_stacked([40], 4, nq=4, pow_bits=1, batch_bits=1, seed=3700 + seed, kind="max")
    shapes = [[(96, 5)], [(32, 3)]]
    assert GP.trace_rounds_k(shapes, 5, 7) == 5
    GP.check_jagged(shapes, 5, 7, seed=3800 + seed, nq=4, pow_bits=1, batch_bits=1, kind="max")


# ---- LogUp-GKR ------------------------------------------------------------------------------------------------------------------------------
GKR_SPEC = [Chip(1000, 4, False, 30, 3, 0, [12, 4, 9, 5, 1, 7, 12, 3]), Chip(600, 3, True, 20, 0, 3, [9] * 6 + [12] * 4),
            Chip(64, 1, False), Chip(0, 2, True, None, 0, 2, [4] * 2), Chip(33, 2, True, None, 1, 1, [12])]


@pytest.mark.parametrize("kind", KINDS)
def test_logup_gkr_on_extreme_traces(kind):
    """calibrated messages of up to 12 values, light interactions, an absent chip and preprocessed columns in the messages"""
    from sp1_b200 import Lib
    mlr = 10
    blob, heights, mains, preps, _, _ = M.spec_machine(np.random.default_rng(3400), GKR_SPEC, kind=kind)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=mlr, gkr_pow_bits=4)
    mach = lib.machine_create(blob)
    GP.check_gkr(lib, mach, blob, heights, mains, preps, mlr, 3401)
    lib.machine_free(mach)
    lib.close()


# ---- zerocheck ------------------------------------------------------------------------------------------------------------------------------
# random programs of degree 3 at every register-file tier (live set 0 / 10 / 24 / 80 / 300: <= 8, <= 16, <= 32 in shared memory, local,
# global), each with the constant whose word is p - 1, next to template chips: both operands of a base-field product are extreme words
ZC_SPEC = [prog_chip(64, 3501, max_word=True, prep=2), prog_chip(48, 3502, live=10, max_word=True),
           prog_chip(33, 3503, live=24, dup=True, max_word=True), prog_chip(100, 3504, live=80, n_asserts=12, max_word=True),
           prog_chip(17, 3505, live=300, n_asserts=12, max_word=True), Chip(256, 2, True, 18, 1, 2), Chip(96, 6, False, deep=True)]


@pytest.mark.parametrize("kind", KINDS)
def test_zerocheck_on_extreme_traces(kind):
    from sp1_b200 import Lib
    mlr = 8
    rng = np.random.default_rng(3500)
    blob, heights, mains, preps, pv, _ = M.spec_machine(rng, ZC_SPEC, interactions=False, kind=kind)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=mlr)
    mach = lib.machine_create(blob)
    for k, c in enumerate(ZC_SPEC):
        if c.program is not None:
            assert M.zc_tier(lib.machine_chip_regs(mach, k)) == M.zc_tier(c.program.live + 4), (k, lib.machine_chip_regs(mach, k))
    GP.check_zerocheck(lib, mach, rng, blob, heights, mains, preps, pv, mlr)
    lib.machine_free(mach)
    lib.close()


# ---- the whole shard ------------------------------------------------------------------------------------------------------------------------
SHARD_SPEC = ([prog_chip(64, 3601, prep=2, max_word=True), Chip(32, 1, True), prog_chip(17, 3602, live=10, dup=True, max_word=True),
               Chip(16, 2, False, vps=()), prog_chip(0, 3603, max_word=True), Chip(40, 2, True, 12, 2, 1, [12, 3])], 5, 7)


@pytest.mark.parametrize("kind", KINDS)
def test_whole_shard_on_extreme_traces(kind):
    """prove_shard equals the oracle's proof and final challenger; the library's verifier and the oracle's accept it; the constraint
    report is clean; for `max`, the proof from the upload slots (device input) is the same"""
    import torch
    from sp1_b200 import Lib
    from sp1_b200.lib import parse_constraint_report, verdict_name
    spec, log_stack, mlr = SHARD_SPEC
    blob, heights, mains, preps, pv, names, ch = M.shard_inputs(spec, 3600, kind=kind)
    och = ch.clone()
    opc, owords = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, och, **M.SMALL)
    lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, **M.SMALL)
    mach = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    assert (pc == opc).all(), "preprocessed commitment differs from the oracle"
    dense = M.dense_main(mains)
    assert parse_constraint_report(lib.debug_constraints_words(mach, prep_round, dense, heights, pv)) == {}, "constraints fail"
    st = ch.st.copy()
    words = lib.prove_shard(mach, prep_round, dense, heights, names, pv, st)
    assert words.size == owords.size and (words == owords).all(), M.shard_diff(words, owords)
    assert (st == och.st).all(), "final challenger state differs from the oracle"
    if kind == "max":
        pinned = torch.from_numpy(dense.view(np.int32)).pin_memory()
        st2 = ch.st.copy()
        words2 = lib.prove_shard(mach, prep_round, lib.upload_begin(pinned, 0), heights, names, pv, st2)
        assert (words2 == owords).all() and (st2 == och.st).all(), "the proof from the upload slot differs"
    verdict, vst = lib.verify_shard(mach, pc, heights, names, words, ch.st.copy())
    assert verdict == 0, f"the library rejects the proof: {verdict_name(verdict)}"
    assert (vst == och.st).all(), "verifier and prover end in different challenger states"
    v = ch.clone()
    assert O.verify_shard(blob, heights, names, log_stack, mlr, v, pc, words, **M.SMALL) == 0, "the oracle rejects the proof"
    lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()
