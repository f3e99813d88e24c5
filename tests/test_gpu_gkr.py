"""GPU parity tests (LogUp-GKR): fraction circuit + per-layer sumchecks through the C ABI vs the oracle (which also runs
the restated LogUpGkrVerifier::verify_logup_gkr on its own proof).  Bit-exact, including the challenger state."""
import numpy as np
import pytest

from tests import gpu_prove as GP
from tests import machines as M
from tests import oracle_lib as O
from tests.machines import Chip, full_table_spec, n_interactions, shard_diff, spec_machine

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("spec,mlr", [
    ([(8, 1, False)], 3),
    ([(5, 1, False), (0, 2, False), (6, 1, True)], 3),
    ([(1, 1, False), (2, 1, True)], 4),
    ([(32, 2, True), (96, 1, False), (128, 1, False)], 7),
    ([(4096, 2, True), (1000, 3, False), (0, 1, False), (2048 + 32, 5, False)], 13),
])
def test_logup_gkr_matches_oracle(spec, mlr):
    from sp1_b200 import Lib
    rng = np.random.default_rng(950 + mlr)
    blob, heights, mains, preps, pv, _ = spec_machine(rng, spec)
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 4))
    och = ch.clone()
    owords = O.gkr_prove_verify(blob, heights, mains, preps, mlr, och, gkr_pow_bits=6)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21), gkr_pow_bits=6)
    mach = lib.machine_create(blob)
    d_mains, d_preps = GP.upload(mains, preps)
    st = ch.st.copy()
    words = lib.logup_gkr(mach, heights, d_mains, d_preps, st)
    assert words.size == owords.size, (words.size, owords.size)
    bad = np.nonzero(words != owords)[0]
    assert bad.size == 0, f"first differing words {bad[:8]} of {words.size}"
    assert (st == och.st).all()
    lib.machine_free(mach)
    lib.close()


def test_logup_gkr_and_whole_shard_with_silent_chips():
    """chips that carry constraints but no LogUp interactions, absent chips, tiny heights: GKR alone and the whole shard proof"""
    from sp1_b200 import Lib
    for spec, silent, mlr in M.GKR_EDGE_CASES:
        rng = np.random.default_rng(960 + mlr)
        blob, heights, mains, preps, pv, names = spec_machine(rng, M.silent(spec, silent), names="Chip{:02d}")
        ch = O.Challenger(); ch.observe(O.rand_field(rng, 4))
        och = ch.clone()
        owords = O.gkr_prove_verify(blob, heights, mains, preps, mlr, och, gkr_pow_bits=4)
        log_stack = min(mlr, 4)
        lib = Lib(0, max_log_row_count=mlr, log_stacking_height=log_stack, gkr_pow_bits=4, num_queries=4, pow_bits=3, batch_pow_bits=2)
        mach = lib.machine_create(blob)
        d_mains, d_preps = GP.upload(mains, preps)
        st = ch.st.copy()
        words = lib.logup_gkr(mach, heights, d_mains, d_preps, st)
        assert words.size == owords.size and (words == owords).all()
        assert (st == och.st).all()
        # whole shard on the same machine
        c2 = O.Challenger(); c2.observe(O.rand_field(rng, 5))
        oc2 = c2.clone()
        opc, ow = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, oc2, num_queries=4, pow_bits=3,
                                       batch_pow_bits=2, gkr_pow_bits=4)
        pc, prep_round = GP.commit_prep(lib, preps)
        assert (pc == opc).all()
        st2 = c2.st.copy()
        w2 = GP.prove(lib, mach, prep_round, mains, heights, names, pv, st2)
        assert w2.size == ow.size and (w2 == ow).all() and (st2 == oc2.st).all()
        if prep_round is not None:
            lib.jagged_round_free(prep_round)
        lib.machine_free(mach)
        lib.close()


# ---- the benchmark's chip shapes: calibrated interactions, >= 2^10 padded interactions, looping grid-stride kernels, mlr = 2, a full
# batch table -------------------------------------------------------------------------------------------------------------------------
PRE = [9] * 50 + [5] * 4          # the calibrated precompile table's messages (sp1_b200.workload.synthetic_machine)
SUM2_THREADS_TOTAL = 396 * 128    # gkr_sum2_kernel: at most 396 blocks of 128 threads (gkr_driver.inc)
FIX_THREADS_TOTAL = 528 * 256     # gkr_fix2_kernel / gkr_fix_sum_kernel: at most 528 blocks of 256 threads


def _gkr_case(spec, mlr, seed):
    from sp1_b200 import Lib
    blob, heights, mains, preps, pv, _ = spec_machine(np.random.default_rng(seed), spec)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21), gkr_pow_bits=4)
    mach = lib.machine_create(blob)
    GP.check_gkr(lib, mach, blob, heights, mains, preps, mlr, seed + 1)
    lib.machine_free(mach)
    lib.close()
    return blob, heights


def _work_items(blob, heights, spec):
    """(quads of gkr_sum2_kernel, pairs of gkr_fix2_kernel, pairs of the first gkr_fix_sum_kernel) on layer 0"""
    from sp1_b200 import synth_air as SA
    q = f2 = fs = 0
    for c, h in zip(spec, heights):
        c = Chip(*c)
        I = SA.synth_interactions_calibrated(c.g, c.wp, list(c.vps))[0] if c.vps else 0
        rows = (h + 1) // 2
        q += I * ((rows + 3) // 4)
        r2 = (rows + 3) // 4
        f2 += I * ((r2 + 1) // 2)
        r3 = (r2 + 1) // 2
        fs += I * ((r3 + 1) // 2)
    return q, f2, fs


def test_logup_gkr_calibrated_ten_interaction_variables():
    """690 interactions (2^10 padded: the interaction rounds take a second stride over 256 threads, the flatten runs over 1024 slots),
    messages of 12 values (16 beta powers), filler columns and four preprocessed columns in the openings, an absent chip"""
    spec = [Chip(1000, 4, False, 30, 3, 0, [12, 4, 9, 5, 1, 7, 12, 3] * 8), Chip(600, 3, True, 20, 0, 3, [9] * 54 + [12] * 100),
            Chip(2048 + 32, 2, False, None, 0, 0, [2, 3] * 60), Chip(0, 2, True, None, 0, 2, [4] * 5)]
    blob, _ = _gkr_case(spec, 12, 970)
    assert 512 < n_interactions(blob) <= 1024


def test_logup_gkr_calibrated_eleven_interaction_variables_and_looping_kernels():
    """nine copies of the calibrated precompile table's messages at full height: 1222 interactions (2^11 padded), and enough work
    items that gkr_sum2_kernel, gkr_fix2_kernel and gkr_fix_sum_kernel loop over their grids with jobs changing inside a block"""
    spec = [Chip(4096, 6, i % 2 == 0, 40, 2, 2 if i % 2 == 0 else 0, PRE + [12] * 10) for i in range(9)] + [Chip(3000, 2, False, None, 0, 0, [12] * 30)]
    blob, heights = _gkr_case(spec, 12, 980)
    assert n_interactions(blob) > 1024
    q, f2, fs = _work_items(blob, heights, spec)
    assert q > SUM2_THREADS_TOTAL and f2 > FIX_THREADS_TOTAL and fs > FIX_THREADS_TOTAL, (q, f2, fs)


MLR2_CASES = [
    # heights 0..4 under max_log_row_count = 2: one row variable per layer, a tree of two levels
    [Chip(4, 1, False, None, 0, 0, [12, 3]), Chip(3, 1, True, None, 0, 2, [5]), Chip(0, 1, False, None, 0, 0, [4]),
     Chip(1, 2, False, 12, 1, 0, [4, 4]), Chip(2, 1, False, None, 0, 0, ())],
    [Chip(2, 1, True), Chip(4, 2, False), Chip(1, 1, False)],
]


@pytest.mark.parametrize("case", range(len(MLR2_CASES)))
def test_logup_gkr_and_whole_shard_two_row_variables(case):
    """max_log_row_count = 2 is the only use of gkr_fix2_kernel<uint32_t, false>, of gkr_sum2_kernel<uint32_t> with two = 0 and of
    gkr_first_level_kernel without level 2: LogUp-GKR alone and the whole shard"""
    from sp1_b200 import Lib
    mlr, log_stack = 2, 2
    seed = 990 + case
    blob, heights, mains, preps, pv, names = spec_machine(np.random.default_rng(seed), MLR2_CASES[case])
    prm = dict(num_queries=4, pow_bits=3, batch_pow_bits=2, gkr_pow_bits=4)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=log_stack, **prm)
    mach = lib.machine_create(blob)
    GP.check_gkr(lib, mach, blob, heights, mains, preps, mlr, seed + 1)
    ch = O.Challenger(); ch.observe(O.rand_field(np.random.default_rng(seed + 2), 9))
    och = ch.clone()
    opc, owords = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, och, **prm)
    pc, prep_round = GP.commit_prep(lib, preps)
    assert (pc == opc).all(), "preprocessed commitment differs from the oracle"
    st = ch.st.copy()
    words = GP.prove(lib, mach, prep_round, mains, heights, names, pv, st)
    assert words.size == owords.size and (words == owords).all(), shard_diff(words, owords)
    assert (st == och.st).all(), "final challenger state differs from the oracle"
    lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()


def test_logup_gkr_full_batch_table_then_one_chip_too_many():
    """96 chips with interactions fill the batch table (find_job at n = MAX_JOBS, the largest parameter block); 97 chips must be a
    clean error, after which the same context proves a valid machine"""
    from sp1_b200 import Lib
    from sp1_b200.lib import Sp1B200Error
    mlr = 5
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=mlr, gkr_pow_bits=4)
    blob, heights, mains, preps, pv, _ = spec_machine(np.random.default_rng(1001), full_table_spec(97, 1000))
    mach = lib.machine_create(blob)
    d_mains, d_preps = GP.upload(mains, preps)
    with pytest.raises(Sp1B200Error, match="batch table"):
        lib.logup_gkr(mach, heights, d_mains, d_preps, O.Challenger().st.copy())
    lib.machine_free(mach)
    for k, absent in enumerate((False, True)):
        blob, heights, mains, preps, pv, _ = spec_machine(np.random.default_rng(1002 + k), full_table_spec(96, 1010 + k, absent))
        mach = lib.machine_create(blob)
        GP.check_gkr(lib, mach, blob, heights, mains, preps, mlr, 1020 + k)
        lib.machine_free(mach)
    lib.close()
