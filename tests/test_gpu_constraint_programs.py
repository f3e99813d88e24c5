"""A seeded sweep of random constraint programs (tests/machines.py random_program) through the GPU zerocheck against the oracle, word
for word: machines of 2 to 6 random-program chips with random register-file tiers, heights and max_log_row_count.  The sweep also
asserts that, across its machines, every tier, the pieces path, every opcode, a direct assert on a leaf, a constant and a public value,
a permuted alpha order, a register asserted twice and chips of constraint degree 1, 2 and 3 each appeared, so that a change to the generator cannot quietly narrow it."""
import collections

import numpy as np
import pytest

from tests import machines as M

pytestmark = pytest.mark.gpu

N_MACHINES = 40
# live-set ranges that land in each register-file tier (the re-scheduled pressure is the live set + 3 to 5 registers)
LIVE = [(0, 3), (6, 11), (14, 26), (32, 110), (130, 400)]


def _sweep_machine(seed):
    """-> (chips, max_log_row_count) of sweep machine `seed`"""
    rng = np.random.default_rng(seed)
    mlr = int(rng.integers(1, 11))
    chips = []
    for k in range(int(rng.integers(2, 7))):
        tier = int(rng.integers(0, 5))
        top = 1 << mlr
        heights = [0, 1, 2, 3, top, 2 * int(rng.integers(0, top // 2 + 1)) + 1, 1 << int(rng.integers(0, mlr + 1))]
        heights.append(heights[-1] + 1)
        h = min(heights[int(rng.integers(0, len(heights)))], top)
        if tier == 4:
            h = min(h, 512)                         # the oracle interprets a ~1000-instruction program per row
        n_asserts = 0 if rng.integers(0, 8) == 0 else int(rng.integers(6, 25))
        chips.append(M.prog_chip(h, seed * 10 + k, n_asserts=n_asserts, live=int(rng.integers(*LIVE[tier])), cols=int(rng.integers(1, 12)),
                                 prep=int(rng.integers(0, 4)), n_ops=int(rng.integers(5, 200)), direct=bool(rng.integers(0, 4)),
                                 dup=bool(rng.integers(0, 4) == 0), max_deg=int(rng.integers(1, 4))))
    return chips, mlr


def test_random_constraint_programs_match_oracle():
    from sp1_b200 import Lib
    tiers, features, pieces, failures = collections.Counter(), set(), 0, []
    for seed in range(N_MACHINES):
        chips, mlr = _sweep_machine(seed)
        rng = np.random.default_rng(50_000 + seed)
        blob, heights, mains, preps, pv, _ = M.spec_machine(rng, chips, interactions=False)
        lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21))
        try:
            mach = lib.machine_create(blob)
            regs = [lib.machine_chip_regs(mach, k) for k in range(len(chips))]
            gp, st0, openings, owords, ost = M.oracle_zerocheck(rng, blob, heights, mains, preps, pv, mlr)
            words, st = M.product_zerocheck(lib, mach, heights, mains, preps, pv, gp, st0, openings)
            lib.machine_free(mach)
        finally:
            lib.close()
        for k, c in enumerate(chips):
            rp = M.random_program(c.program)
            features |= rp.features
            if rp.asserts and heights[k]:
                tiers[M.zc_tier(regs[k])] += 1
                pieces += M.lowered_shape(rp.words)[2]
        if words.size != owords.size or (words != owords).any() or (st != ost).any():
            bad = np.nonzero(words[:min(words.size, owords.size)] != owords[:min(words.size, owords.size)])[0]
            where = ", ".join(f"chip {k}: h {h}, {M.TIER_NAMES[M.zc_tier(r)]} ({r} registers), {c.program}"
                              for k, (c, h, r) in enumerate(zip(chips, heights, regs)))
            failures.append(f"seed {seed} (max_log_row_count {mlr}): {M.first_diff(words, owords, 'zerocheck proof')}"
                            f"{'' if bad.size else '; the challenger state differs'}; first differing word "
                            f"{int(bad[0]) if bad.size else None}; {where}")
    assert not failures, "\n".join(failures)
    print(f"constrained chips per tier: {dict((M.TIER_NAMES[t], n) for t, n in sorted(tiers.items()))}; chips that take pieces: {pieces}")
    missing = [M.TIER_NAMES[t] for t in range(5) if t not in tiers]
    missing += [f for f in M.OPCODE_NAMES + ["assert_leaf", "assert_const", "assert_public", "alpha_permuted", "dup_assert", "cube",
                                            "alias", "overwrite", "dead_code", "degree_1", "degree_2", "degree_3"] if f not in features]
    missing += [] if pieces else ["the pieces path"]
    assert not missing, f"the sweep did not cover: {missing}"
