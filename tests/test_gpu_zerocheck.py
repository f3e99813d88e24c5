"""GPU parity tests (zerocheck): constraint bytecode interpreter + multi-chip sumcheck through the C ABI vs the oracle
(which also runs the restated ShardVerifier::verify_zerocheck on its own proof).  Bit-exact."""
import numpy as np
import pytest

from tests.machines import Chip, oracle_zerocheck, product_zerocheck, spec_machine, workload_machine
from tests.test_oracle import _synth_machine

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("spec,mlr", [
    ([(8, 1, False)], 3),
    ([(5, 1, False), (0, 2, False), (6, 1, True)], 3),
    ([(1, 1, False), (2, 1, True)], 4),
    ([(32, 3, True), (96, 2, False), (128, 1, False)], 7),
    ([(4096, 2, True), (1000, 12, False), (0, 1, False), (2048 + 32, 5, False)], 13),
    # long-lived intermediates: register pressure ~ groups -> every register-file tier (<= 8, <= 16, <= 32 in shared memory,
    # local-memory fallback above) in one proof, next to a flat chip
    ([(512, 6, False, True), (300, 14, True, True), (1024, 28, False, True), (96, 40, False, True), (2048, 3, True)], 12),
    # the reference's largest register tiers (sys/lib/zerocheck/sequential.cu:298-335: 256 / 512 / 1024 registers): programs whose
    # re-scheduled live set is ~250, ~500 and ~1000 registers -> the global-memory register file, next to a shared-memory chip;
    # heights on both sides of the "pieces" threshold (<= 16 blocks of 128 row pairs)
    ([(192, 250, False, True), (64, 500, True, True), (8192, 3, True), (96, 1000, False, True), (6000, 300, False, True)], 13),
])
def test_zerocheck_matches_oracle(spec, mlr):
    from sp1_b200 import Lib
    rng = np.random.default_rng(900 + mlr)
    blob, heights, mains, preps, pv = _synth_machine(rng, spec)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21))
    mach = lib.machine_create(blob)
    if any(len(s_) > 3 and s_[1] >= 250 for s_ in spec):
        regs = [lib.machine_chip_regs(mach, k) for k in range(len(spec))]
        assert max(regs) > 900 and sorted(regs)[-2] > 450 and min(regs) <= 32, regs   # the tiers the case is meant to exercise
    _check_zerocheck(lib, mach, rng, blob, heights, mains, preps, pv, mlr)
    lib.machine_free(mach)
    lib.close()


def _check_zerocheck(lib, mach, rng, blob, heights, mains, preps, pv, mlr):
    gp, st0, openings, owords, ost = oracle_zerocheck(rng, blob, heights, mains, preps, pv, mlr)
    words, st = product_zerocheck(lib, mach, heights, mains, preps, pv, gp, st0, openings)
    assert words.size == owords.size, (words.size, owords.size)
    bad = np.nonzero(words != owords)[0]
    assert bad.size == 0, f"first differing words {bad[:8]} of {words.size}"
    assert (st == ost).all()


# calibrated chips: constraint counts from the workloads' chip_stats.json range (up to 9 per group), filler main columns, several
# further preprocessed columns (LOAD_PREP of column 0 next to committed-only columns)
CALIBRATED_SPECS = [
    ([Chip(700, 4, True, 36, 5, 3), Chip(96, 14, False, 120, 0, 0), Chip(0, 2, True, 18, 1, 2), Chip(33, 1, True, 9, 7, 35),
      Chip(2048, 40, False, 360, 2, 0)], 11),
    ([Chip(1, 2, True, 18, 0, 4), Chip(2, 1, False, 7, 3, 0), Chip(4, 3, True, 20, 2, 1)], 2),
]


@pytest.mark.parametrize("case", range(len(CALIBRATED_SPECS)))
def test_zerocheck_calibrated_chips_match_oracle(case):
    from sp1_b200 import Lib
    spec, mlr = CALIBRATED_SPECS[case]
    rng = np.random.default_rng(1100 + case)
    blob, heights, mains, preps, pv, _ = spec_machine(rng, spec)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21))
    mach = lib.machine_create(blob)
    _check_zerocheck(lib, mach, rng, blob, heights, mains, preps, pv, mlr)
    lib.machine_free(mach)
    lib.close()


@pytest.mark.parametrize("workload,mlr", [("tinyc", 12), ("tinyr", 12)])
def test_zerocheck_workload_machines_match_oracle(workload, mlr):
    """the benchmark's calibrated core machine and compress-shape machine at a quarter of their size"""
    from sp1_b200 import Lib
    blob, heights, mains, preps, pv, _ = workload_machine(workload, seed=1110, max_log_rows=mlr, scale=0.25)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21))
    mach = lib.machine_create(blob)
    _check_zerocheck(lib, mach, np.random.default_rng(1111), blob, heights, mains, preps, pv, mlr)
    lib.machine_free(mach)
    lib.close()
