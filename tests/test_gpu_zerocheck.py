"""GPU parity tests (zerocheck): constraint bytecode interpreter + multi-chip sumcheck through the C ABI vs the oracle
(which also runs the restated ShardVerifier::verify_zerocheck on its own proof).  Bit-exact."""
import numpy as np
import pytest

from tests import gpu_prove as GP
from tests.machines import PROGRAM_ZC_CASES, Chip, lowered_shape, random_program, spec_machine, workload_machine, zc_tier

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("spec,mlr", [
    ([(8, 1, False)], 3),
    ([(5, 1, False), (0, 2, False), (6, 1, True)], 3),
    ([(1, 1, False), (2, 1, True)], 4),
    ([(32, 3, True), (96, 2, False), (128, 1, False)], 7),
    ([(4096, 2, True), (1000, 12, False), (0, 1, False), (2048 + 32, 5, False)], 13),
    # long-lived intermediates: register pressure ~ groups -> every register-file tier (<= 8, <= 16, <= 32 in shared memory,
    # local-memory fallback above) in one proof, next to a flat chip
    ([Chip(512, 6, False, deep=True), Chip(300, 14, True, deep=True), Chip(1024, 28, False, deep=True), Chip(96, 40, False, deep=True),
      (2048, 3, True)], 12),
    # the reference's largest register tiers (sys/lib/zerocheck/sequential.cu:298-335: 256 / 512 / 1024 registers): programs whose
    # re-scheduled live set is ~250, ~500 and ~1000 registers -> the global-memory register file, next to a shared-memory chip;
    # heights on both sides of the "pieces" threshold (<= 16 blocks of 128 row pairs)
    ([Chip(192, 250, False, deep=True), Chip(64, 500, True, deep=True), (8192, 3, True), Chip(96, 1000, False, deep=True),
      Chip(6000, 300, False, deep=True)], 13),
] + PROGRAM_ZC_CASES)   # and random constraint programs (tests/machines.py random_program)
def test_zerocheck_matches_oracle(spec, mlr):
    from sp1_b200 import Lib
    rng = np.random.default_rng(900 + mlr)
    blob, heights, mains, preps, pv, _ = spec_machine(rng, spec, interactions=False)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21))
    mach = lib.machine_create(blob)
    if any(Chip(*s_).deep and s_[1] >= 250 for s_ in spec):
        regs = [lib.machine_chip_regs(mach, k) for k in range(len(spec))]
        assert max(regs) > 900 and sorted(regs)[-2] > 450 and min(regs) <= 32, regs   # the tiers the case is meant to exercise
    for k, c in enumerate(Chip(*s_) for s_ in spec):
        if c.program is not None and c.program.n_asserts:
            # the tier and the path each random chip is meant to exercise: the live set + a few registers; a 150-op body takes pieces
            assert zc_tier(lib.machine_chip_regs(mach, k)) == zc_tier(c.program.live + 4), (k, lib.machine_chip_regs(mach, k))
            assert c.program.n_ops < 150 or lowered_shape(random_program(c.program).words)[2], k
    GP.check_zerocheck(lib, mach, rng, blob, heights, mains, preps, pv, mlr)
    lib.machine_free(mach)
    lib.close()


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
    GP.check_zerocheck(lib, mach, rng, blob, heights, mains, preps, pv, mlr)
    lib.machine_free(mach)
    lib.close()


@pytest.mark.parametrize("workload,mlr", [("tinyc", 12), ("tinyr", 12)])
def test_zerocheck_workload_machines_match_oracle(workload, mlr):
    """the benchmark's calibrated core machine and compress-shape machine at a quarter of their size"""
    from sp1_b200 import Lib
    blob, heights, mains, preps, pv, _ = workload_machine(workload, seed=1110, max_log_rows=mlr, scale=0.25)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21))
    mach = lib.machine_create(blob)
    GP.check_zerocheck(lib, mach, np.random.default_rng(1111), blob, heights, mains, preps, pv, mlr)
    lib.machine_free(mach)
    lib.close()
