"""GPU path against the committed golden fixtures (tests/golden/shard_proofs.json): no oracle call on this path — the CUDA
library alone must reproduce the commitments, every proof word (SHA-256) and the final challenger state."""
import pytest

from tests import golden_util as G
from tests import gpu_prove as GP

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", G.cases(), ids=lambda c: c["name"])
def test_gpu_reproduces_golden_shard_proofs(case):
    from sp1_b200 import Lib
    blob, heights, mains, preps, pv, names, ch = G.inputs_of(case)
    lib = Lib(0, log_stacking_height=case["log_stacking_height"], max_log_row_count=case["max_log_row_count"],
              num_queries=case["num_queries"], pow_bits=case["pow_bits"], batch_pow_bits=case["batch_pow_bits"],
              gkr_pow_bits=case["gkr_pow_bits"])
    mach = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    st = ch.st.copy()
    words = GP.prove(lib, mach, prep_round, mains, heights, names, pv, st)
    G.check_words(case, pc, words, st)
    if prep_round is not None:
        lib.jagged_round_free(prep_round)
    lib.machine_free(mach)
    lib.close()


@pytest.mark.parametrize("case", G.fullsize_cases(), ids=lambda c: c["name"])
def test_gpu_reproduces_baseline_size_golden(case):
    """BASELINE-size bit parity (workloads S1 / S2, CORE protocol parameters): the code paths that only run at scale (fast RS-encode
    tiles, flat compress layers above 2^16, zerocheck pieces, 96-job GKR batches) against the oracle's committed proof."""
    from sp1_b200 import Lib
    blob, heights, mains, preps, pv, names, ch = G.fullsize_inputs(case["workload"], case["seed"])
    lib = Lib(0)   # sp1b200_default_core_params
    m = lib.machine_create(blob)
    pc, prep_round = GP.commit_prep(lib, preps)
    st = ch.st.copy()
    words = GP.prove(lib, m, prep_round, mains, heights, names, pv, st)
    G.check_words(case, pc, words, st)
    lib.jagged_round_free(prep_round)
    lib.machine_free(m)
    lib.close()
