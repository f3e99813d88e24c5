"""Full-size parity property (BASELINE.json's sha-bench-like shard, workloads S1, S2 = 198.5 M trace cells and S3 = the full 402 M-cell shard, 35 chips up to 2^22 rows, core
protocol parameters: stacking height 2^21, 124 queries, 16 + 5 + 12 proof-of-work bits): the oracle cannot PROVE this size in test
time, but the restated reference verifier (ShardVerifier::verify_shard, run by the oracle from the proof words alone) must accept the
proof the CUDA library produces, end in the prover's challenger state, and reject it after a one-bit change."""
import pytest

from tests import machines as M
from tests import oracle_lib as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("workload", ["S1", "S2", "S3", "S2c", "S3c", "R1"])
def test_full_size_gpu_proof_is_accepted_by_the_restated_reference_verifier(workload):
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import workload as W
    from sp1_b200.lib import HostChallenger
    from tools.device_traces import device_traces

    mach = W.synthetic_machine(workload, seed=42)
    specs, names = mach["specs"], mach["names"]
    heights = [s_.h for s_ in specs]
    pv = M.PV
    d_main, d_prep, prep_rows, prep_cols = device_traces(specs, M.PV0, lambda i: 7000 + i, torch.device("cuda", 0))
    prm = W.params_of(workload)                           # core parameters, or the recursion ones for the compress-shape shard
    lib = Lib(device=0, **prm)
    machine = lib.machine_create(mach["blob"])
    pc, h_prep = lib.jagged_commit_dense(d_prep, prep_rows, prep_cols)
    st0 = HostChallenger().st.copy()
    st = st0.copy()
    words = lib.prove_shard(machine, h_prep, d_main, heights, names, pv, st)
    again = lib.prove_shard(machine, h_prep, d_main, heights, names, pv, st0.copy())
    assert (words == again).all(), "the proof is not deterministic"
    lib.jagged_round_free(h_prep)
    lib.machine_free(machine)
    lib.close()
    del d_main, d_prep
    torch.cuda.empty_cache()

    v = O.Challenger(); v.st[:] = st0
    LS, MLR = prm["log_stacking_height"], prm["max_log_row_count"]
    assert O.verify_shard(mach["blob"], heights, names, LS, MLR, v, pc, words) == 0, "restated reference verifier rejected the GPU proof"
    assert (v.st == st).all(), "verifier and prover end in different challenger states"
    n_sec = int(words[0])
    off = 1 + n_sec + int(words[1]) + int(words[2]) // 2      # a word in the middle of the LogUp-GKR section
    bad = words.copy(); bad[off] ^= 1
    v2 = O.Challenger(); v2.st[:] = st0
    assert O.verify_shard(mach["blob"], heights, names, LS, MLR, v2, pc, bad) != 0
