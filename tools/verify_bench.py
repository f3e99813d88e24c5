"""Times sp1b200_verify_shard on full-size GPU proofs and the oracle's restated verifier (orc_verify_shard) on the same words.

    python tools/verify_bench.py --out DIR [--workloads S2c R1] [--reps 5]

Per workload: the proof is made on the device (S2c at the core parameters, R1 at the recursion ones), then verified `reps` times after
one warm-up call.  Reported per call: the host clock around sp1b200_verify_shard (it ends with a device synchronise), the CUDA-event
time of the verifier's kernels (Merkle openings, query fold chains, jagged column sum) and the rest as host time; the oracle's CPU
time on the same words (one call; it runs on this host's cores, whose count is reported).  The card's name, power limit and maximum
SM clock are read in the same run.  Writes verify_bench.json into --out."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def full_size_proof(lib, workload, dev):
    """prove the full-size synthetic shard `workload` on `lib`'s context (fresh transcript) -> machine handle, commitment, proof"""
    import torch
    from sp1_b200 import workload as W
    from sp1_b200.lib import HostChallenger
    from tests import machines as M
    from tests import oracle_lib as O
    from tools.device_traces import device_traces
    mach = W.synthetic_machine(workload, seed=42)
    specs, names = mach["specs"], mach["names"]
    heights = [s.h for s in specs]
    d_main, d_prep, prep_rows, prep_cols = device_traces(specs, M.PV0, lambda i: 7000 + i, dev)
    machine = lib.machine_create(mach["blob"])
    pc, h_prep = lib.jagged_commit_dense(d_prep, prep_rows, prep_cols)
    st = HostChallenger().st.copy()
    words = lib.prove_shard(machine, h_prep, d_main, heights, names, O.to_monty([M.PV0, 5, 6, 7]), st)
    lib.jagged_round_free(h_prep)
    del d_main, d_prep
    torch.cuda.empty_cache()
    return dict(machine=machine, blob=mach["blob"], pc=pc, heights=heights, names=names, words=words, final=st)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["S2c", "R1"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true", help="skip the oracle's CPU verification")
    ap.add_argument("--out", required=True, help="directory for verify_bench.json")
    args = ap.parse_args()
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import workload as W
    from sp1_b200.lib import HostChallenger, verdict_name
    from tests import oracle_lib as O

    assert torch.cuda.is_available(), "verify_bench needs a GPU"
    card = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    power = q.stdout.strip() if q.returncode == 0 else "unknown"
    rows = []
    for wl in args.workloads:
        lib = Lib(device=0, **W.params_of(wl))
        prm = lib.params   # the defaults, updated with the workload's own
        f = full_size_proof(lib, wl, torch.device("cuda", 0))
        start = HostChallenger().st.copy()
        verdict, st = lib.verify_shard(f["machine"], f["pc"], f["heights"], f["names"], f["words"], start)   # warm-up
        assert verdict == 0, verdict_name(verdict)
        assert (st == f["final"]).all()
        wall, kern = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            verdict, _ = lib.verify_shard(f["machine"], f["pc"], f["heights"], f["names"], f["words"], start)
            wall.append((time.perf_counter() - t0) * 1e3)
            kern.append(lib.phase_ms("verify.kernels"))
            assert verdict == 0
        row = {"workload": wl, "card": card, "power_limit_and_max_sm_clock": power, "host_cores": os.cpu_count(),
               "proof_words": int(f["words"].size), "num_queries": prm["num_queries"], "log_stacking_height": prm["log_stacking_height"],
               "verify_ms_median": sorted(wall)[len(wall) // 2], "verify_ms_min": min(wall),
               "kernel_ms_median": sorted(kern)[len(kern) // 2],
               "merkle_ms": lib.phase_ms("verify.merkle"), "fold_ms": lib.phase_ms("verify.fold"),
               "jagged_eval_ms": lib.phase_ms("verify.jagged_eval")}
        row["host_ms_median"] = row["verify_ms_median"] - row["kernel_ms_median"]
        if not args.no_oracle:
            v = O.Challenger(); v.st[:] = start
            t0 = time.perf_counter()
            r = O.verify_shard(f["blob"], f["heights"], f["names"], prm["log_stacking_height"], prm["max_log_row_count"], v, f["pc"], f["words"],
                               log_blowup=prm["log_blowup"], num_queries=prm["num_queries"], pow_bits=prm["pow_bits"],
                               batch_pow_bits=prm["batch_pow_bits"], gkr_pow_bits=prm["gkr_pow_bits"])
            row["oracle_cpu_ms"] = (time.perf_counter() - t0) * 1e3
            assert r == 0
        print(json.dumps(row), flush=True)
        rows.append(row)
        lib.machine_free(f["machine"])
        lib.close()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "verify_bench.json"), "w") as fh:
        json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
