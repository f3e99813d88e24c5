"""Times the two shard checks (sp1b200_debug_constraints / sp1b200_debug_interactions) on full-size shards built on the device.

    python tools/debug_bench.py --out DIR [--workloads S2c S3c] [--reps 3]

Per workload: CUDA-event time of each check after one warm-up call, the algorithmic bytes (4 B per trace cell read; the interaction
check adds the 24 B per (row, interaction) pair of its sort buffers, written and read once by each pass), the growth of device memory
in use over the first call on a fresh context (the context's pool keeps what it allocated, so this is the call's peak), and the card's
name and power limit read in the same run.  Writes debug_bench.json into --out."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["S2c", "S3c"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", required=True, help="directory for debug_bench.json")
    args = ap.parse_args()
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import workload as W
    from tests import machines as M
    from tools.device_traces import device_traces

    assert torch.cuda.is_available(), "debug_bench needs a GPU"
    card = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    power = q.stdout.strip() if q.returncode == 0 else "unknown"
    pv = M.PV
    results = []
    for wl in args.workloads:
        m = W.synthetic_machine(wl, seed=42)
        heights = [sp.h for sp in m["specs"]]
        dense, d_prep, prep_rows, prep_cols = device_traces(m["specs"], M.PV0, lambda i: 700 + i, 0)
        lib = Lib(0, **W.params_of(wl))
        mach = lib.machine_create(m["blob"])
        pr = lib.jagged_commit_dense(d_prep, prep_rows, prep_cols)[1] if d_prep is not None else None
        cells = int(dense.numel()) + (int(d_prep.numel()) if d_prep is not None else 0)
        pairs = sum(int(h) * int(n) for h, n in zip(heights, m["interactions"]))
        row = {"workload": wl, "card": card, "power_limit_and_max_sm_clock": power, "trace_cells": cells, "interaction_pairs": pairs}
        for name, call in (("constraints", lambda: lib.debug_constraints_words(mach, pr, dense, heights, pv)),
                           ("interactions", lambda: lib.debug_interactions_words(mach, pr, dense, heights))):
            torch.cuda.synchronize()
            free0, total = torch.cuda.mem_get_info(0)
            words = call()
            torch.cuda.synchronize()
            free1, _ = torch.cuda.mem_get_info(0)
            times = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); call(); e1.record(); torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            alg = 4 * cells + (24 * 2 * pairs if name == "interactions" else 0)
            row[name] = {"ms": sorted(times), "report_words": int(words.size), "clean": words.tolist() in ([0], [0, 0, 0]),
                         "algorithmic_bytes": alg, "GB_per_s": alg / (min(times) * 1e6), "pool_growth_bytes": int(free0 - free1)}
        results.append(row)
        print(json.dumps(row), flush=True)
        if pr is not None:
            lib.jagged_round_free(pr)
        lib.machine_free(mach)
        lib.close()
        del dense, d_prep
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "debug_bench.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
