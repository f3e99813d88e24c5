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
    import numpy as np
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import synth_air as SA
    from sp1_b200 import workload as W

    assert torch.cuda.is_available(), "debug_bench needs a GPU"
    card = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    power = q.stdout.strip() if q.returncode == 0 else "unknown"
    pv = SA.to_monty(np.array([12345, 5, 6, 7]))
    results = []
    for wl in args.workloads:
        m = W.synthetic_machine(wl, seed=42)
        specs = m["specs"]
        heights = [sp.h for sp in specs]
        parts, preps = [], []
        for i, sp in enumerate(specs):
            a, p = SA.synth_trace_cuda(sp.h, sp.g, sp.wp, 12345, 700 + i, 0, extra_cols=sp.extra, extra_prep=sp.extra_prep)
            parts.append(a); preps.append(p)
        dense = torch.cat(parts).contiguous()
        torch.cuda.synchronize()
        lib = Lib(0, **W.params_of(wl))
        mach = lib.machine_create(m["blob"])
        pts = [p.view(-1, sp.h).cpu().numpy().view(np.uint32) for p, sp in zip(preps, specs) if p is not None]
        pr = lib.jagged_commit(pts)[1] if pts else None
        cells = int(dense.numel()) + sum(int(p.numel()) for p in preps if p is not None)
        pairs = sum(int(h) * int(n) for h, n in zip(heights, _interactions_per_chip(m["blob"])))
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
        del dense, parts, preps
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "debug_bench.json"), "w") as f:
        json.dump(results, f, indent=1)


def _interactions_per_chip(blob):
    b = [int(x) for x in blob]
    p = 1
    for _ in range(b[0]):
        ni, nl, nc, npub, na = b[p + 4:p + 9]
        p += 9 + 2 * ni + 2 * nl + nc + npub + 2 * na
    out = []
    for _ in range(b[0]):
        k = b[p]; out.append(k); p += 1
        for _ in range(k):
            nv = b[p + 2]; p += 3
            for _ in range(nv + 1):
                p += 2 + 3 * b[p]
    return out


if __name__ == "__main__":
    main()
