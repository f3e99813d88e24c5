"""Times sp1b200_program_vk_tail (the verifying key's initial global cumulative sum of a memory image) at several image sizes, beside the
oracle's OpenMP restatement on every host core, and checks that both give the same tail.

  python tools/setup_bench.py [--log-sizes 16 19 22] [--reps 5] [--out FILE]

GPU: one warm-up call, then the median of --reps calls: wall time around the call (it ends in a stream synchronise) and the device time
of the call's CUDA-event phases ("program_vk_tail" = duplicate check + lift + sum, and the lift and the sum alone).  CPU: one call of
the oracle (oracle/lift.hpp, a restatement of the Rust, not the reference's Rust itself).  Images: unique random word-aligned addresses,
random 64-bit words, no page image.  The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def image(n, seed):
    rng = np.random.default_rng(seed)
    addrs = rng.choice(1 << 45, n, replace=False).astype(np.uint64) << np.uint64(3)
    return addrs, rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-sizes", type=int, nargs="+", default=[16, 19, 22])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from sp1_b200 import Lib
    from tests import lift_oracle_lib as LO
    lib = Lib(0)
    rows = []
    for lg in a.log_sizes:
        n = 1 << lg
        addrs, words = image(n, 4242 + lg)
        tail = lib.program_vk_tail(0x2000, addrs, words)   # warm-up
        wall, total, lift, ssum = [], [], [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            t = lib.program_vk_tail(0x2000, addrs, words)
            wall.append((time.perf_counter() - t0) * 1e3)
            total.append(lib.phase_ms("program_vk_tail")); lift.append(lib.phase_ms("program_vk_tail.lift"))
            ssum.append(lib.phase_ms("program_vk_tail.sum"))
            assert (t == tail).all()
        t0 = time.perf_counter()
        ref = LO.initial_global_cumulative_sum(addrs, words)
        cpu = (time.perf_counter() - t0) * 1e3
        assert (tail[3:17] == ref).all(), f"2^{lg}: the device tail differs from the oracle"
        row = dict(entries=n, gpu_wall_ms=statistics.median(wall), gpu_kernel_ms=statistics.median(total),
                   gpu_lift_ms=statistics.median(lift), gpu_sum_ms=statistics.median(ssum),
                   cpu_restatement_ms=cpu, cpu_threads=os.cpu_count())
        rows.append(row)
        print(json.dumps(row), flush=True)
    lib.close()
    res = dict(card=card(), cpu_label="CPU restatement (oracle/lift.hpp, OpenMP), not the reference's Rust", rows=rows)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
