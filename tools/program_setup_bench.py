"""Times sp1b200_program_setup (a core program's preprocessed tables generated and committed on the device, plus its verifying key) at
several program sizes with one memory image, and beside it the host path it replaces: the NumPy restatement of the tables
(tests/program_ref.py) and the host-to-device copy of their words.  Every device result is checked against the restatement.

  python tools/program_setup_bench.py [--log-instrs 12 16 20] [--log-image 20] [--reps 5] [--out FILE]

GPU: one warm-up call per size, then the median of --reps calls of the device time of each CUDA-event phase: "program_setup" (the whole
call), ".tables" (instruction upload, the three tables, the validation read-back), ".vk_tail" (sp1b200_program_vk_tail of the image) and
".commit" (sp1b200_jagged_commit of the tables), and the wall time around the call.  Host: one run of the NumPy restatement of the three
tables (single-threaded NumPy; a restatement, not the reference's Rust generator) and the median of --reps pinned host-to-device copies of
the same words, timed with CUDA events.  The card's name, power limit and maximum SM clock are printed with the numbers."""
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

PHASES = ["program_setup", "program_setup.tables", "program_setup.vk_tail", "program_setup.commit"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def program(n, seed):
    from sp1_b200.lib import MAX_OPCODE, pack_instructions
    rng = np.random.default_rng(seed)
    u64 = lambda: rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
    return pack_instructions(rng.integers(0, MAX_OPCODE + 1, n), rng.integers(0, 32, n), u64(), u64(), rng.integers(0, 2, n),
                             rng.integers(0, 2, n))


def image(n, seed):
    rng = np.random.default_rng(seed)
    return rng.choice(1 << 45, n, replace=False).astype(np.uint64) << np.uint64(3), rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)


def h2d_ms(words, reps):
    import torch
    src = torch.from_numpy(words.view(np.int32)).pin_memory()
    dst = torch.empty_like(src, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dst.copy_(src, non_blocking=True)   # warm-up
    ts = []
    for _ in range(reps):
        e0.record(); dst.copy_(src, non_blocking=True); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-instrs", type=int, nargs="+", default=[12, 16, 20])
    ap.add_argument("--log-image", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from sp1_b200 import Lib
    from tests import program_ref as PR
    lib = Lib(0)
    addrs, words = image(1 << a.log_image, 77)
    pc_base, pc_start = 0x20_0000, 0x20_0000
    rows = []
    for lg in a.log_instrs:
        n = 1 << lg
        instrs = program(n, 4000 + lg)
        t0 = time.perf_counter()
        dense, shapes = PR.dense(pc_base, instrs)
        numpy_ms = (time.perf_counter() - t0) * 1e3
        got, _ = lib.program_preprocessed_traces(pc_base, instrs)
        assert (got == dense).all(), f"2^{lg}: device tables differ from the restatement"
        want_commit, h = lib.jagged_commit_dense(dense, [s[0] for s in shapes], [s[1] for s in shapes])
        lib.jagged_round_free(h)
        key = lib.program_setup(pc_base, instrs, pc_start, addrs, words)   # warm-up
        lib.jagged_round_free(key["round"])
        assert (key["prep_commit"] == want_commit).all(), f"2^{lg}: commitment differs from the commitment of the restated tables"
        wall, ph = [], {p: [] for p in PHASES}
        for _ in range(a.reps):
            t0 = time.perf_counter()
            k = lib.program_setup(pc_base, instrs, pc_start, addrs, words)
            wall.append((time.perf_counter() - t0) * 1e3)
            lib.jagged_round_free(k["round"])
            for p in PHASES:
                ph[p].append(lib.phase_ms(p))
            assert (k["vk_digest"] == key["vk_digest"]).all()
        row = dict(instructions=n, image_entries=1 << a.log_image, dense_words=int(dense.size), gpu_wall_ms=statistics.median(wall),
                   **{"gpu_" + p.replace("program_setup", "total").replace(".", "_") + "_ms": statistics.median(v) for p, v in ph.items()},
                   host_numpy_tables_ms=numpy_ms, host_h2d_tables_ms=h2d_ms(dense, a.reps))
        rows.append(row)
        print(json.dumps(row), flush=True)
    lib.close()
    res = dict(card=card(), host_label="NumPy restatement of the tables (tests/program_ref.py), not the reference's Rust", rows=rows)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
