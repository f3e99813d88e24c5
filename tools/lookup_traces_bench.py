"""Times sp1b200_lookup_traces (a shard's Byte, Program and Range multiplicity traces built on the device from its byte lookups and executed
pcs) on uniform and skewed record streams, and beside it the host-to-device copy of the records and the NumPy restatement of the tables
(tests/lookup_ref.py).  Every device result is checked against the restatement.

  python tools/lookup_traces_bench.py [--log-lookups 22 26] [--log-pcs 22] [--log-instrs 20] [--reps 5] [--out FILE]

GPU: records and outputs in device memory, one warm-up call per stream, then the median of --reps calls of the device time of each
CUDA-event phase: "lookup_traces" (the whole call), ".tables" (zeroing aside, the counting passes) and ".write" (the range check and the
column-major write).  Records per second are (lookup records + pc records) over the whole call.  The bytes floor is what the call must
move at least (the records read once, the 64-bit counters zeroed, read back and the 32-bit words written) over 3.35 TB/s, the HBM3
bandwidth of NVIDIA's H100 SXM data sheet.  The records' host-to-device copy is timed separately from pageable and from pinned memory
with CUDA events.  Host: one run of the NumPy restatement (single-threaded NumPy; a restatement, not the reference's Rust generator).
Streams: "uniform" draws opcode, operands and pcs uniformly; "skewed" sends half the lookups to U8Range(0, 0) and half the pcs to one pc.
The card's name, power limit and maximum SM clock are printed with the numbers."""
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

PHASES = ["lookup_traces", "lookup_traces.tables", "lookup_traces.write"]
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def streams(kind, n_lookups, n_pcs, pc_base, n_instrs, seed):
    from sp1_b200.lib import pack_byte_lookups, pack_pc_counts
    rng = np.random.default_rng(seed)
    op = rng.integers(0, 7, n_lookups)
    bits = rng.integers(0, 17, n_lookups)
    a = np.where(op == 6, rng.integers(0, 1 << 16, n_lookups) & ((1 << bits) - 1), 0)
    b = np.where(op == 6, bits, rng.integers(0, 256, n_lookups))
    c = rng.integers(0, 256, n_lookups)
    pc = np.uint64(pc_base) + np.uint64(4) * rng.integers(0, n_instrs, n_pcs).astype(np.uint64)
    if kind == "skewed":
        hot = rng.random(n_lookups) < 0.5
        op, a, b, c = np.where(hot, 3, op), np.where(hot, 0, a), np.where(hot, 0, b), np.where(hot, 0, c)
        pc = np.where(rng.random(n_pcs) < 0.5, np.uint64(pc_base + 4 * 7), pc)
    return pack_byte_lookups(op, a, b, c, 1), pack_pc_counts(pc, 1)


def copy_ms(recs, reps, pinned):
    import torch
    src = torch.from_numpy(recs.view(np.uint8).reshape(-1))
    if pinned:
        src = src.pin_memory()
    dst = torch.empty_like(src, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dst.copy_(src, non_blocking=pinned)   # warm-up
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0.record(); dst.copy_(src, non_blocking=pinned); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts), dst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-lookups", type=int, nargs="+", default=[22, 26])
    ap.add_argument("--log-pcs", type=int, default=22)
    ap.add_argument("--log-instrs", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from sp1_b200 import Lib
    from tests import lookup_ref as LR
    lib = Lib(0)
    pc_base, n_instrs, n_pcs = 0x20_0000, 1 << a.log_instrs, 1 << a.log_pcs
    h = LR.next_multiple_of_32(n_instrs)
    out = tuple(torch.zeros(s, dtype=torch.int32, device="cuda") for s in ((6, 1 << 16), (1, h), (1, 1 << 17)))
    counters = 6 * (1 << 16) + (1 << 17) + h
    rows = []
    for lg in a.log_lookups:
        for kind in ("uniform", "skewed"):
            n = 1 << lg
            lookups, pcs = streams(kind, n, n_pcs, pc_base, n_instrs, 5000 + lg)
            t0 = time.perf_counter()
            want = LR.main_words(pc_base, n_instrs, lookups, pcs)
            numpy_ms = (time.perf_counter() - t0) * 1e3
            pageable_l, _ = copy_ms(lookups, a.reps, False)
            pageable_p, _ = copy_ms(pcs, a.reps, False)
            pinned_l, d_lookups = copy_ms(lookups, a.reps, True)
            pinned_p, d_pcs = copy_ms(pcs, a.reps, True)
            lib.lookup_traces(pc_base, n_instrs, d_lookups, d_pcs, out=out)   # warm-up
            for o, w in zip(out, want):
                assert (o.cpu().numpy().view(np.uint32) == w).all(), f"2^{lg} {kind}: device tables differ from the restatement"
            wall, ph = [], {p: [] for p in PHASES}
            for _ in range(a.reps):
                t0 = time.perf_counter()
                lib.lookup_traces(pc_base, n_instrs, d_lookups, d_pcs, out=out)
                wall.append((time.perf_counter() - t0) * 1e3)
                for p in PHASES:
                    ph[p].append(lib.phase_ms(p))
            total_ms = statistics.median(ph["lookup_traces"])
            floor_bytes = lookups.nbytes + pcs.nbytes + counters * (8 + 8 + 4)
            row = dict(stream=kind, lookup_records=n, pc_records=n_pcs, instructions=n_instrs, gpu_wall_ms=statistics.median(wall),
                       **{"gpu_" + p.replace("lookup_traces", "total").replace(".", "_") + "_ms": statistics.median(v) for p, v in ph.items()},
                       records_per_s=(n + n_pcs) / (total_ms * 1e-3), floor_bytes=floor_bytes,
                       bytes_floor_ms=floor_bytes / HBM_BYTES_PER_S * 1e3,
                       share_of_bytes_floor=floor_bytes / HBM_BYTES_PER_S * 1e3 / total_ms,
                       h2d_pageable_ms=pageable_l + pageable_p, h2d_pinned_ms=pinned_l + pinned_p, host_numpy_restatement_ms=numpy_ms)
            rows.append(row)
            print(json.dumps(row), flush=True)
            del d_lookups, d_pcs
    lib.close()
    res = dict(card=card(), bound="memory: the call does no arithmetic beyond one Montgomery product per counter, so the bytes floor applies",
               host_label="NumPy restatement of the tables (tests/lookup_ref.py), not the reference's Rust", rows=rows)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
