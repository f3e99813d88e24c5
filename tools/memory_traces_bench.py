"""Times sp1b200_memory_traces (a shard's MemoryGlobalInit / MemoryGlobalFinalize / MemoryLocal traces with their byte lookups and global
interaction events, built on the device from its memory events), and beside it the host-to-device copy of the events and the NumPy
restatement (tests/memory_ref.py).  Device results are checked against the restatement at the sizes the restatement is run.

  python tools/memory_traces_bench.py [--log-events 20 22 24] [--max-log-host 22] [--reps 5] [--out FILE]

Workloads per size n: "global" = n init events and n finalize events (random distinct 48-bit addresses, in random order, address 0
first with previous address 0 for init, a non-zero previous address for finalize); "local" = n local events.  GPU: events and outputs in
device memory, one warm-up call, then the median of --reps calls of the device time of each CUDA-event phase: "memory_traces" (the whole
call), ".sort" (address keys, checks and the radix sort) and ".rows" (the row kernels).  The bytes floor is what the call must move at
least (events read once; trace words, lookup records and global records written once; the sort's traffic not counted) over 3.35 TB/s,
the HBM3 bandwidth of NVIDIA's H100 SXM data sheet.  The events' host-to-device copy is timed from pageable and from pinned memory with
CUDA events.  Host: one run of the NumPy restatement up to 2^max-log-host events (single-threaded NumPy; a restatement, not the
reference's Rust generator).  The card's name, power limit and maximum SM clock are printed with the numbers."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from lookup_traces_bench import HBM_BYTES_PER_S, card, copy_ms   # noqa: E402

PHASES = ["memory_traces", "memory_traces.sort", "memory_traces.rows"]


def global_events(n, rng, previous, with_zero):
    from sp1_b200.lib import pack_memory_events
    addrs = np.unique(rng.integers(previous + 1, 1 << 48, n + n // 8 + 64, dtype=np.uint64))
    addrs = rng.permutation(addrs)[:n]
    values = rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
    if with_zero:
        addrs[0], values[0] = 0, 0
    return pack_memory_events(addrs, values, rng.integers(0, 1 << 48, n, dtype=np.uint64))[rng.permutation(n)]


def local_events(n, rng):
    from sp1_b200.lib import pack_memory_local_events
    u = lambda bits: rng.integers(0, 1 << bits, n, dtype=np.uint64, endpoint=False)
    return pack_memory_local_events(u(48), u(48), u(64), u(48), u(64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-events", type=int, nargs="+", default=[20, 22, 24])
    ap.add_argument("--max-log-host", type=int, default=22)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from sp1_b200 import Lib
    from sp1_b200.lib import BYTE_LOOKUP_DTYPE, GLOBAL_EVENT_DTYPE, MEMORY_EVENT_DTYPE, MEMORY_LOCAL_EVENT_DTYPE
    from tests import memory_ref as MR
    lib = Lib(0)
    rows = []
    for lg in a.log_events:
        n = 1 << lg
        rng = np.random.default_rng(7000 + lg)
        for kind in ("global", "local"):
            empty_g = np.zeros(0, MEMORY_EVENT_DTYPE)
            if kind == "global":
                pf = 1 << 20
                init, fin, local = global_events(n, rng, 0, True), global_events(n, rng, pf, False), np.zeros(0, MEMORY_LOCAL_EVENT_DTYPE)
            else:
                pf = 0
                init, fin, local = empty_g, empty_g, local_events(n, rng)
            events = [x for x in (init, fin, local) if x.size]
            numpy_ms = None
            want = None
            if lg <= a.max_log_host:
                t0 = time.perf_counter()
                want = MR.shard(init, fin, 0, pf, local)
                numpy_ms = (time.perf_counter() - t0) * 1e3
            pageable = sum(copy_ms(e, a.reps, False)[0] for e in events)
            pinned, dev = 0.0, []
            for e in events:
                ms, d = copy_ms(e, a.reps, True)
                pinned += ms
                dev.append(d)
            args = (dev[0], dev[1], 0, pf, None) if kind == "global" else (None, None, 0, 0, dev[0])
            h = [MR.num_rows(x.size) for x in (init, fin, local)]
            n_lk = 12 * (init.size + fin.size) + 10 * local.size
            n_ge = init.size + fin.size + 2 * local.size
            out = (torch.zeros((30, h[0]), dtype=torch.int32, device="cuda"), torch.zeros((30, h[1]), dtype=torch.int32, device="cuda"),
                   torch.zeros((20, h[2]), dtype=torch.int32, device="cuda"),
                   torch.zeros(n_lk * BYTE_LOOKUP_DTYPE.itemsize, dtype=torch.uint8, device="cuda"),
                   torch.zeros(n_ge * GLOBAL_EVENT_DTYPE.itemsize, dtype=torch.uint8, device="cuda"))
            lib.memory_traces(*args, out=out)   # warm-up
            if want is not None:
                for o, t in zip(out[:3], want["traces"]):
                    assert (o.cpu().numpy().view(np.uint32) == MR.main_words(t)).all(), f"2^{lg} {kind}: device trace differs"
                g = out[4].cpu().numpy().view(GLOBAL_EVENT_DTYPE)
                assert (g["message"] == want["globals"][0]).all(), f"2^{lg} {kind}: global events differ"
                lk = out[3].cpu().numpy().view(BYTE_LOOKUP_DTYPE)
                lk = lk[lk["count"] != 0]
                assert all((lk[f].astype(np.int64) == want["lookups"][:, j]).all() for j, f in enumerate(("opcode", "a", "b", "c")))
                del g, lk
            ph = {p: [] for p in PHASES}
            for _ in range(a.reps):
                lib.memory_traces(*args, out=out)
                for p in PHASES:
                    ph[p].append(lib.phase_ms(p))
            total_ms = statistics.median(ph["memory_traces"])
            rows_ms = statistics.median(ph["memory_traces.rows"])
            floor_bytes = sum(e.nbytes for e in events) + sum(o.numel() * o.element_size() for o in out)
            row = dict(workload=kind, events=n, **{"gpu_" + p.replace("memory_traces", "total").replace(".", "_") + "_ms": statistics.median(v)
                                                    for p, v in ph.items()},
                       floor_bytes=floor_bytes, bytes_floor_ms=floor_bytes / HBM_BYTES_PER_S * 1e3,
                       share_of_bytes_floor=floor_bytes / HBM_BYTES_PER_S * 1e3 / total_ms,
                       rows_share_of_bytes_floor=floor_bytes / HBM_BYTES_PER_S * 1e3 / rows_ms,
                       h2d_pageable_ms=pageable, h2d_pinned_ms=pinned, host_numpy_restatement_ms=numpy_ms)
            rows.append(row)
            print(json.dumps(row), flush=True)
            del dev, out
            torch.cuda.empty_cache()
    lib.close()
    res = dict(card=card(), bound="the sort phase against the row phase; the row phase against the bytes floor of the whole call",
               host_label="NumPy restatement of the three chips (tests/memory_ref.py), not the reference's Rust", rows=rows)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
