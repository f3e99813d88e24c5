#!/usr/bin/env python3
"""Where the RS-encode time goes, at the S2c main-commit shape (95 columns, 2^21 -> 2^23 rows, blowup 4).

GPU run (default):
  * the card's name, power limit, SM clock and throttle reasons (nvidia-smi, same process as the timings);
  * lib.rs_encode timed with CUDA events on the library's stream: best and median of --reps calls after --warmup calls;
  * in a run of its own, torch.profiler (CUDA activities): time per launch of every kernel of the call (step A, step B);
  * algorithmic bytes (20 B per padded cell: 4 read + 16 written) per second, Montgomery products per second, and the two floors:
    HBM (algorithmic bytes at the data-sheet 3.35 TB/s) and multiplier pipe (products x slots per product over 64 IMAD slots per SM
    per clock at the card's maximum SM clock).
Static count (--sass OBJ, no GPU): instructions per output cell of both kernels from the sm_90a SASS (tools/sass_dyn.py weighting,
loop trip counts of the S2c shape), split into multiplier-pipe classes (IMAD*, IMAD.HI, IMAD.WIDE and their slots), memory
(LDG/STG/LDS/STS/LDL/STL), SHFL and the rest (ALU, control).  Both sides of a uniform branch are counted.
usage: rs_profile.py [--ncols 95] [--log-h 21] [--log-blowup 2] [--reps 10] [--warmup 3] [--json OUT]
       rs_profile.py --sass sp1_b200/csrc/build/ntt.o"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# multiplier-pipe slots per instruction class (tools/pipe_mix.cu; the same weights as tests/test_codegen.py)
SLOTS = {"IMAD.HI": 2.0, "IMAD.WIDE": 2.65}
HBM_GBS = 3350.0            # H100 SXM data sheet
# Montgomery products per output cell, counted from the kernels' structure (L1 = 10, L2 = 11, 4 cosets): step A per thread and coset
# 3 radix-8 passes x 12 + 8 coset-twist products on 3 of 4 cosets, over 8 cells; step B per thread 3 x 12 + 2 (radix-4 pass) + 8
# inter-step twist + 7 twist-chain products, over 8 cells
PRODUCTS_PER_CELL = {"step_a": (36 + 8 * 3 / 4) / 8, "step_b": (36 + 2 + 8 + 7) / 8}
SLOTS_PER_PRODUCT = 2.65 + 1 + 2.0      # IMAD.WIDE + IMAD + IMAD.HI


def card_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks_throttle_reasons.active"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        return {"nvidia_smi": r.stderr.strip()}
    f = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return dict(zip(["name", "power_limit", "max_sm_clock", "sm_clock", "throttle_reasons"], f))


def sass_count(obj):
    """{kernel: {class: instructions per output cell}} for the two fast kernels"""
    kernels = {"step_a": ("rs_step_a_fastILi10ELi2", "4", 32), "step_b": ("rs_step_b_2048", "", 8)}   # (name, loop trips, cells per thread)
    out = {}
    for key, (frag, trips, cells) in kernels.items():
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_dyn.py"), obj, frag, trips], capture_output=True, text=True)
        if r.returncode != 0:
            sys.exit(r.stderr)
        hist = {}
        for line in r.stdout.splitlines():
            p = line.split()
            if len(p) == 2 and re.fullmatch(r"[\d.]+", p[1]):
                hist[p[0]] = float(p[1])
        imad = sum(v for k, v in hist.items() if k.startswith("IMAD") and k not in SLOTS)
        mem = {k: hist.get(k, 0.0) for k in ("LDG", "STG", "LDS", "STS", "LDL", "STL")}
        shfl = hist.get("SHFL", 0.0)
        total = sum(hist.values())
        slots = imad + sum(w * hist.get(k, 0.0) for k, w in SLOTS.items())
        row = {"IMAD*": imad, "IMAD.HI": hist.get("IMAD.HI", 0.0), "IMAD.WIDE": hist.get("IMAD.WIDE", 0.0), "mul_slots": slots}
        row.update(mem)
        row["SHFL"] = shfl
        row["other"] = total - imad - row["IMAD.HI"] - row["IMAD.WIDE"] - sum(mem.values()) - shfl
        row["total"] = total
        out[key] = {k: round(v / cells, 2) for k, v in row.items()}
    return out


def gpu_profile(a):
    import numpy as np
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import workload as W

    assert torch.cuda.is_available(), "rs_profile needs a GPU (use --sass for the static count)"
    dev = torch.device("cuda:0")
    info = card_info()
    props = torch.cuda.get_device_properties(0)
    lib = Lib(device=0)
    n, lb = a.ncols, a.log_blowup
    g = torch.Generator(device=dev)
    g.manual_seed(7)
    msg = torch.randint(0, W.P, (n, 1 << a.log_h), dtype=torch.int32, device=dev, generator=g)
    cw = torch.empty((n, 1 << (a.log_h + lb)), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    stream = torch.cuda.ExternalStream(lib.stream())

    def call():
        lib.rs_encode(msg, cw, n, a.log_h, lb)

    for _ in range(a.warmup):
        call()
    lib.sync()
    times = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        call()
        e1.record(stream)
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    # checksum of the codeword so that two builds can be compared on the same seeded input
    digest = int(torch.sum(cw.to(torch.int64) * torch.arange(1, cw.shape[1] + 1, device=dev, dtype=torch.int64).remainder_(65521)).item())

    from torch.profiler import ProfilerActivity, profile
    kern = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            call()
        lib.sync()
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and "rs_" in ev.name:
            name = "step_a" if "rs_step_a" in ev.name else "step_b" if "rs_step_b" in ev.name else ev.name
            kern.setdefault(name, []).append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
    lib.close()

    cells_in, cells_out = n << a.log_h, n << (a.log_h + lb)
    best, med = min(times), statistics.median(times)
    algo_bytes = 20.0 * cells_in * (1 << lb) / 4        # 4 B read per input cell + 4 B written per output cell
    products = sum(PRODUCTS_PER_CELL.values()) * cells_out
    try:
        clk_ghz = float(info.get("max_sm_clock", "").split()[0]) / 1000.0
    except (ValueError, IndexError):
        clk_ghz = props.clock_rate / 1e6 if hasattr(props, "clock_rate") else float("nan")
    mul_floor_ms = products * SLOTS_PER_PRODUCT / (props.multi_processor_count * 64 * clk_ghz * 1e9) * 1e3
    hbm_floor_ms = algo_bytes / (HBM_GBS * 1e9) * 1e3
    steps = {}
    for k, v in sorted(kern.items()):
        per = [x / 1e3 for x in v]                       # us -> ms per launch
        steps[k] = {"launches_per_call": len(per) / a.reps, "ms_per_call": sum(per) / a.reps, "ms_launch_median": statistics.median(per)}
    res = {
        "card": info, "sms": props.multi_processor_count,
        "shape": f"{n} cols 2^{a.log_h} -> 2^{a.log_h + lb}",
        "rs_encode_ms": {"best": best, "median": med, "all": times},
        "kernels_profiler": steps,
        "algorithmic_GBps": algo_bytes / (med * 1e-3) / 1e9,
        "products_per_s": products / (med * 1e-3),
        "floors_ms": {"hbm": hbm_floor_ms, "multiplier": mul_floor_ms},
        "codeword_digest": digest,
    }
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--ncols", type=int, default=95)
    ap.add_argument("--log-h", type=int, default=21)
    ap.add_argument("--log-blowup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sass", metavar="OBJ", default=None, help="static SASS count of the kernels in OBJ (no GPU)")
    ap.add_argument("--json", metavar="OUT", default=None)
    a = ap.parse_args()
    if a.sass:
        res = {"sass_per_output_cell": sass_count(a.sass)}
        for k, row in res["sass_per_output_cell"].items():
            print(k, " ".join(f"{c}={v}" for c, v in row.items()))
    else:
        assert a.reps >= 10, "best and median of at least 10 calls"
        res = gpu_profile(a)
        print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
