#!/usr/bin/env python
"""Per-kernel device times of ONE shard proven alone (torch.profiler, CUDA activities), with the modelled HBM bytes of the
LogUp-GKR and jagged-sumcheck kernels computed from the shard's shapes, and the phase times the library reports for an
unprofiled shard.
usage: python tools/gkr_profile.py [--workload S2c] [--warmup 2] [--out FILE]

The GKR byte model counts the fraction-tree and working arrays only (16 B per extension element, 4 B per base element); trace
reads of the first level and the eq tables (at most 2^21 x 16 B per layer) are left out.  The jagged model counts the trace
reads (4 B per cell of the stacked area) and the extension-field working arrays; the eq tables and L2 re-reads are left out."""
import argparse
import os
import re
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sp1_b200 import workload as W  # noqa: E402


def gkr_bytes_model(heights, inters, mlr):
    """modelled bytes per GKR kernel name for the code as it stands: level 0 = base-field numerators + EF denominators, levels 1
    and 2 written by the first-level pass, two row rounds summed and fixed per pass, the remaining row rounds one per pass"""
    half = lambda x: (x + 1) // 2  # noqa: E731
    lens = [list(heights)]
    for _ in range(1, mlr):
        lens.append([half(x) for x in lens[-1]])
    S = [sum(i * x for i, x in zip(inters, ln)) for ln in lens]
    m = defaultdict(float)
    m["gkr_first_level_kernel"] = 20 * S[0] + 32 * S[1] + (32 * S[2] if mlr > 2 else 0)
    for l in range(2, mlr - 1):
        m["gkr_level_kernel"] += 32 * (S[l] + S[l + 1])
    for l in range(mlr - 1):
        seq = (20 if l == 0 else 32) * S[l]
        rows = [half(x) for x in lens[l]]
        m["gkr_sum2_kernel"] += seq
        r = mlr - 1 - l
        n_fix = 2 if r >= 2 else 1
        for _ in range(n_fix):
            rows = [half(x) for x in rows]
        m["gkr_fix2_kernel"] += seq + 64 * sum(i * x for i, x in zip(inters, rows))
        for _ in range(r - n_fix):
            nxt = [half(x) for x in rows]
            m["gkr_fix_sum_kernel"] += 64 * sum(i * (x + y) for i, x, y in zip(inters, rows, nxt))
            rows = nxt
    return m, S


JK_MAX, JK_LOW = 5, 10  # csrc/jagged.cu


def jagged_layout(rounds_heights, ls, mlr):
    """rounds_heights: per jagged round the column heights -> (area, log_m, K) as sp1b200_jagged_prove sees them: each round
    padded to a multiple of 2^ls with dummy columns (sp1b200_jagged_commit), K = the rounds summed straight from the trace"""
    S, R = 1 << ls, 1 << mlr
    heights = []
    for hs in rounds_heights:
        area = sum(hs)
        added = max(-(-area // S) * S, S) - area
        added_cols = max(-(-added // R), 1)
        heights += list(hs) + [R] * (added_cols - 1) + [added - (added_cols - 1) * R]
    total = sum(heights)
    lm = (total - 1).bit_length()
    k = min(JK_MAX, ls, lm - 1, min(JK_LOW, mlr))
    p = 0
    for h in heights:
        p += h
        if p:
            k = min(k, (p & -p).bit_length() - 1)
    return total, lm, k


def jagged_bytes_model(area, lm, k):
    """modelled bytes per jagged-sumcheck kernel for the code as it stands: rounds 0 .. k-1 each one read of the trace, one pass
    that reads it again and writes the level-k dense and eq arrays, then one fix-and-sum pass per round on EF arrays"""
    m = defaultdict(float)
    N = 1 << lm
    if k:
        m["jagged_round_kernel"] = k * 4 * area
    m["jagged_fold_to_kernel"] = 4 * area + 32 * (N >> k)
    m["hadamard_fold_kernel"] = sum(32 * (N >> r) + 32 * (N >> (r + 1)) for r in range(k, lm))
    return m


def kernel_name(n):
    n = n.replace("(anonymous namespace)::", "")
    n = re.sub(r"^void ", "", n)
    return re.sub(r"\(.*", "", n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="S2c", choices=list(W.WORKLOADS))
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the table to this file")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from sp1_b200 import Lib
    from sp1_b200.lib import HostChallenger
    from sp1_b200 import shards as SH
    from tests import machines as M
    from tools.device_traces import device_traces

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    params = W.params_of(args.workload)
    lib = Lib(device=0, **params)
    mach = W.synthetic_machine(args.workload, seed=42)
    inters = mach["interactions"]
    specs, names = mach["specs"], mach["names"]
    heights = [s_[0] for s_ in specs]
    main_heights = [h for h, cols in mach["main_shapes"] if h for _ in range(cols)]
    prep_heights = [h for h, cols in mach["prep_shapes"] if h for _ in range(cols)]
    d_main, d_prep, prep_rows, prep_cols = device_traces(specs, M.PV0, lambda i: SH.shard_seed(0, 0) + i, dev)
    pv = M.PV
    machine = lib.machine_create(mach["blob"])
    _, h_prep = lib.jagged_commit_dense(d_prep, prep_rows, prep_cols)
    chal0 = HostChallenger().st.copy()

    def step():
        st = chal0.copy()
        lib.prove_shard(machine, h_prep, d_main, heights, names, pv, st)
        lib.sync()

    for _ in range(args.warmup):
        step()
    step()   # unprofiled: the library's own phase timers
    phases = {n: lib.phase_ms(n) for n in ("gkr.circuit", "gkr.rounds", "gkr.openings", "gkr.total", "gkr.host_wait",
                                            "jagged.sumcheck", "jagged.total", "shard.total")}
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    tot, cnt = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        n = kernel_name(e.name)
        tot[n] += e.time_range.elapsed_us() / 1e3
        cnt[n] += 1

    mlr = lib.params["max_log_row_count"]
    model, S = gkr_bytes_model(heights, inters, mlr)
    try:
        card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=5).stdout.strip()
    except Exception:
        card = "unavailable"
    allms = sum(tot.values())
    lines = [f"# {args.workload}, one shard alone, card: {card}; rows x interactions at level 0 = {S[0]:.3e}",
             f"# {sum(cnt.values())} device activities, {allms:.2f} ms of device time (serialised)",
             f"{'kernel':40s} {'launches':>8s} {'ms':>9s} {'share':>6s} {'avg us':>9s}"]
    for n in sorted(tot, key=lambda k: -tot[k]):
        lines.append(f"{n:40s} {cnt[n]:8d} {tot[n]:9.3f} {100 * tot[n] / allms:5.1f}% {1e3 * tot[n] / cnt[n]:9.1f}")
    by_base = defaultdict(float)   # template instances summed: the byte model is per kernel family
    for n, v in tot.items():
        if n.startswith(("gkr_", "table_evals_")):   # table_evals_*: the chip openings (sumcheck.cu)
            by_base[re.sub(r"<.*", "", n)] += v
    lines.append(f"{'GKR kernel family':40s} {'ms':>9s} {'model GB':>9s} {'GB/s':>7s}")
    for n in sorted(by_base, key=lambda k: -by_base[k]):
        gb = model.get(n, 0.0) / 1e9
        lines.append(f"{n:40s} {by_base[n]:9.3f}" + (f" {gb:9.3f} {gb / (by_base[n] / 1e3):7.0f}" if gb else ""))
    gkr_ms = sum(by_base.values())
    gkr_gb = sum(model.get(n, 0.0) for n in by_base) / 1e9
    lines.append(f"GKR kernels (gkr_*, table_evals_*): {gkr_ms:.3f} ms ({100 * gkr_ms / allms:.1f}% of device time), modelled {gkr_gb:.2f} GB")
    area, lm, k = jagged_layout([prep_heights, main_heights], lib.params["log_stacking_height"], mlr)
    jmodel = jagged_bytes_model(area, lm, k)
    jfam = defaultdict(float)   # the jagged sumcheck and the PCS passes over the same trace
    for n, v in tot.items():
        b = re.sub(r"<.*", "", n)
        if b.startswith(("hadamard_", "jagged_")) or b in ("column_evals_kernel", "batch_columns_kernel"):
            jfam[b] += v
    lines.append(f"{'jagged kernel family':40s} {'ms':>9s} {'model GB':>9s} {'GB/s':>7s}   (area {area / 1e6:.1f} M cells, log_m {lm}, "
                 f"K = {k} rounds from the trace)")
    for n in sorted(jfam, key=lambda x: -jfam[x]):
        gb = (jmodel.get(n) or (4 * area if n in ("column_evals_kernel", "batch_columns_kernel") else 0.0)) / 1e9
        lines.append(f"{n:40s} {jfam[n]:9.3f}" + (f" {gb:9.3f} {gb / (jfam[n] / 1e3):7.0f}" if gb else ""))
    hj = [n for n in jfam if n in jmodel]
    lines.append(f"jagged sumcheck kernels: {sum(jfam[n] for n in hj):.3f} ms, modelled {sum(jmodel.values()) / 1e9:.2f} GB "
                 "(column_evals / batch_columns: trace bytes only)")
    # the eq tables every sumcheck and PCS driver shares (sumcheck.cu)
    for n in ("eq_table_kernel", "halve_eq_kernel"):
        lines.append(f"shared {n:33s} {tot.get(n, 0.0):9.3f} ms in {cnt.get(n, 0)} launches")
    lines.append("phases of an unprofiled shard (ms): " + ", ".join(f"{k} {v:.3f}" for k, v in phases.items()))
    lines.append(f"gpu_mem_used_gb {(torch.cuda.mem_get_info(dev)[1] - torch.cuda.mem_get_info(dev)[0]) / 2**30:.1f}")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    lib.jagged_round_free(h_prep)
    lib.machine_free(machine)
    lib.close()


if __name__ == "__main__":
    main()
