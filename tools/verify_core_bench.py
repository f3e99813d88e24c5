"""Times sp1b200_verify_core_proof on full-size GPU core proofs against N sequential sp1b200_verify_shard calls and the oracle.

    python tools/verify_core_bench.py --out DIR [--workloads S2c R1] [--shards 8] [--reps 5] [--host-threads 0]

Per workload: N full-size shards (S2c at the core parameters, R1 at the recursion ones) are proved on the device with a valid
public-value chain (tests/core_chain.py) under one verifying key, then verified `reps` times after one warm-up call, three ways:
  core      one sp1b200_verify_core_proof call (host phases on --host-threads threads, 0 = all cores; one launch per kernel)
  per_shard N sp1b200_verify_shard calls, one after the other, each from the transcript that observed the key
  oracle    the oracle's restated verifier, orc_verify_shard on every shard (one pass; --no-oracle skips it)
Reported: the medians and minima of the host clock around each way, the core call's host / kernel split (phase_ms), the card's name,
power limit and maximum SM clock, and the host's core count.  Writes verify_core_bench.json into --out."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def prove_chain(lib, workload, n, dev, seed=900):
    """n full-size shards of `workload` with the public values of a valid core proof -> dict for the verifiers"""
    import numpy as np
    import torch
    from sp1_b200 import synth_air as SA
    from sp1_b200 import workload as W
    from sp1_b200.lib import HostChallenger
    from tests import core_chain as CC
    mach = W.synthetic_machine(workload, seed=42)
    specs, names = mach["specs"], mach["names"]
    heights = [s.h for s in specs]
    machine = lib.machine_create(mach["blob"])
    pvs, tail = CC.chain(n, seed)
    tail = SA.to_monty(np.array(tail))
    prep_round, pc = None, np.zeros(8, np.uint32)
    words, finals = [], []
    for s, pv in enumerate(pvs):
        mains, preps = [], []
        for i, sp in enumerate(specs):   # the same seeds for every shard: identical preprocessed tables, each shard's own pv0
            m_, p_ = SA.synth_trace_cuda(sp.h, sp.g, sp.wp, CC.pv0_of(pv), 7000 + i, dev, extra_cols=sp.extra, extra_prep=sp.extra_prep)
            mains.append(m_)
            if sp.wp:
                preps.append(p_)
        d_main = torch.cat(mains).contiguous()
        del mains
        if prep_round is None and preps:
            d_prep = torch.cat(preps).contiguous()
            pc, prep_round = lib.jagged_commit_dense(d_prep, [s_.h for s_ in specs if s_.wp], [1 + s_.extra_prep for s_ in specs if s_.wp])
            del d_prep
        del preps
        hc = HostChallenger(); hc.observe(pc); hc.observe(tail)
        st = hc.st.copy()
        words.append(lib.prove_shard(machine, prep_round, d_main, heights, names, SA.to_monty(np.array(pv)), st))
        finals.append(st)
        del d_main
        torch.cuda.empty_cache()
    if prep_round is not None:
        lib.jagged_round_free(prep_round)
    hc = HostChallenger(); hc.observe(pc); hc.observe(tail)
    return dict(machine=machine, blob=mach["blob"], pc=pc, has_prep=any(s.wp for s in specs), tail=tail, heights=heights,
                names=names, words=words, finals=finals, start=hc.st.copy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["S2c", "R1"])
    ap.add_argument("--shards", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-threads", type=int, default=0)
    ap.add_argument("--no-oracle", action="store_true", help="skip the oracle's CPU verification")
    ap.add_argument("--out", required=True, help="directory for verify_core_bench.json")
    args = ap.parse_args()
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import workload as W
    from sp1_b200.lib import verdict_name
    from tests import oracle_lib as O

    assert torch.cuda.is_available(), "verify_core_bench needs a GPU"
    card = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    power = q.stdout.strip() if q.returncode == 0 else "unknown"
    med = lambda xs: sorted(xs)[len(xs) // 2]
    rows = []
    for wl in args.workloads:
        lib = Lib(device=0, **W.params_of(wl))
        prm = lib.params
        n = args.shards
        f = prove_chain(lib, wl, n, torch.device("cuda", 0))
        core = lambda: lib.verify_core_proof(f["machine"], f["pc"], f["tail"], [f["heights"]] * n, f["names"], f["words"],
                                             host_threads=args.host_threads)
        v, s, sv, fin = core()   # warm-up
        assert v == 0, (verdict_name(v), s, verdict_name(sv))
        assert all((fin[k] == f["finals"][k]).all() for k in range(n))
        core_ms, core_host, core_kern = [], [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            v, _, _, _ = core()
            core_ms.append((time.perf_counter() - t0) * 1e3)
            core_host.append(lib.phase_ms("verify_core.host"))
            core_kern.append(lib.phase_ms("verify_core.kernels"))
            assert v == 0
        pc_arg = f["pc"] if f["has_prep"] else None
        for w in f["words"][:1]:   # warm-up
            assert lib.verify_shard(f["machine"], pc_arg, f["heights"], f["names"], w, f["start"])[0] == 0
        seq_ms, seq_kern = [], []
        for _ in range(args.reps):
            t0, kern = time.perf_counter(), 0.0
            for w in f["words"]:
                assert lib.verify_shard(f["machine"], pc_arg, f["heights"], f["names"], w, f["start"])[0] == 0
                kern += lib.phase_ms("verify.kernels")
            seq_ms.append((time.perf_counter() - t0) * 1e3)
            seq_kern.append(kern)
        row = {"workload": wl, "shards": n, "card": card, "power_limit_and_max_sm_clock": power, "host_cores": os.cpu_count(),
               "host_threads": args.host_threads or os.cpu_count(), "proof_words_per_shard": int(f["words"][0].size),
               "num_queries": prm["num_queries"], "reps": args.reps,
               "core_ms_median": med(core_ms), "core_ms_min": min(core_ms), "core_host_ms_median": med(core_host),
               "core_kernel_ms_median": med(core_kern), "core_merkle_ms": lib.phase_ms("verify_core.merkle"),
               "core_fold_ms": lib.phase_ms("verify_core.fold"), "core_jagged_eval_ms": lib.phase_ms("verify_core.jagged_eval"),
               "per_shard_ms_median": med(seq_ms), "per_shard_ms_min": min(seq_ms), "per_shard_kernel_ms_median": med(seq_kern)}
        row["speedup_median"] = row["per_shard_ms_median"] / row["core_ms_median"]
        if not args.no_oracle:
            t0 = time.perf_counter()
            for w in f["words"]:
                o = O.Challenger(); o.st[:] = f["start"]
                r = O.verify_shard(f["blob"], f["heights"], f["names"], prm["log_stacking_height"], prm["max_log_row_count"], o, pc_arg, w,
                                   log_blowup=prm["log_blowup"], num_queries=prm["num_queries"], pow_bits=prm["pow_bits"],
                                   batch_pow_bits=prm["batch_pow_bits"], gkr_pow_bits=prm["gkr_pow_bits"])
                assert r == 0
            row["oracle_cpu_ms"] = (time.perf_counter() - t0) * 1e3
        print(json.dumps(row), flush=True)
        rows.append(row)
        lib.machine_free(f["machine"])
        lib.close()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "verify_core_bench.json"), "w") as fh:
        json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
