"""Times sp1b200_verify_compressed on full-size compress-shape (R1) proofs, and the recursion vk tree on the device against the oracle.

    python tools/verify_compressed_bench.py --out DIR [--proofs 8] [--reps 5] [--keys 185862] [--host-threads 0]

proofs  --proofs full-size R1 proofs, each under its own verifying key (distinct vk tails), with valid recursion public values, are
        verified `reps` times after one warm-up, two ways: one sp1b200_verify_compressed call for all of them, and one call per proof.
vk_tree the recursion vk map of --keys seeded digests (the reference's map has 185 862): RecursionVks::from_map with the tree on the
        device (sp1b200_recursion_vks_create, its tree kernels timed with CUDA events), against tests/recursion_ref.py's restatement on the
        host (one call of the oracle's Poseidon2 compression per node, driven from Python).
Reported: medians and minima of the host clock, the card's name, power limit and maximum SM clock.  Writes verify_compressed_bench.json
into --out."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def recursion_pv(rng, vk_root, sp1_vk_digest):
    """187 Montgomery words of RecursionPublicValues that pass verify_compressed's checks: random fields, the given sp1_vk_digest and
    vk_root, is_complete = 1, and digest = the hash of the first 175 words"""
    import numpy as np
    from sp1_b200 import lib as B
    from tests import oracle_lib as O
    pv = O.rand_field(rng, B.PV_MAX_NUM)
    for name, val in (("sp1_vk_digest", sp1_vk_digest), ("vk_root", vk_root), ("is_complete", O.to_monty([1]))):
        at, n = B.RPV[name]
        pv[at:at + n] = val
    at, n = B.RPV["digest"]
    pv[at:at + n] = B.recursion_pv_digest(pv)
    return np.ascontiguousarray(pv, dtype=np.uint32)


def prove_recursion(lib, workload, n, dev, seed=950):
    """n full-size proofs of `workload` under n distinct verifying keys with valid public values -> dict for the verifier"""
    import numpy as np
    import torch
    from sp1_b200 import lib as B
    from sp1_b200 import workload as W
    from tests import oracle_lib as O
    from tools.device_traces import device_traces
    mach = W.synthetic_machine(workload, seed=42)
    specs, names = mach["specs"], mach["names"]
    heights = [s.h for s in specs]
    machine = lib.machine_create(mach["blob"])
    rng = np.random.default_rng(seed)
    pc, prep_round = np.zeros(8, np.uint32), None
    keys, words, finals = [], [], []
    sp1_vk_digest = O.rand_field(rng, 8)
    for i in range(n):
        tail = np.concatenate([O.rand_field(rng, 18), np.zeros(6, np.uint32)])
        keys.append(tail)
    d_main, d_prep, prep_rows, prep_cols = device_traces(specs, 0, lambda i: 7000 + i, dev)
    if d_prep is not None:
        pc, prep_round = lib.jagged_commit_dense(d_prep, prep_rows, prep_cols)
    del d_main, d_prep
    keys = [np.concatenate([pc, t]) for t in keys]
    # the map holds every proof's key and 15 others; its root goes into the public values
    vks = lib.recursion_vks(np.concatenate([np.stack([B.vk_hash(k[:8], k[8:]) for k in keys]), O.rand_field(rng, (15, 8))]))
    root = vks.root()
    for i in range(n):
        pv = recursion_pv(rng, root, sp1_vk_digest)
        d_main, _, _, _ = device_traces(specs, int(O.from_monty(pv[:1])[0]), lambda k: 7000 + k, dev)
        hc = B.HostChallenger(); hc.observe(keys[i])
        st = hc.st.copy()
        words.append(lib.prove_shard(machine, prep_round, d_main, heights, names, pv, st))
        finals.append(st)
        del d_main
        torch.cuda.empty_cache()
    if prep_round is not None:
        lib.jagged_round_free(prep_round)
    proofs = [vks.open(B.vk_hash(k[:8], k[8:])) for k in keys]
    return dict(machine=machine, blob=mach["blob"], keys=keys, heights=heights, names=names, words=words, finals=finals, vks=vks,
                merkle_proofs=proofs, sp1_vk_digest=sp1_vk_digest)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--proofs", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--keys", type=int, default=185862)
    ap.add_argument("--host-threads", type=int, default=0)
    ap.add_argument("--out", required=True, help="directory for verify_compressed_bench.json")
    args = ap.parse_args()
    import numpy as np
    import torch
    from sp1_b200 import Lib
    from sp1_b200 import workload as W
    from sp1_b200.lib import verdict_name
    from tests import oracle_lib as O
    from tests import recursion_ref as RR

    assert torch.cuda.is_available(), "verify_compressed_bench needs a GPU"
    card = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    power = q.stdout.strip() if q.returncode == 0 else "unknown"
    med = lambda xs: sorted(xs)[len(xs) // 2]
    out = {"card": card, "power_limit_and_max_sm_clock": power, "host_cores": os.cpu_count(), "reps": args.reps}

    lib = Lib(device=0, **W.params_of("R1"))
    n = args.proofs
    f = prove_recursion(lib, "R1", n, torch.device("cuda", 0))
    hs = [f["heights"]] * n
    one_call = lambda: lib.verify_compressed(f["machine"], f["vks"], f["keys"], hs, f["names"], f["words"], f["merkle_proofs"],
                                             [f["sp1_vk_digest"]] * n, host_threads=args.host_threads)
    v, sv, fin = one_call()   # warm-up
    assert v == [0] * n, [verdict_name(x) for x in v]
    assert all((fin[k] == f["finals"][k]).all() for k in range(n))
    batch_ms, per_ms = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        assert one_call()[0] == [0] * n
        batch_ms.append((time.perf_counter() - t0) * 1e3)
    for _ in range(args.reps):
        t0 = time.perf_counter()
        for k in range(n):
            assert lib.verify_compressed(f["machine"], f["vks"], f["keys"][k:k + 1], hs[:1], f["names"], f["words"][k:k + 1],
                                         f["merkle_proofs"][k:k + 1], [f["sp1_vk_digest"]], host_threads=args.host_threads)[0] == [0]
        per_ms.append((time.perf_counter() - t0) * 1e3)
    out["proofs"] = {"workload": "R1", "proofs": n, "proof_words": int(f["words"][0].size), "one_call_ms_median": med(batch_ms),
                     "one_call_ms_min": min(batch_ms), "per_proof_calls_ms_median": med(per_ms), "per_proof_calls_ms_min": min(per_ms),
                     "one_call_host_ms": lib.phase_ms("verify_compressed.host"), "one_call_kernel_ms": lib.phase_ms("verify_compressed.kernels")}
    out["proofs"]["speedup_median"] = out["proofs"]["per_proof_calls_ms_median"] / out["proofs"]["one_call_ms_median"]
    print(json.dumps(out["proofs"]), flush=True)
    f["vks"].close()
    lib.machine_free(f["machine"])

    rng = np.random.default_rng(77)
    digests = O.rand_field(rng, (args.keys, 8))
    lib.recursion_vks(digests).close()   # warm-up
    gpu_ms, tree_ms = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        vks = lib.recursion_vks(digests)
        gpu_ms.append((time.perf_counter() - t0) * 1e3)
        tree_ms.append(lib.phase_ms("recursion_vks.tree"))
        root = vks.root()
        vks.close()
    t0 = time.perf_counter()
    ref = RR.VkMap(digests)
    oracle_ms = (time.perf_counter() - t0) * 1e3
    assert (ref.root == root).all()
    out["vk_tree"] = {"keys": args.keys, "create_ms_median": med(gpu_ms), "create_ms_min": min(gpu_ms), "tree_kernels_ms_median": med(tree_ms),
                      "oracle_restatement_host_ms": oracle_ms}
    print(json.dumps(out["vk_tree"]), flush=True)
    lib.close()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "verify_compressed_bench.json"), "w") as fh:
        json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
