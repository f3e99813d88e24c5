#!/usr/bin/env python
"""Generate tests/golden/shard_proofs.json: small whole-shard proofs produced by the CPU oracle (oracle/liboracle.so) on seeded
synthetic machines.  The reference holds no golden vectors for this path and cannot be built in this image (DESIGN.md section 4),
so these fixtures pin the ORACLE against accidental change (and give the GPU suite a committed, oracle-independent target):
every entry stores the preprocessed commitment, the main commitment, the final challenger state, the section lengths and a
SHA-256 of the proof words; the first and last 8 words of every section are stored in clear for debugging.

  python tools/gen_golden_proofs.py            # rewrites tests/golden/shard_proofs.json
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import golden_util as G  # noqa: E402
from tests import oracle_lib as O  # noqa: E402

CASES = [
    # name, spec [(height, groups, with_prep)], log_stack, max_log_rows, seed, queries, pow, batch_pow, gkr_pow
    ("one_chip_full_height", [(8, 1, False)], 3, 3, 101, 4, 3, 2, 2),
    ("odd_heights_empty_chip_prep", [(5, 1, False), (0, 2, False), (6, 1, True)], 3, 3, 102, 4, 3, 2, 2),
    ("four_chips", [(32, 2, True), (96, 1, False), (128, 1, False), (0, 1, True)], 5, 7, 103, 8, 4, 2, 3),
    ("medium", [(4096, 2, True), (1024 + 32, 3, False), (0, 1, False), (8192, 1, True), (2048, 4, False)], 12, 13, 104, 16, 8, 5, 6),
]


def prove_case(spec, log_stack, mlr, seed, nq, pw, bpw, gpw):
    """the oracle's proof of a case's seeded inputs (golden_util.inputs_of) -> (blob, heights, mains, preps, names, prep commitment,
    words, final challenger)"""
    blob, heights, mains, preps, pv, names, ch = G.inputs_of({"spec": spec, "seed": seed})
    pc, words = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, ch, num_queries=nq, pow_bits=pw,
                                     batch_pow_bits=bpw, gkr_pow_bits=gpw)
    return blob, heights, mains, preps, names, pc, words, ch


def run_case(name, spec, log_stack, mlr, seed, nq, pw, bpw, gpw):
    *_, pc, words, ch = prove_case(spec, log_stack, mlr, seed, nq, pw, bpw, gpw)
    d = {"name": name, "spec": [list(s) for s in spec], "log_stacking_height": log_stack, "max_log_row_count": mlr, "seed": seed,
         "num_queries": nq, "pow_bits": pw, "batch_pow_bits": bpw, "gkr_pow_bits": gpw}
    d.update(summarize(name, pc, words, ch, {}))   # the case's parameters first, as the fixture lists them
    return d


def summarize(name, pc, words, ch, extra):
    n_sec = int(words[0])
    lens = [int(x) for x in words[1:1 + n_sec]]
    off = 1 + n_sec
    heads = []
    for ln in lens:
        sec = words[off:off + ln]
        heads.append({"first": [int(x) for x in sec[:8]], "last": [int(x) for x in sec[-8:]]})
        off += ln
    d = {"name": name, "prep_commit": [int(x) for x in pc], "main_commit": [int(x) for x in words[1 + n_sec:1 + n_sec + 8]],
         "final_challenger": [int(x) for x in ch.st], "section_lengths": lens, "n_words": int(words.size),
         "sha256": hashlib.sha256(words.astype("<u4").tobytes()).hexdigest(), "sections": heads}
    d.update(extra)
    return d


def full_size(workloads):
    """BASELINE-size goldens: the bench workloads with the CORE protocol parameters (2^21 stacking, 2^22 rows, 124 queries, 16+5+12 PoW
    bits), proven once by the oracle (minutes on 8 cores) -> tests/golden/shard_proofs_fullsize.json.  Also stores the three grinding
    witnesses so that the replay-mode test can reproduce the same proof with grind_mode = 1."""
    import time
    path = G.FULL_PATH
    old = {c["name"]: c for c in (json.load(open(path))["cases"] if os.path.exists(path) else [])}
    for wl in workloads:
        seed = 9000 + sum(ord(c) for c in wl)
        blob, heights, mains, preps, pv, names, ch = G.fullsize_inputs(wl, seed)
        t0 = time.time()
        pc, words = O.prove_shard_verify(blob, heights, mains, preps, names, pv, 21, 22, ch)
        print(f"{wl}: oracle proved + verified in {time.time() - t0:.0f}s, {words.size} words", flush=True)
        old[wl] = summarize(wl, pc, words, ch, {"workload": wl, "seed": seed, "log_stacking_height": 21, "max_log_row_count": 22,
                                                "num_queries": 124, "pow_bits": 16, "batch_pow_bits": 5, "gkr_pow_bits": 12})
    out = {"generator": "tools/gen_golden_proofs.py --full (oracle/liboracle.so incl. its restated verifier; minimum-witness grinding)",
           "cases": [old[k] for k in sorted(old)]}
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path, [c["sha256"][:12] for c in out["cases"]])


def bincode_case(name, spec, log_stack, mlr, seed, nq, pw, bpw, gpw):
    """the wire bytes of the same seeded proof: bincode(ShardProof) written by the product's host-only converter"""
    from sp1_b200 import lib as PL
    _, heights, mains, preps, names, _, words, _ = prove_case(spec, log_stack, mlr, seed, nq, pw, bpw, gpw)
    main_w, prep_w = [m.shape[0] for m in mains], [0 if p is None else p.shape[0] for p in preps]
    data = PL.shard_proof_to_bincode(words, names, heights, main_w, prep_w, log_stacking_height=log_stack,
                                     max_log_row_count=mlr, num_queries=nq, pow_bits=pw, batch_pow_bits=bpw, gkr_pow_bits=gpw)
    return {"name": name, "words_sha256": hashlib.sha256(words.astype("<u4").tobytes()).hexdigest(), "bincode_bytes": len(data),
            "bincode_sha256": hashlib.sha256(data).hexdigest(), "head_hex": data[:64].hex()}


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--full":
        return full_size(sys.argv[2:] or ["S1"])
    if len(sys.argv) > 1 and sys.argv[1] == "--bincode":
        out = {"generator": "tools/gen_golden_proofs.py --bincode (the proofs of shard_proofs.json as bincode(ShardProof), csrc/wire.cu)",
               "cases": [bincode_case(*c) for c in CASES]}
        path = os.path.join(ROOT, "tests", "golden", "shard_proofs_bincode.json")
        with open(path, "w") as f:
            json.dump(out, f, indent=1)
        print("wrote", path, [c["bincode_sha256"][:12] for c in out["cases"]])
        return
    out = {"generator": "tools/gen_golden_proofs.py (oracle/liboracle.so; minimum-witness grinding)",
           "format": "proof words = [n_sections][lengths] then main commitment | LogUp-GKR | zerocheck + opened values | evaluation proof | "
                     "public values; u32 little-endian for the hash",
           "cases": [run_case(*c) for c in CASES]}
    path = os.path.join(ROOT, "tests", "golden", "shard_proofs.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path, [c["sha256"][:12] for c in out["cases"]])


if __name__ == "__main__":
    main()
