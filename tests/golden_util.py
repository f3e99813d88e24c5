"""Shared helpers for the committed golden fixtures (tests/golden/shard_proofs.json, made by tools/gen_golden_proofs.py)."""
import hashlib
import json
import os

import numpy as np

from tests import machines as M
from tests import oracle_lib as O

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shard_proofs.json")


def cases():
    return json.load(open(PATH))["cases"]


def inputs_of(case):
    """re-create the seeded inputs of a golden case (same generator the fixture script used)
    -> (blob, heights, mains, preps, pv, names, challenger)"""
    return M.shard_inputs(case["spec"], case["seed"])


def check_words(case, prep_commit, words, final_state):
    assert [int(x) for x in prep_commit] == case["prep_commit"], "preprocessed commitment differs from the golden fixture"
    assert int(words.size) == case["n_words"]
    n_sec = int(words[0])
    assert [int(x) for x in words[1:1 + n_sec]] == case["section_lengths"]
    assert [int(x) for x in words[1 + n_sec:1 + n_sec + 8]] == case["main_commit"], "main commitment differs from the golden fixture"
    off = 1 + n_sec
    for ln, sec in zip(case["section_lengths"], case["sections"]):
        got = words[off:off + ln]
        assert [int(x) for x in got[:8]] == sec["first"] and [int(x) for x in got[-8:]] == sec["last"]
        off += ln
    assert hashlib.sha256(words.astype("<u4").tobytes()).hexdigest() == case["sha256"], "proof words differ from the golden fixture"
    assert [int(x) for x in final_state] == case["final_challenger"], "final challenger state differs from the golden fixture"


# ---- BASELINE-size goldens (tests/golden/shard_proofs_fullsize.json): workloads S1 / S2 with the core protocol parameters ------------
FULL_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shard_proofs_fullsize.json")


def fullsize_cases():
    return json.load(open(FULL_PATH))["cases"] if os.path.exists(FULL_PATH) else []


def fullsize_inputs(workload, seed):
    """the seeded full-size inputs of a golden case: the bench machine of `workload` (sp1_b200.workload.synthetic_machine) with numpy
    traces (so that the CPU generator and the GPU test see the same words).  -> (blob, heights, mains, preps, pv, names, challenger)"""
    rng = np.random.default_rng(seed)
    inp = M.workload_machine(workload, rng)
    ch = O.Challenger()
    ch.observe(O.rand_field(rng, 9))
    return inp + (ch,)
