"""Synthetic workload generator (sp1_b200/workload.py, sp1_b200/synth_air.py): shapes follow the reference's bench generator
(sp1-gpu/crates/jagged_tracegen/src/test_utils.rs:107-221) — heights multiples of 32 up to 2^22, target areas within 1 %, chips
in name order — and the synthetic traces satisfy their own constraints and balanced interactions (checked by the oracle)."""
import numpy as np
import pytest

from sp1_b200 import workload as W
from tests import machines as M
from tests import oracle_lib as O


@pytest.mark.parametrize("name", ["S1", "S2", "S3", "tiny"])
def test_shard_shapes(name):
    prep, main = W.shard_shapes(name)
    area = W.area_of(main)
    target = W.WORKLOADS[name][0]
    assert abs(area - target) <= 0.01 * target
    assert all(r % 32 == 0 and 0 <= r <= 1 << 22 for r, _ in main)
    assert sum(1 for r, _ in main if r == 0) >= 1            # absent chips stay in the list with height 0
    assert [c for _, c in main] == [w for _, w in sorted(W.CORE_CHIPS)]
    assert (W.shard_shapes(name) == (prep, main))            # deterministic for a seed
    assert W.shard_shapes(name, seed=43)[1] != main


def test_synthetic_machine_is_consistent():
    m = W.synthetic_machine("tiny", seed=42)
    assert m["names"] == sorted(m["names"])
    assert len(m["names"]) == len(m["specs"]) == len(m["main_shapes"])
    for sp, (rows, cols) in zip(m["specs"], m["main_shapes"]):
        assert rows == sp.h and cols == 6 * sp.g + (1 if sp.wp else 0) + sp.extra
    assert int(m["blob"][0]) == len(m["specs"])
    small = W.synthetic_machine("S2", seed=42, scale=1 / 64)
    assert W.area_of(small["main_shapes"]) < W.area_of(W.synthetic_machine("S2", seed=42)["main_shapes"]) / 32


@pytest.mark.parametrize("workload", ["tiny", "tinyc", "tinyr"])
def test_synthetic_traces_satisfy_constraints_and_interactions(workload):
    """a scaled-down copy of the bench machine (light and calibrated + precompile table): the oracle proves it and its restated
    verifier accepts (constraints hold on every real row, the LogUp cumulative sum is zero)"""
    blob, heights, mains, preps, pv, names = M.workload_machine(workload, seed=3, scale=1 / 256)
    mlr = max(5, int(np.ceil(np.log2(max(heights + [2])))))
    ch = O.Challenger()
    pc, words = O.prove_shard_verify(blob, heights, mains, preps, names, pv, min(mlr, 6), mlr, ch, num_queries=4, pow_bits=2,
                                     batch_pow_bits=1, gkr_pow_bits=2)
    assert words[0] == 5 and words.size > 100


def test_calibrated_machine_follows_the_chip_statistics():
    """calibrated workloads: every core chip carries the constraint count (clamped to 4..9 per 6-column group) and the number /
    lengths of LogUp messages that tools/chip_stats.py read off the reference's Rust eval functions; the precompile-heavy shard
    puts ~30 % of its area into one 682-column table"""
    st = W.chip_stats()
    assert len(st) >= 30 and all("source" in v or "error" in v for v in st.values())
    light, cal = W.synthetic_machine("S2", seed=42), W.synthetic_machine("S2c", seed=42)
    assert light["main_shapes"] == cal["main_shapes"] and light["names"] == cal["names"]
    assert cal["blob"].size > 2 * light["blob"].size          # more constraints and far more interaction words
    m = W.synthetic_machine("S3c", seed=42)
    k = m["names"].index(W.PRECOMPILE[0])
    rows, cols = m["main_shapes"][k]
    assert cols == 682
    share = rows * cols / W.area_of(m["main_shapes"])
    assert 0.27 < share < 0.33
    assert abs(W.area_of(m["main_shapes"]) / W.WORKLOADS["S3c"][0] - 1) < 0.02


def test_calibration_agrees_with_the_reference_recorded_gkr_workloads():
    """reference-held data: sp1-gpu/crates/logup_gkr/layer_workloads.json lists the (chip, interaction) row counts of 119 real shards;
    its interactions-per-chip distribution (summarised into chip_stats.json by tools/chip_stats.py) brackets what the static reading
    of the Rust eval functions produced, and the calibrated S2c shard is at least as heavy as the heaviest recorded shard"""
    import json
    import os
    st = json.load(open(os.path.join(os.path.dirname(W.__file__), "chip_stats.json")))
    ref = st["reference_gkr_workloads"]
    assert ref and ref["shards"] >= 100
    per_chip = [v["interactions"] for k, v in st["chips"].items() if "interactions" in v and k in dict(W.CORE_CHIPS)]
    med = sorted(per_chip)[len(per_chip) // 2]
    assert ref["interactions_per_chip"]["p10"] <= med <= ref["interactions_per_chip"]["p90"]
    m = W.synthetic_machine("S2c", seed=42)
    heavy = 0
    for name, sp in zip(m["names"], m["specs"]):
        v = st["chips"].get(name, {}).get("values_per_interaction", [4] * 8)
        heavy += sp.h * (2 * len(v[::2]) + (2 if sp.wp else 0))
    assert heavy >= ref["sum_rows_times_interactions"]["max"]
