"""Synthetic core-shard workloads (SURVEY.md §8d, BASELINE.md §2.3).

Mirrors the reference's own bench generator (sp1-gpu/crates/jagged_tracegen/src/test_utils.rs:107-221): chip widths from
the core machine's cost table (crates/core/executor/src/artifacts/rv64im_costs.json), heights random multiples of 32
(crates/hypercube/src/util.rs:57) up to 2^22 filling a target area, values uniform field elements, zero padding.
cycles := cells / 45 for synthetic inputs (BASELINE.md).  Test / bench input generation only: no prover logic here.
"""
import collections

import numpy as np

P = 0x7F000001
# one chip of a synthetic machine: height, 6-column constraint groups, has preprocessed columns, filler main columns, further
# preprocessed columns (synth_air.synth_chip / synth_trace take exactly these)
Spec = collections.namedtuple("Spec", "h g wp extra extra_prep")
CELLS_PER_CYCLE = 45

# main-trace chips of the core cluster and their total column counts (rv64im_costs.json, v6.4.0)
CORE_CHIPS = [
    ("Add", 33), ("Addi", 30), ("Addw", 36), ("Bitwise", 51), ("Branch", 45), ("DivRem", 246), ("Global", 241),
    ("InstructionFetch", 36), ("Jal", 31), ("Jalr", 35), ("LoadByte", 47), ("LoadDouble", 39), ("LoadHalf", 44),
    ("LoadWord", 44), ("LoadX0", 48), ("Lt", 44), ("MemoryBump", 15), ("MemoryGlobalFinalize", 30),
    ("MemoryGlobalInit", 30), ("MemoryLocal", 20), ("Mul", 82), ("ShiftLeft", 65), ("ShiftRight", 69), ("StateBump", 14),
    ("StoreByte", 50), ("StoreDouble", 39), ("StoreHalf", 45), ("StoreWord", 44), ("Sub", 33), ("Subw", 32),
    ("SyscallInstrs", 65), ("UType", 31),
]
# preprocessed-only tables (SURVEY.md §8d): committed once at setup, opened with every shard
PREP_CHIPS = [("Byte", 13, 1 << 16), ("Program", 17, 1 << 19), ("Range", 3, 1 << 16)]

WORKLOADS = {
    # name: (target main area in cells, description)
    "S1": (1 << 25, "fibonacci-like shard, 2^20 cycles (reference DEFAULT_RANDOM_LOG_AREA), C=16"),
    "S2": (190_000_000, "sha-bench-like shard, 2^22 cycles, ~1.9e8 cells, C=91"),
    "S3": (402_653_184, "full shard (ELEMENT_THRESHOLD = 2^28 + 2^27 cells), C=192"),
    "tiny": (1 << 21, "smoke-sized shard"),
    # calibrated variants (suffix c): every chip carries the constraint count and the LogUp interaction count / message lengths that
    # tools/chip_stats.py reads off the reference's Rust eval functions (sp1_b200/chip_stats.json) instead of the light template
    "S1c": (1 << 25, "S1 with calibrated chips (constraints + interactions per chip from chip_stats.json)"),
    "S2c": (190_000_000, "S2 with calibrated chips (constraints + interactions per chip from chip_stats.json)"),
    # precompile-heavy shards (BASELINE config 3, SURVEY 8d S3): 30 % of the area in one 682-column precompile table
    "S3p": (402_653_184, "full shard, 30 % of the area in a 682-column precompile table (keccak-permute-like), light chips"),
    "S3c": (402_653_184, "full shard, 30 % of the area in a 682-column precompile table, calibrated chips"),
    "tinyc": (1 << 21, "smoke-sized shard, calibrated chips + a small precompile table"),
    # compress-shape shard (BASELINE config 5 "core+compress", SURVEY.md 8f.3): the recursion machine's eight chips, most columns
    # preprocessed, ~2^27 cells, RECURSION protocol parameters (crates/verifier/src/compressed/config.rs:1-2, fri_params.rs:20-26)
    "R1": (1 << 27, "compress-shape shard: recursion machine (8 chips, preprocessed-heavy), 2^27 main cells, stacking 2^20, rows <= 2^21"),
    "tinyr": (1 << 20, "smoke-sized compress-shape shard"),
}
# protocol parameters per workload family: core = crates/prover/src/components.rs:16-17 + core_fri_config, recursion =
# RECURSION_LOG_STACKING_HEIGHT / RECURSION_MAX_LOG_ROW_COUNT + recursion_fri_config (same blowup 2 -> 124 queries, 16 PoW bits)
CORE_PARAMS = dict(log_stacking_height=21, max_log_row_count=22)
RECURSION_PARAMS = dict(log_stacking_height=20, max_log_row_count=21)


def params_of(workload):
    return dict(RECURSION_PARAMS if workload in RECURSION_WORKLOADS else CORE_PARAMS)


RECURSION_WORKLOADS = {"R1", "tinyr"}
# compress machine (crates/recursion/machine/src/machine.rs:89-105), in name order: (name, main width, preprocessed width, share of the
# main area).  Widths are APPROXIMATE (the column structs' sizes need rustc): what matters for the prover is the shape - a wide
# Poseidon2 table that dominates the area, narrow ALU / memory tables at full height, most columns preprocessed.
RECURSION_CHIPS = [("BaseAlu", 7, 8, 0.10), ("ExtAlu", 13, 8, 0.16), ("MemoryConst", 7, 4, 0.04), ("MemoryVar", 7, 8, 0.10),
                   ("Poseidon2Wide", 157, 36, 0.50), ("PrefixSumChecks", 19, 8, 0.04), ("PublicValues", 7, 16, 0.0), ("Select", 7, 10, 0.06)]
PRECOMPILE = ("KeccakPermute", 682)       # SURVEY.md 8(d): 682-wide precompile columns
PRECOMPILE_SHARE = {"S3p": 0.30, "S3c": 0.30, "tinyc": 0.30}
CALIBRATED = {"S1c", "S2c", "S3c", "tinyc"}
BASE_OF = {"S1c": "S1", "S2c": "S2", "S3p": "S3", "S3c": "S3", "tinyc": "tiny"}


def shard_shapes(workload, seed=42, max_log_rows=22):
    """-> (prep [(rows, cols)], main [(rows, cols)]) in BTreeMap (name) order, as the reference commits them (core chips only; the
    precompile table of the S3p / S3c workloads is added by synthetic_machine)."""
    area = int(WORKLOADS[workload][0] * (1.0 - PRECOMPILE_SHARE.get(workload, 0.0)))
    rng = np.random.default_rng(seed)
    chips = sorted(CORE_CHIPS)
    weights = rng.dirichlet(np.ones(len(chips)) * 2.0)
    rows = []
    for (name, w), share in zip(chips, weights):
        r = int(share * area / w) // 32 * 32
        rows.append(min(r, 1 << max_log_rows))
    # absent chips of the cluster still appear with height 0 in counts/transcript: drop a few deterministically
    for i in rng.choice(len(chips), size=3, replace=False):
        rows[i] = 0
    # top up the widest-margin chips so that the area lands within 1% of the target
    deficit = area - sum(r * w for r, (_, w) in zip(rows, chips))
    for i in np.argsort([-w for _, w in chips]):
        if deficit <= 0:
            break
        if rows[i] == 0:
            continue
        w = chips[i][1]
        add = min(((1 << max_log_rows) - rows[i]), deficit // w) // 32 * 32
        rows[i] += add
        deficit -= add * w
    main = [(r, w) for r, (_, w) in zip(rows, chips)]
    prep_scale = 1.0 if area >= (1 << 27) else max(area / (1 << 27), 1 / 64)
    prep = [(int(h * prep_scale) // 32 * 32 or 32, w) for _, w, h in sorted(PREP_CHIPS)]
    return prep, main


def area_of(shapes):
    return int(sum(r * c for r, c in shapes))


def random_dense_numpy(shapes, seed):
    """flat uint32 array of all real cells (tables back to back, column-major each), uniform in [0, p)"""
    rng = np.random.default_rng(seed)
    return rng.integers(0, P, size=area_of(shapes), dtype=np.uint32)


def random_dense_cuda(shapes, seed, device):
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    return torch.randint(0, P, (area_of(shapes),), dtype=torch.int32, device=device, generator=g)


_STATS = None


def chip_stats():
    """sp1_b200/chip_stats.json (tools/chip_stats.py): per chip {constraints, interactions, values_per_interaction}"""
    global _STATS
    if _STATS is None:
        import json
        import os
        _STATS = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "chip_stats.json")))["chips"]
    return _STATS


# ---- full-shard synthetic machine (constraints + interactions) for bench.py and the scale tests -------------------------------
def synthetic_machine(workload, seed=42, max_log_rows=22, scale=1.0):
    """-> dict(names, specs [(height, groups, with_prep[, extra_cols])], blob, main_shapes [(rows, cols)], prep_shapes,
    interactions [per chip: number of LogUp interactions])
    chips = the core cluster's chips (CORE_CHIPS widths -> 6-column constraint groups) + the three preprocessed tables (+ the
    precompile table of the S3p / S3c workloads), in name order; heights from shard_shapes (multiples of 32), optionally scaled
    down by `scale` (CPU baseline sample).  Calibrated workloads take each chip's constraint count and interaction message
    lengths from chip_stats.json."""
    from . import synth_air as SA
    if workload in RECURSION_WORKLOADS:
        return _recursion_machine(workload, seed, scale)
    prep, main = shard_shapes(workload, seed=seed, max_log_rows=max_log_rows)
    calibrated = workload in CALIBRATED
    stats = chip_stats() if calibrated else {}
    chips = sorted(CORE_CHIPS)
    entries = []   # (name, groups, with_prep, rows, extra_cols)
    for (name, w), (rows, _) in zip(chips, main):
        entries.append((name, max(1, round(w / 6)), False, rows, 0))
    for (name, w, _), (rows, _) in zip(sorted(PREP_CHIPS), prep):
        entries.append((name, max(1, round(w / 6)), True, rows, 0))
    share = PRECOMPILE_SHARE.get(workload, 0.0)
    if share:
        pname, pw = PRECOMPILE
        rows = int(WORKLOADS[workload][0] * share / pw) // 32 * 32
        entries.append((pname, pw // 6, False, min(rows, 1 << max_log_rows), pw - 6 * (pw // 6)))
    entries.sort(key=lambda e: e[0])
    names, specs, words, iwords = [], [], [], []
    for name, g, wp, rows, extra in entries:
        h = int(rows * scale) // 32 * 32 if rows else 0
        if rows and not h:
            h = 32
        names.append(name); specs.append(Spec(h, g, wp, extra, 0))
        st = stats.get(name) if calibrated else None
        if name == PRECOMPILE[0] and calibrated:
            # a permutation precompile: ~2 constraints per column, a handful of wide memory / syscall interactions
            st = {"constraints": 2 * PRECOMPILE[1], "values_per_interaction": [9] * 50 + [5] * 4}
        if st and "constraints" in st:
            cw, _, _ = SA.synth_chip(g, wp, n_constraints=min(max(st["constraints"], 4 * g), 9 * g), extra_cols=extra)
            v = st["values_per_interaction"]
            iw = SA.synth_interactions_calibrated(g, wp, [max(1, min(x, 12)) for x in v[::2]] or [4])   # half are sends, half receives
        else:
            cw, _, _ = SA.synth_chip(g, wp, extra_cols=extra)
            iw = SA.synth_interactions(g, wp, inter_groups=-(-g // 3))
        words.append(cw)
        iwords.append(iw)
    blob = SA.machine_blob_with_interactions(words, iwords)
    return _machine_dict(names, specs, blob, iwords)


def _machine_dict(names, specs, blob, iwords):
    main_shapes = [(s.h, 6 * s.g + (1 if s.wp else 0) + s.extra) for s in specs]
    prep_shapes = [(s.h, 1 + s.extra_prep) for s in specs if s.wp]
    interactions = [int(iw[0]) if len(iw) else 0 for iw in iwords]   # each chip's interaction section starts with its count
    return dict(names=names, specs=specs, blob=blob, main_shapes=main_shapes, prep_shapes=prep_shapes, interactions=interactions)


def _recursion_machine(workload, seed, scale):
    """compress-shape machine: RECURSION_CHIPS with heights (multiples of 32, <= 2^21) that give each chip its share of the main area"""
    from . import synth_air as SA
    area = WORKLOADS[workload][0]
    rng = np.random.default_rng(seed)
    names, specs, words, iwords = [], [], [], []
    for name, mw, pw, share in sorted(RECURSION_CHIPS):
        g = max(1, (mw - 1) // 6)
        extra = mw - 1 - 6 * g
        rows = 32 if share == 0.0 else min(int(share * area * (0.9 + 0.2 * rng.random()) / mw) // 32 * 32, 1 << RECURSION_PARAMS["max_log_row_count"])
        h = max(32, int(rows * scale) // 32 * 32)
        names.append(name); specs.append(Spec(h, g, True, extra, pw - 1))
        cw, _, _ = SA.synth_chip(g, True, n_constraints=min(9 * g, 6 * g), extra_cols=extra, extra_prep=pw - 1)
        words.append(cw)
        # recursion chips talk to the memory argument only: a few 5-value (address, extension value) messages per row
        iwords.append(SA.synth_interactions_calibrated(g, True, [5] * min(2 * g, 12)))
    return _machine_dict(names, specs, SA.machine_blob_with_interactions(words, iwords), iwords)
