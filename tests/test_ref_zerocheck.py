"""The zerocheck round polynomials, claimed sum and opened values pinned to the reference's own zerocheck kernels.

The oracle (oracle/zerocheck.hpp) and the product (sp1_b200/csrc/zerocheck.cu) agree word for word, and the restated verifier accepts
both, but all three read the protocol the same way: the order of the alpha powers and each chip's offset into the reversed table, the
Horner order of the lambda weighting (chip 0 gets lambda^(n-1)), the gamma^1... opening batch with main columns before preprocessed ones,
the padded-row adjustment and the VirtualGeq correction that cancels it on the padding rows, the eq adjustment carried across folds and
the eq root, the zero padding of the folds and the opened values.  A shared slip there would pass every other test.  Here the
reference's kernels (sp1-gpu/crates/sys/lib/zerocheck/*.cu and jagged_assist/{chip_layouts,fold_metadata}.cu, compiled unmodified into
oracle/_ref/libsp1ref.so and launched by oracle/ref_launcher.cu's ref_zerocheck as sp1-gpu/crates/zerocheck/src/prover.rs launches
them) run the padded-row adjustment, the fused first two rounds, every later round and every fold with the oracle's challenges.  Their
raw totals, stored in tests/golden/ref_zerocheck.json, are turned into the proof by the reference's host arithmetic (prover.rs and
grid.rs, restated below with oracle field operations), and every round polynomial, the claimed sum, the final point and evaluation and
every opened value of the oracle's proof (CPU) and of the product's proof (GPU) must equal it.

The reference takes heights that are multiples of 4 up to 2^max_log_row_count, max_log_row_count >= 2 and constraint programs of at
most 1024 registers as the machine blob stores them (one register per node, so the benchmark's tinyc machine is out of range);
ref_zerocheck rejects anything else before launching.  The product's shapes outside that range (odd heights, heights = 2 mod 4,
max_log_row_count < 2, larger programs) stay pinned to the oracle alone (tests/test_gpu_zerocheck.py).

Record the fixture on a GPU machine with oracle/_ref built: `SP1B200_RECORD_REF=1 python -m pytest tests/test_ref_zerocheck.py`."""
import functools

import numpy as np
import pytest

from sp1_b200 import synth_air as SA
from tests import oracle_lib as O
from tests.ext_field import EF, ONE, ZERO, efs, eval_at, interpolate, parse_partial_sumcheck
from tests.machines import PV0, Chip, oracle_zerocheck, product_zerocheck, spec_machine, workload_machine
from tests.ref_golden import Ref, Store

STORE = Store("ref_zerocheck", "tests/test_ref_zerocheck.py")
NODE_XS = [0, 1, 2, 4]                                                                            # grid.rs:26
CONSTRAINT_NODES = [(0, 2), (0, 3), (1, 2), (1, 3), (2, 0), (2, 1), (2, 2), (2, 3), (3, 0), (3, 1), (3, 2), (3, 3)]   # grid.rs:31-44


@pytest.fixture(scope="module", autouse=True)
def _record_golden():
    yield
    STORE.save()


# ---- the reference's host arithmetic (sp1-gpu/crates/zerocheck/src/prover.rs, grid.rs) ----------------------------------------------
def powers(x, n, start=0):
    out, p = [], ONE
    for i in range(start + n):
        if i >= start:
            out.append(p)
        p = p * x
    return out


def host_tables(alpha, gamma, lam, chips):
    """prover.rs:2438-2459: alpha^0 .. alpha^(max_constraints - 1) reversed, gamma^1 .. gamma^max_columns, lambda^0 .. lambda^(n-1)
    reversed"""
    max_nc = max(c["n_constraints"] for c in chips)
    max_cols = max(c["main_w"] + c["prep_w"] for c in chips)
    return powers(alpha, max_nc)[::-1], powers(gamma, max_cols, start=1), powers(lam, len(chips))[::-1]


def claimed_sum(openings, chips, gkr_pows, lam):
    """prover.rs:2461-2483: Horner in lambda over the chips of sum_j gkr_powers[j] * opening_j, main openings before preprocessed"""
    claim, k = ZERO, 0
    for c in chips:
        w = c["main_w"] + c["prep_w"]
        claim = claim * lam
        for j in range(w):
            claim = claim + openings[k + j] * gkr_pows[j]
        k += w
    return claim


def eq_at_nodes(z):
    """grid.rs:47-54"""
    return [ONE - z, z, z * EF.of(3) - ONE, z * EF.of(7) - EF.of(3)]


def eq_root(z):
    """grid.rs:57-59"""
    return (ONE - z) * (ONE - (z + z)).inv()


def assemble_grid(totals):
    """prover.rs:2161-2182: the 12 node totals plus the bilinear extension of the 4 corner GKR totals (corner c = 2x + y)"""
    g00, g01, g10, g11 = totals[12:16]
    gx, gy, gxy = g10 - g00, g01 - g00, g11 - g10 - g01 + g00
    grid = [[ZERO] * 4 for _ in range(4)]
    grid[0][0], grid[0][1], grid[1][0], grid[1][1] = g00, g01, g10, g11
    for e, (ix, iy) in enumerate(CONSTRAINT_NODES):
        x, y = EF.of(NODE_XS[ix]), EF.of(NODE_XS[iy])
        grid[ix][iy] = totals[e] + g00 + gx * x + gy * y + gxy * (x * y)
    return grid


def first_round_message(grid, z_a, z_b, eq_adj):
    """zerocheck_first_round_message_from_grid (grid.rs:65-90)"""
    eq_y = eq_at_nodes(z_b)
    ys = [eq_adj * eq_y[iy] * ((ONE - z_a) * grid[0][iy] + z_a * grid[1][iy]) for iy in range(4)]
    return interpolate([EF.of(x) for x in NODE_XS] + [eq_root(z_b)], ys + [ZERO])


def second_round_message(grid, z_a, z_b, eq_adj, alpha):
    """zerocheck_second_round_message_from_grid (grid.rs:95-131)"""
    nodes = [EF.of(x) for x in NODE_XS]
    weights = []
    for k in range(4):
        num, den = ONE, ONE
        for j in range(4):
            if j != k:
                num, den = num * (alpha - nodes[j]), den * (nodes[k] - nodes[j])
        weights.append(num * den.inv())
    eq_x = eq_at_nodes(z_a)
    eq_y_at_alpha = z_b * alpha + (ONE - z_b) * (ONE - alpha)
    ys = [eq_adj * eq_y_at_alpha * eq_x[ix] * sum((weights[iy] * grid[ix][iy] for iy in range(4)), ZERO) for ix in range(4)]
    return interpolate(nodes + [eq_root(z_a)], ys + [ZERO])


def later_round_message(totals, last, eq_adj, claim):
    """evaluate_zerocheck's finalisation (prover.rs:1777-1795): the totals at {0, 2, 4} times eq(last, x) and the eq adjustment, the
    claim minus the node-0 value at 1, and 0 at the eq root (last - 1) / (2 last - 1)"""
    xs = [EF.of(0), EF.of(2), EF.of(4)]
    ys = [t * ((ONE - x) * (ONE - last) + x * last) * eq_adj for x, t in zip(xs, totals)]
    return interpolate(xs + [ONE, (last - ONE) * (last + last - ONE).inv()], ys + [claim - ys[0], ZERO])


def eq1(z, a):
    return (ONE - z) * (ONE - a) + z * a


def reference_proof(raw, zeta, challenges, claim, n_chips, mlr):
    """zerocheck() (prover.rs:2557-2677) on the raw kernel totals: -> (round polynomials, point (Point::add_dimension order), evaluation,
    the column values)"""
    vals = efs(raw)
    grid = assemble_grid(vals[n_chips:n_chips + 16])
    rounds = vals[n_chips + 16:n_chips + 16 + 3 * (mlr - 2)]
    z = list(zeta)
    z_a, z_b = z[-2], z[-1]
    eq_adj = ONE
    g1 = first_round_message(grid, z_a, z_b, eq_adj)
    assert eval_at(g1, ZERO) + eval_at(g1, ONE) == claim, "the reference's first round message does not sum to the claim"
    g2 = second_round_message(grid, z_a, z_b, eq_adj, challenges[0])
    claim = eval_at(g2, challenges[1])
    eq_adj = eq_adj * eq1(z_b, challenges[0]) * eq1(z_a, challenges[1])     # prover.rs:2328-2330
    z = z[:-2]
    polys = [g1, g2]
    for r in range(2, mlr):
        g = later_round_message(rounds[3 * (r - 2):3 * (r - 1)], z[-1], eq_adj, claim)
        polys.append(g)
        claim = eval_at(g, challenges[r])
        eq_adj = eq_adj * eq1(z[-1], challenges[r])                         # prover.rs:2224-2225
        z = z[:-1]
    point = list(reversed(challenges))                                      # add_dimension inserts at the front
    return polys, point, claim, vals[n_chips + 16 + 3 * (mlr - 2):]


def opened_values(colvals, chips):
    """prover.rs:2695-2732: preprocessed values from column 0, main values from preprocessed_cols on, which counts the padding column
    (zerocheck/src/lib.rs:1303-1324) -> per chip (prep, main)"""
    pp, mp = 0, sum(c["prep_w"] for c in chips) + 1
    out = []
    for c in chips:
        out.append((colvals[pp:pp + c["prep_w"]], colvals[mp:mp + c["main_w"]]))
        pp += c["prep_w"]; mp += c["main_w"]
    return out


def max_reg(chip):
    """the register file the reference's interpreter needs for the blob's program (bytecode.rs:208-209)"""
    return int((chip["instrs"].reshape(-1, 2)[:, 0] >> 16).max()) + 1 if chip["instrs"].size else 0


# ---- cases --------------------------------------------------------------------------------------------------------------------------
def _vanishing_chip():
    """the first three constraints of synth_air's one-group template (c - ab, d (d - 1), e - abd): all vanish on the zero row, so the
    padded-row adjustment is 0 and no geq correction is launched for the chip"""
    a = SA.Asm()
    one = a.const(1)
    A, B, Cc, D, E = (a.leaf(SA.LEAF_MAIN, i) for i in range(5))
    ab = a.op(SA.MUL, A, B)
    a.assert_zero(a.op(SA.SUB, Cc, ab))
    a.assert_zero(a.op(SA.MUL, D, a.op(SA.SUB, D, one)))
    a.assert_zero(a.op(SA.SUB, E, a.op(SA.MUL, ab, D)))
    return a.words(6, 0)


def _synth(rng, spec):
    """spec: list of (height, groups, with_prep, kind), kind "flat", "deep" (long-lived intermediates) or "vanishing" (one group)"""
    words, mains, preps, heights = [], [], [], []
    for h, g, wp, kind in spec:
        assert kind != "vanishing" or (g, wp) == (1, False), "the vanishing chip has one group and no preprocessed column"
        words.append(_vanishing_chip() if kind == "vanishing" else SA.synth_chip(g, wp, deep=kind == "deep")[0])
        m, p = SA.synth_trace(rng, h, g, wp, PV0)
        mains.append(m); preps.append(p); heights.append(h)
    return SA.machine_blob(words), heights, mains, preps, O.to_monty(np.array([PV0, 5, 6, 7]))


# (name, kind, spec, max_log_row_count)
CASES = [
    # only the fused pass runs (no later round); one chip of exactly 2^mlr rows (no padded rows)
    ("mlr2_full_height", "synth", [(4, 1, False, "flat")], 2),
    # heights 4 * odd at several levels: odd pair counts that the folds zero-pad and odd VirtualGeq thresholds; chips with and without
    # a padded-row adjustment
    ("heights_4_mod_8", "synth", [(12, 1, True, "flat"), (20, 1, False, "vanishing"), (4, 1, False, "flat"), (44, 2, True, "flat"),
                                  (108, 1, False, "flat"), (76, 1, False, "vanishing")], 7),
    # the MAX_REGS = 1024 template and the 64-thread block (a 1024-register program), next to narrow chips
    ("registers_1024", "synth", [(192, 68, False, "deep"), (64, 3, True, "flat"), (96, 10, False, "deep")], 8),
    # a tier split: eleven chunks, one above 256 registers (MAX_REGS 512) and a 256-register tier 0 on 64-thread blocks
    ("tier_split", "synth", [(16 * (k + 1), 1 + k % 3, k % 2 == 0, "flat") for k in range(9)]
     + [(96, 16, False, "deep"), (64, 33, True, "deep")], 8),
    # a 682-column chip (the decoupled gkr_sweep) next to narrow chips (the inline carrier GKR)
    ("wide_682", "spec", [Chip(256, 4, False, None, 658), Chip(64, 1, True), Chip(100, 2, False)], 9),
    # calibrated chips: up to 36 preprocessed columns, heights that are not multiples of 32, an empty chip
    ("calibrated", "spec", [Chip(700, 4, True, 36, 5, 3), Chip(96, 14, False, 60, 0, 0), Chip(0, 2, True, 18, 1, 2), Chip(36, 1, True, 9, 7, 35),
                            Chip(2044, 12, False, 100, 2, 0)], 11),
    # the benchmark's compress-shape machine at a quarter of its size
    ("tinyr_quarter", "tinyr", None, 12),
    # an empty chip between chips
    ("empty_between", "synth", [(16, 1, False, "flat"), (0, 2, True, "flat"), (8, 1, False, "vanishing"), (0, 1, False, "flat"),
                                (12, 1, True, "flat")], 4),
]
IDS = [c[0] for c in CASES]


@functools.lru_cache(maxsize=None)
def _machine(name):
    _, kind, spec, mlr = CASES[IDS.index(name)]
    seed = 4000 + IDS.index(name)
    if kind == "synth":
        blob, heights, mains, preps, pv = _synth(np.random.default_rng(seed), spec)
    elif kind == "spec":
        blob, heights, mains, preps, pv, _ = spec_machine(np.random.default_rng(seed), spec)
    else:
        blob, heights, mains, preps, pv, _ = workload_machine(kind, seed, max_log_rows=mlr, scale=0.25)
    from tests.ref_lib import parse_chip_words
    return blob, heights, mains, preps, pv, mlr, parse_chip_words(blob)[0]


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """the oracle's proof: (GKR point, challenger state before it, openings at the GKR point, proof words, recorded inputs)"""
    blob, heights, mains, preps, pv, mlr, _ = _machine(name)
    gp, st0, openings, words, _ = oracle_zerocheck(np.random.default_rng(5000 + IDS.index(name)), blob, heights, mains, preps, pv, mlr)
    return gp, st0, openings, words, O.zerocheck_last_inputs()


def _prep_pad_rows(chips, heights, mlr):
    """the preprocessed padding column: the preprocessed section padded to a multiple of 2^min(mlr, 4) rows, at least one multiple"""
    stacking = 1 << min(mlr, 4)
    total = sum(c["prep_w"] * h for c, h in zip(chips, heights))
    return (-total) % stacking or stacking


@functools.lru_cache(maxsize=None)
def _run_reference(name):
    """the reference kernels on the case with the oracle's inputs (recording runs only; once per case for both tests)"""
    from tests import ref_lib as R
    blob, heights, mains, preps, pv, mlr, chips = _machine(name)
    gp, _, _, _, (alpha, gamma, lam, _, challenges) = _oracle(name)
    a_pows, g_pows, l_pows = host_tables(EF(alpha), EF(gamma), EF(lam), chips)
    w = lambda xs: np.stack([x.w for x in xs])
    return R.zerocheck(blob, heights, mains, preps, _prep_pad_rows(chips, heights, mlr), pv, w(a_pows), w(g_pows), w(l_pows), mlr, gp, challenges)


def _reference(name):
    return Ref(f"zerocheck.{name}", lambda: _run_reference(name), keep=True, store=STORE)


def _check_case_shape(name, raw):
    """each case exercises what it is there for"""
    _, heights, _, _, _, mlr, chips = _machine(name)
    pad = efs(raw[:4 * len(chips)])
    regs = [max_reg(c) for c in chips]
    if name == "mlr2_full_height":
        assert mlr == 2 and heights == [1 << mlr]
    elif name == "heights_4_mod_8":
        assert all(h % 8 == 4 for h in heights) and len({h for h in heights}) >= 5
        assert any(p == ZERO for p in pad) and any(p != ZERO for p in pad), "needs chips with and without a padded-row adjustment"
    elif name == "registers_1024":
        assert 512 < max(regs) <= 1024, regs
    elif name == "tier_split":
        high = [r for r in regs if r > 256]
        assert len(chips) >= 10 and len(high) == 1 and len(high) * 10 <= len(chips), regs
        assert 128 < max(r for r in regs if r <= 256) <= 256 and 256 < high[0] <= 512, regs
    elif name == "wide_682":
        widths = [c["main_w"] + c["prep_w"] for c in chips]
        assert 682 in widths and min(widths) <= 256, widths
    elif name == "calibrated":
        assert max(c["prep_w"] for c in chips) == 36 and any(h % 32 for h in heights if h)
    elif name == "empty_between":
        assert 0 in heights[1:-1]


def _check(name, words, who):
    blob, heights, mains, preps, pv, mlr, chips = _machine(name)
    gp, _, openings, _, (alpha, gamma, lam, claim, challenges) = _oracle(name)
    ref = _reference(name)
    raw = ref.words
    _check_case_shape(name, raw)
    _, g_pows, _ = host_tables(EF(alpha), EF(gamma), EF(lam), chips)
    claim = claimed_sum(efs(openings), chips, g_pows, EF(lam))
    sc, o = parse_partial_sumcheck(words, 0)
    assert sc["claim"] == claim, f"{name}: {who}: the claimed sum differs from the reference's: {sc['claim']} != {claim}"
    polys, point, final, colvals = reference_proof(raw, efs(gp), efs(challenges), claim, len(chips), mlr)
    assert len(sc["polys"]) == len(polys) == mlr, f"{name}: {who}: {len(sc['polys'])} rounds, the reference {len(polys)}"
    for r, (got, exp) in enumerate(zip(sc["polys"], polys)):
        assert len(got) == len(exp), f"{name}: {who}: round {r} has {len(got)} coefficients, the reference {len(exp)}"
        for k, (g, e) in enumerate(zip(got, exp)):
            assert g == e, f"{name}: {who}: round {r} coefficient {k} differs from the reference kernels' round polynomial: {g} != {e}"
    assert sc["point"] == point, f"{name}: {who}: the sumcheck point differs from the reference's"
    assert sc["eval"] == final, f"{name}: {who}: the sumcheck evaluation differs from the reference's last round polynomial at the point"
    vals = efs(words[o:])
    v = 0
    for k, (c, (rp, rm)) in enumerate(zip(chips, opened_values(colvals, chips))):
        for kind, exp in (("preprocessed", rp), ("main", rm)):
            for j, e in enumerate(exp):
                assert vals[v] == e, f"{name}: {who}: chip {k} {kind} column {j}: opened value differs from the reference's folded column"
                v += 1
    assert v == len(vals), f"{name}: {who}: {len(vals)} opened values, the reference {v}"


@pytest.mark.parametrize("name", IDS)
def test_zerocheck_oracle_vs_reference(name):
    _check(name, _oracle(name)[3], "oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("name", IDS)
def test_zerocheck_product_vs_reference(name):
    from sp1_b200 import Lib
    blob, heights, mains, preps, pv, mlr, _ = _machine(name)
    gp, st0, openings, _, _ = _oracle(name)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21))
    try:
        mach = lib.machine_create(blob)
        words, _ = product_zerocheck(lib, mach, heights, mains, preps, pv, gp, st0, openings)
        lib.machine_free(mach)
    finally:
        lib.close()
    _check(name, words, "product")
