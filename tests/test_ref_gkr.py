"""The LogUp-GKR circuit and every GKR sumcheck round polynomial pinned to the reference's own kernels.

The oracle (oracle/gkr.hpp) and the product (sp1_b200/csrc/gkr.cu, gkr_driver.inc) agree word for word, but both apply the same reading
of the round-polynomial corrections: the eq-mass correction (pad_adj - eq_sum) with its (1 - z) factor, the x4 / /8 scaling of the 1/2
node, the eq root b = (1 - z) / (1 - 2z), the hand-off of the padding adjustment into the eq adjustment when the row variables run out,
the padding values (n = 0, d = 1) of short and empty chips and the padding of the interaction count to 2^v.  A shared slip there would pass
every other test and the restated verifier alike.  Here the reference's kernels (sp1-gpu/crates/sys/lib/logup_gkr/*.cu,
jagged_assist/fold_metadata.cu, mle/mle.cu and mle/fixlastvariable.cu, compiled unmodified into oracle/_ref/libsp1ref.so and launched by
oracle/ref_launcher.cu's ref_logup_gkr as sp1-gpu/crates/logup_gkr launches them) build the first layer, run the forward circuit and
every layer's sumcheck rounds with the oracle's lambdas, evaluation points and challenges.  Their output fractions and raw block sums,
stored in tests/golden/ref_gkr.json, are turned into round polynomials by the reference's host arithmetic (logup_gkr/src/sumcheck.rs,
restated below with oracle field operations), and the output fractions, every round polynomial, each layer's claimed sum, sumcheck
evaluation and n_0, n_1, d_0, d_1 of the oracle's proof (CPU) and of the product's proof (GPU) must equal them.

The reference only takes chips of height 0 or a multiple of 4 of at least 8 rows (a multiple of 8 when the leaf takes the two-round
lookahead), max_log_row_count >= 3 and at least two interactions; ref_logup_gkr rejects anything else before launching.  The product's
shapes outside that range (max_log_row_count 2, odd heights, heights below 8) stay pinned to the oracle alone (tests/test_gpu_gkr.py).

Record the fixture on a GPU machine with oracle/_ref built: `SP1B200_RECORD_REF=1 python -m pytest tests/test_ref_gkr.py`."""
import functools

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.ext_field import EF, HALF, ONE, ZERO, efs, eval_at, interpolate, parse_partial_sumcheck
from tests.machines import Chip, n_interactions, spec_machine, workload_machine
from tests.ref_golden import Ref, Store
from tests.ref_lib import gkr_layer_words

STORE = Store("ref_gkr", "tests/test_ref_gkr.py")
POW_BITS = 4
FOUR, INV8 = EF.of(4), EF.of(8).inv()


@pytest.fixture(scope="module", autouse=True)
def _record_golden():
    yield
    STORE.save()


# ---- the reference's host arithmetic (sp1-gpu/crates/logup_gkr/src/sumcheck.rs) ----------------------------------------------------
def eq1(z, a):
    """eq(z, a) of one coordinate: the padding-adjustment factor of a fixed variable (sumcheck.rs:473-474, 569-570, 700-702)"""
    return z * a + (ONE - z) * (ONE - a)


def finalize_univariate(e0, eh, eq_sum, claim, last, eq_adj, pad_adj):
    """sumcheck.rs:58-100: correct the sums by the eq mass of the padded rows, descale the 1/2 node by 8, and interpolate through
    {0, 1, 1/2, b} with g(b) = 0, b = (1 - z) / (1 - 2z) the root of the eq factor"""
    corr = pad_adj - eq_sum
    e0 = (e0 + corr * (ONE - last)) * eq_adj
    eh = (eh + corr * FOUR) * INV8 * eq_adj
    b = (ONE - last) * (ONE - (last + last)).inv()
    return interpolate([ZERO, ONE, HALF, b], [e0, claim - e0, eh, ZERO])


def two_round_univariates(grid, z_y, z_x, eq_adj, pad_adj, claim, a1):
    """sumcheck.rs:151-215: rounds 1 and 2 from the 10-value grid of two_round_sum_* -> (g1, g2)"""
    h00, h01, h0h, h10, h1h, hh0, hh1, hhh, eq_y0, eq_y1 = grid
    corr = pad_adj - (eq_y0 + eq_y1)
    e0 = (h00 + h10 + corr * (ONE - z_y)) * eq_adj
    eh = (h0h + h1h + corr * FOUR) * INV8 * eq_adj
    b_y = (ONE - z_y) * (ONE - (z_y + z_y)).inv()
    g1 = interpolate([ZERO, ONE, HALF, b_y], [e0, claim - e0, eh, ZERO])
    claim2 = eval_at(g1, a1)
    # round 2: each grid column interpolated through {0, 1, 1/2, b_y} and evaluated at alpha_1; the eq masses by the same interpolation
    nodes = [ZERO, ONE, HALF, b_y]
    col = lambda y0, y1, yh: eval_at(interpolate(nodes, [y0, y1, yh, ZERO]), a1)
    f0, fh = col(h00, h01, h0h * INV8), col(hh0, hh1, hhh * INV8)
    corr = pad_adj * eq1(z_y, a1) - (eq_y0 + a1 * (eq_y1 - eq_y0))
    e0 = (f0 + corr * (ONE - z_x)) * eq_adj
    eh = (fh + corr * FOUR) * INV8 * eq_adj
    b_x = (ONE - z_x) * (ONE - (z_x + z_x)).inv()
    return g1, interpolate([ZERO, ONE, HALF, b_x], [e0, claim2 - e0, eh, ZERO])


def reference_layer(raw, claim, point, challenges, v):
    """materialized_round_sumcheck / first_round_sumcheck (sumcheck.rs:918-1142) on one layer's raw kernel sums.  point: the layer's
    evaluation point (interaction variables first); challenges in round order.  -> (round polynomials, evaluation, [n0, n1, d0, d1])"""
    vals = efs(raw)
    n = len(point)
    rows = n - v
    pt = list(point)
    eq_adj = pad_adj = ONE
    polys, i, r0 = [], 0, 0
    lookahead = rows > 2
    if lookahead:   # sumcheck.rs:941-973, 1043-1082: both rounds' updates at once (two_round_fix_and_sum_*, :285-393)
        polys += two_round_univariates(vals[:10], pt[-1], pt[-2], eq_adj, pad_adj, claim, challenges[0])
        z_y, z_x = pt.pop(), pt.pop()
        pad_adj = pad_adj * eq1(z_y, challenges[0]) * eq1(z_x, challenges[1])
        rows -= 2
        i, r0 = 10, 2
    rc = claim if r0 == 0 else eval_at(polys[-1], challenges[1])
    interactions = False
    for r in range(r0, n):
        if r > 0 and not (lookahead and r == 2):   # fix_and_sum_* with the previous round's challenge
            pad_adj = pad_adj * eq1(pt.pop(), challenges[r - 1])
            if not interactions:
                if rows == 1:   # the last row variable: fixAndSumLastCircuitLayer hands the padding adjustment to the eq adjustment
                    eq_adj, pad_adj, interactions = pad_adj, ONE, True
                else:
                    rows -= 1
        e0, eh, eq_sum = vals[i:i + 3]
        i += 3
        polys.append(finalize_univariate(e0, eh, eq_sum, rc, pt[-1], eq_adj, pad_adj))
        rc = eval_at(polys[-1], challenges[r])
    assert i + 4 == len(vals), (i, len(vals))
    return polys, rc, vals[i:]


# ---- the LogUp-GKR proof words (oracle/capi.cpp put(GkrProof)) ----------------------------------------------------------------------
def parse_gkr_proof(w):
    """-> dict(out (the output numerator and denominator words), rounds: per layer dict(n0, n1, d0, d1, sc))"""
    w = np.asarray(w, np.uint32)
    n_out = int(w[0])
    o = 1 + 8 * n_out
    out = w[1:o]
    rounds = []
    nr = int(w[o]); o += 1
    for _ in range(nr):
        n0, n1, d0, d1 = efs(w[o:o + 16]); o += 16
        sc, o = parse_partial_sumcheck(w, o)
        rounds.append(dict(n0=n0, n1=n1, d0=d0, d1=d1, sc=sc))
    return dict(out=out, rounds=rounds)


# ---- cases --------------------------------------------------------------------------------------------------------------------------
# (name, machine, max_log_row_count).  Chip order = the proof's chip order = the reference's chip-name order (spec_machine names the
# chips Chip000, Chip001, ...; the workload machines' names are sorted).  Heights are 0 or multiples of 8 of at least 8 rows.
PRE = [9] * 50 + [5] * 4
CASES = [
    # v = 1 (one send and one receive); a chip without interactions; leaf one round at a time (max_log_row_count 3)
    ("mlr3_v1", [Chip(8, 1, False, None, 0, 0, [3]), Chip(0, 1, False, None, 0, 0, ())], 3),
    # 18 interactions (2^5 padded: interaction layers of odd height 9); an empty chip between chips; height 8 = the max(h, 8) minimum
    ("mlr3_empty_between", [Chip(8, 1, False), Chip(0, 2, False), Chip(8, 1, True)], 3),
    # v = 3; lookahead leaf, single-round circuit layers; heights 16, 0 and 8 (remainderModFour pads inside the transitions and folds)
    ("mlr4_leaf_lookahead", [Chip(16, 1, False, None, 0, 0, [4, 2]), Chip(0, 1, True, None, 0, 0, [5]), Chip(8, 1, True, None, 0, 0, ())], 4),
    ("mlr4_light", [Chip(16, 1, False), Chip(8, 2, True), Chip(0, 1, False)], 4),
    # lookahead circuit layers; height 24 (a multiple of 8, not of 16)
    ("mlr5_circuit_lookahead", [Chip(32, 2, True), Chip(8, 1, False), Chip(0, 1, False), Chip(24, 1, True, None, 0, 0, [12, 1])], 5),
    # heights that are multiples of 32 but not powers of two; messages of 12 values
    ("mlr8_multiples_of_32", [Chip(96, 2, True), Chip(0, 1, False), Chip(128, 1, False), Chip(32, 1, True, None, 0, 0, [12, 5]), Chip(16, 1, False),
                              Chip(160, 2, False, None, 0, 1, [7, 7, 3])], 8),
    # max_log_row_count 14: every kernel strides over its grid
    ("mlr14_strides", [Chip(16384, 2, False, None, 0, 0, [12, 3, 7]), Chip(12288, 1, True, None, 0, 0, [9, 4]), Chip(0, 1, False),
                       Chip(4096 + 32, 2, False)], 14),
    # the calibrated shapes of tests/test_gpu_gkr.py: 690 interactions (v = 10) and 1222 (v = 11)
    ("calibrated_690", [Chip(1000, 4, False, 30, 3, 0, [12, 4, 9, 5, 1, 7, 12, 3] * 8), Chip(600, 3, True, 20, 0, 3, [9] * 54 + [12] * 100),
                        Chip(2048 + 32, 2, False, None, 0, 0, [2, 3] * 60), Chip(0, 2, True, None, 0, 2, [4] * 5)], 12),
    ("calibrated_1222", [Chip(4096, 6, i % 2 == 0, 40, 2, 2 if i % 2 == 0 else 0, PRE + [12] * 10) for i in range(9)]
     + [Chip(3000, 2, False, None, 0, 0, [12] * 30)], 12),
    # the benchmark's tinyc machine at quarter size
    ("tinyc_quarter", "tinyc", 11),
]
IDS = [c[0] for c in CASES]


@functools.lru_cache(maxsize=None)
def _machine(name):
    _, spec, mlr = CASES[IDS.index(name)]
    seed = 2000 + IDS.index(name)
    if isinstance(spec, str):
        blob, heights, mains, preps, _, _ = workload_machine(spec, seed, max_log_rows=mlr, scale=0.25)
    else:
        blob, heights, mains, preps, _, _ = spec_machine(np.random.default_rng(seed), spec)
    return blob, heights, mains, preps, mlr


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """the oracle's proof: (challenger state before it, proof words, its unrecorded inputs)"""
    blob, heights, mains, preps, mlr = _machine(name)
    ch = O.Challenger()
    ch.observe(O.rand_field(np.random.default_rng(3000 + IDS.index(name)), 4))
    st0 = ch.st.copy()
    words = O.gkr_prove_verify(blob, heights, mains, preps, mlr, ch, gkr_pow_bits=POW_BITS)
    return st0, words, O.gkr_last_inputs()


@functools.lru_cache(maxsize=None)
def _run_reference(name):
    """the reference kernels on the case with the oracle's inputs (recording runs only; once per case for both tests)"""
    from tests import ref_lib as R
    blob, heights, mains, preps, mlr = _machine(name)
    _, words, (alpha, beta_seed, layers) = _oracle(name)
    chips, off = R.parse_chip_words(blob)
    inters = R.parse_interactions(blob, off, len(chips))
    challenges = [np.stack([p.w for p in reversed(r["sc"]["point"])]) for r in parse_gkr_proof(words)["rounds"]]
    return R.logup_gkr(inters, heights, mains, preps, alpha, O.partial_lagrange(beta_seed), mlr, np.stack([l[0] for l in layers]),
                       [l[2] for l in layers], challenges)


def _reference(name, v):
    """the reference kernels' raw outputs on the case (stored; run live while recording): the output fractions (digest only) and the
    per-layer sums (words)"""
    n_out = 2 << v
    out = Ref(f"gkr.{name}.out", lambda: _run_reference(name)[:8 * n_out], store=STORE)
    sums = Ref(f"gkr.{name}.rounds", lambda: _run_reference(name)[8 * n_out:], keep=True, store=STORE)
    return out, sums


def _check(name, words, who):
    blob, _, _, _, mlr = _machine(name)
    _, _, (_, _, layers) = _oracle(name)
    v = max(n_interactions(blob) - 1, 0).bit_length()
    pf = parse_gkr_proof(words)
    out, sums = _reference(name, v)
    raw = sums.words
    assert out.eq(pf["out"]), f"{who}: output fractions differ from the reference's extractOutput"
    assert len(pf["rounds"]) == len(layers) == mlr - 1
    o = 0
    for p, (rp, (_, claim, point)) in enumerate(zip(pf["rounds"], layers)):
        n = v + p + 1
        size = gkr_layer_words(v, p)
        sc = rp["sc"]
        assert sc["claim"] == EF(claim), f"{who}: layer {p}: claimed sum differs from num_eval * lambda + den_eval"
        challenges = list(reversed(sc["point"]))
        polys, final, comps = reference_layer(raw[o:o + size], EF(claim), efs(point), challenges, v)
        o += size
        assert len(sc["polys"]) == len(polys) == n, f"{who}: layer {p} has {len(sc['polys'])} rounds, the reference {len(polys)}"
        for r, (got, exp) in enumerate(zip(sc["polys"], polys)):
            assert len(got) == 4, f"{who}: layer {p} round {r} has {len(got)} coefficients"
            for k, (g, e) in enumerate(zip(got, exp)):
                assert g == e, f"{who}: layer {p} round {r} coefficient {k} differs from the reference kernels' round polynomial: {g} != {e}"
        assert sc["eval"] == final, f"{who}: layer {p}: sumcheck evaluation differs from the reference's last round polynomial at the point"
        for label, g, e in zip(("n0", "n1", "d0", "d1"), (rp["n0"], rp["n1"], rp["d0"], rp["d1"]), comps):
            assert g == e, f"{who}: layer {p}: {label} differs from the reference's fixLastVariableInteractionsLayer: {g} != {e}"
    assert o == raw.size


@pytest.mark.parametrize("name", IDS)
def test_gkr_round_polys_oracle_vs_reference(name):
    _check(name, _oracle(name)[1], "oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("name", IDS)
def test_gkr_round_polys_product_vs_reference(name):
    import torch
    from sp1_b200 import Lib
    blob, heights, mains, preps, mlr = _machine(name)
    st0, owords, _ = _oracle(name)
    lib = Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21), gkr_pow_bits=POW_BITS)
    try:
        mach = lib.machine_create(blob)
        d_mains = [torch.from_numpy(np.ascontiguousarray(m).view(np.int32)).cuda() for m in mains]
        d_preps = [torch.from_numpy(np.ascontiguousarray(p).view(np.int32)).cuda() if p is not None else None for p in preps]
        torch.cuda.synchronize()
        words = lib.logup_gkr(mach, heights, d_mains, d_preps, st0.copy())
        lib.machine_free(mach)
    finally:
        lib.close()
    _check(name, words, "product")
