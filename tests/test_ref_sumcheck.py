"""Jagged Hadamard sumcheck round polynomials pinned to the reference's own round kernels.

The oracle and the product agree word for word, but both restate the same reading of the reference, so a shared protocol slip (an
evaluation node, the order in which the first two variables are bound, the 1/2-node scaling, the zero padding of a dense length that is
not a power of two) would pass every other test and the restated verifier alike.  Here the reference's kernels
(sp1-gpu/crates/sys/lib/jagged_sumcheck/jagged_sumcheck.cu, hadamard.cu and mle/fixlastvariable.cu, compiled unmodified into
oracle/_ref/libsp1ref.so and launched by oracle/ref_launcher.cu's ref_jagged_sumcheck) are run on each case's dense trace with the
challenges of the oracle's proof.  Their raw block sums, stored in tests/golden/ref_sumcheck.json, are turned into round polynomials
by the reference's host arithmetic (sp1-gpu/crates/jagged_sumcheck/src/sumcheck.rs, restated below with oracle field operations), and
every round polynomial, the final evaluations and the stacked-PCS batch evaluations of the oracle's proof (CPU) and of the product's
proof (GPU) must equal them.

Record the fixture on a GPU machine with oracle/_ref built: `SP1B200_RECORD_REF=1 python -m pytest tests/test_ref_sumcheck.py`."""
import functools

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.ext_field import EF, HALF, ONE, QUARTER, ZERO, efs as _efs, eval_at, interpolate
from tests.jagged_layout import column_heights, dense, parse_jagged_proof, stacked_cols
from tests.ref_golden import Ref, Store

STORE = Store("ref_sumcheck", "tests/test_ref_sumcheck.py")
NQ, POW_BITS, BATCH_BITS, LOG_BLOWUP = 8, 4, 2, 2


@pytest.fixture(scope="module", autouse=True)
def _record_golden():
    yield
    STORE.save()


def reference_round_polys(raw, claim, challenges):
    """The reference's host loop (jagged_sumcheck/src/sumcheck.rs:233-355) on the raw kernel sums of R.jagged_sumcheck.
    -> (round polynomials, final evaluation, p_eval, q_eval, stacked evals)"""
    log_m = len(challenges)
    v = _efs(raw)
    nodes = [ZERO, ONE, HALF]                                                     # sumcheck.rs:271-275, hadamard.rs:192-199
    h00, h01, h0h, h10, h1h, hh0, hh1, hhh = v[:8]
    # sumcheck.rs:262-269: descale the midpoint sums by 1/4, the centre by 1/16, and deduce h(1, 1) from the claim
    h0h, h1h, hh0, hh1, hhh = h0h * QUARTER, h1h * QUARTER, hh0 * QUARTER, hh1 * QUARTER, hhh * QUARTER * QUARTER
    h11 = claim - h00 - h01 - h10
    # sumcheck.rs:277-283, round 0: g(Y) = h(0, Y) + h(1, Y)
    polys = [interpolate(nodes, [h00 + h10, h01 + h11, h0h + h1h])]
    # sumcheck.rs:285-301, round 1: g(X) = h(X, alpha_1), each grid column interpolated through the nodes and evaluated at alpha_1
    col = lambda y0, y1, yh: eval_at(interpolate(nodes, [y0, y1, yh]), challenges[0])
    polys.append(interpolate(nodes, [col(h00, h01, h0h), col(h10, h11, h1h), col(hh0, hh1, hhh)]))
    claim_r = eval_at(polys[-1], challenges[1])
    # sumcheck.rs:195-206 (round 2, from the fused two-challenge fold) and hadamard.rs:181-200 (rounds 3 .. log_m - 1):
    # eval_1 = claim - eval_0, the 1/2 node descaled by 1/4
    sums = v[8:10] + v[10:10 + 2 * (log_m - 3)]
    for r in range(2, log_m):
        e0, eh = sums[2 * (r - 2)], sums[2 * (r - 2) + 1]
        polys.append(interpolate(nodes, [e0, claim_r - e0, eh * QUARTER]))
        claim_r = eval_at(polys[-1], challenges[r])
    p_eval, q_eval = v[10 + 2 * (log_m - 3):12 + 2 * (log_m - 3)]
    return polys, claim_r, p_eval, q_eval, v[12 + 2 * (log_m - 3):]


# ---- cases --------------------------------------------------------------------------------------------------------------------------
# (name, tables per commitment round as (rows, cols), log_stacking_height, max_log_row_count).  Heights are multiples of 16, the dense
# length a multiple of 8: the preconditions of the reference's fused kernels (sumcheck.rs:107, 150).  K = the product's number of rounds
# summed from the base-field trace (2^K divides every column start, K <= 5).
CASES = [
    # K = 4 (a 16-row table), empty tables between tables
    ("k4_empty_tables", [[(48, 3), (0, 4), (16, 2)], [(80, 2), (0, 1), (16, 9)]], 6, 7),
    # K = 4; preprocessed then main round, the first round's segment (80 words) ends inside a 2^5 block; dense length 400 (zero padding)
    ("k4_segment_inside_block", [[(32, 2), (16, 1)], [(64, 3), (0, 2), (32, 4)]], 4, 6),
    # K = 5, dense length 1088: paddedHadamardFixAndSum pads odd layers with zeros
    ("k5_not_power_of_two", [[(96, 2), (32, 3)], [(0, 2), (160, 4), (32, 5)]], 5, 8),
    # log_stacking_height 3: the stacked evaluations are taken in the first loop round
    ("stacking_3", [[(64, 3), (32, 2)], [(96, 1), (0, 2), (32, 1)]], 3, 7),
    # log_stacking_height = log_m - 1: taken in the last loop round; a 160-row dummy padding column
    ("stacking_last_round", [[(128, 3), (64, 2)], [(256, 1), (32, 3)]], 9, 8),
    # heights of 2^12 and 2^13: several 2^10-row runs per column
    ("row_runs", [[(8192, 2), (4096, 3), (2048 + 32, 5), (0, 2)], [(1024, 7), (4096, 2)]], 12, 13),
    # log_m = 21 (dense length 1.5 * 2^20): every kernel loops over its grid
    ("log_m_21", [[(2 ** 17, 3), (0, 3), (2 ** 16 + 32, 5)], [(2 ** 17 - 160, 6)]], 16, 17),
]
IDS = [c[0] for c in CASES]


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """the case's tables and the oracle's proof: (rounds, z_row, challenger state before the proof, proof words, z_col, claim)"""
    _, shapes_rounds, log_stack, mlr = CASES[IDS.index(name)]
    rng = np.random.default_rng(1000 + IDS.index(name))
    rounds = [O.random_tables(rng, s) for s in shapes_rounds]
    z_row = O.rand_field(rng, (mlr, 4))
    ch = O.Challenger()
    ch.observe(O.rand_field(rng, 3))
    st0 = ch.st.copy()
    _, _, proof = O.jagged_prove_verify(rounds, log_stack, mlr, z_row, ch, log_blowup=LOG_BLOWUP, num_queries=NQ, pow_bits=POW_BITS,
                                        batch_pow_bits=BATCH_BITS)
    z_col, claim = O.jagged_last_inputs()
    return rounds, z_row, st0, proof, z_col, claim


def _reference(name, pf):
    """the reference kernels' raw sums on the case (stored words; run live while recording)"""
    _, shapes_rounds, log_stack, mlr = CASES[IDS.index(name)]

    @functools.lru_cache(maxsize=1)
    def run():
        from tests import ref_lib as R
        rounds, z_row, _, _, z_col, _ = _oracle(name)
        heights = column_heights(pf["rc_cc"])
        challenges = np.stack([p.w for p in reversed(pf["sumcheck"]["point"])])
        return R.jagged_sumcheck(dense(rounds, log_stack), heights, O.partial_lagrange(z_row), O.partial_lagrange(z_col), challenges,
                                 log_stack)
    n_rounds = 12 + 2 * (pf["log_m"] - 3)
    sums = Ref(f"jagged.{name}.rounds", lambda: run()[:4 * n_rounds], keep=True, store=STORE)
    stacked = Ref(f"jagged.{name}.stacked", lambda: run()[4 * n_rounds:], store=STORE)
    return sums, stacked


def _check(name, words, who):
    _, shapes_rounds, log_stack, _ = CASES[IDS.index(name)]
    _, _, _, _, z_col, claim = _oracle(name)
    pf = parse_jagged_proof(words, stacked_cols(shapes_rounds, log_stack), log_stack, NQ, LOG_BLOWUP)
    sc = pf["sumcheck"]
    assert sc["claim"] == EF(claim), f"{who}: Hadamard sumcheck claim differs from the oracle's z_col claim"
    sums, stacked = _reference(name, pf)
    challenges = list(reversed(sc["point"]))
    polys, final, p_eval, q_eval, _ = reference_round_polys(sums.words, EF(claim), challenges)
    assert len(sc["polys"]) == len(polys) == pf["log_m"]
    for r, (got, exp) in enumerate(zip(sc["polys"], polys)):
        for k, (g, e) in enumerate(zip(got, exp)):
            assert g == e, f"{who}: round {r} coefficient {k} differs from the reference kernels' round polynomial: {g} != {e}"
        assert len(got) == len(exp) == 3, f"{who}: round {r} has {len(got)} coefficients"
    assert sc["eval"] == final, f"{who}: sumcheck evaluation differs from the reference's last round polynomial at the point"
    assert pf["expected_eval"] == p_eval, f"{who}: trace evaluation (p_eval) differs from the reference's final fold"
    assert p_eval * q_eval == sc["eval"], f"{who}: p_eval * q_eval of the reference differs from the sumcheck evaluation"
    batch = np.stack([e.w for e in pf["batch_evals"]])
    assert stacked.eq(batch), f"{who}: stacked-PCS batch evaluations differ from the reference's stacked_evals snapshot"


@pytest.mark.parametrize("name", IDS)
def test_jagged_round_polys_oracle_vs_reference(name):
    _check(name, _oracle(name)[3], "oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("name", IDS)
def test_jagged_round_polys_product_vs_reference(name):
    from sp1_b200 import Lib
    _, shapes_rounds, log_stack, mlr = CASES[IDS.index(name)]
    rounds, z_row, st0, _, _, _ = _oracle(name)
    lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, num_queries=NQ, pow_bits=POW_BITS, batch_pow_bits=BATCH_BITS)
    try:
        handles, claims = [], []
        for tabs in rounds:
            _, h = lib.jagged_commit(tabs)
            handles.append(h)
            claims.append(lib.jagged_column_claims(h, z_row, sum(t.shape[0] for t in tabs)))
        st = st0.copy()
        proof = lib.jagged_prove(handles, z_row, np.concatenate(claims), st)
        for h in handles:
            lib.jagged_round_free(h)
    finally:
        lib.close()
    _check(name, proof, "product")
