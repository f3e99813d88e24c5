"""The jagged evaluation (branching-program) sumcheck pinned to the reference's own jagged_assist kernels.

The oracle (oracle/jagged.hpp BranchingProgram, jagged_eval_prove) and the product (csrc/jagged.cu bp_suffix_kernel / bp_round_kernel /
bp_update_kernel, csrc/sumcheck.cuh bp_transition) share one reading of the reference: the transition function, the condensing of equal
merged prefix sums, the order in which variables are bound, the 1/2 node and where the claimed sum enters the transcript.  The shard
verifier calls the same bp_transition.  A slip shared by all of them passes every other test and both restated verifiers.  Here the
reference's kernels (sp1-gpu/crates/sys/lib/jagged_assist/branching_program.cu: branchingProgram, interpolateAndObserve on the device
DuplexChallenger, fixLastVariable and transition, compiled unmodified into oracle/_ref/libsp1ref.so and launched by
oracle/ref_launcher.cu's ref_jagged_eval and ref_bp_transitions) run each case from the challenger state the oracle had before the
claimed sum was observed.  Their outputs, stored in tests/golden/ref_jagged_eval.json, are turned into the proof by the reference's host
arithmetic (sp1-gpu/crates/jagged_assist/src/sync_eval_sumcheck.rs, restated below), and the claimed sum, every round polynomial, the
point and the final evaluation of the oracle's proof (CPU) and of the product's proof (GPU) must equal them.  The oracle's challenger
after the sumcheck must also equal the reference's.

Record the fixture on a GPU machine with oracle/_ref built: `SP1B200_RECORD_REF=1 python -m pytest tests/test_ref_jagged_eval.py`."""
import ctypes as C
import functools
import itertools

import numpy as np
import pytest

from tests import machines as M
from tests import oracle_lib as O
from tests.ext_field import HALF, ONE, ZERO, efs, eval_at, interpolate
from tests.jagged_layout import column_heights, parse_jagged_proof, stacked_cols
from tests.ref_golden import Ref, Store

STORE = Store("ref_jagged_eval", "tests/test_ref_jagged_eval.py")
NQ, POW_BITS, BATCH_BITS, LOG_BLOWUP = 8, 4, 2, 2


@pytest.fixture(scope="module", autouse=True)
def _record_golden():
    yield
    STORE.save()


def log2_ceil(n):
    """sync_eval_sumcheck.rs:25-31: 0 for n <= 1"""
    return 0 if n <= 1 else (n - 1).bit_length()


def condensed(heights, z_col):
    """new_jagged_eval_sumcheck_poly_sync (sync_eval_sumcheck.rs:59-91) on the column heights of the jagged layout.
    -> (log_m, merged prefix sums [nk, 2 (log_m + 1)] as 0/1, condensed z_col eq values [nk] EF)"""
    prefix = [0] + list(itertools.accumulate(heights))
    log_m = log2_ceil(prefix[-1])
    # Point::from_usize(x, log_m + 1): most significant bit first (slop/crates/multilinear/src/point.rs:93-103)
    bits = [tuple((x >> i) & 1 for i in reversed(range(log_m + 1))) for x in prefix]
    merged = [a + b for a, b in zip(bits, bits[1:])]                                    # windows(2), current || next
    eq = efs(O.partial_lagrange(z_col))                                                 # Mle::blocking_partial_lagrange(z_col)
    # zip stops at the shorter side, chunk_by groups equal consecutive merged prefix sums and sums their eq values
    groups = [(m, [e for _, e in g]) for m, g in itertools.groupby(zip(merged, eq), key=lambda t: t[0])]
    zc = [functools.reduce(lambda a, b: a + b, g, ZERO) for _, g in groups]
    return log_m, np.array([m for m, _ in groups], np.uint32), zc


def reference_proof(sum_values, point):
    """prove_jagged_eval_sumcheck_sync's host tail (sync_eval_sumcheck.rs:215-238) on the stored sums: each (y_0, y_1/2, y_1) through
    interpolate_univariate_polynomial at (0, 1/2, 1); the final claim is the last polynomial at the point's first (most recent)
    coordinate.  -> (round polynomials, final evaluation)"""
    polys = [interpolate([ZERO, HALF, ONE], efs(ys)) for ys in np.asarray(sum_values, np.uint32).reshape(-1, 12)]
    return polys, eval_at(polys[-1], efs(point)[0])


# ---- cases --------------------------------------------------------------------------------------------------------------------------
# (name, tables per commitment round as (rows, cols) or a benchmark workload at quarter size, log_stacking_height, max_log_row_count,
# the edge the case reaches).  Every round is padded to a multiple of 2^log_stacking_height by two dummy tables (jagged_commit): up to
# 2^mlr-row columns and one last column, which may be empty.  An edge reads the layout the proof records:
#   L.real   heights of the real columns (dummy tables left out),  L.heights  every column,  L.total  the last prefix sum
#   L.ncols  the columns (the z_col eq table has 2^log2_ceil(ncols) entries),  L.nk  the merged prefix sums after condensing
CASES = [
    # odd heights, one-row tables
    ("odd_heights_one_row", [[(1, 1), (7, 3), (1, 2), (13, 1)], [(5, 2), (1, 1), (3, 4)]], 2, 4,
     lambda L: 1 in L.real and sum(h % 2 for h in L.real) >= 5),
    # the last prefix sum is exactly 2^log_m: the only next prefix sum whose top bit is set
    ("total_pow2", [[(16, 3), (8, 2)], [(32, 2)]], 3, 5, lambda L: L.total == 1 << L.log_m),
    # real heights sum to 2^(log_m - 1) + 1; stacking pads the round to 2^(log_m - 1) + 4, the least total above 2^(log_m - 1)
    ("total_half_plus_1", [[(32, 2), (0, 3), (1, 1)]], 2, 5,
     lambda L: sum(L.real) == (1 << (L.log_m - 1)) + 1 and L.total == (1 << (L.log_m - 1)) + 4),
    # empty multi-column tables at the start, in the middle and at the end of a round: merged prefix sums repeat, so condensing sums
    # z_col eq values, and the first merged prefix sum is (0, 0)
    ("empty_tables", [[(0, 3), (9, 2), (0, 4), (5, 3), (0, 2)], [(0, 2), (6, 1), (0, 5)]], 2, 4,
     lambda L: L.rc[0][0] == (0, 3) and L.rc[0][2] == (0, 4) and L.rc[0][4] == (0, 2) and L.rc[1][0] == (0, 2) and L.rc[1][2] == (0, 5)
     and L.heights[0] == 0 and L.ncols - L.nk == 2 + 3 + 1 + 1 + 4),
    # max_log_row_count = log_m + 1 (the largest the product takes): the reference walks one layer more than there are prefix-sum bits
    ("mlr_log_m_plus_1", [[(40, 1), (3, 5)], [(9, 2)]], 3, 8, lambda L: L.mlr == L.log_m + 1),
    # max_log_row_count = log_m
    ("mlr_log_m", [[(100, 1), (20, 1)]], 2, 7, lambda L: L.mlr == L.log_m),
    # max_log_row_count well below log_m: z_row runs out six layers below the top
    ("mlr_far_below", [[(8, 40), (3, 9)]], 3, 3, lambda L: L.mlr + 6 == L.log_m),
    # 257 columns, the dummy one included, none condensed: a second block of the reference's grid with one live thread
    ("cols_257", [[(3, 200), (5, 56)]], 2, 3, lambda L: L.ncols == 257 and L.nk == 257),
    # 512 columns, the dummy one included: two full blocks, a z_col eq table with no spare entry
    ("cols_512", [[(2, 300), (1, 211)]], 2, 2, lambda L: L.ncols == 512 and L.nk == 512),
    # more than 512 merged prefix sums after condensing (three blocks), a 40-column empty table condensed inside them
    ("three_blocks", [[(6, 333), (0, 40), (11, 200)], [(4, 120)]], 3, 4, lambda L: L.nk > 512 and L.ncols - L.nk == 39),
    # a single real column
    ("single_column", [[(37, 1)]], 2, 6, lambda L: len(L.real) == 1),
    # the benchmark's tinyc table layout at quarter size: a preprocessed round and 2425 main columns
    ("tinyc_quarter", "tinyc", 10, 11, lambda L: L.nk > 2000 and len(L.rc) == 2),
    # log_m = 21: 44 rounds
    ("log_m_21", [[(2 ** 17, 6), (2 ** 16 + 5, 3), (0, 2)], [(2 ** 17 - 3, 1)]], 16, 17, lambda L: L.log_m == 21 and 2 * (L.log_m + 1) == 44),
]
IDS = [c[0] for c in CASES]


class Layout:
    """the jagged layout a proof records (see CASES)"""

    def __init__(self, rc_cc, mlr, z_col):
        self.rc, self.mlr = rc_cc, mlr
        self.heights = column_heights(rc_cc)
        self.real = [rows for rc in rc_cc for rows, cols in rc[:-2] for _ in range(cols)]
        self.total, self.ncols = sum(self.heights), len(self.heights)
        self.log_m, self.merged, self.zc = condensed(self.heights, z_col)
        self.nk = len(self.zc)


@functools.lru_cache(maxsize=None)
def _rounds(name):
    _, spec, _, mlr, _ = CASES[IDS.index(name)]
    seed = 5000 + IDS.index(name)
    if isinstance(spec, str):
        _, _, mains, preps, _, _ = M.workload_machine(spec, seed, max_log_rows=mlr, scale=0.25)
        return [[p for p in preps if p is not None], mains]
    rng = np.random.default_rng(seed)
    return [O.random_tables(rng, s) for s in spec]


def _shapes(name):
    return [[(t.shape[1], t.shape[0]) for t in tabs] for tabs in _rounds(name)]


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """the oracle's proof: (z_row, challenger state before the proof, proof words, z_col, challenger before the evaluation sumcheck's
    claim, challenger after its last sample)"""
    _, _, log_stack, mlr, _ = CASES[IDS.index(name)]
    rng = np.random.default_rng(6000 + IDS.index(name))
    z_row = O.rand_field(rng, (mlr, 4))
    ch = O.Challenger()
    ch.observe(O.rand_field(rng, 5))
    st0 = ch.st.copy()
    _, _, proof = O.jagged_prove_verify(_rounds(name), log_stack, mlr, z_row, ch, log_blowup=LOG_BLOWUP, num_queries=NQ, pow_bits=POW_BITS,
                                        batch_pow_bits=BATCH_BITS)
    z_col, _ = O.jagged_last_inputs()
    before, after = O.jagged_eval_states()
    return z_row, st0, proof, z_col, before, after


def _parse(name, words):
    _, _, log_stack, mlr, _ = CASES[IDS.index(name)]
    pf = parse_jagged_proof(words, stacked_cols(_shapes(name), log_stack), log_stack, NQ, LOG_BLOWUP)
    return pf, Layout(pf["rc_cc"], mlr, _oracle(name)[3])


@functools.lru_cache(maxsize=None)
def _reference(name):
    """the reference kernels' outputs on the case, from the oracle's inputs (stored words; run live while recording)"""
    pf, L = _parse(name, _oracle(name)[2])

    @functools.lru_cache(maxsize=1)
    def run():
        from tests import ref_lib as R
        z_row, _, _, _, before, _ = _oracle(name)
        z_index = np.stack([p.w for p in pf["sumcheck"]["point"]])      # the Hadamard sumcheck point, as jagged_prove passes it
        bp, sums, point, st = R.jagged_eval(O.to_monty(L.merged), np.stack([e.w for e in L.zc]), z_row, z_index,
                                            pf["eval_sumcheck"]["claim"].w, before)
        assert (bp[0] == bp[1]).all(), "the round_num = -1 launch differs between its two lambda rows"
        return bp[0], sums, point, st
    return {k: Ref(f"eval.{name}.{k}", functools.partial(lambda i: run()[i], i), keep=True, store=STORE)
            for i, k in enumerate(("bp", "sum_values", "point", "challenger"))}


def _check(name, words, who):
    pf, L = _parse(name, words)
    assert CASES[IDS.index(name)][4](L), f"{name}: the layout {pf['rc_cc']} does not reach the case's edge"
    assert pf["log_m"] == L.log_m
    ref = _reference(name)
    esc = pf["eval_sumcheck"]
    dim = 2 * (L.log_m + 1)
    # the claimed sum: sum_k zc_k * bp_k over the program values at the boolean prefix sums
    bp = efs(ref["bp"].words)
    assert len(bp) == L.nk
    claim = functools.reduce(lambda a, b: a + b, (z * v for z, v in zip(L.zc, bp)), ZERO)
    assert esc["claim"] == claim, f"{who}: claimed sum differs from sum_k zc_k * bp_k of the reference's branching program"
    polys, final = reference_proof(ref["sum_values"].words, ref["point"].words)
    assert len(esc["polys"]) == len(polys) == dim
    for r, (got, exp) in enumerate(zip(esc["polys"], polys)):
        assert len(got) == len(exp) == 3, f"{who}: round {r} has {len(got)} coefficients"
        for k, (g, e) in enumerate(zip(got, exp)):
            assert g == e, f"{who}: round {r} coefficient {k} differs from the reference kernels' round polynomial: {g} != {e}"
    point = efs(ref["point"].words)
    for i, (g, e) in enumerate(zip(esc["point"], point)):
        assert g == e, f"{who}: point coordinate {i} (most recent first) differs from the reference's sample"
    assert len(esc["point"]) == len(point) == dim
    assert esc["eval"] == final, f"{who}: final evaluation differs from the reference's last round polynomial at the point"
    return L


@pytest.mark.parametrize("name", IDS)
def test_jagged_eval_oracle_vs_reference(name):
    _check(name, _oracle(name)[2], "oracle")
    after = _oracle(name)[5]
    assert (after == _reference(name)["challenger"].words).all(), \
        "oracle: the challenger after the evaluation sumcheck differs from the reference's device challenger"


@pytest.mark.gpu
@pytest.mark.parametrize("name", IDS)
def test_jagged_eval_product_vs_reference(name):
    from sp1_b200 import Lib
    _, _, log_stack, mlr, _ = CASES[IDS.index(name)]
    z_row, st0 = _oracle(name)[:2]
    lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, num_queries=NQ, pow_bits=POW_BITS, batch_pow_bits=BATCH_BITS)
    try:
        handles, claims = [], []
        for tabs in _rounds(name):
            _, h = lib.jagged_commit(tabs)
            handles.append(h)
            claims.append(lib.jagged_column_claims(h, z_row, sum(t.shape[0] for t in tabs)))
        proof = lib.jagged_prove(handles, z_row, np.concatenate(claims), st0.copy())
        for h in handles:
            lib.jagged_round_free(h)
    finally:
        lib.close()
    _check(name, proof, "product")


def test_bp_transition_matches_reference_table():
    """bp_transition (csrc/sumcheck.cuh), compiled for the host, on every (bit state, memory state) pair against the reference's
    TRANSITIONS table as its transition_kernel writes it"""
    from tests import hostcheck_lib

    def run():
        from tests import ref_lib as R
        return R.bp_transitions()
    table = Ref("transitions", run, keep=True, store=STORE).words.reshape(16, 5).astype(np.int64)
    assert (table[:, 4] == 4).all(), "the reference's FAIL state must stay FAIL"
    got = np.zeros(64, np.int32)
    hostcheck_lib.load().sp1b200_hostcheck_bp_transitions(got.ctypes.data_as(C.POINTER(C.c_int32)))
    got = np.where(got.reshape(16, 4) < 0, 4, got.reshape(16, 4))
    for b in range(16):
        for s in range(4):
            assert got[b, s] == table[b, s], (f"bp_transition(row={b >> 3}, index={(b >> 2) & 1}, cur={(b >> 1) & 1}, next={b & 1}, "
                                              f"state={s}) = {got[b, s]}, the reference's TRANSITIONS gives {table[b, s]}")
