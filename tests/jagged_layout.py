"""The jagged PCS proof words and the dense layout of its tables, shared by the tests that rerun the jagged sumchecks on the reference's own
kernels (tests/test_ref_sumcheck.py, tests/test_ref_jagged_eval.py)."""
import numpy as np

from tests.ext_field import EF, efs, parse_partial_sumcheck


def parse_jagged_proof(w, stacked_cols, log_stack, num_queries, log_blowup):
    """the jagged PCS proof words (oracle/capi.cpp put(JaggedProof)).  stacked_cols: the stacked columns of each commitment round.
    -> dict(batch_evals, sumcheck, eval_sumcheck, rc_cc, expected_eval, log_m): the Hadamard sumcheck and the jagged evaluation sumcheck
    as parse_partial_sumcheck reads them, rc_cc the (rows, cols) of every table of every round, the dummy padding tables included"""
    w = np.asarray(w, np.uint32)
    lh = log_stack + log_blowup
    o = 2 * 4 * log_stack + 8 * log_stack                                 # univariate messages, FRI commitments
    for width in stacked_cols:                                            # component openings
        o += num_queries * width + 8 + 2 + num_queries * lh * 8
    for q in range(log_stack):                                            # query phase
        o += num_queries * 8 + 8 + 2 + num_queries * (lh - q - 1) * 8
    o += 4 + 1 + 1                                                        # final poly, two witnesses
    batch = []
    for width in stacked_cols:
        batch += efs(w[o:o + 4 * width]); o += 4 * width
    sc, o = parse_partial_sumcheck(w, o)
    esc, o = parse_partial_sumcheck(w, o)
    rc_cc = []
    for _ in stacked_cols:
        cnt = int(w[o]); o += 1
        rc_cc.append([(int(w[o + 2 * i]), int(w[o + 2 * i + 1])) for i in range(cnt)]); o += 2 * cnt
    o += 8 * len(stacked_cols)
    expected = EF(w[o:o + 4]); o += 4
    log_m = int(w[o + 1]); o += 2
    assert o == w.size, (o, w.size)
    return dict(batch_evals=batch, sumcheck=sc, eval_sumcheck=esc, rc_cc=rc_cc, expected_eval=expected, log_m=log_m)


def stacked_cols(shapes_rounds, log_stack):
    """the stacked columns of each commitment round of tables (rows, cols)"""
    S = 1 << log_stack
    return [max(-(-sum(r * c for r, c in shapes) // S), 1) for shapes in shapes_rounds]


def dense(rounds, log_stack):
    """the committed words of all rounds back to back, each round zero-padded to a multiple of 2^log_stack (jagged_commit)"""
    parts = []
    S = 1 << log_stack
    for tabs in rounds:
        d = np.concatenate([t.reshape(-1) for t in tabs if t.size] or [np.zeros(0, np.uint32)])
        parts += [d, np.zeros(max(-(-d.size // S) * S, S) - d.size, np.uint32)]
    return np.concatenate(parts)


def column_heights(rc_cc):
    """the height of every column of the jagged layout, dummy padding tables included, as the proof's table sizes record them"""
    return [rows for rc in rc_cc for rows, cols in rc for _ in range(cols)]
