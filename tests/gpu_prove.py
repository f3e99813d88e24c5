"""How the tests drive the library to prove a shard: commit the preprocessed tables and prove from numpy main traces; and the jagged
PCS parity harness.  Full-size traces on the device come from tools/device_traces.py."""
import numpy as np

from tests import machines as M
from tests import oracle_lib as O


def commit_prep(lib, preps):
    """commit the chips' preprocessed tables (preps[k] None for a chip without them) -> (commitment, round).  A machine without any
    preprocessed table has no round (None) and the zero commitment, the one its verifying key holds."""
    tabs = [p for p in preps if p is not None]
    return lib.jagged_commit(tabs) if tabs else (np.zeros(8, np.uint32), None)


def prove(lib, mach, prep_round, mains, heights, names, pv, state, replay=None):
    """Lib.prove_shard on numpy main traces; state: the challenger, updated in place"""
    return lib.prove_shard(mach, prep_round, M.dense_main(mains), heights, names, pv, state, replay=replay)


def check_jagged(shapes_rounds, log_stack, max_log_rows, seed, nq=8, pow_bits=4, batch_bits=2, between=None):
    """jagged PCS on random tables of the given (rows, cols) shapes per round: every commitment, column claim and proof word and the
    final challenger state equal the oracle's.  between(lib): called before every call into the library and once after the proof"""
    between = between or (lambda lib: None)
    from sp1_b200 import Lib
    rng = np.random.default_rng(seed)
    rounds = [O.random_tables(rng, s) for s in shapes_rounds]
    z_row = O.rand_field(rng, (max_log_rows, 4))
    ch = O.Challenger()
    ch.observe(O.rand_field(rng, 3))
    och = ch.clone()
    ocommits, oclaims, oproof = O.jagged_prove_verify(rounds, log_stack, max_log_rows, z_row, och, num_queries=nq,
                                                      pow_bits=pow_bits, batch_pow_bits=batch_bits)
    lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=max_log_rows, num_queries=nq, pow_bits=pow_bits,
              batch_pow_bits=batch_bits)
    handles, claims = [], []
    for i, tabs in enumerate(rounds):
        between(lib)
        commit, h = lib.jagged_commit(tabs)
        assert (commit == ocommits[i]).all(), f"round {i} jagged commitment differs"
        handles.append(h)
        between(lib)
        claims.append(lib.jagged_column_claims(h, z_row, sum(t.shape[0] for t in tabs)))
    claims = np.concatenate(claims)
    assert (claims == oclaims).all(), "column claims differ"
    st = ch.st.copy()
    between(lib)
    proof = lib.jagged_prove(handles, z_row, claims, st)
    between(lib)
    assert proof.size == oproof.size, (proof.size, oproof.size)
    bad = np.nonzero(proof != oproof)[0]
    assert bad.size == 0, f"first differing proof words {bad[:8]} of {proof.size}"
    assert (st == och.st).all()
    for h in handles:
        lib.jagged_round_free(h)
    lib.close()
