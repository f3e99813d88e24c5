"""How the tests drive the library to prove a shard: commit the preprocessed tables and prove from numpy main traces; and the parity
harnesses that several test modules share (stacked BaseFold, jagged PCS, LogUp-GKR, zerocheck).  Full-size traces on the device come
from tools/device_traces.py."""
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


def check_jagged(shapes_rounds, log_stack, max_log_rows, seed, nq=8, pow_bits=4, batch_bits=2, between=None, kind=None):
    """jagged PCS on random tables of the given (rows, cols) shapes per round: every commitment, column claim and proof word and the
    final challenger state equal the oracle's.  between(lib): called before every call into the library and once after the proof.
    kind: the word kind (O.words) of the tables and of z_row; None: uniform"""
    between = between or (lambda lib: None)
    from sp1_b200 import Lib
    rng = np.random.default_rng(seed)
    rounds = [O.random_tables(rng, s, kind) for s in shapes_rounds]
    z_row = O.words(rng, (max_log_rows, 4), kind)
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


JK_MAX = 5   # the most jagged sumcheck rounds summed straight from the base-field trace (sp1_b200/csrc/jagged.cu)


def trace_rounds_k(shapes_rounds, log_stack, mlr):
    """K as sp1b200_jagged_prove picks it: the column heights of all rounds, dummy padding columns included (jagged_commit)"""
    heights, S, R = [], 1 << log_stack, 1 << mlr
    for shapes in shapes_rounds:
        area = 0
        for rows, cols in shapes:
            heights += [rows] * cols
            area += rows * cols
        padded = max(-(-area // S) * S, S)
        added = padded - area
        added_cols = max(-(-added // R), 1)
        heights += [R] * (added_cols - 1) + [added - (added_cols - 1) * R]
    prefix, s = [], 0
    for h in heights:
        s += h
        prefix.append(s)
    lm = (s - 1).bit_length()
    k = min(JK_MAX, log_stack, lm - 1, min(10, mlr))
    for p in prefix:
        if p:
            k = min(k, (p & -p).bit_length() - 1)
    return k


def check_stacked(ncols_rounds, log_h, nq, pow_bits, batch_bits, seed, keep_codeword=True, device_input=False, kind=None):
    """stacked commit + BaseFold evaluation proof on random rounds of 2^log_h rows: every commitment, proof word and the final
    challenger state equal the oracle's, and a second context replaying the proof's grinding witnesses gives the same proof.  kind: the
    word kind (O.words) of the columns and of the evaluation point's coordinates (a coordinate whose four words are all zero gets the
    word p - 1 in its first limb: BaseFold divides the claim by each coordinate, so a zero lies outside the protocol and the oracle
    rejects it); None: uniform"""
    from sp1_b200 import Lib
    rng = np.random.default_rng(seed)
    rounds = [O.words(rng, (c, 1 << log_h), kind) for c in ncols_rounds]
    extra = max(1, int(np.ceil(np.log2(sum(ncols_rounds)))))
    point = O.words(rng, (extra + log_h, 4), kind)
    if kind is not None:
        point[(point == 0).all(axis=1), 0] = O.P - 1
    ch = O.Challenger()
    ch.observe(O.rand_field(rng, 5))
    och = ch.clone()
    ocommits, oproof = O.stacked_prove_verify(rounds, log_h, point, och, num_queries=nq, pow_bits=pow_bits,
                                              batch_pow_bits=batch_bits)
    lib = Lib(0, log_stacking_height=log_h, num_queries=nq, pow_bits=pow_bits, batch_pow_bits=batch_bits)
    handles, keep = [], []
    for i, r in enumerate(rounds):
        src = r
        if device_input:
            import torch
            src = torch.from_numpy(r.view(np.int32)).cuda()
            torch.cuda.synchronize()
            keep.append(src)
        commit, h = lib.stacked_commit(src, r.shape[0], keep_codeword=keep_codeword)
        assert (commit == ocommits[i]).all(), f"round {i} commitment differs"
        handles.append(h)
    st = ch.st.copy()
    proof = lib.stacked_prove(handles, point, st)
    assert proof.size == oproof.size, (proof.size, oproof.size)
    bad = np.nonzero(proof != oproof)[0]
    assert bad.size == 0, f"first differing proof word {bad[:5]} of {proof.size}"
    assert (st == och.st).all()
    # replay mode: same witnesses -> same proof
    nev = sum(ncols_rounds) * 4
    pow_w, batch_w = proof[-nev - 2], proof[-nev - 1]
    lib2 = Lib(0, log_stacking_height=log_h, num_queries=nq, pow_bits=pow_bits, batch_pow_bits=batch_bits, grind_mode=1)
    hs2 = [lib2.stacked_commit(r, r.shape[0])[1] for r in rounds]
    st2 = ch.st.copy()
    proof2 = lib2.stacked_prove(hs2, point, st2, replay=[batch_w, pow_w])
    assert (proof2 == oproof).all() and (st2 == och.st).all()
    for h in handles:
        lib.commit_free(h)
    for h in hs2:
        lib2.commit_free(h)
    lib.close(); lib2.close()


def upload(mains, preps):
    """per chip device tensors of the main and preprocessed traces (None for a chip without preprocessed columns)"""
    import torch
    d_mains = [torch.from_numpy(np.ascontiguousarray(m).view(np.int32)).cuda() for m in mains]
    d_preps = [torch.from_numpy(np.ascontiguousarray(p).view(np.int32)).cuda() if p is not None else None for p in preps]
    torch.cuda.synchronize()
    return d_mains, d_preps


def check_gkr(lib, mach, blob, heights, mains, preps, mlr, seed, pow_bits=4):
    """Lib.logup_gkr from a random transcript state drawn from `seed`: every proof word and the final challenger state equal the
    oracle's"""
    rng = np.random.default_rng(seed)
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 4))
    och = ch.clone()
    owords = O.gkr_prove_verify(blob, heights, mains, preps, mlr, och, gkr_pow_bits=pow_bits)
    d_mains, d_preps = upload(mains, preps)
    st = ch.st.copy()
    words = lib.logup_gkr(mach, heights, d_mains, d_preps, st)
    assert words.size == owords.size and (words == owords).all(), M.first_diff(words, owords, "LogUp-GKR proof")
    assert (st == och.st).all(), "final challenger state differs from the oracle"


def check_zerocheck(lib, mach, rng, blob, heights, mains, preps, pv, mlr):
    """Lib.zerocheck at a random GKR point from a random transcript state, both drawn from rng: every proof word and the final
    challenger state equal the oracle's"""
    gp, st0, openings, owords, ost = M.oracle_zerocheck(rng, blob, heights, mains, preps, pv, mlr)
    words, st = M.product_zerocheck(lib, mach, heights, mains, preps, pv, gp, st0, openings)
    assert words.size == owords.size, (words.size, owords.size)
    bad = np.nonzero(words != owords)[0]
    assert bad.size == 0, f"first differing words {bad[:8]} of {words.size}"
    assert (st == ost).all()
