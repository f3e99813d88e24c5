"""GPU tests of the shard checks (sp1b200_debug_constraints / sp1b200_debug_interactions) against the restated reference checks
(oracle/debug.hpp), word for word: register-file tiers, calibrated and workload machines, odd heights and height 0, clean traces and
corruptions, crafted fingerprint collisions, the three kinds of main-trace pointer, errors, memory, and a full-size S2c shard."""
import numpy as np
import pytest

from sp1_b200 import synth_air as SA
from sp1_b200.lib import parse_constraint_report, parse_interaction_report
from tests import debug_oracle_lib as DO
from tests import gpu_prove as GP
from tests import machines as M
from tests import oracle_lib as O
from tests.machines import Chip, colliding_keys, constant_key_machine, cross_chip_machine

pytestmark = pytest.mark.gpu
P = O.P

TIER_SPECS = [
    ([(5, 1, False), (0, 2, False), (6, 1, True)], 3),
    ([Chip(512, 6, False, deep=True), Chip(300, 14, True, deep=True), Chip(1024, 28, False, deep=True), Chip(96, 40, False, deep=True),
      (2047, 3, True)], 12),
    ([Chip(192, 250, False, deep=True), Chip(64, 500, True, deep=True), (8191, 3, True), Chip(96, 1000, False, deep=True),
      Chip(600, 300, False, deep=True)], 13),
]


def _lib(mlr):
    from sp1_b200 import Lib
    return Lib(0, max_log_row_count=mlr, log_stacking_height=min(mlr, 21))


def _check(lib, mach, prep_round, blob, heights, mains, preps, pv, max_rows=3, max_keys=16, inter=True):
    dense = M.dense_main(mains)
    got = lib.debug_constraints_words(mach, prep_round, dense, heights, pv, max_rows)
    want_c = want = DO.debug_constraints(blob, heights, mains, preps, pv, max_rows)
    assert got.tolist() == want.tolist(), (parse_constraint_report(got), parse_constraint_report(want))
    if inter:
        got = lib.debug_interactions_words(mach, prep_round, dense, heights, max_keys)
        want = DO.debug_interactions(blob, heights, mains, preps, max_keys)
        assert got.tolist() == want.tolist(), (parse_interaction_report(got), parse_interaction_report(want))
    return parse_constraint_report(want_c)


def _corrupt_cells(rng, mains, n_chips=3):
    live = [k for k, m in enumerate(mains) if m.size]
    for k in rng.choice(live, size=min(n_chips, len(live)), replace=False):
        m = mains[k]
        for _ in range(2):
            c, r = int(rng.integers(0, m.shape[0])), int(rng.integers(0, m.shape[1]))
            m[c, r] = (int(m[c, r]) + 1 + int(rng.integers(0, 1000))) % P


@pytest.mark.parametrize("spec,mlr", TIER_SPECS)
def test_constraint_report_register_tiers(spec, mlr):
    rng = np.random.default_rng(1700 + mlr)
    blob, heights, mains, preps, pv, _ = M.spec_machine(rng, spec, interactions=False)
    lib = _lib(mlr)
    mach = lib.machine_create(blob)
    pr = GP.commit_prep(lib, preps)[1]
    assert _check(lib, mach, pr, blob, heights, mains, preps, pv, inter=False) == {}
    _corrupt_cells(rng, mains)
    assert _check(lib, mach, pr, blob, heights, mains, preps, pv, inter=False)
    # more failing rows than max_rows: a broken column of the widest chip; a changed public value fails every row that loads it
    k = int(np.argmax(heights))
    mains[k][2, :] = (mains[k][2, :].astype(np.uint64) + 1).astype(np.uint32) % P
    rep = _check(lib, mach, pr, blob, heights, mains, preps, pv, max_rows=2, inter=False)
    assert rep[k]["n_failing_rows"] > 2 and len(rep[k]["rows"]) == 2
    pv2 = pv.copy(); pv2[0] = (int(pv2[0]) + 1) % P
    rep = _check(lib, mach, pr, blob, heights, mains, preps, pv2, max_rows=5, inter=False)
    assert all(rep[c]["n_failing_rows"] == heights[c] for c in range(len(heights)) if heights[c])
    if pr is not None:
        lib.jagged_round_free(pr)
    lib.machine_free(mach)
    lib.close()


def test_constraint_report_random_programs():
    """random constraint programs (tests/machines.py random_program) in every register-file tier, a chip without constraints and a
    chip of more than 2^16 main columns: clean -> nothing; one witness cell nudged -> exactly that chip, that row and that constraint's
    alpha index (twice-asserted registers: both); the zero column of a direct leaf assert nudged -> that assert alone; the constant 0 of
    a direct constant assert made 1 -> that assert on every row; the zero public value, which every program loads and one assert
    reads directly, changed -> every row of every constrained chip, with that assert"""
    spec = [M.prog_chip(300, 81, dup=True), M.prog_chip(77, 82, live=10, prep=2), M.prog_chip(64, 83, live=24, n_asserts=16, n_ops=150),
            M.prog_chip(40, 84, n_asserts=0), M.prog_chip(129, 85, live=80, dup=True), M.prog_chip(50, 86, live=300, n_asserts=10),
            M.prog_chip(3, 87, wide=65600, n_asserts=6, n_ops=20), M.prog_chip(0, 88)]
    rng = np.random.default_rng(1750)
    blob, heights, mains, preps, pv, _ = M.spec_machine(rng, spec, interactions=False)
    lib = _lib(9)
    mach = lib.machine_create(blob)
    assert {M.zc_tier(lib.machine_chip_regs(mach, k)) for k in range(len(spec))} == set(range(5))
    pr = GP.commit_prep(lib, preps)[1]
    assert _check(lib, mach, pr, blob, heights, mains, preps, pv, inter=False) == {}
    for k in (0, 2, 4, 5, 6):
        rp = M.random_program(spec[k].program)
        row = int(rng.integers(0, heights[k]))
        w = min(rp.witness, key=lambda x: (x is None, -rp.witness.count(x), rng.random()))   # a twice-asserted one first
        mains[k][w, row] = (int(mains[k][w, row]) + 1) % P
        rep = _check(lib, mach, pr, blob, heights, mains, preps, pv, inter=False)
        alphas = sorted(a for (_, a), w2 in zip(rp.asserts, rp.witness) if w2 == w)
        assert list(rep) == [k] and rep[k]["n_failing_rows"] == 1 and rep[k]["rows"] == {row: alphas}, (k, w, row, rep)
        mains[k][w, row] = (int(mains[k][w, row]) - 1) % P
    # the three direct asserts (leaf, constant 0, zero public value).  On a clean trace each is the zero polynomial, so the zerocheck
    # cannot see whether the lowering kept them; the report can.  The zero column nudged: the leaf assert alone fails
    rp = M.random_program(spec[0].program)
    leaf_alpha, const_alpha, pub_alpha = [a for (_, a), w in zip(rp.asserts, rp.witness) if w is None]
    mains[0][rp.zero_col, 5] = 1
    rep = _check(lib, mach, pr, blob, heights, mains, preps, pv, inter=False)
    assert list(rep) == [0] and rep[0]["rows"] == {5: [leaf_alpha]}, rep
    mains[0][rp.zero_col, 5] = 0
    # the constant 0 made 1 in chip 0's constant table (a blob edit): the constant assert fails on every row, next to the constraints
    # that read the constant elsewhere
    blob2 = blob.copy()
    blob2[1 + 9 + 2 * len(rp.instrs) + 2 * len(rp.leaves)] = O.to_monty(np.array([1]))[0]
    mach2 = lib.machine_create(blob2)
    rep = _check(lib, mach2, pr, blob2, heights, mains, preps, pv, inter=False)
    lib.machine_free(mach2)
    assert list(rep) == [0] and rep[0]["n_failing_rows"] == heights[0] and all(const_alpha in c for c in rep[0]["rows"].values()), rep
    # the zero public value changed, which every program loads: every row of every constrained chip fails, chip 0's public assert too
    pv2 = pv.copy(); pv2[4] = (int(pv2[4]) + 1) % P
    rep = _check(lib, mach, pr, blob, heights, mains, preps, pv2, max_rows=4, inter=False)
    failing = {k for k, s in enumerate(spec) if heights[k] and s.program.n_asserts}
    assert set(rep) == failing and all(rep[k]["n_failing_rows"] == heights[k] for k in failing), rep
    assert all(pub_alpha in c for c in rep[0]["rows"].values()), rep
    if pr is not None:
        lib.jagged_round_free(pr)
    lib.machine_free(mach)
    lib.close()


CALIBRATED = [M.Chip(700, 4, True, 36, 5, 3), M.Chip(96, 14, False, 120, 0, 0, [12, 4, 9, 5]), M.Chip(0, 2, True, 18, 1, 2),
              M.Chip(33, 1, True, 9, 7, 35), M.Chip(2048, 40, False, 360, 2, 0, [9] * 6)]


@pytest.mark.parametrize("case", ["calibrated", "tinyc", "tinyr"])
def test_reports_on_calibrated_and_workload_machines(case):
    rng = np.random.default_rng(1800)
    if case == "calibrated":
        blob, heights, mains, preps, pv, _ = M.spec_machine(rng, CALIBRATED)
        mlr = 11
    else:
        blob, heights, mains, preps, pv, _ = M.workload_machine(case, seed=1801, max_log_rows=12, scale=0.25)
        mlr = 12
    lib = _lib(mlr)
    mach = lib.machine_create(blob)
    pr = GP.commit_prep(lib, preps)[1]
    _check(lib, mach, pr, blob, heights, mains, preps, pv)
    words = lib.debug_interactions_words(mach, pr, M.dense_main(mains), heights)
    assert words.tolist() == [0, 0, 0]
    _corrupt_cells(rng, mains)
    _check(lib, mach, pr, blob, heights, mains, preps, pv)
    if pr is not None:
        lib.jagged_round_free(pr)
    lib.machine_free(mach)
    lib.close()


def _inter_case(blob, heights, mains, preps, max_keys=16, mlr=8):
    lib = _lib(mlr)
    mach = lib.machine_create(blob)
    pr = GP.commit_prep(lib, preps)[1]
    got = lib.debug_interactions_words(mach, pr, M.dense_main(mains), heights, max_keys)
    want = DO.debug_interactions(blob, heights, mains, preps, max_keys)
    if pr is not None:
        lib.jagged_round_free(pr)
    lib.machine_free(mach)
    lib.close()
    assert got.tolist() == want.tolist(), (parse_interaction_report(got), parse_interaction_report(want))
    return parse_interaction_report(want)


def test_interaction_report_cross_chip():
    rng = np.random.default_rng(1900)
    blob, heights, mains, preps = cross_chip_machine(rng, h=200, mult_col_kind4=True)
    assert _inter_case(blob, heights, mains, preps)["n_unbalanced"] == 0
    mains[1][0, 17] = (int(mains[1][0, 17]) + 1) % P                       # one changed value
    _inter_case(blob, heights, mains, preps)
    blob, heights, mains, preps = cross_chip_machine(rng, h=200, mult_col_kind4=True)
    one = int(O.to_monty(np.array([1]))[0])
    r = int(np.nonzero(mains[1][3] == one)[0][0])
    mains[1][3, r] = 0                                                     # one changed multiplicity
    assert _inter_case(blob, heights, mains, preps)["n_unbalanced"] == 2
    mains[0][3, :] = 0                                                     # the sender's multiplicity column zeroed: > max_keys keys
    rep = _inter_case(blob, heights, mains, preps, max_keys=5)
    assert rep["n_unbalanced"] > 5 and len(rep["keys"]) == 5


def _blob_segments(blob):
    """-> (per chip program words, per chip interaction words) of a machine blob"""
    segs = M.chip_segments(blob)
    return [s[2] for s in segs], [s[3] for s in segs]


def _bump_first_receive(iw):
    """interaction words of one chip with the constant of the first receive's first value column + 1"""
    iw = list(iw)
    q = 1
    for _ in range(iw[0]):
        is_send, nv = iw[q], iw[q + 2]
        q += 3
        q += 2 + 3 * iw[q]                                  # multiplicity vcol
        if not is_send and nv:
            iw[q + 1] = (iw[q + 1] + int(O.to_monty(np.array([1]))[0])) % P
            return iw
        for _ in range(nv):
            q += 2 + 3 * iw[q]
    raise ValueError("no receive with a value")


def test_interaction_report_edited_receive():
    """an existing calibrated blob with one receive's virtual-column constant changed"""
    rng = np.random.default_rng(1901)
    blob, heights, mains, preps, pv, _ = M.spec_machine(rng, [M.Chip(300, 2, False, None, 0, 0, [4, 5]), M.Chip(129, 1, True, 9, 0, 1, [9])])
    progs, inters = _blob_segments(blob)
    inters[1] = _bump_first_receive(inters[1])
    blob2 = SA.machine_blob_with_interactions(progs, inters)
    assert blob2.size == blob.size and (blob2 != blob).sum() == 1
    rep = _inter_case(blob2, heights, mains, preps, mlr=9)
    assert rep["n_unbalanced"] > 0 and all(set(k["chips"]) == {1} for k in rep["keys"])


def test_interaction_report_fingerprint_collisions():
    rng = np.random.default_rng(1902)
    A, B = colliding_keys(rng)
    # A sent, B received: two keys (grouping by fingerprint alone would find them balanced)
    blob, heights, mains, preps = constant_key_machine(rng, [[(1, 5, A)], [(0, 5, B)]], [7, 7])
    rep = _inter_case(blob, heights, mains, preps)
    assert rep["n_unbalanced"] == 2
    # A and B each sent and received: nothing
    blob, heights, mains, preps = constant_key_machine(rng, [[(1, 5, A), (1, 5, B)], [(0, 5, B), (0, 5, A)]], [9, 9])
    assert _inter_case(blob, heights, mains, preps)["n_unbalanced"] == 0


def test_pointer_kinds_errors_memory_and_proof_unchanged():
    import torch
    rng = np.random.default_rng(2000)
    spec = [(1024, 2, True), (256 + 32, 3, False), (0, 1, False), (2048, 1, True)]
    blob, heights, mains, preps, pv, names = M.spec_machine(rng, spec, names="Chip{:02d}")
    mains[1][2, 7] = (int(mains[1][2, 7]) + 3) % P
    lib = _lib(11)
    mach = lib.machine_create(blob)
    pr = GP.commit_prep(lib, preps)[1]
    dense = M.dense_main(mains)
    ref_c = lib.debug_constraints_words(mach, pr, dense, heights, pv)
    ref_i = lib.debug_interactions_words(mach, pr, dense, heights)
    assert ref_c.tolist() == DO.debug_constraints(blob, heights, mains, preps, pv).tolist()
    assert ref_i.tolist() == DO.debug_interactions(blob, heights, mains, preps).tolist()
    d = torch.from_numpy(dense.view(np.int32)).cuda()
    pinned = torch.from_numpy(dense.view(np.int32)).pin_memory()
    for src in (d, lib.upload_begin(pinned, 0)):
        assert lib.debug_constraints_words(mach, pr, src, heights, pv).tolist() == ref_c.tolist()
        assert lib.debug_interactions_words(mach, pr, src, heights).tolist() == ref_i.tolist()
    # errors: capacity, mismatched preprocessed round; the context stays usable
    from sp1_b200.lib import Sp1B200Error
    with pytest.raises(Sp1B200Error, match="capacity"):
        lib.debug_constraints_words(mach, pr, dense, heights, pv, cap_words=2)
    with pytest.raises(Sp1B200Error, match="capacity"):
        lib.debug_interactions_words(mach, pr, dense, heights, cap_words=2)
    with pytest.raises(Sp1B200Error, match="preprocessed"):
        lib.debug_constraints_words(mach, None, dense, heights, pv)
    with pytest.raises(Sp1B200Error, match="preprocessed"):
        lib.debug_interactions_words(mach, None, dense, heights)
    assert lib.debug_constraints_words(mach, pr, dense, heights, pv).tolist() == ref_c.tolist()
    # repeated calls: device memory in use stays flat after the first
    used = []
    for _ in range(4):
        lib.debug_constraints_words(mach, pr, dense, heights, pv); lib.debug_interactions_words(mach, pr, dense, heights)
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info(0)
        used.append(total - free)
    assert max(used[1:]) - min(used[1:]) < (8 << 20), used
    # a proof after either check equals the proof without it (clean trace)
    mains[1][2, 7] = (int(mains[1][2, 7]) - 3) % P
    dense = M.dense_main(mains)
    proofs = []
    for pre in (None, "c", "i"):
        if pre == "c":
            assert lib.debug_constraints_words(mach, pr, dense, heights, pv).tolist() == [0]
        if pre == "i":
            assert lib.debug_interactions_words(mach, pr, dense, heights).tolist() == [0, 0, 0]
        st = O.Challenger().st.copy()
        proofs.append(GP.prove(lib, mach, pr, mains, heights, names, pv, st))
    assert all((p_.size == proofs[0].size and (p_ == proofs[0]).all()) for p_ in proofs)
    lib.jagged_round_free(pr)
    lib.machine_free(mach)
    lib.close()


def _write_cell(dense, cell, value):
    """a torch write into a trace the library reads next: the library runs on its own stream, so the write must have finished"""
    import torch
    dense[cell] = value
    torch.cuda.current_stream(dense.device).synchronize()


def test_full_size_s2c_shard():
    """one full-size S2c shard built on the device: clean -> both reports empty; one corrupted cell -> that (chip, row) with the
    constraints the oracle finds for that row alone; one chip's receive made unbalanced in the blob -> the oracle's report for that chip"""
    from sp1_b200 import Lib
    from sp1_b200 import workload as W
    from tools.device_traces import device_traces
    mach_d = W.synthetic_machine("S2c", seed=42)
    specs, blob = mach_d["specs"], mach_d["blob"]
    heights = [sp.h for sp in specs]
    dense, d_prep, prep_rows, prep_cols = device_traces(specs, M.PV0, lambda i: 500 + i, 0)
    wd = M.widths(blob)

    def chip_table(d, k, side):
        """chip k's main (side 0) or preprocessed (side 1) table on the device, [cols, rows]"""
        off = sum(h * w[side] for h, w in zip(heights[:k], wd[:k]))
        return d[off:off + heights[k] * wd[k][side]].view(-1, heights[k])

    def host(t):
        return np.ascontiguousarray(t.cpu().numpy().view(np.uint32))
    pv = M.PV
    lib = Lib(0)
    mach = lib.machine_create(blob)
    pr = lib.jagged_commit_dense(d_prep, prep_rows, prep_cols)[1] if d_prep is not None else None
    assert lib.debug_constraints_words(mach, pr, dense, heights, pv).tolist() == [0]
    assert lib.debug_interactions_words(mach, pr, dense, heights).tolist() == [0, 0, 0]
    k = int(np.argmax(heights)); row = heights[k] - 5
    cell = sum(h * w[0] for h, w in zip(heights[:k], wd[:k])) + 2 * heights[k] + row
    _write_cell(dense, cell, int((int(dense[cell].item()) + 1) % P))
    rep = parse_constraint_report(lib.debug_constraints_words(mach, pr, dense, heights, pv))
    one_row = host(chip_table(dense, k, 0)[:, row:row + 1])
    prep_row = host(chip_table(d_prep, k, 1)[:, row:row + 1]) if wd[k][1] else None
    # the oracle on chip k's row alone (a one-chip machine with that chip's program)
    alone = DO.debug_constraints(SA.machine_blob([M.chip_segments(blob)[k][2]]), [1], [one_row], [prep_row], pv)
    want = parse_constraint_report(alone)
    assert list(rep) == [k] and rep[k]["n_failing_rows"] == 1 and rep[k]["rows"] == {row: want[0]["rows"][0]}
    _write_cell(dense, cell, int((int(dense[cell].item()) - 1) % P))
    # one chip's receive made unbalanced in the blob (the smallest chip with interactions, so that the oracle runs on it alone)
    progs, inters = _blob_segments(blob)
    c = min((i for i in range(len(specs)) if heights[i] and inters[i][0]), key=lambda i: heights[i])
    inters2 = list(inters); inters2[c] = _bump_first_receive(inters[c])
    mach2 = lib.machine_create(SA.machine_blob_with_interactions(progs, inters2))
    got = parse_interaction_report(lib.debug_interactions_words(mach2, pr, dense, heights, max_keys=1 << 17))
    lib.machine_free(mach2)
    prep_c = host(chip_table(d_prep, c, 1)) if wd[c][1] else None
    want = parse_interaction_report(DO.debug_interactions(SA.machine_blob_with_interactions([progs[c]], [inters2[c]]), [heights[c]],
                                                         [host(chip_table(dense, c, 0))], [prep_c], max_keys=1 << 17))
    # the same unbalanced keys and nets; chip c carries the whole net.  A key can also occur (balanced) in other chips - the synthetic
    # traces share small values such as 0 between chips - and those chips are listed with net 0, possibly as the first occurrence.
    assert 0 < want["n_unbalanced"] == got["n_unbalanced"] == len(want["keys"]) == len(got["keys"])
    by_key = lambda rep: {(k["kind"], tuple(k["values"])): k for k in rep["keys"]}
    g_, w_ = by_key(got), by_key(want)
    assert set(g_) == set(w_)
    for key, w in w_.items():
        g = g_[key]
        assert g["net"] == w["net"] and g["chips"][c] == w["net"] and all(x == 0 for ch, x in g["chips"].items() if ch != c)
        if set(g["chips"]) == {c}:
            assert g["first"] == (c,) + w["first"][1:]
    lib.jagged_round_free(pr) if pr is not None else None
    lib.machine_free(mach)
    lib.close()
