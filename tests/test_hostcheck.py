"""CPU tests of the DEVICE arithmetic sources compiled for the host (sp1_b200/csrc/hostcheck.cu): the exact
kb31.cuh / poseidon2.cuh code the kernels run, checked against the oracle on the CPU box (edge values included)."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O


def _L():
    from tests import hostcheck_lib as H
    return H.load()


def _edge_states(rng, n):
    st = O.rand_field(rng, (n, 16))
    st[0] = 0
    st[1] = O.P - 1            # largest canonical Montgomery word in every lane
    st[2] = 1
    st[3, ::2] = O.P - 1
    st[4, 0] = O.P - 1
    return st


def test_device_poseidon2_source_on_host_matches_oracle():
    rng = np.random.default_rng(5)
    st = _edge_states(rng, 400)
    exp = np.stack([O.permute(s) for s in st])
    got = st.copy()
    _L().sp1b200_hostcheck_permute(got.ctypes.data_as(O.u32p), C.c_uint64(got.shape[0]))
    assert (got == exp).all()
    assert (got < O.P).all()   # canonical outputs


@pytest.mark.parametrize("mode", [-1] + list(range(16)) + [19, 21, 23])
def test_every_permutation_mode_on_host_matches_oracle(mode):
    """permute_m<MODE> (s-box reduction form, pipe placement of the additions) computes the same words as the oracle; -1 = the round-1 code"""
    rng = np.random.default_rng(50 + mode)
    st = _edge_states(rng, 300)
    exp = np.stack([O.permute(s) for s in st])
    got = st.copy()
    assert _L().sp1b200_hostcheck_permute_mode(got.ctypes.data_as(O.u32p), C.c_uint64(got.shape[0]), C.c_int(mode)) == 1
    assert (got == exp).all() and (got < O.P).all()


def test_device_field_and_ext_sources_on_host():
    rng = np.random.default_rng(6)
    n = 2000
    a, b = O.rand_field(rng, n), O.rand_field(rng, n)
    a[:4] = [0, O.P - 1, 1, O.P - 1]
    b[:4] = [0, O.P - 1, O.P - 1, 0]
    add, sub, mul = (np.zeros(n, np.uint32) for _ in range(3))
    _L().sp1b200_hostcheck_field(a.ctypes.data_as(O.u32p), b.ctypes.data_as(O.u32p), add.ctypes.data_as(O.u32p),
                                 sub.ctypes.data_as(O.u32p), mul.ctypes.data_as(O.u32p), C.c_uint64(n))
    L = O.lib()
    for i in range(n):
        assert add[i] == L.orc_add(int(a[i]), int(b[i]))
        assert sub[i] == L.orc_sub(int(a[i]), int(b[i]))
        assert mul[i] == L.orc_mul(int(a[i]), int(b[i]))
    x, y = O.rand_field(rng, (300, 4)), O.rand_field(rng, (300, 4))
    x[0] = O.P - 1
    y[0] = O.P - 1
    out = np.zeros((300, 4), np.uint32)
    _L().sp1b200_hostcheck_ext_mul(x.ctypes.data_as(O.u32p), y.ctypes.data_as(O.u32p), out.ctypes.data_as(O.u32p), C.c_uint64(300))
    inv = np.zeros((300, 4), np.uint32)
    _L().sp1b200_hostcheck_ext_inv(x.ctypes.data_as(O.u32p), inv.ctypes.data_as(O.u32p), C.c_uint64(300))
    e = np.zeros(4, np.uint32)
    for i in range(300):
        L.orc_ext_mul(O.ptr(x[i]), O.ptr(y[i]), O.ptr(e))
        assert (out[i] == e).all()
        L.orc_ext_inv(O.ptr(x[i]), O.ptr(e))
        assert (inv[i] == e).all()


def _check_lowering(chip_words, main_w, prep_w, n_constraints, seed, window=24):
    rng = np.random.default_rng(seed)
    cw = np.array(chip_words, dtype=np.uint32)
    out = np.zeros(12, np.uint32)
    nl = C.c_uint32(0)
    regs = None
    for _ in range(6):
        main_row = O.rand_field(rng, max(main_w, 1))
        prep_row = O.rand_field(rng, max(prep_w, 1))
        pv = O.rand_field(rng, 8)
        ap = O.rand_field(rng, (max(n_constraints, 1), 4))
        regs = _L().sp1b200_hostcheck_zc_lower(cw.ctypes.data_as(O.u32p), main_row.ctypes.data_as(O.u32p), prep_row.ctypes.data_as(O.u32p),
                                               pv.ctypes.data_as(O.u32p), ap.ctypes.data_as(O.u32p), C.c_uint32(window),
                                               out.ctypes.data_as(O.u32p), C.byref(nl))
        assert regs > 0
        assert (out[:4] == out[4:8]).all()
        assert (out[:4] == out[8:12]).all()     # ... and as a sum of self-contained pieces
        assert out[:4].any()          # random rows do not satisfy the constraints: a non-trivial comparison
    return regs, nl.value


def test_constraint_lowering_preserves_the_row_polynomial():
    """zc_lower (re-scheduling for the shared-memory register file) vs the bytecode as given, same row, same alpha powers"""
    from sp1_b200 import synth_air as SA
    for groups, wp in [(1, False), (3, True), (7, False), (41, True)]:
        words, main_w, prep_w = SA.synth_chip(groups, wp)
        n_constraints = words[2]
        for window in (0, 4, 24, 10_000):
            regs, _ = _check_lowering(words, main_w, prep_w, n_constraints, seed=groups + window, window=window)
            # SSA input: one register per instruction; lowered: a handful regardless of the chip's size
            assert regs <= 16, (groups, wp, window, regs)


def test_constraint_lowering_pressure_tracks_live_values():
    """deep programs (all products first, consumed in reverse): the lowered pressure follows the live set, results unchanged"""
    from sp1_b200 import synth_air as SA
    for groups in (6, 14, 28, 40):
        words, main_w, prep_w = SA.synth_chip(groups, False, deep=True)
        regs, _ = _check_lowering(words, main_w, prep_w, words[2], seed=groups)
        assert groups <= regs <= groups + 8, (groups, regs)


def test_constraint_lowering_handles_register_reuse_dead_code_and_leaf_asserts():
    from sp1_b200 import synth_air as SA
    a = SA.Asm()
    x = a.leaf(SA.LEAF_MAIN, 0)
    y = a.leaf(SA.LEAF_MAIN, 1)
    k = a.const(5)
    t = a.op(SA.MUL, x, y)
    dead = a.op(SA.ADD, t, k)                       # never asserted
    u = a.op(SA.SUB, t, k)
    a.assert_zero(u)
    a.assert_zero(x)                                # assert directly on a leaf
    v = a.op(SA.NEG, u)
    a.assert_zero(v)
    a.assert_zero(u)                                # the same value under a second alpha power
    # overwrite a register in place (non-SSA): reg[t] = reg[t] * reg[y]; assert it
    a.instrs.append((SA.MUL, t, t, y))
    a.assert_zero(t)
    words = a.words(2, 0)
    regs, n_low = _check_lowering(words, 2, 0, words[2], seed=99, window=2)
    assert regs <= 4
    assert dead >= 0


def _ext_eval(coeffs, x):
    """Horner with the oracle's ext arithmetic"""
    L = O.lib()
    acc = np.zeros(4, np.uint32)
    tmp = np.zeros(4, np.uint32)
    for c in coeffs[::-1]:
        L.orc_ext_mul(O.ptr(acc), O.ptr(np.ascontiguousarray(x)), O.ptr(tmp))
        acc = ((tmp.astype(np.uint64) + c) % O.P).astype(np.uint32)
    return acc


def test_host_transcript_arithmetic_matches_oracle():
    """hostfield.hpp's E4 over kb31.cuh (the library's host transcript math): ext product / inverse vs the oracle, and the batched-inversion Lagrange
    interpolation through 3, 4 and 5 nodes reproduces the node values"""
    rng = np.random.default_rng(8)
    n = 200
    a, b = O.rand_field(rng, (n, 4)), O.rand_field(rng, (n, 4))
    a[0] = O.P - 1; b[0] = O.P - 1; a[1] = [1, 0, 0, 0]
    mul, inv = np.zeros((n, 4), np.uint32), np.zeros((n, 4), np.uint32)
    _L().sp1b200_hostcheck_e4(a.ctypes.data_as(O.u32p), b.ctypes.data_as(O.u32p), mul.ctypes.data_as(O.u32p), inv.ctypes.data_as(O.u32p),
                              C.c_uint64(n))
    e = np.zeros(4, np.uint32)
    for i in range(n):
        O.lib().orc_ext_mul(O.ptr(a[i]), O.ptr(b[i]), O.ptr(e)); assert (mul[i] == e).all()
        O.lib().orc_ext_inv(O.ptr(a[i]), O.ptr(e)); assert (inv[i] == e).all()
    for deg in (3, 4, 5):
        for _ in range(5):
            xs, ys = O.rand_field(rng, (deg, 4)), O.rand_field(rng, (deg, 4))
            xs[0] = 0                                    # the drivers' node sets start with 0 and 1
            xs[1] = [int(O.to_monty(np.array([1]))[0]), 0, 0, 0]
            coeffs = np.zeros((deg, 4), np.uint32)
            assert _L().sp1b200_hostcheck_interpolate(xs.ctypes.data_as(O.u32p), ys.ctypes.data_as(O.u32p), C.c_uint32(deg),
                                                      coeffs.ctypes.data_as(O.u32p)) == 0
            for i in range(deg):
                assert (_ext_eval(coeffs, xs[i]) == ys[i]).all()


def test_constraint_lowering_fuzz():
    """random register-reusing programs (tests/machines.py random_program): the re-scheduled stream and its partition into pieces
    evaluate to the same row polynomial as the bytecode as given; the lowered pressure never exceeds the number of registers the input
    used by much.  Half the programs are satisfiable ones as the GPU tests run them, half need satisfy nothing: 1 to 60 asserts on any
    register at any point, read and overwritten afterwards, direct asserts on loads that ops also read, bodies of 1 to 400 instructions"""
    from tests import machines as M
    rng = np.random.default_rng(2024)
    for it in range(80):
        sat = it % 2 == 0
        prog = M.Prog(2024 + it, n_asserts=int(rng.integers(6, 60)) if sat else int(rng.integers(1, 60)), live=int(rng.integers(0, 40)),
                      cols=int(rng.integers(1, 30)), prep=int(rng.integers(0, 4)), n_ops=int(rng.integers(1, 400)),
                      direct=bool(rng.integers(0, 2)), dup=bool(rng.integers(0, 2)), max_deg=int(rng.integers(1, 4)), sat=sat)
        rp = M.random_program(prog)
        words, main_w, prep_w, n_regs, n_asserts = rp.words, rp.main_w, rp.prep_w, rp.words[3], len(rp.asserts)
        cw = np.array(words, dtype=np.uint32)
        out = np.zeros(12, np.uint32)
        nl = C.c_uint32(0)
        for window in (0, 24):
            mr, pr, pv = O.rand_field(rng, main_w), O.rand_field(rng, max(prep_w, 1)), O.rand_field(rng, 8)
            ap = O.rand_field(rng, (n_asserts, 4))
            regs = _L().sp1b200_hostcheck_zc_lower(cw.ctypes.data_as(O.u32p), mr.ctypes.data_as(O.u32p), pr.ctypes.data_as(O.u32p),
                                                   pv.ctypes.data_as(O.u32p), ap.ctypes.data_as(O.u32p), C.c_uint32(window),
                                                   out.ctypes.data_as(O.u32p), C.byref(nl))
            assert regs > 0, (prog, window)
            assert out[:4].any() or not sat, (prog, window, "random rows do not satisfy the program")   # (x - x can zero a free one)
            assert (out[:4] == out[4:8]).all(), (prog, window, "full stream")
            assert (out[:4] == out[8:12]).all(), (prog, window, "pieces")
            assert regs <= n_regs + 4, (prog, window, regs, n_regs)
