"""CPU tests of the lazily reduced field arithmetic at the ends of its domains: the exact kb31.cuh / septic.cuh / poseidon2.cuh code the
kernels run (compiled for the host by sp1_b200/csrc/hostcheck.cu), against plain Python integers (x * 2^-32 mod p), not the oracle.

The hot kernels sum up to four 32 x 32-bit products in a 64-bit accumulator and reduce once (kb::monty_reduce2, domain x < 2p 2^32).
Four products of canonical words reach 4 (p-1)^2 = 0.992 * 2p 2^32, so the bound holds with less than 1 % margin, and only operands
near the Montgomery word p - 1 come close to it: these tests put exactly those operands through every primitive that reduces lazily."""
import ctypes as C

import numpy as np
import pytest

from tests import septic as S

P = 0x7F000001
R = 1 << 32
R_INV = pow(R, P - 2, P)
ONE = R % P                          # the Montgomery word of 1
W_MAX = P - 1                        # the largest canonical word (the value 0x3FFF0001)
W_THIRD = W_MAX * pow(3, P - 2, P) % P   # 3 * W_THIRD = p - 1 mod p: kb::ext_mul triples b_1..b_3 into the word p - 1
u64p = C.POINTER(C.c_uint64)


def _L():
    from tests import hostcheck_lib as H
    return H.load()


def _u32(a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    return a, a.ctypes.data_as(C.POINTER(C.c_uint32))


def _reduce(xs):
    x = np.ascontiguousarray(np.array(xs, dtype=np.uint64))
    outs = [np.zeros(x.size, np.uint32) for _ in range(3)]
    _L().sp1b200_hostcheck_reduce(x.ctypes.data_as(u64p), *(_u32(o)[1] for o in outs), C.c_uint64(x.size))
    return outs


def _domain_points(rng, hi):
    """inputs of a reduction whose domain is [0, hi): both ends, k 2^32 +- 1, low word 0 and all ones, just below and above p 2^32,
    and a random sample"""
    xs = {0, 1, 2, hi - 1, hi - 2, R - 1, R, R + 1}
    for k in [1, 2, 3, P - 1, P, P + 1, (hi >> 32) - 1, (hi >> 32) - 2, int(rng.integers(1, hi >> 32))]:
        for d in (-1, 0, 1, R - 1):
            xs.add(k * R + d)
    for d in range(-3, 4):
        xs.add(P * R + d)
    xs |= {int(x) for x in rng.integers(0, hi, 4000, dtype=np.uint64)}
    xs |= {int(x) << 32 for x in rng.integers(0, hi >> 32, 200, dtype=np.uint64)}            # low word 0
    xs |= {(int(x) << 32) | (R - 1) for x in rng.integers(0, hi >> 32, 200, dtype=np.uint64)}  # low word 2^32 - 1
    return sorted(x for x in xs if 0 <= x < hi)


@pytest.mark.parametrize("which,hi", [("monty_reduce", P * R), ("monty_reduce2", 2 * P * R), ("monty_reduce_lazy", P * R)])
def test_montgomery_reductions_over_their_whole_domain(which, hi):
    rng = np.random.default_rng({"monty_reduce": 1, "monty_reduce2": 2, "monty_reduce_lazy": 3}[which])
    xs = _domain_points(rng, hi)
    assert xs[-1] == hi - 1 and (P * R - 1) in xs and (hi == P * R or P * R in xs)
    r, r2, rl = _reduce(xs)
    got = {"monty_reduce": r, "monty_reduce2": r2, "monty_reduce_lazy": rl}[which]
    bad = []
    for x, g in zip(xs, got.tolist()):
        want = x * R_INV % P
        ok = (g == want) if which != "monty_reduce_lazy" else (g < 2 * P and g % P == want)
        if not ok:
            bad.append((hex(x), g, want))
    assert not bad, f"{which}: {len(bad)} wrong results, first {bad[:4]}"


def test_mul_takes_any_32_bit_first_operand():
    """kb::mul(a, b) for a < 2^32 and b < p, its stated contract (a b < 2^32 p): canonical a b 2^-32"""
    rng = np.random.default_rng(4)
    a_edge = [0, 1, ONE, P - 2, P - 1, P, P + 1, 2 * P - 1, 2 * P, R - 2, R - 1, 1 << 31, (1 << 31) - 1]
    b_edge = [0, 1, 2, ONE, P - ONE, P - 2, P - 1]
    a = [x for x in a_edge for _ in b_edge] + [int(x) for x in rng.integers(0, R, 3000, dtype=np.uint64)]
    b = [y for _ in a_edge for y in b_edge] + [int(x) for x in rng.integers(P - 64, P, 1000)] + [int(x) for x in rng.integers(0, P, 2000)]
    n = len(a)
    (aa, pa), (bb, pb) = _u32(a), _u32(b)
    outs = [np.zeros(n, np.uint32) for _ in range(3)]
    _L().sp1b200_hostcheck_field(pa, pb, *(_u32(o)[1] for o in outs), C.c_uint64(n))
    mul = outs[2].tolist()
    bad = [(x, y, g) for x, y, g in zip(a, b, mul) if g != x * y * R_INV % P]
    assert not bad, f"{len(bad)} wrong products, first {bad[:4]}"
    assert (R - 1, P - 1) in zip(a, b)


# ---- the degree-4 extension F[x]/(x^4 - 3) ---------------------------------------------------------------------------------------------
def _ext_words_mul(a, b):
    """the product of two extension elements given as Montgomery words, in Python integers -> words"""
    x = [w * R_INV % P for w in a]
    y = [w * R_INV % P for w in b]
    t = [0] * 7
    for i in range(4):
        for j in range(4):
            t[i + j] += x[i] * y[j]
    c = [(t[k] + (3 * t[k + 4] if k < 3 else 0)) % P for k in range(4)]
    return [v * R % P for v in c]


def _ext_cases(rng):
    """(a, b) pairs of extension words: the worst case of kb::ext_mul (a = all p - 1, b = (p - 1, (p-1)/3, (p-1)/3, (p-1)/3), whose
    tripled b_j are all p - 1), all p - 1 on both sides, and mixtures with 0 and ONE"""
    worst_b = [W_MAX, W_THIRD, W_THIRD, W_THIRD]
    vals = [0, ONE, W_MAX, W_THIRD]
    cases = [([W_MAX] * 4, worst_b), (worst_b, [W_MAX] * 4), ([W_MAX] * 4, [W_MAX] * 4), (worst_b, worst_b)]
    for _ in range(400):
        cases.append(([vals[int(k)] for k in rng.integers(0, 4, 4)], [vals[int(k)] for k in rng.integers(0, 4, 4)]))
    for _ in range(100):   # one side extreme, the other uniform
        u = [int(x) for x in rng.integers(0, P, 4)]
        cases += [([W_MAX] * 4, u), (u, worst_b)]
    return cases


def test_ext_mul_and_inv_at_the_accumulator_bound():
    assert 3 * W_THIRD % P == W_MAX and W_THIRD == 0x54AAAAAB
    cases = _ext_cases(np.random.default_rng(5))
    n = len(cases)
    (_, pa), (_, pb) = _u32([a for a, _ in cases]), _u32([b for _, b in cases])
    out = np.zeros((n, 4), np.uint32)
    _L().sp1b200_hostcheck_ext_mul(pa, pb, _u32(out)[1], C.c_uint64(n))
    bad = [(a, b) for (a, b), g in zip(cases, out.tolist()) if g != _ext_words_mul(a, b)]
    assert not bad, f"ext_mul: {len(bad)} wrong products, first {bad[:2]}"
    # the inverse of every non-zero operand: a * inv(a) = 1 in Python integers
    xs = [x for a, b in cases for x in (a, b) if any(x)]
    inv = np.zeros((len(xs), 4), np.uint32)
    (_, px) = _u32(xs)
    _L().sp1b200_hostcheck_ext_inv(px, _u32(inv)[1], C.c_uint64(len(xs)))
    assert (inv < P).all()
    bad = [x for x, v in zip(xs, inv.tolist()) if _ext_words_mul(x, v) != [ONE, 0, 0, 0]]
    assert not bad, f"ext_inv: {len(bad)} wrong inverses, first {bad[:2]}"


# ---- the septic extension F[z]/(z^7 - 3z - 5) ------------------------------------------------------------------------------------------
def _septic_cases(rng):
    """every coefficient at the word p - 1, one coefficient at a time at p - 1 (the rest 0 or uniform), and mixtures with 0 and ONE"""
    cases = [[W_MAX] * 7]
    for k in range(7):
        e = [0] * 7; e[k] = W_MAX
        cases.append(e)
        u = [int(x) for x in rng.integers(0, P, 7)]; u[k] = W_MAX
        cases.append(u)
        m = [W_MAX] * 7; m[k] = 0
        cases.append(m)
    vals = [0, ONE, W_MAX]
    for _ in range(20):
        cases.append([vals[int(k)] for k in rng.integers(0, 3, 7)])
    return cases


def test_septic_mul_and_frobenius_at_the_accumulator_bound():
    rng = np.random.default_rng(6)
    xs = _septic_cases(rng)
    ys = [[W_MAX] * 7] * len(xs)                    # every product against all p - 1 ...
    ys = ys + xs[::-1]                              # ... and against the cases themselves
    xs = xs + xs
    n = len(xs)
    (_, pa), (_, pb) = _u32(xs), _u32(ys)
    mul, inv = np.zeros((n, 7), np.uint32), np.zeros((n, 7), np.uint32)
    S.lib().sp1b200_hostcheck_septic(pa, pb, _u32(mul)[1], _u32(inv)[1], C.c_uint64(n))
    for x, y, g in zip(xs, ys, mul.tolist()):
        assert g == list(S.mont(S.smul(S.canon(x), S.canon(y)))), (x, y)
    for x, g in zip(xs, inv.tolist()):
        if any(x):
            assert S.smul(S.canon(x), S.canon(g)) == [1, 0, 0, 0, 0, 0, 0], x
    half = n // 2
    fr, dfr = np.zeros((half, 7), np.uint32), np.zeros((half, 7), np.uint32)
    _L().sp1b200_hostcheck_septic_frobenius(_u32(xs[:half])[1], _u32(fr)[1], _u32(dfr)[1], C.c_uint64(half))
    for x, f, d in zip(xs[:half], fr.tolist(), dfr.tolist()):
        a = S.canon(x)
        assert f == list(S.mont(S.spow(a, P))), ("frobenius", x)
        assert d == list(S.mont(S.spow(a, P * P))), ("double_frobenius", x)


# ---- the Poseidon2 s-box products ------------------------------------------------------------------------------------------------------
def test_poseidon2_lazy_products_at_their_largest_inputs():
    """mont_lazy (result in (0, 2p)) and mont_wide_lazy ([0, 2p)) for a b just below 2^32 p, operands < 2p included; sbox on canonical
    state words and round constants up to p - 1"""
    rng = np.random.default_rng(7)
    a = [2 * P - 1, 2 * P - 2, 2 * P - 1, P - 1, P - 1, R - 1, R - 1, P, 1, ONE]
    b = [P - 1, P - 1, 2 * P - 2, P - 1, 0, P, P - 1, P - 1, P - 1, W_MAX]
    for x in rng.integers(1, R, 2000, dtype=np.uint64):
        x = int(x)
        a.append(x); b.append(min((P * R - 1) // x, R - 1))     # the largest b with a b < 2^32 p
    for x in rng.integers(P, 2 * P, 500):
        a.append(int(x)); b.append(int(rng.integers(P - 8, 2 * P)))
    keep = [(x, y) for x, y in zip(a, b) if x * y < P * R]
    assert len(keep) > 2000 and (2 * P - 1, P - 1) in keep
    a, b = [x for x, _ in keep], [y for _, y in keep]
    n = len(a)
    outs = [np.zeros(n, np.uint32) for _ in range(3)]
    _L().sp1b200_hostcheck_p2_products(_u32(a)[1], _u32(b)[1], *(_u32(o)[1] for o in outs), C.c_uint64(n))
    lazy, wide = outs[0].tolist(), outs[1].tolist()
    for x, y, g, w in zip(a, b, lazy, wide):
        want = x * y * R_INV % P
        assert 0 < g < 2 * P and g % P == want, ("mont_lazy", x, y, g)
        assert 0 <= w < 2 * P and w % P == want, ("mont_wide_lazy", x, y, w)
    # sbox(s, rc) = (s + rc)^3 for canonical words s and rc
    s = [W_MAX, W_MAX, 0, W_MAX, P - 2, ONE, P - ONE] + [int(x) for x in rng.integers(P - 16, P, 300)] + [int(x) for x in rng.integers(0, P, 300)]
    rc = [W_MAX, 0, W_MAX, 1, 1, P - ONE, ONE] + [int(x) for x in rng.integers(P - 16, P, 300)] + [int(x) for x in rng.integers(0, P, 300)]
    n = len(s)
    outs = [np.zeros(n, np.uint32) for _ in range(3)]
    _L().sp1b200_hostcheck_p2_products(_u32(s)[1], _u32(rc)[1], *(_u32(o)[1] for o in outs), C.c_uint64(n))
    for x, y, g in zip(s, rc, outs[2].tolist()):
        v = (x + y) % P
        assert g == v * v % P * v % P * R_INV % P * R_INV % P, ("sbox", x, y, g)
