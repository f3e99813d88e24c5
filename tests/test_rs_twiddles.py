"""CPU check of the RS-encode kernels' per-pass twiddle table (sp1_b200/csrc/rs_twiddles.cuh), built on the host by the same source the
device builder runs: entry 2^(s-3) + low of a radix-8 pass with a 2^s-point top stage holds wA[0..3], wB[0..1], wC and a zero, the
powers of the two-adic generator w = 3^127 that the passes used to gather from TH (TH[i] = w^(i 2^12))."""
import ctypes as C

import numpy as np

from tests import oracle_lib as O

P = O.P
W = pow(3, 127, P)          # canonical generator of the 2^24-th roots of unity


def _table():
    from tests import hostcheck_lib as H
    L = H.load()
    L.sp1b200_hostcheck_rs_tw8.restype = C.c_uint32
    out = np.zeros(512 * 8, np.uint32)
    n = L.sp1b200_hostcheck_rs_tw8(out.ctypes.data_as(O.u32p))
    assert n == out.size
    return out.reshape(512, 8)


def _th(i):
    """TH[i] as a canonical value"""
    return pow(W, i << 12, P)


def test_generator_has_order_two_to_the_24():
    assert pow(W, 1 << 23, P) == P - 1 and pow(W, 1 << 24, P) == 1


def test_per_pass_table_matches_the_th_gathers():
    got = O.from_monty(_table()).astype(np.int64)
    assert (got[:2] == 0).all()                      # entries 0 and 1 are unused
    for s in range(4, 12):
        stride = 1 << (s - 3)
        for low in range(stride):
            exp = [_th((j * stride + low) << (12 - s)) for j in range(4)]
            exp += [_th((j * stride + low) << (13 - s)) for j in range(2)]
            exp += [_th(low << (14 - s)), 0]
            assert got[stride + low].tolist() == exp, (s, low)


def test_table_words_are_canonical_montgomery():
    t = _table()
    assert (t < P).all()
    assert (O.to_monty(O.from_monty(t)) == t).all()
