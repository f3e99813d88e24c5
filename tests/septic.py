"""Python restatement of the core-proof verifier's septic arithmetic in canonical integers: the extension F_p[z]/(z^7 - 3z - 5), the
curve y^2 = x^3 + 45x + 41z^3, its constant points and SepticDigest addition; Montgomery-word conversions; and the library's host
code for it (libsp1b200_hostcheck.so)."""
import ctypes as C

import numpy as np

from tests import hostcheck_lib

P = 0x7F000001
R_INV = pow(1 << 32, P - 2, P)


def smul(a, b):
    t = [0] * 13
    for i in range(7):
        for j in range(7):
            t[i + j] = (t[i + j] + a[i] * b[j]) % P
    r = t[:7]
    for i in range(7, 13):
        r[i - 7] = (r[i - 7] + 5 * t[i]) % P
        r[i - 6] = (r[i - 6] + 3 * t[i]) % P
    return r


def spow(a, e):
    r, b = [1, 0, 0, 0, 0, 0, 0], a
    while e:
        if e & 1:
            r = smul(r, b)
        b = smul(b, b)
        e >>= 1
    return r


def sinv(a):
    return spow(a, P ** 7 - 2)


def sadd(a, b):
    return [(x + y) % P for x, y in zip(a, b)]


def ssub(a, b):
    return [(x - y) % P for x, y in zip(a, b)]


def curve_add(p, q):
    """SepticCurve::add_incomplete; None on the exceptional case"""
    dx = ssub(q[0], p[0])
    if not any(dx):
        return None
    s = smul(ssub(q[1], p[1]), sinv(dx))
    x = ssub(ssub(smul(s, s), p[0]), q[0])
    y = ssub(smul(s, ssub(p[0], x)), p[1])
    return (x, y)


def curve_neg(p):
    return (p[0], [(-v) % P for v in p[1]])


def on_curve(p):
    x, y = p
    rhs = sadd(sadd(smul(smul(x, x), x), [45 * v % P for v in x]), [0, 0, 0, 41, 0, 0, 0])
    return smul(y, y) == rhs


def multiples(base, k):
    """[base, 2 base, ..., k base]: the doubling by the tangent, slope (3x^2 + 45) / 2y, then incomplete additions"""
    x, y = base
    s = smul(sadd(smul([3, 0, 0, 0, 0, 0, 0], smul(x, x)), [45, 0, 0, 0, 0, 0, 0]), sinv(sadd(y, y)))
    x2 = ssub(ssub(smul(s, s), x), x)
    out = [base, (x2, ssub(smul(s, ssub(x, x2)), y))]
    while len(out) < k:
        out.append(curve_add(out[-1], base))
    return out[:k]


ZERO = ([0x1414213, 0x5623730, 0x9504880, 0x1688724, 0x2096980, 0x7856967, 0x1875376],
        [2020310104, 1513506566, 1843922297, 2003644209, 805967281, 1882435203, 1623804682])
START = ([0x1732050, 0x8075688, 0x7729352, 0x7446341, 0x5058723, 0x6694280, 0x5253810],
         [1095433104, 7540207, 1124564165, 2035506693, 11121645, 102781365, 398772161])
DUMMY = ([0x2718281 + (1 << 24), 0x8284590, 0x4523536, 0x0287471, 0x3526624, 0x9775724, 0x7093699],
         [1250555984, 1592495468, 656721246, 420301347, 2125819749, 819876460, 17687681])


def digest_add(a, b):
    """SepticDigest + SepticDigest (septic_digest.rs:67-83)"""
    s = curve_add(START, a)
    s = s and curve_add(s, curve_neg(ZERO))
    s = s and curve_add(s, b)
    s = s and curve_add(s, curve_neg(ZERO))
    s = s and curve_add(s, ZERO)
    return s and curve_add(s, curve_neg(START))


def mont(v):
    return np.array([(x << 32) % P for x in v], np.uint32)


def canon(w):
    return [int(x) * R_INV % P for x in w]


def pt_words(p):
    return np.concatenate([mont(p[0]), mont(p[1])])


def words_pt(w):
    return (canon(w[:7]), canon(w[7:14]))


# ---- the library's host code ------------------------------------------------------------------------------------------------------
def lib():
    L = hostcheck_lib.load()
    L.sp1b200_hostcheck_septic_digest_add.restype = C.c_int
    return L


def ptr(a):
    return C.c_void_p(a.ctypes.data)
