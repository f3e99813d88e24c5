"""Extension-field arithmetic on Montgomery words for the tests that restate the reference's host arithmetic (tests/test_ref_sumcheck.py,
tests/test_ref_gkr.py): oracle multiplication and inversion, the plain addition, and slop_algebra's univariate interpolation."""
import numpy as np

from tests import oracle_lib as O


# ---- extension-field arithmetic on Montgomery words (oracle multiplication and inversion; addition is the plain one) ----------------
class EF:
    __slots__ = ("w",)

    def __init__(self, w):
        self.w = np.ascontiguousarray(w, np.uint32).reshape(4)

    @staticmethod
    def of(n):
        return EF(O.to_monty(np.array([n % O.P, 0, 0, 0])))

    def __add__(self, o):
        return EF((self.w.astype(np.uint64) + o.w) % O.P)

    def __sub__(self, o):
        return EF((self.w.astype(np.uint64) + O.P - o.w) % O.P)

    def __mul__(self, o):
        out = np.zeros(4, np.uint32)
        O.lib().orc_ext_mul(O.ptr(self.w), O.ptr(o.w), O.ptr(out))
        return EF(out)

    def inv(self):
        out = np.zeros(4, np.uint32)
        O.lib().orc_ext_inv(O.ptr(self.w), O.ptr(out))
        return EF(out)

    def __eq__(self, o):
        return bool((self.w == o.w).all())

    def __repr__(self):
        return f"EF({[int(x) for x in O.from_monty(self.w)]})"


ZERO, ONE = EF.of(0), EF.of(1)
HALF, QUARTER = EF.of(2).inv(), EF.of(4).inv()


def interpolate(xs, ys):
    """slop_algebra::interpolate_univariate_polynomial: the coefficients (constant first) of the polynomial of degree < len(xs)"""
    coeffs = [ZERO] * len(xs)
    for i, (xi, yi) in enumerate(zip(xs, ys)):
        num, den = [yi], ONE
        for j, xj in enumerate(xs):
            if j == i:
                continue
            den = den * (xi - xj)
            nxt = [ZERO] * (len(num) + 1)
            for k, c in enumerate(num):
                nxt[k + 1] = nxt[k + 1] + c
                nxt[k] = nxt[k] - c * xj
            num = nxt
        dinv = den.inv()
        coeffs = [a + c * dinv for a, c in zip(coeffs, num)]
    return coeffs


def eval_at(coeffs, x):
    r = ZERO
    for c in reversed(coeffs):
        r = r * x + c
    return r


def efs(words):
    """flat Montgomery words -> a list of EF, four words each"""
    return [EF(w) for w in np.asarray(words, np.uint32).reshape(-1, 4)]


def parse_partial_sumcheck(w, o):
    """one PartialSumcheckProof at word o of a proof (oracle/capi.cpp put): n | per round polynomial {m | m coefficients} | claimed sum |
    point[n] | evaluation.  -> (dict(polys, claim, point, eval), the offset after it)"""
    n = int(w[o]); o += 1
    polys = []
    for _ in range(n):
        m = int(w[o]); o += 1
        polys.append(efs(w[o:o + 4 * m])); o += 4 * m
    claim = EF(w[o:o + 4]); o += 4
    point = efs(w[o:o + 4 * n]); o += 4 * n
    ev = EF(w[o:o + 4]); o += 4
    return dict(polys=polys, claim=claim, point=point, eval=ev), o
