"""CPU tests of the core-proof verifier's host arithmetic (sp1_b200/csrc/septic.hpp, through libsp1b200_hostcheck.so): the septic
extension F_p[z]/(z^7 - 3z - 5), the curve y^2 = x^3 + 45x + 41z^3 and SepticDigest addition, against a Python restatement in
canonical integers; and the PublicValues word offsets of sp1_b200.lib.PV against the struct's field list."""
import ctypes as C

import numpy as np
import pytest

from tests import hostcheck_lib

P = 0x7F000001
R_INV = pow(1 << 32, P - 2, P)

# ---- Python restatement (canonical integers) ---------------------------------------------------------------------------------------


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


def _lib():
    L = hostcheck_lib.load()
    L.sp1b200_hostcheck_septic_digest_add.restype = C.c_int
    return L


def _p(a):
    return C.c_void_p(a.ctypes.data)


def test_constant_points_are_on_the_curve():
    for p in (ZERO, START, DUMMY):
        assert on_curve(p)
    out = np.zeros(42, np.uint32)
    _lib().sp1b200_hostcheck_septic_constants(_p(out))
    for i, p in enumerate((ZERO, START, DUMMY)):
        assert words_pt(out[14 * i:14 * i + 14]) == (p[0], p[1])


def test_septic_mul_and_inverse_match_the_restatement():
    rng = np.random.default_rng(7)
    n = 24
    a = [[int(x) for x in rng.integers(0, P, 7)] for _ in range(n)]
    b = [[int(x) for x in rng.integers(0, P, 7)] for _ in range(n)]
    a[0] = [5, 0, 0, 0, 0, 0, 0]          # a base-field element
    a[1] = [0, 1, 0, 0, 0, 0, 0]          # z
    a[2] = [0, 0, 0, 0, 0, 0, P - 1]      # -z^6
    A = np.concatenate([mont(x) for x in a]); B = np.concatenate([mont(x) for x in b])
    mul, inv = np.zeros(7 * n, np.uint32), np.zeros(7 * n, np.uint32)
    _lib().sp1b200_hostcheck_septic(_p(A), _p(B), _p(mul), _p(inv), C.c_uint64(n))
    for i in range(n):
        assert canon(mul[7 * i:7 * i + 7]) == smul(a[i], b[i]), i
        assert canon(inv[7 * i:7 * i + 7]) == sinv(a[i]), i
        assert smul(canon(inv[7 * i:7 * i + 7]), a[i]) == [1, 0, 0, 0, 0, 0, 0]
    # z^7 = 3z + 5
    assert spow([0, 1, 0, 0, 0, 0, 0], 7) == [5, 3, 0, 0, 0, 0, 0]


def _multiples(base, k):
    """base, 2 base, ..., k base by repeated incomplete addition (the doubling 2 base by the tangent)"""
    x, y = base
    # 2P by the tangent: slope = (3x^2 + 45) / 2y
    s = smul(sadd(smul([3, 0, 0, 0, 0, 0, 0], smul(x, x)), [45, 0, 0, 0, 0, 0, 0]), sinv(sadd(y, y)))
    x2 = ssub(ssub(smul(s, s), x), x)
    two = (x2, ssub(smul(s, ssub(x, x2)), y))
    out = [base, two]
    while len(out) < k:
        out.append(curve_add(out[-1], base))
    return out


def test_curve_add_matches_the_restatement():
    pts = _multiples(DUMMY, 8) + _multiples(START, 4)
    for p in pts:
        assert on_curve(p)
    pairs = [(pts[i], pts[j]) for i in range(len(pts)) for j in range(len(pts)) if i != j][:40]
    pairs.append((pts[2], pts[2]))                      # the exceptional case: equal x
    pairs.append((pts[3], curve_neg(pts[3])))           # and P + (-P)
    n = len(pairs)
    Pw = np.concatenate([pt_words(a) for a, _ in pairs]); Qw = np.concatenate([pt_words(b) for _, b in pairs])
    out, ok = np.zeros(14 * n, np.uint32), np.zeros(n, np.uint32)
    _lib().sp1b200_hostcheck_septic_curve_add(_p(Pw), _p(Qw), _p(out), _p(ok), C.c_uint64(n))
    for i, (a, b) in enumerate(pairs):
        want = curve_add(a, b)
        assert bool(ok[i]) == (want is not None), i
        if want is not None:
            assert words_pt(out[14 * i:14 * i + 14]) == want, i
            assert on_curve(want)


def test_digest_sum_of_multiples_cancels():
    """the core verifier's sum: initial + (zero + P_1) + ... + (zero + P_n) == zero when the initial sum is zero - Σ P_i"""
    L = _lib()
    mult = _multiples(DUMMY, 12)
    rng = np.random.default_rng(11)
    ks = [int(k) for k in rng.integers(1, 5, 3)]            # shard i's digest = zero + k_i · dummy
    digests = [curve_add(ZERO, mult[k - 1]) for k in ks]
    initial = curve_add(ZERO, curve_neg(mult[sum(ks) - 1]))
    acc_py, acc = initial, pt_words(initial)
    for d in digests:
        acc_py = digest_add(acc_py, d)
        out = np.zeros(14, np.uint32)
        assert L.sp1b200_hostcheck_septic_digest_add(_p(acc), _p(pt_words(d)), _p(out)) == 1
        assert words_pt(out) == acc_py
        acc = out
    assert words_pt(acc) == (ZERO[0], ZERO[1])


def test_digest_add_reports_the_exceptional_case():
    """a digest equal to the starting digest makes the first incomplete addition divide by zero"""
    out = np.zeros(14, np.uint32)
    assert _lib().sp1b200_hostcheck_septic_digest_add(_p(pt_words(START)), _p(pt_words(ZERO)), _p(out)) == 0
    assert digest_add(START, ZERO) is None


# PublicValues<[F; 4], [F; 3], [F; 4], F> (crates/hypercube/src/air/public_values.rs), without the mprotect fields: (field, words)
PUBLIC_VALUES_FIELDS = [
    ("prev_committed_value_digest", 8 * 4), ("committed_value_digest", 8 * 4), ("prev_deferred_proofs_digest", 8),
    ("deferred_proofs_digest", 8), ("pc_start", 3), ("next_pc", 3), ("prev_exit_code", 1), ("exit_code", 1),
    ("is_execution_shard", 1), ("previous_init_addr", 3), ("last_init_addr", 3), ("previous_finalize_addr", 3),
    ("last_finalize_addr", 3), ("previous_init_page_idx", 3), ("last_init_page_idx", 3), ("previous_finalize_page_idx", 3),
    ("last_finalize_page_idx", 3), ("initial_timestamp", 4), ("last_timestamp", 4), ("is_timestamp_high_eq", 1),
    ("inv_timestamp_high", 1), ("is_timestamp_low_eq", 1), ("inv_timestamp_low", 1), ("global_init_count", 1),
    ("global_finalize_count", 1), ("global_page_prot_init_count", 1), ("global_page_prot_finalize_count", 1), ("global_count", 1),
    ("global_cumulative_sum", 14), ("prev_commit_syscall", 1), ("commit_syscall", 1), ("prev_commit_deferred_syscall", 1),
    ("commit_deferred_syscall", 1), ("initial_timestamp_inv", 1), ("last_timestamp_inv", 1), ("is_first_execution_shard", 1),
    ("is_untrusted_programs_enabled", 1), ("proof_nonce", 4), ("empty", 4),
]


def test_public_values_offsets_match_the_struct():
    from sp1_b200 import lib as B
    at = 0
    for name, n in PUBLIC_VALUES_FIELDS:
        assert B.PV[name] == (at, n), name
        at += n
    assert at == B.PV_NUM_ELTS == 160
    assert set(B.PV) == {n for n, _ in PUBLIC_VALUES_FIELDS}
    assert B.PV_MAX_NUM == 187 and B.VK_TAIL_WORDS == 24


def test_core_verdict_names():
    from sp1_b200 import lib as B
    assert B.verdict_name(42) == "InvalidShape(chip tables)"
    assert B.verdict_name(43) == "EmptyProof"
    assert B.verdict_name(44) == "TooManyShards"
    assert B.verdict_name(45) == "InvalidShardProof"
    assert B.verdict_name(50) == "InvalidPublicValues(invalid initial timestamp)"
    assert B.verdict_name(74) == "InvalidPublicValues(global cumulative sum is not zero)"
    assert B.verdict_name(75) == "InvalidPublicValues(global cumulative sum: exceptional point addition)"
    assert B.verdict_name(76) == "Unknown"
    names = [B.verdict_name(v) for v in range(46, 76)]
    assert all(n.startswith("InvalidPublicValues(") for n in names) and len(set(names)) == 30
