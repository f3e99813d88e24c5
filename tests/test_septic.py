"""CPU tests of the core-proof verifier's arithmetic (sp1_b200/csrc/septic.cuh, through libsp1b200_hostcheck.so): the septic
extension F_p[z]/(z^7 - 3z - 5), the curve y^2 = x^3 + 45x + 41z^3 and SepticDigest addition, against the Python restatement in
tests/septic.py; and the PublicValues word offsets of sp1_b200.lib.PV against the struct's field list."""
import ctypes as C

import numpy as np

from tests.septic import DUMMY, P, START, ZERO, canon, curve_add, curve_neg, digest_add, lib, mont, multiples, on_curve, ptr, pt_words, \
    sinv, smul, spow, words_pt


def test_constant_points_are_on_the_curve():
    for p in (ZERO, START, DUMMY):
        assert on_curve(p)
    out = np.zeros(42, np.uint32)
    lib().sp1b200_hostcheck_septic_constants(ptr(out))
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
    lib().sp1b200_hostcheck_septic(ptr(A), ptr(B), ptr(mul), ptr(inv), C.c_uint64(n))
    for i in range(n):
        assert canon(mul[7 * i:7 * i + 7]) == smul(a[i], b[i]), i
        assert canon(inv[7 * i:7 * i + 7]) == sinv(a[i]), i
        assert smul(canon(inv[7 * i:7 * i + 7]), a[i]) == [1, 0, 0, 0, 0, 0, 0]
    # z^7 = 3z + 5
    assert spow([0, 1, 0, 0, 0, 0, 0], 7) == [5, 3, 0, 0, 0, 0, 0]


def test_curve_add_matches_the_restatement():
    pts = multiples(DUMMY, 8) + multiples(START, 4)
    for p in pts:
        assert on_curve(p)
    pairs = [(pts[i], pts[j]) for i in range(len(pts)) for j in range(len(pts)) if i != j][:40]
    pairs.append((pts[2], pts[2]))                      # the exceptional case: equal x
    pairs.append((pts[3], curve_neg(pts[3])))           # and P + (-P)
    n = len(pairs)
    Pw = np.concatenate([pt_words(a) for a, _ in pairs]); Qw = np.concatenate([pt_words(b) for _, b in pairs])
    out, ok = np.zeros(14 * n, np.uint32), np.zeros(n, np.uint32)
    lib().sp1b200_hostcheck_septic_curve_add(ptr(Pw), ptr(Qw), ptr(out), ptr(ok), C.c_uint64(n))
    for i, (a, b) in enumerate(pairs):
        want = curve_add(a, b)
        assert bool(ok[i]) == (want is not None), i
        if want is not None:
            assert words_pt(out[14 * i:14 * i + 14]) == want, i
            assert on_curve(want)


def test_digest_sum_of_multiples_cancels():
    """the core verifier's sum: initial + (zero + P_1) + ... + (zero + P_n) == zero when the initial sum is zero - Σ P_i"""
    L = lib()
    mult = multiples(DUMMY, 12)
    rng = np.random.default_rng(11)
    ks = [int(k) for k in rng.integers(1, 5, 3)]            # shard i's digest = zero + k_i · dummy
    digests = [curve_add(ZERO, mult[k - 1]) for k in ks]
    initial = curve_add(ZERO, curve_neg(mult[sum(ks) - 1]))
    acc_py, acc = initial, pt_words(initial)
    for d in digests:
        acc_py = digest_add(acc_py, d)
        out = np.zeros(14, np.uint32)
        assert L.sp1b200_hostcheck_septic_digest_add(ptr(acc), ptr(pt_words(d)), ptr(out)) == 1
        assert words_pt(out) == acc_py
        acc = out
    assert words_pt(acc) == (ZERO[0], ZERO[1])


def test_digest_add_reports_the_exceptional_case():
    """a digest equal to the starting digest makes the first incomplete addition divide by zero"""
    out = np.zeros(14, np.uint32)
    assert lib().sp1b200_hostcheck_septic_digest_add(ptr(pt_words(START)), ptr(pt_words(ZERO)), ptr(out)) == 0
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
