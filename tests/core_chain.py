"""Public values of a valid N-shard core proof (PublicValues<[F; 4], [F; 3], [F; 4], F>, sp1_b200.lib.PV) and the verifying-key tail
they chain from, for the core-proof verifier's tests and benchmark.

The chain: timestamps from [0, 0, 0, 1]; program counters from the key's pc_start to HALT_PC = [1, 0, 0]; exactly one first execution
shard (shard 0); optionally one non-execution shard (timestamps, pc and exit code unchanged across it); the commit-syscall flags at 1
from the first shard on; non-zero init / finalize addresses; one proof nonce; and global cumulative sums zero + k_i · dummy whose k_i
cancel against the key's initial sum zero - (Σ k_i) · dummy.  Everything is canonical integers; the synthetic chips read public value
0 = prev_committed_value_digest[0][0], so shard i's traces are built with pv0_of(pvs[i])."""
import numpy as np

from tests.test_septic import DUMMY, ZERO, curve_add, curve_neg, sadd, sinv, smul, ssub

P = 0x7F000001
PV_MAX_NUM = 187


def _off(name):
    from sp1_b200.lib import PV
    return PV[name]


def setf(pv, name, vals):
    at, n = _off(name)
    vals = list(vals) if hasattr(vals, "__len__") else [vals]
    assert len(vals) == n, name
    pv[at:at + n] = [int(v) % P for v in vals]


def getf(pv, name):
    at, n = _off(name)
    return list(pv[at:at + n])


def multiples(base, k):
    """[base, 2 base, ..., k base]: the doubling by the tangent, then incomplete additions"""
    x, y = base
    s = smul(sadd(smul([3, 0, 0, 0, 0, 0, 0], smul(x, x)), [45, 0, 0, 0, 0, 0, 0]), sinv(sadd(y, y)))
    x2 = ssub(ssub(smul(s, s), x), x)
    out = [base, (x2, ssub(smul(s, ssub(x, x2)), y))]
    while len(out) < k:
        out.append(curve_add(out[-1], base))
    return out[:k]


def vk_tail(pc_start, initial_sum, untrusted=0):
    """pc_start[3] | initial_global_cumulative_sum x[7] y[7] | enable_untrusted_programs | 6 zeros, canonical"""
    return [int(v) for v in pc_start] + list(initial_sum[0]) + list(initial_sum[1]) + [untrusted] + [0] * 6


def chain(n, seed, non_execution=None, untrusted=0):
    """-> (pvs: list of n lists of PV_MAX_NUM canonical ints, vk tail: 24 canonical ints).  non_execution: index of a shard (not 0)
    that executes nothing."""
    rng = np.random.default_rng(seed)
    r16 = lambda k: [int(v) for v in rng.integers(1, 1 << 16, k)]
    pc_start = r16(3)
    ks = [int(k) for k in rng.integers(1, 4, n)]
    mult = multiples(DUMMY, max(1, sum(ks)))
    initial = curve_add(ZERO, curve_neg(mult[sum(ks) - 1])) if n else ZERO
    nonce = [int(v) for v in rng.integers(0, P, 4)]
    pvs = []
    ts, pc, exit_code = [0, 0, 0, 1], pc_start, 0
    ia, fa, ip, fp = [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]
    cvd, dpd, commit, commit_def = [0] * 32, [0] * 8, 0, 0
    for i in range(n):
        pv = [0] * PV_MAX_NUM
        execn = i != non_execution
        setf(pv, "is_execution_shard", int(execn))
        setf(pv, "is_first_execution_shard", int(i == 0))
        setf(pv, "initial_timestamp", ts)
        ts = ts[:3] + [ts[3] + int(rng.integers(1, 1000))] if execn else ts
        setf(pv, "last_timestamp", ts)
        setf(pv, "pc_start", pc)
        pc = ([1, 0, 0] if i == n - 1 else r16(3)) if execn else pc
        setf(pv, "next_pc", pc)
        setf(pv, "prev_exit_code", exit_code)
        setf(pv, "exit_code", exit_code)
        setf(pv, "proof_nonce", nonce)
        for name, prev, last in (("init_addr", ia, None), ("finalize_addr", fa, None), ("init_page_idx", ip, None), ("finalize_page_idx", fp, None)):
            setf(pv, "previous_" + name, prev)
        ia, fa, ip, fp = r16(3), r16(3), r16(3), r16(3)
        setf(pv, "last_init_addr", ia); setf(pv, "last_finalize_addr", fa)
        setf(pv, "last_init_page_idx", ip); setf(pv, "last_finalize_page_idx", fp)
        setf(pv, "prev_committed_value_digest", cvd)
        cvd = [int(v) for v in rng.integers(1, 256, 32)]
        setf(pv, "committed_value_digest", cvd)
        setf(pv, "prev_deferred_proofs_digest", dpd)
        dpd = [int(v) for v in rng.integers(0, P, 8)]
        setf(pv, "deferred_proofs_digest", dpd)
        setf(pv, "prev_commit_syscall", commit); commit = 1; setf(pv, "commit_syscall", commit)
        setf(pv, "prev_commit_deferred_syscall", commit_def); commit_def = 1; setf(pv, "commit_deferred_syscall", commit_def)
        setf(pv, "is_untrusted_programs_enabled", untrusted)
        d = curve_add(ZERO, mult[ks[i] - 1])
        setf(pv, "global_cumulative_sum", list(d[0]) + list(d[1]))
        pvs.append(pv)
    return pvs, vk_tail(pc_start, initial, untrusted)


def pv0_of(pv):
    return int(pv[0])
