"""Public values of a valid N-shard core proof (PublicValues<[F; 4], [F; 3], [F; 4], F>, sp1_b200.lib.PV) and the verifying-key tail
they chain from, for the core-proof verifier's tests and benchmark.

The chain: timestamps from [0, 0, 0, 1]; program counters from the key's pc_start to HALT_PC = [1, 0, 0]; exactly one first execution
shard (shard 0); optionally one non-execution shard (timestamps, pc and exit code unchanged across it); the commit-syscall flags at 1
from the first shard on; non-zero init / finalize addresses; one proof nonce; and global cumulative sums zero + k_i · dummy whose k_i
cancel against the key's initial sum zero - (Σ k_i) · dummy.  Everything is canonical integers; the synthetic chips read public value
0 = prev_committed_value_digest[0][0], so shard i's traces are built with pv0_of(pvs[i]).

PV_CASES: one chain fault per reason the public-value checks across shards give, with the verdict and shard the reference's loop stops at."""
import numpy as np

from tests.septic import DUMMY, START, ZERO, curve_add, curve_neg, multiples

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


# (name, mutation of the valid 3-shard chain with a non-execution shard 1, expected verdict, expected shard)
def _set(s, name, vals):
    return lambda pvs, tail: setf(pvs[s], name, vals)


def _m_len(pvs, tail):
    pvs[1][:] = pvs[1][:186]


def _m_never(field):
    def f(pvs, tail):
        for pv in pvs:
            setf(pv, "previous_" + field, [0, 0, 0]); setf(pv, "last_" + field, [0, 0, 0])
    return f


def _m_commit(field):
    def f(pvs, tail):
        for pv in pvs:
            setf(pv, "prev_" + field, 0); setf(pv, field, 0)
    return f


def _m_ts_changed(pvs, tail):
    last = getf(pvs[1], "last_timestamp"); last[3] += 1
    setf(pvs[1], "last_timestamp", last); setf(pvs[2], "initial_timestamp", last)


def _m_pc_nonexec(pvs, tail):
    setf(pvs[1], "next_pc", [7, 7, 7]); setf(pvs[2], "pc_start", [7, 7, 7])


def _m_exit_nonexec(pvs, tail):
    setf(pvs[1], "exit_code", 3); setf(pvs[2], "prev_exit_code", 3); setf(pvs[2], "exit_code", 3)


def _m_exit_changed(pvs, tail):
    setf(pvs[0], "exit_code", 3)
    for s in (1, 2):
        setf(pvs[s], "prev_exit_code", 3); setf(pvs[s], "exit_code", 3)
    setf(pvs[2], "exit_code", 4)


def _m_digest(pvs, tail):
    g = getf(pvs[1], "global_cumulative_sum")
    p = (g[:7], g[7:])
    q = curve_add(p, DUMMY)
    setf(pvs[1], "global_cumulative_sum", list(q[0]) + list(q[1]))


def _m_exceptional(pvs, tail):
    tail[3:17] = list(START[0]) + list(START[1])


def _m_bump(s, name, k=0):
    def f(pvs, tail):
        v = getf(pvs[s], name); v[k] = (v[k] + 1) % P
        setf(pvs[s], name, v)
    return f


PV_CASES = [
    ("length", _m_len, 46, 1),
    ("first shard twice", _set(2, "is_first_execution_shard", 1), 47, 2),
    ("first shard not boolean", _set(1, "is_first_execution_shard", 2), 48, 1),
    ("first shard not set", _set(0, "is_first_execution_shard", 0), 49, 3),
    ("initial timestamp", _m_bump(2, "initial_timestamp", 3), 50, 2),
    ("timestamp unchanged on an execution shard", _set(1, "is_execution_shard", 1), 51, 1),
    ("timestamp changed on a non-execution shard", _m_ts_changed, 52, 1),
    ("pc_start != vk.pc_start", _m_bump(0, "pc_start", 1), 53, 0),
    ("pc_start != prev_next_pc", _m_bump(2, "pc_start", 0), 54, 2),
    ("pc changed on a non-execution shard", _m_pc_nonexec, 55, 1),
    ("not halted", _set(2, "next_pc", [5, 0, 0]), 56, 3),
    ("prev_exit_code", _set(0, "prev_exit_code", 1), 57, 0),
    ("exit code changed on a non-execution shard", _m_exit_nonexec, 58, 1),
    ("exit code changed twice", _m_exit_changed, 59, 2),
    ("proof nonce", _m_bump(2, "proof_nonce", 1), 60, 2),
    ("previous_init_addr", _m_bump(1, "previous_init_addr"), 61, 1),
    ("previous_finalize_addr", _m_bump(1, "previous_finalize_addr", 2), 62, 1),
    ("previous_init_page_idx", _m_bump(2, "previous_init_page_idx"), 63, 2),
    ("previous_finalize_page_idx", _m_bump(2, "previous_finalize_page_idx", 1), 64, 2),
    ("untrusted programs flag", _set(0, "is_untrusted_programs_enabled", 1), 65, 0),
    ("zero address never initialized", _m_never("init_addr"), 66, 3),
    ("zero address never finalized", _m_never("finalize_addr"), 67, 3),
    ("committed value digest", _m_bump(1, "prev_committed_value_digest", 5), 68, 1),
    ("deferred proofs digest", _m_bump(2, "prev_deferred_proofs_digest", 7), 69, 2),
    ("commit syscall", _set(0, "prev_commit_syscall", 1), 70, 0),
    ("commit deferred syscall", _set(1, "prev_commit_deferred_syscall", 0), 71, 1),
    ("COMMIT never called", _m_commit("commit_syscall"), 72, 3),
    ("COMMIT_DEFERRED_PROOFS never called", _m_commit("commit_deferred_syscall"), 73, 3),
    ("global cumulative sum", _m_digest, 74, 3),
    ("exceptional point addition", _m_exceptional, 75, 0),
]
