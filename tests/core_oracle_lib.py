"""ctypes binding of oracle/libcoreoracle.so: the restated core-proof verifier (oracle/core.hpp, built by oracle/core.mk) and its septic
arithmetic.  Test infrastructure only.  Field elements are u32 Montgomery words."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests.oracle_lib import ptr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(ROOT, "oracle", "libcoreoracle.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "core.mk"])
        L = C.CDLL(_SO)
        L.orc_verify_core_proof.restype = C.c_int64
        L.orc_septic_digest_add.restype = C.c_int
        _lib = L
    return _lib


def septic_mul(a, b):
    """[n, 7] x [n, 7] -> [n, 7]"""
    a = np.ascontiguousarray(a, dtype=np.uint32); b = np.ascontiguousarray(b, dtype=np.uint32)
    out = np.zeros_like(a)
    lib().orc_septic_mul(ptr(a), ptr(b), ptr(out), C.c_uint64(a.shape[0]))
    return out


def septic_inv(a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    out = np.zeros_like(a)
    lib().orc_septic_inv(ptr(a), ptr(out), C.c_uint64(a.shape[0]))
    return out


def curve_add(p, q):
    """[n, 14] points (x then y) -> ([n, 14] sums, [n] ok flags: 0 on the exceptional case)"""
    p = np.ascontiguousarray(p, dtype=np.uint32); q = np.ascontiguousarray(q, dtype=np.uint32)
    out, ok = np.zeros_like(p), np.zeros(p.shape[0], np.uint32)
    lib().orc_septic_curve_add(ptr(p), ptr(q), ptr(out), ptr(ok), C.c_uint64(p.shape[0]))
    return out, ok


def digest_add(a, b):
    """SepticDigest + SepticDigest of two 14-word points -> 14 words, or None on the exceptional case"""
    a = np.ascontiguousarray(a, dtype=np.uint32); b = np.ascontiguousarray(b, dtype=np.uint32)
    out = np.zeros(14, np.uint32)
    return out if lib().orc_septic_digest_add(ptr(a), ptr(b), ptr(out)) else None


def verify_core_proof(blob, heights_per_shard, names, log_stack, max_log_rows, prep_commit, vk_tail, words_per_shard, log_blowup=2,
                      num_queries=124, pow_bits=16, batch_pow_bits=5, gkr_pow_bits=12):
    """the restated SP1Prover::verify -> (verdict, shard, shard_result): verdict 0 accepts, -2 when a shard does not parse, else a code
    of include/sp1b200.h; for InvalidShardProof shard_result is orc_verify_shard's result on that shard (its reason is on stderr)"""
    n, nch = len(words_per_shard), len(names)
    H = np.ascontiguousarray(np.asarray(heights_per_shard, dtype=np.uint64).reshape(-1) if n else np.zeros(1, np.uint64))
    nm = b"".join(s.encode() + b"\0" for s in names)
    ws = [np.ascontiguousarray(w, dtype=np.uint32) for w in words_per_shard]
    P = (C.c_void_p * max(1, n))(*[w.ctypes.data for w in ws])
    NW = (C.c_uint64 * max(1, n))(*[w.size for w in ws])
    blob = np.ascontiguousarray(blob, dtype=np.uint32)
    pc = np.ascontiguousarray(prep_commit if prep_commit is not None else np.zeros(8), dtype=np.uint32)
    tail = np.ascontiguousarray(vk_tail, dtype=np.uint32)
    shard, res = C.c_uint32(), C.c_int64()
    v = lib().orc_verify_core_proof(ptr(blob), C.c_uint32(nch), C.c_void_p(H.ctypes.data), C.c_char_p(nm), C.c_uint32(log_stack),
                                    C.c_uint32(max_log_rows), C.c_uint32(log_blowup), C.c_uint32(num_queries), C.c_uint32(pow_bits),
                                    C.c_uint32(batch_pow_bits), C.c_uint32(gkr_pow_bits), ptr(pc), ptr(tail), C.c_uint32(n), P, NW,
                                    C.byref(shard), C.byref(res))
    return int(v), int(shard.value), int(res.value)
