"""ctypes binding of oracle/libliftoracle.so: the restated SepticCurve::lift_x, SepticExtension::sqrt, SepticCurveComplete addition and
Program::initial_global_cumulative_sum (oracle/lift.hpp, built by oracle/lift.mk).  Test infrastructure only.  Field elements are u32
Montgomery words."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests.oracle_lib import ptr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(ROOT, "oracle", "libliftoracle.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "lift.mk"])
        L = C.CDLL(_SO)
        L.orc_initial_global_cumulative_sum.restype = C.c_int
        _lib = L
    return _lib


def lift_x(msgs):
    """SepticCurve::lift_x of [n, 8] messages (Montgomery words) -> ([n] offsets, -1 where the reference panics; [n, 14] points)"""
    m = np.ascontiguousarray(msgs, dtype=np.uint32).reshape(-1, 8)
    off, pts = np.zeros(m.shape[0], np.int32), np.zeros((m.shape[0], 14), np.uint32)
    lib().orc_lift_x(ptr(m), C.c_void_p(off.ctypes.data), ptr(pts), C.c_uint64(m.shape[0]))
    return off, pts


def septic_sqrt(a):
    """SepticExtension::sqrt of [n, 7] elements -> ([n, 7] roots, [n] ok flags: 0 for a non-square)"""
    a = np.ascontiguousarray(a, dtype=np.uint32).reshape(-1, 7)
    out, ok = np.zeros_like(a), np.zeros(a.shape[0], np.uint32)
    lib().orc_septic_sqrt(ptr(a), ptr(out), ptr(ok), C.c_uint64(a.shape[0]))
    return out, ok


def curve_add_complete(p, q):
    """SepticCurveComplete + of [n, 14] point pairs (infinity = 14 zero words) -> [n, 14]"""
    p = np.ascontiguousarray(p, dtype=np.uint32).reshape(-1, 14); q = np.ascontiguousarray(q, dtype=np.uint32).reshape(-1, 14)
    out = np.zeros_like(p)
    lib().orc_curve_add_complete(ptr(p), ptr(q), ptr(out), C.c_uint64(p.shape[0]))
    return out


def initial_global_cumulative_sum(addrs, words, pages=None, prots=None, untrusted=0):
    """Program::initial_global_cumulative_sum of a memory image (and page image) -> 14 words; raises where the reference panics"""
    a = np.ascontiguousarray(addrs, dtype=np.uint64); w = np.ascontiguousarray(words, dtype=np.uint64)
    pg = np.ascontiguousarray(pages if pages is not None else [], dtype=np.uint64)
    pr = np.ascontiguousarray(prots if prots is not None else [], dtype=np.uint8)
    out, bad = np.zeros(14, np.uint32), C.c_uint64()
    r = lib().orc_initial_global_cumulative_sum(C.c_void_p(a.ctypes.data), C.c_void_p(w.ctypes.data), C.c_uint64(a.size),
                                                C.c_void_p(pg.ctypes.data), C.c_void_p(pr.ctypes.data), C.c_uint64(pg.size),
                                                C.c_int(untrusted), ptr(out), C.byref(bad))
    if r == 1:
        raise ValueError(f"entry {bad.value} has no curve point after 256 offsets")
    if r == 2:
        raise ValueError("the sum is the point at infinity")
    return out
