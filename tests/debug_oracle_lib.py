"""ctypes binding of oracle/libdebugoracle.so: the restated shard checks (oracle/debug.hpp, built by oracle/debug.mk).  Test
infrastructure only.  Both calls return the report words of sp1b200_debug_constraints / sp1b200_debug_interactions."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests.oracle_lib import ptr, u32p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(ROOT, "oracle", "libdebugoracle.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "debug.mk"])
        L = C.CDLL(_SO)
        L.orc_debug_constraints.restype = C.c_uint64
        L.orc_debug_interactions.restype = C.c_uint64
        _lib = L
    return _lib


def _chip_ptrs(mains, preps, keep):
    def arr_ptr(a):
        a = np.ascontiguousarray(a if a is not None and a.size else np.zeros(1, np.uint32), dtype=np.uint32)
        keep.append(a)
        return ptr(a)
    n = len(mains)
    return (u32p * n)(*[arr_ptr(m) for m in mains]), (u32p * n)(*[arr_ptr(p) for p in preps])


def debug_constraints(blob, heights, mains, preps, pv, max_rows=3):
    """the restated debug_constraints_all_chips: report words of sp1b200_debug_constraints"""
    keep = []
    M, Pp = _chip_ptrs(mains, preps, keep)
    H = (C.c_uint64 * len(heights))(*heights)
    blob = np.ascontiguousarray(blob, dtype=np.uint32)
    pv = np.ascontiguousarray(pv, dtype=np.uint32)
    f = lib().orc_debug_constraints
    n = f(ptr(blob), H, M, Pp, ptr(pv), C.c_uint32(pv.size), C.c_uint32(max_rows), None, C.c_uint64(0))
    out = np.zeros(n, np.uint32)
    f(ptr(blob), H, M, Pp, ptr(pv), C.c_uint32(pv.size), C.c_uint32(max_rows), ptr(out), C.c_uint64(n))
    return out


def debug_interactions(blob, heights, mains, preps, max_keys=16):
    """the restated debug_interactions_with_all_chips: report words of sp1b200_debug_interactions"""
    keep = []
    M, Pp = _chip_ptrs(mains, preps, keep)
    H = (C.c_uint64 * len(heights))(*heights)
    blob = np.ascontiguousarray(blob, dtype=np.uint32)
    f = lib().orc_debug_interactions
    n = f(ptr(blob), H, M, Pp, C.c_uint32(max_keys), None, C.c_uint64(0))
    out = np.zeros(n, np.uint32)
    f(ptr(blob), H, M, Pp, C.c_uint32(max_keys), ptr(out), C.c_uint64(n))
    return out
