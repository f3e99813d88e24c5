"""The shard checks on the CPU: the restated debug_constraints_all_chips / debug_interactions_with_all_chips (oracle/debug.hpp) on
satisfiable and corrupted machines, the interaction check's key fingerprint (linear, so colliding keys can be built from it), and
the code ptxas generates for the constraint-check kernel.  Helpers here build the machines tests/test_gpu_debug.py checks on the GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from sp1_b200 import synth_air as SA
from sp1_b200 import workload as W
from sp1_b200.lib import parse_constraint_report, parse_interaction_report
from tests import hostcheck_lib
from tests import debug_oracle_lib as DO
from tests import oracle_lib as O

P = O.P
PV = O.to_monty(np.array([12345, 5, 6, 7]))


def _inter_words(inters):
    """inters: [(is_send, kind, mult vcol words, [value vcol words])] -> the chip's interaction words"""
    w = [len(inters)]
    for is_send, kind, mult, vals in inters:
        w += [is_send, kind, len(vals)] + mult
        for v in vals:
            w += v
    return w


def cross_chip_machine(rng, h=64, mult_col_kind4=False):
    """two one-group chips whose sends (chip 0) and receives (chip 1) sit in different chips: chip 1's trace is chip 0's with the rows
    reversed.  Interactions (sends in chip 0, receives in chip 1, same order): kind 4 (a, 9) with multiplicity 1 (or column d when
    mult_col_kind4), kind 6 (b) with multiplicity d."""
    w, _, _ = SA.synth_chip(1, False)
    m0, _ = SA.synth_trace(rng, h, 1, False, 12345)
    m1 = np.ascontiguousarray(m0[:, ::-1])
    a, b, d = (SA.LEAF_MAIN, 0, 1), (SA.LEAF_MAIN, 1, 1), (SA.LEAF_MAIN, 3, 1)
    mult4 = SA._vcol([d]) if mult_col_kind4 else SA._vcol([], constant=1)
    inter = lambda s: [(s, 4, mult4, [SA._vcol([a]), SA._vcol([], constant=9)]), (s, 6, SA._vcol([d]), [SA._vcol([b])])]
    blob = SA.machine_blob_with_interactions([w, w], [_inter_words(inter(1)), _inter_words(inter(0))])
    return blob, [h, h], [m0, m1], [None, None]


def fingerprint(kind, values):
    L = hostcheck_lib.load()
    f = L.sp1b200_hostcheck_fingerprint
    f.restype = C.c_uint64
    v = np.ascontiguousarray(values, dtype=np.uint32)
    return int(f(C.c_uint32(kind), C.c_uint32(v.size), v.ctypes.data_as(C.POINTER(C.c_uint32)) if v.size else None))


def colliding_keys(rng, kind=5):
    """two different 3-value keys (canonical values) with equal fingerprints, from the two linear forms read off basis vectors"""
    def forms(vals):
        x = fingerprint(kind, O.to_monty(np.array(vals)))
        return x >> 31, x & 0x7fffffff
    base = forms([0, 0, 0])
    c = []
    for t in range(3):
        e = [0, 0, 0]; e[t] = 1
        f = forms(e)
        c.append(((f[0] - base[0]) % P, (f[1] - base[1]) % P))
    # d = c0 x c1 (componentwise forms over the three values) is in the kernel of both forms
    u, v = [x[0] for x in c], [x[1] for x in c]
    d = [(u[1] * v[2] - u[2] * v[1]) % P, (u[2] * v[0] - u[0] * v[2]) % P, (u[0] * v[1] - u[1] * v[0]) % P]
    A = [int(x) for x in rng.integers(0, P, 3)]
    B = [(x + y) % P for x, y in zip(A, d)]
    assert A != B
    return A, B


def constant_key_machine(rng, chip_inters, heights):
    """one-group chips whose interactions have constant values: chip_inters[k] = [(is_send, kind, canonical values)], multiplicity 1"""
    words, iws, mains = [], [], []
    for inters, h in zip(chip_inters, heights):
        w, _, _ = SA.synth_chip(1, False)
        words.append(w)
        iws.append(_inter_words([(s, k, SA._vcol([], constant=1), [SA._vcol([], constant=x) for x in vals]) for s, k, vals in inters]))
        mains.append(SA.synth_trace(rng, h, 1, False, 12345)[0])
    return SA.machine_blob_with_interactions(words, iws), list(heights), mains, [None] * len(heights)


def _small_workload(name):
    m = W.synthetic_machine(name, seed=42, scale=1 / 256)
    rng = np.random.default_rng(3)
    mains, preps = [], []
    for sp in m["specs"]:
        a, p = SA.synth_trace(rng, sp.h, sp.g, sp.wp, 12345, extra_cols=sp.extra, extra_prep=sp.extra_prep)
        mains.append(a); preps.append(p)
    return m["blob"], [sp.h for sp in m["specs"]], mains, preps


@pytest.mark.parametrize("workload", ["tiny", "tinyc", "tinyr"])
def test_oracle_reports_nothing_on_satisfiable_machines(workload):
    blob, heights, mains, preps = _small_workload(workload)
    assert DO.debug_constraints(blob, heights, mains, preps, PV).tolist() == [0]
    assert DO.debug_interactions(blob, heights, mains, preps).tolist() == [0, 0, 0]


def test_oracle_constraint_report_names_the_corrupted_row():
    blob, heights, mains, preps = _small_workload("tinyc")
    k = max(range(len(heights)), key=lambda i: heights[i])
    row = heights[k] // 3
    mains[k][2, row] = (int(mains[k][2, row]) + 1) % P          # column c of group 0: breaks c = a b
    rep = parse_constraint_report(DO.debug_constraints(blob, heights, mains, preps, PV))
    assert list(rep) == [k] and rep[k]["n_failing_rows"] == 1 and list(rep[k]["rows"]) == [row]
    n_constraints = int(blob[1 + 3]) if k == 0 else None
    idx = rep[k]["rows"][row]
    assert idx and idx == sorted(set(idx)) and (n_constraints is None or max(idx) < n_constraints)
    mains[k][2, row] = (int(mains[k][2, row]) - 1) % P
    assert DO.debug_constraints(blob, heights, mains, preps, PV).tolist() == [0]


def test_oracle_interaction_report_on_cross_chip_corruptions():
    rng = np.random.default_rng(7)
    blob, heights, mains, preps = cross_chip_machine(rng)
    h = heights[0]
    assert DO.debug_interactions(blob, heights, mains, preps).tolist() == [0, 0, 0]
    # one changed value: chip 1 row r receives (a + 1, 9) instead of (a, 9)
    r = 5
    a_old = int(mains[1][0, r])
    mains[1][0, r] = (a_old + 1) % P
    rep = parse_interaction_report(DO.debug_interactions(blob, heights, mains, preps))
    mains[1][0, r] = a_old
    nine = int(O.to_monty(np.array([9]))[0])
    assert rep["n_unbalanced"] == 2
    k0, k1 = rep["keys"]
    one = int(O.to_monty(np.array([1]))[0])
    assert (k0["kind"], k0["values"], k0["net"], k0["first"], k0["chips"]) == (4, [a_old, nine], one, (0, 0, h - 1 - r), {0: one})
    assert (k1["kind"], k1["values"], k1["net"], k1["first"], k1["chips"]) == (4, [(a_old + 1) % P, nine], P - one, (1, 0, r), {1: P - one})
    # one changed multiplicity: chip 1 stops receiving (6, b) at a row where d = 1
    r = int(np.nonzero(mains[1][3] == one)[0][0])
    mains[1][3, r] = 0
    rep = parse_interaction_report(DO.debug_interactions(blob, heights, mains, preps))
    assert rep["n_unbalanced"] == 1 and rep["keys"][0]["kind"] == 6 and rep["keys"][0]["net"] == one
    assert rep["keys"][0]["first"] == (0, 1, h - 1 - r) and rep["keys"][0]["chips"] == {0: one}


def test_fingerprint_is_linear_and_collisions_can_be_built():
    rng = np.random.default_rng(11)
    x, y = O.rand_field(rng, 4), O.rand_field(rng, 4)
    s = ((x.astype(np.uint64) + y) % P).astype(np.uint32)
    fx, fy, fs, f0 = (fingerprint(3, v) for v in (x, y, s, np.zeros(4, np.uint32)))
    for sh, mask in ((31, 0x7fffffff), (0, 0x7fffffff)):
        part = lambda f: (f >> sh) & mask
        assert part(fs) == (part(fx) + part(fy) - part(f0)) % P      # affine in the values: the kind / n_values terms are constant
    assert fingerprint(3, x) < 1 << 62 and fingerprint(3, x) != fingerprint(4, x) and fingerprint(3, x[:3]) != fingerprint(3, x)
    A, B = colliding_keys(rng)
    assert fingerprint(5, O.to_monty(np.array(A))) == fingerprint(5, O.to_monty(np.array(B)))


BUILD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sp1_b200", "csrc", "build")


@pytest.mark.skipif(not os.path.exists(os.path.join(BUILD, "zerocheck.ptxas.log")), reason="needs the build directory")
def test_constraint_check_codegen():
    """the constraint-check kernels do not spill in the shared-memory tier, and the zerocheck sum kernels keep the registers / spills they
    had before the register file took a node count"""
    figs, cur = {}, None
    for line in open(os.path.join(BUILD, "zerocheck.ptxas.log")):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1); figs[cur] = [None, None]; continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and cur:
            figs[cur][1] = int(m.group(1))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            figs[cur][0] = int(m.group(1))
    dbg = [v for k, v in figs.items() if "zc_debug_kernelILi0E" in k]
    assert len(dbg) == 2 and all(s == 0 for _, s in dbg), dbg
    sums = sorted(tuple(v) for k, v in figs.items() if "zc_sum_kernel" in k)
    assert sums == [(64, 0), (66, 0), (70, 0), (94, 0), (96, 0), (96, 12)], sums
