"""The shard checks on the CPU: the restated debug_constraints_all_chips / debug_interactions_with_all_chips (oracle/debug.hpp) on
satisfiable and corrupted machines, the interaction check's key fingerprint (linear, so colliding keys can be built from it), and
the code ptxas generates for the constraint-check kernel."""
import os
import re

import numpy as np
import pytest

from sp1_b200.lib import parse_constraint_report, parse_interaction_report
from tests import debug_oracle_lib as DO
from tests import machines as M
from tests import oracle_lib as O
from tests.machines import colliding_keys, cross_chip_machine, fingerprint

P = O.P
PV = M.PV


def _small_workload(name):
    return M.workload_machine(name, seed=3, scale=1 / 256)[:4]


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
