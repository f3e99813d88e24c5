"""CPU tests of the shard's memory chips: the NumPy restatement (tests/memory_ref.py) against rows, lookups and global events checked by
hand, and the C records of sp1b200_memory_traces against what sp1_b200.lib packs."""
import os
import subprocess
import tempfile

import numpy as np

from tests import memory_ref as MR

ROOT = os.path.dirname(os.path.abspath(__file__)).rsplit(os.sep, 1)[0]
P = MR.P


def _events(addrs, values=None, timestamps=None):
    from sp1_b200.lib import pack_memory_events
    n = len(addrs)
    return pack_memory_events(addrs, [0] * n if values is None else values, [0] * n if timestamps is None else timestamps)


def _row(t, i):
    return {name: int(t[i, k]) for k, name in enumerate(MR.INIT_COLS)}


def _lt(row):
    return [row["lt.bit"]] + [row[f"lt.u16_flags[{k}]"] for k in range(4)] + [row["lt.not_eq_inv"], row["lt.comparison_limbs[0]"],
                                                                                 row["lt.comparison_limbs[1]"]]


def test_column_counts_match_the_library():
    from sp1_b200.lib import MEMORY_CHIP_COLS, MEMORY_GLOBAL_LOOKUPS, MEMORY_LOCAL_LOOKUPS
    assert MR.NUM_MEMORY_INIT_COLS == MEMORY_CHIP_COLS["MemoryGlobalInit"] == MEMORY_CHIP_COLS["MemoryGlobalFinalize"] == 30
    assert MR.NUM_MEMORY_LOCAL_INIT_COLS == MEMORY_CHIP_COLS["MemoryLocal"] == 20
    assert (MEMORY_GLOBAL_LOOKUPS, MEMORY_LOCAL_LOOKUPS) == (12, 10)
    assert [MR.num_rows(n) for n in (0, 1, 15, 16, 17, 31, 32, 33)] == [0, 32, 32, 32, 32, 32, 32, 64]


def test_init_rows_checked_by_hand():
    # given out of order: the chip sorts by address
    addrs = [0x2_0000_0005, 0, 0x10007, 7, (1 << 48) - 1]
    values = [0, 0, 0x0000_ABCD_1234_5678, 0xFFFF_FFFF_0000_0001, 1]
    ts = [(3 << 24) | 0x123456, 0, 0xFFFF_FFFF_FFFF, 1, 2]
    t = MR.global_trace(_events(addrs, values, ts), 0)
    assert t.shape == (32, 30)
    assert not t[5:].any()                                   # padding rows are zero
    r0, r1, r2, r3, r4 = (_row(t, i) for i in range(5))
    # address 0 first with previous address 0: no comparison
    assert [r0[f"addr[{k}]"] for k in range(3)] == [0, 0, 0] and r0["is_comp"] == 0 and r0["prev_valid"] == 1
    assert _lt(r0) == [0] * 8
    assert (r0["is_prev_addr_zero.inverse"], r0["is_prev_addr_zero.result"], r0["is_index_zero.inverse"], r0["is_index_zero.result"]) == (0, 1, 0, 1)
    assert (r0["is_real"], r0["index"], r0["clk_high"], r0["clk_low"]) == (1, 0, 0, 0)
    # the row after it: prev_addr 0 at i = 1, so prev_valid 0; 0 < 7 differs first in limb 0
    assert [r1[f"prev_addr[{k}]"] for k in range(3)] == [0, 0, 0] and r1["prev_valid"] == 0 and r1["is_comp"] == 1
    assert _lt(r1) == [1, 1, 0, 0, 0, pow(P - 7, P - 2, P), 0, 7]
    assert (r1["is_prev_addr_zero.result"], r1["is_index_zero.inverse"], r1["is_index_zero.result"]) == (1, 1, 0)
    assert (r1["clk_high"], r1["clk_low"], r1["value_lower"], r1["value_upper"]) == (0, 1, 0xFF, 0xFF)
    assert [r1[f"value[{k}]"] for k in range(4)] == [1, 0, 0xFFFF, 0xFFFF]
    # 7 < 0x10007 differs first in limb 1: (0 - 1)^-1 = p - 1; a value with bytes 4 and 5 set
    assert [r2[f"prev_addr[{k}]"] for k in range(3)] == [7, 0, 0] and [r2[f"addr[{k}]"] for k in range(3)] == [7, 1, 0]
    assert _lt(r2) == [1, 0, 1, 0, 0, P - 1, 0, 1] and r2["prev_valid"] == 1
    assert (r2["is_prev_addr_zero.inverse"], r2["is_prev_addr_zero.result"]) == (pow(7, P - 2, P), 0)
    assert (r2["is_index_zero.inverse"] * 2) % P == 1
    assert [r2[f"value[{k}]"] for k in range(4)] == [0x5678, 0x1234, 0xABCD, 0] and (r2["value_lower"], r2["value_upper"]) == (0xCD, 0xAB)
    assert (r2["clk_high"], r2["clk_low"]) == (0xFFFFFF, 0xFFFFFF)
    # 0x10007 < 0x2_0000_0005 differs first in limb 2: (0 - 2)^-1 = (p - 1) / 2
    assert _lt(r3) == [1, 0, 0, 1, 0, (P - 1) // 2, 0, 2]
    assert (r3["is_prev_addr_zero.inverse"] * 8) % P == 1 and (r3["clk_high"], r3["clk_low"]) == (3, 0x123456)
    # the largest address 2^48 - 1: limb 2 again, (2 - 0xFFFF)^-1
    assert [r4[f"addr[{k}]"] for k in range(3)] == [0xFFFF] * 3
    assert _lt(r4) == [1, 0, 0, 1, 0, pow((2 - 0xFFFF) % P, P - 2, P), 2, 0xFFFF]
    assert r4["index"] == 4 and (r4["is_index_zero.inverse"] * 4) % P == 1


def test_nonzero_previous_address_at_row_0():
    t = MR.global_trace(_events([0x1_0000_0105]), 0x1_0000_0100)
    r = _row(t, 0)
    assert [r[f"prev_addr[{k}]"] for k in range(3)] == [0x100, 0, 1] and r["is_comp"] == 1 and r["prev_valid"] == 1
    assert _lt(r) == [1, 1, 0, 0, 0, pow(P - 5, P - 2, P), 0x100, 0x105]
    assert (r["is_prev_addr_zero.inverse"] * 0x101) % P == 1 and r["is_prev_addr_zero.result"] == 0
    assert (r["is_index_zero.inverse"], r["is_index_zero.result"]) == (0, 1)
    lk, msg, rcv, kind = MR.global_dependencies(_events([0x1_0000_0105], [0x0000_0201_0000_0009], [(9 << 24) | 4]), 0x1_0000_0100, True)
    assert lk.tolist() == ([[6, 9, 16, 0], [6, 0, 16, 0], [6, 0x0201, 16, 0], [6, 0, 16, 0]] + [[6, 0x100, 16, 0], [6, 0, 16, 0], [6, 1, 16, 0]]
                           + [[6, 0x105, 16, 0], [6, 0, 16, 0], [6, 1, 16, 0]] + [[3, 0, 0x01, 0x02], [6, (0x100 - 0x105) & 0xFFFF, 16, 0]])
    # Finalize receives with the event's clk; the value limbs fold bytes 4 and 5 in at 2^16
    assert msg.tolist() == [[9, 4, 0x105, 0, 1, 9 + (0x01 << 16), 0 + (0x02 << 16), 0]] and rcv.tolist() == [1] and kind.tolist() == [1]


def test_init_dependencies_checked_by_hand():
    ev = _events([7, 0], [0x0000_ABCD_1234_5678, 0], [(1 << 24) | 2, 5])
    lk, msg, rcv, kind = MR.global_dependencies(ev, 0, False)
    row0 = [[6, 0, 16, 0]] * 4 + [[6, 0, 16, 0]] * 3 + [[6, 0, 16, 0]] * 3 + [[3, 0, 0, 0]]          # address 0: no comparison
    row1 = ([[6, 0x5678, 16, 0], [6, 0x1234, 16, 0], [6, 0xABCD, 16, 0], [6, 0, 16, 0]] + [[6, 0, 16, 0]] * 3
            + [[6, 7, 16, 0], [6, 0, 16, 0], [6, 0, 16, 0]] + [[3, 0, 0xCD, 0xAB], [6, 0xFFF9, 16, 0]])
    assert lk.tolist() == row0 + row1
    # Init sends with clk 0, 0, in sorted order
    assert msg.tolist() == [[0, 0, 0, 0, 0, 0, 0, 0], [0, 0, 7, 0, 0, 0x5678 + (0xCD << 16), 0x1234 + (0xAB << 16), 0]]
    assert rcv.tolist() == [0, 0] and kind.tolist() == [1, 1]


def test_local_row_checked_by_hand():
    from sp1_b200.lib import pack_memory_local_events
    ev = pack_memory_local_events([0x1_0002_0003], [(5 << 24) | 7], [0x0102_0304_0506_0708], [(6 << 24) | 0xFFFFFF], [0xFFEE_DDCC_BBAA_9988])
    t = MR.local_trace(ev)
    assert t.shape == (32, 20) and not t[1:].any()
    r = {name: int(t[0, k]) for k, name in enumerate(MR.LOCAL_COLS)}
    assert [r[f"addr[{k}]"] for k in range(3)] == [3, 2, 1]
    assert (r["initial_clk_high"], r["initial_clk_low"], r["final_clk_high"], r["final_clk_low"]) == (5, 7, 6, 0xFFFFFF)
    assert [r[f"initial_value[{k}]"] for k in range(4)] == [0x0708, 0x0506, 0x0304, 0x0102]
    assert [r[f"final_value[{k}]"] for k in range(4)] == [0x9988, 0xBBAA, 0xDDCC, 0xFFEE]
    assert (r["initial_value_lower"], r["initial_value_upper"], r["final_value_lower"], r["final_value_upper"]) == (0x04, 0x03, 0xCC, 0xDD)
    assert r["is_real"] == 1
    assert list(t[0]) == [3, 2, 1, 5, 6, 7, 0xFFFFFF, 0x0708, 0x0506, 0x0304, 0x0102, 0x9988, 0xBBAA, 0xDDCC, 0xFFEE, 4, 3, 0xCC, 0xDD, 1]
    lk, msg, rcv, kind = MR.local_dependencies(ev)
    assert lk.tolist() == ([[3, 0, 0x04, 0x03]] + [[6, x, 16, 0] for x in (0x0708, 0x0506, 0x0304, 0x0102)]
                           + [[3, 0, 0xCC, 0xDD]] + [[6, x, 16, 0] for x in (0x9988, 0xBBAA, 0xDDCC, 0xFFEE)])
    # the initial access is received, the final access sent
    assert msg.tolist() == [[5, 7, 3, 2, 1, 0x0708 + (0x04 << 16), 0x0506 + (0x03 << 16), 0x0102],
                            [6, 0xFFFFFF, 3, 2, 1, 0x9988 + (0xCC << 16), 0xBBAA + (0xDD << 16), 0xFFEE]]
    assert rcv.tolist() == [1, 0] and kind.tolist() == [1, 1]


def test_main_words_are_column_major_montgomery():
    t = MR.global_trace(_events([0, 3]), 0)
    w = MR.main_words(t)
    assert w.shape == (30, 32) and w.dtype == np.uint32
    assert int(w[MR.IC["addr[0]"], 1]) == (3 << 32) % P and int(w[MR.IC["is_real"], 0]) == (1 << 32) % P


def test_record_layouts_match_the_header():
    """sizeof / offsetof of the three memory records, compiled from include/sp1b200.h, equal the numpy records lib.py packs"""
    from sp1_b200.lib import GLOBAL_EVENT_DTYPE, MEMORY_EVENT_DTYPE, MEMORY_LOCAL_EVENT_DTYPE
    src = r'''#include <stdio.h>
#include <stddef.h>
#include "sp1b200.h"
int main(void) {
    printf("%zu %zu %zu %zu\n", sizeof(sp1b200_memory_event), offsetof(sp1b200_memory_event, addr), offsetof(sp1b200_memory_event, value),
           offsetof(sp1b200_memory_event, timestamp));
    printf("%zu %zu %zu %zu %zu %zu\n", sizeof(sp1b200_memory_local_event), offsetof(sp1b200_memory_local_event, addr),
           offsetof(sp1b200_memory_local_event, initial_timestamp), offsetof(sp1b200_memory_local_event, initial_value),
           offsetof(sp1b200_memory_local_event, final_timestamp), offsetof(sp1b200_memory_local_event, final_value));
    printf("%zu %zu %zu %zu %zu\n", sizeof(sp1b200_global_event), offsetof(sp1b200_global_event, message),
           offsetof(sp1b200_global_event, is_receive), offsetof(sp1b200_global_event, kind), offsetof(sp1b200_global_event, pad));
    printf("%u %u %u %u\n", SP1B200_MEMORY_GLOBAL_COLS, SP1B200_MEMORY_LOCAL_COLS, SP1B200_MEMORY_GLOBAL_LOOKUPS, SP1B200_MEMORY_LOCAL_LOOKUPS);
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "layout.c"), "w") as f:
            f.write(src)
        exe = os.path.join(d, "layout")
        subprocess.run(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", exe, os.path.join(d, "layout.c")], check=True)
        lines = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    got_m, got_l, got_g, consts = [[int(v) for v in l.split()] for l in lines]
    fm, fl, fg = MEMORY_EVENT_DTYPE.fields, MEMORY_LOCAL_EVENT_DTYPE.fields, GLOBAL_EVENT_DTYPE.fields
    assert got_m == [MEMORY_EVENT_DTYPE.itemsize] + [fm[n][1] for n in ("addr", "value", "timestamp")] and got_m[0] == 24
    assert got_l == [MEMORY_LOCAL_EVENT_DTYPE.itemsize] + [fl[n][1] for n in MEMORY_LOCAL_EVENT_DTYPE.names] and got_l[0] == 40
    assert got_g == [GLOBAL_EVENT_DTYPE.itemsize] + [fg[n][1] for n in ("message", "is_receive", "kind", "pad")] and got_g[0] == 36
    assert consts == [MR.NUM_MEMORY_INIT_COLS, MR.NUM_MEMORY_LOCAL_INIT_COLS, 12, 10]


def test_memory_traces_symbol_is_exported():
    from sp1_b200 import lib as B
    assert hasattr(B.load(), "sp1b200_memory_traces") and "sp1b200_memory_traces" in B.ERR_FUNCS
