"""CPU tests of the shard's lookup multiplicity traces: the NumPy restatement (tests/lookup_ref.py) against rows and public-value lookups
checked by hand, and the C records of sp1b200_lookup_traces against what sp1_b200.lib packs."""
import os
import subprocess
import tempfile

import numpy as np

from tests import lookup_ref as LR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lookups(rows):
    from sp1_b200.lib import pack_byte_lookups
    r = np.array(rows, np.int64).reshape(-1, 5)
    return pack_byte_lookups(r[:, 0], r[:, 1], r[:, 2], r[:, 3], r[:, 4])


def test_byte_rows_checked_by_hand():
    from sp1_b200.lib import BYTE_OPCODES as OP
    recs = []
    for k, (b, c) in enumerate([(0, 0), (0xFF, 0x01), (0x80, 0x7F)]):
        for name in ("AND", "OR", "XOR", "U8Range", "LTU", "MSB"):
            recs.append((OP[name], 0xBEEF, b, c, 10 * k + OP[name] + 1))   # a is not read
    recs.append((OP["AND"], 0, 0xFF, 0x01, 1000))       # a second record of one key adds
    recs.append((OP["Range"], 5, 0xFF, 0x01, 7))         # a Range record does not reach the Byte table
    t = LR.byte_trace(_lookups(recs))
    assert t.shape == (1 << 16, 6)
    #                       AND   OR  XOR  U8R  LTU  MSB
    assert [int(v) for v in t[0x0000]] == [1, 2, 3, 4, 5, 6]
    assert [int(v) for v in t[0xFF01]] == [1011, 12, 13, 14, 15, 16]
    assert [int(v) for v in t[0x807F]] == [21, 22, 23, 24, 25, 26]
    assert int(t.sum()) == sum(range(1, 7)) + sum(range(11, 17)) + sum(range(21, 27)) + 1000


def test_range_rows_checked_by_hand():
    R = 6
    recs = [(R, 0, 0, 0, 3),          # a = 0 < 2^0: row 1
            (R, 1, 1, 0, 4),          # row 2 + 1 = 3
            (R, 8191, 13, 0, 5),      # row 2^13 + 8191
            (R, 0, 16, 9, 6),         # row 2^16 (c is not read)
            (R, 65535, 16, 0, 7),     # the last row
            (R, 0, 16, 0, 1),         # adds to row 2^16
            (3, 0, 0, 0, 99)]         # U8Range: not a Range record
    t = LR.range_trace(_lookups(recs))
    assert t.shape == (1 << 17, 1)
    want = {1: 3, 3: 4, (1 << 13) + 8191: 5, 1 << 16: 7, (1 << 17) - 1: 7}
    assert {int(r): int(t[r, 0]) for r in np.nonzero(t[:, 0])[0]} == want


def test_program_rows_checked_by_hand():
    from sp1_b200.lib import pack_pc_counts
    base = 0x2000
    pcs = pack_pc_counts([base, base + 8, base + 8, base + 6, base - 4, base + 4 * 17, base + 4 * 16, 3],
                         [5, 1, 2, 100, 100, 100, 9, 100])
    t = LR.program_trace(base, 17, pcs)   # rows 0..16 are instructions, 17..31 padding
    assert t.shape == (32, 1)
    want = {0: 5, 2: 3, 16: 9}            # misaligned, below and above the window dropped
    assert {int(r): int(t[r, 0]) for r in np.nonzero(t[:, 0])[0]} == want
    assert [LR.next_multiple_of_32(n) for n in (1, 15, 16, 17, 32, 33)] == [32, 32, 32, 32, 32, 64]


def _pv():
    pv = [0] * 187
    pv[LR.INITIAL_TIMESTAMP:LR.INITIAL_TIMESTAMP + 4] = [0x1234, 0xAB, 0xCD, 0]        # low limb 0: (0 - 1) / 8 wraps to 8191
    pv[LR.LAST_TIMESTAMP:LR.LAST_TIMESTAMP + 4] = [0xFFFF, 0x01, 0x02, 0x0009]
    pv[LR.PC_START:LR.PC_START + 3] = [0x1111, 0x2222, 0x3333]
    pv[LR.NEXT_PC:LR.NEXT_PC + 3] = [1, 0, 0]
    pv[LR.LAST_FINALIZE_ADDR:LR.LAST_FINALIZE_ADDR + 3] = [0xFFFF, 0xFFFF, 0xFFFF]
    pv[LR.COMMITTED_VALUE_DIGEST:LR.COMMITTED_VALUE_DIGEST + 4] = [0x01, 0x02, 0x03, 0x04]
    pv[LR.PREV_COMMITTED_VALUE_DIGEST + 28:LR.PREV_COMMITTED_VALUE_DIGEST + 32] = [0xFF, 0x00, 0x7F, 0x80]
    return pv


def test_public_value_lookups_checked_by_hand():
    pv = _pv()
    byte = LR.byte_dependencies(pv)
    assert len(byte) == 2 + 8 * 2 * 2
    assert byte[:2] == [(3, 0, 0xAB, 0xCD), (3, 0, 0x01, 0x02)]
    assert (3, 0, 0x01, 0x02) in byte[2:6] and (3, 0, 0x03, 0x04) in byte[2:6]           # word 0 of committed_value_digest
    assert byte[-4:-2] == [(3, 0, 0xFF, 0x00), (3, 0, 0x7F, 0x80)]                        # word 7 of prev_committed_value_digest
    assert sum(1 for e in byte if e == (3, 0, 0, 0)) == 34 - 2 - 2 - 2                    # every other digest pair is zero
    rng = LR.range_dependencies(pv)
    assert len(rng) == 4 + 6 * 3
    assert rng[:4] == [(6, 0x1234, 16, 0), (6, 0xFFFF // 8, 13, 0), (6, 0xFFFF, 16, 0), (6, (9 - 1) // 8, 13, 0)]
    assert rng[4:7] == [(6, 0x1111, 16, 0), (6, 0x2222, 16, 0), (6, 0x3333, 16, 0)]
    assert rng[7:10] == [(6, 1, 16, 0), (6, 0, 16, 0), (6, 0, 16, 0)]
    assert rng[-3:] == [(6, 0xFFFF, 16, 0)] * 3
    t = LR.tables(0, 1, _lookups([]), _pcs_none(), pv)
    assert int(t["Range"][(1 << 13) + 8191, 0]) == 1 and int(t["Range"][(1 << 16) + 0xFFFF, 0]) == 4
    assert int(t["Byte"][0, 3]) == 28 and int(t["Byte"].sum()) == 34


def _pcs_none():
    from sp1_b200.lib import pack_pc_counts
    return pack_pc_counts(np.zeros(0, np.uint64), np.zeros(0, np.uint32))


def test_main_words_are_column_major_montgomery():
    from sp1_b200.lib import pack_pc_counts
    byte, prog, rng = LR.main_words(0x1000, 40, _lookups([(2, 0, 1, 2, 9), (6, 3, 2, 0, 4)]), pack_pc_counts([0x1000 + 4 * 39], [6]))
    assert byte.shape == (6, 1 << 16) and prog.shape == (1, 64) and rng.shape == (1, 1 << 17)
    assert byte[2, 0x0102] == LR.to_monty(9) and rng[0, 7] == LR.to_monty(4) and prog[0, 39] == LR.to_monty(6)
    assert np.count_nonzero(byte) == 1 and np.count_nonzero(prog) == 1 and np.count_nonzero(rng) == 1


def test_record_layouts_match_the_header():
    """sizeof / offsetof of sp1b200_byte_lookup and sp1b200_pc_count, compiled from include/sp1b200.h, equal the numpy records lib.py packs"""
    from sp1_b200.lib import BYTE_LOOKUP_DTYPE, PC_COUNT_DTYPE
    src = r'''#include <stdio.h>
#include <stddef.h>
#include "sp1b200.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(sp1b200_byte_lookup), offsetof(sp1b200_byte_lookup, a), offsetof(sp1b200_byte_lookup, b),
           offsetof(sp1b200_byte_lookup, c), offsetof(sp1b200_byte_lookup, opcode), offsetof(sp1b200_byte_lookup, pad),
           offsetof(sp1b200_byte_lookup, count));
    printf("%zu %zu %zu %zu\n", sizeof(sp1b200_pc_count), offsetof(sp1b200_pc_count, pc), offsetof(sp1b200_pc_count, count),
           offsetof(sp1b200_pc_count, pad));
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "layout.c"), "w") as f:
            f.write(src)
        exe = os.path.join(d, "layout")
        subprocess.run(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", exe, os.path.join(d, "layout.c")], check=True)
        lines = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    got_b, got_p = [[int(v) for v in l.split()] for l in lines]
    fb, fp = BYTE_LOOKUP_DTYPE.fields, PC_COUNT_DTYPE.fields
    assert got_b == [BYTE_LOOKUP_DTYPE.itemsize] + [fb[n][1] for n in ("a", "b", "c", "opcode", "pad", "count")]
    assert got_p == [PC_COUNT_DTYPE.itemsize] + [fp[n][1] for n in ("pc", "count", "pad")]


def test_lookup_traces_symbol_is_exported():
    from sp1_b200 import lib as B
    assert hasattr(B.load(), "sp1b200_lookup_traces") and "sp1b200_lookup_traces" in B.ERR_FUNCS
