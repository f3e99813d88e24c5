"""CPU tests of the program setup's table generators: the NumPy restatement (tests/program_ref.py) against rows checked by hand, and the C
records of the instruction list (sp1b200_instruction) against what sp1_b200.lib packs."""
import os
import subprocess
import tempfile

import numpy as np

from tests import program_ref as PR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64_MAX = (1 << 64) - 1


def test_byte_rows_checked_by_hand():
    t = PR.byte_trace()
    assert t.shape == (1 << 16, 7)
    #            b     c     and   or    xor   ltu msb
    want = {(0x00, 0x00): (0x00, 0x00, 0x00, 0x00, 0x00, 0, 0),
            (0xFF, 0x01): (0xFF, 0x01, 0x01, 0xFF, 0xFE, 0, 1),
            (0x01, 0xFF): (0x01, 0xFF, 0x01, 0xFF, 0xFE, 1, 0),
            (0x80, 0x7F): (0x80, 0x7F, 0x00, 0xFF, 0xFF, 0, 1),
            (0xFF, 0xFF): (0xFF, 0xFF, 0xFF, 0xFF, 0x00, 0, 1)}
    for (b, c), row in want.items():
        assert tuple(int(v) for v in t[256 * b + c]) == row, (b, c)


def test_range_rows_checked_by_hand():
    t = PR.range_trace()
    assert t.shape == (1 << 17, 2)
    want = {0: (0, 0), 1: (0, 0), 2: (0, 1), 3: (1, 1), 4: (0, 2), 1 << 16: (0, 16), (1 << 17) - 1: ((1 << 16) - 1, 16)}
    for r, row in want.items():
        assert tuple(int(v) for v in t[r]) == row, r


def test_program_rows_and_padding_checked_by_hand():
    from sp1_b200.lib import pack_instructions
    pc_base = (1 << 48) - 16
    instrs = pack_instructions(opcode=[52, 0, 1], op_a=[0, 31, 5], op_b=[U64_MAX, 0x0001_0002_0003_0004, 0],
                               op_c=[U64_MAX, 5, U64_MAX], imm_b=[1, 0, 0], imm_c=[1, 0, 1])
    t = PR.program_trace(pc_base, instrs)
    assert t.shape == (32, 16)
    #       pc[3]                   opcode op_a op_b[4]                         op_c[4]                         op_a_0 imm_b imm_c
    row0 = [0xFFF0, 0xFFFF, 0xFFFF, 52, 0, 0xFFFF, 0xFFFF, 0xFFFF, 0xFFFF, 0xFFFF, 0xFFFF, 0xFFFF, 0xFFFF, 1, 1, 1]
    row1 = [0xFFF4, 0xFFFF, 0xFFFF, 0, 31, 4, 3, 2, 1, 5, 0, 0, 0, 0, 0, 0]
    row2 = [0xFFF8, 0xFFFF, 0xFFFF, 1, 5, 0, 0, 0, 0, 0xFFFF, 0xFFFF, 0xFFFF, 0xFFFF, 0, 0, 1]
    assert [int(v) for v in t[0]] == row0
    assert [int(v) for v in t[1]] == row1
    assert [int(v) for v in t[2]] == row2
    for r in range(3, 32):   # padding rows repeat row 0, its pc included
        assert [int(v) for v in t[r]] == row0, r


def test_program_heights():
    assert [PR.next_multiple_of_32(n) for n in (1, 15, 16, 17, 31, 32, 33, 1000)] == [32, 32, 32, 32, 32, 32, 64, 1024]
    assert PR.next_multiple_of_32(0) == 16


def test_dense_layout_is_byte_program_range_column_major():
    from sp1_b200.lib import pack_instructions
    instrs = pack_instructions(opcode=[3] * 40, op_a=np.arange(40), op_b=np.arange(40) << 20, op_c=7, imm_b=0, imm_c=1)
    words, shapes = PR.dense(0x1000, instrs)
    assert shapes == [(1 << 16, 7), (64, 16), (1 << 17, 2)]
    assert words.size == 7 * (1 << 16) + 16 * 64 + 2 * (1 << 17)
    prog = words[7 << 16: (7 << 16) + 16 * 64].reshape(16, 64)   # column-major: column k is a row of this view
    assert (prog[4, :40] == PR.to_monty(np.arange(40))).all()    # op_a
    assert (prog[0, 40:] == PR.to_monty(0x1000)).all()            # padding pc = pc_base


def test_instruction_record_layout_matches_the_header():
    """sizeof / offsetof of sp1b200_instruction, compiled from include/sp1b200.h, equal the numpy record lib.py packs"""
    from sp1_b200.lib import INSTRUCTION_DTYPE
    src = r'''#include <stdio.h>
#include <stddef.h>
#include "sp1b200.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(sp1b200_instruction), offsetof(sp1b200_instruction, opcode),
           offsetof(sp1b200_instruction, op_a), offsetof(sp1b200_instruction, imm_b), offsetof(sp1b200_instruction, imm_c),
           offsetof(sp1b200_instruction, pad), offsetof(sp1b200_instruction, op_b), offsetof(sp1b200_instruction, op_c));
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "layout.c"), "w") as f:
            f.write(src)
        exe = os.path.join(d, "layout")
        subprocess.run(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", exe, os.path.join(d, "layout.c")], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    f = INSTRUCTION_DTYPE.fields
    assert got == [INSTRUCTION_DTYPE.itemsize] + [f[n][1] for n in ("opcode", "op_a", "imm_b", "imm_c", "pad", "op_b", "op_c")]


def test_program_setup_symbols_are_exported():
    from sp1_b200 import lib as B
    L = B.load()
    for s in ("sp1b200_program_preprocessed_traces", "sp1b200_program_setup"):
        assert hasattr(L, s), s
        assert s in B.ERR_FUNCS
