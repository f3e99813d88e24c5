"""Static checks of the code ptxas generates for the hot kernels (no GPU needed: nvcc cross-compiles sm_90a, cuobjdump reads the objects).
The measured speed of these kernels follows their instruction mix (DESIGN.md 3.1: the Poseidon2 kernels run at the throughput of the fmaheavy
pipe, time proportional to the IMAD* slot count), so the mix is pinned here: a compiler flag, a header change or a refactor that silently
brings back the 64-bit-addend s-box reduction, spills the sponge state or drops the occupancy of the NTT tiles fails on the CPU, before any
GPU time is spent.  Skipped where the build directory is absent (the GPU box receives the built .so only)."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "sp1_b200", "csrc", "build")

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(BUILD, "merkle.o")) or shutil.which("cuobjdump") is None,
                                reason="needs the build directory and cuobjdump")


def _ptxas(tu):
    """{demangled kernel name fragment: (registers, spill store bytes, shared bytes)} from the -Xptxas -v log of a translation unit"""
    out, cur = {}, None
    for line in open(os.path.join(BUILD, tu + ".ptxas.log")):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            out[cur] = [None, None, 0]
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m:
            out[cur][1] = int(m.group(1))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            out[cur][0] = int(m.group(1))
            sm = re.search(r"(\d+) bytes smem", line)
            out[cur][2] = int(sm.group(1)) if sm else 0
    return out


def _find(table, frag):
    hits = [v for k, v in table.items() if frag in k]
    assert len(hits) == 1, (frag, [k for k in table if frag in k])
    return hits[0]


def test_poseidon2_kernels_keep_the_state_in_registers_at_full_occupancy():
    t = _ptxas("merkle")
    for k in ("16leaf_hash_kernel", "compress_layer_kernel", "permute_states_kernel"):   # 16 = Itanium length prefix (not fri_leaf_hash_kernel)
        regs, spill, _ = _find(t, k)
        assert regs <= 32 and spill == 0, (k, regs, spill)      # 32 registers x 256 threads -> 2048 threads per SM
    regs, spill, _ = _find(t, "20fri_leaf_hash_kernel")
    assert regs <= 40 and spill == 0


def test_rs_encode_tiles_keep_their_occupancy():
    t = _ptxas("ntt")
    regs, spill, _ = _find(t, "rs_step_a_fastILi10ELi2")
    assert regs <= 32 and spill <= 64            # two 1024-thread tiles per SM (a handful of spilled words is the measured optimum)
    regs, spill, smem = _find(t, "rs_step_b_2048")
    assert regs <= 32 and spill == 0 and smem == 8192


def test_jagged_fold_to_kernels_keep_their_shared_memory():
    """the level-0 fold pass (odd column starts) needs an eq_lo table of 2^10 EF; the instances the aligned traces run keep 2^9,
    so their occupancy does not change with it"""
    t = _ptxas("jagged")
    for k in range(6):
        regs, spill, smem = _find(t, f"jagged_fold_to_kernelILi{k}E")
        assert spill == 0 and smem == (16640 if k == 0 else 8448), (k, regs, spill, smem)


def test_permutation_instruction_mix():
    """dynamic opcode histogram of one permutation (tools/sass_dyn.py, loop trip counts 4 / 5 / 4): the subtractive s-box reduction keeps it
    at ~4.9 k instructions (round-1 code: 5 456) with no IMAD.MOV negations and (almost) no IMAD.X carries, 296 wide products"""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_dyn.py"), os.path.join(BUILD, "merkle.o"), "permute_states_kernel", "4,5,4"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    hist = {}
    for line in r.stdout.splitlines():
        p = line.split()
        if len(p) >= 2 and re.fullmatch(r"[\d.]+", p[1]):
            hist[p[0]] = float(p[1])
    total = float(re.search(r"total ([\d.]+) instr", r.stdout).group(1))
    assert 4700 <= total <= 5000, total
    assert hist.get("IMAD.MOV", 0) <= 20 and hist.get("IMAD.X", 0) <= 40, hist
    assert 290 <= hist.get("IMAD.WIDE", 0) <= 310 and 620 <= hist.get("IMAD.HI", 0) <= 650, hist
    # multiplier-pipe slots per permutation (IMAD* = 1, IMAD.HI = 2, IMAD.WIDE = 2.65, the slot costs tools/pipe_mix.cu measures); round-1 code: 3 724
    slots = sum(v for k, v in hist.items() if k.startswith("IMAD") and k not in ("IMAD.HI", "IMAD.WIDE")) + 2 * hist["IMAD.HI"] + 2.65 * hist["IMAD.WIDE"]
    assert slots <= 3500, slots
