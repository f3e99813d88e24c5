"""GPU tests of the program setup (sp1b200_program_vk_tail): the 24-word vk_tail of a memory image (and page image) equals pc_start, the
oracle's restated Program::initial_global_cumulative_sum and the untrusted-programs word, for images from empty to 2^20 entries, from
host and device memory and in any entry order; duplicate keys and NULL arrays are errors that leave the context usable; the key digest
of the produced tail is the oracle's sponge; a core proof verifies against the key of its image and not against the key of a changed
image; a poisoned context pool gives the same tail."""
import ctypes as C

import numpy as np
import pytest

from tests import core_chain as CC
from tests import lift_oracle_lib as LO
from tests import machines as M
from tests import oracle_lib as O
from tests import recursion_ref as RR
from tests import septic as S
from tests.provers import Core, specs_machine

pytestmark = pytest.mark.gpu

V_GLOBAL_CUMULATIVE_SUM = 74


def _lib():
    from sp1_b200 import Lib
    return Lib(0)


def _image(n, seed):
    """n unique 48-bit addresses (word-aligned, as a program's) and random u64 words"""
    rng = np.random.default_rng(seed)
    addrs = rng.choice(1 << 45, n, replace=False).astype(np.uint64) << np.uint64(3)
    return addrs, rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)


def _pages(n, seed):
    rng = np.random.default_rng(seed)
    return rng.choice(1 << 36, n, replace=False).astype(np.uint64), rng.integers(0, 8, n).astype(np.uint8)


def _expected(pc_start_abs, addrs, words, pages=None, prots=None, untrusted=0):
    s = LO.initial_global_cumulative_sum(addrs, words, pages, prots, untrusted)
    pc = O.to_monty(np.array([pc_start_abs & 0xFFFF, (pc_start_abs >> 16) & 0xFFFF, (pc_start_abs >> 32) & 0xFFFF], np.uint32))
    return np.concatenate([pc, s, O.to_monty(np.array([untrusted], np.uint32)), np.zeros(6, np.uint32)])


@pytest.mark.parametrize("n", [0, 1, 2, 3, 255, 256, 257, 4097, 1 << 20])
def test_tail_matches_the_oracle(n):
    lib = _lib()
    addrs, words = _image(n, 9000 + n)
    pages, prots = _pages(17, 9100 + n)
    pc = 0x0000_7654_3210_2468 + 4 * n
    got = lib.program_vk_tail(pc, addrs, words, pages, prots, 0)   # pages are not read without untrusted programs
    assert (got == _expected(pc, addrs, words)).all()
    if n == 0:
        assert (got[3:17] == S.pt_words(S.ZERO)).all()   # SepticDigest::zero()
    lib.close()


@pytest.mark.parametrize("n_mem,n_pages", [(0, 1), (1, 1), (300, 40), (4097, 513)])
def test_tail_with_untrusted_programs_matches_the_oracle(n_mem, n_pages):
    lib = _lib()
    addrs, words = _image(n_mem, 9200 + n_mem)
    pages, prots = _pages(n_pages, 9300 + n_pages)
    got = lib.program_vk_tail(0x2000, addrs, words, pages, prots, 1)
    assert (got == _expected(0x2000, addrs, words, pages, prots, 1)).all()
    assert got[17] == O.to_monty(np.array([1], np.uint32))[0]
    lib.close()


def test_device_pointers_and_entry_order_give_the_same_tail():
    import torch
    lib = _lib()
    addrs, words = _image(5000, 9400)
    pages, prots = _pages(300, 9401)
    want = lib.program_vk_tail(0x10074, addrs, words, pages, prots, 1)
    dev = lambda a: torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()
    assert (lib.program_vk_tail(0x10074, dev(addrs), dev(words), dev(pages), dev(prots), 1) == want).all()
    perm, pperm = np.random.default_rng(1).permutation(5000), np.random.default_rng(2).permutation(300)
    assert (lib.program_vk_tail(0x10074, addrs[perm], words[perm], pages[pperm], prots[pperm], 1) == want).all()
    assert (want == _expected(0x10074, addrs, words, pages, prots, 1)).all()
    lib.close()


def test_errors_name_the_key_and_leave_the_context_usable():
    from sp1_b200.lib import Sp1B200Error
    lib = _lib()
    addrs, words = _image(1000, 9500)
    pages, prots = _pages(100, 9501)
    want = _expected(0x4000, addrs, words, pages, prots, 1)
    dup = addrs.copy(); dup[700] = dup[123]
    with pytest.raises(Sp1B200Error, match=f"duplicate memory address 0x{int(addrs[123]):x}"):
        lib.program_vk_tail(0x4000, dup, words, pages, prots, 1)
    assert (lib.program_vk_tail(0x4000, addrs, words, pages, prots, 1) == want).all()
    pdup = pages.copy(); pdup[99] = pdup[0]
    with pytest.raises(Sp1B200Error, match=f"duplicate page index 0x{int(pages[0]):x}"):
        lib.program_vk_tail(0x4000, addrs, words, pdup, prots, 1)
    assert (lib.program_vk_tail(0x4000, addrs, words, pages, prots, 1) == want).all()
    out = np.zeros(24, np.uint32)
    for args in ((None, C.c_void_p(words.ctypes.data), 5, None, None, 0),
                 (C.c_void_p(addrs.ctypes.data), C.c_void_p(words.ctypes.data), 5, None, C.c_void_p(prots.ctypes.data), 3)):
        a, w, n, p, pr, npg = args
        e = lib.L.sp1b200_program_vk_tail(lib.ctx, C.c_uint64(0), a, w, C.c_uint64(n), p, pr, C.c_uint64(npg), C.c_int(1),
                                          C.c_void_p(out.ctypes.data))
        assert e and b"NULL" in e
        assert (lib.program_vk_tail(0x4000, addrs, words, pages, prots, 1) == want).all()
    lib.close()


def test_key_digest_of_the_produced_tail_is_the_oracle_sponge():
    from sp1_b200 import lib as B
    lib = _lib()
    addrs, words = _image(777, 9600)
    tail = lib.program_vk_tail(0x20_0000, addrs, words)
    commit = O.rand_field(np.random.default_rng(9601), 8)
    assert (B.vk_hash(commit, tail) == RR.vk_hash(np.concatenate([commit, tail]))).all()
    lib.close()


def test_core_proof_verifies_against_the_key_of_its_image():
    """a core chain whose key takes its initial sum from an image, the last shard's global cumulative sum chosen so that the total is the
    zero digest: accepted; the key of the image with one word changed: rejected by the cumulative-sum check"""
    pvs, tail = CC.chain(3, 9700)
    initial0 = (tail[3:10], tail[10:17])
    c = Core(specs_machine(M.NO_PREP), 7, 8)
    addrs, words = _image(2000, 9701)
    pc_abs = tail[0] | (tail[1] << 16) | (tail[2] << 32)
    img_tail = c.lib.program_vk_tail(pc_abs, addrs, words)
    initial = S.words_pt(img_tail[3:17])
    # I0 + d_1 + ... + d_n - n zero = zero (group sums) stays true with I0 -> I and d_n -> d_n + I0 - I
    g = CC.getf(pvs[-1], "global_cumulative_sum")
    d = S.curve_add(S.curve_add((g[:7], g[7:]), initial0), S.curve_neg(initial))
    CC.setf(pvs[-1], "global_cumulative_sum", list(d[0]) + list(d[1]))
    canon_tail = [int(v) for v in O.from_monty(img_tail)]
    assert canon_tail[:3] == tail[:3] and canon_tail[17:] == tail[17:]
    words_, _, mtail = c.prove(pvs, canon_tail)
    assert (mtail == img_tail).all()
    v, shard, sv, _ = c.verify(words_, img_tail)
    assert (v, shard, sv) == (0, 0, 0)
    changed = words.copy(); changed[1234] ^= np.uint64(1 << 40)
    bad_tail = c.lib.program_vk_tail(pc_abs, addrs, changed)
    assert not (bad_tail[3:17] == img_tail[3:17]).all()
    v, shard, _, _ = c.verify(words_, bad_tail)
    assert (v, shard) == (V_GLOBAL_CUMULATIVE_SUM, 3)
    c.close()


def test_poisoned_pool_gives_the_same_tail():
    """every block of the context's pool holds a non-zero pattern before the call (a freed pool keeps its blocks)"""
    lib = _lib()
    addrs, words = _image(1 << 16, 9800)
    pages, prots = _pages(4096, 9801)
    want = _expected(0x8000, addrs, words, pages, prots, 1)
    blocks = []
    for size in [256 << k for k in range(0, 18)] * 2 + [64 << 20, 64 << 20]:
        p = C.c_void_p()
        lib._chk(lib.L.sp1b200_malloc(lib.ctx, C.c_size_t(size), C.byref(p)))
        fill = np.full(size // 4, 0x7effffff, np.uint32)
        lib._chk(lib.L.sp1b200_memcpy_h2d(lib.ctx, p, C.c_void_p(fill.ctypes.data), C.c_size_t(size)))
        lib.sync()
        blocks.append(p)
    for p in blocks:
        lib._chk(lib.L.sp1b200_free(lib.ctx, p))
    lib.sync()
    assert (lib.program_vk_tail(0x8000, addrs, words, pages, prots, 1) == want).all()
    lib.close()
