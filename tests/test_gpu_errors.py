"""Error behaviour of the C ABI on a GPU box: every fallible entry point returns a message (raised as Sp1B200Error by the ctypes mirror) instead
of reading out of bounds, hanging or silently accepting bad input — the reference's FFI convention (CudaRustError, sys/src/runtime.rs:5-20)."""
import numpy as np
import pytest

from tests import gpu_prove as GP
from tests import machines as M
from tests import oracle_lib as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from sp1_b200 import Lib
    L = Lib(0, log_stacking_height=10, max_log_row_count=11, num_queries=8, pow_bits=4, batch_pow_bits=2, gkr_pow_bits=3)
    yield L
    L.close()


def _machine(rng):
    spec = [(1024, 2, True), (256 + 32, 3, False), (2048, 1, True)]
    return M.spec_machine(rng, spec, names="Chip{:02d}")


def test_machine_create_rejects_malformed_blobs(lib):
    from sp1_b200.lib import Sp1B200Error
    rng = np.random.default_rng(1)
    blob, *_ = _machine(rng)
    good = lib.machine_create(blob)
    lib.machine_free(good)
    with pytest.raises(Sp1B200Error, match="truncated"):
        lib.machine_create(blob[:40].copy())
    # header word 4 of chip 0 = n_instrs: a count that overruns the blob (and would wrap a 32-bit size sum)
    bad = blob.copy(); bad[1 + 4] = 0x7FFFFFFF
    with pytest.raises(Sp1B200Error, match="truncated"):
        lib.machine_create(bad)
    # first leaf of chip 0: column far outside the main width  (records: 9 header words, then instrs, then leaves {source|pad, col})
    ni = int(blob[1 + 4])
    bad = blob.copy(); bad[1 + 9 + 2 * ni + 1] = 10_000
    with pytest.raises(Sp1B200Error, match="leaf column"):
        lib.machine_create(bad)
    # unknown opcode in the first instruction (low byte of the first instruction word)
    bad = blob.copy(); bad[1 + 9] = (int(bad[1 + 9]) & ~0xFF) | 0x2A
    with pytest.raises(Sp1B200Error, match="opcode"):
        lib.machine_create(bad)
    # operand register beyond n_regs in an arithmetic instruction: find the first ADD/SUB/MUL and blow up operand a
    for k in range(ni):
        w0 = int(blob[1 + 9 + 2 * k])
        if (w0 & 0xFF) in (3, 4, 5):
            bad = blob.copy(); bad[1 + 9 + 2 * k + 1] = (int(bad[1 + 9 + 2 * k + 1]) & 0xFFFF0000) | 0xFFFE
            with pytest.raises(Sp1B200Error, match="operand out of range"):
                lib.machine_create(bad)
            break
    else:
        pytest.fail("no arithmetic instruction found")
    # interaction section cut in the middle
    with pytest.raises(Sp1B200Error, match="interaction"):
        lib.machine_create(blob[:-7].copy())


def test_prove_shard_capacity_error_leaves_the_transcript_untouched(lib):
    """a too-small proof buffer reports the needed size and does NOT advance the caller's challenger (a retry with a larger buffer
    proves from the same transcript)"""
    from sp1_b200.lib import Sp1B200Error
    rng = np.random.default_rng(2)
    blob, heights, mains, preps, pv, names = _machine(rng)
    mach = lib.machine_create(blob)
    _, prep_round = GP.commit_prep(lib, preps)
    dense = M.dense_main(mains)
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 5))
    st = ch.st.copy()
    with pytest.raises(Sp1B200Error, match="capacity"):
        lib.prove_shard(mach, prep_round, dense, heights, names, pv, st, cap_words=1000)
    assert (st == ch.st).all(), "a failed call must not advance the challenger"
    words = lib.prove_shard(mach, prep_round, dense, heights, names, pv, st)
    st2 = ch.st.copy()
    again = lib.prove_shard(mach, prep_round, dense, heights, names, pv, st2)
    assert (words == again).all() and (st == st2).all()
    lib.jagged_round_free(prep_round)
    lib.machine_free(mach)


def test_shape_errors_are_reported(lib):
    from sp1_b200.lib import Sp1B200Error
    rng = np.random.default_rng(3)
    blob, heights, mains, preps, pv, names = _machine(rng)
    mach = lib.machine_create(blob)
    dense = M.dense_main(mains)
    st = O.Challenger().st.copy()
    # preprocessed round missing although the machine has preprocessed columns
    with pytest.raises(Sp1B200Error, match="preprocessed"):
        lib.prove_shard(mach, None, dense, heights, names, pv, st)
    # a table taller than 2^max_log_row_count
    with pytest.raises(Sp1B200Error, match="rows"):
        lib.jagged_commit_dense(np.zeros(8, np.uint32), [1 << 12], [1])
    # too few public values for the programs' LOAD_PUBLIC indices
    _, prep_round = GP.commit_prep(lib, preps)
    with pytest.raises(Sp1B200Error, match="public value"):
        lib.prove_shard(mach, prep_round, dense, heights, names, pv[:0], st)
    lib.jagged_round_free(prep_round)
    lib.machine_free(mach)


def test_context_rejects_a_missing_device():
    from sp1_b200 import Lib
    from sp1_b200.lib import Sp1B200Error
    with pytest.raises(Sp1B200Error, match="not present"):
        Lib(device=64)


def test_repeated_contexts_and_proofs_do_not_leak_device_memory():
    """create / prove / destroy in a loop: device memory in use returns to its starting level (contexts own their pools, slots,
    mailboxes; failure paths of ctx_create and jagged_commit release what they allocated)"""
    import torch
    from sp1_b200 import Lib
    rng = np.random.default_rng(4)
    blob, heights, mains, preps, pv, names = _machine(rng)
    dense = M.dense_main(mains)
    torch.cuda.synchronize()
    used = []
    ref = None
    for it in range(6):
        L = Lib(0, log_stacking_height=10, max_log_row_count=11, num_queries=8, pow_bits=4, batch_pow_bits=2, gkr_pow_bits=3)
        mach = L.machine_create(blob)
        _, prep_round = GP.commit_prep(L, preps)
        for _ in range(3):
            w = L.prove_shard(mach, prep_round, dense, heights, names, pv, O.Challenger().st.copy())
            if ref is None:
                ref = w
            assert (w == ref).all()
        L.jagged_round_free(prep_round)
        L.machine_free(mach)
        L.close()
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info(0)
        used.append(total - free)
    assert max(used[1:]) - min(used[1:]) < (64 << 20), used     # steady after the first iteration (CUDA context / module loading)
