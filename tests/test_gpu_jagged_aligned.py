"""GPU parity tests (jagged PCS) for the rounds summed straight from the base-field trace: K = the number of Hadamard sumcheck
rounds that never materialise the extension-field arrays, chosen by the library from the column alignment (2^K divides every
column prefix sum), log_stacking_height and log_m.  K = 0 (some column starts at an odd index) is the same path with no trace
rounds: the fold pass to level 0 sums round 0.  Each case names the K it reaches and is checked word for word against the
oracle through the same harness as tests/test_gpu_jagged.py (gpu_prove.check_jagged)."""
import pytest

from tests.gpu_prove import check_jagged, trace_rounds_k

pytestmark = pytest.mark.gpu

CASES = [
    # column starts aligned exactly to 2, 4, 8, 16 and 32 (K = 1 .. 5), empty chips in between
    ("align2", [[(6, 3), (0, 2), (10, 2)], [(18, 5)]], 4, 5, 1),
    ("align4", [[(12, 3), (20, 2)], [(0, 1), (36, 2), (4, 7)]], 4, 6, 2),
    ("align8", [[(24, 2), (8, 5), (0, 3)], [(40, 3)]], 5, 6, 3),
    ("align16", [[(48, 3), (0, 4), (16, 2)], [(80, 2), (16, 9)]], 6, 7, 4),
    ("align32", [[(96, 2), (32, 3)], [(0, 2), (160, 4), (32, 5)]], 6, 8, 5),
    # log_m = 5 = the alignment: K is clamped by log_m - 1
    ("clamp_log_m", [[(32, 1)]], 5, 5, 4),
    # log_stacking_height 3 below the alignment of 32
    ("clamp_stacking", [[(32, 3), (64, 2)], [(96, 1)]], 3, 7, 3),
    # two rounds; the first round's segment ends where a 2^5 block ends (segment boundary inside the rounds' blocks)
    ("segment_boundary", [[(32, 1)], [(64, 2), (0, 3), (32, 3)]], 5, 6, 5),
    # heights of 2^12 rows, 2^12 stacking: several runs of 2^10 rows per column (the eq_hi factor changes inside a column)
    ("row_runs", [[(4096, 3), (2048 + 32, 5), (0, 2)], [(1024, 7), (4096, 2)]], 12, 12, 5),
    # odd heights (K = 0), several runs of 2^10 rows per column
    ("unaligned", [[(4096 - 1, 3), (0, 2), (2048 + 5, 2)], [(1024 + 3, 5)]], 12, 12, 0),
]


@pytest.mark.parametrize("name,shapes,log_stack,mlr,k", CASES, ids=[c[0] for c in CASES])
def test_jagged_trace_rounds_match_oracle(name, shapes, log_stack, mlr, k):
    assert trace_rounds_k(shapes, log_stack, mlr) == k, name
    check_jagged(shapes, log_stack, mlr, seed=900 + log_stack + mlr + k)


@pytest.mark.parametrize("shapes,log_stack,mlr,k", [
    ([[(2 ** 16 + 1, 9), (0, 3), (2 ** 15 + 7, 7)], [(2 ** 16 - 31, 12)]], 16, 17, 0),  # log_m = 21
    ([[(2 ** 16 + 2, 9), (0, 3), (2 ** 15 + 6, 7)], [(2 ** 16 - 30, 12)]], 16, 17, 1),  # log_m = 21
    ([[(2 ** 20, 9), (0, 2), (2 ** 19 + 32, 7)], [(2 ** 20 - 160, 10)]], 20, 20, 5),    # log_m = 25
], ids=["k0", "k1", "k5"])
def test_jagged_trace_rounds_grid_loops(shapes, log_stack, mlr, k):
    # the fold pass to level K writes 2^(log_m - K) entries: 2^20 pairs for k0 and 2^19 for k1 and k5, so each of its 132 x 8
    # blocks of 256 threads loops over the grid; every warp of the trace-round passes walks a span of many blocks
    assert trace_rounds_k(shapes, log_stack, mlr) == k
    check_jagged(shapes, log_stack, mlr, seed=913 + k)
