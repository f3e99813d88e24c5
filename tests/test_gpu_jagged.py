"""GPU parity tests (jagged PCS): commit of chip tables, column claims, Hadamard + branching-program sumchecks and the
stacked/BaseFold proof through the C ABI vs the oracle (which also runs the restated JaggedPcsVerifier)."""
import pytest

from tests.gpu_prove import check_jagged

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shapes,log_stack,mlr", [
    ([[(5, 3), (0, 2), (8, 1)]], 3, 3),
    ([[(3, 2), (7, 1)], [(16, 2), (0, 4), (9, 3)]], 3, 4),
    ([[(1, 1)]], 2, 2),
    ([[(32, 5), (17, 3)], [(20, 7)]], 4, 5),
])
def test_jagged_matches_oracle_small(shapes, log_stack, mlr):
    check_jagged(shapes, log_stack, mlr, seed=600 + log_stack + mlr)


def test_jagged_matches_oracle_medium():
    # heights that are multiples of 32 (the reference's trace heights), two rounds, empty chips, 2^12 stacking height
    shapes = [[(4096, 3), (96, 17), (0, 5)], [(8192, 9), (2048 + 32, 40), (0, 3), (64, 13), (8192, 2)]]
    check_jagged(shapes, 12, 13, seed=77, nq=16, pow_bits=8, batch_bits=5)
