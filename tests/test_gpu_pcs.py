"""GPU parity tests (PCS level): stacked commit + BaseFold evaluation proof through the C ABI vs the oracle.
Bit-exact: commitments, every proof word, and the post-proof challenger state.  The oracle also runs the restated
reference verifier on its own proof, so equality here implies the CUDA proof verifies."""
import pytest

from tests.gpu_prove import check_stacked

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("ncols,log_h", [([1], 1), ([3], 4), ([2, 5], 5), ([9, 17], 8), ([33], 10)])
def test_stacked_basefold_matches_oracle(ncols, log_h):
    check_stacked(ncols, log_h, nq=10, pow_bits=6, batch_bits=3, seed=1000 + log_h)


def test_stacked_basefold_two_step_ntt_sizes():
    # log_h = 13 exercises the strided (step A) + contiguous (step B) split of the RS-encode kernels
    check_stacked([3, 2], 13, nq=16, pow_bits=8, batch_bits=5, seed=77)


def test_recomputed_codeword_and_device_input():
    check_stacked([4, 3], 9, nq=12, pow_bits=5, batch_bits=2, seed=78, keep_codeword=False, device_input=True)


def test_core_parameters_small_trace():
    # real FRI parameters (124 queries, 16 + 5 PoW bits) on a reduced stacking height
    check_stacked([5, 11], 12, nq=124, pow_bits=16, batch_bits=5, seed=79)
