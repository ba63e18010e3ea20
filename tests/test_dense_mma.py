"""The in-tree blocked Cholesky (16 x 8 DMMA trailing updates and panel solves) at the LM bench's own dense size.

test_dense_cholesky_solve_matches_numpy covers small sizes against numpy's solve; this checks the normwise
backward error at n_d = 13 080 with 512-wide block columns (what one GPU factors per LM attempt at config 2) and
at an odd size near it whose last tiles and panel are partial."""
import numpy as np
import pytest

from camera_calibration_b200 import api

pytestmark = pytest.mark.gpu


def _spd(n, seed):
    # symmetric random matrix shifted past its spectral radius (condition number about 10); O(n^2) to make
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    A += A.T
    A *= 0.5
    A[np.diag_indices(n)] += 1.2 * np.sqrt(2.0 * n)
    return A, rng.standard_normal(n)


@pytest.mark.parametrize("n", [13080, 13001])
def test_dense_cholesky_backward_error_at_bench_size(n):
    A, b = _spd(n, n)
    x, _, _ = api.dense_cholesky_solve(A, b, 512)
    inf = lambda v: np.linalg.norm(v, np.inf)
    berr = inf(A @ x - b) / (inf(A) * inf(x) + inf(b))
    assert berr <= 1e-13, berr
