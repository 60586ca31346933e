"""The rounds of the Chebyshev HOPE solve (algorithm 2) keep their results bit for bit however their steps are scheduled.

tests/golden/hope_rounds.npz (make_golden_hope_rounds.py) holds the output of the build that computed the stop rule's
residuals z^T (AV)^T (AV) z - l^2 on the host from two matrices it read back, symmetrised the Rayleigh-Ritz matrix in a
kernel of its own and extracted X with one apply launch per half.  The solver now forms the quadratic forms on the
device (ritz_quadform_kernel, same order of the fp64 sums), symmetrises while the Jacobi kernel loads its matrix, and
extracts whole rows of X with one launch over [M1 | M2]: same arithmetic per element, so X, sigma, the residual estimate
and the number of rounds and sweeps must be equal, not close."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, golden_path

sys.path.insert(0, GOLDEN)
import make_golden_hope_rounds as mk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def gold():
    return np.load(golden_path('hope_rounds.npz'))


def test_sbm_solve_is_bit_identical_with_one_launch_extraction(gpu_ctx, gold):
    """n = 20 000 (tensor-core Gram / apply), bench solver setting: filtered rounds, residual stop rule, d = 128 > b."""
    rows, Xs, sig, st = mk.sbm_case(gpu_ctx)
    assert (st['iters'], st['spmm_count']) == (int(gold['sbm_iters']), int(gold['sbm_spmm']))
    assert np.array_equal(rows, gold['sbm_rows'])
    assert np.array_equal(sig, gold['sbm_sigma'])
    assert np.array_equal(Xs, gold['sbm_X'])
    assert np.float32(st['resid_est']) == gold['sbm_resid_est']
    assert np.float32(st['ritz_change']) == gold['sbm_ritz_change']


def test_solve_that_drops_and_refills_columns_is_bit_identical(gpu_ctx, gold):
    """Undirected Karate: block width 36 > 34 nodes, so the rank test drops columns in every orthonormalisation and the
    refill reads the rank back between the round's steps (CUDA-core Gram / apply below 4096 rows)."""
    X, sig, st = mk.karate_case(gpu_ctx)
    assert st['iters'] == int(gold['karate_iters'])
    assert np.array_equal(sig, gold['karate_sigma'])
    assert np.array_equal(X, gold['karate_X'])
    assert np.float32(st['resid_est']) == gold['karate_resid_est']
    assert np.float32(st['ritz_change']) == gold['karate_ritz_change']
