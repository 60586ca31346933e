"""oracle/gf_oracle.py pinned BIT-FOR-BIT against the unmodified reference class gem.embedding.gf.GraphFactorization run with a
seeded global NumPy RNG (tests/golden/ref_gf_*.npz, made by tests/golden/make_golden_gf.py).  CPU only."""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, golden_path

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import gf_oracle as go


@pytest.mark.parametrize('name', ['ref_gf_karate_d2_it300', 'ref_gf_randw60_d8_it60', 'ref_gf_randw60_d128_it60'])
def test_reference_class_outputs_bit_exact(name):
    z = np.load(golden_path(name + '.npz'))
    e = z['edges']
    X = go.gf_sequential(int(z['n']), e[:, 0].astype(int), e[:, 1].astype(int), e[:, 2], z['X0'].shape[1], float(z['eta']),
                         float(z['regu']), int(z['max_iter']), z['X0'])
    assert np.array_equal(X, z['X'])


def test_rows_schedule_equals_the_reference_sweep_on_row_major_edge_lists():
    """gemb_gf mode 1 (rows in parallel, partners from the previous epoch's table) IS the reference's sequential sweep whenever the
    edge list is grouped by ascending source: only j > i is read, and row j > i has not been touched yet in the current epoch."""
    z = np.load(golden_path('ref_gf_randw60_d8_it60.npz'))
    e = z['edges']
    order = np.lexsort((np.arange(len(e)), e[:, 0]))         # grouped by source, input order inside a row
    es = e[order]
    args = lambda ee: (int(z['n']), ee[:, 0].astype(int), ee[:, 1].astype(int), ee[:, 2], 8, float(z['eta']), float(z['regu']),
                       int(z['max_iter']), z['X0'])
    assert np.array_equal(go.gf_sequential(*args(es)), go.gf_rows_jacobi(*args(es)))
    # a different edge order is a different (equally valid) SGD schedule
    rev = es[::-1]
    assert not np.array_equal(go.gf_sequential(*args(rev)), go.gf_sequential(*args(es)))
