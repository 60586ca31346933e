"""oracle/eval_gauss_oracle.py (the Gaussian score of LaplacianEigenmaps / LocallyLinearEmbedding) pinned against the
reference's own evaluation functions: goldens made by tests/golden/make_golden_eval_gauss.py with the unmodified
gem.evaluation.evaluate_graph_reconstruction, at the bar of test_oracle_eval.py."""
import os
import sys

import numpy as np
import pytest

from conftest import REPO
from gauss_golden import gauss_golden

sys.path.insert(0, os.path.join(REPO, 'oracle'))

CASES = [('eval_karate_lap', ('und', 'dir', 'dirw')), ('eval_karate_lle', ('und', 'dir', 'dirw')),
         ('eval_randw200_gauss', ('und', 'dir', 'dirw')), ('eval_sbm1024_lap', ('und',))]


@pytest.mark.parametrize('name,variants', CASES)
def test_gaussian_oracle_matches_reference_evaluation(eval_oracle, name, variants):
    import eval_gauss_oracle as go
    eo = eval_oracle
    z, n, (indptr, indices, w) = gauss_golden(name)
    assert str(z['score']) == 'gaussian'
    edges = eo.EdgeSet(n, indptr, indices)
    adj = go.reconstruct_gaussian(z['X'], exact=True)
    for tag in variants:
        und = tag == 'und'
        r = eo.evaluate(adj, edges, weights=w, is_undirected=und, is_weighted=(tag == 'dirw'), node_order=z['nodes'])
        assert r['n_pred'] == int(z[tag + '_n_pred'])
        assert abs(r['MAP'] - float(z[tag + '_MAP'])) < 1e-13
        assert np.array_equal(r['prec_curve'][:4096], z[tag + '_prec_head'])
        assert np.array_equal(r['prec_curve'][::997], z[tag + '_prec_stride'])
        if tag == 'dirw':
            assert abs(r['err'] - float(z[tag + '_err'])) < 1e-10
            assert abs(r['err_baseline'] - float(z[tag + '_err_baseline'])) < 1e-12


@pytest.mark.parametrize('name', ['eval_karate_lap', 'eval_karate_lle', 'eval_randw200_gauss'])
def test_vectorised_gaussian_equals_the_loops(name):
    import eval_gauss_oracle as go
    z, _, _ = gauss_golden(name)
    A = go.reconstruct_gaussian(z['X'], exact=True)
    B = go.reconstruct_gaussian(z['X'], exact=False)
    assert np.all(np.diag(A) == 0) and np.all(np.diag(B) == 0)
    assert np.array_equal(A == 0, B == 0)                     # the same entries underflow
    assert np.allclose(A, B, rtol=1e-13, atol=0)


def test_randw200_golden_has_ties_and_underflow():
    """The random case exercises what it was built for: exact delta = 0 ties and scores that underflow to 0."""
    import eval_gauss_oracle as go
    z, n, _ = gauss_golden('eval_randw200_gauss')
    A = go.reconstruct_gaussian(z['X'], exact=False)
    off = ~np.eye(n, dtype=bool)
    assert np.sum((A == 1.0) & off) >= 60
    assert np.sum((A == 0.0) & off) >= 3000
    assert int(z['und_n_pred']) == n * (n - 1) // 2 - np.sum(np.triu(A == 0.0, 1))
