"""oracle/lle_composite_oracle.py, the composite-operator form of oracle/lle_oracle.py (lle_composite: eigsh on -M^T M as a LinearOperator, dense eigh at small n)
pinned against the explicit oracle lle_dense, the reference class outputs tests/golden/ref_lle_*.npz and the reference's
Karate golden.  CPU only."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import REPO, golden_path, load_karate_nx

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import lap_oracle as lo
import lle_composite_oracle as lc
import lle_oracle as le


def _adj_from_npz(z):
    e, n = z['edges'], int(z['n'])
    return sp.csr_matrix((e[:, 2], (e[:, 0].astype(int), e[:, 1].astype(int))), shape=(n, n))


def _gap_ok(s, j, bar):
    lo_gap = s[j + 1] ** 2 - s[j] ** 2
    hi_gap = (s[j + 2] ** 2 - s[j + 1] ** 2) if j + 2 < len(s) else 1.0
    return min(lo_gap, hi_gap) > bar


@pytest.mark.parametrize('name,d', [('karate', 2), ('karate', 4), ('sbm1024', 16), ('randw120', 8)])
@pytest.mark.parametrize('dense_max', [2000, 0])          # dense eigh, and eigsh on the LinearOperator
def test_composite_matches_explicit_and_reference(name, d, dense_max):
    z = np.load(golden_path('ref_lle_%s_d%d.npz' % (name, d)))
    A = _adj_from_npz(z)
    X, s, V = lc.lle_composite(A, d, dense_max=dense_max)
    Xe, se, Ve = le.lle_dense(A, d)
    assert np.allclose(s ** 2, se ** 2, atol=1e-10), np.abs(s ** 2 - se ** 2).max()
    assert s[0] < 1e-6                                     # rows of P sum to one: sigma_0 = 0
    ref = np.real(z['X'])
    for j in range(d):
        if _gap_ok(se, j, 1e-6):
            assert np.allclose(lo.align_signs(X[:, j:j + 1], Xe[:, j:j + 1]), Xe[:, j:j + 1], atol=1e-7)
    Q = np.linalg.qr(ref)[0]
    assert np.linalg.norm(X - Q @ (Q.T @ X), 2) < 1e-6
    res, nrm = lc.composite_residuals(A, V, s)
    assert res.max() < 1e-8 and nrm > 0


def test_karate_golden():
    import networkx as nx
    G = load_karate_nx()
    A = nx.to_scipy_sparse_array(G, nodelist=list(G.nodes), weight='weight', format='csr')
    gold = np.loadtxt(golden_path('karate_LocallyLinearEmbedding.txt'))
    for dense_max in (2000, 0):
        X, s, V = lc.lle_composite(A, 2, dense_max=dense_max)
        assert np.allclose(lo.align_signs(X, gold), gold, atol=1e-7), np.abs(lo.align_signs(X, gold) - gold).max()


def test_residual_helper_sees_a_wrong_pair():
    z = np.load(golden_path('ref_lle_randw120_d8.npz'))
    A = _adj_from_npz(z)
    X, s, V = lc.lle_composite(A, 8)
    good, nrm = lc.composite_residuals(A, V, s)
    bad, _ = lc.composite_residuals(A, V, s * 1.1)
    M = le.lle_matrix(A).toarray()
    assert abs(nrm - np.linalg.norm(M, 2) ** 2) < 1e-6 * nrm
    assert good.max() < 1e-10 and bad[1:].min() > 1e-4
