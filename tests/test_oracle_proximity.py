"""oracle/proximity_oracle.py pinned on the CPU: common neighbours against networkx's count, Adamic-Adar against a brute-force
sum over z, rooted PageRank rows against networkx's personalised PageRank, the truncated series against the inverse, and
the matrix-free operator against the dense matrix."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import REPO, load_karate_nx, load_sbm1024_nx

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import proximity_oracle as po


def _karate_undirected():
    import networkx as nx
    G = nx.Graph(load_karate_nx().to_undirected())
    return G, nx.to_scipy_sparse_array(G, nodelist=list(G.nodes), weight=None, dtype=np.float64, format='csr')


def test_common_neighbors_is_networkx_count():
    import networkx as nx
    G, A = _karate_undirected()
    S = po.proximity_dense(A, 'common_neighbors')
    nodes = list(G.nodes)
    want = np.array([[len(list(nx.common_neighbors(G, i, j))) for j in nodes] for i in nodes], dtype=np.float64)
    np.fill_diagonal(want, np.diag(S))            # networkx has no pair (i, i); S_ii = deg(i)
    assert np.array_equal(S, want)
    assert np.array_equal(np.diag(S), np.asarray(A.sum(axis=1)).ravel())


def test_adamic_adar_is_the_brute_force_sum():
    A = po.random_digraph(n=40, seed=9, p=0.15)
    Ad = A.toarray()
    n = Ad.shape[0]
    deg = Ad.sum(axis=1) + Ad.sum(axis=0)
    D = np.array([1.0 / deg[z] if deg[z] > 0 else 0.0 for z in range(n)])
    want = np.zeros((n, n))
    for i in range(n):
        for j in range(n):
            want[i, j] = sum(Ad[i, z] * Ad[z, j] * D[z] for z in range(n))
    S = po.proximity_dense(A, 'adamic_adar')
    assert np.abs(S - want).max() <= 1e-14 * max(1.0, np.abs(want).max())
    assert D[7] == 0.0 and po.inv_degree(A)[7] == 0.0


@pytest.mark.parametrize('alpha', [0.5, 0.85])
def test_rooted_pagerank_rows_are_personalised_pagerank(alpha):
    import networkx as nx
    G, A = _karate_undirected()
    assert np.all(np.asarray(A.sum(axis=1)).ravel() > 0)          # no dangling nodes
    S = po.proximity_dense(A, 'rooted_pagerank', alpha=alpha)
    nodes = list(G.nodes)
    worst = 0.0
    for i, v in enumerate(nodes):
        pr = nx.pagerank(G, alpha=alpha, personalization={v: 1}, tol=1e-14, max_iter=1000, weight=None)
        worst = max(worst, np.abs(S[i] - np.array([pr[u] for u in nodes])).max())
    print('alpha %.2f: max |S_i - pagerank_i| = %.2e (bar 1e-10)' % (alpha, worst))
    assert worst < 1e-10
    assert np.allclose(S.sum(axis=1), 1.0, atol=1e-12)             # each row a distribution


@pytest.mark.parametrize('alpha', [0.3, 0.5, 0.85])
@pytest.mark.parametrize('katz_tol', [1e-7, 1e-10])
def test_truncated_series_matches_the_inverse_at_katz_tol(alpha, katz_tol):
    A = po.random_digraph()
    J = po.rooted_pagerank_terms(alpha, katz_tol)
    S = po.proximity_dense(A, 'rooted_pagerank', alpha=alpha)
    St = po.proximity_dense(A, 'rooted_pagerank', alpha=alpha, terms=J)
    err = np.abs(S - St).sum(axis=1).max()                          # ||.||_inf: the tail is alpha^(J+1) at most
    print('alpha %.2f tol %.0e: J = %d, ||S - S_J||_inf = %.2e' % (alpha, katz_tol, J, err))
    assert err <= alpha * katz_tol * (1 + 1e-9)
    assert alpha ** J <= katz_tol < alpha ** (J - 1)


@pytest.mark.parametrize('proximity', po.PROXIMITIES)
@pytest.mark.parametrize('graph', ['karate', 'sbm1024', 'randw200'])
def test_matrix_free_equals_dense(proximity, graph):
    import networkx as nx
    if graph == 'karate':
        G = load_karate_nx()
        A = nx.to_scipy_sparse_array(G, nodelist=list(G.nodes), weight='weight', dtype=np.float64, format='csr')
    elif graph == 'sbm1024':
        G, _ = load_sbm1024_nx()
        A = nx.to_scipy_sparse_array(G, nodelist=list(G.nodes), weight='weight', dtype=np.float64, format='csr')
    else:
        A = po.random_digraph()
    alpha = 0.6 if proximity == 'rooted_pagerank' else None
    S = po.proximity_dense(A, proximity, alpha=alpha)
    op = po.proximity_operator(A, proximity, alpha=alpha)
    X = np.random.default_rng(0).standard_normal((A.shape[0], 5))
    scale = np.abs(S).max() * np.abs(X).sum(axis=0).max()
    assert np.abs(op @ X - S @ X).max() <= 1e-13 * scale
    assert np.abs(op.T @ X - S.T @ X).max() <= 1e-13 * scale
    assert np.abs(op.matvec(X[:, 0]) - S @ X[:, 0]).max() <= 1e-13 * scale


@pytest.mark.parametrize('proximity', po.PROXIMITIES)
def test_embedding_layout_and_residuals(proximity):
    A = po.random_digraph()
    alpha = 0.5 if proximity == 'rooted_pagerank' else None
    X, s = po.embedding(A, proximity, 8, alpha=alpha)
    assert X.shape == (200, 8) and np.all(np.diff(s) >= 0)
    S = po.proximity_dense(A, proximity, alpha=alpha)
    sv = np.linalg.svd(S, compute_uv=False)
    assert np.allclose(s, sv[:4][::-1], rtol=1e-12)
    X1, X2 = X[:, :4], X[:, 4:]
    assert np.allclose(np.sum(X1 ** 2, axis=0), s) and np.allclose(np.sum(X2 ** 2, axis=0), s)
    r1, r2 = po.residuals(A, proximity, X, s, alpha=alpha)
    assert r1.max() < 1e-12 and r2.max() < 1e-12
    # the matrix-free route gives the same triplets
    Xm, sm = po.embedding(A, proximity, 8, alpha=alpha, dense_max=0)
    assert np.allclose(sm, s, rtol=1e-10)
    assert np.linalg.norm(Xm[:, :4] @ Xm[:, 4:].T - X1 @ X2.T) < 1e-9 * np.linalg.norm(X1 @ X2.T)
