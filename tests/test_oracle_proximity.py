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


# ----------------------------------------------------------------- operator_apply / operator_abs (gemb_hope_apply's oracle)
def _dense_operator(A, mode, transpose, coef, terms, absolute=False):
    """The dense matrix operator_apply (absolute: operator_abs) multiplies by, built independently of it."""
    Ad = A.toarray()
    n = Ad.shape[0]
    if absolute:
        Ad, coef = np.abs(Ad), (None if coef is None else abs(coef))
    if mode == 0:
        S, T = np.zeros((n, n)), np.eye(n)
        for _ in range(terms):
            T = coef * Ad @ T
            S += T
    elif mode == 1:
        S = Ad
    elif mode == 2:
        M = np.eye(n) + Ad if absolute else np.eye(n) - Ad
        S = M.T @ M if absolute else -(M.T @ M)
    elif mode in (3, 4):
        if absolute:
            D = np.abs(po.inv_degree(A)) if mode == 4 else np.ones(n)
            S = Ad @ np.diag(D) @ Ad
        else:
            S = po.proximity_dense(A, 'common_neighbors' if mode == 3 else 'adamic_adar')
    else:
        S, T = np.eye(n), np.eye(n)
        for _ in range(terms):
            T = coef * Ad @ T
            S += T
        S = (1.0 - coef) * S
    return S.T if transpose and mode not in (1, 2) else S


def _signed_digraph():
    A = po.random_digraph(n=60, seed=5, p=0.12)
    A.data = A.data * np.random.default_rng(1).choice([-1.0, 1.0], A.nnz)
    return A


@pytest.mark.parametrize('transpose', [False, True])
@pytest.mark.parametrize('mode,coef,terms', [(0, 0.07, 1), (0, 0.07, 6), (1, None, None), (2, None, None),
                                             (3, None, None), (4, None, None), (5, 0.6, 1), (5, 0.6, 9)])
def test_operator_apply_equals_dense(mode, coef, terms, transpose):
    """operator_apply and operator_abs against dense matrices on a directed graph with an isolated node and a row
    without out-edges (signed for operator_abs, so that |.| matters), and the mode-5 series against proximity_dense's on
    P = transition(A)."""
    A = po.random_digraph(n=60, seed=5, p=0.12)
    if mode == 1:
        A = (A + A.T).tocsr()
    if mode == 2:
        A = po.transition(A)
    X = np.random.default_rng(2).standard_normal((A.shape[0], 7))
    for absolute, B in ((False, A), (True, _signed_digraph() if mode != 1 else (_signed_digraph() + _signed_digraph().T))):
        fn = po.operator_abs if absolute else po.operator_apply
        Y = fn(B, mode, X, transpose=transpose, coef=coef, terms=terms)
        S = _dense_operator(B, mode, transpose, coef, terms, absolute)
        ref = S @ (np.abs(X) if absolute else X)
        assert np.abs(Y - ref).max() <= 1e-13 * max(1.0, np.abs(ref).max())
    if mode == 5:
        S = po.proximity_dense(po.random_digraph(n=60, seed=5, p=0.12), 'rooted_pagerank', alpha=coef, terms=terms)
        Y = po.operator_apply(po.transition(po.random_digraph(n=60, seed=5, p=0.12)), 5, X, transpose, coef, terms)
        assert np.abs(Y - (S.T if transpose else S) @ X).max() <= 1e-13


@pytest.mark.parametrize('transpose', [False, True])
@pytest.mark.parametrize('mode,coef,terms', [(0, 0.05, 4), (1, None, None), (2, None, None), (3, None, None),
                                             (4, None, None), (5, 0.5, 7)])
def test_operator_abs_bounds_operator(mode, coef, terms, transpose):
    """A >= 0 and X >= 0: operator_abs is operator_apply (mode 2, whose S is signed: it bounds it).  Signed: it bounds
    |operator_apply| entry by entry."""
    A = po.random_digraph(n=80, seed=4, p=0.08)
    if mode == 1:
        A = (A + A.T).tocsr()
    if mode in (2, 5):
        A = po.transition(A)
    rng = np.random.default_rng(3)
    Xp = rng.random((A.shape[0], 5))
    Y, B = (f(A, mode, Xp, transpose, coef, terms) for f in (po.operator_apply, po.operator_abs))
    if mode == 2:
        assert np.all(np.abs(Y) <= B * (1 + 1e-14)) and not np.allclose(np.abs(Y), B)
    else:
        assert np.abs(Y - B).max() <= 1e-14 * np.abs(B).max()
    Xs = rng.standard_normal((A.shape[0], 5))
    Y, B = (f(A, mode, Xs, transpose, coef, terms) for f in (po.operator_apply, po.operator_abs))
    assert np.all(np.abs(Y) <= B * (1 + 1e-14))


def test_operator_apply_empty_graph():
    """No edges: S = 0 (modes 0, 1, 3, 4), -I (mode 2), (1 - alpha) I (mode 5)."""
    A = sp.csr_matrix((50, 50))
    X = np.random.default_rng(4).standard_normal((50, 4))
    for mode in (0, 1, 3, 4):
        assert not np.any(po.operator_apply(A, mode, X, coef=0.1, terms=3))
    assert np.array_equal(po.operator_apply(A, 2, X), -X)
    assert np.array_equal(po.operator_apply(A, 5, X, coef=0.25, terms=5), 0.75 * X)
    assert not np.any(po.inv_degree(A))
