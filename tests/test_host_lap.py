"""Host logic of gem_b200.embedding.lap (CPU): the undirected, degree-normalised matrix the GPU solver receives equals
I - L_sym of the pinned oracle (oracle/lap_oracle.py <- nx.normalized_laplacian_matrix(graph.to_undirected()), lap.py:25-26),
including networkx's rule for a pair whose two directions carry different weights, self loops and isolated vertices."""
import os
import sys

import numpy as np
import pytest

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, 'oracle'))


def test_undirected_normalised_matches_oracle():
    import networkx as nx
    import lap_oracle as lo
    from gem_b200 import graph as hg
    from gem_b200.embedding.lap import undirected_normalised
    rng = np.random.default_rng(5)
    G = nx.DiGraph()
    G.add_nodes_from(range(60))                       # nodes 57..59 stay isolated
    for _ in range(400):
        u, v = int(rng.integers(0, 57)), int(rng.integers(0, 57))
        G.add_edge(u, v, weight=float(np.round(rng.uniform(0.3, 2.5), 3)))      # includes a few self loops
    csr = hg.from_networkx(G)
    ahat, l_fro2 = undirected_normalised(csr)
    A = nx.to_scipy_sparse_array(G, nodelist=list(G.nodes), weight='weight', format='csr')
    W = lo.undirected_weights(A)
    assert np.array_equal(W.toarray(), nx.to_numpy_array(G.to_undirected(), nodelist=list(G.nodes), weight='weight'))
    L = lo.normalized_laplacian(W).toarray()
    assert np.allclose(ahat.to_scipy().toarray(), np.eye(60) - L, atol=1e-14)
    assert abs(l_fro2 - np.sum(L * L)) < 1e-10
    assert ahat.is_symmetric()


def test_errors_and_names():
    from gem_b200.embedding.lap import LaplacianEigenmaps
    LaplacianEigenmaps.hyper_params.clear(); LaplacianEigenmaps.hyper_params.update({'method_name': 'lap_eigmap_svd'})
    m = LaplacianEigenmaps(d=2)
    assert m.get_method_name() == 'lap_eigmap_svd' and m.get_method_summary() == 'lap_eigmap_svd_2'
    with pytest.raises(ValueError, match='graph needed'):
        m.learn_embedding(graph=None)
    with pytest.raises(ValueError, match='Embedding not learned yet'):
        m.get_embedding()


def test_lle_operator_matches_oracle():
    """gem_b200.embedding.lle.lle_operator: C = c I - (I - P)^T (I - P) against the pinned oracle's I - P (lle.py:25-28)."""
    import networkx as nx
    import lle_oracle as le
    from gem_b200 import graph as hg
    from gem_b200.embedding.lle import lle_operator, LocallyLinearEmbedding
    rng = np.random.default_rng(8)
    G = nx.DiGraph()
    G.add_nodes_from(range(50))                       # 48, 49 isolated
    for _ in range(300):
        u, v = int(rng.integers(0, 48)), int(rng.integers(0, 48))
        if u != v:
            G.add_edge(u, v, weight=float(np.round(rng.uniform(0.3, 2.5), 3)))
    C, c = lle_operator(hg.from_networkx(G))
    A = nx.to_scipy_sparse_array(G, nodelist=list(G.nodes), weight='weight', format='csr')
    M = le.lle_matrix(A).toarray()
    assert c >= np.linalg.norm(M, 2) ** 2 - 1e-12
    assert np.allclose(C.to_scipy().toarray(), c * np.eye(50) - M.T @ M, atol=1e-13)
    assert C.is_symmetric()
    LocallyLinearEmbedding.hyper_params.clear(); LocallyLinearEmbedding.hyper_params.update({'method_name': 'lle_svd'})
    m = LocallyLinearEmbedding(d=2)
    assert m.get_method_summary() == 'lle_svd_2'
    with pytest.raises(ValueError, match='graph needed'):
        m.learn_embedding(graph=None)


def test_gf_host_logic():
    import networkx as nx
    from gem_b200.embedding.gf import GraphFactorization
    GraphFactorization.hyper_params.clear()
    GraphFactorization.hyper_params.update({'print_step': 10000, 'method_name': 'graph_factor_sgd'})
    m = GraphFactorization(d=2, max_iter=10, eta=1e-3, regu=1.0, data_set='x')
    assert m.get_method_summary() == 'graph_factor_sgd_2'
    with pytest.raises(ValueError, match='graph needed'):
        m.learn_embedding(graph=None)
    G = nx.DiGraph()
    G.add_edge(2, 0, weight=0.5); G.add_edge(0, 1); G.add_node(3)
    n, src, dst, w = m._edges(G)
    assert n == 4 and src.tolist() == [2, 0] and dst.tolist() == [0, 1] and w.tolist() == [0.5, 1.0]      # graph.edges order
    H = nx.DiGraph(); H.add_edge(5, 1)
    with pytest.raises(ValueError, match='labels must be 0..n-1'):
        m._edges(H)


def test_gf_schedule_choice(monkeypatch):
    """Which gemb_gf mode the plugin asks for: rows in parallel when graph.edges() is grouped by ascending source, the reference's
    order on one warp otherwise, regrouping (with a warning) beyond sequential_limit."""
    import networkx as nx
    from gem_b200 import _native
    from gem_b200.embedding.gf import GraphFactorization
    calls = []

    class FakeCtx:
        def __init__(self, device=0): pass
        def close(self): pass
        def __enter__(self): return self
        def __exit__(self, *exc): self.close()

    def fake_gf(ctx, n, src, dst, w, d, eta, regu, max_iter, X0, mode=0):
        calls.append((mode, src.tolist()))
        return np.zeros((n, d), np.float32), 0.0

    monkeypatch.setattr(_native, 'Context', FakeCtx)
    monkeypatch.setattr(_native, 'graph_factorization', fake_gf)
    GraphFactorization.hyper_params.clear()
    GraphFactorization.hyper_params.update({'print_step': 10000, 'method_name': 'graph_factor_sgd'})
    G = nx.DiGraph(); G.add_nodes_from(range(4)); G.add_edges_from([(0, 1), (1, 2), (2, 3), (3, 0)])
    GraphFactorization(d=2, max_iter=5, eta=1e-3, regu=1.0).learn_embedding(graph=G)
    assert calls[-1][0] == 1
    H = nx.DiGraph(); H.add_edges_from([(2, 3), (0, 1), (1, 2)])            # node order 2, 3, 0, 1: sources 2, 0, 1
    GraphFactorization(d=2, max_iter=5, eta=1e-3, regu=1.0).learn_embedding(graph=H)
    assert calls[-1] == (0, [2, 0, 1])
    with pytest.warns(RuntimeWarning, match='grouped by source'):
        GraphFactorization(d=2, max_iter=5, eta=1e-3, regu=1.0, sequential_limit=10).learn_embedding(graph=H)
    assert calls[-1] == (1, [0, 1, 2])
