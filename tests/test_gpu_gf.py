"""Graph Factorization parity on the GPU (gem_b200.embedding.gf.GraphFactorization -> gemb_gf) against outputs of the unmodified
reference class with the same start X0 (tests/golden/ref_gf_*.npz; the oracle reproduces those bit-for-bit, tests/test_oracle_gf.py)
and against the reference's golden tests/karate_res/GraphFactorization.txt at the reference's own bar (tests/test_karate.py:37-40,85:
|mean(target - X)| < 0.3 -- the start is random there).  fp32 SGD vs the reference's fp64: 2e-4 relative after 60-300 epochs."""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, golden_path, load_karate_nx

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(REPO, 'oracle'))


def _fresh(**kw):
    from gem_b200.embedding.gf import GraphFactorization
    GraphFactorization.hyper_params.clear()
    GraphFactorization.hyper_params.update({'print_step': 10000, 'method_name': 'graph_factor_sgd'})
    return GraphFactorization(**kw)


def _nx_from(z):
    """A DiGraph whose graph.edges() yields the stored edge list in the stored order (it came from graph.edges() of the graph the
    reference ran on: grouped by source, sources in node-insertion order)."""
    import networkx as nx
    G = nx.DiGraph()
    e = z['edges']
    seen = list(dict.fromkeys(int(u) for u in e[:, 0]))
    G.add_nodes_from(seen)
    G.add_nodes_from(i for i in range(int(z['n'])) if i not in set(seen))
    for u, v, w in e:
        G.add_edge(int(u), int(v), weight=float(w))
    assert [(u, v) for u, v in G.edges()] == [(int(u), int(v)) for u, v, _ in e]
    return G


@pytest.mark.parametrize('name', ['ref_gf_karate_d2_it300', 'ref_gf_randw60_d8_it60', 'ref_gf_randw60_d128_it60'])
def test_reference_class_outputs(native_lib, name):
    z = np.load(golden_path(name + '.npz'))
    G = _nx_from(z)
    m = _fresh(d=z['X0'].shape[1], max_iter=int(z['max_iter']), eta=float(z['eta']), regu=float(z['regu']))
    X = m.learn_embedding(graph=G, is_weighted=True, no_python=True, X0=z['X0'])
    # karate: the reference's node order is not sorted -> the sweep runs in the reference's order on one warp (mode 0);
    # randw60: nodes inserted in order -> graph.edges() is grouped by ascending source -> rows in parallel (mode 1), same result
    assert m.stats['mode'] == (0 if 'karate' in name else 1)
    ref = z['X']
    assert np.abs(X - ref).max() < 2e-4 * max(np.abs(ref).max(), 1e-3), np.abs(X - ref).max()
    assert abs(m.get_edge_weight(0, 1) - float(ref[0] @ ref[1])) < 1e-5


def test_sequential_mode_equals_rows_mode_and_handles_any_order(native_lib):
    import gf_oracle as go
    from gem_b200 import _native
    z = np.load(golden_path('ref_gf_randw60_d8_it60.npz'))
    e = z['edges']
    n, d = int(z['n']), 8
    ctx = _native.Context(0)
    try:
        kw = dict(d=d, eta=float(z['eta']), regu=float(z['regu']), max_iter=int(z['max_iter']), X0=z['X0'])
        src, dst, w = e[:, 0].astype(np.int32), e[:, 1].astype(np.int32), e[:, 2].astype(np.float32)
        X0s, _ = _native.graph_factorization(ctx, n, src, dst, w, mode=0, **kw)
        X1s, _ = _native.graph_factorization(ctx, n, src, dst, w, mode=1, **kw)
        assert np.array_equal(X0s, X1s)                          # same arithmetic in the same order: bit-identical
        # reversed edge list: not grouped by source -> the plugin's mode 0; against the oracle on the same order
        rs, rd, rw = src[::-1].copy(), dst[::-1].copy(), w[::-1].copy()
        Xr, _ = _native.graph_factorization(ctx, n, rs, rd, rw, mode=0, **kw)
        Xo = go.gf_sequential(n, rs, rd, rw, d, float(z['eta']), float(z['regu']), int(z['max_iter']), z['X0'])
        assert np.abs(Xr - Xo).max() < 2e-4 * np.abs(Xo).max()
        with pytest.raises(RuntimeError, match='grouped by source'):
            _native.graph_factorization(ctx, n, rs, rd, rw, mode=1, **kw)
    finally:
        ctx.close()


def test_karate_reference_config(native_lib):
    """tests/test_karate.py:37-40: GraphFactorization(d=2, max_iter=50000, eta=1e-4, regu=1.0) on the Karate graph (to_directed)."""
    G = load_karate_nx().to_undirected().to_directed()
    m = _fresh(d=2, max_iter=50000, eta=1e-4, regu=1.0, data_set='karate')
    np.random.seed(0)
    X = m.learn_embedding(graph=G, is_weighted=True, no_python=True)
    gold = np.loadtxt(golden_path('karate_GraphFactorization.txt'))
    assert X.shape == gold.shape and np.isfinite(X).all()
    assert abs(np.mean(gold - X)) < 0.3
