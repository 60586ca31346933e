"""Host steps of link prediction without a GPU: split_di_graph_to_train_test and sample_graph give the reference's
split and sample (the linkpred_*.npz goldens, made by the reference's functions) for networkx and HostCSR inputs;
the reference's quirks are kept; the evaluation itself has no CPU fallback."""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, golden_path

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import linkpred_oracle as lo  # noqa: E402

CASES = ['linkpred_karate_hope', 'linkpred_sbm1024_hope', 'linkpred_sbm1024_hope_s300', 'linkpred_randw200_dot',
         'linkpred_sbm1024_lap']


def _nx(n, e):
    import networkx as nx
    G = nx.DiGraph()
    G.add_nodes_from(range(n))
    G.add_weighted_edges_from((int(a), int(b), float(w)) for a, b, w in e)
    return G


def _csr(n, e):
    from gem_b200 import graph as hg
    return hg.from_edges(n, e[:, 0].astype(np.int64), e[:, 1].astype(np.int64), e[:, 2])


def _csr_edges(c):
    rows = np.repeat(np.arange(c.n), np.diff(c.indptr))
    w = np.ones(c.nnz) if c.data is None else c.data
    return np.column_stack((rows, c.indices, w)).astype(np.float64)


@pytest.mark.parametrize('name', CASES)
def test_split_and_sample_equal_the_reference(name):
    from gem_b200.utils import evaluation_util, graph_util
    z = np.load(golden_path(name + '.npz'))
    n, e, und, s = int(z['n']), z['edges'], bool(z['is_undirected']), int(z['n_sample'])
    seed, ratio = int(z['seed']), float(z['train_ratio'])
    # networkx, global np.random as in the reference
    G = _nx(n, e)
    np.random.seed(seed)
    tr, te = evaluation_util.split_di_graph_to_train_test(G, ratio, und)
    assert np.array_equal(np.array([(a, b, w) for a, b, w in tr.edges(data='weight')]).reshape(-1, 3), z['train_edges'])
    assert np.array_equal(np.array([(a, b, w) for a, b, w in te.edges(data='weight')]).reshape(-1, 3), z['test_edges'])
    assert list(tr.nodes) == list(G.nodes) and list(te.nodes) == list(G.nodes)
    tes, node_l = graph_util.sample_graph(te, s or None)
    assert np.array_equal(node_l, z['node_l'])
    # HostCSR with a RandomState: the golden graphs are in row-major order, so the draws are the same
    rng = np.random.RandomState(seed)
    ctr, cte = evaluation_util.split_di_graph_to_train_test(_csr(n, e), ratio, und, rng=rng)
    assert np.array_equal(_csr_edges(ctr), z['train_edges']) and np.array_equal(_csr_edges(cte), z['test_edges'])
    ctes, cnode_l = graph_util.sample_graph(cte, s or None, rng=rng)
    assert np.array_equal(cnode_l, z['node_l'])
    if s:
        ref, _ = lo.sample_loops([tuple(x) for x in z['test_edges'].tolist()], n, s, None, node_l=node_l)
        got = [(a, b, w) for a, b, w in tes.edges(data='weight')]
        assert sorted(got) == sorted((int(a), int(b), w) for a, b, w in ref)
        assert np.array_equal(_csr_edges(ctes), np.array(sorted(ref), dtype=np.float64).reshape(-1, 3))
        trs = graph_util.induced_graph(ctr, cnode_l)
        ref, _ = lo.sample_loops([tuple(x) for x in z['train_edges'].tolist()], n, s, None, node_l=node_l)
        assert np.array_equal(_csr_edges(trs), np.array(sorted(ref), dtype=np.float64).reshape(-1, 3))


def test_one_vector_draw_is_the_scalar_draws():
    a = np.random.RandomState(5).uniform(size=4097)
    r = np.random.RandomState(5)
    assert np.array_equal(a, np.array([r.uniform() for _ in range(4097)]))


def test_reference_quirks():
    import networkx as nx
    from gem_b200.utils import evaluation_util
    G = nx.DiGraph([(0, 1), (1, 0), (1, 2), (2, 2)])                # (1, 2) has no reverse
    with pytest.raises(nx.NetworkXError):
        evaluation_util.split_di_graph_to_train_test(G, 0.5, True, rng=np.random.RandomState(0))
    with pytest.raises(nx.NetworkXError):
        evaluation_util.split_di_graph_to_train_test(_csr(3, np.array([(0, 1, 1.0), (1, 0, 1.0), (1, 2, 1.0)])), 0.5,
                                                     True, rng=np.random.RandomState(0))
    G = nx.DiGraph([(0, 1), (1, 0), (2, 2), (3, 1)])                # self-loop; (3, 1) never draws
    G.add_node(4)
    for ratio in (0.0, 1.0):
        tr, te = evaluation_util.split_di_graph_to_train_test(G, ratio, True, rng=np.random.RandomState(0))
        assert tr.has_edge(2, 2) and te.has_edge(2, 2) and tr.has_edge(3, 1) and te.has_edge(3, 1)
        assert len(tr.nodes) == len(te.nodes) == 5
        assert tr.has_edge(0, 1) == tr.has_edge(1, 0) == (ratio == 1.0) != te.has_edge(0, 1)
    # directed: every edge draws, self-loops included
    tr, te = evaluation_util.split_di_graph_to_train_test(G, 0.0, False, rng=np.random.RandomState(0))
    assert tr.number_of_edges() == 0 and te.number_of_edges() == 4


def test_no_cpu_fallback(native_lib):
    if native_lib.gemb_device_count() > 0:
        pytest.skip('a GPU is present')
    from gem_b200.embedding.hope import HOPE
    from gem_b200.evaluation.evaluate_link_prediction import evaluateStaticLinkPrediction
    z = np.load(golden_path('linkpred_karate_hope.npz'))
    G = _nx(int(z['n']), z['edges'])
    with pytest.raises(RuntimeError):
        evaluateStaticLinkPrediction(G, HOPE(d=4, beta=0.01), is_undirected=False, seed=1)
