"""oracle/cc_oracle.py and the networkx path of get_lcc pinned against networkx and the reference's get_lcc recipe
(goldens made by tests/golden/make_golden_cc.py): labels, node list, map, edges and weights exact; link prediction with
the largest-component step exact given the golden X (MAP to 1e-13, the precision curve bit for bit); and
split_and_sample(lcc=True) reproduces the golden's training and test graphs."""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, golden_path

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import cc_oracle as co  # noqa: E402

CC_CASES = ['cc_karate_s2', 'cc_rmat12', 'cc_tie', 'cc_oneway']
LP_CASES = ['linkpred_lcc_karate_s2', 'linkpred_lcc_rmat10']


def nx_graph(z):
    import networkx as nx
    G = nx.DiGraph()
    G.add_nodes_from(z['nodes'].tolist())
    G.add_weighted_edges_from((int(a), int(b), float(w)) for a, b, w in z['edges'])
    return G


def positions(z):
    """The golden graph as a CSR over rows = node order: (n, indptr, indices, weights, position of every label)."""
    nodes = z['nodes']
    pos = np.full(int(nodes.max()) + 1, -1, dtype=np.int64)
    pos[nodes] = np.arange(nodes.size)
    e = z['edges']
    src, dst = pos[e[:, 0].astype(np.int64)], pos[e[:, 1].astype(np.int64)]
    order = np.lexsort((dst, src))
    indptr = np.zeros(nodes.size + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=nodes.size), out=indptr[1:])
    return nodes.size, indptr, dst[order].astype(np.int32), e[order, 2], pos


def sorted_edges(indptr, indices, w):
    rows = np.repeat(np.arange(indptr.size - 1), np.diff(indptr))
    e = np.stack([rows, indices, np.ones(indices.size) if w is None else w], 1).astype(np.float64)
    return e[np.lexsort((e[:, 2], e[:, 1], e[:, 0]))]


@pytest.mark.parametrize('name', CC_CASES)
def test_oracle_matches_networkx(name):
    z = np.load(golden_path(name + '.npz'))
    n, indptr, indices, w, pos = positions(z)
    lab = co.labels(n, indptr, indices)
    assert np.array_equal(lab, z['labels'])
    node_l, ip, ix, ww = co.lcc_csr(n, indptr, indices, w, lab)
    keys = z['map_keys']
    assert np.array_equal(node_l, np.sort(pos[keys]))
    assert np.array_equal(z['map_values'], np.arange(node_l.size))
    if 2 * keys.size >= n:                                # networkx keeps G's node order: the map is the row order
        assert np.array_equal(node_l, pos[keys])
        assert np.array_equal(sorted_edges(ip, ix, ww), z['lcc_edges'])
    # in the graph's own node labels, whatever order the map has
    new_of_row = np.full(n, -1)
    new_of_row[pos[keys]] = z['map_values']
    ours = sorted_edges(ip, ix, ww)
    ours[:, :2] = new_of_row[node_l[ours[:, :2].astype(np.int64)]]
    assert np.array_equal(ours[np.lexsort((ours[:, 2], ours[:, 1], ours[:, 0]))], z['lcc_edges'])
    assert np.all(np.diff(node_l) > 0)
    for r in range(node_l.size):                          # columns stay sorted within each row
        assert np.all(np.diff(ix[ip[r]:ip[r + 1]]) >= 0)


@pytest.mark.parametrize('name', CC_CASES)
def test_get_lcc_networkx_path_matches_reference_recipe(name):
    from gem_b200.utils.graph_util import get_lcc
    z = np.load(golden_path(name + '.npz'))
    H, m = get_lcc(nx_graph(z))
    assert list(m.keys()) == z['map_keys'].tolist() and list(m.values()) == z['map_values'].tolist()
    assert list(H.nodes) == list(range(len(m)))           # copy=True: the nodes iterate as 0..k-1
    e = np.array([(u, v, w) for u, v, w in H.edges(data='weight')], dtype=np.float64).reshape(-1, 3)
    assert np.array_equal(e[np.lexsort((e[:, 2], e[:, 1], e[:, 0]))], z['lcc_edges'])


def test_get_lcc_rejects_undirected_networkx():
    import networkx as nx
    from gem_b200.utils.graph_util import get_lcc
    with pytest.raises(nx.NetworkXNotImplemented):
        get_lcc(nx.path_graph(4))


def test_tie_goes_to_the_component_met_first():
    z = np.load(golden_path('cc_tie.npz'))
    sizes = np.bincount(z['labels'])
    assert np.sum(sizes == sizes.max()) == 2 and sorted(z['map_keys'].tolist()) == [1, 2, 9, 10]


@pytest.mark.parametrize('name', LP_CASES)
def test_oracle_link_prediction_with_lcc_matches_reference(name):
    z = np.load(golden_path(name + '.npz'))
    e = z['edges']
    r = co.linkpred_lcc(e[:, 0], e[:, 1], z['nodes'], z['X'], str(z['score']), int(z['seed']), float(z['train_ratio']),
                        bool(z['is_undirected']))
    assert list(r['node_map'].keys()) == z['map_keys'].tolist()
    assert list(r['node_map'].values()) == z['map_values'].tolist()
    assert r['n_pred'] == int(z['n_pred'])
    assert abs(r['MAP'] - float(z['MAP'])) < 1e-13
    assert np.array_equal(r['prec_curve'][:4096], z['prec_head'])
    assert np.array_equal(r['prec_curve'][::997], z['prec_stride'])


@pytest.mark.parametrize('name', LP_CASES)
def test_split_and_sample_lcc_matches_golden(name):
    from gem_b200.evaluation.evaluate_link_prediction import split_and_sample
    z = np.load(golden_path(name + '.npz'))
    G = nx_graph(z)
    tr, te, tr_s, node_l = split_and_sample(G, float(z['train_ratio']), None, bool(z['is_undirected']),
                                            np.random.RandomState(int(z['seed'])), lcc=True)
    k = int(z['k'])
    assert list(tr.nodes) == list(range(k)) and list(te.nodes) == list(range(k)) and tr_s is tr
    assert np.array_equal(node_l, np.arange(k))
    e = np.array(list(tr.edges(data='weight')), dtype=np.float64).reshape(-1, 3)
    assert np.array_equal(e[np.lexsort((e[:, 2], e[:, 1], e[:, 0]))], z['train_edges'])
    assert np.array_equal(np.array(list(te.edges(data='weight')), dtype=np.float64).reshape(-1, 3), z['test_edges'])


def test_split_and_sample_lcc_is_a_no_op_on_one_component():
    """The SBM-1024 split of linkpred_sbm1024_hope keeps one component: lcc=True returns the very same graphs."""
    from gem_b200.evaluation.evaluate_link_prediction import split_and_sample
    z = np.load(golden_path('linkpred_sbm1024_hope.npz'))
    G = nx_graph(dict(nodes=np.arange(int(z['n'])), edges=z['edges']))
    a = split_and_sample(G, float(z['train_ratio']), None, True, np.random.RandomState(int(z['seed'])))
    b = split_and_sample(G, float(z['train_ratio']), None, True, np.random.RandomState(int(z['seed'])), lcc=True)
    for x, y in zip(a[:3], b[:3]):
        assert list(x.nodes) == list(y.nodes) and list(x.edges(data='weight')) == list(y.edges(data='weight'))
    assert np.array_equal(a[3], b[3])
