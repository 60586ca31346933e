"""tests/golden/make_golden_cc.py -- goldens of get_lcc (graph_util.py:29-34) and of link prediction with upstream GEM's
largest-component step, produced with networkx and the reference's get_lcc recipe.  The reference's own get_lcc calls
nx.weakly_connected_component_subgraphs, which networkx 2.4 removed, so its three statements are written out here with
the helper replaced by what it returned (the component's subgraph, copied) -- see ref_get_lcc.  The link-prediction
goldens use the UNMODIFIED reference functions (split_di_graph_to_train_test, get_edge_list_from_adj_mtrx,
computeMAP, computePrecisionCurve) through make_golden_linkpred.py.  Runs only in the build container; writes
tests/golden/cc_*.npz and linkpred_lcc_*.npz.

Cases (get_lcc)
  cc_karate_s2    the training graph of the Karate split with seed 2 (directed, train_ratio 0.8, the fixture loaded
                  as tests/test_karate.py does: node order of first appearance): components 33 and 1 (node 18)
  cc_rmat12       host R-MAT at scale 12 (gem_b200.synth.rmat, seed 42), nodes 0..4095, edges row-major
  cc_tie          two largest components of the same size (the one with the smaller first node wins), weighted
  cc_oneway       a weighted digraph whose edges all point from the larger id to the smaller, 400 nodes
Cases (link prediction with the LCC step, a fixed X of the LCC's k rows with entries in {-1.5, -1.25, ..., 1.5} so
that every score is exact in fp32, no node sample)
  linkpred_lcc_karate_s2   the Karate split above, split score (hope.py:43-44), d = 8
  linkpred_lcc_rmat10      host R-MAT at scale 10 (seed 3), undirected, seed 6, dot score (node2vec.py:56-57), d = 16

    python make_golden_cc.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.dont_write_bytecode = True
import make_golden_linkpred as mgl  # noqa: E402  (reference imports, networkx shims, score classes)

nx = mgl.nx
mge = mgl.mge
reu, rmetrics = mgl.reu, mgl.rmetrics


def ref_get_lcc(di_graph):
    """graph_util.py:29-34 with max(nx.weakly_connected_component_subgraphs(G), key=len) written out."""
    di_graph = max((di_graph.subgraph(c).copy() for c in nx.weakly_connected_components(di_graph)), key=len)
    tdl_nodes = list(di_graph.nodes())
    nodeListMap = dict(zip(tdl_nodes, range(len(tdl_nodes))))
    nx.relabel_nodes(di_graph, nodeListMap, copy=False)
    return di_graph, nodeListMap


def edges_array(G):
    return np.array([(u, v, w) for u, v, w in G.edges(data='weight', default=1)], dtype=np.float64).reshape(-1, 3)


def karate_train(seed=2):
    np.random.seed(seed)
    train, _ = reu.split_di_graph_to_train_test(mgl.mg.load_karate_nx(), 0.8, False)
    return train


def rmat_nx(scale, seed):
    from gem_b200 import synth
    csr = synth.rmat(scale, seed=seed)
    G = nx.DiGraph()
    G.add_nodes_from(range(csr.n))
    rows = np.repeat(np.arange(csr.n), np.diff(csr.indptr))
    G.add_weighted_edges_from(zip(rows.tolist(), csr.indices.tolist(), [1.0] * csr.nnz))
    return G


def tie_graph():
    """components {0, 3, 11}, {1, 2, 9, 10}, {4}, {5, 6, 7, 8}: the two of size 4 tie, {1, 2, 9, 10} comes first."""
    rng = np.random.default_rng(5)
    G = nx.DiGraph()
    G.add_nodes_from(range(12))
    for u, v in [(3, 0), (0, 11), (10, 1), (2, 9), (9, 10), (5, 6), (7, 6), (8, 7), (8, 5), (4, 4)]:
        G.add_edge(u, v, weight=float(np.round(rng.uniform(0.1, 2.0), 3)))
    return G


def oneway_graph():
    rng = np.random.default_rng(9)
    G = nx.DiGraph()
    G.add_nodes_from(range(400))
    for _ in range(330):
        u, v = (int(x) for x in rng.integers(0, 400, 2))
        if u != v:
            G.add_edge(max(u, v), min(u, v), weight=float(np.round(rng.uniform(0.1, 2.0), 3)))
    return G


def save_cc(name, G):
    nodes = list(G.nodes)
    pos = {u: i for i, u in enumerate(nodes)}
    comps = list(nx.weakly_connected_components(G))
    labels = np.empty(len(nodes), dtype=np.int32)
    for c, members in enumerate(comps):
        for u in members:
            labels[pos[u]] = c
    H, m = ref_get_lcc(G)
    out = dict(nodes=np.array(nodes, dtype=np.int64), edges=edges_array(G), labels=labels,
               map_keys=np.array(list(m.keys()), dtype=np.int64), map_values=np.array(list(m.values()), dtype=np.int64),
               lcc_nodes=np.array(sorted(H.nodes), dtype=np.int64),
               lcc_edges=np.array(sorted(edges_array(H).tolist()), dtype=np.float64).reshape(-1, 3))
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    print(name, 'n', len(nodes), 'components', len(comps), 'lcc', len(m), 'lcc edges', H.number_of_edges(), flush=True)


def save_linkpred(name, G, seed, is_undirected, score, d, xseed, train_ratio=0.8):
    """make_golden_linkpred.run with the LCC step after the split (upstream GEM's link prediction)."""
    np.random.seed(seed)
    train, test = reu.split_di_graph_to_train_test(G, train_ratio, is_undirected)
    n_comp = nx.number_weakly_connected_components(train)
    assert n_comp > 1
    train, m = ref_get_lcc(train)
    test = nx.relabel_nodes(test.subgraph(list(m)), m, copy=True)
    k = len(m)
    X = np.random.default_rng(xseed).integers(-6, 7, (k, d)) / 4.0   # dyadic: every score is exact in fp32 and fp64
    model = {'split': mge.SplitModel, 'dot': mge.DotModel}[score](d)
    adj = model.get_reconstructed_adj(X)
    pred = reu.get_edge_list_from_adj_mtrx(adj, is_undirected=is_undirected)
    filtered = [e for e in pred if not train.has_edge(e[0], e[1])]
    MAP = rmetrics.computeMAP(filtered, test)
    prec, _ = rmetrics.computePrecisionCurve(filtered, test)
    prec = np.asarray(prec, dtype=np.float64)
    out = dict(seed=np.int64(seed), train_ratio=np.float64(train_ratio), is_undirected=np.int32(is_undirected),
               n_sample=np.int64(0), n=np.int64(len(G)), k=np.int64(k), score=np.array(score),
               nodes=np.array(list(G.nodes), dtype=np.int64), edges=edges_array(G),
               map_keys=np.array(list(m.keys()), dtype=np.int64), map_values=np.array(list(m.values()), dtype=np.int64),
               train_edges=np.array(sorted(edges_array(train).tolist())).reshape(-1, 3),
               test_edges=edges_array(test), X=X, MAP=np.float64(MAP), n_pred=np.int64(len(filtered)),
               prec_head=prec[:4096], prec_stride=prec[::997])
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    print(name, 'components', n_comp, 'k', k, 'MAP', MAP, 'n_pred', len(filtered), flush=True)


def main():
    save_cc('cc_karate_s2', karate_train(2))
    save_cc('cc_rmat12', rmat_nx(12, 42))
    save_cc('cc_tie', tie_graph())
    save_cc('cc_oneway', oneway_graph())
    save_linkpred('linkpred_lcc_karate_s2', mgl.mg.load_karate_nx(), 2, False, 'split', 8, 21)
    save_linkpred('linkpred_lcc_rmat10', rmat_nx(10, 3), 6, True, 'dot', 16, 22)


if __name__ == '__main__':
    main()
