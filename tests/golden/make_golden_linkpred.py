"""tests/golden/make_golden_linkpred.py -- goldens of link prediction, produced by the UNMODIFIED reference functions
(gem.utils.evaluation_util.split_di_graph_to_train_test / get_edge_list_from_adj_mtrx, gem.utils.graph_util.sample_graph,
gem.evaluation.metrics.computeMAP / computePrecisionCurve) and the reference classes HOPE and LaplacianEigenmaps,
imported from the reference tree with the networkx shims of make_golden*.py.  Runs only in the build container;
writes tests/golden/linkpred_*.npz.

The task (np.random seeded once, then used in this order):
    train, test = split_di_graph_to_train_test(G, train_ratio, is_undirected)
    [n_sample: test, node_l = sample_graph(test, s); the train graph induced on the same node_l -- sample_graph
     again from the same random state]
    X = <reference class>.learn_embedding(graph=train)            (or a given random X)
    pred = get_edge_list_from_adj_mtrx(<reconstruction of X[node_l]>, is_undirected=is_undirected)
    filtered = [e for e in pred if not train.has_edge(e[0], e[1])]
    MAP = computeMAP(filtered, test); prec, _ = computePrecisionCurve(filtered, test)
The reconstruction uses the score classes of make_golden_eval*.py (the reference's get_edge_weight with d // 2).
Every graph is rebuilt with nodes 0..n-1 and its edges in row-major order, so a CSR drawn row by row makes the same
draws.

Cases
  linkpred_karate_hope        karate, directed (the fixture is upper-triangular), HOPE d = 4, beta = 0.01
  linkpred_sbm1024_hope       SBM-1024, undirected, HOPE d = 16, beta = 0.01
  linkpred_sbm1024_hope_s300  the same with n_sample_nodes = 300
  linkpred_randw200_dot       the weighted 200-node random digraph of make_golden_eval.py, directed, its random X
  linkpred_randw200_split     the same, split score
  linkpred_sbm1024_lap        SBM-1024, undirected, LaplacianEigenmaps d = 16 (Gaussian score)

    python make_golden_linkpred.py [case ...]      (default: every case)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.dont_write_bytecode = True
import make_golden_eval as mge  # noqa: E402  (reference imports, networkx shim, score classes)
import make_golden_eval_gauss as mgg  # noqa: E402

mg = mge.mg
nx = mge.nx
from gem.utils import evaluation_util as reu  # noqa: E402
from gem.utils import graph_util as rgu  # noqa: E402
from gem.evaluation import metrics as rmetrics  # noqa: E402


def canonical(G):
    """nodes 0..n-1, edges in row-major order, weights kept."""
    H = nx.DiGraph()
    H.add_nodes_from(range(len(G.nodes)))
    H.add_weighted_edges_from(sorted((int(u), int(v), float(w)) for u, v, w in G.edges(data='weight', default=1)))
    return H


def learn_hope(d, beta):
    return lambda train: mg.ref_hope(train, d, beta)


def learn_lap(d):
    import make_golden_lap as mgl
    return lambda train: mgl.run(train, d)


def edges_array(G):
    return np.array([(u, v, w) for u, v, w in G.edges(data='weight', default=1)], dtype=np.float64).reshape(-1, 3)


def run(name, G, seed, is_undirected, score, learn=None, X=None, train_ratio=0.8, n_sample=None):
    G = canonical(G)
    n = len(G.nodes)
    np.random.seed(seed)
    train, test = reu.split_di_graph_to_train_test(G, train_ratio, is_undirected)
    if n_sample:
        state = np.random.get_state()
        test_s, node_l = rgu.sample_graph(test, n_sample)
        np.random.set_state(state)
        train_s, node_l2 = rgu.sample_graph(train, n_sample)
        assert np.array_equal(node_l, node_l2)
    else:
        test_s, train_s, node_l = test, train, np.arange(n)
    if X is None:
        X = np.asarray(learn(train))
    cls = {'split': mge.SplitModel, 'dot': mge.DotModel, 'gaussian': mgg.GaussModel}[score]
    Xs = X[np.asarray(node_l)]
    model = cls(Xs.shape[1])
    adj = model.get_reconstructed_adj(Xs)
    pred = reu.get_edge_list_from_adj_mtrx(adj, is_undirected=is_undirected)
    filtered = [e for e in pred if not train_s.has_edge(e[0], e[1])]
    MAP = rmetrics.computeMAP(filtered, test_s)
    prec, _ = rmetrics.computePrecisionCurve(filtered, test_s)
    prec = np.asarray(prec, dtype=np.float64)
    out = dict(seed=np.int64(seed), train_ratio=np.float64(train_ratio), is_undirected=np.int32(is_undirected),
               n_sample=np.int64(n_sample or 0), n=np.int64(n), score=np.array(score), edges=edges_array(G),
               train_edges=edges_array(train), test_edges=edges_array(test), node_l=np.asarray(node_l, dtype=np.int64),
               X=X, MAP=np.float64(MAP), n_pred=np.int64(len(filtered)), n_pred_unfiltered=np.int64(len(pred)),
               prec_head=prec[:4096], prec_stride=prec[::997])
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    print(name, 'MAP', MAP, 'n_pred', len(filtered), 'of', len(pred), flush=True)


def randw200():
    rng = np.random.default_rng(7)                    # the graph and X of make_golden_eval.py's eval_randw200_*
    n = 200
    R = nx.DiGraph()
    R.add_nodes_from(range(n))
    for _ in range(1500):
        u, v = rng.integers(0, n, 2)
        R.add_edge(int(u), int(v), weight=float(np.round(rng.uniform(0.1, 2.0), 3)))
    X = rng.standard_normal((n, 16)) * 0.4
    X[:, 3] = np.round(X[:, 3], 1)
    return R, np.round(X, 1)


CASES = ('linkpred_karate_hope', 'linkpred_sbm1024_hope', 'linkpred_sbm1024_hope_s300', 'linkpred_randw200_dot',
         'linkpred_randw200_split', 'linkpred_sbm1024_lap')


def main(cases):
    if 'linkpred_karate_hope' in cases:
        run('linkpred_karate_hope', mg.load_karate_nx(), 11, False, 'split', learn=learn_hope(4, 0.01))
    if 'linkpred_sbm1024_hope' in cases:
        run('linkpred_sbm1024_hope', mg.load_sbm_nx(), 12, True, 'split', learn=learn_hope(16, 0.01))
    if 'linkpred_sbm1024_hope_s300' in cases:
        run('linkpred_sbm1024_hope_s300', mg.load_sbm_nx(), 13, True, 'split', learn=learn_hope(16, 0.01), n_sample=300)
    if 'linkpred_randw200_dot' in cases or 'linkpred_randw200_split' in cases:
        R, X = randw200()
        if 'linkpred_randw200_dot' in cases:
            run('linkpred_randw200_dot', R, 14, False, 'dot', X=X)
        if 'linkpred_randw200_split' in cases:
            run('linkpred_randw200_split', R, 15, False, 'split', X=X)
    if 'linkpred_sbm1024_lap' in cases:
        run('linkpred_sbm1024_lap', mg.load_sbm_nx(), 16, True, 'gaussian', learn=learn_lap(16))


if __name__ == '__main__':
    main(sys.argv[1:] or CASES)
