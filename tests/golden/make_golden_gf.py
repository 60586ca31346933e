"""tests/golden/make_golden_gf.py -- fixtures of the UNMODIFIED reference class gem.embedding.gf.GraphFactorization (imported from
/root/reference; build container only).  The class draws X0 = 0.01 * np.random.randn(n, d) from the global NumPy RNG: the script seeds
it (np.random.seed(s)) right before the call and stores the same draw, the edge list in graph.edges order, and the result.
matplotlib (imported by gf.py:5 for a plot helper the path never calls) is absent from the image: a harness-side stub module stands in."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.dont_write_bytecode = True
import make_golden as mg

for name in ('matplotlib', 'matplotlib.pyplot'):
    sys.modules.setdefault(name, types.ModuleType(name))
sys.path.insert(0, mg.REF)
import networkx as nx
from gem.embedding.gf import GraphFactorization


def save(name, G, d, max_iter, eta, regu, seed):
    GraphFactorization.hyper_params = {'print_step': 10000, 'method_name': 'graph_factor_sgd'}
    m = GraphFactorization(d=d, max_iter=max_iter, eta=eta, regu=regu, data_set=name)
    n = len(G.nodes)
    X0 = 0.01 * np.random.RandomState(seed).randn(n, d)
    np.random.seed(seed)
    cwd = os.getcwd()
    os.chdir('/tmp')                      # the class creates gem/intermediate relative to the CWD before it looks for gem/c_exe/gf
    try:
        X = np.array(m.learn_embedding(graph=G, is_weighted=True, no_python=True))
    finally:
        os.chdir(cwd)
    nodes = list(G.nodes)
    assert nodes == list(range(n)) or True
    e = np.array([[u, v, w] for u, v, w in G.edges(data='weight', default=1)], dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, 'ref_gf_%s_d%d_it%d.npz' % (name, d, max_iter)), X=X, X0=X0, edges=e, n=n,
                        eta=eta, regu=regu, max_iter=max_iter)
    print(name, d, max_iter, X.shape, float(np.abs(X).max()))


if __name__ == '__main__':
    # `python make_golden_gf.py NAME ...` rewrites only the named fixtures (file names without .npz)
    only = set(sys.argv[1:])
    want = lambda name, d, it: not only or 'ref_gf_%s_d%d_it%d' % (name, d, it) in only
    K = mg.load_karate_nx().to_undirected().to_directed()      # tests/test_karate.py:35 works on G.to_directed()
    K = nx.convert_node_labels_to_integers(K, ordering='sorted') if sorted(K.nodes) != list(range(len(K.nodes))) else K
    if want('karate', 2, 300):
        save('karate', K, 2, 300, 1e-2, 1.0, 7)
    rng = np.random.default_rng(3)
    R = nx.DiGraph()
    R.add_nodes_from(range(60))
    for _ in range(400):
        u, v = int(rng.integers(0, 60)), int(rng.integers(0, 60))
        if u != v:
            R.add_edge(u, v, weight=float(np.round(rng.uniform(0.2, 2.0), 3)))
    for d in (8, 128):                    # d = 128: four values per lane in gf.cu
        if want('randw60', d, 60):
            save('randw60', R, d, 60, 2e-2, 0.05, 9)
