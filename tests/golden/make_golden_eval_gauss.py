"""tests/golden/make_golden_eval_gauss.py -- goldens of the reconstruction evaluation for the Gaussian score of
LaplacianEigenmaps and LocallyLinearEmbedding (get_edge_weight = exp(-|x_i - x_j|^2), lap.py:39-42, lle.py:37-40),
produced like make_golden_eval.py by the UNMODIFIED reference evaluateStaticGraphReconstruction.  Runs only in the
build container; writes tests/golden/eval_*_lap.npz, eval_*_lle.npz and eval_randw200_gauss.npz.

Cases
  eval_karate_lap, eval_karate_lle   karate, X = tests/karate_res/{LaplacianEigenmaps,LocallyLinearEmbedding}.txt,
                                     variants und / dir / dirw (structurally equivalent nodes: delta ~ 1e-33)
  eval_sbm1024_lap                   tests/data/sbm.gpickle, X = tests/smb_res/LaplacianEigenmaps.txt rounded to fp32,
                                     und.  The graph and X are the committed fixtures sbm1024.npz and
                                     sbm1024_LaplacianEigenmaps.npy (the same graph; that X cast to fp32), so this golden
                                     stores only the reference's results and the names of those two files
  eval_randw200_gauss                200-node weighted digraph (both directions of many edges), d = 6, with
                                     duplicated rows (exact delta = 0 ties) and a few far rows (delta > 745.14:
                                     score 0, dropped by the full scan, kept by the sampled branch)

    python make_golden_eval_gauss.py [case ...]      (default: every case)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_eval as mge  # noqa: E402  (reference imports, networkx shim, loaders)

mg = mge.mg
nx = mge.nx
gr = mge.gr


class GaussModel(mge.SplitModel):               # get_edge_weight of lap.py:39-42 (= lle.py:37-40)
    def get_edge_weight(self, i, j):
        return np.exp(
            -np.power(np.linalg.norm(self._X[i, :] - self._X[j, :]), 2)
        )


def run(name, G, X, variants, fixtures=None):
    """fixtures = (graph .npz, X .npy) already committed under tests/golden: stored by name instead of by value."""
    model = GaussModel(X.shape[1])
    out = {'score': np.array('gaussian'), 'n': np.int64(len(G.nodes))}
    if fixtures:
        out['graph_fixture'], out['X_fixture'] = np.array(fixtures[0]), np.array(fixtures[1])
    else:
        out['X'] = X
        out['edges'] = np.array([(u, v, w) for u, v, w in G.edges(data='weight', default=1)], dtype=np.float64)
        out['nodes'] = np.array(list(G.nodes), dtype=np.int64)
    for tag, kw in variants.items():
        MAP, prec, err, err_b = gr.evaluateStaticGraphReconstruction(G, model, X, None, **kw)
        prec = np.asarray(prec, dtype=np.float64)
        out[tag + '_MAP'] = np.float64(MAP)
        out[tag + '_n_pred'] = np.int64(len(prec))
        out[tag + '_prec_head'] = prec[:4096]
        out[tag + '_prec_stride'] = prec[::997]
        out[tag + '_err'] = np.float64(-1.0 if err is None else err)
        out[tag + '_err_baseline'] = np.float64(-1.0 if err_b is None else err_b)
        print(name, tag, 'MAP', MAP, 'n_pred', len(prec), 'err', err, err_b, flush=True)
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)


def randw200():
    rng = np.random.default_rng(11)
    n = 200
    R = nx.DiGraph()
    R.add_nodes_from(range(n))
    for _ in range(1200):
        u, v = rng.integers(0, n, 2)
        w = float(np.round(rng.uniform(0.1, 2.0), 3))
        R.add_edge(int(u), int(v), weight=w)
        if rng.uniform() < 0.4:
            R.add_edge(int(v), int(u), weight=w)          # both directions
    X = rng.standard_normal((n, 6)) * 0.5
    X[100:130] = X[0:30]                                  # duplicated rows: delta = 0 exactly, ties among them
    X[190:195] += 40.0                                    # far rows: delta ~ 9600 to the rest -> score 0
    X[195:200] -= 40.0
    return R, X


def sbm1024_lap():
    """The reference's SBM graph and LE golden, checked against the committed fixtures that stand in for them."""
    S = mg.load_sbm_nx()
    X = np.loadtxt(os.path.join(mg.REF, 'tests/smb_res/LaplacianEigenmaps.txt')).astype(np.float32)
    fx = np.load(os.path.join(HERE, 'sbm1024_LaplacianEigenmaps.npy'))
    f = np.load(os.path.join(HERE, 'sbm1024.npz'))
    assert np.array_equal(X, fx)
    assert list(S.nodes) == f['nodes'].tolist()
    assert sorted(S.edges()) == sorted(zip(f['src'].tolist(), f['dst'].tolist()))
    return S, X.astype(np.float64)


def main(cases):
    V = {'und': dict(is_undirected=True), 'dir': dict(is_undirected=False),
         'dirw': dict(is_undirected=False, is_weighted=True)}
    if 'eval_karate_lap' in cases or 'eval_karate_lle' in cases:
        K = mg.load_karate_nx()
        K.add_nodes_from(range(34))
    if 'eval_karate_lap' in cases:
        run('eval_karate_lap', K, np.loadtxt(os.path.join(mg.REF, 'tests/karate_res/LaplacianEigenmaps.txt')), V)
    if 'eval_karate_lle' in cases:
        run('eval_karate_lle', K, np.loadtxt(os.path.join(mg.REF, 'tests/karate_res/LocallyLinearEmbedding.txt')), V)
    if 'eval_randw200_gauss' in cases:
        R, X = randw200()
        run('eval_randw200_gauss', R, X, V)
    if 'eval_sbm1024_lap' in cases:
        S, X = sbm1024_lap()
        run('eval_sbm1024_lap', S, X, {'und': dict(is_undirected=True)},
            fixtures=('sbm1024.npz', 'sbm1024_LaplacianEigenmaps.npy'))


CASES = ('eval_karate_lap', 'eval_karate_lle', 'eval_randw200_gauss', 'eval_sbm1024_lap')

if __name__ == '__main__':
    main(sys.argv[1:] or CASES)
