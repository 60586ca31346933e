"""tests/golden/make_golden_tsne.py -- goldens of t-SNE, made with sklearn 1.9 (the library the reference's
plot_embedding2D calls: TSNE(n_components=2).fit_transform).  Only this script imports sklearn.
Writes tests/golden/tsne_*.npz.

Every case feeds sklearn the fp32 rounding of its embedding (as float64), i.e. exactly the data gem_b200's fp32 path
sees.  The inputs are not stored: inputs() rebuilds them from the fixtures named below (and a seed), and the tests call
it.  Each golden holds
    knn_idx           NearestNeighbors(k).kneighbors() without the query row, k = min(n - 1, int(3 perplexity + 1)):
                      each row's neighbour SET, ascending ids (int16)
    p_rows, p_cond    _binary_search_perplexity (sklearn's float64, stored as float32) on rows p_rows = every eighth
                      row, its columns in the order of knn_idx
    nnz_P             entries of _joint_probabilities_nn's symmetrised CSR (zeros dropped)
    Y0                the PCA start as TSNE._fit makes it (fp32); pca_solver: the solver PCA picked
    Y250, Y1000       TSNE(random_state=0, max_iter=250 / default 1000).embedding_
    grad_bh{a}_{pos}, kl_bh{a}_{pos}  _kl_divergence_bh at angle a in {0, 0.5} (files: '0', '05') and pos in
                      {Y0, Y250, Y1000} (gradient including the factor 4, KL error; float32)
    grad_exact_{pos}, kl_exact_{pos}  _kl_divergence (method='exact') on the same P (dense)
    kl_final, n_iter, trust12        TSNE(random_state=0).kl_divergence_, n_iter_ and trustworthiness(X, Y, 12)
    nn_same           (SBM cases) the share of nodes whose nearest 2-D neighbour in sklearn's embedding shares its
                      community (labels: sbm1024_node_labels.npz)

Cases
    tsne_karate_d4      tests/golden/karate_HOPE.txt (34 x 4; k = 33: every other node)
    tsne_sbm1024_d16    ref_hope_sbm1024_d16.npz with sbm1024_node_labels.npz
    tsne_sbm1024_d256   ref_hope_sbm1024_d256.npz (n < 10 d: sklearn's PCA is randomized there)
    tsne_mix2000_d64    seeded 2000-point mixture of 6 Gaussians in 64 dimensions with 40 duplicated rows

    python make_golden_tsne.py
"""
import os
import sys

import numpy as np
from scipy.spatial.distance import squareform

HERE = os.path.dirname(os.path.abspath(__file__))


def inputs():
    """(name, X float32, community labels or None) of every case, rebuilt from the fixtures."""
    for name, X, labels in _inputs64():
        yield name, X.astype(np.float32), labels


def _inputs64():
    yield 'tsne_karate_d4', np.loadtxt(os.path.join(HERE, 'karate_HOPE.txt')), None
    lab = np.load(os.path.join(HERE, 'sbm1024_node_labels.npz'))
    labels = lab['indices'][np.argsort(np.repeat(np.arange(1024), np.diff(lab['indptr'])), kind='stable')]
    for d in (16, 256):
        yield 'tsne_sbm1024_d%d' % d, np.load(os.path.join(HERE, 'ref_hope_sbm1024_d%d.npz' % d))['X'], labels
    rng = np.random.RandomState(20)
    centres = rng.randn(6, 64) * 3.0
    X = centres[rng.randint(0, 6, 2000)] + rng.randn(2000, 64)
    X[1960:] = X[rng.choice(1960, 40, replace=False)]
    yield 'tsne_mix2000_d64', X, None


def main():
    import sklearn
    from sklearn.decomposition import PCA
    from sklearn.manifold import TSNE, trustworthiness
    from sklearn.manifold._t_sne import _joint_probabilities_nn, _kl_divergence, _kl_divergence_bh
    from sklearn.manifold._utils import _binary_search_perplexity
    from sklearn.neighbors import NearestNeighbors
    print('sklearn', sklearn.__version__)
    perplexity = 30.0
    for name, X32, labels in inputs():
        X = X32.astype(np.float64)
        n = X.shape[0]
        k = min(n - 1, int(3.0 * perplexity + 1))
        nn = NearestNeighbors(n_neighbors=k).fit(X)
        dist, idx = nn.kneighbors()
        d2 = dist ** 2
        p_cond = _binary_search_perplexity(d2.astype(np.float32), perplexity, 0)
        G = nn.kneighbors_graph(mode='distance')
        G.data **= 2
        P = _joint_probabilities_nn(G, perplexity, 0).tocsr()
        P.sort_indices()
        pca = PCA(n_components=2, random_state=0)
        pca.set_output(transform='default')
        Y0 = pca.fit_transform(X).astype(np.float32, copy=False)
        Y0 = Y0 / np.std(Y0[:, 0]) * 1e-4
        order = np.argsort(idx, axis=1, kind='stable')
        rows = np.arange(0, n, 8)
        out = dict(perplexity=perplexity, knn_idx=np.take_along_axis(idx, order, 1).astype(np.int16),
                   p_rows=rows.astype(np.int32),
                   p_cond=np.take_along_axis(p_cond, order, 1)[rows].astype(np.float32), nnz_P=int(P.nnz),
                   Y0=Y0, pca_solver=pca._fit_svd_solver)
        runs = {}
        for it in (250, 1000):
            t = TSNE(random_state=0, max_iter=it).fit(X)
            runs[it] = t
            out['Y%d' % it] = t.embedding_.astype(np.float32)
        t = runs[1000]
        out['kl_final'], out['n_iter'] = float(t.kl_divergence_), int(t.n_iter_)
        out['trust12'] = float(trustworthiness(X, t.embedding_, n_neighbors=12))
        Pc = squareform(P.toarray(), checks=False)
        for pos in ('Y0', 'Y250', 'Y1000'):
            Y = out[pos].astype(np.float32)
            for a, tag in ((0.0, '0'), (0.5, '05')):
                e, g = _kl_divergence_bh(Y.ravel().copy(), P, 1, n, 2, angle=a, compute_error=True)
                out['grad_bh%s_%s' % (tag, pos)] = g.reshape(n, 2).astype(np.float32)
                out['kl_bh%s_%s' % (tag, pos)] = float(e)
            e, g = _kl_divergence(Y.ravel().astype(np.float64), Pc, 1, n, 2)
            out['grad_exact_%s' % pos] = g.reshape(n, 2)
            out['kl_exact_%s' % pos] = float(e)
        if labels is not None:
            E = t.embedding_
            D = ((E[:, None, :] - E[None, :, :]) ** 2).sum(-1)
            np.fill_diagonal(D, np.inf)
            out['nn_same'] = float(np.mean(labels[D.argmin(1)] == labels))
        np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
        print('%s: %d bytes, n %d d %d k %d nnz %d solver %s kl %.6f n_iter %d trust12 %.4f%s'
              % (name, os.path.getsize(os.path.join(HERE, name + '.npz')), n, X.shape[1], k, P.nnz, out['pca_solver'],
                 out['kl_final'], out['n_iter'], out['trust12'], '' if labels is None else ' nn_same %.4f' % out['nn_same']))


if __name__ == '__main__':
    sys.exit(main())
