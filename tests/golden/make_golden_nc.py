"""tests/golden/make_golden_nc.py -- goldens of node classification, made with sklearn (the library upstream GEM's
evaluateNodeClassification builds on): train_test_split, OneVsRestClassifier(LogisticRegression()) and f1_score.
Only this script imports sklearn.  Writes tests/golden/nc_*.npz and sbm1024_node_labels.npz.

Each golden: the embedding X (rows in node-id order), the 0/1 labels Y, the split (train_test_split with
random_state = RandomState(seed)), sklearn's coefficients at tol 1e-12, the TopKRanker predictions restated per the
contract of gem_b200/evaluation/evaluate_node_classification.py (p = 1 / (1 + exp(-z)) from those coefficients,
argsort(kind='stable')[-k:], k = 0: every label), micro / macro F1 of those predictions, and -- for information --
the F1 of sklearn at its default settings (tol 1e-4, 100 iterations).

Cases
  nc_karate_hope      tests/golden/karate_HOPE.txt (rows in list(graph.nodes) order, put in id order here) and
                      networkx's `club` attribute (2 labels); test_ratio 0.5
  nc_sbm1024_hope     the reference's HOPE d = 16 SBM-1024 embedding (ref_hope_sbm1024_d16.npz) and its label fixture
                      tests/data/sbm_node_labels.pickle (one-hot, 3 labels), converted to sbm1024_node_labels.npz
  nc_multilabel       synthetic, n = 400, d = 12, L = 7, rows with 0-3 labels; label 5 on no training row, label 6 on
                      every training row, test rows with k = 0

    python make_golden_nc.py [REFERENCE_CHECKOUT]      (default: $GEM_REFERENCE, as make_golden.py)
"""
import os
import pickle
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _karate():
    import networkx as nx
    G = nx.DiGraph()                                   # loaded as tests/test_karate.py:31-35 of the reference does
    with open(os.path.join(HERE, 'karate.edgelist')) as f:
        for line in f:
            e = line.split()
            G.add_edge(int(e[0]), int(e[1]))
    order = np.array(list(G.nodes), dtype=np.int64)
    Xf = np.loadtxt(os.path.join(HERE, 'karate_HOPE.txt'))
    X = np.empty_like(Xf)
    X[order] = Xf                                      # file row r is node order[r] (SURVEY F6)
    club = nx.get_node_attributes(nx.karate_club_graph(), 'club')
    Y = np.zeros((34, 2), dtype=np.int8)
    for v in range(34):
        Y[v, 0 if club[v] == 'Mr. Hi' else 1] = 1
    return X, Y, 0.5, 7


def _sbm(ref):
    z = np.load(os.path.join(HERE, 'ref_hope_sbm1024_d16.npz'))
    X = np.empty_like(z['X'])
    X[z['nodes'].astype(np.int64)] = z['X']
    with open(os.path.join(ref, 'tests/data/sbm_node_labels.pickle'), 'rb') as f:
        lab = pickle.load(f, encoding='latin1').tocsr()
    lab.sort_indices()
    np.savez_compressed(os.path.join(HERE, 'sbm1024_node_labels.npz'), indptr=lab.indptr.astype(np.int64),
                        indices=lab.indices.astype(np.int32), shape=np.array(lab.shape, dtype=np.int64))
    return X, (lab.toarray() > 0).astype(np.int8), 0.3, 11


def _multilabel():
    rng = np.random.RandomState(2024)
    n, d, L = 400, 12, 7
    centers = rng.randn(L, d) * 1.5
    Y = np.zeros((n, L), dtype=np.int8)
    X = rng.randn(n, d) * 0.8
    for i in range(n):
        k = rng.randint(0, 4)
        labs = rng.choice(5, size=k, replace=False)
        Y[i, labs] = 1
        X[i] += centers[labs].sum(0)
    seed, ratio = 5, 0.25
    test, train = split_rows(n, ratio, seed)
    Y[:, 5] = 0
    Y[test[:6], 5] = 1                                 # label 5: test rows only
    Y[train, 6] = 1                                    # label 6: every training row
    Y[test[::2], 6] = 1
    Y[test[1:8:2]] = 0                                 # k = 0 test rows
    return X, Y, ratio, seed


def split_rows(n, ratio, seed):
    from sklearn.model_selection import train_test_split
    idx = np.arange(n)
    te_tr = train_test_split(idx, test_size=ratio, random_state=np.random.RandomState(seed))
    return te_tr[1], te_tr[0]


def make(name, X, Y, ratio, seed, C=1.0):
    from sklearn.linear_model import LogisticRegression
    from sklearn.metrics import f1_score
    from sklearn.multiclass import OneVsRestClassifier, _ConstantPredictor
    n, L = Y.shape
    test, train = split_rows(n, ratio, seed)

    def fitted(**kw):
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            return OneVsRestClassifier(LogisticRegression(C=C, **kw)).fit(X[train], Y[train])

    def predict(W):
        z = X[test] @ W[:, :-1].T + W[:, -1]
        with np.errstate(over='ignore'):
            P = 1.0 / (1.0 + np.exp(-z))
        k = Y[test].sum(1)
        pred = [np.sort(np.argsort(P[i], kind='stable')[-int(k[i]):] if k[i] else np.arange(L)) for i in range(len(test))]
        Yp = np.zeros((len(test), L), dtype=np.int8)
        for i, p in enumerate(pred):
            Yp[i, p] = 1
        return pred, (f1_score(Y[test], Yp, average='micro', zero_division=0),
                      f1_score(Y[test], Yp, average='macro', zero_division=0))

    def weights(clf):
        W = np.zeros((L, X.shape[1] + 1))
        for c, e in enumerate(clf.estimators_):
            if isinstance(e, _ConstantPredictor):
                W[c, -1] = np.inf if e.y_.ravel()[0] else -np.inf
            else:
                W[c, :-1], W[c, -1] = e.coef_[0], e.intercept_[0]
        return W

    W = weights(fitted(tol=1e-12, max_iter=100000))
    pred, (mi, ma) = predict(W)
    _, (mi0, ma0) = predict(weights(fitted()))
    lens = np.array([p.size for p in pred], dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, name + '.npz'), X=X, Y=Y, test_ratio=ratio, seed=seed, C=C,
                        test_idx=test, train_idx=train, W=W,
                        pred_indptr=np.concatenate(([0], np.cumsum(lens))), pred_indices=np.concatenate(pred),
                        micro=mi, macro=ma, micro_sklearn_default=mi0, macro_sklearn_default=ma0)
    print('%-16s n=%d d=%d L=%d micro %.6f macro %.6f (sklearn defaults: %.6f %.6f)'
          % (name, n, X.shape[1], L, mi, ma, mi0, ma0))


if __name__ == '__main__':
    ref = sys.argv[1] if len(sys.argv) > 1 else os.environ.get('GEM_REFERENCE', '/root/reference')
    make('nc_karate_hope', *_karate())
    make('nc_sbm1024_hope', *_sbm(ref))
    make('nc_multilabel', *_multilabel())
