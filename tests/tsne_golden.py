"""Loader of the t-SNE goldens (tests/golden/make_golden_tsne.py).

The goldens keep what only sklearn can say (neighbour sets, a sample of calibrated rows, PCA starts, positions,
gradients, KL, trustworthiness) and not what follows from it: the inputs are rebuilt by the generator's inputs() from
the committed fixtures, and the joint P is the oracle's chain on sklearn's neighbour sets (fp64 d^2 of those pairs
rounded to fp32, calibrate, joint), which tests/test_oracle_tsne.py pins to the stored rows and to sklearn's nnz.
-> dict of the golden's arrays plus X (float32), labels (or None), knn_d2 (fp32 d^2 aligned with knn_idx) and P (CSR)."""
import functools
import os
import sys

import numpy as np

from conftest import GOLDEN, REPO

sys.path.insert(0, GOLDEN)
sys.path.insert(0, os.path.join(REPO, 'oracle'))
import make_golden_tsne  # noqa: E402
import tsne_oracle as to  # noqa: E402

CASES = ['tsne_karate_d4', 'tsne_sbm1024_d16', 'tsne_sbm1024_d256', 'tsne_mix2000_d64']


@functools.lru_cache(maxsize=None)
def _inputs():
    return {name: (X, labels) for name, X, labels in make_golden_tsne.inputs()}


@functools.lru_cache(maxsize=None)
def _load(name):
    z = np.load(os.path.join(GOLDEN, name + '.npz'))
    z = {k: z[k] for k in z.files}
    X, labels = _inputs()[name]
    n = X.shape[0]
    idx = z['knn_idx'].astype(np.int64)
    rows = np.repeat(np.arange(n), idx.shape[1])
    d2 = ((X[rows].astype(np.float64) - X[idx.ravel()].astype(np.float64)) ** 2).sum(1).astype(np.float32)
    z.update(X=X, labels=labels, knn_idx=idx, knn_d2=d2.reshape(idx.shape))
    z['p_cond_oracle'] = to.calibrate(z['knn_d2'], float(z['perplexity']))
    z['P'] = to.joint(idx, z['p_cond_oracle'], n)
    return z


def load(name):
    """A fresh dict (the arrays are shared: do not modify them)."""
    return dict(_load(name))
