"""Loader of the Gaussian-score evaluation goldens (tests/golden/make_golden_eval_gauss.py).

A golden either holds its graph and X itself, like every eval_*.npz, or names committed fixtures instead
(`graph_fixture`: an .npz with nodes / src / dst, unit weights; `X_fixture`: an .npy) so that large inputs are stored
once.  -> (z, n, (indptr, indices, weights)) as conftest.eval_golden, with z['X'] fp64 and z['nodes'] filled in."""
import numpy as np

from conftest import eval_golden, golden_path


def gauss_golden(name):
    z = np.load(golden_path(name + '.npz'))
    if 'graph_fixture' not in z.files:
        z, n, csr = eval_golden(name)
        return dict(z), n, csr
    z = dict(z)
    g = np.load(golden_path(str(z['graph_fixture'])))
    src, dst = g['src'].astype(np.int64), g['dst'].astype(np.int64)
    n = int(z['n'])
    z['nodes'] = g['nodes'].astype(np.int64)
    z['X'] = np.load(golden_path(str(z['X_fixture']))).astype(np.float64)
    assert z['nodes'].size == n and z['X'].shape[0] == n
    order = np.lexsort((dst, src))
    src, dst = src[order], dst[order]
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, src + 1, 1)
    return z, n, (np.cumsum(indptr), dst, np.ones(dst.size))
