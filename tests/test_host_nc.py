"""Host side of node classification without a GPU: every ValueError of evaluateNodeClassification comes before any
device call, there is no CPU fallback, and the product never imports sklearn."""
import os
import re

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import REPO


@pytest.fixture
def no_device(monkeypatch):
    """Fail loudly if the evaluation reaches the library."""
    from gem_b200 import _native

    def boom(*a, **k):
        raise AssertionError('device call before validation')
    monkeypatch.setattr(_native, 'Context', boom)
    monkeypatch.setattr(_native, 'lib', boom)


def _data(n=20, d=3, L=4):
    rng = np.random.RandomState(0)
    X = rng.randn(n, d)
    Y = np.zeros((n, L), dtype=np.int8)
    Y[np.arange(n), rng.randint(0, L, n)] = 1
    return X, Y


@pytest.mark.parametrize('bad', [
    lambda X, Y: (X[:-1], Y, 0.5),                                   # shape mismatch
    lambda X, Y: (X[:, 0], Y, 0.5),                                  # X not 2-D
    lambda X, Y: (X, Y[:, :0], 0.5),                                 # no labels
    lambda X, Y: (X, np.where(Y > 0, 2, 0), 0.5),                    # a value other than 0/1
    lambda X, Y: (X, sp.csr_matrix(np.where(Y > 0, 0.5, 0)), 0.5),   # sparse, not 0/1
    lambda X, Y: (X, Y, 0.0),                                        # test_ratio outside (0, 1)
    lambda X, Y: (X, Y, 1.0),
    lambda X, Y: (X, Y, -0.2),
    lambda X, Y: (X, Y, 0.99),                                       # empty training split
    lambda X, Y: (np.where(X > 1, np.nan, X), Y, 0.5),               # non-finite X
], ids=['shape', 'x1d', 'nolabels', 'value', 'sparse-value', 'ratio0', 'ratio1', 'ratio-neg', 'empty-train', 'nan'])
def test_value_errors_before_any_device_call(no_device, bad):
    from gem_b200.evaluation.evaluate_node_classification import evaluateNodeClassification
    X, Y, r = bad(*_data())
    with pytest.raises(ValueError):
        evaluateNodeClassification(X, Y, r, seed=1)


def test_label_csr_dense_and_sparse_agree():
    from gem_b200.evaluation.evaluate_node_classification import _label_csr, _rows
    X, Y = _data()
    Y[3] = 0
    Y[4, :3] = 1
    a, b = _label_csr(Y), _label_csr(sp.csr_matrix(Y))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    rows = np.array([4, 3, 0])
    p, ix = _rows(a[0], a[1], rows)
    assert np.array_equal(np.diff(p), Y[rows].sum(1))
    assert np.array_equal(ix, np.concatenate([np.flatnonzero(Y[r]) for r in rows]))


def test_no_cpu_fallback(native_lib):
    if native_lib.gemb_device_count() > 0:
        pytest.skip('a GPU is present')
    from gem_b200.evaluation.evaluate_node_classification import evaluateNodeClassification
    X, Y = _data()
    with pytest.raises(RuntimeError):
        evaluateNodeClassification(X, Y, 0.5, seed=1)


def test_product_does_not_import_sklearn():
    pat = re.compile(r'^\s*(import\s+sklearn|from\s+sklearn)', re.M)
    hits = []
    for root, _, files in os.walk(os.path.join(REPO, 'gem_b200')):
        for f in files:
            if f.endswith('.py'):
                with open(os.path.join(root, f)) as fh:
                    if pat.search(fh.read()):
                        hits.append(f)
    assert not hits


def test_warning_names_each_cause(monkeypatch):
    """A label stopped by max_iter and one whose line search stalled are reported as such (the fit itself is faked)."""
    import warnings
    from gem_b200 import _native
    from gem_b200.evaluation import evaluate_node_classification as enc

    class Ctx:
        def __init__(self, device):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *exc):
            return False

    def fake_fit(ctx, X, indptr, labels, L, C, tol, max_iter):
        status = np.full(L, _native.NC_CONVERGED, dtype=np.int32)
        status[1], status[3] = _native.NC_MAXITER, _native.NC_STALLED
        return np.zeros((L, X.shape[1] + 1)), np.ones(L, dtype=np.int32), status, {}

    def fake_topk(ctx, X, W, koff):
        return np.zeros(int(koff[-1]), dtype=np.int32)
    monkeypatch.setattr(_native, 'Context', Ctx)
    monkeypatch.setattr(_native, 'nc_fit', fake_fit)
    monkeypatch.setattr(_native, 'nc_topk', fake_topk)
    X, Y = _data()
    st = {}
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        enc.evaluateNodeClassification(X, Y, 0.5, seed=1, max_iter=7, stats=st)
    msg = ' '.join(str(x.message) for x in w if issubclass(x.category, RuntimeWarning))
    assert '2 of 4 labels' in msg and '1 stopped at max_iter=7 (first: [1])' in msg
    assert 'line search found no acceptable step (first: [3])' in msg
    assert np.array_equal(st['unconverged'], [1, 3])
