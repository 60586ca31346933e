"""The fp64 oracle of node classification (oracle/nc_oracle.py) reproduces every nc_*.npz golden made with sklearn:
the split, the tight fit, the TopKRanker predictions and micro / macro F1; the host F1 of the product agrees."""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, golden_path

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import nc_oracle as no  # noqa: E402

CASES = ['nc_karate_hope', 'nc_sbm1024_hope', 'nc_multilabel']


@pytest.fixture(scope='module', params=CASES)
def case(request):
    z = np.load(golden_path(request.param + '.npz'))
    test, train = no.split(z['Y'].shape[0], float(z['test_ratio']), int(z['seed']))
    W = no.fit(z['X'][train], z['Y'][train], float(z['C']))
    return z, test, train, W


def _golden_pred(z):
    p, ix = z['pred_indptr'], z['pred_indices']
    return [ix[p[i]:p[i + 1]] for i in range(len(p) - 1)]


def test_split(case):
    z, test, train, _ = case
    assert np.array_equal(test, z['test_idx']) and np.array_equal(train, z['train_idx'])


def test_fit_matches_sklearn_tight(case):
    z, _, train, W = case
    Wg = z['W']
    const = ~np.isfinite(Wg[:, -1])
    assert np.array_equal(Wg[const], W[const])
    scale = np.abs(Wg[~const]).max(1, keepdims=True)
    assert np.abs(W[~const] - Wg[~const]).max() <= 1e-6 * scale.max()
    cert = no.certificate(z['X'][train], z['Y'][train], float(z['C']), W)
    assert np.nanmax(cert) < 1e-8


def test_predictions_and_f1(case):
    z, test, _, W = case
    Y = z['Y']
    L = Y.shape[1]
    P = no.probabilities(z['X'][test], W)
    k = Y[test].sum(1)
    pred = no.topk(P, k)
    gold = _golden_pred(z)
    assert all(np.array_equal(a, b) for a, b in zip(pred, gold))
    mi, ma = no.f1(Y[test], pred, L)
    assert abs(mi - float(z['micro'])) <= 1e-12 and abs(ma - float(z['macro'])) <= 1e-12
    # the product's host F1 from the CSR predictions
    from gem_b200.evaluation import metrics
    from gem_b200.evaluation.evaluate_node_classification import _label_csr
    tp, ti = _label_csr(Y[test])
    mi2, ma2 = metrics.f1_from_predictions(L, tp, ti, z['pred_indptr'], z['pred_indices'])
    assert abs(mi2 - float(z['micro'])) <= 1e-12 and abs(ma2 - float(z['macro'])) <= 1e-12


def test_multilabel_case_covers_the_corners():
    z = np.load(golden_path('nc_multilabel.npz'))
    Y, train, test = z['Y'], z['train_idx'], z['test_idx']
    ntr = Y[train].sum(0)
    assert (ntr == 0).any() and (ntr == len(train)).any()
    k = Y[test].sum(1)
    assert (k == 0).any() and k.max() >= 3


def test_sbm_labels_are_the_reference_fixture():
    z = np.load(golden_path('sbm1024_node_labels.npz'))
    g = np.load(golden_path('sbm1024.npz'))
    assert tuple(z['shape']) == (1024, 3) and np.array_equal(np.diff(z['indptr']), np.ones(1024))
    assert np.array_equal(z['indices'], g['labels'])
    nc = np.load(golden_path('nc_sbm1024_hope.npz'))
    assert np.array_equal(nc['Y'].argmax(1), g['labels'])
