"""Node classification on the GPU: the goldens end to end, optimality of the batched L-BFGS fit against the fp64
certificate of oracle/nc_oracle.py, the top-k kernel against the oracle's ranking, repeatability, the unconverged
path and ownership of device blocks."""
import os
import sys
import warnings

import numpy as np
import pytest

from conftest import REPO, golden_path

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import nc_oracle as no  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = ['nc_karate_hope', 'nc_sbm1024_hope', 'nc_multilabel']
CERT_BAR = 1e-4          # 10x the default tol of 1e-5


def _pred_rows(p, ix):
    return [np.sort(ix[p[i]:p[i + 1]]) for i in range(len(p) - 1)]


@pytest.mark.parametrize('name', CASES)
def test_goldens_end_to_end(native_lib, name):
    from gem_b200.evaluation.evaluate_node_classification import evaluateNodeClassification
    z = np.load(golden_path(name + '.npz'))
    st = {}
    mi, ma = evaluateNodeClassification(z['X'], z['Y'], float(z['test_ratio']), seed=int(z['seed']), C=float(z['C']),
                                        stats=st)
    assert np.array_equal(st['test_idx'], z['test_idx'])
    test = z['test_idx']
    k = z['Y'][test].sum(1)
    P = no.probabilities(z['X'][test], z['W'])
    skip = set(no.near_tie_rows(P, k).tolist())
    got, ref = _pred_rows(st['pred_indptr'], st['pred_indices']), no.topk(P, k)
    bad = [i for i in range(len(test)) if not np.array_equal(got[i], ref[i])]
    print('%s: %d near-tie rows, micro %.6f macro %.6f' % (name, len(skip), mi, ma))
    assert not skip                 # no near ties on these goldens: every row is compared
    assert not bad
    assert abs(mi - float(z['micro'])) <= 1e-12 and abs(ma - float(z['macro'])) <= 1e-12
    cert = no.certificate(z['X'][z['train_idx']], z['Y'][z['train_idx']], float(z['C']), st['W'])
    assert np.nanmax(cert) <= CERT_BAR


def _multilabel(n, d, L, seed):
    rng = np.random.RandomState(seed)
    k = rng.randint(0, 4, n)
    lab = [np.sort(rng.choice(L, size=int(kk), replace=False)) for kk in k]
    centers = rng.randn(L, d) / np.sqrt(max(d, 1)) * 1.5
    X = rng.randn(n, d).astype(np.float32)
    for i, ls in enumerate(lab):
        if ls.size:
            X[i] += centers[ls].sum(0)
    Y = np.zeros((n, L), dtype=np.int8)
    for i, ls in enumerate(lab):
        Y[i, ls] = 1
    return X.astype(np.float32), Y


@pytest.fixture(scope='module', params=[2, 64, 128, 182], ids=lambda d: 'd%d' % d)
def big(request):
    return _multilabel(40_000, request.param, 300, 100 + request.param)


@pytest.mark.parametrize('C', [1.0, 0.01])
def test_optimality_and_predictions(gpu_ctx, big, C):
    """n = 40 000, L = 300 (panels of 128, 128 and 44), multi-label: every label's fp64 certificate at the GPU's
    weights is <= 1e-4, and the top-k kernel picks the oracle's labels on every row that is not a near tie."""
    from gem_b200 import _native
    from gem_b200.evaluation.evaluate_node_classification import _label_csr
    X, Y = big
    n, d = X.shape
    ntr = 30_000
    ptr, lab = _label_csr(Y[:ntr])
    W, iters, status, st = _native.nc_fit(gpu_ctx, X[:ntr], ptr, lab, Y.shape[1], C=C)
    cert = no.certificate(X[:ntr], Y[:ntr], C, W)
    print('d=%d C=%g: certificate max %.3g median %.3g, iterations %d / %d / %d, %d evaluations, %d unconverged'
          % (d, C, np.nanmax(cert), np.nanmedian(cert), iters.min(), np.median(iters), iters.max(), st['evaluations'],
             st['unconverged']))
    assert st['panels'] == 3
    assert np.nanmax(cert) <= CERT_BAR
    Xt, Yt = X[ntr:], Y[ntr:]
    tp, _ = _label_csr(Yt)
    pred = _native.nc_topk(gpu_ctx, Xt, W, tp)
    k = np.diff(tp)
    P = no.probabilities(Xt, W)
    skip = set(no.near_tie_rows(P, k).tolist())
    ref = no.topk(P, k)
    got = _pred_rows(tp, pred)
    bad = [i for i in range(len(k)) if k[i] and i not in skip and not np.array_equal(got[i], ref[i])]
    print('  predictions: %d of %d rows excluded as near ties, %d differ' % (len(skip), len(k), len(bad)))
    assert not bad


def test_repeatable_bits(gpu_ctx):
    from gem_b200 import _native
    from gem_b200.evaluation.evaluate_node_classification import _label_csr
    X, Y = _multilabel(12_000, 64, 140, 7)
    ptr, lab = _label_csr(Y[:9000])
    tp, _ = _label_csr(Y[9000:])
    runs = []
    for _ in range(2):
        W, iters, status, _ = _native.nc_fit(gpu_ctx, X[:9000], ptr, lab, 140)
        runs.append((W.tobytes(), iters.tobytes(), status.tobytes(), _native.nc_topk(gpu_ctx, X[9000:], W, tp).tobytes()))
    assert runs[0] == runs[1]


def test_unconverged_warns_and_flags(native_lib):
    from gem_b200 import _native
    from gem_b200.evaluation.evaluate_node_classification import evaluateNodeClassification
    X, Y = _multilabel(6000, 16, 20, 9)
    st = {}
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        evaluateNodeClassification(X, Y, 0.5, seed=3, max_iter=2, stats=st)
    msgs = [x for x in w if issubclass(x.category, RuntimeWarning) and 'stopped at max_iter=2' in str(x.message)]
    assert msgs and msgs[0].filename == __file__
    assert st['unconverged'].size > 0
    assert np.all(st['status'][st['unconverged']] == _native.NC_MAXITER)
    assert np.all(st['iters'] <= 2)


@pytest.mark.skipif(os.environ.get('GEMB_CACHE_MB', '').strip() == '0',
                    reason='GEMB_CACHE_MB=0: no block cache, gemb_mem_live_blocks is always 0')
def test_no_block_leaked(gpu_ctx):
    from gem_b200 import _native
    from gem_b200.evaluation.evaluate_node_classification import _label_csr
    X, Y = _multilabel(5000, 24, 30, 11)
    ptr, lab = _label_csr(Y[:4000])
    tp, _ = _label_csr(Y[4000:])
    W = _native.nc_fit(gpu_ctx, X[:4000], ptr, lab, 30)[0]
    for call in (lambda: _native.nc_fit(gpu_ctx, X[:4000], ptr, lab, 30),
                 lambda: _native.nc_topk(gpu_ctx, X[4000:], W, tp)):
        call()
        before = _native.mem_live_blocks()
        call()
        assert _native.mem_live_blocks() == before
    bad = lab.copy()
    bad[0] = 30                                   # out of range: rejected before any allocation
    before = _native.mem_live_blocks()
    with pytest.raises(RuntimeError, match='label id'):
        _native.nc_fit(gpu_ctx, X[:4000], ptr, bad, 30)
    assert _native.mem_live_blocks() == before
