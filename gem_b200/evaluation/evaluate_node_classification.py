"""evaluateNodeClassification on an H100: one-vs-rest logistic regression on the embedding, TopKRanker prediction and
micro / macro F1 -- upstream GEM's evaluateNodeClassification (OneVsRestClassifier(LogisticRegression()) with its
TopKRanker), which the reference checkout does not ship.

    1. split    sklearn's train_test_split(X, Y, test_size=test_ratio, random_state=rng), restated: rng is
                np.random.RandomState(seed) (the global np.random when seed is None), n_test = ceil(test_ratio n),
                perm = rng.permutation(n), test rows perm[:n_test], training rows perm[n_test:]
    2. fit      for every label c the minimiser of 1/2 |w|^2 + C sum_i log(1 + exp(-s_i (w . x_i + b))) over the
                training rows (s_i = +1 where the row carries c, else -1; b not penalised) -- gemb_nc_fit, batched
                L-BFGS on the GPU.  A label no training row carries is the constant p = 0, one that every training
                row carries the constant p = 1 (sklearn's _ConstantPredictor)
    3. predict  test row i with k_i true labels gets the k_i labels of largest p = 1 / (1 + exp(-(w . x + b))), exact
                ties to the larger label index (argsort(kind='stable')[-k:]) -- gemb_nc_topk.  A row with k_i = 0
                gets every label, as upstream's argsort()[-0:] does
    4. score    micro and macro F1 over the labels (sklearn.metrics.f1_score; a label with tp + fp + fn = 0 counts 0
                in the macro average), on the host from the O(sum k) predictions

tol is relative: label c stops when max|grad f_c| <= tol * max|grad f_c(0, 0)|.  A label that reaches max_iter first,
or whose line search finds no acceptable step in 40 trials, warns (RuntimeWarning, pointing at the caller; the message
names the two causes apart).  No CPU fallback: without a GPU this raises RuntimeError.
"""
import math
import time
import warnings

import numpy as np

from gem_b200 import _native
from gem_b200.evaluation import metrics


def _label_csr(Y):
    """0/1 indicator (dense or scipy.sparse) -> (indptr int64, label ids int32, ascending per row); ValueError on any
    other value."""
    if hasattr(Y, 'tocsr'):
        Y = Y.tocsr(copy=True)
        Y.sum_duplicates()
        Y.eliminate_zeros()
        Y.sort_indices()
        if Y.data.size and not np.all(Y.data == 1):
            raise ValueError('Y must hold only 0 and 1')
        return np.asarray(Y.indptr, dtype=np.int64), np.asarray(Y.indices, dtype=np.int32)
    Y = np.asarray(Y)
    if Y.size and not np.all((Y == 0) | (Y == 1)):
        raise ValueError('Y must hold only 0 and 1')
    r, c = np.nonzero(Y)
    indptr = np.zeros(Y.shape[0] + 1, dtype=np.int64)
    np.cumsum(np.bincount(r, minlength=Y.shape[0]), out=indptr[1:])
    return indptr, c.astype(np.int32)


def _rows(indptr, indices, rows):
    """The CSR rows `rows`, in that order."""
    lens = np.diff(indptr)[rows]
    out_ptr = np.zeros(rows.size + 1, dtype=np.int64)
    np.cumsum(lens, out=out_ptr[1:])
    starts = np.repeat(indptr[rows] - out_ptr[:-1], lens)
    return out_ptr, indices[np.arange(out_ptr[-1], dtype=np.int64) + starts]


def split(n, test_ratio, seed=None):
    """Step 1: (test rows, training rows)."""
    rng = np.random if seed is None else np.random.RandomState(seed)
    n_test = int(math.ceil(test_ratio * n))
    perm = rng.permutation(n)
    return perm[:n_test], perm[n_test:]


def evaluateNodeClassification(X, Y, test_ratio, seed=None, C=1.0, tol=1e-5, max_iter=1000, device=None, stats=None):
    """-> (micro_f1, macro_f1).  X: n x d embedding (rows = node ids); Y: n x L 0/1 indicator, dense or scipy.sparse.
    stats: an optional dict, filled with the split, the weights (L x (d + 1)), the per-label iterations and status
    (gem_b200._native.NC_*), the labels that did not converge, the predictions and the host-clock times in ms."""
    X = np.asarray(X)
    if X.ndim != 2 or X.shape[0] == 0 or X.shape[1] == 0:
        raise ValueError('X must be a non-empty n x d matrix, got shape %s' % (X.shape,))
    if not np.all(np.isfinite(X)):
        raise ValueError('X must be finite')
    if len(getattr(Y, 'shape', ())) != 2 or Y.shape[0] != X.shape[0] or Y.shape[1] == 0:
        raise ValueError('Y must be an n x L indicator with n = %d rows, got shape %s'
                         % (X.shape[0], getattr(Y, 'shape', None)))
    if not 0.0 < float(test_ratio) < 1.0:
        raise ValueError('test_ratio must lie in (0, 1), got %r' % (test_ratio,))
    if not (C > 0 and tol >= 0 and max_iter >= 0):
        raise ValueError('need C > 0, tol >= 0 and max_iter >= 0')
    n, L = int(X.shape[0]), int(Y.shape[1])
    if int(math.ceil(float(test_ratio) * n)) >= n:
        raise ValueError('test_ratio %r leaves no training row of %d' % (test_ratio, n))
    indptr, labels = _label_csr(Y)
    t0 = time.perf_counter()
    test, train = split(n, float(test_ratio), seed)
    tr_ptr, tr_lab = _rows(indptr, labels, train)
    te_ptr, te_lab = _rows(indptr, labels, test)
    Xf = np.ascontiguousarray(X, dtype=np.float32)
    X_train, X_test = Xf[train], Xf[test]
    t1 = time.perf_counter()
    with _native.Context(0 if device is None else int(device)) as ctx:
        W, iters, status, st = _native.nc_fit(ctx, X_train, tr_ptr, tr_lab, L, C, tol, max_iter)
        t2 = time.perf_counter()
        pred = _native.nc_topk(ctx, X_test, W, te_ptr)
        t3 = time.perf_counter()
    # k = 0 rows: every label
    k = np.diff(te_ptr)
    lens = np.where(k == 0, L, k)
    p_ptr = np.zeros(test.size + 1, dtype=np.int64)
    np.cumsum(lens, out=p_ptr[1:])
    p_lab = np.empty(int(p_ptr[-1]), dtype=np.int32)
    own = np.repeat(k > 0, lens)
    p_lab[own] = pred
    p_lab[~own] = np.tile(np.arange(L, dtype=np.int32), int((k == 0).sum()))
    micro, macro = metrics.f1_from_predictions(L, te_ptr, te_lab, p_ptr, p_lab)
    maxit = np.flatnonzero(status == _native.NC_MAXITER)
    stalled = np.flatnonzero(status == _native.NC_STALLED)
    bad = np.union1d(maxit, stalled)
    if stats is not None:
        stats.update(test_idx=test, train_idx=train, W=W, iters=iters, status=status, unconverged=bad,
                     pred_indptr=p_ptr, pred_indices=p_lab, split_ms=1e3 * (t1 - t0), fit_ms=1e3 * (t2 - t1),
                     topk_ms=1e3 * (t3 - t2), fit_stats=st)
    if bad.size:
        why = []
        if maxit.size:
            why.append('%d stopped at max_iter=%d (first: %s)' % (maxit.size, max_iter, maxit[:8].tolist()))
        if stalled.size:
            why.append('%d stopped because the line search found no acceptable step (first: %s)'
                       % (stalled.size, stalled[:8].tolist()))
        warnings.warn('evaluateNodeClassification: %d of %d labels did not meet tol=%g: %s'
                      % (bad.size, L, tol, '; '.join(why)), RuntimeWarning, stacklevel=2)
    return micro, macro
