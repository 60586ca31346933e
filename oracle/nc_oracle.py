"""oracle/nc_oracle.py -- fp64 NumPy / SciPy restatement of node classification (upstream GEM's
evaluateNodeClassification with its TopKRanker over OneVsRestClassifier(LogisticRegression())).

    split      sklearn's train_test_split(X, Y, test_size=r, random_state=rng): n_test = ceil(r n),
               perm = rng.permutation(n), test = perm[:n_test], train = perm[n_test:]
    objective  f_c(w, b) = 1/2 |w|^2 + C sum_i log(1 + exp(-s_i (w . x_i + b))), s_i = +-1, b not penalised
    fit        the minimiser of every f_c by scipy L-BFGS-B run tight; labels with no positive (every row positive)
               training row: the constant p = 0 (p = 1), stored as w = 0, b = -inf (+inf)
    certificate  max|grad f_c(w, b)| / max|grad f_c(0, 0)| at any given weights
    top-k      p = 1 / (1 + exp(-z)); row i gets argsort(p, kind='stable')[-k_i:] (ties to the larger label), k_i = 0:
               every label (upstream's argsort()[-0:])
    F1         micro and macro over the labels as sklearn.metrics.f1_score (a label with tp + fp + fn = 0 counts 0)

Checker only: nothing under gem_b200/ imports this file.
"""
import math

import numpy as np
from scipy.optimize import minimize


def split(n, test_ratio, seed=None):
    """-> (test rows, train rows)"""
    rng = np.random if seed is None else np.random.RandomState(seed)
    n_test = int(math.ceil(test_ratio * n))
    perm = rng.permutation(n)
    return perm[:n_test], perm[n_test:]


def objective(X, y, C, wb):
    """f_c and its gradient (fp64) at wb = (w, b) for the 0/1 label column y."""
    X = np.asarray(X, dtype=np.float64)
    w, b = wb[:-1], wb[-1]
    z = X @ w + b
    s = np.where(y > 0, 1.0, -1.0)
    f = 0.5 * w @ w + C * np.logaddexp(0.0, -s * z).sum()
    r = C * (_sigmoid(z) - (y > 0))
    return f, np.concatenate([X.T @ r + w, [r.sum()]])


def _sigmoid(z):
    e = np.exp(-np.abs(z))
    return np.where(z >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def fit(X, Y, C=1.0):
    """-> W, L x (d + 1): row c = (w_c, b_c), the minimiser of f_c (constants as +-inf intercepts)."""
    X = np.asarray(X, dtype=np.float64)
    Y = np.asarray(Y)
    n, d = X.shape
    W = np.zeros((Y.shape[1], d + 1))
    for c in range(Y.shape[1]):
        y = Y[:, c]
        npos = int((y > 0).sum())
        if npos == 0 or npos == n:
            W[c, d] = np.inf if npos else -np.inf
            continue
        r = minimize(lambda v: objective(X, y, C, v), np.zeros(d + 1), jac=True, method='L-BFGS-B',
                     options=dict(gtol=1e-13, ftol=1e-16, maxiter=100000, maxcor=30))
        W[c] = r.x
    return W


def certificate(X, Y, C, W):
    """max|grad f_c(W_c)| / max|grad f_c(0, 0)| per label (nan for the constant labels)."""
    X = np.asarray(X, dtype=np.float64)
    Y = np.asarray(Y) > 0
    W = np.asarray(W, dtype=np.float64)
    Z = X @ W[:, :-1].T + W[:, -1]
    const = ~np.isfinite(W[:, -1])
    Z[:, const] = 0.0
    R = C * (_sigmoid(Z) - Y)
    g = np.vstack([X.T @ R + W[:, :-1].T, R.sum(0)])
    R0 = C * (0.5 - Y)
    g0 = np.vstack([X.T @ R0, R0.sum(0)])
    out = np.abs(g).max(0) / np.abs(g0).max(0)
    out[const] = np.nan
    return out


def probabilities(X, W):
    """p = 1 / (1 + exp(-(X w + b))) in fp64, m x L."""
    X = np.asarray(X, dtype=np.float64)
    W = np.asarray(W, dtype=np.float64)
    with np.errstate(over='ignore'):
        return 1.0 / (1.0 + np.exp(-(X @ W[:, :-1].T + W[:, -1])))


def topk(P, k):
    """TopKRanker: row i -> sorted label ids of argsort(P[i], kind='stable')[-k_i:] (k_i = 0: every label)."""
    out = []
    for i in range(P.shape[0]):
        o = np.argsort(P[i], kind='stable')
        out.append(np.sort(o[-int(k[i]):] if k[i] else o))
    return out


def near_tie_rows(P, k, eps=1e-6):
    """Rows whose k-th and (k+1)-th largest probabilities lie within eps (k = 0 and k = L rows are never near ties)."""
    rows = []
    for i in range(P.shape[0]):
        ki = int(k[i])
        if 0 < ki < P.shape[1]:
            s = np.sort(P[i])[::-1]
            if s[ki - 1] - s[ki] <= eps:
                rows.append(i)
    return np.array(rows, dtype=np.int64)


def f1(Y_true, pred, L):
    """(micro F1, macro F1) of the predicted label sets `pred` (list of id arrays) against the 0/1 matrix Y_true."""
    Y_true = np.asarray(Y_true) > 0
    Yp = np.zeros_like(Y_true)
    for i, p in enumerate(pred):
        Yp[i, p] = True
    tp = (Y_true & Yp).sum(0).astype(np.float64)
    fp = (~Y_true & Yp).sum(0).astype(np.float64)
    fn = (Y_true & ~Yp).sum(0).astype(np.float64)
    den = 2 * tp + fp + fn
    micro = 2 * tp.sum() / den.sum() if den.sum() else 0.0
    per = np.where(den > 0, 2 * tp / np.maximum(den, 1), 0.0)
    return float(micro), float(per.mean())
