"""oracle/tsne_oracle.py -- fp64 NumPy restatement of the t-SNE stages of gem_b200 (sklearn 1.9's TSNE, barnes_hut,
init='pca'), the checker of tests/test_oracle_tsne.py and tests/test_gpu_tsne.py.  Dense: for n up to a few thousand.

    knn(X, k)                     exact neighbours by (d^2, index) ascending, the row itself excluded
    neighbour_mismatches(...)     rows whose neighbour sets differ other than by swaps at the k-th distance
    calibrate(d2, perplexity)     _binary_search_perplexity (fp64 on fp32 d^2)
    joint(idx, p_cond, n)         _joint_probabilities_nn: (P + P^T) / sum as a scipy CSR (fp64)
    pca_start(X)                  the PCA scores with svd_flip's signs, column 0 scaled to standard deviation 1e-4
    exact_gradient(Y, P, exag)    4 sum_j (exag p_ij - q_ij / Z) q_ij (y_i - y_j) and KL(exag P || Q), q = 1 / (1 + d^2)
    descend(Y, P, iters, ...)     _gradient_descent's update on the exact gradient
    trustworthiness(X, Y, k)      sklearn.manifold.trustworthiness, restated
"""
import numpy as np
import scipy.sparse as sp


def sqdist(A, B):
    """|a - b|^2 in fp64 (difference form)."""
    A = np.asarray(A, np.float64)
    B = np.asarray(B, np.float64)
    return ((A[:, None, :] - B[None, :, :]) ** 2).sum(-1)


def knn(X, k):
    """(idx n x k, d2 n x k): each row's k nearest other rows, ascending by (d^2, index)."""
    D = sqdist(X, X)
    n = D.shape[0]
    np.fill_diagonal(D, np.inf)
    idx = np.empty((n, k), np.int64)
    for i in range(n):
        o = np.lexsort((np.arange(n), D[i]))[:k]
        idx[i] = o
    return idx, np.take_along_axis(D, idx, 1)


def neighbour_mismatches(idx, d2, ref_idx, ref_d2, rel=1e-5):
    """Rows i whose neighbour set differs from the reference's by more than swaps at the k-th distance: every index in
    only one of the two sets must lie within rel * d2_k of the reference's k-th (largest) d^2.  Rows in any order."""
    bad = []
    for i in range(idx.shape[0]):
        a, b = set(idx[i].tolist()), set(ref_idx[i].tolist())
        if a == b:
            continue
        kth = float(np.max(ref_d2[i]))
        where = {int(j): float(v) for j, v in zip(ref_idx[i], ref_d2[i])}
        where.update({int(j): float(v) for j, v in zip(idx[i], d2[i]) if int(j) not in where})
        if not all(abs(where[j] - kth) <= rel * max(kth, 1e-30) for j in a ^ b):
            bad.append(i)
    return bad


def calibrate(d2, perplexity, steps=100):
    """The conditional P of each row: beta bisection from 1, at most 100 steps, |H - log perplexity| <= 1e-5."""
    d2 = np.asarray(d2, np.float32).astype(np.float64)
    n, k = d2.shape
    target = np.log(np.float64(np.float32(perplexity)))
    tol, floor = np.float64(np.float32(1e-5)), np.float64(np.float32(1e-8))
    P = np.zeros((n, k))
    for i in range(n):
        beta, lo, hi = 1.0, -np.inf, np.inf
        for _ in range(steps):
            p = np.exp(-d2[i] * beta)
            s = p.sum()
            if s == 0.0:
                s = floor
            p = p / s
            H = np.log(s) + beta * np.dot(d2[i], p)
            P[i] = p
            diff = H - target
            if abs(diff) <= tol:
                break
            if diff > 0:
                lo = beta
                beta = beta * 2.0 if hi == np.inf else (beta + hi) / 2.0
            else:
                hi = beta
                beta = beta / 2.0 if lo == -np.inf else (beta + lo) / 2.0
    return P


def entropy(d2, p):
    """Shannon entropy (nats) of each row's conditional distribution."""
    with np.errstate(divide='ignore', invalid='ignore'):
        return -np.sum(np.where(p > 0, p * np.log(p), 0.0), axis=1)


def joint(idx, p_cond, n):
    """(P_cond + P_cond^T) / sum as CSR, zeros dropped, column ids ascending."""
    k = idx.shape[1]
    C = sp.csr_matrix((np.asarray(p_cond, np.float64).ravel(), np.asarray(idx).ravel(), np.arange(0, n * k + 1, k)),
                      shape=(n, n))
    P = (C + C.T).tocsr()
    P.eliminate_zeros()
    P.sort_indices()
    P.data /= max(P.sum(), np.finfo(np.float64).eps)
    return P


def pca_start(X):
    """The two leading principal-component scores (svd_flip(u_based_decision=False) signs), scaled so that column 0
    has standard deviation 1e-4."""
    X = np.asarray(X, np.float64)
    Xc = X - X.mean(0)
    w, V = np.linalg.eigh(Xc.T @ Xc)
    V = V[:, ::-1][:, :2]
    if V.shape[1] < 2:
        V = np.hstack([V, np.zeros((V.shape[0], 1))])
    for q in range(2):
        a = np.argmax(np.abs(V[:, q]))
        if V[a, q] < 0:
            V[:, q] = -V[:, q]
    Y = Xc @ V
    return Y / Y[:, 0].std() * 1e-4


def exact_gradient(Y, P, exaggeration=1.0, tree_pairs=False):
    """(grad n x 2, KL) with every pair counted (sklearn's method='exact', including its factor 4).  tree_pairs: leave
    out of the repulsion (and of Z) the pairs within 1e-6 of each other on both axes, as sklearn's quadtree does (its
    leaves hold such duplicates, and a leaf that duplicates the query is skipped) -- the exact sum behind angle 0."""
    Y = np.asarray(Y, np.float64)
    Pd = exaggeration * (P.toarray() if sp.issparse(P) else np.asarray(P, np.float64))
    W = 1.0 / (1.0 + sqdist(Y, Y))
    np.fill_diagonal(W, 0.0)
    if tree_pairs:
        Y32 = np.asarray(Y, np.float32)
        dup = np.all(np.abs(Y32[:, None, :] - Y32[None, :, :]) <= np.float32(1e-6), axis=-1)
        Wr = np.where(dup, 0.0, W)
        Z = Wr.sum()
        grad = 4.0 * ((Pd * W).sum(1)[:, None] * Y - (Pd * W) @ Y - ((Wr * Wr).sum(1)[:, None] * Y - (Wr * Wr) @ Y) / Z)
        Q = W / Z
        with np.errstate(divide='ignore', invalid='ignore'):
            kl = np.sum(np.where(Pd > 0, Pd * np.log(np.maximum(Pd, 1e-300) / np.maximum(Q, 1e-300)), 0.0))
        return grad, kl
    Z = W.sum()
    Q = W / Z
    M = (Pd - Q) * W
    grad = 4.0 * (M.sum(1)[:, None] * Y - M @ Y)
    with np.errstate(divide='ignore', invalid='ignore'):
        kl = np.sum(np.where(Pd > 0, Pd * np.log(np.maximum(Pd, 1e-300) / np.maximum(Q, 1e-300)), 0.0))
    return grad, kl


def step(Y, update, gains, grad, momentum, learning_rate, min_gain=0.01):
    """One _gradient_descent update (fp64): (Y, update, gains, |gains * grad|)."""
    inc = update * grad < 0.0
    gains = np.where(inc, gains + 0.2, gains * 0.8)
    gains = np.maximum(gains, min_gain)
    g = grad * gains
    update = momentum * update - learning_rate * g
    return Y + update, update, gains, np.linalg.norm(g)


def descend(Y, P, iters, exaggeration, momentum, learning_rate, tree_pairs=False):
    """iters steps from Y (fresh update 0, gains 1) on the exact gradient; returns the positions."""
    Y = np.asarray(Y, np.float64).copy()
    update = np.zeros_like(Y)
    gains = np.ones_like(Y)
    for _ in range(iters):
        g, _ = exact_gradient(Y, P, exaggeration, tree_pairs)
        Y, update, gains, _ = step(Y, update, gains, g, momentum, learning_rate)
    return Y


def trustworthiness(X, Y, k):
    """sklearn.manifold.trustworthiness(X, Y, n_neighbors=k), restated (euclidean)."""
    n = X.shape[0]
    DX = sqdist(X, X)
    np.fill_diagonal(DX, np.inf)
    rank = np.empty((n, n), np.int64)
    order = np.argsort(DX, axis=1, kind='stable')
    rank[np.arange(n)[:, None], order] = np.arange(n)[None, :]
    DY = sqdist(Y, Y)
    np.fill_diagonal(DY, np.inf)
    nbr = np.argsort(DY, axis=1, kind='stable')[:, :k]
    r = rank[np.arange(n)[:, None], nbr] + 1 - k
    t = np.sum(r[r > 0])
    return 1.0 - t * (2.0 / (n * k * (2.0 * n - 3.0 * k - 1.0)))
