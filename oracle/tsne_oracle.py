"""oracle/tsne_oracle.py -- NumPy restatement of the t-SNE stages of gem_b200 (sklearn 1.9's TSNE, barnes_hut,
init='pca'), the checker of tests/test_oracle_tsne.py, tests/test_gpu_tsne.py and tests/test_gpu_tsne_edges.py.  fp64 except where a
function restates sklearn's float32 steps (bh_gradient).  knn and sqdist work in row blocks (n d up to a few million);
the gradients are dense and the quadtree is pure Python: for n up to a few thousand.

    knn(X, k)                     exact neighbours by (d^2, index) ascending, the row itself excluded
    neighbour_mismatches(...)     rows whose neighbour sets differ other than by swaps at the k-th distance
    calibrate(d2, perplexity)     _binary_search_perplexity (fp64 on fp32 d^2)
    joint(idx, p_cond, n)         _joint_probabilities_nn: (P + P^T) / sum as a scipy CSR (fp64)
    pca_start(X)                  the PCA scores with svd_flip's signs, column 0 scaled to standard deviation 1e-4
    exact_gradient(Y, P, exag)    4 sum_j (exag p_ij - q_ij / Z) q_ij (y_i - y_j) and KL(exag P || Q), q = 1 / (1 + d^2)
    QuadTree(Y)                   _quad_tree.pyx's tree of the float32 positions, cell by cell
    bh_gradient(Y, P, angle)      _kl_divergence_bh: the Barnes-Hut gradient and KL on that tree, in sklearn's float32 steps
    descend(Y, P, iters, ...)     _gradient_descent's update on the exact gradient
    trustworthiness(X, Y, k)      sklearn.manifold.trustworthiness, restated
"""
import numpy as np
import scipy.sparse as sp


_BLOCK_ELEMS = 1 << 23     # fp64 elements of one row block's difference array (64 MB)


def _row_blocks(n, width):
    step = max(1, _BLOCK_ELEMS // max(1, width))
    for r0 in range(0, n, step):
        yield r0, min(n, r0 + step)


def sqdist(A, B):
    """|a - b|^2 in fp64 (difference form), in blocks of rows of A: every entry is the same sum over the same
    contiguous row of differences whatever the block, so the result does not depend on the blocking."""
    A = np.asarray(A, np.float64)
    B = np.asarray(B, np.float64)
    D = np.empty((A.shape[0], B.shape[0]))
    for r0, r1 in _row_blocks(A.shape[0], B.shape[0] * A.shape[1]):
        D[r0:r1] = ((A[r0:r1, None, :] - B[None, :, :]) ** 2).sum(-1)
    return D


def knn(X, k):
    """(idx n x k, d2 n x k): each row's k nearest other rows, ascending by (d^2, index).  Rows are processed in blocks,
    so n x n is never stored."""
    X = np.asarray(X, np.float64)
    n = X.shape[0]
    idx = np.empty((n, k), np.int64)
    d2 = np.empty((n, k))
    for r0, r1 in _row_blocks(n, n * X.shape[1]):
        D = sqdist(X[r0:r1], X)
        D[np.arange(r1 - r0), np.arange(r0, r1)] = np.inf
        o = np.argsort(D, axis=1, kind='stable')[:, :k]           # stable: equal d^2 by ascending index
        idx[r0:r1] = o
        d2[r0:r1] = np.take_along_axis(D, o, 1)
    return idx, d2


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
        Z = max(Wr.sum(), np.finfo(np.float64).eps)        # compute_gradient_negative's floor (all points coincident)
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


_F32 = np.float32
_EPSILON = _F32(1e-6)          # _quad_tree.pyx EPSILON


def _widen(M):
    """QuadTree.build_tree's upper bound: max(M (1 + 1e-3 sign M), M + 1e-3), as numpy evaluates it on float32 M."""
    return _F32(np.maximum(M * (1. + 1e-3 * np.sign(M)), M + 1e-3))


class QuadTree:
    """_quad_tree.pyx's _QuadTree for 2-D points, built as build_tree builds it: the root [min, widened max] in float32,
    points inserted in index order, a leaf's barycentre its first point, a point within EPSILON of it on both axes
    merged into it, any other point splitting the leaf until the two separate, and every cell's barycentre the running
    float32 mean (n b + p) / (n + 1) of the points that passed through it.  Every float operation is one numpy float32
    operation where sklearn's is one C float operation, so the cells, widths and barycentres are sklearn's bits.

    barycentre='sum': each non-leaf cell's barycentre is instead the fp64 sum of its points' coordinates divided by
    their count, rounded to float32 (a leaf's stays its first point) -- how gem_b200's tree forms them.

    Arrays (one entry per cell, cell 0 the root): bary (C x 2 float32), sqw (C float32, squared_max_width), size
    (C int64, cumulative_size), leaf (C bool), children (C x 4 int64, -1 where absent; slot 2 [x >= cx] + [y >= cy])."""

    def __init__(self, Y, barycentre='sklearn'):
        if barycentre not in ('sklearn', 'sum'):
            raise ValueError(barycentre)
        Y = np.asarray(Y, np.float32)
        lo = [_F32(v) for v in Y.min(0)]
        hi = [_F32(v) for v in _widen(Y.max(0))]
        self._lo, self._hi, self._ctr, self._bary, self._sqw = [], [], [], [], []
        self._size, self._leaf, self._pidx, self._ch, self._sum = [], [], [], [], []
        self._new(lo, hi)
        for i in range(Y.shape[0]):
            self._insert([_F32(Y[i, 0]), _F32(Y[i, 1])], i)
        if barycentre == 'sum':
            self._barycentres_from_sums(Y)
        self.bary = np.array(self._bary, np.float32).reshape(-1, 2)
        self.sqw = np.array(self._sqw, np.float32)
        self.size = np.array(self._size, np.int64)
        self.leaf = np.array(self._leaf, bool)
        self.children = np.array(self._ch, np.int64).reshape(-1, 4)

    def _new(self, lo, hi):
        ctr = [_F32((hi[a] + lo[a]) / _F32(2)) for a in range(2)]
        w = [_F32(hi[a] - lo[a]) for a in range(2)]
        sqw = _F32(0)
        for a in range(2):
            sqw = max(sqw, _F32(w[a] * w[a]))
        self._lo.append(lo); self._hi.append(hi); self._ctr.append(ctr); self._bary.append([_F32(0), _F32(0)])
        self._sqw.append(sqw); self._size.append(0); self._leaf.append(True); self._pidx.append(-1)
        self._ch.append([-1, -1, -1, -1])
        return len(self._lo) - 1

    def _slot(self, c, pt):
        return 2 * int(pt[0] >= self._ctr[c][0]) + int(pt[1] >= self._ctr[c][1])

    def _child(self, c, pt, pidx, size):
        """_insert_point_in_new_child: a new leaf under c holding pt (size points)."""
        s = self._slot(c, pt)
        lo = [self._ctr[c][a] if (s >> (1 - a)) & 1 else self._lo[c][a] for a in range(2)]
        hi = [self._hi[c][a] if (s >> (1 - a)) & 1 else self._ctr[c][a] for a in range(2)]
        k = self._new(lo, hi)
        self._leaf[c] = False
        self._pidx[c] = -1
        self._bary[k] = list(pt)
        self._pidx[k] = pidx
        self._size[k] = size
        self._ch[c][s] = k
        return k

    def _insert(self, pt, pidx):
        c = 0
        while True:
            n = self._size[c]
            if n == 0:
                self._size[c] = 1
                self._bary[c] = list(pt)
                self._pidx[c] = pidx
                return
            if not self._leaf[c]:
                fn, fn1 = _F32(n), _F32(n + 1)
                self._bary[c] = [_F32(_F32(fn * self._bary[c][a] + pt[a]) / fn1) for a in range(2)]
                self._size[c] = n + 1
                nxt = self._ch[c][self._slot(c, pt)]
                if nxt == -1:
                    self._child(c, pt, pidx, 1)
                    return
                c = nxt
                continue
            b = self._bary[c]
            if abs(_F32(pt[0] - b[0])) <= _EPSILON and abs(_F32(pt[1] - b[1])) <= _EPSILON:
                self._size[c] = n + 1
                return
            self._child(c, b, self._pidx[c], n)       # the leaf moves down, then pt is inserted again at c

    def _barycentres_from_sums(self, Y):
        """Each non-leaf cell's barycentre as (float32) (fp64 sum of its points / count)."""
        C = len(self._lo)
        pts = [[] for _ in range(C)]
        for i in range(Y.shape[0]):
            c = 0
            while True:
                pts[c].append(i)
                if self._leaf[c]:
                    break
                nxt = self._ch[c][self._slot(c, [_F32(Y[i, 0]), _F32(Y[i, 1])])]
                if nxt == -1:       # a duplicate that landed in a leaf sklearn reached through another slot
                    break
                c = nxt
        for c in range(C):
            if not self._leaf[c] and pts[c]:
                s = Y[pts[c]].astype(np.float64).sum(0)
                self._bary[c] = [_F32(s[0] / len(pts[c])), _F32(s[1] / len(pts[c]))]


def bh_summaries(tree, Y, angle):
    """compute_gradient_negative's summaries: for every query point the cells summarize() accepts, in its depth-first
    order (children in slot order).  A cell at d^2 = (y - b)_x^2 + (y - b)_y^2 (float32) is skipped when it is a leaf
    within EPSILON of the query on both axes, accepted when it is a leaf or squared_max_width / d^2 < angle^2 (float32),
    and opened otherwise.  -> (query, cell, dx, dy, d2) arrays (float32 differences), grouped by query in order."""
    Y = np.asarray(Y, np.float32)
    n = Y.shape[0]
    theta2 = _F32(_F32(angle) * _F32(angle))
    ch = tree.children
    nch = (ch >= 0).sum(1)
    packed = np.full_like(ch, -1)                      # existing children first, in slot order
    for c in range(ch.shape[0]):
        e = ch[c][ch[c] >= 0]
        packed[c, :e.size] = e
    q = np.arange(n)
    c = np.zeros(n, np.int64)
    done = np.zeros(n, bool)
    while not done.all():
        dx = Y[q, 0] - tree.bary[c, 0]
        dy = Y[q, 1] - tree.bary[c, 1]
        d2 = dx * dx + dy * dy
        leaf = tree.leaf[c]
        skip = ~done & leaf & (np.abs(dx) <= _EPSILON) & (np.abs(dy) <= _EPSILON)
        with np.errstate(divide='ignore', invalid='ignore'):
            accept = leaf | (tree.sqw[c] / d2 < theta2)
        opened = ~done & ~skip & ~accept
        reps = np.where(opened, nch[c], np.where(skip, 0, 1))
        src = np.repeat(np.arange(q.size), reps)
        start = np.cumsum(reps) - reps
        j = np.arange(src.size) - start[src]
        op = opened[src]
        q = q[src]
        c = np.where(op, packed[c[src], np.minimum(j, 3)], c[src])
        done = ~op
    dx = Y[q, 0] - tree.bary[c, 0]
    dy = Y[q, 1] - tree.bary[c, 1]
    return q, c, dx, dy, dx * dx + dy * dy


def bh_gradient(Y, P, angle, exaggeration=1.0, barycentre='sklearn', kl_float32=False):
    """(grad n x 2, KL) of _kl_divergence_bh (dof 1, including its factor 4) at positions Y (rounded to float32) for the
    joint P (CSR): _barnes_hut_tsne.pyx's gradient on the QuadTree of Y.  The float32 steps are sklearn's: the summary
    d^2, q = 1 / (1 + d^2), mult = (float32) (size q^2), the repulsive force summed in float32 in the walk's order, the
    attractive force pij q (y_i - y_j) summed in float32 in CSR order with pij = (float32) (exaggeration P), and the
    gradient (float32) (pos - neg / sum_Q) times 4.  sum_Q is summed in fp64, and so is the KL unless kl_float32, which
    adds its terms one by one into a float32 total in CSR order as sklearn does.  barycentre: see QuadTree."""
    Y = np.asarray(Y, np.float32)
    n = Y.shape[0]
    tree = QuadTree(Y, barycentre)
    q, c, dx, dy, d2 = bh_summaries(tree, Y, angle)
    qz = (_F32(1) / (_F32(1) + d2)).astype(np.float64)
    size = tree.size[c].astype(np.float32).astype(np.float64)
    sum_q = max(float(np.sum(size * qz)), float(_F32(np.finfo(np.float64).eps)))
    mult = (size * qz * qz).astype(np.float32)
    neg = np.zeros((n, 2), np.float32)
    np.add.at(neg[:, 0], q, mult * dx)
    np.add.at(neg[:, 1], q, mult * dy)
    P = sp.csr_matrix(P)
    rows = np.repeat(np.arange(n), np.diff(P.indptr))
    pij = (exaggeration * P.data).astype(np.float32)
    b = Y[rows] - Y[P.indices]
    dij = b[:, 0] * b[:, 0] + b[:, 1] * b[:, 1]
    qij = _F32(1) / (_F32(1) + dij)
    w = pij * qij
    pos = np.zeros((n, 2), np.float32)
    np.add.at(pos[:, 0], rows, w * b[:, 0])
    np.add.at(pos[:, 1], rows, w * b[:, 1])
    qn = (qij.astype(np.float64) / sum_q).astype(np.float32)
    tiny = np.finfo(np.float32).tiny
    terms = pij.astype(np.float64) * np.log((np.maximum(pij, tiny) / np.maximum(qn, tiny)).astype(np.float64))
    if kl_float32:
        kl = _F32(0)
        for t in terms.tolist():
            kl = _F32(float(kl) + t)
        kl = float(kl)
    else:
        kl = float(np.sum(terms))
    grad = (pos.astype(np.float64) - neg.astype(np.float64) / sum_q).astype(np.float32) * _F32(4)
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
