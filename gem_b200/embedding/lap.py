"""Laplacian Eigenmaps on an H100 -- drop-in for reference gem/embedding/lap.py:8-42 (SURVEY 8(f) rank 4).

Same class name, hyper-parameter (d), method name ('lap_eigmap_svd'), call signature, error behaviour
(ValueError('graph needed')), row order (list(graph.nodes)), result (eigenvectors 1..d of the normalised Laplacian of the
UNDIRECTED graph, ascending eigenvalue, the first one dropped -- lap.py:25-32), printed diagnostic (:34-36) and
get_edge_weight (:39-42).  The reference calls scipy.sparse.linalg.eigs(l_sym, k=d+1, which='SM'); here the same
eigenvectors come from the d+1 LARGEST algebraic eigenpairs of A_hat = D^-1/2 W D^-1/2 (L_sym = I - A_hat on the vertices
that have edges), computed by the Chebyshev-filtered subspace iteration of libgemb200.so (gemb_hope with
opts.spectral_mode = 1: the CSR SpMM, tensor-core Gram / apply and Rayleigh-Ritz kernels HOPE uses) -- no shift-invert, no CPU path.

Extra, optional hyper-parameters: tol (default 1e-6: relative change of every wanted eigenvalue between two Rayleigh-Ritz rounds;
stop_rule=1 switches to the residual estimate, which fp32 Gram matrices cannot certify below ~3e-4), max_iters, oversample,
cheb_degree, cheb_range_log2, seed, device, dtype, strict, verbose.
`graph` may also be a scipy.sparse matrix or a gem_b200.graph.HostCSR (rows = 0..n-1)."""
import numpy as np

from gem_b200 import _native
from gem_b200 import graph as _graph
from gem_b200.embedding.static_graph_embedding import StaticGraphEmbedding

_OPT_KEYS = ('tol', 'max_iters', 'min_iters', 'oversample', 'seed', 'verbose', 'cheb_degree', 'cheb_range_log2', 'stop_rule')


def undirected_coo(csr):
    """graph.to_undirected() (lap.py:25, lle.py:25) on the adjacency matrix, as symmetric COO (src, dst, weight) with every
    off-diagonal pair in both directions and the self loops once.  The pair {u, v} exists when either direction does; when
    both do, networkx copies the nodes in order and, for each, its out-edges, so the edge out of the LATER node is written
    last and wins: W[u, v] = A[max, min] if present, else A[min, max]."""
    n = csr.n
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(csr.indptr).astype(np.int64))
    cols = csr.indices.astype(np.int64)
    w = np.ones(cols.shape[0]) if csr.data is None else np.asarray(csr.data, dtype=np.float64)
    off = rows != cols
    lo, hi = np.minimum(rows[off], cols[off]), np.maximum(rows[off], cols[off])
    lower = rows[off] > cols[off]
    pair = lo * np.int64(n) + hi
    order = np.lexsort((~lower, pair))                       # per pair: the (later -> earlier) entry first
    pair_s = pair[order]
    first = np.ones(pair_s.shape[0], dtype=bool)
    first[1:] = pair_s[1:] != pair_s[:-1]
    sel = order[first]
    pl, ph, pw = lo[sel], hi[sel], w[off][sel]
    dr, dw = rows[~off], w[~off]                             # self loops stay as they are
    return np.concatenate((pl, ph, dr)), np.concatenate((ph, pl, dr)), np.concatenate((pw, pw, dw))


def undirected_normalised(csr):
    """(HostCSR of A_hat' = D^-1/2 W D^-1/2 + [isolated vertices: 1 on the diagonal], ||L_sym||_F^2), W = undirected_coo.
    D = row sums of W, 1/sqrt(0) -> 0 (nx.normalized_laplacian_matrix).  An isolated vertex has a zero row in L_sym
    (eigenvalue 0, eigenvector e_i); a unit self loop in A_hat' gives it the matching eigenvalue 1."""
    n = csr.n
    src, dst, ww = undirected_coo(csr)
    deg = np.bincount(src, weights=ww, minlength=n)
    with np.errstate(divide='ignore'):
        dh = 1.0 / np.sqrt(deg)
    dh[~np.isfinite(dh)] = 0.0
    ah = ww * dh[src] * dh[dst]
    iso = np.flatnonzero(deg == 0)
    # ||L_sym||_F^2 = sum_i (1[deg_i > 0] - A_hat_ii)^2 + sum_{i != j} A_hat_ij^2
    dm = src == dst
    diag_hat = np.bincount(src[dm], weights=ah[dm], minlength=n) if dm.any() else np.zeros(n)
    l_fro2 = float(np.sum(((deg > 0).astype(np.float64) - diag_hat) ** 2) + np.sum(ah[~dm] ** 2))
    src = np.concatenate((src, iso)); dst = np.concatenate((dst, iso)); ah = np.concatenate((ah, np.ones(iso.shape[0])))
    out = _graph.from_edges(n, src, dst, ah, nodes=csr.nodes, unit_if_all_ones=False)
    out.symmetric = True
    return out, l_fro2


def spectral_solve(model, op, d, name):
    """(V, lam): the d + 1 largest algebraic eigenpairs of the symmetric HostCSR `op` by the Chebyshev-filtered subspace
    iteration of gemb_hope (spectral_mode = 1), with the model's solver options; sets model.stats and warns (raises
    under strict) when the solver stopped unconverged."""
    opts = {k: getattr(model, '_' + k) for k in _OPT_KEYS if hasattr(model, '_' + k)}
    opts.setdefault('tol', 1e-6)
    opts.setdefault('max_iters', 300)
    with _native.Context(int(getattr(model, '_device', 0))) as ctx, \
            _native.DeviceGraph(ctx, op.n, op.indptr, op.indices, op.data_f32()) as g:
        V, lam, st = g.hope(d + 1, 0.0, spectral_mode=1, **opts)
    model.stats = st
    model._check_converged(st, '%s: the solver stopped at max_iters=%d without meeting tol=%g (eigenvalues still moving '
                           'by %.3g per round)' % (name, st['iters'], opts['tol'], st['ritz_change']), stacklevel=4)
    return V, lam


class LaplacianEigenmaps(StaticGraphEmbedding):

    _recon_score = 'gaussian'      # get_edge_weight is exp(-|x_i - x_j|^2): reconstructed and evaluated on the GPU

    hyper_params = {
        'method_name': 'lap_eigmap_svd'
    }

    def __init__(self, *args, **kwargs):
        """ Initialize the LaplacianEigenmaps class

        Args:
            d: dimension of the embedding
        """
        super(LaplacianEigenmaps, self).__init__(*args, **kwargs)
        self.stats = None
        self._w = None

    def learn_embedding(self, graph=None, is_weighted=False, no_python=False, **ignored):
        csr = self._to_csr(graph)
        d = int(self._d)
        if d + 1 > csr.n:
            raise ValueError('d + 1 eigenvectors asked of a %d-node graph' % csr.n)
        ahat, l_fro2 = undirected_normalised(csr)
        V, lam = spectral_solve(self, ahat, d, 'LaplacianEigenmaps')
        w = 1.0 - np.asarray(lam, dtype=np.float64)              # ascending eigenvalues of L_sym (lap.py:29-31)
        self._w = w
        self._result(V[:, 1:], csr.n)
        # lap.py:34-36: || V diag(w) V^T - L_sym ||_F; with orthonormal eigenvectors that is sqrt(||L_sym||_F^2 - sum w_i^2)
        eig_err = float(np.sqrt(max(l_fro2 - float(np.sum(w * w)), 0.0)))
        self._eig_err = eig_err
        print('Laplacian matrix recon. error (low rank): %f' % eig_err)
        return self._X

    def get_edge_weight(self, i, j):
        return np.exp(
            -np.power(np.linalg.norm(self._X[i, :] - self._X[j, :]), 2)
        )
