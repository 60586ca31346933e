"""Locally Linear Embedding on an H100 -- drop-in for reference gem/embedding/lle.py:10-40 (SURVEY 8(f) rank 4).

Same class name, hyper-parameter (d), method name ('lle_svd'), call signature, error behaviour (ValueError('graph needed')),
row order (list(graph.nodes)), result (right singular vectors 1..d of M = I - D^-1 W for the d+1 smallest singular values of
the UNDIRECTED graph, ascending, the first one dropped -- lle.py:25-32) and get_edge_weight (:37-40).

The reference calls scipy.sparse.linalg.svds(I - P, k=d+1, which='SM').  Here the right singular vectors of M for its smallest
singular values come from the Chebyshev-filtered subspace iteration of libgemb200.so (gemb_hope) -- the same CSR SpMM,
tensor-core Gram / apply and Rayleigh-Ritz kernels HOPE and LaplacianEigenmaps run on -- in one of two operator forms,
chosen by the `operator` hyper-parameter:
  'explicit'   the eigenvectors of C = c I - M^T M for its LARGEST eigenvalues (c = ||M||_1 ||M||_inf >= ||M||_2^2;
               spectral_mode 1).  C is formed on the host (scipy.sparse product P^T P) and uploaded: sum_v deg(v)^2
               entries, which power-law hubs make far larger than W, and more than one upload takes (2^31) on R-MAT
               scale 20.  In fp32 with c on the diagonal, C cannot resolve sigma^2 below ~6e-8 c.
  'composite'  the eigenvectors of -M^T M for its largest algebraic eigenvalues -sigma^2, never formed (spectral_mode 2):
               P and P^T are uploaded (W's pattern twice) and every application of -M^T M is two SpMM sweeps,
               T = X - P X and P^T T - T.  Unshifted, so the small sigma^2 are resolved relative to themselves.
  'auto'       (default) 'explicit' while sum_v deg(v)^2 + n <= 2^31 - 1 (deg = entries per row of W, the bound on
               C's entries), else 'composite'.
No CPU path for the solve.  model.stats['operator'] says which form ran.

Extra, optional hyper-parameters: operator, tol (default 1e-6; explicit: change of every wanted eigenvalue of C between two
Rayleigh-Ritz rounds, relative to itself and at least 1e-3 max|eigenvalue|, as in lap.py; composite: the change of every
wanted -sigma^2 relative to ||M||_2^2; stop_rule=1: the residual estimate max_j ||C v_j - l_j v_j|| / max_j |l_j|, or
max_j ||M^T M v_j - sigma_j^2 v_j|| / ||M||_2^2), max_iters, oversample, cheb_degree, cheb_range_log2, seed, device, dtype,
strict."""
import numpy as np

from gem_b200 import graph as _graph
from gem_b200.embedding.lap import spectral_solve, undirected_coo
from gem_b200.embedding.static_graph_embedding import StaticGraphEmbedding


def lle_operator(csr, coo=None):
    """(HostCSR of C = c I - (I - P)^T (I - P), c) with P = D^-1 W (sklearn normalize(..., 'l1', axis=1): rows over the sum of
    their absolute values, zero rows stay zero), W = graph.to_undirected().  coo: undirected_coo(csr), if already made."""
    import scipy.sparse as sp
    n = csr.n
    src, dst, ww = undirected_coo(csr) if coo is None else coo
    s = np.bincount(src, weights=np.abs(ww), minlength=n)
    inv = np.where(s > 0, 1.0 / np.where(s > 0, s, 1.0), 0.0)
    P = sp.csr_matrix((ww * inv[src], (src, dst)), shape=(n, n))
    M = sp.identity(n, format='csr') - P
    c = float(abs(M).sum(axis=0).max() * abs(M).sum(axis=1).max())          # ||M||_1 ||M||_inf >= ||M||_2^2
    C = (c * sp.identity(n, format='csr') - (M.T @ M)).tocsr()
    C = ((C + C.T) * 0.5).tocsr()                                            # symmetric to the last bit
    C.sort_indices()
    out = _graph.HostCSR(n, C.indptr.astype(np.int64), C.indices.astype(np.int32), C.data.astype(np.float64), nodes=csr.nodes,
                         symmetric=True)
    return out, c


def lle_composite_operator(csr, coo=None):
    """(HostCSR of P = D^-1 W, HostCSR of P^T): the same P as lle_operator's, uploaded with its transpose for the composite
    form (spectral_mode 2).  W is symmetric, so P^T has W's pattern with the values w_ij / s_j.  coo: as in lle_operator."""
    import scipy.sparse as sp
    n = csr.n
    src, dst, ww = undirected_coo(csr) if coo is None else coo
    s = np.bincount(src, weights=np.abs(ww), minlength=n)
    inv = np.where(s > 0, 1.0 / np.where(s > 0, s, 1.0), 0.0)
    pv = ww * inv[src]
    out = []
    for r, c in ((src, dst), (dst, src)):
        Q = sp.csr_matrix((pv, (r, c)), shape=(n, n))
        Q.sort_indices()
        out.append(_graph.HostCSR(n, Q.indptr.astype(np.int64), Q.indices.astype(np.int32), Q.data.astype(np.float64),
                                  nodes=csr.nodes, symmetric=False))
    return out[0], out[1]


EXPLICIT_ENTRY_LIMIT = 2 ** 31 - 1


def choose_operator(csr, operator='auto', coo=None):
    """'explicit' or 'composite' for `operator`; 'auto': explicit while sum_v deg(v)^2 + n <= 2^31 - 1, deg(v) the
    entries of row v of W = graph.to_undirected() -- the bound on the entries of C = c I - M^T M.  The degrees are counted
    on W's entries (O(nnz) given coo = undirected_coo(csr), which the chosen operator then reuses)."""
    if operator in ('explicit', 'composite'):
        return operator
    if operator != 'auto':
        raise ValueError("operator must be 'auto', 'explicit' or 'composite', not %r" % (operator,))
    src = (undirected_coo(csr) if coo is None else coo)[0]
    deg = np.bincount(src, minlength=csr.n).astype(np.int64)
    return 'explicit' if int(np.sum(deg * deg)) + csr.n <= EXPLICIT_ENTRY_LIMIT else 'composite'


class LocallyLinearEmbedding(StaticGraphEmbedding):

    _recon_score = 'gaussian'      # get_edge_weight is exp(-|x_i - x_j|^2): reconstructed and evaluated on the GPU

    hyper_params = {
        'method_name': 'lle_svd'
    }

    def __init__(self, *args, **kwargs):
        """ Initialize the LocallyLinearEmbedding class

        Args:
            d: dimension of the embedding
        """
        super(LocallyLinearEmbedding, self).__init__(*args, **kwargs)
        self.stats = None
        self._s = None

    def learn_embedding(self, graph=None, is_weighted=False, no_python=False, **ignored):
        csr = self._to_csr(graph)
        d = int(self._d)
        if d + 1 > csr.n:
            raise ValueError('d + 1 singular vectors asked of a %d-node graph' % csr.n)
        coo = undirected_coo(csr)                  # W = graph.to_undirected(), once for the rule and the operator
        operator = choose_operator(csr, getattr(self, '_operator', 'auto'), coo)
        if operator == 'explicit':
            C, c = lle_operator(csr, coo)
            V, lam = spectral_solve(self, C, d, 'LocallyLinearEmbedding')
            self._s = np.sqrt(np.maximum(c - np.asarray(lam, dtype=np.float64), 0.0))     # ascending singular values of I - P
        else:
            P, PT = lle_composite_operator(csr, coo)
            V, lam = spectral_solve(self, P, d, 'LocallyLinearEmbedding', op_t=PT)
            self._s = np.sqrt(np.maximum(-np.asarray(lam, dtype=np.float64), 0.0))       # lam = -sigma^2, descending
        self.stats['operator'] = operator
        return self._result(V[:, 1:], csr.n)

    def get_edge_weight(self, i, j):
        return np.exp(
            -np.power(np.linalg.norm(self._X[i, :] - self._X[j, :]), 2)
        )
