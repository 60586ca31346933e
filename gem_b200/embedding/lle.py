"""Locally Linear Embedding on an H100 -- drop-in for reference gem/embedding/lle.py:10-40 (SURVEY 8(f) rank 4).

Same class name, hyper-parameter (d), method name ('lle_svd'), call signature, error behaviour (ValueError('graph needed')),
row order (list(graph.nodes)), result (right singular vectors 1..d of M = I - D^-1 W for the d+1 smallest singular values of
the UNDIRECTED graph, ascending, the first one dropped -- lle.py:25-32) and get_edge_weight (:37-40).

The reference calls scipy.sparse.linalg.svds(I - P, k=d+1, which='SM').  Here: the right singular vectors of M for its smallest
singular values are the eigenvectors of C = c I - M^T M for its LARGEST eigenvalues (c = ||M||_1 ||M||_inf >= ||M||_2^2), and
those come from the Chebyshev-filtered subspace iteration of libgemb200.so (gemb_hope, opts.spectral_mode = 1) -- the same CSR SpMM,
tensor-core Gram / apply and Rayleigh-Ritz kernels HOPE and LaplacianEigenmaps run on.  First version: C is formed explicitly on the
host (scipy.sparse product P^T P, sum_v deg(v)^2 entries -- fine for bounded degrees, not for power-law hubs); applying M and M^T as
two fused sweeps inside the solver instead is the next step (DESIGN.md section 9).  No CPU path for the solve.

Extra, optional hyper-parameters: tol (default 1e-6), max_iters, oversample, cheb_degree, cheb_range_log2, seed, device, dtype, strict."""
import numpy as np

from gem_b200 import graph as _graph
from gem_b200.embedding.lap import spectral_solve, undirected_coo
from gem_b200.embedding.static_graph_embedding import StaticGraphEmbedding


def lle_operator(csr):
    """(HostCSR of C = c I - (I - P)^T (I - P), c) with P = D^-1 W (sklearn normalize(..., 'l1', axis=1): rows over the sum of
    their absolute values, zero rows stay zero), W = graph.to_undirected()."""
    import scipy.sparse as sp
    n = csr.n
    src, dst, ww = undirected_coo(csr)
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
        C, c = lle_operator(csr)
        V, lam = spectral_solve(self, C, d, 'LocallyLinearEmbedding')
        self._s = np.sqrt(np.maximum(c - np.asarray(lam, dtype=np.float64), 0.0))     # ascending singular values of I - P
        return self._result(V[:, 1:], csr.n)

    def get_edge_weight(self, i, j):
        return np.exp(
            -np.power(np.linalg.norm(self._X[i, :] - self._X[j, :]), 2)
        )
