"""Graph Factorization on an H100 -- drop-in for reference gem/embedding/gf.py:12-108 (SURVEY 8(f) rank 4).

Same class name, hyper-parameters (d, eta, regu, max_iter, print_step; data_set accepted), method name ('graph_factor_sgd'),
call signature, error behaviour (ValueError('graph needed')), start (0.01 * np.random.randn(n, d) from NumPy's global RNG, gf.py:94),
update rule and edge order (gf.py:95-104; its C++ twin gem/c_src/gf.cpp:143-164), get_edge_weight (:107-108).  The SGD runs in
libgemb200.so (gemb_gf, gem_b200/csrc/gf.cu) in fp32; there is no CPU path and nothing shells out to gem/c_exe/gf.

Schedule: the reference sweeps graph.edges() sequentially.  When that order is grouped by ascending source row (any graph whose nodes
were inserted in sorted order -- every fixture of the reference), the sweep equals "all rows in parallel, partners read from the previous
epoch's table" exactly (only j > i is read, and row j > i is untouched so far in the epoch): gemb_gf mode 1, one warp per row.  Any other
order runs on one warp in the order given (mode 0) up to `sequential_limit` edge updates (default 2e7); beyond that the edges are grouped
by source (a different, equally valid SGD schedule) and a warning says so.
Node labels must be the integers 0..n-1 (the reference indexes X[i] with the label)."""
import warnings

import numpy as np

from gem_b200 import _native
from gem_b200 import graph as _graph
from gem_b200.embedding.static_graph_embedding import StaticGraphEmbedding


class GraphFactorization(StaticGraphEmbedding):

    _recon_split = False     # get_edge_weight = <X[i], X[j]>: the GPU reconstruction of the base class applies

    hyper_params = {
        'print_step': 10000,
        'method_name': 'graph_factor_sgd'
    }

    def __init__(self, *args, **kwargs):
        """ Initialize the GraphFactorization class
        Args:
            d: dimension of the embedding
            eta: learning rate of sgd
            regu: regularization coefficient of magnitude of weights
            max_iter: max iterations in sgd
            print_step: #iterations to log the prgoress (step%print_step)
        """
        super(GraphFactorization, self).__init__(*args, **kwargs)
        self.stats = None

    @staticmethod
    def _edges(graph):
        """(n, src, dst, w) in graph.edges(data='weight', default=1) order; HostCSR / scipy input: row-major order."""
        if isinstance(graph, _graph.HostCSR) or not (hasattr(graph, 'nodes') and hasattr(graph, 'edges')):
            csr = graph if isinstance(graph, _graph.HostCSR) else _graph.from_scipy(graph)
            src = np.repeat(np.arange(csr.n, dtype=np.int64), np.diff(csr.indptr).astype(np.int64))
            w = None if csr.data is None else np.asarray(csr.data, dtype=np.float32)
            return csr.n, src.astype(np.int32), csr.indices.astype(np.int32), w
        n = len(graph.nodes)
        m = graph.number_of_edges()
        e = np.fromiter((x for u, v, ww in graph.edges(data='weight', default=1) for x in (u, v, ww)), dtype=np.float64,
                        count=3 * m).reshape(m, 3)
        if m and (e[:, :2].min() < 0 or e[:, :2].max() >= n):
            raise ValueError('GraphFactorization indexes the embedding with the node label: labels must be 0..n-1')
        return n, e[:, 0].astype(np.int32), e[:, 1].astype(np.int32), e[:, 2].astype(np.float32)

    def learn_embedding(self, graph=None, is_weighted=False, no_python=True, X0=None, **ignored):
        self._check_graph(graph)
        n, src, dst, w = self._edges(graph)
        d = int(self._d)
        if X0 is None:
            X0 = 0.01 * np.random.randn(n, d)                      # gf.py:94 (NumPy's global RNG, like the reference)
        mode = 1 if (src.size < 2 or bool(np.all(src[1:] >= src[:-1]))) else 0
        if mode == 0 and float(src.size) * float(self._max_iter) > float(getattr(self, '_sequential_limit', 2e7)):
            order = np.argsort(src, kind='stable')
            src, dst = src[order], dst[order]
            w = None if w is None else w[order]
            mode = 1
            warnings.warn('GraphFactorization: graph.edges() is not grouped by source and %d x %d sequential updates exceed '
                          'sequential_limit; the edges were grouped by source row (a different SGD schedule)' % (src.size, self._max_iter),
                          RuntimeWarning, stacklevel=2)
        with _native.Context(int(getattr(self, '_device', 0))) as ctx:
            X, ms = _native.graph_factorization(ctx, n, src, dst, w, d, float(self._eta), float(self._regu), int(self._max_iter),
                                                np.asarray(X0, dtype=np.float32), mode=mode)
        self.stats = {'device_ms': ms, 'mode': mode, 'edges': int(src.size), 'epochs': int(self._max_iter)}
        return self._result(X, n)

    def get_edge_weight(self, i, j):
        return np.dot(self._X[i, :], self._X[j, :])
