"""Plugin API of GEM, kept verbatim in behaviour (reference gem/embedding/static_graph_embedding.py:5-83):
same constructor plumbing (class-level hyper_params dict updated by kwargs, then mirrored into
self._<key>: SURVEY F13), same getters, same error strings.  get_reconstructed_adj is the one method
whose n^2 Python loop (reference :59-64) is replaced: a subclass that declares `_recon_split` (True: split
halves, hope.py:43-44; False: dot product, node2vec.py:56-57) or `_recon_score = 'gaussian'`
(exp(-|x_i - x_j|^2), lap.py:39-42 / lle.py:37-40) gets the matrix from the GPU (gemb_recon_create /
gemb_recon_dense, fp32 arithmetic, returned as fp64 with a zero diagonal); there is no CPU path for it -- without a
GPU it raises RuntimeError."""
import warnings
from abc import ABC, abstractmethod

import numpy as np

from gem_b200 import graph as _graph


def _graph_is_empty(graph):
    """`if not graph` of the reference for every accepted input type, checked in this order: HostCSR (.n), anything with
    a .shape (scipy sparse matrices AND arrays raise TypeError from __len__), then len() (networkx graphs, tuples)."""
    if graph is None:
        return True
    if isinstance(graph, _graph.HostCSR):
        return graph.n == 0
    if hasattr(graph, 'shape'):
        return graph.shape[0] == 0
    if hasattr(graph, '__len__'):
        return len(graph) == 0
    return False


def recon_kind(model):
    """The gemb_recon_create kind of a model's get_edge_weight: 2 for `_recon_score = 'gaussian'`, 1 / 0 for
    `_recon_split` True / False, None when it declares neither (its score is evaluated entry by entry)."""
    if getattr(model, '_recon_score', None) == 'gaussian':
        return 2
    split = getattr(model, '_recon_split', None)
    if split is None:
        return None
    return 1 if split else 0


class StaticGraphEmbedding(ABC):
    """Base of the drop-in embedding classes.  Subclasses provide a class-level `hyper_params` dict (at least
    'method_name'), `learn_embedding` and `get_edge_weight`; a subclass whose score is one of the three reference
    forms declares `_recon_split` or `_recon_score` so that reconstruction and evaluation run on the GPU."""

    def __init__(self, *param_dicts, **params):
        self._method_name = self._d = self._X = None
        # SURVEY F13, kept on purpose: keyword arguments are merged into the dict shared by the CLASS (later instances
        # inherit them); every entry then becomes an attribute with a leading underscore.  Positional dicts are
        # applied last, override, and do not touch the shared dict.
        shared = self.hyper_params
        shared.update(params)
        settings = dict(shared)
        for extra in param_dicts:
            settings.update(extra)
        for name, value in settings.items():
            setattr(self, '_' + name, value)

    # -- getters (same strings and errors as the reference, :21-46)
    def get_embedding(self):
        if self._X is None:
            raise ValueError("Embedding not learned yet")
        return self._X

    def get_method_name(self):
        return self._method_name

    def get_method_summary(self):
        return '{}_{:d}'.format(self._method_name, self._d)

    # -- steps shared by the learn_embedding of the subclasses
    @staticmethod
    def _check_graph(graph):
        if _graph_is_empty(graph):
            raise ValueError('graph needed')

    def _to_csr(self, graph):
        """The input step: the empty-graph guard, then a HostCSR of a HostCSR, networkx graph or scipy.sparse matrix."""
        self._check_graph(graph)
        if isinstance(graph, _graph.HostCSR):
            return graph
        if hasattr(graph, 'nodes') and hasattr(graph, 'edges'):
            return _graph.from_networkx(graph)
        return _graph.from_scipy(graph)

    def _check_converged(self, stats, msg, stacklevel=3):
        """A solver that stopped unconverged raises RuntimeError(msg) under `strict` and warns otherwise.  stacklevel
        counts the frames from here up to the line that called learn_embedding, which the warning points at."""
        if stats['converged']:
            return
        if getattr(self, '_strict', False):
            raise RuntimeError(msg)
        warnings.warn(msg, RuntimeWarning, stacklevel=stacklevel)

    def _result(self, X, node_num):
        """The result step: X in the requested dtype (default float32, returned as it is), C-contiguous; the node count."""
        self._node_num = node_num
        dt = np.dtype(getattr(self, '_dtype', np.float32))
        self._X = X if X.dtype == dt and X.flags.c_contiguous else np.ascontiguousarray(X, dtype=dt)
        return self._X

    def get_reconstructed_adj(self, X=None, node_l=None):
        """A_hat[i, j] = get_edge_weight(i, j) off the diagonal, 0 on it (reference :48-65).  As there, a given X
        replaces the stored embedding and `node_l` is accepted but unused."""
        if X is None:
            rows = self._node_num
        else:
            self._X = X
            rows = X.shape[0]
        kind = recon_kind(self)
        if kind is None:
            # a subclass with a score function of its own: evaluate it entry by entry, like the reference
            score = self.get_edge_weight
            return np.array([[0.0 if i == j else score(i, j) for j in range(rows)] for i in range(rows)],
                            dtype=np.float64).reshape(rows, rows)
        from gem_b200 import _native
        with _native.Context(getattr(self, '_device', 0)) as ctx, \
                _native.Reconstruction(ctx, np.asarray(self._X)[:rows], kind) as rec:
            A = rec.dense().astype(np.float64)
        return np.exp(-A) if kind == _native.RECON_GAUSS else A     # delta is +inf on the diagonal: exp gives 0

    @abstractmethod
    def learn_embedding(self, graph):
        """graph: networkx DiGraph (or the CSR forms the subclass documents) -> n x d ndarray, also stored."""

    @abstractmethod
    def get_edge_weight(self, i, j):
        """Score of the edge i -> j from rows i and j of the embedding."""
