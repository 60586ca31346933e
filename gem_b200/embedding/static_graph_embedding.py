"""Plugin API of GEM, kept verbatim in behaviour (reference gem/embedding/static_graph_embedding.py:5-83):
same constructor plumbing (class-level hyper_params dict updated by kwargs, then mirrored into
self._<key>: SURVEY F13), same getters, same error strings.  get_reconstructed_adj is the one method
whose n^2 Python loop (reference :59-64) is replaced: a subclass that declares `_recon_split` (True: split
halves, hope.py:43-44; False: dot product, node2vec.py:56-57) or `_recon_score = 'gaussian'`
(exp(-|x_i - x_j|^2), lap.py:39-42 / lle.py:37-40) gets the matrix from the GPU (gemb_recon_create /
gemb_recon_dense, fp32 arithmetic, returned as fp64 with a zero diagonal); there is no CPU path for it -- without a
GPU it raises RuntimeError."""
from abc import ABC, abstractmethod

import numpy as np


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
        ctx = _native.Context(getattr(self, '_device', 0))
        try:
            rec = _native.Reconstruction(ctx, np.asarray(self._X)[:rows], kind)
            try:
                if kind == _native.RECON_GAUSS:
                    return np.exp(-rec.dense().astype(np.float64))     # delta is +inf on the diagonal: exp gives 0
                return rec.dense().astype(np.float64)
            finally:
                rec.free()
        finally:
            ctx.close()

    @abstractmethod
    def learn_embedding(self, graph):
        """graph: networkx DiGraph (or the CSR forms the subclass documents) -> n x d ndarray, also stored."""

    @abstractmethod
    def get_edge_weight(self, i, j):
        """Score of the edge i -> j from rows i and j of the embedding."""
