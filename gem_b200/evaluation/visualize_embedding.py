"""plot_embedding2D on an H100: the reference's plot (gem/evaluation/visualize_embedding.py:7-31) with its
TSNE(n_components=2).fit_transform(node_pos) reduction run on the GPU by tsne().

tsne() restates sklearn 1.9's TSNE with its defaults (init='pca', method='barnes_hut', metric='euclidean') stage by
stage -- exact kNN, perplexity calibration, symmetrised P, PCA start, Barnes-Hut gradient on sklearn's quadtree cells,
and sklearn's gradient descent -- in gem_b200/csrc/tsne.cu (gemb_tsne in include/gemb200.h).  Results are deterministic
to the bit on one device.  No CPU fallback: without a GPU it raises RuntimeError.  Neither sklearn nor matplotlib is
imported here; matplotlib only inside plot_embedding2D, where the reference needs it.
"""
import numbers
import time

import numpy as np

from gem_b200 import _native


def _positive(name, v):
    if not isinstance(v, numbers.Real) or not np.isfinite(v) or v <= 0:
        raise ValueError('%s must be a positive number, got %r' % (name, v))
    return float(v)


def tsne(X, perplexity=30.0, early_exaggeration=12.0, learning_rate='auto', max_iter=1000, n_iter_without_progress=300,
         min_grad_norm=1e-7, angle=0.5, device=None, stats=None):
    """The n x 2 float32 t-SNE positions of the rows of X (sklearn's TSNE(n_components=2).fit_transform(X) with the
    same parameters).  learning_rate 'auto' is sklearn's max(n / early_exaggeration / 4, 50).  X has at most 1024
    columns (the width of the PCA start's eigensolver).
    stats: an optional dict, filled with kl_divergence, n_iter, learning_rate, n_neighbors, nnz_P and the host-clock
    milliseconds of every stage (knn_ms, calib_ms, sym_ms, pca_ms, opt_ms, total_ms; tree_ms and grad_ms are the
    device time of the quadtree builds and of the gradient steps, summed over the iterations) and of the whole call
    (wall_ms).  Every ValueError comes before any device call."""
    X = np.asarray(X)
    if X.ndim != 2 or X.shape[0] < 2 or X.shape[1] < 1:
        raise ValueError('X must be an n x d matrix with n >= 2 and d >= 1, got shape %s' % (X.shape,))
    if not np.issubdtype(X.dtype, np.number) or not np.all(np.isfinite(X)):
        raise ValueError('X must be finite')
    if X.shape[1] > 1024:
        raise ValueError('X has %d columns; the Jacobi eigensolver of the PCA start takes at most 1024' % X.shape[1])
    n = X.shape[0]
    perplexity = _positive('perplexity', perplexity)
    if perplexity >= n:
        raise ValueError('perplexity (%g) must be less than n_samples (%d)' % (perplexity, n))
    early_exaggeration = _positive('early_exaggeration', early_exaggeration)
    if isinstance(learning_rate, str):
        if learning_rate != 'auto':
            raise ValueError("learning_rate must be 'auto' or a positive number, got %r" % learning_rate)
        learning_rate = max(n / early_exaggeration / 4, 50.0)
    learning_rate = _positive('learning_rate', learning_rate)
    if not isinstance(max_iter, numbers.Integral) or max_iter < 250:
        raise ValueError('max_iter must be an integer >= 250, got %r' % (max_iter,))
    if not isinstance(n_iter_without_progress, numbers.Integral) or n_iter_without_progress < -1:
        raise ValueError('n_iter_without_progress must be an integer >= -1, got %r' % (n_iter_without_progress,))
    if not isinstance(min_grad_norm, numbers.Real) or not min_grad_norm >= 0:
        raise ValueError('min_grad_norm must be >= 0, got %r' % (min_grad_norm,))
    if not isinstance(angle, numbers.Real) or not 0.0 <= angle <= 1.0:
        raise ValueError('angle must be in [0, 1], got %r' % (angle,))
    t0 = time.perf_counter()
    with _native.Context(0 if device is None else int(device)) as ctx:
        Y, st = _native.tsne(ctx, X, perplexity, early_exaggeration, learning_rate, int(max_iter),
                             max(int(n_iter_without_progress), 0), float(min_grad_norm), float(angle))
    if stats is not None:
        stats.update(st)
        stats['learning_rate'] = learning_rate
        stats['wall_ms'] = (time.perf_counter() - t0) * 1e3
    return Y


def plot_embedding2D(node_pos, node_colors=None, di_graph=None, labels=None):
    """The reference's plot: a scatter of the 2-D positions, or a networkx drawing of di_graph at them.  An embedding
    wider than 2 is reduced by tsne() first."""
    try:
        import matplotlib.pyplot as plt
    except ImportError as e:
        raise ImportError('plot_embedding2D needs matplotlib (pip install matplotlib)') from e
    import networkx as nx
    node_num, embedding_dimension = node_pos.shape
    if embedding_dimension > 2:
        print("Embedding dimension greater than 2, use tSNE to reduce it to 2")
        node_pos = tsne(node_pos)

    if di_graph is None:
        plt.scatter(node_pos[:, 0], node_pos[:, 1], c=node_colors)
        return
    pos = {i: node_pos[i, :] for i in range(node_num)}
    style = dict(width=0.1, arrows=False, alpha=0.8, labels=labels)
    if node_colors is None:
        nx.draw_networkx(di_graph, pos, node_color=None, node_size=300, font_size=12, **style)
    else:
        nx.draw_networkx_nodes(di_graph, pos, node_color=node_colors, node_size=100, font_size=5, **style)
