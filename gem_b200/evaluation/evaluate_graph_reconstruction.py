"""evaluateStaticGraphReconstruction on an H100 -- drop-in for reference
gem/evaluation/evaluate_graph_reconstruction.py:8-46 (same arguments, same return tuple).

The reference materialises the n x n reconstruction with n^2 Python calls (static_graph_embedding.py:59-64),
scans it into an edge list (evaluation_util.py:20-36) and sorts that list once globally and once per node
(metrics.py:6-46).  Here the matrix lives on the device only (gemb_recon_create), the per-node ranking is a counting
kernel (gemb_recon_ranks), the global precision curve a threshold selection (gemb_recon_top), and the weighted error
a gather of the true edges (gemb_recon_pairs).  No CPU fallback: without a GPU this raises RuntimeError.

The score function is the model's get_edge_weight: split halves for HOPE (hope.py:43-44), plain dot product for
node2vec (node2vec.py:56-57), exp(-|x_i - x_j|^2) for LaplacianEigenmaps and LocallyLinearEmbedding (lap.py:39-42,
lle.py:37-40); a model says which through its `_recon_split` or `_recon_score` attribute.  For the Gaussian score the
device returns delta = |x_i - x_j|^2 and the order is delta ascending (stable), which is the reference's descending
score order; the weighted error uses exp(-delta) in fp64.
`max_k` (extra, optional): length of the precision curve to return; the reference always returns all
n_pred entries (max_k = -1, default here too).  When the reconstruction does not fit in device memory it is
regenerated block by block (gemb_recon_create); the full curve is then every positive entry of a matrix too large for
the device, so max_k < 0 raises ValueError before any pass over it.
"""
import numpy as np

from gem_b200 import _native
from gem_b200.embedding.static_graph_embedding import recon_kind
from gem_b200.evaluation import metrics


def _true_csr(digraph, node_num):
    """CSR of the true graph by node ID (the reference calls digraph.has_edge(i, j) with matrix positions).
    A gem_b200.graph.HostCSR is taken as it is (rows = node ids), so that graphs too large for networkx can be
    evaluated."""
    from gem_b200.graph import HostCSR
    if isinstance(digraph, HostCSR):
        return np.asarray(digraph.indptr, dtype=np.int64), np.asarray(digraph.indices, dtype=np.int64)
    e = np.array([(int(u), int(v)) for u, v in digraph.edges()], dtype=np.int64).reshape(-1, 2)
    if e.size and (e.min() < 0 or e.max() >= node_num):
        raise ValueError('node ids must be 0..n-1 (the reference indexes the reconstruction by node id)')
    if e.size and not digraph.is_directed():
        # an nx.Graph lists every edge once, in one direction, but has_edge(i, j) (metrics.py:17) is true both ways
        e = np.concatenate((e, e[e[:, 0] != e[:, 1]][:, ::-1]))
    if e.size:
        e = np.unique(e, axis=0)                       # rows sorted by (src, dst); MultiGraph duplicates dropped
    order = np.lexsort((e[:, 1], e[:, 0]))
    e = e[order]
    indptr = np.zeros(node_num + 1, dtype=np.int64)
    np.add.at(indptr, e[:, 0] + 1, 1)
    return np.cumsum(indptr), e[:, 1].copy()


def check_max_k(rec, max_k):
    """ValueError when the whole precision curve (max_k < 0) is asked of a reconstruction regenerated in blocks.
    Stand-ins for the handle without `blocks` hold their matrix whole."""
    blocks = getattr(rec, 'blocks', 1)
    if max_k < 0 and blocks > 1:
        raise ValueError('max_k = %d asks for every predicted edge of a %d x %d reconstruction that does not fit in '
                         'device memory (regenerated in %d blocks); pass max_k >= 0' % (max_k, rec.n, rec.n, blocks))


def evaluateStaticGraphReconstruction(digraph, graph_embedding, X_stat, node_l=None, file_suffix=None,
                                      sample_ratio_e=None, is_undirected=True, is_weighted=False, max_k=-1,
                                      device=None):
    from gem_b200.graph import HostCSR
    node_num = digraph.n if isinstance(digraph, HostCSR) else len(digraph.nodes)
    kind = recon_kind(graph_embedding)
    if kind is None:
        raise TypeError("%s declares neither _recon_split (True: hope.py:43-44, False: node2vec.py:56-57) nor "
                        "_recon_score ('gaussian': lap.py:39-42)" % type(graph_embedding).__name__)
    gauss = kind == _native.RECON_GAUSS
    if X_stat is not None:
        graph_embedding._X = X_stat                   # get_reconstructed_adj(X) does this (static_graph_embedding.py:56)
    X = graph_embedding.get_embedding()
    if X.shape[0] != node_num:
        raise ValueError('embedding has %d rows, graph has %d nodes' % (X.shape[0], node_num))
    indptr, indices = _true_csr(digraph, node_num)
    has_edge = metrics.csr_has_edge(node_num, indptr, indices)
    dev = device if device is not None else getattr(graph_embedding, '_device', 0)
    with _native.Context(dev) as ctx, _native.Reconstruction(ctx, X, kind) as rec:
        if sample_ratio_e:
            # evaluation_util.py:5-18 + :25-28: random pairs, kept when A_hat >= 0
            from gem_b200.utils import evaluation_util
            pairs = np.array(evaluation_util.get_random_edge_pairs(node_num, sample_ratio_e, is_undirected),
                             dtype=np.int64).reshape(-1, 2)
            w = rec.pairs(pairs[:, 0], pairs[:, 1])
            if gauss:
                # exp(-delta) >= 0 keeps every pair; ordering by -delta (exact) is ordering by the score
                keep = np.ones(w.shape, dtype=bool)
                w = -w
            else:
                keep = w >= 0.0
            pi, pj, pw = pairs[keep, 0], pairs[keep, 1], w[keep]
            total, count = metrics.node_ap_sum(node_num, pi, pj, pw, has_edge, np.diff(indptr), is_undirected)
            MAP = total / count if count else float('nan')
            prec_curv, _ = metrics.precision_curve(pi, pj, pw, has_edge)
        else:
            check_max_k(rec, max_k)
            ranks, _ = rec.ranks(indptr, indices, is_undirected)
            MAP, _, _ = metrics.map_from_ranks(node_num, indptr, ranks, is_undirected)
            ti, tj, tw = rec.top(is_undirected, max_k)
            if gauss:
                tw = -tw                              # delta ascending = -delta descending
            prec_curv, _ = metrics.precision_curve_from_top(ti, tj, tw, has_edge, max_k)
        if is_weighted:
            # :37-40 -- nx.to_numpy_matrix(digraph) has rows/columns in list(digraph.nodes) order while the
            # reconstruction is indexed by node id; edge (u -> v) is therefore compared with A_hat[pos u][pos v]
            if isinstance(digraph, HostCSR):                  # rows already in id order
                pos = np.arange(node_num, dtype=np.int64)
                eu = np.repeat(np.arange(node_num, dtype=np.int64), np.diff(indptr))
                ev = indices
                a = np.ones(ev.size) if digraph.data is None else np.asarray(digraph.data, dtype=np.float64)
            else:
                pos = np.empty(node_num, dtype=np.int64)
                pos[np.array([int(u) for u in digraph.nodes], dtype=np.int64)] = np.arange(node_num)
                ed = [(int(u), int(v), float(wt)) for u, v, wt in digraph.edges(data='weight', default=1)]
                if not digraph.is_directed():             # nx.to_numpy_matrix of an nx.Graph is symmetric
                    ed = ed + [(v, u, wt) for u, v, wt in ed if u != v]
                eu = np.array([t[0] for t in ed], dtype=np.int64)
                ev = np.array([t[1] for t in ed], dtype=np.int64)
                a = np.array([t[2] for t in ed], dtype=np.float64)
            est = rec.pairs(pos[eu], pos[ev]).astype(np.float64)
            if gauss:
                est = np.exp(-est)
            nz = a != 0
            err = float(np.sqrt(np.sum((a[nz] - est[nz]) ** 2)))
            err_baseline = float(np.sqrt(np.sum(a ** 2)))
        else:
            err = None
            err_baseline = None
    return MAP, prec_curv, err, err_baseline
