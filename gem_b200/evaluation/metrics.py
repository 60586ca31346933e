"""Host-side finish of GEM's metrics (reference gem/evaluation/metrics.py:1-46).

The n^2 part -- ranking every candidate edge of every node -- runs on the GPU (gemb_recon_ranks / gemb_recon_top,
gem_b200/csrc/recon.cu); what is left here is O(nnz) bookkeeping in the reference's own summation order.
"""
import numpy as np

precision_pos = [2, 10, 100, 200, 300, 500, 1000]          # metrics.py:3


def map_from_ranks(n, indptr, ranks, is_undirected, out_degree=None):
    """metrics.py:28-46 given, for every true edge (CSR order), its 1-based rank among the predicted edges of its
    source node (0 = not predicted).  AP_i = (sum over hits, in rank order, of (#hits so far) / rank) / #hits;
    nodes without out-edges are skipped unless is_undirected (:38-39); MAP = sum(AP) / count, summed in node order.
    -> (MAP, node_ap, count)"""
    indptr = np.asarray(indptr, dtype=np.int64)
    ranks = np.asarray(ranks, dtype=np.int64)
    outdeg = np.diff(indptr) if out_degree is None else np.asarray(out_degree)
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(indptr))
    hit = ranks > 0
    hr, rk = rows[hit], ranks[hit]
    order = np.lexsort((rk, hr))                              # by node, then by rank
    hr, rk = hr[order], rk[order]
    hits = np.bincount(hr, minlength=n)                       # sum(delta_factors) per node
    first = np.cumsum(hits) - hits
    t = np.arange(1, hr.size + 1, dtype=np.int64) - first[hr]  # number of hits up to and including this one
    # np.bincount adds its weights one by one in input order = rank order: the reference's sequential sum()
    sums = np.bincount(hr, weights=t.astype(np.float64) / rk.astype(np.float64), minlength=n)
    node_ap = np.where(hits > 0, sums / np.maximum(hits, 1), 0.0)
    counted = np.ones(n, dtype=bool) if is_undirected else (outdeg > 0)
    count = int(counted.sum())
    total = 0.0
    for a in node_ap[counted].tolist():                       # sum(node_ap): sequential, in node order
        total += a
    return (total / count if count else float('nan')), node_ap, count


def precision_curve_from_top(i, j, w, has_edge, max_k=-1):
    """metrics.py:6-25 given the (unordered) candidates that reach the max_k-th weight: order them as the reference's
    stable descending sort of the row-major list does (weight desc, then i, then j), cut at max_k.
    -> (precision_scores, delta_factors) as python lists"""
    i = np.asarray(i, dtype=np.int64); j = np.asarray(j, dtype=np.int64); w = np.asarray(w)
    order = np.lexsort((j, i, -w.astype(np.float64)))
    if max_k >= 0:
        order = order[:max_k]
    delta = has_edge(i[order], j[order]).astype(np.float64)
    correct = np.cumsum(delta)
    prec = correct / np.arange(1, order.size + 1, dtype=np.float64)
    return prec.tolist(), delta.tolist()


def csr_has_edge(n, indptr, indices):
    """Vectorised has_edge(i, j) of an n-node CSR graph whose rows hold sorted column ids: a binary search of the
    sorted keys i * n + j."""
    keys = np.repeat(np.arange(n, dtype=np.int64), np.diff(indptr)) * n + np.asarray(indices, dtype=np.int64)

    def has_edge(i, j):
        if keys.size == 0:
            return np.zeros(np.shape(i), dtype=bool)
        q = np.asarray(i, dtype=np.int64) * n + np.asarray(j, dtype=np.int64)
        pos = np.minimum(np.searchsorted(keys, q), keys.size - 1)
        return keys[pos] == q
    return has_edge


def precision_curve(i, j, w, has_edge, max_k=-1):
    """metrics.py:6-24 on an explicit predicted-edge list (arrays i, j, w in list order): precision@1..max_k of the list
    sorted by weight (descending, stable).  -> (precision_scores, delta_factors) as python lists"""
    max_k = i.size if max_k == -1 else min(max_k, i.size)
    order = np.argsort(-np.asarray(w, dtype=np.float64), kind='stable')[:max_k]
    delta = has_edge(i[order], j[order]).astype(np.float64) if max_k else np.zeros(0)
    prec = np.cumsum(delta) / np.arange(1, max_k + 1, dtype=np.float64)
    return prec.tolist(), delta.tolist()


def node_ap_sum(node_num, i, j, w, has_edge, outdeg, is_undirected, max_k=-1):
    """metrics.py:28-46 on an explicit predicted-edge list (arrays i, j, w in list order): the average precision of
    each node's edges (list order, sorted by weight descending and stable, cut at max_k), nodes without out-edges
    skipped unless is_undirected.  -> (sum of the APs in node order, number of nodes counted); MAP = sum / count."""
    order = np.argsort(i, kind='stable')                      # node_edges[st].append(...) keeps list order per node
    i, j, w = i[order], j[order], np.asarray(w, dtype=np.float64)[order]
    starts = np.searchsorted(i, np.arange(node_num + 1))
    total = 0.0
    count = 0
    for v in range(node_num):
        if not is_undirected and outdeg[v] == 0:
            continue
        count += 1
        s, e = int(starts[v]), int(starts[v + 1])
        k = e - s if max_k == -1 else min(max_k, e - s)
        if k == 0:
            continue
        o = np.argsort(-w[s:e], kind='stable')[:k]
        delta = has_edge(i[s:e][o], j[s:e][o]).astype(np.float64)
        prec = np.cumsum(delta) / np.arange(1, k + 1, dtype=np.float64)
        sp = sd = 0.0
        for p, dl in zip(prec.tolist(), delta.tolist()):      # sum(precision_rectified), sum(delta_factors): sequential
            sp += p * dl
            sd += dl
        if sd != 0:
            total += float(sp / sd)
    return total, count


def f1_from_predictions(n_labels, true_indptr, true_indices, pred_indptr, pred_indices):
    """Micro and macro F1 over n_labels labels (sklearn.metrics.f1_score, average='micro' / 'macro') of predicted label
    sets against true ones, both as CSR rows of label ids (unique per row).  In the macro average a label with
    tp + fp + fn = 0 counts as 0.  O(sum of the row lengths).  -> (micro, macro)"""
    rows_t = np.repeat(np.arange(len(true_indptr) - 1, dtype=np.int64), np.diff(true_indptr))
    rows_p = np.repeat(np.arange(len(pred_indptr) - 1, dtype=np.int64), np.diff(pred_indptr))
    kt = rows_t * n_labels + np.asarray(true_indices, dtype=np.int64)
    kp = rows_p * n_labels + np.asarray(pred_indices, dtype=np.int64)
    hit = np.isin(kp, kt)
    lab_p = np.asarray(pred_indices, dtype=np.int64)
    tp = np.bincount(lab_p[hit], minlength=n_labels).astype(np.float64)
    fp = np.bincount(lab_p[~hit], minlength=n_labels).astype(np.float64)
    fn = np.bincount(np.asarray(true_indices, dtype=np.int64), minlength=n_labels) - tp
    den = 2.0 * tp + fp + fn
    micro = 2.0 * tp.sum() / den.sum() if den.sum() else 0.0
    per = np.where(den > 0, 2.0 * tp / np.maximum(den, 1.0), 0.0)
    return float(micro), float(per.mean())


# ---- the reference's own entry points (gem/evaluation/metrics.py:6-46), same names, arguments and results, for
# callers that already hold an explicit predicted edge list [(st, ed, w), ...].  The list sorts are NumPy stable
# argsorts (= Python's stable sorted(..., reverse=True) on the weight), the sums run in the reference's order.
def _has_edge_fn(true_digraph):
    from gem_b200.graph import HostCSR
    if isinstance(true_digraph, HostCSR):
        outdeg = np.diff(true_digraph.indptr)
        return csr_has_edge(true_digraph.n, true_digraph.indptr, true_digraph.indices), true_digraph.n, outdeg
    n = len(true_digraph.nodes)
    he = true_digraph.has_edge

    def has_edge(i, j):
        return np.fromiter((he(int(a), int(b)) for a, b in zip(np.atleast_1d(i), np.atleast_1d(j))), dtype=bool,
                           count=np.size(i))
    outdeg = np.array([true_digraph.out_degree(i) if true_digraph.has_node(i) else 0 for i in range(n)]) \
        if true_digraph.is_directed() else np.array([true_digraph.degree(i) if true_digraph.has_node(i) else 0 for i in range(n)])
    return has_edge, n, outdeg


def _edge_arrays(predicted_edge_list):
    m = len(predicted_edge_list)
    if m == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float64)
    a = np.asarray(predicted_edge_list, dtype=np.float64).reshape(m, 3)
    return a[:, 0].astype(np.int64), a[:, 1].astype(np.int64), a[:, 2]


def computePrecisionCurve(predicted_edge_list, true_digraph, max_k=-1):
    """metrics.py:6-24: precision@1..max_k of the edge list sorted by weight (descending, stable)."""
    has_edge, _, _ = _has_edge_fn(true_digraph)
    return precision_curve(*_edge_arrays(predicted_edge_list), has_edge, max_k)


def computeMAP(predicted_edge_list, true_digraph, max_k=-1, is_undirected=False):
    """metrics.py:27-46: mean over the counted nodes of the average precision of each node's predicted edges."""
    has_edge, node_num, outdeg = _has_edge_fn(true_digraph)
    total, count = node_ap_sum(node_num, *_edge_arrays(predicted_edge_list), has_edge, outdeg, is_undirected, max_k)
    return total / count
