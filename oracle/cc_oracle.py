"""oracle/cc_oracle.py -- TEST INFRASTRUCTURE ONLY (not shipped, never imported by gem_b200/).

CPU restatement of get_lcc (graph_util.py:29-34) and of link prediction with upstream GEM's largest-component step:

    labels()       scipy.sparse.csgraph.connected_components(connection='weak'), renumbered so that component c is
                   the c-th in the order of the components' smallest members (networkx's yield order over row order)
    lcc_label()    the largest component; on a tie the one with the smallest member (max(..., key=len) keeps the
                   first maximal component networkx yields)
    lcc_csr()      the LCC's CSR: new id = rank of the old id among the LCC's rows, every edge of a kept row kept
    split_lcc()    the split of linkpred_oracle.split, then the training graph cut to its largest component and the
                   test graph induced on the same nodes with the same relabelling (nothing changes when the training
                   graph is one component)
Pinned: yes -- tests/test_oracle_cc.py compares with goldens made by networkx (tests/golden/make_golden_cc.py).
"""
import numpy as np

import eval_gauss_oracle as go
import eval_oracle as eo
import linkpred_oracle as lo


def labels(n, indptr, indices):
    """Component number of every row, 0..k-1 in the order of each component's smallest row."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    if n == 0:
        return np.zeros(0, dtype=np.int32)
    indptr = np.asarray(indptr, dtype=np.int64)
    nnz = int(indptr[-1])
    A = sp.csr_matrix((np.ones(nnz, dtype=np.int8), np.asarray(indices[:nnz], dtype=np.int64), indptr), shape=(n, n))
    k, lab = connected_components(A, directed=True, connection='weak')
    _, first = np.unique(lab, return_index=True)           # smallest row of every scipy component
    rank = np.empty(k, dtype=np.int64)
    rank[np.argsort(first, kind='stable')] = np.arange(k)
    return rank[lab].astype(np.int32)


def lcc_label(lab):
    """The largest component's number (the first maximal size: the smallest member wins a tie); -1 when empty."""
    return int(np.argmax(np.bincount(lab))) if lab.size else -1


def lcc_csr(n, indptr, indices, data, lab):
    """-> (node_l int64, indptr int64, indices int32, data or None) of the largest component."""
    c = lcc_label(lab)
    indptr = np.asarray(indptr, dtype=np.int64)
    keep = lab == c
    node_l = np.flatnonzero(keep).astype(np.int64)
    new = np.full(n, -1, dtype=np.int64)
    new[node_l] = np.arange(node_l.size)
    ip = np.zeros(node_l.size + 1, dtype=np.int64)
    np.cumsum(np.diff(indptr)[node_l], out=ip[1:])
    emask = np.repeat(keep, np.diff(indptr))
    nnz = int(indptr[-1])
    ix = new[np.asarray(indices[:nnz], dtype=np.int64)[emask]]
    assert ix.size == 0 or ix.min() >= 0                   # a weak component holds every edge of its rows
    w = None if data is None else np.asarray(data[:nnz], dtype=np.float64)[emask]
    return node_l, ip, ix.astype(np.int32), w


def csr_of_edges(n, src, dst):
    """Row-major CSR (columns sorted, duplicates kept) of edge arrays."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    order = np.lexsort((dst, src))
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=indptr[1:])
    return indptr, dst[order].astype(np.int32)


def split_lcc(src, dst, nodes, train_ratio, is_undirected, rng):
    """Edges in the graph's edge order, src / dst node labels, nodes = the node labels in the graph's node order.
    -> (train mask, test mask, new id of every edge end of train / test: (tu, tv, eu, ev), map label -> new id)
    where train / test masks select the kept edges in edge order."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    nodes = np.asarray(nodes, dtype=np.int64)
    n = nodes.size
    pos = np.full(int(max(nodes.max(), src.max(initial=0), dst.max(initial=0))) + 1, -1, dtype=np.int64)
    pos[nodes] = np.arange(n)
    tr, te = lo.split(src, dst, train_ratio, is_undirected, rng)
    ps, pd = pos[src], pos[dst]
    lab = labels(n, *csr_of_edges(n, ps[tr], pd[tr]))
    if lab.size and lab.max() > 0:
        keep = lab == lcc_label(lab)
    else:
        keep = np.ones(n, dtype=bool)
    new = np.full(n, -1, dtype=np.int64)
    new[keep] = np.arange(int(keep.sum()))
    tr &= (new[ps] >= 0) & (new[pd] >= 0)
    te &= (new[ps] >= 0) & (new[pd] >= 0)
    node_map = {int(nodes[i]): int(new[i]) for i in np.flatnonzero(keep)}
    return tr, te, (new[ps[tr]], new[pd[tr]], new[ps[te]], new[pd[te]]), node_map


def linkpred_lcc(src, dst, nodes, X, score, seed, train_ratio, is_undirected, n_sample=None):
    """Link prediction with the LCC step, the model's embedding given (X: k x d, rows = new ids).
    -> dict(MAP, prec_curve, n_pred, train mask, test mask, node_map, node_l)"""
    rng = np.random.RandomState(seed)
    tr, te, (tu, tv, eu, ev), node_map = split_lcc(src, dst, nodes, train_ratio, is_undirected, rng)
    k = len(node_map)
    node_l = rng.choice(k, n_sample, replace=False) if n_sample and k > n_sample else np.arange(k)
    s = len(node_l)
    _, utr, vtr = lo.induce(tu, tv, k, node_l)
    _, ute, vte = lo.induce(eu, ev, k, node_l)
    Xs = np.asarray(X)[node_l]
    adj = go.reconstruct_gaussian(Xs) if score == 'gaussian' else eo.reconstruct(Xs, score == 'split')
    r = lo.evaluate(adj, lo.edge_set(s, ute, vte), lo.edge_set(s, utr, vtr), is_undirected=is_undirected)
    r.update(train=tr, test=te, node_map=node_map, node_l=node_l)
    return r
