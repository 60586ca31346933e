"""oracle/linkpred_oracle.py -- TEST INFRASTRUCTURE ONLY (not shipped, never imported by gem_b200/).

CPU restatement of link prediction built from the reference's functions plus one filter:

    split()        evaluation_util.py:39-53  split_di_graph_to_train_test (one uniform() per edge in edge order;
                                             under is_undirected only st < ed draws, both directions move together)
    sample()       graph_util.py:42-58       sample_graph (node_l = choice(n, s, replace=False), induced graph
                                             relabelled by position in node_l)
    filtered()     [e for e in pred if not train.has_edge(e[0], e[1])]
    evaluate()     computeMAP(filtered, test) (is_undirected=False) and computePrecisionCurve(filtered, test),
                   metrics.py:6-46, through eval_oracle.py

Graphs are edge arrays (src, dst, w) in the networkx graph's edge order; a split or a sample keeps that order, as the
reference's graph copies and its sampled graph do.  *_loops follow the reference statement by statement (small
inputs); the vectorised forms must equal them (tests/test_oracle_linkpred.py).
Pinned: yes -- tests/test_oracle_linkpred.py compares with goldens made by the reference's own functions
(tests/golden/make_golden_linkpred.py -> linkpred_*.npz).
"""
import numpy as np

import eval_oracle as eo


# ------------------------------------------------------------------------------------------- split
def split_loops(edges, train_ratio, is_undirected, rng):
    """edges: [(st, ed, w), ...] in edge order.  -> (train edges, test edges), lists in edge order."""
    present = {(st, ed) for st, ed, _ in edges}
    in_train = {(st, ed): True for st, ed, _ in edges}
    in_test = {(st, ed): True for st, ed, _ in edges}
    for (st, ed, w) in edges:
        if is_undirected and st >= ed:
            continue
        if rng.uniform() <= train_ratio:
            in_test[(st, ed)] = False
            if is_undirected:
                if (ed, st) not in present:
                    raise KeyError((ed, st))
                in_test[(ed, st)] = False
        else:
            in_train[(st, ed)] = False
            if is_undirected:
                if (ed, st) not in present:
                    raise KeyError((ed, st))
                in_train[(ed, st)] = False
    return ([e for e in edges if in_train[(e[0], e[1])]], [e for e in edges if in_test[(e[0], e[1])]])


def split(src, dst, train_ratio, is_undirected, rng):
    """Vectorised split of edge arrays in edge order.  -> (train mask, test mask)."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    n = int(max(src.max(), dst.max())) + 1 if src.size else 0
    draw = src < dst if is_undirected else np.ones(src.size, dtype=bool)
    to_train = rng.uniform(size=int(draw.sum())) <= train_ratio
    train = np.ones(src.size, dtype=bool)
    test = np.ones(src.size, dtype=bool)
    train[draw] = to_train
    test[draw] = ~to_train
    if is_undirected:
        keys = src * n + dst
        order = np.argsort(keys)
        rk = dst[draw] * n + src[draw]
        pos = np.minimum(np.searchsorted(keys[order], rk), max(keys.size - 1, 0))
        if not np.all(keys[order][pos] == rk):
            raise KeyError('missing reverse edge')
        train[order[pos]] = to_train
        test[order[pos]] = ~to_train
    return train, test


# ------------------------------------------------------------------------------------------- sample
def sample_loops(edges, node_num, n_sampled_nodes, rng, node_l=None):
    """-> (edges of the induced graph relabelled, in edge order; node_l).  node_l given: no draw."""
    if node_l is None:
        if not (n_sampled_nodes and node_num > n_sampled_nodes):
            return list(edges), np.arange(node_num)
        node_l = rng.choice(node_num, n_sampled_nodes, replace=False)
    inv = {}
    for k, v in enumerate(node_l):
        inv[int(v)] = k
    out = []
    for st, ed, w in edges:
        if st in inv and ed in inv:
            out.append((inv[st], inv[ed], w))
    return out, node_l


def induce(src, dst, node_num, node_l):
    """Vectorised induced graph: -> (kept mask in edge order, relabelled src, relabelled dst)."""
    inv = np.full(node_num, -1, dtype=np.int64)
    inv[np.asarray(node_l, dtype=np.int64)] = np.arange(len(node_l))
    u, v = inv[np.asarray(src, dtype=np.int64)], inv[np.asarray(dst, dtype=np.int64)]
    keep = (u >= 0) & (v >= 0)
    return keep, u[keep], v[keep]


# ------------------------------------------------------------------------------------------- filter and metrics
def edge_set(n, src, dst):
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    key = np.unique(src * n + dst)
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, key // n + 1, 1)
    return eo.EdgeSet(n, np.cumsum(indptr), key % n)


def filtered_loops(pred, train_edges):
    train = {(st, ed) for st, ed, _ in train_edges}
    return [e for e in pred if (e[0], e[1]) not in train]


def filtered(i, j, w, train):
    keep = ~train.has_edge(i, j)
    return i[keep], j[keep], w[keep]


def evaluate(adj, test, train, is_undirected=True, max_k=-1, edge_pairs=None):
    """Steps 4-6 on a reconstruction adj (n x n) of the evaluated rows: test, train = EdgeSet of the (sampled)
    graphs.  -> dict(MAP, node_ap, count, prec_curve, delta, n_pred, i, j, w)"""
    i, j, w = eo.edge_list_from_adj(adj, is_undirected=is_undirected, edge_pairs=edge_pairs)
    i, j, w = filtered(i, j, w, train)
    MAP, node_ap, count = eo.compute_map(i, j, w, test, is_undirected=False)
    prec, delta = eo.precision_curve(i, j, w, test, max_k)
    return {'MAP': MAP, 'node_ap': node_ap, 'count': count, 'prec_curve': prec, 'delta': delta, 'n_pred': len(w),
            'i': i, 'j': j, 'w': w}


def ranks(adj, test, train, is_undirected):
    """1-based rank of every test edge (CSR order of `test`) among its row's filtered candidates sorted by weight
    (descending, stable in j), 0 when it is not a candidate; and the candidates per row."""
    n = test.n
    i, j, w = eo.edge_list_from_adj(adj, is_undirected=is_undirected)
    i, j, w = filtered(i, j, w, train)
    n_pred_row = np.bincount(i, minlength=n)
    starts = np.searchsorted(i, np.arange(n + 1))
    out = np.zeros(len(test.indices), dtype=np.int64)
    for v in range(n):
        a, b = test.indptr[v], test.indptr[v + 1]
        if a == b:
            continue
        s, e = starts[v], starts[v + 1]
        order = np.argsort(-np.asarray(w[s:e], dtype=np.float64), kind='stable')
        pos = np.zeros(n, dtype=np.int64)
        pos[j[s:e][order]] = np.arange(1, e - s + 1)
        out[a:b] = pos[test.indices[a:b]]
    return out, n_pred_row
