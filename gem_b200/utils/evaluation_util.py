"""Sampling and splitting helpers of the evaluation (reference gem/utils/evaluation_util.py:5-53)."""
import secrets

import numpy as np


def get_random_edge_pairs(node_num, sample_ratio=0.01, is_undirected=True, seed=None):
    """Distinct random (st, ed) pairs: int(sample_ratio * n * (n - 1)) of them, half that for undirected graphs, where
    (a, b) and (b, a) count as the same pair; self pairs are possible, as in the reference.  The reference draws from
    `secrets` (not reproducible); `seed` (extra) makes the sample reproducible."""
    num_pairs = int(sample_ratio * node_num * (node_num - 1))
    if is_undirected:
        num_pairs = num_pairs / 2
    rng = np.random.default_rng(secrets.randbits(64) if seed is None else seed)
    chosen = set()
    out = []
    while len(out) < num_pairs:
        a, b = (int(x) for x in rng.integers(0, node_num, 2))
        if (a, b) in chosen or (is_undirected and (b, a) in chosen):
            continue
        chosen.add((a, b))
        out.append((a, b))
    return out


def get_edge_list_from_adj_mtrx(adj, threshold=0.0, is_undirected=True, edge_pairs=None):
    """gem/utils/evaluation_util.py:20-36: [(i, j, adj[i, j]), ...] in row-major order -- entries > threshold off the
    diagonal (i < j only when is_undirected), or the given pairs with adj >= threshold.  Vectorised; same list."""
    adj = np.asarray(adj)
    node_num = adj.shape[0]
    if edge_pairs:
        ep = np.asarray(edge_pairs, dtype=np.int64).reshape(-1, 2)
        w = adj[ep[:, 0], ep[:, 1]]
        keep = w >= threshold
        return [(int(a), int(b), c) for a, b, c in zip(ep[keep, 0], ep[keep, 1], w[keep])]
    mask = adj > threshold
    mask[np.arange(node_num), np.arange(node_num)] = False
    if is_undirected:
        mask &= np.triu(np.ones((node_num, node_num), dtype=bool), 1)
    ii, jj = np.nonzero(mask)                                  # row-major order, like the reference's double loop
    return [(int(a), int(b), c) for a, b, c in zip(ii, jj, adj[ii, jj])]


def _uniform(rng, m):
    """m draws of rng.uniform() (the global np.random when rng is None); one vector call gives the same m numbers."""
    return (np.random if rng is None else rng).uniform(size=m)


def split_di_graph_to_train_test(di_graph, train_ratio, is_undirected=True, rng=None):
    """gem/utils/evaluation_util.py:39-53: one uniform() per edge in edge order, <= train_ratio -> train, otherwise
    test; under is_undirected only st < ed edges draw and both directions move together.  Both graphs keep every node.
    Kept from the reference: under is_undirected self-loops (and an st > ed edge whose reverse is absent) stay in both
    graphs, and a drawing edge whose reverse is missing is an error (networkx.NetworkXError).
    di_graph: a networkx DiGraph (returns two networkx graphs, copies of it with edges removed) or a
    gem_b200.graph.HostCSR (edges drawn in row-major order; returns two HostCSR).  rng: a np.random.RandomState,
    None = the global np.random (the reference)."""
    from gem_b200.graph import HostCSR
    if isinstance(di_graph, HostCSR):
        return _split_csr(di_graph, train_ratio, is_undirected, rng)
    import networkx as nx
    e = list(di_graph.edges())
    st = np.array([int(a) for a, _ in e], dtype=np.int64)
    ed = np.array([int(b) for _, b in e], dtype=np.int64)
    draw = st < ed if is_undirected else np.ones(st.size, dtype=bool)
    to_train = _uniform(rng, int(draw.sum())) <= train_ratio
    ds, dd = st[draw], ed[draw]
    if is_undirected:
        for a, b in zip(ds.tolist(), dd.tolist()):
            if not di_graph.has_edge(b, a):
                raise nx.NetworkXError('The edge %s-%s is not in the graph' % (b, a))
    train_digraph = di_graph.copy()
    test_digraph = di_graph.copy()
    for g, sel in ((test_digraph, to_train), (train_digraph, ~to_train)):
        rm = list(zip(ds[sel].tolist(), dd[sel].tolist()))
        g.remove_edges_from(rm)
        if is_undirected:
            g.remove_edges_from([(b, a) for a, b in rm])
    return train_digraph, test_digraph


def _split_csr(csr, train_ratio, is_undirected, rng):
    from gem_b200.graph import HostCSR
    n = csr.n
    indptr = np.asarray(csr.indptr, dtype=np.int64)
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(indptr))
    cols = np.asarray(csr.indices, dtype=np.int64)
    keys = rows * n + cols                                    # ascending: rows, then sorted columns
    draw = rows < cols if is_undirected else np.ones(rows.size, dtype=bool)
    to_train = _uniform(rng, int(draw.sum())) <= train_ratio
    in_train = np.ones(rows.size, dtype=bool)
    in_test = np.ones(rows.size, dtype=bool)
    in_train[draw] = to_train
    in_test[draw] = ~to_train
    if is_undirected:
        # the reverse of every drawing edge must exist; an st > ed edge follows the draw of its reverse
        rk = cols[draw] * n + rows[draw]
        pos = np.minimum(np.searchsorted(keys, rk), max(keys.size - 1, 0))
        found = keys[pos] == rk
        if not found.all():
            import networkx as nx
            t = int(np.flatnonzero(~found)[0])
            raise nx.NetworkXError('The edge %d-%d is not in the graph' % (cols[draw][t], rows[draw][t]))
        in_train[pos] = to_train
        in_test[pos] = ~to_train
    out = []
    for keep in (in_train, in_test):
        ip = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(np.bincount(rows[keep], minlength=n), out=ip[1:])
        out.append(HostCSR(n, ip, cols[keep].astype(np.int32), None if csr.data is None else csr.data[keep],
                           nodes=csr.nodes))
    return out[0], out[1]
