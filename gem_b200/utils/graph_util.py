"""Wire formats on either side of the hot path, byte-compatible with the reference
gem/utils/graph_util.py: saveGraphToEdgeListTxt (:129-134), saveGraphToEdgeListTxtn2v (:137-140),
loadGraphFromEdgeListTxt (:143-158), loadEmbedding (:161-169).  saveEmbedding writes the `.emb`
text that SNAP's WriteOutput (bin@0x406ef0) produces and loadEmbedding reads.

The functions with the reference's names keep its signatures (networkx graphs in and out; loadEmbedding /
saveEmbedding use the native parallel reader / writer of libgemb200.so -- host code, no GPU needed -- and fall back
to the per-line loop only when the library has not been built).  loadEdgeListCSR / saveEdgeListCSR / saveCSR / loadCSR
go straight between files and gem_b200.graph.HostCSR, which is what a 20 M-edge input needs: the reference's
per-line Python loops take minutes there (SURVEY 8(f) rank 2).  get_lcc (:29-34) takes either form; on a HostCSR it
runs on the GPU."""
import os

import numpy as np


def _lib_or_none():
    from gem_b200 import _native
    return _native.lib() if os.path.exists(_native.LIB_PATH) else None


def _check(status):
    from gem_b200 import _native
    _native.check(status)


def _ptr(a):
    import ctypes
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def readEdgeList(file_name, skip_header=0):
    """-> (src int64[m], dst int64[m], w float64[m] or None when every weight is 1.0), in file order; the token
    rules of loadGraphFromEdgeListTxt (graph_util.py:149-156).  Needs libgemb200.so."""
    import ctypes
    from gem_b200 import _native
    L = _native.lib()
    path = os.fsencode(file_name)
    m = ctypes.c_int64(0)
    _check(L.gemb_edge_list_scan(path, int(skip_header), ctypes.byref(m)))
    m = int(m.value)
    src = np.empty(m, dtype=np.int64)
    dst = np.empty(m, dtype=np.int64)
    w = np.empty(m, dtype=np.float64)
    unit = ctypes.c_int32(1)
    _check(L.gemb_edge_list_parse(path, int(skip_header), m, _ptr(src), _ptr(dst), _ptr(w), ctypes.byref(unit)))
    return src, dst, (None if unit.value else w)


def loadEdgeListCSR(file_name, directed=True, n=None, skip_header=0, node_order='id'):
    """Edge-list text -> HostCSR without networkx.  Equivalent to
        graph.from_networkx(loadGraphFromEdgeListTxt(file_name, directed), by_label=(node_order == 'id'))
    node_order='id': row = integer node id, n = max id + 1 (what node2vec / loadEmbedding assume);
    node_order='appearance': row r = r-th distinct node in reading order = list(graph.nodes) of the graph the
    reference would build (what HOPE's nx.to_numpy_matrix uses, hope.py:28).  A repeated edge keeps its LAST weight
    (nx add_edge overwrites); directed=False adds the reverse of every edge (nx.Graph)."""
    from gem_b200 import graph as hg
    src, dst, w = readEdgeList(file_name, skip_header)
    nodes = None
    if node_order == 'appearance':
        inter = np.empty(2 * src.size, dtype=np.int64)
        inter[0::2] = src
        inter[1::2] = dst
        uniq, first = np.unique(inter, return_index=True)
        order = np.argsort(first, kind='stable')
        nodes = uniq[order]
        rank = np.empty(uniq.size, dtype=np.int64)
        rank[order] = np.arange(uniq.size)
        src = rank[np.searchsorted(uniq, src)]
        dst = rank[np.searchsorted(uniq, dst)]
        n_rows = uniq.size
    elif node_order == 'id':
        n_rows = int(max(src.max(), dst.max())) + 1 if src.size else 0
    else:
        raise ValueError("node_order must be 'id' or 'appearance'")
    if n is not None:
        if n < n_rows:
            raise ValueError('n = %d is smaller than the %d nodes of the file' % (n, n_rows))
        n_rows = int(n)
    if not directed:
        # nx.Graph: one undirected edge; in matrix form both directions, the later line wins for either direction
        src, dst = np.concatenate((src, dst)), np.concatenate((dst, src))
        order = np.argsort(np.concatenate((np.arange(src.size // 2), np.arange(src.size // 2))), kind='stable')
        src, dst = src[order], dst[order]
        w = None if w is None else np.concatenate((w, w))[order]
    csr = hg.from_edges(n_rows, src, dst, w, nodes=(nodes.tolist() if nodes is not None else None))
    return csr


def saveEdgeListCSR(csr, file_name, n2v=False):
    """HostCSR -> the bytes saveGraphToEdgeListTxt (n2v=False: two header lines) / saveGraphToEdgeListTxtn2v
    (n2v=True) write for the same graph with edges in row-major order."""
    L = _lib_or_none()
    if L is None:
        raise RuntimeError('libgemb200.so has not been built (python -m gem_b200.build)')
    src = np.repeat(np.arange(csr.n, dtype=np.int64), np.diff(csr.indptr))
    dst = np.ascontiguousarray(csr.indices, dtype=np.int64)
    w = None if csr.data is None else np.ascontiguousarray(csr.data, dtype=np.float64)
    _check(L.gemb_edge_list_write(os.fsencode(file_name), int(src.size), _ptr(src), _ptr(dst), _ptr(w),
                                  -1 if n2v else int(csr.n)))


def saveCSR(csr, file_name):
    """Binary CSR (NumPy .npz): the loader a 268 M-edge graph wants instead of text."""
    d = {'n': np.int64(csr.n), 'indptr': csr.indptr, 'indices': csr.indices}
    if csr.data is not None:
        d['data'] = csr.data
    if csr.symmetric is not None:
        d['symmetric'] = np.bool_(csr.symmetric)
    np.savez(file_name, **d)


def loadCSR(file_name):
    from gem_b200.graph import HostCSR
    z = np.load(file_name)
    return HostCSR(int(z['n']), z['indptr'], z['indices'], z['data'] if 'data' in z else None,
                   symmetric=(bool(z['symmetric']) if 'symmetric' in z else None))


def saveGraphToEdgeListTxt(graph, file_name):
    with open(file_name, 'w') as f:
        f.write('%d\n' % len(graph.nodes))
        f.write('%d\n' % len(graph.edges))
        for i, j, w in graph.edges(data='weight', default=1):
            f.write('%d %d %f\n' % (i, j, w))


def saveGraphToEdgeListTxtn2v(graph, file_name):
    with open(file_name, 'w') as f:
        for i, j, w in graph.edges(data='weight', default=1):
            f.write('%d %d %f\n' % (i, j, w))


def loadGraphFromEdgeListTxt(file_name, directed=True):
    import networkx as nx
    with open(file_name, 'r') as f:
        G = nx.DiGraph() if directed else nx.Graph()
        for line in f:
            edge = line.strip().split()
            if not edge:
                continue
            w = float(edge[2]) if len(edge) == 3 else 1.0
            G.add_edge(int(edge[0]), int(edge[1]), weight=w)
    return G


def loadEmbedding(file_name):
    L = _lib_or_none()
    if L is not None:
        import ctypes
        path = os.fsencode(file_name)
        rows, d = ctypes.c_int64(0), ctypes.c_int32(0)
        _check(L.gemb_emb_read(path, ctypes.byref(rows), ctypes.byref(d), None))
        X = np.zeros((int(rows.value), int(d.value)))
        _check(L.gemb_emb_read(path, ctypes.byref(rows), ctypes.byref(d), _ptr(X)))
        return X
    with open(file_name, 'r') as f:
        n, d = f.readline().strip().split()
        X = np.zeros((int(n), int(d)))
        for line in f:
            emb = line.strip().split()
            X[int(emb[0]), :] = [float(e) for e in emb[1:]]
    return X


def saveEmbedding(X, file_name, ids=None):
    """'<V> <d>' then '<id> v1 ... vd' with ~6 significant digits (C++ ostream default)."""
    X = np.asarray(X)
    L = _lib_or_none()
    if L is not None:
        X64 = np.ascontiguousarray(X, dtype=np.float64)
        idv = None if ids is None else np.ascontiguousarray(list(ids), dtype=np.int64)
        _check(L.gemb_emb_write(os.fsencode(file_name), int(X.shape[0] if idv is None else idv.size), _ptr(idv),
                                int(X.shape[1]), _ptr(X64), int(X.shape[0])))
        return
    ids = range(X.shape[0]) if ids is None else ids
    with open(file_name, 'w') as f:
        f.write('%d %d\n' % X.shape)
        for i in ids:
            f.write('%d %s\n' % (i, ' '.join('%g' % v for v in X[i])))


def get_lcc(di_graph, device=None):
    """gem/utils/graph_util.py:29-34: the largest weakly connected component, relabelled 0..k-1.
    networkx DiGraph: the reference's recipe with the helper networkx 2.4 removed written out --
        c = max(nx.weakly_connected_components(G), key=len); H = G.subgraph(c).copy()
        nodeListMap = dict(zip(list(H.nodes), range(len(H))))
    -> (H relabelled by nodeListMap, nodeListMap).  The relabelling makes a copy, so H's nodes iterate as 0..k-1 (the
    reference relabels in place: same nodes, edges and map, but a scrambled node order, and every embedding takes
    list(graph.nodes) as its row order).  Plain networkx, no device.  An undirected nx.Graph raises, as in the
    reference.  On a tie the component whose first node comes first in G's node order wins.  H's node order (and so
    the map) is the order networkx's subgraph view yields: G's node order when the component holds at least half of
    G's nodes, the component set's own iteration order otherwise.
    gem_b200.graph.HostCSR: labelled and cut on the device (gemb_cc_*), every stored edge joining its two ends.
    -> (HostCSR of the component, node_l): node_l (int64, ascending) maps new row -> old row, as sample_graph's does;
    `nodes` and `symmetric` are carried over.  On a tie the component with the smallest row wins -- the networkx
    rule over row order.  device: the CUDA device (default 0)."""
    from gem_b200.graph import HostCSR
    if isinstance(di_graph, HostCSR):
        return _lcc_csr(di_graph, 0 if device is None else int(device))
    import networkx as nx
    c = max(nx.weakly_connected_components(di_graph), key=len)
    H = di_graph.subgraph(c).copy()
    nodeListMap = dict(zip(list(H.nodes), range(len(H))))
    return nx.relabel_nodes(H, nodeListMap, copy=True), nodeListMap


def _check_csr(csr):
    """The input rules of gemb_cc_create, raised as ValueError before any device call."""
    n = int(csr.n)
    if not 0 <= n < 2 ** 31:
        raise ValueError('get_lcc: n = %d; vertex ids are int32 (n < 2^31)' % n)
    indptr = np.asarray(csr.indptr)
    if indptr.shape != (n + 1,):
        raise ValueError('get_lcc: indptr has %d entries, n + 1 = %d' % (indptr.size, n + 1))
    if int(indptr[0]) != 0:
        raise ValueError('get_lcc: indptr[0] = %d, not 0' % int(indptr[0]))
    if n and np.any(indptr[1:] < indptr[:-1]):
        raise ValueError('get_lcc: indptr is not non-decreasing')
    nnz = int(indptr[-1])
    if np.asarray(csr.indices).shape[0] < nnz:
        raise ValueError('get_lcc: indptr ends at %d, indices holds %d' % (nnz, np.asarray(csr.indices).shape[0]))
    ix = np.asarray(csr.indices)[:nnz]
    if nnz and (int(ix.min()) < 0 or int(ix.max()) >= n):
        raise ValueError('get_lcc: a column id lies outside [0, %d)' % n)
    if csr.data is not None and np.asarray(csr.data).shape[0] < nnz:
        raise ValueError('get_lcc: %d weights for %d stored edges' % (np.asarray(csr.data).shape[0], nnz))


def _lcc_csr(csr, device):
    from gem_b200 import _native
    from gem_b200.graph import HostCSR
    _check_csr(csr)
    nnz = int(csr.indptr[-1])
    with _native.Context(device) as ctx, _native.Components(ctx, csr.n, csr.indptr, csr.indices[:nnz]) as cc:
        node_l, indptr, indices, w = cc.lcc(None if csr.data is None else csr.data[:nnz])
    nodes = csr.nodes
    if nodes is not None:
        nodes = nodes[node_l] if isinstance(nodes, np.ndarray) else [nodes[i] for i in node_l.tolist()]
    return HostCSR(node_l.size, indptr, indices, w, nodes=nodes, symmetric=csr.symmetric), node_l


def sample_graph(di_graph, n_sampled_nodes=None, rng=None):
    """gem/utils/graph_util.py:42-58: when n_sampled_nodes is given and smaller than the node count,
    node_l = choice(n, n_sampled_nodes, replace=False) and the graph induced on node_l, node node_l[k] relabelled k;
    otherwise (di_graph, arange(n)) without a draw.  di_graph: a networkx graph with nodes 0..n-1 (returns a
    networkx DiGraph whose edges carry 'weight', default 1, added in di_graph.edges order, as the reference does) or
    a gem_b200.graph.HostCSR (returns a HostCSR).  rng: a np.random.RandomState, None = the global np.random."""
    from gem_b200.graph import HostCSR
    node_num = di_graph.n if isinstance(di_graph, HostCSR) else len(di_graph.nodes)
    if not (n_sampled_nodes and node_num > n_sampled_nodes):
        return di_graph, np.arange(node_num)
    node_l = (np.random if rng is None else rng).choice(node_num, n_sampled_nodes, replace=False)
    return induced_graph(di_graph, node_l), node_l


def induced_graph(di_graph, node_l):
    """The graph sample_graph builds for a given node_l: the edges with both ends in node_l, node node_l[k] -> k."""
    from gem_b200.graph import HostCSR, from_edges
    node_l = np.asarray(node_l, dtype=np.int64)
    s = node_l.size
    if isinstance(di_graph, HostCSR):
        inv = np.full(di_graph.n, -1, dtype=np.int64)
        inv[node_l] = np.arange(s)
        rows = np.repeat(np.arange(di_graph.n, dtype=np.int64), np.diff(np.asarray(di_graph.indptr, dtype=np.int64)))
        u, v = inv[rows], inv[np.asarray(di_graph.indices, dtype=np.int64)]
        keep = (u >= 0) & (v >= 0)
        return from_edges(s, u[keep], v[keep], None if di_graph.data is None else di_graph.data[keep])
    import networkx as nx
    inv = {int(v): k for k, v in enumerate(node_l.tolist())}
    sampled_graph = nx.DiGraph()
    sampled_graph.add_nodes_from(range(s))
    sampled_graph.add_weighted_edges_from((inv[st], inv[ed], w) for st, ed, w in di_graph.edges(data='weight', default=1)
                                          if st in inv and ed in inv)
    return sampled_graph
