"""evaluateStaticLinkPrediction on an H100: hold out a share of the edges, train on the rest, and rank the held-out
edges among the node pairs that are not training edges.

The task, in the reference's own functions (rng = one np.random.RandomState(seed), or the global np.random):
    train, test = split_di_graph_to_train_test(G, train_ratio, is_undirected)      evaluation_util.py:39-53
    [lcc=True, only when train has more than one weak component -- upstream GEM's step:
     train, nodeListMap = get_lcc(train)                                            graph_util.py:29-34
     test = test.subgraph(nodeListMap) relabelled by nodeListMap (HostCSR: induced_graph(test, node_l))]
    test, node_l = sample_graph(test, n_sample_nodes)  (optional; the train graph    graph_util.py:42-58
                   is induced on the same node_l, relabelled the same way)
    X = model.learn_embedding(graph=train)[node_l]
    pred = get_edge_list_from_adj_mtrx(get_reconstructed_adj(X), is_undirected)     evaluation_util.py:20-36
           (or the sampled pairs, sample_ratio_e)
    filtered = [e for e in pred if not train.has_edge(e[0], e[1])]
    MAP = computeMAP(filtered, test); prec_curv, _ = computePrecisionCurve(filtered, test)   metrics.py:6-46
computeMAP keeps its default is_undirected=False: a node without held-out out-edges has nothing to predict and is
skipped.  On the device, the training edges are an exclusion set of the reconstruction (gemb_recon_exclude): the
counting kernels rank and select over the remaining candidates, so the n^2 list is never built on the host.  In the
sampled-pairs branch the few pairs are filtered on the host.  No CPU fallback: without a GPU this raises RuntimeError.

digraph: a networkx DiGraph with nodes 0..n-1 or a gem_b200.graph.HostCSR (then the split and the sample stay in
CSR form: no networkx at any size).  The embedding's rows are taken as node ids, as evaluateStaticGraphReconstruction
does.  With lcc=True the embedding is learned on the largest component, and node ids are its 0..k-1.  The default
lcc=False keeps every node; on a training graph that is one component both give the same bits.  -> (MAP, prec_curv)
A reconstruction too large for device memory is regenerated block by block; max_k < 0 then raises ValueError (as in
evaluateStaticGraphReconstruction).
"""
import numpy as np

from gem_b200 import _native
from gem_b200.embedding.static_graph_embedding import recon_kind
from gem_b200.evaluation import metrics
from gem_b200.evaluation.evaluate_graph_reconstruction import _true_csr, check_max_k


def split_and_sample(digraph, train_ratio=0.8, n_sample_nodes=None, is_undirected=True, rng=None, lcc=False,
                     device=None):
    """The host steps 1-2: -> (train, test_sampled, train_sampled, node_l).  train is the whole training graph (what
    the model learns on); the sampled graphs are induced on node_l (all nodes when no sample is drawn).  lcc=True:
    when the training graph has more than one weak component, train is its largest one (get_lcc, on the GPU `device`
    for a HostCSR), the test graph is induced on the same nodes with the same relabelling, and node_l indexes them."""
    from gem_b200.utils import evaluation_util, graph_util
    train, test = evaluation_util.split_di_graph_to_train_test(digraph, train_ratio, is_undirected, rng)
    if lcc:
        train, test = _largest_component(train, test, device)
    test_s, node_l = graph_util.sample_graph(test, n_sample_nodes, rng)
    train_s = train if test_s is test else graph_util.induced_graph(train, node_l)
    return train, test_s, train_s, np.asarray(node_l, dtype=np.int64)


def _largest_component(train, test, device):
    """(train, test) cut to train's largest weak component, or unchanged when train is one component."""
    from gem_b200.graph import HostCSR
    from gem_b200.utils import graph_util
    if isinstance(train, HostCSR):
        train_l, node_l = graph_util.get_lcc(train, device)
        if train_l.n == train.n:
            return train, test
        return train_l, graph_util.induced_graph(test, node_l)
    import networkx as nx
    train_l, node_map = graph_util.get_lcc(train)
    if len(node_map) == len(train):
        return train, test
    return train_l, nx.relabel_nodes(test.subgraph(list(node_map)), node_map, copy=True)


def evaluateStaticLinkPrediction(digraph, graph_embedding, train_ratio=0.8, n_sample_nodes=None, sample_ratio_e=None,
                                 is_undirected=True, max_k=-1, seed=None, device=None, lcc=False):
    from gem_b200.graph import HostCSR
    kind = recon_kind(graph_embedding)
    if kind is None:
        raise TypeError("%s declares neither _recon_split (True: hope.py:43-44, False: node2vec.py:56-57) nor "
                        "_recon_score ('gaussian': lap.py:39-42)" % type(graph_embedding).__name__)
    gauss = kind == _native.RECON_GAUSS
    rng = None if seed is None else np.random.RandomState(seed)
    dev = device if device is not None else getattr(graph_embedding, '_device', 0)
    train, test_s, train_s, node_l = split_and_sample(digraph, train_ratio, n_sample_nodes, is_undirected, rng, lcc, dev)
    node_num = train.n if isinstance(train, HostCSR) else len(train.nodes)
    X = np.asarray(graph_embedding.learn_embedding(graph=train))
    if X.shape[0] != node_num:
        raise ValueError('embedding has %d rows, graph has %d nodes' % (X.shape[0], node_num))
    X = X[node_l]
    n = node_l.size
    te_indptr, te_indices = _true_csr(test_s, n)
    tr_indptr, tr_indices = _true_csr(train_s, n)
    in_test = metrics.csr_has_edge(n, te_indptr, te_indices)
    with _native.Context(dev) as ctx, _native.Reconstruction(ctx, X, kind) as rec:
        if sample_ratio_e:
            # evaluation_util.py:5-18 + :25-28, then the pairs that are training edges dropped
            from gem_b200.utils import evaluation_util
            pairs = np.array(evaluation_util.get_random_edge_pairs(n, sample_ratio_e, is_undirected, seed=seed),
                             dtype=np.int64).reshape(-1, 2)
            w = rec.pairs(pairs[:, 0], pairs[:, 1])
            if gauss:
                keep = np.ones(w.shape, dtype=bool)      # exp(-delta) >= 0 keeps every pair; order by -delta
                w = -w
            else:
                keep = w >= 0.0
            keep &= ~metrics.csr_has_edge(n, tr_indptr, tr_indices)(pairs[:, 0], pairs[:, 1])
            pi, pj, pw = pairs[keep, 0], pairs[keep, 1], w[keep]
            total, count = metrics.node_ap_sum(n, pi, pj, pw, in_test, np.diff(te_indptr), False)
            MAP = total / count if count else float('nan')
            prec_curv, _ = metrics.precision_curve(pi, pj, pw, in_test, max_k)
        else:
            check_max_k(rec, max_k)
            rec.exclude(tr_indptr, tr_indices)
            ranks, _ = rec.ranks(te_indptr, te_indices, is_undirected)
            MAP, _, _ = metrics.map_from_ranks(n, te_indptr, ranks, False)
            ti, tj, tw = rec.top(is_undirected, max_k)
            if gauss:
                tw = -tw
            prec_curv, _ = metrics.precision_curve_from_top(ti, tj, tw, in_test, max_k)
    return MAP, prec_curv
