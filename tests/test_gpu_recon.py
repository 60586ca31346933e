"""Reconstruction + MAP / precision-curve parity on the GPU (SURVEY 8(f) rank 1), through the reference-facing
functions (gem_b200.evaluation.evaluate_graph_reconstruction.evaluateStaticGraphReconstruction,
StaticGraphEmbedding.get_reconstructed_adj -> ctypes -> gemb_recon_*).

Two levels of parity:
  * the reconstruction itself vs the fp64 oracle: |A_hat - L R^T| <= 4e-6 * |L_i| |R_j|  (3xTF32 / fp32 arithmetic);
  * the evaluation logic BIT-EXACT: the oracle's metrics (pinned against the reference's own functions,
    tests/test_oracle_eval.py) evaluated on the matrix the GPU produced must give the same ranks, n_pred, precision
    curve (exact equality) and MAP (1e-13) as the GPU's counting kernels;
and the reference's goldens (tests/golden/eval_*.npz) within the fp32 tolerance of the scores: |MAP - golden| < 2e-3.
"""
import numpy as np
import pytest

from conftest import eval_golden

pytestmark = pytest.mark.gpu


def _nx_from(n, indptr, indices, w):
    import networkx as nx
    G = nx.DiGraph()
    G.add_nodes_from(range(n))
    rows = np.repeat(np.arange(n), np.diff(indptr))
    for u, v, ww in zip(rows.tolist(), indices.tolist(), w.tolist()):
        G.add_edge(u, v, weight=ww)
    return G


def _model(split, d):
    from gem_b200.embedding.hope import HOPE
    from gem_b200.embedding.node2vec import node2vec
    if split:
        HOPE.hyper_params.clear(); HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
        return HOPE(d=d, beta=0.01)
    node2vec.hyper_params.clear(); node2vec.hyper_params.update({'method_name': 'node2vec_rw'})
    return node2vec(d=d)


def _check_dense(A, X, split):
    X = np.asarray(X, dtype=np.float64)
    k = X.shape[1] // 2
    L, R = (X[:, :k], X[:, k:]) if split else (X, X)
    ref = L @ R.T
    np.fill_diagonal(ref, 0.0)
    bound = 4e-6 * np.outer(np.linalg.norm(L, axis=1), np.linalg.norm(R, axis=1)) + 1e-30
    assert np.all(np.abs(A - ref) <= bound), float(np.max(np.abs(A - ref) / bound))
    assert np.all(np.diag(A) == 0)


@pytest.mark.parametrize('name,variants', [('eval_karate_hope', ('und', 'dir', 'dirw')),
                                           ('eval_karate_n2v', ('und', 'dir', 'dirw')),
                                           ('eval_randw200_split', ('und', 'dir', 'dirw')),
                                           ('eval_randw200_dot', ('und', 'dir', 'dirw')),
                                           ('eval_sbm1024_hope', ('und',))])
def test_evaluation_matches_oracle_and_reference_goldens(gpu_ctx, eval_oracle, name, variants):
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    eo = eval_oracle
    z, n, (indptr, indices, w) = eval_golden(name)
    split = bool(z['split'])
    X = z['X']
    G = _nx_from(n, indptr, indices, w)
    # the weighted error depends on list(G.nodes) order (oracle docstring): rebuild it as the golden had it
    import networkx as nx
    H = nx.DiGraph()
    H.add_nodes_from(int(u) for u in z['nodes'])
    H.add_edges_from(G.edges(data=True))
    m = _model(split, X.shape[1])
    A = m.get_reconstructed_adj(X=X)
    assert A.dtype == np.float64 and m.get_embedding() is X
    _check_dense(A, X, split)
    edges = eo.EdgeSet(n, indptr, indices)
    for tag in variants:
        und = tag == 'und'
        MAP, prec, err, err_b = evaluateStaticGraphReconstruction(H, m, X, None, is_undirected=und,
                                                                  is_weighted=(tag == 'dirw'))
        r = eo.evaluate(A, edges, weights=w, is_undirected=und, is_weighted=(tag == 'dirw'), node_order=z['nodes'])
        assert len(prec) == r['n_pred']
        assert np.array_equal(np.array(prec), r['prec_curve'])                 # evaluation logic: exact
        assert abs(MAP - r['MAP']) < 1e-13
        assert abs(MAP - float(z[tag + '_MAP'])) < 2e-3                          # reference golden (fp64 scores)
        if 'randw200' not in name:      # that case has thousands of exactly-zero scores: '> 0' is knife-edge in fp32
            assert abs(len(prec) - int(z[tag + '_n_pred'])) <= 2
        h = min(len(prec), 200)
        assert np.mean(np.abs(np.array(prec[:h]) - z[tag + '_prec_head'][:h])) < 0.02
        if tag == 'dirw':
            assert abs(err - r['err']) < 1e-9 and abs(err_b - r['err_baseline']) < 1e-12
            assert abs(err - float(z[tag + '_err'])) < 1e-4 and abs(err_b - float(z[tag + '_err_baseline'])) < 1e-9
        else:
            assert err is None and err_b is None


@pytest.mark.parametrize('split,d,n', [(True, 128, 4500), (False, 128, 4200), (True, 32, 5000)])
def test_large_reconstruction_tensor_core_path(gpu_ctx, eval_oracle, split, d, n):
    """n >= 4096: the 64-column panels go through the wgmma 3xTF32 kernel (128-row tiles for k <= 64, 64-row tiles for
    k = 128); n not a multiple of 64 exercises the padded last panel.
    Ranks / n_pred / top-k selection are checked exactly against the oracle run on the GPU's own matrix."""
    from gem_b200 import _native
    eo = eval_oracle
    rng = np.random.default_rng(n)
    X = (rng.standard_normal((n, d)) * 0.3).astype(np.float32)
    X[:50] = np.round(X[:50], 1)                                  # exact ties among the first rows
    deg = 12
    src = np.repeat(np.arange(n), deg)
    dst = rng.integers(0, n, n * deg)
    key = np.unique(src.astype(np.int64) * n + dst)
    src, dst = key // n, key % n
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, src + 1, 1)
    indptr = np.cumsum(indptr)
    edges = eo.EdgeSet(n, indptr, dst)
    rec = _native.Reconstruction(gpu_ctx, X, split)
    A = rec.dense()
    _check_dense(A.astype(np.float64), X, split)
    for und in (True, False):
        ranks, n_pred_row = rec.ranks(indptr, dst, und)
        i, j, w = eo.edge_list_from_adj(A, is_undirected=und)
        assert np.array_equal(np.bincount(i, minlength=n), n_pred_row)
        # oracle ranks of the true edges: position within the row's stable descending order
        rows = np.repeat(np.arange(n), np.diff(indptr))
        exp = np.zeros(len(dst), dtype=np.int64)
        starts = np.searchsorted(i, np.arange(n + 1))
        for v in rng.choice(n, 300, replace=False):
            s, e = starts[v], starts[v + 1]
            order = np.argsort(-w[s:e].astype(np.float64), kind='stable')
            pos = {int(c): r + 1 for r, c in enumerate(j[s:e][order])}
            for t in range(indptr[v], indptr[v + 1]):
                exp[t] = pos.get(int(dst[t]), 0)
            assert np.array_equal(ranks[indptr[v]:indptr[v + 1]], exp[indptr[v]:indptr[v + 1]]), v
        for max_k in (1, 1000, 50000):
            ti, tj, tw = rec.top(und, max_k)
            order = np.lexsort((tj, ti, -tw.astype(np.float64)))[:max_k]
            ref = np.argsort(-w.astype(np.float64), kind='stable')[:max_k]
            assert np.array_equal(ti[order], i[ref]) and np.array_equal(tj[order], j[ref])
            assert np.array_equal(tw[order], w[ref])
    pi = rng.integers(0, n, 5000); pj = rng.integers(0, n, 5000)
    pi[:10] = pj[:10]
    assert np.array_equal(rec.pairs(pi, pj), A[pi, pj])
    rec.free()


def test_sampled_pairs_branch_and_errors(gpu_ctx):
    import networkx as nx
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    rng = np.random.default_rng(5)
    n = 300
    G = nx.gnp_random_graph(n, 0.05, seed=1, directed=True)
    X = rng.standard_normal((n, 8)) * 0.5
    m = _model(True, 8)
    MAP, prec, err, err_b = evaluateStaticGraphReconstruction(G, m, X, None, sample_ratio_e=0.1, is_undirected=False)
    assert 0.0 <= MAP <= 1.0 and len(prec) > 0 and all(0.0 <= p <= 1.0 for p in prec) and err is None

    class Other:
        def get_embedding(self): return X
    with pytest.raises(TypeError, match='_recon_split'):
        evaluateStaticGraphReconstruction(G, Other(), None)
    with pytest.raises(ValueError, match='rows'):
        evaluateStaticGraphReconstruction(G, m, X[:10], None)
