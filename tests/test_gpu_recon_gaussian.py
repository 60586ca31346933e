"""Gaussian-score reconstruction and evaluation on the GPU: LaplacianEigenmaps / LocallyLinearEmbedding
(get_edge_weight = exp(-|x_i - x_j|^2), lap.py:39-42, lle.py:37-40) through gemb_recon_create kind 2,
StaticGraphEmbedding.get_reconstructed_adj and evaluateStaticGraphReconstruction.

The device stores an order key of delta = |x_i - x_j|^2 and returns delta itself (+inf on the diagonal and where the
fp64 score underflows).  Levels of parity, as in test_gpu_recon.py:
  * delta against fp64 on the same fp32 X: |delta - delta64| <= max(2d, d + 2) * 2^-24 * delta64 (the worst case of
    d fp32 differences squared and summed with FMA; for d >= 2 that is 2d * 2^-24), exactly 0 for equal rows;
  * the evaluation logic BIT-EXACT against the pinned oracle run on the GPU's own delta matrix.  The oracle gets
    1 / delta as its score: in fp64 that orders exactly as delta does for every fp32 delta (exp(-delta) would merge
    distances below ~1e-16) and is > 0 exactly where delta is finite;
  * the reference's goldens (tests/golden/eval_*_lap / _lle / _gauss .npz; fp64 X, except SBM-1024 whose X is the
    reference's golden rounded to fp32): MAP within 2e-3.  Casting X to fp32 moves the oracle's MAP on these goldens
    by less than 1e-4, so the goldens are compared as they are.
"""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, load_karate_nx
from gauss_golden import gauss_golden

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings('ignore::RuntimeWarning')]   # an unconverged learn_embedding warns
sys.path.insert(0, os.path.join(REPO, 'oracle'))

U = 2.0 ** -24
DELTA_MAX = np.uint32(0x443a4886).view(np.float32)          # 745.1332f: the last delta with fp64 exp(-delta) > 0


def _sqdist64(X):
    """fp64 |x_i - x_j|^2 of the given (fp32) rows, difference form, in row blocks."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    D = np.empty((n, n))
    for b in range(0, n, 32):
        T = X[b:b + 32, None, :] - X[None, :, :]
        D[b:b + 32] = np.einsum('ijk,ijk->ij', T, T)
    return D


def _bound(d):
    return max(2 * d, d + 2) * U


def _order_score(D):
    """fp64 score that the oracle ranks exactly as the device ranks delta (module docstring)."""
    with np.errstate(divide='ignore'):
        return 1.0 / np.asarray(D, dtype=np.float64)


def _nx_from(n, indptr, indices, w, nodes=None):
    import networkx as nx
    G = nx.DiGraph()
    G.add_nodes_from(range(n) if nodes is None else (int(u) for u in nodes))
    rows = np.repeat(np.arange(n), np.diff(indptr))
    for u, v, ww in zip(rows.tolist(), indices.tolist(), w.tolist()):
        G.add_edge(u, v, weight=ww)
    return G


def _model(cls_name, d=2):
    if cls_name == 'lle':
        from gem_b200.embedding.lle import LocallyLinearEmbedding as C
        method = 'lle_svd'
    else:
        from gem_b200.embedding.lap import LaplacianEigenmaps as C
        method = 'lap_eigmap_svd'
    C.hyper_params.clear()
    C.hyper_params.update({'method_name': method})
    return C(d=d)


def _random_graph(rng, n, deg):
    src = np.repeat(np.arange(n), deg)
    dst = rng.integers(0, n, n * deg)
    key = np.unique(src.astype(np.int64) * n + dst)
    src, dst = key // n, key % n
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, src + 1, 1)
    return np.cumsum(indptr), dst


# ---- 1. delta accuracy
@pytest.mark.parametrize('d,n', [(1, 1), (2, 63), (3, 65), (1, 1024), (128, 1024), (300, 1024), (2, 4500),
                                 (128, 4500), (300, 65)])
def test_delta_accuracy(gpu_ctx, d, n):
    from gem_b200 import _native
    rng = np.random.default_rng(1000 * d + n)
    X = (rng.standard_normal((n, d)) * (1.0 / np.sqrt(d))).astype(np.float32)
    if n > 40:
        X[20:30] = X[0:10]                                   # equal rows: delta exactly 0
    rec = _native.Reconstruction(gpu_ctx, X, 2)
    try:
        D = rec.dense()
        assert D.dtype == np.float32 and D.shape == (n, n)
        assert np.all(np.isposinf(np.diag(D)))
        ref = _sqdist64(X)
        off = ~np.eye(n, dtype=bool)
        assert np.all(np.isfinite(D[off]))
        err = np.abs(D.astype(np.float64) - ref)
        assert np.all(err[off] <= _bound(d) * ref[off]), float(np.max(err[off] / np.maximum(ref[off], 1e-300)))
        if n > 40:
            assert np.all(D[np.arange(20, 30), np.arange(0, 10)] == 0) and np.all(D[np.arange(0, 10), np.arange(20, 30)] == 0)
        # the padded columns of the last panel are never reported: every off-diagonal pair, nothing more
        ti, tj, tw = rec.top(False, -1)
        assert ti.size == n * (n - 1) and np.all(tj < n) and np.all(ti != tj)
        assert np.array_equal(tw, D[ti, tj])
        pi = rng.integers(0, n, 3000); pj = rng.integers(0, n, 3000)
        assert np.array_equal(rec.pairs(pi, pj), D[pi, pj])
    finally:
        rec.free()


# ---- 2 + 3. evaluation logic exact against the oracle on the GPU's delta, and the reference goldens
@pytest.mark.parametrize('name,variants', [('eval_karate_lap', ('und', 'dir', 'dirw')),
                                           ('eval_karate_lle', ('und', 'dir', 'dirw')),
                                           ('eval_randw200_gauss', ('und', 'dir', 'dirw')),
                                           ('eval_sbm1024_lap', ('und',))])
def test_evaluation_matches_oracle_and_reference_goldens(gpu_ctx, eval_oracle, name, variants):
    from gem_b200 import _native
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    eo = eval_oracle
    z, n, (indptr, indices, w) = gauss_golden(name)
    X = z['X']
    H = _nx_from(n, indptr, indices, w, nodes=z['nodes'])
    m = _model('lap' if 'lle' not in name else 'lle', X.shape[1])
    A = m.get_reconstructed_adj(X=X)
    assert A.dtype == np.float64 and m.get_embedding() is X and np.all(np.diag(A) == 0)
    rec = _native.Reconstruction(gpu_ctx, X, 2)
    D = rec.dense()
    rec.free()
    assert np.array_equal(A, np.exp(-D.astype(np.float64)))
    S = _order_score(D)
    edges = eo.EdgeSet(n, indptr, indices)
    for tag in variants:
        und = tag == 'und'
        MAP, prec, err, err_b = evaluateStaticGraphReconstruction(H, m, X, None, is_undirected=und,
                                                                  is_weighted=(tag == 'dirw'))
        r = eo.evaluate(S, edges, is_undirected=und)
        assert len(prec) == r['n_pred']
        assert np.array_equal(np.array(prec), r['prec_curve'])                 # evaluation logic: exact
        assert abs(MAP - r['MAP']) < 1e-13
        assert len(prec) == int(z[tag + '_n_pred'])                              # only underflowed pairs dropped
        assert abs(MAP - float(z[tag + '_MAP'])) < 2e-3                          # reference golden (fp64 X)
        h = min(len(prec), 200)
        assert np.mean(np.abs(np.array(prec[:h]) - z[tag + '_prec_head'][:h])) < 0.02
        if tag == 'dirw':
            rw = eo.evaluate(A, edges, weights=w, is_undirected=False, is_weighted=True, node_order=z['nodes'])
            assert abs(err - rw['err']) < 1e-9 and abs(err_b - rw['err_baseline']) < 1e-12
            assert abs(err - float(z[tag + '_err'])) < 1e-4 and abs(err_b - float(z[tag + '_err_baseline'])) < 1e-9
        else:
            assert err is None and err_b is None


@pytest.mark.parametrize('d,n', [(128, 4500), (2, 4200)])
def test_large_ranks_and_top_match_oracle(gpu_ctx, eval_oracle, d, n):
    """Many CTAs, n not a multiple of 64; ranks / n_pred / top-k exact against the oracle on the GPU's delta."""
    from gem_b200 import _native
    eo = eval_oracle
    rng = np.random.default_rng(n + d)
    X = (rng.standard_normal((n, d)) * (1.0 / np.sqrt(d))).astype(np.float32)
    X[:50] = np.round(X[:50], 1)
    X[60:80] = X[0:20]                                        # exact delta = 0 ties
    indptr, dst = _random_graph(rng, n, 12)
    rec = _native.Reconstruction(gpu_ctx, X, 2)
    try:
        D = rec.dense()
        S = _order_score(D)
        for und in (True, False):
            ranks, n_pred_row = rec.ranks(indptr, dst, und)
            i, j, w = eo.edge_list_from_adj(S, is_undirected=und)
            assert np.array_equal(np.bincount(i, minlength=n), n_pred_row)
            starts = np.searchsorted(i, np.arange(n + 1))
            for v in list(range(0, 80, 7)) + rng.choice(n, 200, replace=False).tolist():
                s, e = starts[v], starts[v + 1]
                order = np.argsort(-w[s:e], kind='stable')
                pos = {int(c): r + 1 for r, c in enumerate(j[s:e][order])}
                exp = [pos.get(int(dst[t]), 0) for t in range(indptr[v], indptr[v + 1])]
                assert np.array_equal(ranks[indptr[v]:indptr[v + 1]], exp), v
            ref = np.argsort(-w, kind='stable')
            for max_k in (1, 1000, 50000):
                ti, tj, tw = rec.top(und, max_k)
                order = np.lexsort((tj, ti, tw.astype(np.float64)))[:max_k]     # delta ascending, then i, j
                assert np.array_equal(ti[order], i[ref[:max_k]]) and np.array_equal(tj[order], j[ref[:max_k]])
                assert np.array_equal(tw[order], D[i[ref[:max_k]], j[ref[:max_k]]])
    finally:
        rec.free()


# ---- 4. the underflow boundary
def _boundary_embedding():
    """Rows 0, 1, 2 with fp32 delta(0, 1) = 745.1332f exactly and delta(0, 2) = the next float.  fl(t * t) skips
    745.1332f for every fp32 t, so the rows have d = 2: delta(0, 1) = fl(fl(t^2) + s^2) with s^2 = m ulps exact."""
    T = np.uint32(0x443a4886)
    t0 = np.float32(np.sqrt(745.1332)).view(np.uint32)
    ts = (t0 + np.arange(-400, 400)).astype(np.uint32).view(np.float32)
    sq = (ts * ts).view(np.uint32)
    ulp = np.float32(2.0 ** -14)                              # spacing of fp32 at 745
    for r in range(1, 12):
        hit = ts[sq == T - np.uint32(r * r)]
        if hit.size:
            t1, s1 = hit[0], np.float32(r * 2.0 ** -7)       # s1^2 = r^2 ulps, exact
            break
    assert np.float32(t1 * t1 + s1 * s1).view(np.uint32) == T and s1 * s1 == np.float32(r * r) * ulp
    hit2 = ts[sq == T + np.uint32(1)]
    assert hit2.size
    X = np.array([[0.0, 0.0], [t1, s1], [-hit2[0], 0.0]], dtype=np.float32)
    return X


def test_underflow_boundary(gpu_ctx, eval_oracle, monkeypatch):
    import networkx as nx
    from gem_b200 import _native
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    from gem_b200.utils import evaluation_util
    X = _boundary_embedding()
    rec = _native.Reconstruction(gpu_ctx, X, 2)
    try:
        D = rec.dense()
        assert D[0, 1] == DELTA_MAX and D[1, 0] == DELTA_MAX
        assert np.isposinf(D[0, 2]) and np.isposinf(D[2, 0]) and np.isposinf(D[1, 2])
        assert np.exp(-np.float64(DELTA_MAX)) > 0
        assert np.exp(-np.float64(np.nextafter(DELTA_MAX, np.float32(np.inf)))) == 0
        indptr = np.array([0, 2, 3, 4]); indices = np.array([1, 2, 0, 0])
        for und in (True, False):
            ranks, n_pred_row = rec.ranks(indptr, indices, und)
            assert ranks.tolist() == ([1, 0, 0, 0] if und else [1, 0, 1, 0])
            assert n_pred_row.tolist() == ([1, 0, 0] if und else [1, 1, 0])
            for max_k in (-1, 1, 5):
                ti, tj, tw = rec.top(und, max_k)           # (0, 1) and (1, 0) tie: both reach the 1st weight
                assert sorted(zip(ti.tolist(), tj.tolist())) == ([(0, 1)] if und else [(0, 1), (1, 0)])
                assert np.all(tw == DELTA_MAX)
        w = rec.pairs(np.array([0, 0, 1, 2]), np.array([1, 2, 2, 2]))
        assert w[0] == DELTA_MAX and np.all(np.isposinf(w[1:]))
    finally:
        rec.free()
    # the sampled-pairs branch keeps every pair (exp(-delta) >= 0), underflowed and diagonal ones included
    G = nx.DiGraph()
    G.add_nodes_from(range(3))
    G.add_edges_from([(0, 1), (0, 2), (1, 0), (2, 0)])
    pairs = [(0, 2), (0, 1), (2, 2), (1, 2), (2, 0)]
    monkeypatch.setattr(evaluation_util, 'get_random_edge_pairs', lambda *a, **k: list(pairs))
    m = _model('lap', 2)
    MAP, prec, _, _ = evaluateStaticGraphReconstruction(G, m, X, None, sample_ratio_e=1.0, is_undirected=False)
    eo = eval_oracle
    A = np.exp(-D.astype(np.float64))                        # the reference's scores of the GPU's delta: 5e-324 and 0
    assert A[0, 1] > 0 and np.count_nonzero(A) == 2
    edges = eo.EdgeSet.from_networkx(G)
    r = eo.evaluate(A, edges, is_undirected=False, edge_pairs=pairs)
    assert len(prec) == len(pairs) == r['n_pred']
    assert np.array_equal(np.array(prec), r['prec_curve']) and abs(MAP - r['MAP']) < 1e-13


# ---- 5. end to end: the reference's call after learn_embedding
@pytest.mark.parametrize('cls_name', ['lap', 'lle'])
def test_learn_then_evaluate_karate(gpu_ctx, eval_oracle, cls_name):
    import eval_gauss_oracle as go
    from gem_b200 import _native
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    eo = eval_oracle
    G = load_karate_nx()
    m = _model(cls_name, 2)
    X = m.learn_embedding(graph=G, is_weighted=True, no_python=True)
    MAP, prec, err, err_b = evaluateStaticGraphReconstruction(G, m, X, None)
    assert 0.0 < MAP <= 1.0 and err is None
    n = len(G.nodes)
    rec = _native.Reconstruction(gpu_ctx, X, 2)
    D = rec.dense()
    rec.free()
    edges = eo.EdgeSet.from_networkx(G)
    r = eo.evaluate(_order_score(D), edges, is_undirected=True)
    assert abs(MAP - r['MAP']) < 1e-13 and np.array_equal(np.array(prec), r['prec_curve'])
    A = m.get_reconstructed_adj()
    assert A.dtype == np.float64 and A.shape == (n, n) and np.all(np.diag(A) == 0)
    ref = go.reconstruct_gaussian(np.asarray(X, dtype=np.float32), exact=True)
    delta64 = _sqdist64(np.asarray(X, dtype=np.float32))
    off = ~np.eye(n, dtype=bool)
    tol = ref * (np.expm1(_bound(2) * delta64) + 4e-16)
    assert np.all(np.abs(A - ref)[off] <= tol[off])


# ---- 6. reproducibility and ownership
def test_two_creates_give_identical_bits(gpu_ctx):
    from gem_b200 import _native
    X = np.random.default_rng(3).standard_normal((3000, 24)).astype(np.float32)
    out = []
    for _ in range(2):
        rec = _native.Reconstruction(gpu_ctx, X, 2)
        ti, tj, tw = rec.top(True, 1000)
        o = np.lexsort((tj, ti, tw))                          # top returns its entries unordered
        out.append((rec.dense().tobytes(), ti[o].tobytes(), tj[o].tobytes(), tw[o].tobytes()))
        rec.free()
    assert out[0] == out[1]


@pytest.mark.skipif(os.environ.get('GEMB_CACHE_MB', '').strip() == '0',
                    reason='GEMB_CACHE_MB=0: no block cache, gemb_mem_live_blocks is always 0')
def test_no_leak_and_non_finite_input(gpu_ctx):
    from gem_b200 import _native
    n = 700
    X = np.random.default_rng(5).standard_normal((n, 16)).astype(np.float32)
    nbr = np.sort(np.stack(((np.arange(n) + 1) % n, (np.arange(n) + 7) % n), axis=1), axis=1).ravel()

    def cycle():
        r = _native.Reconstruction(gpu_ctx, X, 2)
        out = (r.dense(), r.pairs(np.arange(10), np.arange(10, 20)), r.ranks(np.arange(0, 2 * n + 1, 2), nbr, True),
               r.top(True, max_k=50))
        r.free()
        return out

    ref = cycle()
    before = _native.mem_live_blocks()
    again = cycle()
    assert _native.mem_live_blocks() == before
    assert ref[0].tobytes() == again[0].tobytes()
    for bad_value in (np.nan, np.inf, -np.inf):
        B = X.copy()
        B[n // 2, 3] = bad_value
        with pytest.raises(RuntimeError, match='finite'):
            _native.Reconstruction(gpu_ctx, B, 2)
        assert _native.mem_live_blocks() == before
    assert cycle()[0].tobytes() == ref[0].tobytes()
