"""The reconstruction in column blocks (gemb_recon_create_blocked): a handle that regenerates its matrix block by block
in every call gives the same bits as the handle that keeps it whole (automatic at these sizes).

Every comparison is np.array_equal; float outputs are compared as bit patterns, and the entries of top in (i, j)
order (the pairs are distinct, so that order is canonical; callers sort the same set by w first).  Covered: the three
kinds at n = 1000 (CUDA-core apply), 4200 and 5000 (tensor-core apply, padded last panel), exact ties (rounded and duplicated rows) and underflowing Gaussian pairs, 1, 3 and 7 panels per
block (7: a short last block), dense / pairs / ranks / top, with an exclusion set and after clearing it; a 16-block
run at n = 65 536; the public evaluation functions forced to one panel per block; device-block ownership; two
blocked runs.
"""
import numpy as np
import pytest

from conftest import eval_golden, golden_path
from test_gpu_linkpred import _case, _keys

pytestmark = pytest.mark.gpu

MAX_KS = (0, 1, 1000, 50000, -1)


def _inputs(kind, n):
    rng = np.random.default_rng(100 * n + kind)
    d = {0: 64, 1: 32, 2: 8}[kind]
    X = (rng.standard_normal((n, d)) * (0.3 if kind != 2 else 0.6)).astype(np.float32)
    X[:50] = np.round(X[:50], 1)                             # exact ties
    X[100:150] = X[0:50]                                     # duplicated rows
    if kind == 2:
        X[200:260] *= 30.0                                   # pairs past 745.1332: the fp64 score underflows
    deg = 12
    key = np.unique(np.repeat(np.arange(n, dtype=np.int64), deg) * n + rng.integers(0, n, n * deg))
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, key // n + 1, 1)
    return rng, X, np.cumsum(indptr), key % n


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _top(rec, und, max_k):
    i, j, w = rec.top(und, max_k)
    o = np.argsort(i.astype(np.int64) * rec.n + j)
    return i[o], j[o], _bits(w[o])


def _tied_max_k(rec, und):
    """A max_k that cuts inside a run of equal values: its top returns more than max_k entries."""
    _, _, w = rec.top(und, 20000)
    w = np.sort(w)[::-1]
    return int(np.flatnonzero(w[1:] == w[:-1])[0]) + 1


def _results(rec, indptr, indices, pi, pj, max_ks):
    out = {'pairs': _bits(rec.pairs(pi, pj))}
    for und in (True, False):
        r, npr = rec.ranks(indptr, indices, und)
        out['ranks', und] = r
        out['npred', und] = npr
        for k in max_ks[und]:
            out['top', und, k] = _top(rec, und, k)
    return out


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for key in a:
        x, y = a[key], b[key]
        if isinstance(x, tuple):
            assert all(np.array_equal(u, v) for u, v in zip(x, y)), key
        else:
            assert np.array_equal(x, y), key


@pytest.mark.parametrize('n', [1000, 4200, 5000])
@pytest.mark.parametrize('kind', [0, 1, 2])
def test_blocked_equals_resident(gpu_ctx, kind, n):
    from gem_b200 import _native
    rng, X, indptr, indices = _inputs(kind, n)
    pi = rng.integers(0, n, 20000)
    pj = rng.integers(0, n, 20000)
    pi[:50] = pj[:50]                                        # diagonal pairs
    with _native.Reconstruction(gpu_ctx, X, kind) as auto:
        assert auto.blocks == 1 and auto.panels_per_block == (n + 63) // 64
        D = auto.dense()
        max_ks = {und: MAX_KS + (_tied_max_k(auto, und),) for und in (True, False)}
        for und in (True, False):
            k = max_ks[und][-1]
            assert auto.top(und, k)[0].size > k
        ref = _results(auto, indptr, indices, pi, pj, max_ks)
        A = _keys(D) if kind == 2 else D.astype(np.float64)
        cases = {und: _case(np.random.default_rng(n + 7), n, A, und) for und in (True, False)}
        ref_ex = {}
        for und in (True, False):
            (tp, ti), (xp, xi) = cases[und]
            auto.exclude(xp, xi)
            ref_ex[und] = auto.ranks(tp, ti, und), [_top(auto, und, k) for k in (0, 1, 1000, -1)]
            auto.exclude(None, None)
    for ppb in (1, 3, 7):
        with _native.Reconstruction(gpu_ctx, X, kind, panels_per_block=ppb) as rec:
            assert rec.panels_per_block == ppb and rec.blocks == -(-((n + 63) // 64) // ppb) > 1
            assert np.array_equal(_bits(rec.dense()), _bits(D))
            _assert_same(_results(rec, indptr, indices, pi, pj, max_ks), ref)
            for und in (True, False):
                (tp, ti), (xp, xi) = cases[und]
                rec.exclude(xp, xi)
                r, npr = rec.ranks(tp, ti, und)
                assert np.array_equal(r, ref_ex[und][0][0]) and np.array_equal(npr, ref_ex[und][0][1])
                for got, exp in zip([_top(rec, und, k) for k in (0, 1, 1000, -1)], ref_ex[und][1]):
                    assert all(np.array_equal(u, v) for u, v in zip(got, exp))
                xr = np.repeat(np.arange(n), np.diff(xp))    # the excluded entries are back after each call
                assert np.array_equal(_bits(rec.pairs(xr, xi)), _bits(D[xr, xi]))
                rec.exclude(None, None)
            cleared = {und: tuple(k for k in max_ks[und] if k >= 0) for und in (True, False)}
            _assert_same(_results(rec, indptr, indices, pi, pj, cleared),
                         {key: v for key, v in ref.items() if key[0] != 'top' or key[2] >= 0})


def test_sixteen_blocks_at_65536_nodes(gpu_ctx):
    from gem_b200 import _native
    n, d = 65536, 128
    rng = np.random.default_rng(65536)
    X = (rng.standard_normal((n, d)) * 0.3).astype(np.float32)
    key = np.unique(np.repeat(np.arange(n, dtype=np.int64), 12) * n + rng.integers(0, n, n * 12))
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, key // n + 1, 1)
    indptr, indices = np.cumsum(indptr), key % n
    out = []
    for ppb in (0, 64):
        with _native.Reconstruction(gpu_ctx, X, _native.RECON_SPLIT, panels_per_block=ppb) as rec:
            assert rec.blocks == (1 if ppb == 0 else 16)
            out.append((rec.ranks(indptr, indices, True), _top(rec, True, 1000)))
    (ra, ta), (rb, tb) = out
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
    assert all(np.array_equal(u, v) for u, v in zip(ta, tb))


class _FixedX:
    def __init__(self, X):
        self.X, self._recon_split = X, True

    def learn_embedding(self, graph=None, **kw):
        return self.X

    def get_embedding(self):
        return self.X


def _force_one_panel(monkeypatch):
    from gem_b200 import _native
    base = _native.Reconstruction

    class OnePanel(base):
        def __init__(self, ctx, X, kind):
            super().__init__(ctx, X, kind, panels_per_block=1)
    monkeypatch.setattr(_native, 'Reconstruction', OnePanel)


def _nx(n, indptr, indices, w):
    import networkx as nx
    G = nx.DiGraph()
    G.add_nodes_from(range(n))
    rows = np.repeat(np.arange(n), np.diff(indptr))
    G.add_weighted_edges_from(zip(rows.tolist(), indices.tolist(), w.tolist()))
    return G


@pytest.mark.parametrize('name', ['eval_karate_hope', 'eval_sbm1024_hope'])
def test_graph_reconstruction_forced_to_one_panel_per_block(gpu_ctx, monkeypatch, name):
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    z, n, (indptr, indices, w) = eval_golden(name)
    G = _nx(n, indptr, indices, w)
    m = _FixedX(z['X'])
    runs = []
    for forced in (False, True):
        if forced:
            _force_one_panel(monkeypatch)
        runs.append([evaluateStaticGraphReconstruction(G, m, z['X'], None, is_undirected=und, is_weighted=True, max_k=k)
                     for und in (True, False) for k in (100, 1000)])
    for a, b in zip(*runs):
        assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2] and a[3] == b[3]
    if n > 64:                                               # more than one panel: the forced handle has blocks
        with pytest.raises(ValueError, match='max_k'):
            evaluateStaticGraphReconstruction(G, m, z['X'], None)


@pytest.mark.parametrize('name', ['linkpred_karate_hope', 'linkpred_sbm1024_hope'])
def test_link_prediction_forced_to_one_panel_per_block(gpu_ctx, monkeypatch, name):
    from gem_b200 import graph as hg
    from gem_b200.evaluation.evaluate_link_prediction import evaluateStaticLinkPrediction
    z = np.load(golden_path(name + '.npz'))
    n, e = int(z['n']), z['edges']
    C = hg.from_edges(n, e[:, 0].astype(np.int64), e[:, 1].astype(np.int64), e[:, 2])
    X = np.random.default_rng(n).standard_normal((n, 16)).astype(np.float32) * 0.5
    kw = dict(train_ratio=float(z['train_ratio']), is_undirected=bool(z['is_undirected']), seed=int(z['seed']))
    runs = []
    for forced in (False, True):
        if forced:
            _force_one_panel(monkeypatch)
        runs.append([evaluateStaticLinkPrediction(C, _FixedX(X), max_k=k, **kw) for k in (100, 1000)])
    assert runs[0] == runs[1]
    if n > 64:
        with pytest.raises(ValueError, match='max_k'):
            evaluateStaticLinkPrediction(C, _FixedX(X), **kw)


def test_blocked_handles_own_their_device_blocks(gpu_ctx, native_lib):
    from gem_b200 import _native
    rng, X, indptr, indices = _inputs(1, 1000)
    live = native_lib.gemb_mem_live_blocks()
    with _native.Reconstruction(gpu_ctx, X, 1, panels_per_block=3) as rec:
        assert native_lib.gemb_mem_live_blocks() > live
        rec.exclude(indptr, indices)
        rec.dense()
        rec.pairs(np.arange(10), np.arange(10, 20))
        rec.ranks(indptr, indices, True)
        rec.top(True, 50)
        with pytest.raises(RuntimeError, match='out of range'):
            rec.ranks(indptr, np.where(np.arange(indices.size) == 5, 1000, indices), True)
        with pytest.raises(RuntimeError, match='out of range'):
            rec.pairs(np.array([0]), np.array([1000]))
        with pytest.raises(RuntimeError, match='ascending'):
            rec.exclude(indptr, indices[::-1].copy())
    assert native_lib.gemb_mem_live_blocks() == live
    with pytest.raises(RuntimeError, match='panels_per_block'):
        _native.Reconstruction(gpu_ctx, X, 1, panels_per_block=-1)
    assert native_lib.gemb_mem_live_blocks() == live


def test_two_blocked_runs_are_identical(gpu_ctx):
    from gem_b200 import _native
    _, X, indptr, indices = _inputs(2, 4200)
    runs = []
    for _ in range(2):
        with _native.Reconstruction(gpu_ctx, X, 2, panels_per_block=7) as rec:
            runs.append((rec.ranks(indptr, indices, False), _top(rec, False, 1000)))
    (ra, ta), (rb, tb) = runs
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
    assert all(np.array_equal(u, v) for u, v in zip(ta, tb))
