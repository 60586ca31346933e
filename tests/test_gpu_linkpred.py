"""Link prediction on the GPU: the exclusion set of gemb_recon_exclude and evaluateStaticLinkPrediction.

  1. ranks, n_pred_row and top-k with an exclusion set are BIT-EXACT against oracle/linkpred_oracle.py run on the
     matrix the GPU produced (for the Gaussian kind: on the order keys the device stores, which order as the score),
     and dense / pairs still return the unmasked values while the exclusion is set;
  2. an empty exclusion, and a cleared one, give exactly what the calls give without one;
  3. end to end with the repository's HOPE / LaplacianEigenmaps on the golden graphs and seeds: the split and the
     sample are the reference's, MAP is within 2e-3 of the reference's (the bar of test_gpu_recon.py), HostCSR and
     networkx inputs give identical results, and no device block is left behind.
"""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, golden_path

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import eval_oracle as eo  # noqa: E402
import linkpred_oracle as lo  # noqa: E402

pytestmark = pytest.mark.gpu

GAUSS_DELTA_MAX = 0x443a4886


def _keys(D):
    """delta (dense of the Gaussian kind) -> the order key the device stores: bits 0x7f800000 - bits(delta), 0 past
    745.1332f and on the diagonal (delta = +inf)."""
    b = np.ascontiguousarray(D, dtype=np.float32).view(np.uint32)
    k = np.where(b <= GAUSS_DELTA_MAX, np.uint32(0x7f800000) - b, np.uint32(0)).astype(np.uint32)
    return k.view(np.float32).astype(np.float64)


def _csr(n, keys):
    keys = np.unique(np.asarray(keys, dtype=np.int64))
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, keys // n + 1, 1)
    return np.cumsum(indptr), keys % n


def _case(rng, n, A, und):
    """Test and train CSRs (disjoint but for a few edges in both) built to hit the corners: excluded entries tied with
    held-out edges (duplicated rows), the max_k = 1 and 1000 thresholds excluded, one row with every candidate
    excluded, held-out edges that are themselves excluded."""
    test = rng.integers(0, n, (n * 6, 2))
    train = rng.integers(0, n, (n * 10, 2))
    test_k = test[:, 0] * n + test[:, 1]
    train_k = train[:, 0] * n + train[:, 1]
    train_k = train_k[~np.isin(train_k, test_k)]
    extra = []
    for i in range(0, 60, 3):                            # rows 100..149 duplicate 0..49: a[i][j] == a[i][j + 100]
        j = int(rng.integers(0, 50))
        test_k = np.append(test_k, i * n + j)
        extra.append(i * n + j + 100)
    i, j, w = eo.edge_list_from_adj(A, is_undirected=und)
    order = np.argsort(-w, kind='stable')
    for pos in (0, 1, 999, 1000):                        # around the thresholds of max_k = 1 and 1000
        extra.append(int(i[order[pos]]) * n + int(j[order[pos]]))
    r = 7
    extra += [r * n + c for c in range(n) if c != r]     # every candidate of row 7
    test_k = np.append(test_k, [r * n + 8, r * n + 4000])
    both = test_k[:5]                                    # held-out edges that are also excluded
    train_k = np.concatenate((train_k, extra, both))
    return _csr(n, test_k), _csr(n, train_k)


@pytest.mark.parametrize('kind,n,d', [(1, 4500, 32), (0, 4200, 64), (2, 5000, 8)])
def test_ranks_and_top_with_exclusion_exact(gpu_ctx, kind, n, d):
    from gem_b200 import _native
    rng = np.random.default_rng(n + kind)
    X = (rng.standard_normal((n, d)) * (0.3 if kind != 2 else 0.6)).astype(np.float32)
    X[:50] = np.round(X[:50], 1)
    X[100:150] = X[0:50]                                 # duplicated rows: exact ties
    with _native.Reconstruction(gpu_ctx, X, kind) as rec:
        D = rec.dense()
        A = _keys(D) if kind == 2 else D.astype(np.float64)
        for und in (True, False):
            (tp, ti_), (xp, xi) = _case(rng, n, A, und)
            test, train = eo.EdgeSet(n, tp, ti_), eo.EdgeSet(n, xp, xi)
            base_r, base_np = rec.ranks(tp, ti_, und)
            base_top = rec.top(und, 1000)
            rec.exclude(xp, xi)
            ranks, n_pred_row = rec.ranks(tp, ti_, und)
            exp_r, exp_np = lo.ranks(A, test, train, und)
            assert np.array_equal(n_pred_row, exp_np)
            assert np.array_equal(ranks, exp_r)
            assert n_pred_row[7] == 0 and np.all(ranks[tp[7]:tp[8]] == 0)
            rows = np.repeat(np.arange(n), np.diff(tp))
            assert np.all(ranks[train.has_edge(rows, ti_)] == 0)          # held-out edges that are excluded
            i, j, w = lo.filtered(*eo.edge_list_from_adj(A, is_undirected=und), train)
            vals = np.sort(w)[::-1]
            for max_k in (-1, 0, 1, 1000):
                ti, tj, tw = rec.top(und, max_k)
                if max_k == 0:
                    assert ti.size == 0
                    continue
                sel = np.ones(w.size, dtype=bool) if max_k == -1 else w >= vals[max_k - 1]
                assert ti.size == int(sel.sum())
                got = np.sort(ti.astype(np.int64) * n + tj)
                assert np.array_equal(got, np.sort(i[sel] * n + j[sel]))
                assert np.array_equal(tw, D[ti, tj])
            # ranks and top zero the excluded entries only while they run: dense and pairs see the plain values
            assert np.array_equal(rec.dense().view(np.uint32), D.view(np.uint32))
            xr = np.repeat(np.arange(n), np.diff(xp))
            assert np.array_equal(rec.pairs(xr, xi).view(np.uint32), D[xr, xi].view(np.uint32))
            # clearing gives back the plain results
            rec.exclude(None, None)
            r2, np2 = rec.ranks(tp, ti_, und)
            assert np.array_equal(r2, base_r) and np.array_equal(np2, base_np)
            t2 = rec.top(und, 1000)
            assert all(np.array_equal(np.sort(a), np.sort(b)) for a, b in zip(t2, base_top))


def test_empty_exclusion_is_no_exclusion(gpu_ctx):
    from gem_b200 import _native
    rng = np.random.default_rng(3)
    n = 700
    X = np.round(rng.standard_normal((n, 16)), 1).astype(np.float32)
    tp, ti_ = _csr(n, rng.integers(0, n * n, n * 8))
    for kind in (0, 1, 2):
        with _native.Reconstruction(gpu_ctx, X, kind) as rec:
            for und in (True, False):
                base = rec.ranks(tp, ti_, und), [rec.top(und, k) for k in (-1, 1, 1000)]
                rec.exclude(np.zeros(n + 1, dtype=np.int32), np.zeros(0, dtype=np.int32))
                got = rec.ranks(tp, ti_, und), [rec.top(und, k) for k in (-1, 1, 1000)]
                rec.exclude(None, None)
                for a, b in zip(base[0], got[0]):
                    assert np.array_equal(a, b)
                for ta, tb in zip(base[1], got[1]):
                    oa = np.lexsort((ta[1], ta[0])); ob = np.lexsort((tb[1], tb[0]))
                    assert all(np.array_equal(x[oa], y[ob]) for x, y in zip(ta, tb))


class FixedX:
    """A model whose learn_embedding returns a given X (the golden's random X) with a reference score."""

    def __init__(self, X, split):
        self.X, self._recon_split = X, split

    def learn_embedding(self, graph=None, **kw):
        return self.X


def _make(name, z):
    if 'randw200' in name:
        return FixedX(z['X'], str(z['score']) == 'split')
    if name.endswith('lap'):
        from gem_b200.embedding.lap import LaplacianEigenmaps as C
        C.hyper_params.clear(); C.hyper_params.update({'method_name': 'lap_eigmap_svd'})
        return C(d=z['X'].shape[1])
    from gem_b200.embedding.hope import HOPE
    HOPE.hyper_params.clear(); HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
    return HOPE(d=z['X'].shape[1], beta=0.01, max_iters=500)      # converged: compared with the reference's exact SVD


@pytest.mark.parametrize('name', ['linkpred_karate_hope', 'linkpred_sbm1024_hope', 'linkpred_sbm1024_hope_s300',
                                  'linkpred_randw200_dot', 'linkpred_randw200_split', 'linkpred_sbm1024_lap'])
def test_end_to_end_against_reference(gpu_ctx, native_lib, name):
    import networkx as nx
    from gem_b200 import graph as hg
    from gem_b200.evaluation.evaluate_link_prediction import evaluateStaticLinkPrediction, split_and_sample
    z = np.load(golden_path(name + '.npz'))
    n, e, und, s = int(z['n']), z['edges'], bool(z['is_undirected']), int(z['n_sample'])
    seed, ratio = int(z['seed']), float(z['train_ratio'])
    G = nx.DiGraph()
    G.add_nodes_from(range(n))
    G.add_weighted_edges_from((int(a), int(b), float(w)) for a, b, w in e)
    C = hg.from_edges(n, e[:, 0].astype(np.int64), e[:, 1].astype(np.int64), e[:, 2])
    tr, te, _, node_l = split_and_sample(G, ratio, s or None, und, np.random.RandomState(seed))
    assert np.array_equal(np.array(list(tr.edges(data='weight'))).reshape(-1, 3), z['train_edges'])
    if not s:
        assert np.array_equal(np.array(list(te.edges(data='weight'))).reshape(-1, 3), z['test_edges'])
    assert np.array_equal(node_l, z['node_l'])
    live = native_lib.gemb_mem_live_blocks()
    kw = dict(train_ratio=ratio, n_sample_nodes=s or None, is_undirected=und, seed=seed)
    MAP, prec = evaluateStaticLinkPrediction(G, _make(name, z), **kw)
    MAP_c, prec_c = evaluateStaticLinkPrediction(C, _make(name, z), **kw)
    assert native_lib.gemb_mem_live_blocks() == live
    assert MAP == MAP_c and prec == prec_c
    assert abs(MAP - float(z['MAP'])) < 2e-3, (MAP, float(z['MAP']))
    h = min(len(prec), 200)
    assert np.mean(np.abs(np.array(prec[:h]) - z['prec_head'][:h])) < 0.05
    MAP_k, prec_k = evaluateStaticLinkPrediction(C, _make(name, z), max_k=100, **kw)
    assert prec_k == prec[:100] and MAP_k == MAP
