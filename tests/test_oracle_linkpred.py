"""oracle/linkpred_oracle.py pinned against the reference's own functions (goldens made by
tests/golden/make_golden_linkpred.py): split, node_l, filtered list, precision curve and MAP exact given the golden X;
its vectorised forms against the statement-by-statement loops; and the identity the device's exclusion relies on:
filtering out the training edges is setting their entries to 0."""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, golden_path
from test_gpu_linkpred import _case

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import eval_gauss_oracle as go  # noqa: E402
import eval_oracle as eo  # noqa: E402
import linkpred_oracle as lo  # noqa: E402

CASES = ['linkpred_karate_hope', 'linkpred_sbm1024_hope', 'linkpred_sbm1024_hope_s300', 'linkpred_randw200_dot',
         'linkpred_randw200_split', 'linkpred_sbm1024_lap']


def oracle_inputs(z):
    """Steps 1-3 of the oracle with the golden's seed and X: split, sample, reconstruct.
    -> (adj of the sample, test and train EdgeSet of the sample, train and test masks of the edges, node_l)"""
    n = int(z['n'])
    e = z['edges']
    src, dst = e[:, 0].astype(np.int64), e[:, 1].astype(np.int64)
    und = bool(z['is_undirected'])
    rng = np.random.RandomState(int(z['seed']))
    tr, te = lo.split(src, dst, float(z['train_ratio']), und, rng)
    s = int(z['n_sample'])
    node_l = rng.choice(n, s, replace=False) if s and n > s else np.arange(n)
    ns = len(node_l)
    ktr, utr, vtr = lo.induce(src[tr], dst[tr], n, node_l)
    kte, ute, vte = lo.induce(src[te], dst[te], n, node_l)
    Xs = z['X'][node_l]
    score = str(z['score'])
    adj = go.reconstruct_gaussian(Xs) if score == 'gaussian' else eo.reconstruct(Xs, score == 'split')
    return adj, lo.edge_set(ns, ute, vte), lo.edge_set(ns, utr, vtr), tr, te, node_l


def oracle_run(z):
    """Steps 1-6 of the oracle with the golden's seed and X.  -> dict"""
    adj, test, train, tr, te, node_l = oracle_inputs(z)
    r = lo.evaluate(adj, test, train, is_undirected=bool(z['is_undirected']))
    r.update(train=z['edges'][tr], test=z['edges'][te], node_l=node_l)
    return r


@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_reference_link_prediction(name):
    z = np.load(golden_path(name + '.npz'))
    r = oracle_run(z)
    assert np.array_equal(r['train'], z['train_edges']) and np.array_equal(r['test'], z['test_edges'])
    assert np.array_equal(r['node_l'], z['node_l'])
    assert r['n_pred'] == int(z['n_pred'])
    assert abs(r['MAP'] - float(z['MAP'])) < 1e-13
    assert np.array_equal(r['prec_curve'][:4096], z['prec_head'])
    assert np.array_equal(r['prec_curve'][::997], z['prec_stride'])


def _assert_zeroing_is_filtering(adj, test, train, und):
    """What gemb_recon_ranks / _top rely on: an entry that holds 0 is not a candidate, so ranks, n_pred_row and the
    candidate list among the candidates not in train equal those on adj with the entries of train set to 0 and no
    exclusion."""
    masked = np.array(adj, dtype=np.float64)
    masked[np.repeat(np.arange(train.n), np.diff(train.indptr)), train.indices] = 0
    none = lo.edge_set(train.n, [], [])
    for got, exp in zip(lo.ranks(masked, test, none, und), lo.ranks(adj, test, train, und)):
        assert np.array_equal(got, exp)
    full = eo.edge_list_from_adj(adj, is_undirected=und)
    kept = lo.filtered(*full, train)
    assert kept[0].size < full[0].size
    for got, exp in zip(eo.edge_list_from_adj(masked, is_undirected=und), kept):
        assert np.array_equal(got, exp)


@pytest.mark.parametrize('name', CASES)
def test_zeroed_training_entries_are_the_filter_on_goldens(name):
    z = np.load(golden_path(name + '.npz'))
    adj, test, train = oracle_inputs(z)[:3]
    _assert_zeroing_is_filtering(adj, test, train, bool(z['is_undirected']))


@pytest.mark.parametrize('und', [True, False])
@pytest.mark.parametrize('kind', [0, 1, 2])
def test_zeroed_training_entries_are_the_filter_on_corner_cases(kind, und):
    """_case's corners: excluded entries tied with held-out ones, excluded entries at the max_k = 1 and 1000
    thresholds, a row with every candidate excluded, held-out edges that are excluded."""
    n = 500 + 100 * kind
    rng = np.random.default_rng(n + kind)
    X = rng.standard_normal((n, 16)) * (0.3 if kind != 2 else 0.6)
    X[:50] = np.round(X[:50], 1)
    X[100:150] = X[0:50]                                 # duplicated rows: exact ties
    adj = go.reconstruct_gaussian(X, exact=False) if kind == 2 else eo.reconstruct(X, kind == 1, exact=False)
    (tp, ti), (xp, xi) = _case(rng, n, adj, und)
    _assert_zeroing_is_filtering(adj, eo.EdgeSet(n, tp, ti), eo.EdgeSet(n, xp, xi), und)


def _graph(rng, n, m, sym):
    e = {}
    while len(e) < m:
        u, v = (int(x) for x in rng.integers(0, n, 2))
        e[(u, v)] = float(np.round(rng.uniform(0.1, 2.0), 2))
        if sym:
            e[(v, u)] = e[(u, v)]
    return sorted((u, v, w) for (u, v), w in e.items())


@pytest.mark.parametrize('und', [True, False])
def test_vectorised_forms_equal_the_loops(und):
    rng = np.random.default_rng(21)
    n = 50
    edges = _graph(rng, n, 300, und)
    src = np.array([a for a, _, _ in edges]); dst = np.array([b for _, b, _ in edges])
    trl, tel = lo.split_loops(edges, 0.7, und, np.random.RandomState(4))
    tr, te = lo.split(src, dst, 0.7, und, np.random.RandomState(4))
    assert [edges[k] for k in np.flatnonzero(tr)] == trl and [edges[k] for k in np.flatnonzero(te)] == tel
    if und:
        assert any(a == b for a, b, _ in trl) == any(a == b for a, b, _ in edges)     # self-loops stay in both
        with pytest.raises(KeyError):
            lo.split_loops([(0, 1, 1.0)], 0.5, True, np.random.RandomState(0))
        with pytest.raises(KeyError):
            lo.split(np.array([0]), np.array([1]), 0.5, True, np.random.RandomState(0))
    sl, node_l = lo.sample_loops(tel, n, 20, np.random.RandomState(8))
    assert np.array_equal(node_l, np.random.RandomState(8).choice(n, 20, replace=False))
    keep, u, v = lo.induce(src[te], dst[te], n, node_l)
    assert [(a, b) for a, b, _ in sl] == list(zip(u.tolist(), v.tolist()))
    trs, _ = lo.sample_loops(trl, n, 20, None, node_l=node_l)
    X = np.round(rng.standard_normal((20, 4)), 1)                  # coarse values: exact ties
    adj = eo.reconstruct(X, True)
    pred = eo.edge_list_from_adj_loops(adj, is_undirected=und)
    fl = lo.filtered_loops(pred, trs)
    ku, kv = lo.induce(src[tr], dst[tr], n, node_l)[1:]
    train = lo.edge_set(20, ku, kv)
    i, j, w = lo.filtered(*eo.edge_list_from_adj(adj, is_undirected=und), train)
    assert [(a, b) for a, b, _ in fl] == list(zip(i.tolist(), j.tolist()))
    import networkx as nx
    T = nx.DiGraph()
    T.add_nodes_from(range(20))
    T.add_edges_from((a, b) for a, b, _ in sl)
    r = lo.evaluate(adj, lo.edge_set(20, u, v), train, is_undirected=und)
    assert abs(eo.compute_map_loops(fl, T) - r['MAP']) < 1e-15
    assert np.array_equal(np.array(eo.precision_curve_loops(fl, T)[0]), r['prec_curve'])
