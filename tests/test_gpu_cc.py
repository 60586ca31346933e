"""Weakly connected components on the GPU (gemb_cc_*, get_lcc on a HostCSR) and link prediction with lcc=True.

  1. labels equal oracle/cc_oracle.py (scipy) exactly, the LCC's CSR equals the oracle's bit for bit (fp64 weights,
     `nodes`, node_l), and two runs give the same bits -- on the goldens, 2^20-vertex paths in three numberings, a
     2^22-vertex path in the zigzag numbering that makes linking by index build Theta(n)-deep chains (with and without
     chords that walk them again; its labelling must stay under a second), a star with 2^20 leaves both ways round,
     self loops only, no edges, n = 0 and 1, device R-MAT at scale 20 and the 1M-node SBM;  get_lcc on a HostCSR and on
     the same networkx graph keep the same component with the same edges, in the same order when it is the majority;
  2. bad input is rejected, and no device block is left behind after a success or a rejected call;
  3. link prediction: lcc=True is bit-identical to lcc=False on a training graph that is one component; on the LCC
     goldens (fixed dyadic X: every score exact in fp32) MAP equals the reference's and the oracle's to 1e-12, the
     precision curve equals the oracle's, and HostCSR and networkx inputs give identical results.
"""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, golden_path
from test_oracle_cc import LP_CASES, nx_graph, positions

sys.path.insert(0, os.path.join(REPO, 'oracle'))
import cc_oracle as co  # noqa: E402

pytestmark = pytest.mark.gpu


def _check(ctx, n, indptr, indices, data=None, nodes=None, symmetric=None):
    """Device against oracle, twice; get_lcc(HostCSR) against the oracle.  -> the oracle's labels"""
    from gem_b200 import _native
    from gem_b200.graph import HostCSR
    from gem_b200.utils.graph_util import get_lcc
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int32)
    lab = co.labels(n, indptr, indices)
    runs = []
    for _ in range(2):
        with _native.Components(ctx, n, indptr, indices) as cc:
            runs.append((cc.labels(), cc.lcc(data), (cc.n_comp, cc.lcc_root, cc.lcc_size, cc.lcc_nnz)))
    (l1, lcc1, info1), (l2, lcc2, info2) = runs
    assert np.array_equal(l1, lab) and np.array_equal(l1, l2) and info1 == info2
    if n == 0:
        assert info1 == (0, -1, 0, 0) and lcc1[0].size == 0 and lcc1[1].tolist() == [0]
        return lab
    exp = co.lcc_csr(n, indptr, indices, data, lab)
    assert info1 == (int(lab.max()) + 1, int(exp[0][0]), exp[0].size, exp[2].size)
    for got, again, want in zip(lcc1, lcc2, exp):
        if want is None:
            assert got is None and again is None
            continue
        assert got.dtype == want.dtype and np.array_equal(got, want) and np.array_equal(got, again)
        if got.dtype == np.float64:
            assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    H, node_l = get_lcc(HostCSR(n, indptr, indices, data, nodes=nodes, symmetric=symmetric))
    assert np.array_equal(node_l, exp[0]) and H.n == exp[0].size and H.symmetric == symmetric
    assert np.array_equal(H.indptr, exp[1]) and np.array_equal(H.indices, exp[2])
    assert (H.data is None and exp[3] is None) or np.array_equal(H.data, exp[3])
    if nodes is not None:
        assert list(H.nodes) == [nodes[i] for i in exp[0]]
    return lab


@pytest.mark.parametrize('name', ['cc_karate_s2', 'cc_rmat12', 'cc_tie', 'cc_oneway'])
def test_goldens(gpu_ctx, name):
    z = np.load(golden_path(name + '.npz'))
    n, indptr, indices, w, _ = positions(z)
    lab = _check(gpu_ctx, n, indptr, indices, w, nodes=z['nodes'].tolist())
    assert np.array_equal(lab, z['labels'])
    # the networkx path: the same nodes and edges; its map is in row order when the component holds half the graph
    # or more, and in the component set's iteration order otherwise (the reference recipe's networkx subgraph view)
    from gem_b200.graph import HostCSR
    from gem_b200.utils.graph_util import get_lcc
    Hc, node_l = get_lcc(HostCSR(n, indptr, indices, w, nodes=z['nodes'].tolist()))
    Hn, m = get_lcc(nx_graph(z))
    assert sorted(m) == sorted(Hc.nodes) and Hn.number_of_edges() == Hc.nnz
    if 2 * node_l.size >= n:
        assert list(m) == list(Hc.nodes)
    label_of = list(m)
    rows = np.repeat(np.arange(Hc.n), np.diff(Hc.indptr))
    ec = sorted(zip((Hc.nodes[i] for i in rows), (Hc.nodes[j] for j in Hc.indices), Hc.data.tolist()))
    en = sorted((label_of[u], label_of[v], wt) for u, v, wt in Hn.edges(data='weight'))
    assert ec == en


def _one_way(n, src, dst):
    return co.csr_of_edges(n, src, dst)


@pytest.mark.parametrize('order', ['forward', 'reverse', 'random'])
def test_path_of_2_20(gpu_ctx, order):
    n = 1 << 20
    ids = np.arange(n)
    if order == 'reverse':
        ids = ids[::-1].copy()
    elif order == 'random':
        ids = np.random.default_rng(1).permutation(n)
    lab = _check(gpu_ctx, n, *_one_way(n, ids[:-1], ids[1:]))
    assert lab.max() == 0


def _zigzag(n, chords):
    """A path numbered h, h-1, h+1, h-2, h+2, ... (h = n // 2): the component's minimum keeps falling as the rows
    advance, so linking by index alone builds a chain of depth ~n / 2.  chords: one more edge from every row h + t to
    h, which makes every hook walk that chain again when finds do not shorten it (Theta(n^2) in total)."""
    h = n // 2
    t = np.arange(1, h + 1)
    s = np.empty(n, dtype=np.int64)
    s[0] = h
    s[1::2] = h - t[:n // 2]
    s[2::2] = (h + t)[:(n - 1) // 2]
    src, dst = s[:-1], s[1:]
    if chords:
        up = np.arange(h + 1, n)
        src, dst = np.concatenate((src, up)), np.concatenate((dst, np.full(up.size, h)))
    return n, src, dst


@pytest.mark.parametrize('chords', [False, True])
def test_zigzag_numbering_stays_linear(gpu_ctx, chords):
    """The adversarial numbering of _zigzag at 2^22 vertices: exact labels and LCC, and the labelling takes well under a
    second (without path halving its finds would make ~10^12 dependent reads)."""
    from gem_b200 import _native
    n, src, dst = _zigzag(1 << 22, chords)
    assert np.array_equal(np.sort(np.unique(np.concatenate((src, dst)))), np.arange(n))
    indptr, indices = _one_way(n, src, dst)
    lab = _check(gpu_ctx, n, indptr, indices)
    assert lab.max() == 0
    with _native.Components(gpu_ctx, n, indptr, indices) as cc:
        label_ms, _ = cc.times()
    assert label_ms < 1000.0, label_ms


@pytest.mark.parametrize('inward', [False, True])
def test_star_with_2_20_leaves(gpu_ctx, inward):
    n = (1 << 20) + 1
    hub = n // 2
    leaves = np.delete(np.arange(n), hub)
    hubs = np.full(leaves.size, hub)
    src, dst = (leaves, hubs) if inward else (hubs, leaves)
    lab = _check(gpu_ctx, n, *_one_way(n, src, dst))
    assert lab.max() == 0


def test_degenerate_graphs(gpu_ctx):
    n = 5000
    lab = _check(gpu_ctx, n, np.arange(n + 1), np.arange(n), data=np.linspace(0.5, 2.0, n))     # self loops only
    assert lab.tolist() == list(range(n))
    lab = _check(gpu_ctx, n, np.zeros(n + 1), np.zeros(0))                                      # no edges
    assert lab.tolist() == list(range(n))
    _check(gpu_ctx, 1, [0, 0], [])
    _check(gpu_ctx, 1, [0, 1], [0], data=np.array([3.5]))
    _check(gpu_ctx, 0, [0], [])


def test_device_rmat_scale_20(gpu_ctx):
    from gem_b200 import _native
    indptr, indices, _ = _native.synth_rmat(gpu_ctx, 20, permute=True)
    data = np.random.default_rng(4).uniform(0.1, 2.0, indices.size)
    lab = _check(gpu_ctx, 1 << 20, indptr, indices, data, symmetric=True)
    assert lab.max() > 1000


def test_sbm_1m_is_one_component(gpu_ctx):
    from gem_b200 import synth
    csr = synth.sbm(n=1_000_000, block=1000, seed=42)
    lab = _check(gpu_ctx, csr.n, csr.indptr, csr.indices, symmetric=True)
    assert lab.max() == 0


def test_rejected_input_and_no_leak(gpu_ctx, native_lib):
    from gem_b200 import _native
    live = native_lib.gemb_mem_live_blocks()
    with _native.Components(gpu_ctx, 4, [0, 1, 2, 2, 3], [1, 0, 3]) as cc:
        cc.labels(), cc.lcc(np.ones(3))
    assert native_lib.gemb_mem_live_blocks() == live
    for indptr, indices in (([0, 2, 1, 3, 3], [1, 0, 3]),      # non-monotone
                            ([1, 1, 2, 2, 3], [1, 0, 3]),      # indptr[0] != 0
                            ([0, 1, 2, 2, 3], [1, 0, 4]),      # column id = n
                            ([0, 1, 2, 2, 3], [1, -1, 3])):    # negative column id
        with pytest.raises(RuntimeError, match='bad argument'):
            _native.Components(gpu_ctx, 4, indptr, indices)
        assert native_lib.gemb_mem_live_blocks() == live


class FixedX:
    """A model whose learn_embedding returns a given X with a reference score."""

    def __init__(self, X, split):
        self.X, self._recon_split = X, split

    def learn_embedding(self, graph=None, **kw):
        return self.X


def test_lcc_is_bit_identical_on_one_component(gpu_ctx, native_lib):
    from gem_b200 import graph as hg
    from gem_b200.evaluation.evaluate_link_prediction import evaluateStaticLinkPrediction
    z = np.load(golden_path('linkpred_sbm1024_hope.npz'))
    n, e = int(z['n']), z['edges']
    G = nx_graph(dict(nodes=np.arange(n), edges=e))
    C = hg.from_edges(n, e[:, 0].astype(np.int64), e[:, 1].astype(np.int64), e[:, 2])
    kw = dict(train_ratio=float(z['train_ratio']), is_undirected=True, seed=int(z['seed']))
    for g in (G, C):
        a = evaluateStaticLinkPrediction(g, FixedX(z['X'], True), **kw)
        b = evaluateStaticLinkPrediction(g, FixedX(z['X'], True), lcc=True, **kw)
        assert np.float64(a[0]).tobytes() == np.float64(b[0]).tobytes() and a[1] == b[1]


@pytest.mark.parametrize('name', LP_CASES)
def test_link_prediction_on_lcc_goldens(gpu_ctx, native_lib, name):
    from gem_b200 import _native
    from gem_b200 import graph as hg
    from gem_b200.evaluation.evaluate_link_prediction import evaluateStaticLinkPrediction
    z = np.load(golden_path(name + '.npz'))
    e, und, split = z['edges'], bool(z['is_undirected']), str(z['score']) == 'split'
    kw = dict(train_ratio=float(z['train_ratio']), is_undirected=und, seed=int(z['seed']), lcc=True)
    live = native_lib.gemb_mem_live_blocks()
    MAP, prec = evaluateStaticLinkPrediction(nx_graph(z), FixedX(z['X'], split), **kw)
    assert native_lib.gemb_mem_live_blocks() == live
    assert abs(MAP - float(z['MAP'])) < 1e-12, (MAP, float(z['MAP']))
    r = co.linkpred_lcc(e[:, 0], e[:, 1], z['nodes'], z['X'], str(z['score']), int(z['seed']), float(z['train_ratio']),
                        und)
    assert abs(MAP - r['MAP']) < 1e-12
    assert np.array_equal(np.array(prec), r['prec_curve'])
    with _native.Reconstruction(gpu_ctx, z['X'], int(split)) as rec:     # every score exact: the fp64 matrix itself
        assert np.array_equal(rec.dense().astype(np.float64), co.eo.reconstruct(z['X'], split, exact=False)
                              * (1 - np.eye(z['X'].shape[0])))
    if np.array_equal(z['nodes'], np.arange(int(z['n']))):                # row-major edge order: the same draws
        C = hg.from_edges(int(z['n']), e[:, 0].astype(np.int64), e[:, 1].astype(np.int64), e[:, 2])
        MAP_c, prec_c = evaluateStaticLinkPrediction(C, FixedX(z['X'], split), **kw)
        assert MAP_c == MAP and prec_c == prec
