"""The host plumbing the embedding classes and the evaluation share, on CPU: fakes of the _native handles record that
every per-call context is closed and every device graph freed, whether the solve returns or raises; the unconverged
step warns at the caller's line or raises under strict; evaluateStaticGraphReconstruction, run on a NumPy
reconstruction, reproduces the reference goldens (full branch) and metrics.computeMAP / computePrecisionCurve of the
same kept pair list (sampled branch)."""
import networkx as nx
import numpy as np
import pytest

from conftest import eval_golden
from test_host_eval import _emulated_kernel_outputs


class FakeSolveError(RuntimeError):
    pass


class _FakeHandle:
    released = False

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self._release()

    def _release(self):
        self.released = True


@pytest.fixture
def fake_native(monkeypatch):
    """Replaces _native.Context / DeviceGraph / graph_factorization; `log` lists every handle made, `cfg` sets whether
    the solve raises and whether it reports convergence."""
    from gem_b200 import _native
    log, cfg = [], {'fail': False, 'converged': 1, 'svd_error_probes': []}

    class Context(_FakeHandle):
        def __init__(self, device=0):
            log.append(self)
        close = _FakeHandle._release

    class DeviceGraph(_FakeHandle):
        def __init__(self, ctx, n, indptr, indices, data=None, indptr_t=None, indices_t=None, data_t=None, row0=0):
            assert not ctx.released
            self.n = int(n)
            log.append(self)
        free = _FakeHandle._release

        def hope(self, d, beta, out=None, want_output=True, **opts):
            if cfg['fail']:
                raise FakeSolveError('fake solve failed')
            st = {'converged': cfg['converged'], 'iters': 7, 'ritz_change': 0.25, 'beta_used': 0.0}
            return np.zeros((self.n, d), np.float32) if out is None else out, np.zeros(d, np.float32), st

        def hope_svd_error(self, d, beta, X, n_probe=0, seed=1):
            cfg['svd_error_probes'].append(n_probe)
            return 0.0

        def node2vec(self, nids, d, walk_len, num_walks, con_size, max_iter, p=1.0, q=1.0, seed=1, sequential=False,
                     n_rows=None, weights64=None, out=None, want_output=True):
            if cfg['fail']:
                raise FakeSolveError('fake solve failed')
            return np.zeros((n_rows, d), np.float32), {}

    def graph_factorization(ctx, n, src, dst, w, d, eta, regu, max_iter, X0, mode=0):
        assert not ctx.released
        if cfg['fail']:
            raise FakeSolveError('fake solve failed')
        return np.zeros((n, d), np.float32), 0.0

    monkeypatch.setattr(_native, 'Context', Context)
    monkeypatch.setattr(_native, 'DeviceGraph', DeviceGraph)
    monkeypatch.setattr(_native, 'graph_factorization', graph_factorization)
    return log, cfg


def _model(name, **extra):
    """A fresh model; settings go in through a positional dict so that the class-level hyper_params stay untouched."""
    from gem_b200.embedding.gf import GraphFactorization
    from gem_b200.embedding.hope import HOPE
    from gem_b200.embedding.lap import LaplacianEigenmaps
    from gem_b200.embedding.lle import LocallyLinearEmbedding
    from gem_b200.embedding.node2vec import node2vec
    make = {'HOPE': lambda: HOPE({'d': 4, 'beta': 0.01}),
            'LaplacianEigenmaps': lambda: LaplacianEigenmaps({'d': 2}),
            'LocallyLinearEmbedding': lambda: LocallyLinearEmbedding({'d': 2}),
            'GraphFactorization': lambda: GraphFactorization({'d': 2, 'eta': 1e-3, 'regu': 1.0, 'max_iter': 5}),
            'node2vec': lambda: node2vec({'d': 4, 'max_iter': 1, 'walk_len': 5, 'num_walks': 2, 'con_size': 2,
                                          'ret_p': 1.0, 'inout_p': 1.0})}[name]
    m = make()
    for k, v in extra.items():
        setattr(m, '_' + k, v)
    return m


def _graph():
    G = nx.DiGraph()
    G.add_nodes_from(range(8))
    G.add_edges_from((i, (i + 1) % 8) for i in range(8))
    G.add_edges_from([(0, 4), (5, 2)])
    return G


ALL = ['HOPE', 'LaplacianEigenmaps', 'LocallyLinearEmbedding', 'GraphFactorization', 'node2vec']
ITERATIVE = ['HOPE', 'LaplacianEigenmaps', 'LocallyLinearEmbedding']


@pytest.mark.parametrize('name', ALL)
def test_handles_are_released_after_success_and_failure(fake_native, name):
    log, cfg = fake_native
    X = _model(name).learn_embedding(graph=_graph())
    assert X.shape[0] == 8 and X.dtype == np.float32
    assert log and all(h.released for h in log)
    n_ok = len(log)
    cfg['fail'] = True
    with pytest.raises(FakeSolveError):
        _model(name).learn_embedding(graph=_graph())
    assert len(log) == 2 * n_ok and all(h.released for h in log)


@pytest.mark.parametrize('name', ALL)
def test_empty_graph_is_refused(fake_native, name):
    log, _ = fake_native
    for g in (None, nx.DiGraph()):
        with pytest.raises(ValueError, match='graph needed'):
            _model(name).learn_embedding(graph=g)
    assert not log


@pytest.mark.parametrize('name', ITERATIVE)
def test_unconverged_solve_warns_at_the_caller_or_raises_under_strict(fake_native, name):
    log, cfg = fake_native
    cfg['converged'] = 0
    with pytest.warns(RuntimeWarning, match=name + ': the solver stopped at max_iters=7') as rec:
        X = _model(name).learn_embedding(graph=_graph())
    assert X.shape[0] == 8
    assert [w.filename for w in rec if 'the solver stopped' in str(w.message)] == [__file__]
    with pytest.raises(RuntimeError, match=name + ': the solver stopped at max_iters=7'):
        _model(name, strict=True).learn_embedding(graph=_graph())
    assert all(h.released for h in log)


@pytest.mark.parametrize('name', ITERATIVE + ['GraphFactorization', 'node2vec'])
def test_dtype_of_the_result(fake_native, name):
    m = _model(name, dtype=np.float64)
    X = m.learn_embedding(graph=_graph())
    assert X.dtype == np.float64 and X.flags.c_contiguous and m._node_num == 8 and m.get_embedding() is X


def test_hope_returns_the_out_buffer_itself(fake_native):
    buf = np.empty((8, 4), np.float32)
    assert _model('HOPE').learn_embedding(graph=_graph(), out=buf) is buf


@pytest.mark.parametrize('n', [4096, 4097])
@pytest.mark.parametrize('setting', ['unset', True, False, 8])
def test_hope_svd_error_selection(fake_native, capsys, n, setting):
    """When HOPE computes hope.py:38-40's 'SVD error' line and how: exact (n_probe = 0) up to 4096 nodes, above that
    only when svd_error_probes asks -- True for the exact value, an int for a Hutchinson estimate with that many
    probes -- and never under svd_error_probes=False."""
    import scipy.sparse as sp
    _, cfg = fake_native
    extra = {} if setting == 'unset' else {'svd_error_probes': setting}
    A = sp.csr_matrix((np.ones(n - 1), (np.arange(n - 1), np.arange(1, n))), shape=(n, n))
    _model('HOPE', **extra).learn_embedding(graph=A)
    expected = {'unset': [0] if n <= 4096 else [], True: [0], False: [], 8: [0] if n <= 4096 else [8]}[setting]
    assert cfg['svd_error_probes'] == expected
    assert capsys.readouterr().out.count('SVD error (low rank): 0.000000') == len(expected)


# ---- evaluateStaticGraphReconstruction on a NumPy reconstruction

@pytest.fixture
def numpy_recon(monkeypatch, eval_oracle):
    """_native.Context / Reconstruction replaced by the fp64 oracle matrix (the device's fp32 scores are checked against
    the same goldens by the GPU tests); ranks / top return what test_host_eval emulates for the kernels."""
    from gem_b200 import _native

    class Context(_FakeHandle):
        def __init__(self, device=0):
            pass

    class Reconstruction(_FakeHandle):
        def __init__(self, ctx, X, kind):
            assert kind in (_native.RECON_DOT, _native.RECON_SPLIT)
            self.adj = eval_oracle.reconstruct(X, kind == _native.RECON_SPLIT)

        def pairs(self, i, j):
            return self.adj[i, j].astype(np.float32)

        def ranks(self, indptr, indices, is_undirected):
            ranks, _, _, _ = _emulated_kernel_outputs(self.adj, indptr, indices, is_undirected)
            return ranks, None

        def top(self, is_undirected, max_k=-1):
            assert max_k == -1
            n = self.adj.shape[0]
            _, i, j, w = _emulated_kernel_outputs(self.adj, np.zeros(n + 1, np.int64), np.zeros(0, np.int64),
                                                  is_undirected)
            return i, j, w

    monkeypatch.setattr(_native, 'Context', Context)
    monkeypatch.setattr(_native, 'Reconstruction', Reconstruction)


def _golden_case(name):
    from gem_b200.embedding.hope import HOPE
    z, n, (indptr, indices, w) = eval_golden(name)
    H = nx.DiGraph()
    H.add_nodes_from(int(u) for u in z['nodes'])           # list(H.nodes) order decides the weighted error
    H.add_weighted_edges_from((int(a), int(b), float(c)) for a, b, c in z['edges'])
    assert bool(z['split'])
    return z, H, HOPE({'d': z['X'].shape[1], 'beta': 0.01})


@pytest.mark.parametrize('name', ['eval_karate_hope', 'eval_randw200_split'])
def test_evaluation_full_branch_matches_the_reference_goldens(numpy_recon, name):
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    z, H, m = _golden_case(name)
    for tag in ('und', 'dir', 'dirw'):
        MAP, prec, err, err_b = evaluateStaticGraphReconstruction(H, m, z['X'], None, is_undirected=(tag == 'und'),
                                                                  is_weighted=(tag == 'dirw'))
        assert abs(MAP - float(z[tag + '_MAP'])) < 1e-13
        assert len(prec) == int(z[tag + '_n_pred'])
        assert np.array_equal(np.array(prec[:4096]), z[tag + '_prec_head'])
        assert np.array_equal(np.array(prec[::997]), z[tag + '_prec_stride'])
        if tag == 'dirw':
            assert abs(err - float(z[tag + '_err'])) < 1e-4 and abs(err_b - float(z[tag + '_err_baseline'])) < 1e-9
        else:
            assert err is None and err_b is None


@pytest.mark.parametrize('name', ['eval_karate_hope', 'eval_randw200_split'])
def test_evaluation_sampled_branch_equals_the_list_metrics(numpy_recon, monkeypatch, name):
    from gem_b200.evaluation import metrics
    from gem_b200.evaluation.evaluate_graph_reconstruction import evaluateStaticGraphReconstruction
    from gem_b200.utils import evaluation_util
    z, H, m = _golden_case(name)
    n = int(z['n'])
    rng = np.random.default_rng(11)
    pairs = [(int(a), int(b)) for a, b in rng.integers(0, n, (4 * n, 2)) if a != b]
    monkeypatch.setattr(evaluation_util, 'get_random_edge_pairs', lambda *a, **k: pairs)
    from gem_b200 import _native
    w = _native.Reconstruction(None, z['X'], _native.RECON_SPLIT).pairs(*np.array(pairs).T)
    kept = [(a, b, float(x)) for (a, b), x in zip(pairs, w) if x >= 0]
    assert 0 < len(kept) < len(pairs)
    for und in (True, False):
        MAP, prec, err, err_b = evaluateStaticGraphReconstruction(H, m, z['X'], None, sample_ratio_e=0.5,
                                                                  is_undirected=und)
        assert MAP == metrics.computeMAP(kept, H, is_undirected=und)
        assert prec == metrics.computePrecisionCurve(kept, H)[0]
        assert err is None and err_b is None
