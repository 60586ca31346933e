"""t-SNE on the GPU, stage by stage against sklearn's goldens (tests/golden/make_golden_tsne.py) and the fp64 oracle
(oracle/tsne_oracle.py): kNN sets, P, the PCA start, the Barnes-Hut gradient at angle 0 and 0.5, the first optimiser steps,
full default runs, bit-determinism, device-block ownership, refusals, a 100k-node run and plot_embedding2D."""
import io
import os
import sys
import types
from contextlib import redirect_stdout

import numpy as np
import pytest
import scipy.sparse as sp

from tsne_golden import CASES, load, to

pytestmark = pytest.mark.gpu

POSITIONS = ['Y0', 'Y250', 'Y1000']


@pytest.fixture(scope='module')
def affinities(gpu_ctx):
    from gem_b200 import _native
    return {name: _native.tsne_affinities(gpu_ctx, load(name)['X'], 30.0) for name in CASES}


@pytest.mark.parametrize('name', CASES)
def test_knn_sets(affinities, name):
    z, a = load(name), affinities[name]
    assert a['knn_idx'].shape == z['knn_idx'].shape
    assert not to.neighbour_mismatches(a['knn_idx'], a['knn_d2'], z['knn_idx'], z['knn_d2'])
    ref = np.sort(z['knn_d2'], 1)
    assert np.all(np.abs(a['knn_d2'] - ref) <= 1e-5 * ref + 1e-7 * ref.max())
    # ascending by (d^2, index)
    d, i = a['knn_d2'], a['knn_idx']
    assert np.all((d[:, 1:] > d[:, :-1]) | ((d[:, 1:] == d[:, :-1]) & (i[:, 1:] > i[:, :-1])))


@pytest.mark.parametrize('name', CASES)
def test_probabilities(affinities, name):
    z, a = load(name), affinities[name]
    H = to.entropy(a['knn_d2'], a['p_cond'])
    assert np.all(np.abs(H - np.log(30.0)) <= 1e-5 + 1e-9)          # every row calibrated within sklearn's tolerance
    n = z['X'].shape[0]
    G = sp.csr_matrix((a['p_val'], a['p_indices'], a['p_indptr']), shape=(n, n))
    R = z['P']
    # neighbours swapped at an exactly tied k-th distance (the mixture's duplicated rows; test_knn_sets allows those
    # swaps and no others) change the entries (i, j) and (j, i) of such a row i: the rest is compared entry by entry
    swapped = np.array([set(a['knn_idx'][i].tolist()) != set(z['knn_idx'][i].tolist()) for i in range(n)])
    keep = sp.diags((~swapped).astype(float))
    Gk, Rk = (keep @ G @ keep).tocsr(), (keep @ R @ keep).tocsr()
    Gk.eliminate_zeros()
    Rk.eliminate_zeros()
    print('%s: %d rows with tie-swapped neighbours' % (name, int(swapped.sum())))
    assert swapped.sum() <= 0.02 * n          # the mixture duplicates 40 of its 2000 rows
    assert np.array_equal(Gk.indptr, Rk.indptr) and np.array_equal(Gk.indices, Rk.indices)
    assert np.all(np.abs(Gk.data - Rk.data) <= 1e-5 * Rk.data + 1e-9 * Rk.data.max())
    assert abs(G.data.sum() - 1.0) < 1e-12
    assert G.nnz == int(z['nnz_P']) or swapped.any()
    # sklearn's calibrated rows, where the neighbour sets agree (GPU rows are in (d^2, index) order)
    for r, ref in zip(z['p_rows'], z['p_cond']):
        if not swapped[r]:
            o = np.argsort(a['knn_idx'][r])
            assert np.all(np.abs(a['p_cond'][r][o] - ref) <= 1e-5 * ref + 1e-12)


@pytest.mark.parametrize('name', CASES)
def test_pca_start(gpu_ctx, name):
    from gem_b200 import _native
    z = load(name)
    Y0, st = _native.tsne(gpu_ctx, z['X'], 30.0, 12.0, 50.0, 0, 300, 1e-7, 0.5)
    tol = 1e-3 if str(z['pca_solver']) == 'randomized' else 1e-5
    err = np.linalg.norm(Y0 - z['Y0']) / np.linalg.norm(z['Y0'])
    print('%s: PCA start rel err %.2e (sklearn solver %s)' % (name, err, z['pca_solver']))
    assert err <= tol
    assert st['n_iter'] == -1 and st['n_neighbors'] == z['knn_idx'].shape[1] and st['nnz_P'] == int(z['nnz_P'])


@pytest.mark.parametrize('name', CASES)
@pytest.mark.parametrize('pos', POSITIONS)
def test_gradient_angle0(gpu_ctx, name, pos):
    """At angle 0 every cell is opened down to sklearn's leaves: the fp64 exact gradient over the pairs the tree counts
    (sklearn's leaves merge points within 1e-6 of each other, and a leaf that duplicates the query is skipped; where no
    two points are that close this is the exact gradient)."""
    from gem_b200 import _native
    z = load(name)
    Y = z[pos]
    P = z['P']
    g, kl = _native.tsne_gradient(gpu_ctx, Y, P.indptr, P.indices, P.data, 0.0)
    ge, kle = to.exact_gradient(Y, z['P'], tree_pairs=True)
    err = np.linalg.norm(g - ge) / np.linalg.norm(ge)
    print('%s %s: |g - g_exact| / |g_exact| = %.2e, KL %.8f vs %.8f' % (name, pos, err, kl, kle))
    assert err <= 1e-4
    assert abs(kl - kle) <= 1e-5 * max(abs(kle), 1e-3)


@pytest.mark.parametrize('name', CASES)
@pytest.mark.parametrize('pos', POSITIONS)
def test_gradient_angle05(gpu_ctx, name, pos):
    from gem_b200 import _native
    z = load(name)
    Y = z[pos]
    P = z['P']
    g, kl = _native.tsne_gradient(gpu_ctx, Y, P.indptr, P.indices, P.data, 0.5)
    ge, _ = to.exact_gradient(Y, z['P'], tree_pairs=True)
    sk = np.linalg.norm(z['grad_bh05_' + pos] - ge)
    mine = np.linalg.norm(g - ge)
    print('%s %s: |g - g_exact| %.3e, sklearn BH %.3e (|g_exact| %.3e); KL %.6f sklearn %.6f'
          % (name, pos, mine, sk, np.linalg.norm(ge), kl, z['kl_bh05_' + pos]))
    assert mine <= 1.5 * sk + 1e-6 * np.linalg.norm(ge)


def test_optimiser_steps(gpu_ctx):
    """The first iterations at angle 0 on Karate (momentum 0.5, exaggeration 12, learning rate max(34 / 48, 50) = 50)
    against the oracle's update driven by the fp64 exact gradient, from the same start and P.  Later iterates are not
    comparable at 1e-4: on Karate the gains flip with the sign of near-zero gradient components, and sklearn's own fp32
    run departs from the fp64 oracle by 9e-5 after 10 steps and 13 % after 20.  The 20-step run is checked for its
    iteration count and finite positions."""
    from gem_b200 import _native
    z = load('tsne_karate_d4')
    a = _native.tsne_affinities(gpu_ctx, z['X'], 30.0)
    n = z['X'].shape[0]
    P = sp.csr_matrix((a['p_val'], a['p_indices'], a['p_indptr']), shape=(n, n))
    Y0, _ = _native.tsne(gpu_ctx, z['X'], 30.0, 12.0, 50.0, 0, 300, 1e-7, 0.0)
    for m in (1, 2, 5):
        Ym, st = _native.tsne(gpu_ctx, z['X'], 30.0, 12.0, 50.0, m, 300, 1e-7, 0.0)
        ref = to.descend(Y0, P, m, 12.0, 0.5, 50.0, tree_pairs=True)
        err = np.linalg.norm(Ym - ref) / np.linalg.norm(ref)
        print('%d steps: rel err %.2e' % (m, err))
        assert st['n_iter'] == m - 1 and err <= 1e-4
    Y20, st = _native.tsne(gpu_ctx, z['X'], 30.0, 12.0, 50.0, 20, 300, 1e-7, 0.0)
    assert st['n_iter'] == 19 and np.all(np.isfinite(Y20))


@pytest.fixture(scope='module')
def full_runs():
    from gem_b200.evaluation.visualize_embedding import tsne
    out = {}
    for name in CASES:
        st = {}
        Y = tsne(load(name)['X'], stats=st)
        out[name] = (Y, st)
    return out


@pytest.mark.parametrize('name', CASES)
def test_full_run(full_runs, name):
    z = load(name)
    Y, st = full_runs[name]
    assert Y.dtype == np.float32 and Y.shape == (z['X'].shape[0], 2) and np.all(np.isfinite(Y))
    tw = to.trustworthiness(z['X'].astype(np.float64), Y.astype(np.float64), 12)
    print('%s: KL %.5f (sklearn %.5f), n_iter %d, trustworthiness %.4f (sklearn %.4f), %s'
          % (name, st['kl_divergence'], float(z['kl_final']), st['n_iter'], tw, float(z['trust12']),
             {k: round(v, 2) for k, v in st.items() if k.endswith('_ms')}))
    if name != 'tsne_karate_d4':
        # Karate's 34 points all attract each other (k = 33) and its trajectory is chaotic (test_optimiser_steps):
        # the run ends in another local minimum, so only its trustworthiness is compared
        assert abs(st['kl_divergence'] - float(z['kl_final'])) <= 0.05 * float(z['kl_final'])
    assert tw >= float(z['trust12']) - 0.01
    assert st['n_neighbors'] == z['knn_idx'].shape[1] and st['nnz_P'] == int(z['nnz_P'])
    assert st['learning_rate'] == max(z['X'].shape[0] / 12.0 / 4.0, 50.0)
    if z['labels'] is not None:
        lab = z['labels']
        D = to.sqdist(Y, Y)
        np.fill_diagonal(D, np.inf)
        share = float(np.mean(lab[D.argmin(1)] == lab))
        print('%s: 2-D nearest neighbour in the same community: %.4f (sklearn %.4f)' % (name, share, float(z['nn_same'])))
        assert share >= 0.95


def test_deterministic(full_runs):
    from gem_b200.evaluation.visualize_embedding import tsne
    z = load('tsne_sbm1024_d16')
    st = {}
    Y = tsne(z['X'], stats=st)
    Y0, st0 = full_runs['tsne_sbm1024_d16']
    assert Y.tobytes() == Y0.tobytes() and st['kl_divergence'] == st0['kl_divergence']


@pytest.mark.skipif(os.environ.get('GEMB_CACHE_MB', '').strip() == '0',
                    reason='GEMB_CACHE_MB=0: no block cache, gemb_mem_live_blocks is always 0')
def test_no_device_blocks_leak(gpu_ctx):
    from gem_b200 import _native
    X = load('tsne_karate_d4')['X']
    z = load('tsne_karate_d4')
    calls = [lambda: _native.tsne(gpu_ctx, X, 30.0, 12.0, 50.0, 300, 300, 1e-7, 0.5),
             lambda: _native.tsne_affinities(gpu_ctx, X, 10.0),
             lambda: _native.tsne_gradient(gpu_ctx, z['Y250'], z['P'].indptr, z['P'].indices, z['P'].data, 0.5)]
    for call in calls:
        call()
        before = _native.mem_live_blocks()
        call()
        assert _native.mem_live_blocks() == before
    # an error after the device work: cap below nnz
    before = _native.mem_live_blocks()
    with pytest.raises(RuntimeError):
        _native.check(_native.lib().gemb_tsne_affinities(gpu_ctx._h, 34, 4, _native._ptr(np.ascontiguousarray(X)), 10.0, 1,
                                                         *([None] * 6), None, None))
    assert _native.mem_live_blocks() == before


def test_refusals_launch_nothing(gpu_ctx):
    from gem_b200 import _native
    X = load('tsne_karate_d4')['X']
    bad = [dict(X=X, perplexity=34.0), dict(X=X, angle=1.5), dict(X=X, learning_rate=0.0),
           dict(X=X, early_exaggeration=-1.0), dict(X=np.where(X > 0.05, np.nan, X)), dict(X=X[:1])]
    for b in bad:
        args = dict(X=X, perplexity=30.0, early_exaggeration=12.0, learning_rate=50.0, max_iter=300,
                    n_iter_without_progress=300, min_grad_norm=1e-7, angle=0.5)
        args.update(b)
        n0 = _native.lib().gemb_launch_count()
        with pytest.raises(RuntimeError):
            _native.tsne(gpu_ctx, **args)
        assert _native.lib().gemb_launch_count() == n0, b


def test_scale_100k(gpu_ctx):
    """n = 100 000: the HOPE d = 128 embedding of bench.py's SBM (1000-node blocks), reduced with the defaults."""
    from gem_b200 import _native, synth
    from gem_b200.evaluation.visualize_embedding import tsne
    csr = synth.sbm(n=100_000, block=1000, seed=42)
    g = _native.DeviceGraph(gpu_ctx, csr.n, csr.indptr, csr.indices, None)
    X, _, _ = g.hope(128, 0.01, tol=4e-3, stop_rule=1, cheb_degree=16, cheb_range_log2=14, max_iters=30, min_iters=2,
                     oversample=8, seed=1234)
    g.free()
    st = {}
    Y = tsne(X, stats=st)
    print('100k: %s' % {k: (round(v, 3) if isinstance(v, float) else v) for k, v in st.items()})
    assert Y.shape == (100_000, 2) and np.all(np.isfinite(Y))
    assert st['n_iter'] >= 249 and np.isfinite(st['kl_divergence'])


@pytest.fixture
def stub_pyplot(monkeypatch):
    calls = []
    plt = types.ModuleType('matplotlib.pyplot')
    plt.scatter = lambda x, y, c=None: calls.append((np.array(x), np.array(y), c))
    mpl = types.ModuleType('matplotlib')
    mpl.pyplot = plt
    monkeypatch.setitem(sys.modules, 'matplotlib', mpl)
    monkeypatch.setitem(sys.modules, 'matplotlib.pyplot', plt)
    return calls


def test_plot_embedding2D_scatters_tsne_positions(stub_pyplot):
    from gem_b200.evaluation.visualize_embedding import plot_embedding2D, tsne
    X = load('tsne_karate_d4')['X']
    buf = io.StringIO()
    with redirect_stdout(buf):
        plot_embedding2D(X, node_colors=np.arange(34))
    assert buf.getvalue() == 'Embedding dimension greater than 2, use tSNE to reduce it to 2\n'
    Y = tsne(X)
    (x, y, c), = stub_pyplot
    assert np.array_equal(x, Y[:, 0]) and np.array_equal(y, Y[:, 1]) and np.array_equal(c, np.arange(34))


def test_plot_embedding2D_2d_makes_no_device_call(stub_pyplot, monkeypatch):
    from gem_b200 import _native
    from gem_b200.evaluation.visualize_embedding import plot_embedding2D

    def boom(*a, **k):
        raise AssertionError('device call for a 2-D embedding')
    monkeypatch.setattr(_native, 'Context', boom)
    monkeypatch.setattr(_native, 'lib', boom)
    X = np.random.RandomState(0).randn(10, 2)
    buf = io.StringIO()
    with redirect_stdout(buf):
        plot_embedding2D(X)
    assert buf.getvalue() == ''
    (x, y, c), = stub_pyplot
    assert np.array_equal(x, X[:, 0]) and np.array_equal(y, X[:, 1]) and c is None
