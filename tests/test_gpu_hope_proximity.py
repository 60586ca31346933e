"""HOPE on the common-neighbour, Adamic-Adar and rooted-PageRank proximities (gemb_hope spectral_modes 3, 4, 5: S applied
matrix-free by the general solver) against the fp64 oracle of oracle/proximity_oracle.py.

- small graphs (undirected Karate at d = 4 and 16, SBM-1024 and a directed weighted 200-node graph at d = 16): sigma against the dense
  oracle, the rank-k product X1 X2^T (invariant to rotations inside degenerate subspaces), fp64 residuals and resid_max;
- hub rows (R-MAT scale 12: rows above SPMM_HEAVY_DEG take the chunked SpMM path, with the per-row scale in its finish
  kernel) against the matrix-free oracle, at the bars of test_gpu_hope.py::test_power_law_graph_skewed_spectrum;
- SBM at 100k nodes at the bars of test_gpu_hope.py::test_large_sparse_input_properties;
- the refusals, bit-identical repeated calls, released device blocks, and Katz unchanged by the new keyword."""
import os
import sys
import warnings

import numpy as np
import pytest

from conftest import REPO, load_karate_nx, load_sbm1024_nx

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings('ignore::RuntimeWarning')]   # tol = 1e-8 is below fp32's floor
sys.path.insert(0, os.path.join(REPO, 'oracle'))
import hope_oracle as ho
import proximity_oracle as po

ALPHA = 0.5


def _fresh(**kw):
    from gem_b200.embedding.hope import HOPE
    HOPE.hyper_params.clear()
    HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
    return HOPE(**kw)


@pytest.fixture(autouse=True)
def _keep_hyper_params():
    """HOPE's keyword arguments stay in the class-level dict (GEM's behaviour): put it back as it was, so that no later
    test inherits a proximity."""
    from gem_b200.embedding.hope import HOPE
    saved = dict(HOPE.hyper_params)
    yield
    HOPE.hyper_params.clear()
    HOPE.hyper_params.update(saved)


def _alpha(proximity):
    return ALPHA if proximity == 'rooted_pagerank' else None


def _bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _small(name):
    """(graph given to learn_embedding, fp64 adjacency in the same node order).  Karate is taken undirected: loaded
    directed it is strictly upper triangular, A A has rank 7, and at d = 16 the eighth triplet (sigma = 0) is not
    defined by S."""
    import networkx as nx
    from gem_b200 import graph as hg
    if name == 'karate':
        G = nx.Graph(load_karate_nx().to_undirected())
        return G, ho.adjacency_from_nx(G)
    if name == 'sbm1024':
        G, _ = load_sbm1024_nx()
        return G, ho.adjacency_from_nx(G)
    A = po.random_digraph()
    return hg.from_scipy(A), A


@pytest.mark.parametrize('proximity', po.PROXIMITIES)
@pytest.mark.parametrize('name,d', [('karate', 4), ('karate', 16), ('sbm1024', 16), ('randw200', 16)])
def test_small_graphs_against_dense_oracle(native_lib, proximity, name, d):
    G, A = _small(name)
    alpha = _alpha(proximity)
    m = _fresh(d=d, beta=0.01, proximity=proximity, alpha=alpha, tol=1e-8, oversample=48, max_iters=400,
               compute_residual=1)
    X = m.learn_embedding(graph=G)
    st = m.stats
    assert st['proximity'] == proximity and st['algorithm'] == 1 and m._svd_error is None
    assert st['spmm_count'] > 0 and st['norm2_A'] == 0.0
    if proximity == 'rooted_pagerank':
        assert st['katz_terms'] == po.rooted_pagerank_terms(ALPHA, 1e-7) and st['beta_used'] == np.float32(ALPHA)
    else:
        assert st['katz_terms'] == 0 and st['beta_used'] == 0.0
    sig = np.asarray(m._sigma, dtype=np.float64)
    Xo, so = po.embedding(A, proximity, d, alpha=alpha)
    S = po.proximity_dense(A, proximity, alpha=alpha)
    smax = so[-1]
    e_sig = np.abs(sig - so).max() / smax
    e_rec = ho.recon_rel_err(X, Xo)
    r1, r2 = po.residuals(A, proximity, X, sig, S=S)
    print('%s d=%d %s: |sigma - fp64| / sigma_max %.2e (bar 1e-5), X1 X2^T rel err %.2e (bar 1e-4), residuals %.2e %.2e '
          '(bar 1e-4), resid_max %.3e vs fp64 %.3e, iters %d sweeps %d'
          % (name, d, proximity, e_sig, e_rec, r1.max(), r2.max(), st['resid_max'], r2.max(), st['iters'], st['spmm_count']))
    assert np.all(np.diff(sig) >= 0)
    assert e_sig <= 1e-5
    assert e_rec <= 1e-4
    assert r1.max() < 1e-4 and r2.max() < 1e-4
    assert abs(st['resid_max'] - r2.max()) <= 2e-3


@pytest.mark.parametrize('proximity', po.PROXIMITIES)
def test_hub_rows_rmat12(native_lib, proximity):
    from gem_b200 import synth
    csr = synth.rmat(scale=12, edge_factor=8, seed=3)
    assert np.diff(csr.indptr).max() > 128                        # hub rows: the chunked SpMM path
    A = csr.to_scipy().astype(np.float64)
    alpha = _alpha(proximity)
    m = _fresh(d=16, beta=0.01, proximity=proximity, alpha=alpha, tol=1e-6, max_iters=200, min_iters=4)
    with warnings.catch_warnings():
        warnings.simplefilter('error')                           # converged: no warning
        X = m.learn_embedding(graph=csr)
    assert m.stats['algorithm'] == 1 and m.stats['converged'] == 1
    sig = np.asarray(m._sigma, dtype=np.float64)
    Xo, so = po.embedding(A, proximity, 16, alpha=alpha, tol=1e-10)
    k = 8
    rec = X[:, :k].astype(np.float64) @ X[:, k:].astype(np.float64).T
    reco = Xo[:, :k] @ Xo[:, k:].T
    e_rec = np.linalg.norm(rec - reco) / np.linalg.norm(reco)
    print('R-MAT 12 %s: max |sigma / fp64 - 1| %.2e (bar 2e-4), X1 X2^T rel err %.2e (bar 5e-3), iters %d'
          % (proximity, np.abs(sig / so - 1).max(), e_rec, m.stats['iters']))
    assert np.allclose(sig, so, rtol=2e-4)
    assert e_rec <= 5e-3


@pytest.mark.parametrize('proximity', po.PROXIMITIES)
def test_sbm100k(native_lib, proximity):
    """Size-independent properties at 100k nodes.  Rooted PageRank runs at alpha = 0.2 (J = 11 terms) and the oracle
    applies the same truncated series, so that its CPU svds stays short."""
    from gem_b200 import synth
    csr = synth.sbm(n=100_000, block=1000, seed=11)
    alpha = 0.2 if proximity == 'rooted_pagerank' else None
    m = _fresh(d=16, beta=0.01, proximity=proximity, alpha=alpha, tol=1e-8, max_iters=100, min_iters=4,
               compute_residual=1)
    X = m.learn_embedding(graph=csr)
    sig = np.asarray(m._sigma, dtype=np.float64)
    assert np.all(np.diff(sig) >= 0)
    A = csr.to_scipy().astype(np.float64)
    terms = m.stats['katz_terms'] if proximity == 'rooted_pagerank' else None
    op = po.proximity_operator(A, proximity, alpha=alpha, terms=terms)
    r1, r2 = po.residuals(A, proximity, X, sig, S=op)
    k = 8
    U = X[:, :k].astype(np.float64) / np.sqrt(sig)[None, :]
    V = X[:, k:].astype(np.float64) / np.sqrt(sig)[None, :]
    Xo, so = po.embedding(A, proximity, 16, alpha=alpha, tol=1e-6, terms=terms)
    print('SBM 100k %s: residuals %.2e %.2e (bar 5e-3), resid_max %.2e, top sigma rel err %.2e (bar 1e-5), '
          'max sigma rel err %.2e (bar 2e-3), iters %d'
          % (proximity, r1.max(), r2.max(), m.stats['resid_max'], abs(sig[-1] / so[-1] - 1),
             np.abs(sig / so - 1).max(), m.stats['iters']))
    assert np.abs(U.T @ U - np.eye(k)).max() < 1e-4 and np.abs(V.T @ V - np.eye(k)).max() < 1e-4
    assert r1.max() < 5e-3 and r2.max() < 5e-3
    assert m.stats['resid_max'] < 5e-3
    assert np.allclose(sig[-1], so[-1], rtol=1e-5)
    assert np.allclose(sig, so, rtol=2e-3)


def test_refusals(gpu_ctx):
    from gem_b200 import _native
    G, A = _small('randw200')
    AT = A.T.tocsr()
    P = po.transition(A).astype(np.float32)
    PT = P.T.tocsr()
    lib = _native.lib()
    with _native.DeviceGraph(gpu_ctx, A.shape[0], A.indptr, A.indices, A.data, AT.indptr, AT.indices, AT.data) as g, \
            _native.DeviceGraph(gpu_ctx, A.shape[0], P.indptr, P.indices, P.data, PT.indptr, PT.indices, PT.data) as gp:
        for mode in (3, 4, 5):
            for algorithm in (2, 3):
                n0 = lib.gemb_launch_count()
                with pytest.raises(RuntimeError, match='general solver'):
                    (gp if mode == 5 else g).hope(8, 0.5, spectral_mode=mode, algorithm=algorithm)
                assert lib.gemb_launch_count() == n0              # refused before any launch
        for alpha in (0.0, 1.0, 1.5, -0.5):
            n0 = lib.gemb_launch_count()
            with pytest.raises(RuntimeError, match='0 < alpha < 1'):
                gp.hope(8, alpha, spectral_mode=5)
            assert lib.gemb_launch_count() == n0
        with pytest.raises(RuntimeError, match='row sum <= 1'):
            g.hope(8, 0.5, spectral_mode=5)                     # A, not P = D_out^-1 A
        with pytest.raises(RuntimeError, match='d must be even'):
            g.hope(7, 0.0, spectral_mode=3)
        X, sig, st = g.hope(8, 0.0, spectral_mode=3, max_iters=5)   # the same upload is accepted for mode 3
        assert sig.shape == (4,) and st['algorithm'] == 1
    An = A.copy()
    An.data[5] = -An.data[5]
    ATn = An.T.tocsr()
    with _native.DeviceGraph(gpu_ctx, An.shape[0], An.indptr, An.indices, An.data, ATn.indptr, ATn.indices, ATn.data) as g:
        with pytest.raises(RuntimeError, match='non-negative weights'):
            g.hope(8, 0.0, spectral_mode=4)
        X, sig, st = g.hope(8, 0.0, spectral_mode=3, max_iters=5)   # A A takes signed weights
        assert np.all(np.isfinite(X))


@pytest.mark.parametrize('proximity', po.PROXIMITIES)
def test_repeated_calls_are_bit_identical_and_release_their_blocks(native_lib, proximity):
    from gem_b200 import _native
    G, _ = load_sbm1024_nx()

    def run():
        m = _fresh(d=16, beta=0.01, proximity=proximity, alpha=_alpha(proximity), tol=1e-8, max_iters=30,
                   compute_residual=1)
        return m.learn_embedding(graph=G).copy(), m._sigma.copy()

    X1, s1 = run()
    before = _native.mem_live_blocks()
    X2, s2 = run()
    if os.environ.get('GEMB_CACHE_MB', '').strip() != '0':
        assert _native.mem_live_blocks() == before
    assert _bits(X1, X2) and _bits(s1, s2)


@pytest.mark.parametrize('algorithm', [1, 2])
def test_katz_keyword_changes_nothing(native_lib, algorithm):
    G, _ = load_sbm1024_nx()
    kw = dict(d=16, beta=0.01, tol=1e-8, max_iters=60, algorithm=algorithm, svd_error_probes=False)
    m0 = _fresh(**kw)
    X0 = m0.learn_embedding(graph=G).copy()
    m1 = _fresh(proximity='katz', **kw)
    X1 = m1.learn_embedding(graph=G)
    assert m0.stats['algorithm'] == algorithm and m1.stats['proximity'] == 'katz'
    assert _bits(X0, X1) and _bits(m0._sigma, m1._sigma)
