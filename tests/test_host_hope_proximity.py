"""HOPE(proximity=...) on the host: every refused setting raises ValueError before any device call (these tests run without
a GPU and would fail with RuntimeError if the library were reached), and rooted PageRank's uploaded P is D_out^-1 A."""
import numpy as np
import pytest
import scipy.sparse as sp

from conftest import load_karate_nx


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


@pytest.fixture
def no_device(monkeypatch):
    """Any attempt to open a device context fails the test."""
    from gem_b200 import _native

    def boom(*a, **k):
        raise AssertionError('a device call was made')
    monkeypatch.setattr(_native, 'Context', boom)
    monkeypatch.setattr(_native, 'DeviceGraph', boom)


@pytest.mark.parametrize('kw,match', [
    (dict(proximity='katz_index'), 'proximity must be one of'),
    (dict(proximity='rooted_pagerank'), 'needs alpha'),
    (dict(proximity='rooted_pagerank', alpha=0.0), 'needs alpha'),
    (dict(proximity='rooted_pagerank', alpha=1.0), 'needs alpha'),
    (dict(proximity='rooted_pagerank', alpha=-0.5), 'needs alpha'),
    (dict(proximity='katz', alpha=0.5), 'takes none'),
    (dict(alpha=0.5), 'takes none'),
    (dict(proximity='common_neighbors', alpha=0.5), 'takes none'),
    (dict(proximity='adamic_adar', beta_over_rho=0.5), 'beta_over_rho'),
    (dict(proximity='rooted_pagerank', alpha=0.5, beta_over_rho=0.5), 'beta_over_rho'),
])
def test_refused_settings(no_device, kw, match):
    m = _fresh(d=4, beta=0.01, **kw)
    with pytest.raises(ValueError, match=match):
        m.learn_embedding(graph=load_karate_nx())


@pytest.mark.parametrize('proximity,alpha', [('adamic_adar', None), ('rooted_pagerank', 0.5)])
def test_negative_weights_refused(no_device, proximity, alpha):
    from gem_b200 import graph as hg
    A = sp.random(50, 50, density=0.1, random_state=1, format='csr')
    A.data[3] = -0.25
    m = _fresh(d=4, beta=0.01, proximity=proximity, alpha=alpha)
    with pytest.raises(ValueError, match='non-negative'):
        m.learn_embedding(graph=hg.from_scipy(A))


@pytest.mark.parametrize('proximity,alpha', [('common_neighbors', None), ('adamic_adar', None), ('rooted_pagerank', 0.5)])
def test_multi_gpu_refused(no_device, monkeypatch, proximity, alpha):
    from gem_b200 import dist as gd
    monkeypatch.setattr(gd, 'spmd', lambda device=None: (object(), 0, 2, 0))
    m = _fresh(d=4, beta=0.01, proximity=proximity, alpha=alpha)
    with pytest.raises(ValueError, match='single-GPU'):
        m.learn_embedding(graph=load_karate_nx())


def test_check_proximity_accepts_the_valid_settings():
    from gem_b200.embedding.hope import check_proximity
    from gem_b200 import graph as hg
    A = hg.from_scipy(sp.csr_matrix(np.array([[0, 2.0], [-1.0, 0]])))
    check_proximity('katz', None, 0.5, 2, A)                  # Katz: beta_over_rho, multi-GPU and signed weights
    check_proximity('common_neighbors', None, None, 1, A)     # signed weights are fine for A A
    check_proximity('rooted_pagerank', 0.999, None, 1, None)


def test_rooted_pagerank_operator_is_row_normalised():
    import os
    import sys
    from conftest import REPO
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import proximity_oracle as po
    from gem_b200 import graph as hg
    from gem_b200.embedding.hope import rooted_pagerank_operator
    rng = np.random.default_rng(4)
    M = (rng.random((60, 60)) < 0.1) * rng.uniform(0.5, 2.0, (60, 60))
    M[5, :] = 0.0                                              # out-degree 0: the row stays zero
    for csr in (hg.from_scipy(sp.csr_matrix(M)), hg.from_scipy(sp.csr_matrix((M > 0).astype(float)))):
        P = rooted_pagerank_operator(csr)
        assert not P.is_symmetric()
        assert np.abs(P.to_scipy() - po.transition(csr.to_scipy())).max() < 1e-15
        assert np.abs(P.transpose().to_scipy() - P.to_scipy().T).max() == 0.0
