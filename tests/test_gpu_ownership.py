"""Every entry point gives back the device blocks it takes from the block cache, on success and on the error returns an
input can reach after allocation (gemb_mem_live_blocks: blocks handed out and not yet released).  A failed call must
also leave the library usable: the same valid call gives the same bits before and after it."""
import ctypes
import os

import numpy as np
import pytest

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(os.environ.get('GEMB_CACHE_MB', '').strip() == '0',
                       reason='GEMB_CACHE_MB=0: no block cache, gemb_mem_live_blocks is always 0'),
]


def _live():
    from gem_b200 import _native
    return _native.mem_live_blocks()


def _same_bits(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_same_bits(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return a == b


def _no_leak(call):
    call()                      # warm-up: grows the context's scratch blocks
    before = _live()
    call()
    assert _live() == before


def _fails_without_leak(bad, good, match=None):
    ref = good()
    before = _live()
    with pytest.raises(RuntimeError, match=match):
        bad()
    assert _live() == before
    assert _same_bits(good(), ref)


def _upload(ctx, csr, weighted=False):
    from gem_b200 import _native
    data = np.linspace(0.5, 1.5, csr.nnz).astype(np.float32) if weighted else None
    return _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, data)


@pytest.fixture(scope='module')
def sbm(gpu_ctx):
    from gem_b200 import synth
    csr = synth.sbm(n=4096, block=512, seed=11)
    g = _upload(gpu_ctx, csr)
    yield csr, g
    g.free()


def _hope(g, **opts):
    X, sig, _ = g.hope(16, 0.01, tol=1e-4, max_iters=8, **opts)
    return X, sig


@pytest.mark.parametrize('opts', [
    dict(algorithm=1), dict(algorithm=2), dict(algorithm=3), dict(spectral_mode=1),
    dict(algorithm=1, compute_residual=1), dict(algorithm=2, compute_residual=1),
    dict(algorithm=1, oversample=4, compute_residual=1),      # d > block width: X in its own block
    dict(algorithm=2, oversample=4, compute_residual=1),
], ids=lambda o: '-'.join('%s%d' % kv for kv in o.items()))
def test_hope_releases_its_blocks(sbm, opts):
    _, g = sbm
    _no_leak(lambda: _hope(g, **opts))


def test_hope_svd_error_releases_its_blocks(sbm):
    csr, g = sbm
    X = np.random.default_rng(1).standard_normal((csr.n, 16)).astype(np.float32)
    _no_leak(lambda: g.hope_svd_error(16, 0.01, X, n_probe=8))


def test_spmm_and_dense_hooks_release_their_blocks(gpu_ctx, sbm):
    csr, g = sbm
    rng = np.random.default_rng(2)
    X = rng.standard_normal((csr.n, 16)).astype(np.float32)
    _no_leak(lambda: g.spmm(X, alpha=0.5, X0=X, gamma=0.25, Xself=X, delta=2.0))
    P, Q = rng.standard_normal((5000, 32)).astype(np.float32), rng.standard_normal((5000, 16)).astype(np.float32)
    _no_leak(lambda: gpu_ctx.gram(P, Q))
    _no_leak(lambda: gpu_ctx.apply(P, rng.standard_normal((32, 16)).astype(np.float32)))
    B = rng.standard_normal((40, 24))
    G = B.T @ B
    _no_leak(lambda: gpu_ctx.chol_inverse(G))
    _no_leak(lambda: gpu_ctx.eigh(G))


@pytest.mark.parametrize('p,q', [(1.0, 1.0), (0.5, 2.0)])
def test_node2vec_releases_its_blocks(gpu_ctx, p, q):
    from gem_b200 import synth
    csr = synth.sbm(n=2048, block=256, seed=12)
    g = _upload(gpu_ctx, csr)
    w = np.linspace(0.5, 1.5, csr.nnz)
    nids = np.arange(csr.n, dtype=np.int32)
    try:
        if p == 1.0:
            _no_leak(lambda: g.n2v_alias(w))
        _no_leak(lambda: g.n2v_walks(nids, 10, 2, p=p, q=q, seed=3, weights64=w))
        _no_leak(lambda: g.node2vec(nids, 16, 10, 2, 3, 1, p=p, q=q, seed=3, weights64=w))
    finally:
        g.free()


@pytest.mark.parametrize('mode', [0, 1])
def test_gf_releases_its_blocks(gpu_ctx, mode):
    from gem_b200 import _native
    rng = np.random.default_rng(4)
    n, m = 500, 4000
    src = np.sort(rng.integers(0, n, m)).astype(np.int32)
    dst = rng.integers(0, n, m).astype(np.int32)
    X0 = (0.01 * rng.standard_normal((n, 24))).astype(np.float32)
    _no_leak(lambda: _native.graph_factorization(gpu_ctx, n, src, dst, None, 24, 0.01, 0.1, 3, X0, mode=mode))


def test_synth_rmat_releases_its_blocks(gpu_ctx):
    from gem_b200 import _native
    _no_leak(lambda: _native.synth_rmat(gpu_ctx, 10))


def test_graph_and_reconstruction_lifetimes(gpu_ctx, sbm):
    from gem_b200 import _native
    csr, _ = sbm
    before = _live()
    g = _upload(gpu_ctx, csr, weighted=True)
    assert _live() > before
    g.free()
    assert _live() == before
    n = 700
    X = np.abs(np.random.default_rng(5).standard_normal((n, 16))).astype(np.float32)
    r = _native.Reconstruction(gpu_ctx, X, kind=_native.RECON_SPLIT)
    r.dense()
    r.pairs(np.arange(10), np.arange(10, 20))
    nbr = np.stack(((np.arange(n) + 1) % n, (np.arange(n) + 7) % n), axis=1)
    r.ranks(np.arange(0, 2 * n + 1, 2), np.sort(nbr, axis=1).ravel(), True)
    r.top(True, max_k=50)
    r.free()
    assert _live() == before


# ---- error returns after allocation

def test_hope_negative_beta_on_edgeless_graph(gpu_ctx, sbm):
    from gem_b200 import _native
    _, g = sbm
    n = 512
    empty = _native.DeviceGraph(gpu_ctx, n, np.zeros(n + 1, dtype=np.int32), np.zeros(0, dtype=np.int32))
    try:
        _fails_without_leak(lambda: empty.hope(16, -0.5), lambda: _hope(g), match='empty graph')
    finally:
        empty.free()


def test_hope_divergent_katz_series(sbm):
    _, g = sbm
    _fails_without_leak(lambda: g.hope(16, 1.0, algorithm=2), lambda: _hope(g))


def test_hope_lanczos_basis_too_small(sbm):
    _, g = sbm
    _fails_without_leak(lambda: g.hope(16, 0.01, algorithm=3, algorithm3_basis=16), lambda: _hope(g, algorithm=3))


def test_upload_with_out_of_range_column(gpu_ctx, sbm):
    from gem_b200 import _native
    csr, g = sbm
    bad = csr.indices.copy()
    bad[len(bad) // 2] = csr.n
    X = np.random.default_rng(6).standard_normal((csr.n, 8)).astype(np.float32)
    _fails_without_leak(lambda: _native.DeviceGraph(gpu_ctx, csr.n, csr.indptr, bad), lambda: g.spmm(X))


def test_recon_top_with_too_small_cap(gpu_ctx):
    from gem_b200 import _native
    X = np.abs(np.random.default_rng(7).standard_normal((300, 16))).astype(np.float32)
    r = _native.Reconstruction(gpu_ctx, X, kind=_native.RECON_SPLIT)
    try:
        i, j, w = (np.empty(1, dtype=t) for t in (np.int32, np.int32, np.float32))
        m = ctypes.c_int64(0)
        bad = lambda: _native.check(_native.lib().gemb_recon_top(r._h, 1, 50, 1, _native._ptr(i), _native._ptr(j),
                                                                  _native._ptr(w), ctypes.byref(m)))
        def good():          # entries are collected through an atomic counter: compare them in (i, j) order
            i_, j_, w_ = r.top(True, max_k=50)
            o = np.lexsort((j_, i_))
            return i_[o], j_[o], w_[o]
        _fails_without_leak(bad, good)
    finally:
        r.free()


def test_second_order_tables_that_do_not_fit(gpu_ctx):
    """Star with a hub of degree 100 000: the p, q != 1 tables need sum over edges (t -> v) of outdeg(v) ~ 1e10 entries
    (160 GB), so the walks return GEMB_ERR_NOMEM after the edge offsets were built."""
    from gem_b200 import _native
    hub = 100_000
    n = hub + 1
    indptr = np.concatenate(([0, hub], hub + np.arange(1, hub + 1))).astype(np.int32)
    indices = np.concatenate((np.arange(1, n), np.zeros(hub))).astype(np.int32)
    g = _native.DeviceGraph(gpu_ctx, n, indptr, indices)
    nids = np.arange(n, dtype=np.int32)
    try:
        _fails_without_leak(lambda: g.n2v_walks(nids, 5, 1, p=0.5, q=2.0, seed=9),
                            lambda: g.n2v_walks(nids, 5, 1, seed=9)[0], match='do not fit')
    finally:
        g.free()
