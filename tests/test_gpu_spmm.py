"""SpMM parity on the GPU: gemb_spmm (through the C ABI, host buffers) vs scipy.sparse on the same
seeded inputs, Y = alpha op(A) X + gamma Xself + delta X0 (the Horner sweep: gamma = 0, delta = 1; the Chebyshev step:
Xself = X).  fp32 accumulate in row order -> tolerance 2e-6 relative to the row's
|alpha| |A| |X| + |gamma| |Xself| + |delta| |X0| bound; with small-integer data every partial sum is exact and the
result must be exact."""
import numpy as np
import pytest

from conftest import load_karate_nx, load_sbm1024_nx

pytestmark = pytest.mark.gpu

BULK_CAP = 3072            # spmm.cu: ids staged per row tile (+ 4), above that the tile reads its ids from global memory
HEAVY_DEG, HEAVY_CHUNK = 128, 512   # common.cuh: rows above HEAVY_DEG go to the chunk kernels, HEAVY_CHUNK per chunk


def _check(ctx, csr, b, alpha, use_x0, transpose, seed=0, gamma=0.0, use_self=False, delta=1.0, exact=False):
    from gem_b200 import _native
    rng = np.random.default_rng(seed)
    alpha, gamma, delta = (float(np.float32(v)) for v in (alpha, gamma, delta))     # what the kernel computes with
    t = csr.transpose()
    g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, csr.data_f32(), t.indptr, t.indices, t.data_f32())
    if exact:
        draw = lambda: rng.integers(-4, 5, (csr.n, b)).astype(np.float32)
    else:
        draw = lambda: rng.standard_normal((csr.n, b)).astype(np.float32)
    X = draw()
    X0 = draw() if use_x0 else None
    Y = g.spmm(X, alpha=alpha, X0=X0, transpose=transpose, gamma=gamma, Xself=X if use_self else None, delta=delta)
    g.free()
    A = csr.to_scipy().astype(np.float64)
    if transpose:
        A = A.T.tocsr()
    X64 = X.astype(np.float64)
    ref = alpha * (A @ X64)
    bound = abs(alpha) * (abs(A) @ np.abs(X64)) + 1e-30
    if use_self:
        ref = ref + gamma * X64
        bound = bound + abs(gamma) * np.abs(X64)
    if use_x0:
        ref = ref + delta * X0.astype(np.float64)
        bound = bound + abs(delta) * np.abs(X0.astype(np.float64))
    if exact:
        assert np.array_equal(Y, ref), np.abs(Y - ref).max()
        return
    err = np.abs(Y - ref) / bound
    assert err.max() < 2e-6, err.max()


@pytest.mark.parametrize('b', [4, 8, 20, 80, 96, 144, 260])
def test_spmm_karate(gpu_ctx, b):
    from gem_b200 import graph as hg
    csr = hg.from_networkx(load_karate_nx())
    _check(gpu_ctx, csr, b, 0.01, True, False)
    _check(gpu_ctx, csr, b, 1.0, False, True)


def test_spmm_sbm1024_weighted(gpu_ctx):
    from gem_b200 import graph as hg
    G, _ = load_sbm1024_nx()
    csr = hg.from_networkx(G)
    rng = np.random.default_rng(1)
    csr.data = rng.uniform(0.1, 2.0, csr.nnz)                   # weighted variant
    for tr in (False, True):
        _check(gpu_ctx, csr, 80, 0.37, True, tr)
        _check(gpu_ctx, csr, 80, -1.5, False, tr)


def test_spmm_rmat_skewed_and_empty_rows(gpu_ctx):
    from gem_b200 import synth
    csr = synth.rmat(scale=12, edge_factor=8, seed=3)           # heavy skew + isolated nodes
    deg = np.diff(csr.indptr)
    assert deg.max() > 50 * max(1, np.median(deg)) and (deg == 0).any()
    _check(gpu_ctx, csr, 80, 0.5, True, False)
    _check(gpu_ctx, csr, 16, 1.0, False, False)
    # hubs of several thousand neighbours: rows above 128 nonzeros go through the chunked heavy-row kernels
    # (several 512-nonzero chunks per hub), weighted and unweighted, wide and narrow blocks, A and A^T
    big = synth.rmat(scale=15, edge_factor=8, seed=4)
    assert np.diff(big.indptr).max() > 4 * 512
    _check(gpu_ctx, big, 80, 0.5, True, False)
    _check(gpu_ctx, big, 8, -1.0, False, True)
    big.data = np.random.default_rng(9).uniform(0.1, 2.0, big.nnz)
    _check(gpu_ctx, big, 80, 0.25, True, True)
    _check(gpu_ctx, big, 144, 1.0, False, False)


def test_spmm_linearity_full_size_property(gpu_ctx):
    """Size-independent property at a size the CPU check would still finish: A(x+y) = Ax + Ay, and the
    Horner epilogue X0 + alpha*A*X is consistent with the plain product."""
    from gem_b200 import _native, synth
    csr = synth.sbm(n=200_000, block=1000, seed=5)
    g = _native.DeviceGraph(gpu_ctx, csr.n, csr.indptr, csr.indices, None)
    rng = np.random.default_rng(2)
    X = rng.standard_normal((csr.n, 80)).astype(np.float32)
    Z = rng.standard_normal((csr.n, 80)).astype(np.float32)
    a, b2, c = g.spmm(X), g.spmm(Z), g.spmm(X + Z)
    assert np.abs(c - (a + b2)).max() <= 2e-5 * np.abs(c).max()
    d = g.spmm(X, alpha=0.25, X0=Z)
    assert np.abs(d - (Z + 0.25 * a)).max() <= 2e-6 * np.abs(d).max()
    ref = csr.to_scipy() @ X.astype(np.float64)
    assert np.abs(a - ref).max() <= 1e-5 * np.abs(ref).max()
    g.free()


def _hub_graph(weights=None):
    """R-MAT scale 12: 4096 rows, 79 of them above HEAVY_DEG (one above HEAVY_CHUNK), 1102 empty rows.
    weights: None (unweighted), 'real' (uniform 0.1..2) or 'eighths' (signed multiples of 1/8, exact in fp32)."""
    from gem_b200 import synth
    csr = synth.rmat(scale=12, edge_factor=8, seed=3)
    deg = np.diff(csr.indptr)
    assert (deg > HEAVY_DEG).any() and (deg <= HEAVY_DEG).any() and (deg > HEAVY_CHUNK).any()
    rng = np.random.default_rng(11)
    if weights == 'real':
        csr.data = rng.uniform(0.1, 2.0, csr.nnz)
    elif weights == 'eighths':
        csr.data = _eighths(rng, csr.nnz)
    return csr


def _eighths(rng, m):
    """nonzero multiples of 1/8 in [-2, 2]: with X in {-4..4} every partial sum of a row stays exact in fp32"""
    return rng.integers(1, 17, m) * rng.choice([-1.0, 1.0], m) / 8


def _csr_from_degrees(deg, n, rng):
    """n_rows = len(deg) rows of the given degrees, distinct sorted column ids in [0, n)."""
    from gem_b200 import graph as hg
    deg = np.asarray(deg, dtype=np.int64)
    indptr = np.zeros(deg.size + 1, dtype=np.int64)
    np.cumsum(deg, out=indptr[1:])
    cols = [np.sort(rng.choice(n, int(d), replace=False)) for d in deg]
    indices = np.concatenate(cols).astype(np.int32) if indptr[-1] else np.zeros(0, np.int32)
    return hg.HostCSR(n, indptr, indices)


def _tile_slices(csr, tile_rows):
    """Staged slice length of every row tile by the bulk kernel's formula: a0 = s & ~3, cnt = (e - a0 + 3) & ~3."""
    s = csr.indptr[0:csr.n:tile_rows]
    e = csr.indptr[np.minimum(np.arange(tile_rows, csr.n + tile_rows, tile_rows), csr.n)]
    a0 = s & ~3
    return s, e, (e - a0 + 3) & ~3


@pytest.mark.parametrize('weights', [None, 'real'])
def test_spmm_three_term_epilogue(gpu_ctx, weights):
    """Y = alpha A X + gamma X + delta X0 as the Chebyshev step calls it (Xself = X), on light and heavy rows, A and
    A^T; Xself without X0; alpha = 0 (the epilogue alone)."""
    csr = _hub_graph(weights)
    for tr in (False, True):
        _check(gpu_ctx, csr, 80, 0.37, True, tr, gamma=-1.3, use_self=True, delta=-0.45)
        _check(gpu_ctx, csr, 80, -2.5, False, tr, gamma=0.7, use_self=True)
    _check(gpu_ctx, csr, 80, 0.0, True, False, gamma=1.7, use_self=True, delta=-3.2)
    _check(gpu_ctx, csr, 16, 1.1, True, False, gamma=-0.3, use_self=True, delta=2.0)


@pytest.mark.parametrize('weights', [None, 'eighths'])
def test_spmm_exact_arithmetic(gpu_ctx, weights):
    """Small integers and multiples of 1/8: every partial sum is exact in fp32, so Y must equal the fp64 result
    exactly whatever the summation order -- a missed or double-counted nonzero shows at any magnitude."""
    csr = _hub_graph(weights)
    for tr in (False, True):
        _check(gpu_ctx, csr, 80, 3, True, tr, gamma=-2, use_self=True, delta=5, exact=True)
        _check(gpu_ctx, csr, 80, -1, True, tr, exact=True)
        _check(gpu_ctx, csr, 80, 2, False, tr, gamma=3, use_self=True, exact=True)
    _check(gpu_ctx, csr, 80, 0, True, False, gamma=-3, use_self=True, delta=2, exact=True)


@pytest.mark.parametrize('b', [4, 12, 1024])
def test_spmm_block_widths_hub_graph(gpu_ctx, b):
    """b = 4: one thread per row; b = 12: groups of 3 threads, which do not divide the 256 threads of a CTA;
    b = 1024: one row per CTA pass (4-row tiles)."""
    csr = _hub_graph('real')
    _check(gpu_ctx, csr, b, 0.5, True, False)
    _check(gpu_ctx, csr, b, -1.25, True, True, gamma=0.6, use_self=True, delta=-1.5)
    exact = _hub_graph('eighths')
    _check(gpu_ctx, exact, b, 2, True, False, gamma=-1, use_self=True, delta=3, exact=True)
    _check(gpu_ctx, _hub_graph(), b, 1, False, True, exact=True)


def _threshold_graph(rng):
    """Light rows (degree 0..8) with single rows of degree 128 (the last light degree), 129 (one chunk), 512, 513
    (two chunks: 512 + 1) and 1025 (three chunks) at the first, last and inner positions of 48-row tiles."""
    n = 6000
    deg = rng.integers(0, 9, n)
    special = {144: 128, 2001: 128, 287: 129, 2000: 129, 452: 512, 673: 513, 1006: 1025, 5999: 1025}
    for r, d in special.items():
        deg[r] = d
    csr = _csr_from_degrees(deg, n, rng)
    got = np.diff(csr.indptr)
    assert sorted(got[got > 8].tolist()) == sorted(special.values())
    return csr


@pytest.mark.parametrize('b', [80, 12, 4])
def test_spmm_heavy_threshold_and_chunk_boundaries(gpu_ctx, b):
    rng = np.random.default_rng(21)
    csr = _threshold_graph(rng)
    _, _, cnt = _tile_slices(csr, 4 * (256 // (b // 4)))
    if b == 80:
        assert (cnt <= BULK_CAP + 4).all()       # every tile is staged, the heavy rows among them are skipped
    for tr in (False, True):
        _check(gpu_ctx, csr, b, 0.8, True, tr, gamma=-0.4, use_self=True, delta=1.3)
        _check(gpu_ctx, csr, b, 1.0, False, tr)
    csr.data = _eighths(rng, csr.nnz)
    _check(gpu_ctx, csr, b, 3, True, False, gamma=2, use_self=True, delta=-1, exact=True)
    _check(gpu_ctx, csr, b, -2, True, True, exact=True)


def _capacity_graph(rng, n_tiles=16, tile=48):
    """Tiles of light rows (degree <= 128, a few empty) whose staged slices alternate between cnt = BULK_CAP + 4
    (the largest that is staged) and BULK_CAP + 8 (the smallest that is not), from every start alignment."""
    deg, s = [], 0
    for t in range(n_tiles):
        cnt = BULK_CAP + 4 if t % 2 == 0 else BULK_CAP + 8
        a0 = s & ~3
        e = a0 + cnt - int(rng.integers(0, 4))       # (e - a0 + 3) & ~3 == cnt
        d = np.zeros(tile, dtype=np.int64)
        full = rng.choice(tile, tile - 4, replace=False)
        d[full] = rng.multinomial(e - s, np.full(full.size, 1.0 / full.size))
        deg.append(d)
        s = e
    return _csr_from_degrees(np.concatenate(deg), n_tiles * tile, rng)


def test_spmm_staging_capacity_boundary(gpu_ctx):
    """b = 80 (48-row tiles), no heavy row: tiles just under the staging capacity read their ids from shared memory,
    tiles just over read them from global memory -- both must give the same exact result."""
    rng = np.random.default_rng(31)
    csr = _capacity_graph(rng)
    assert np.diff(csr.indptr).max() <= HEAVY_DEG
    s, e, cnt = _tile_slices(csr, 48)
    assert (cnt == BULK_CAP + 4).sum() == 8 and (cnt == BULK_CAP + 8).sum() == 8
    assert len(set((s % 4).tolist())) > 1                          # staged slices start at several alignments
    _check(gpu_ctx, csr, 80, 0.9, True, False, gamma=-0.7, use_self=True, delta=0.3)
    _check(gpu_ctx, csr, 80, 1.0, False, False)
    _check(gpu_ctx, csr, 80, -1.5, True, True, gamma=0.25, use_self=True, delta=2.0)
    csr.data = _eighths(rng, csr.nnz)
    _check(gpu_ctx, csr, 80, 3, True, False, gamma=-2, use_self=True, delta=1, exact=True)
    _check(gpu_ctx, csr, 80, 1, False, False, exact=True)


def test_spmm_graph_without_edges(gpu_ctx):
    """No nonzeros: Y is the epilogue alone, exactly (gamma, delta powers of two: both products are exact and the
    kernel's fma rounds the sum once, as fp32 addition does)."""
    from gem_b200 import _native
    n, b = 5000, 80
    g = _native.DeviceGraph(gpu_ctx, n, np.zeros(n + 1, np.int32), np.zeros(0, np.int32), None)
    rng = np.random.default_rng(41)
    X = rng.standard_normal((n, b)).astype(np.float32)
    X0 = rng.standard_normal((n, b)).astype(np.float32)
    assert np.array_equal(g.spmm(X, alpha=0.7, X0=X0, gamma=0.5, Xself=X, delta=-2.0),
                          np.float32(0.5) * X + np.float32(-2.0) * X0)
    assert np.array_equal(g.spmm(X, alpha=0.7, X0=X0), X0)
    assert np.array_equal(g.spmm(X, alpha=-1.0, gamma=0.25, Xself=X), np.float32(0.25) * X)
    assert np.array_equal(g.spmm(X, transpose=True), np.zeros((n, b), np.float32))
    g.free()


def test_spmm_rejects_bad_block_width(gpu_ctx):
    from gem_b200 import _native
    from gem_b200 import graph as hg
    csr = hg.from_networkx(load_karate_nx())
    g = _native.DeviceGraph(gpu_ctx, csr.n, csr.indptr, csr.indices, None)
    for b in (1028, 6):
        with pytest.raises(RuntimeError, match='bad argument'):
            g.spmm(np.ones((csr.n, b), np.float32))
    deg = np.diff(csr.indptr).astype(np.float32)
    assert np.array_equal(g.spmm(np.ones((csr.n, 4), np.float32)), np.repeat(deg[:, None], 4, axis=1))   # still usable
    g.free()


def test_spmm_three_term_is_reproducible(gpu_ctx):
    """The heavy rows are summed in a fixed chunk order (no atomics): the same input gives the same bits."""
    from gem_b200 import _native, synth
    csr = synth.rmat(scale=15, edge_factor=8, seed=4)
    assert np.diff(csr.indptr).max() > 4 * HEAVY_CHUNK
    csr.data = np.random.default_rng(9).uniform(0.1, 2.0, csr.nnz)
    g = _native.DeviceGraph(gpu_ctx, csr.n, csr.indptr, csr.indices, csr.data_f32())
    rng = np.random.default_rng(5)
    X = rng.standard_normal((csr.n, 80)).astype(np.float32)
    X0 = rng.standard_normal((csr.n, 80)).astype(np.float32)
    Y1 = g.spmm(X, alpha=0.3, X0=X0, gamma=-1.1, Xself=X, delta=0.6)
    Y2 = g.spmm(X, alpha=0.3, X0=X0, gamma=-1.1, Xself=X, delta=0.6)
    g.free()
    assert np.array_equal(Y1, Y2)
