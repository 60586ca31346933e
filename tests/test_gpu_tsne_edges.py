"""t-SNE's kernels at the edges the sklearn goldens (tests/test_gpu_tsne.py) do not reach, each against the oracle
(oracle/tsne_oracle.py) on inputs built here from a seed:

    kNN           k from 1 to TSNE_KMAX = 320 (and the refusal at 321), n around the 64-row query block and the
                  128-column candidate tile, d around the 32-dimension stage up to 1000; exact on small-integer X (ties
                  included), within the derived fp32 selection bound on real X
    calibration   rows whose beta doubles or halves many times, exp underflow (p exactly 0), all-equal d^2
    joint P       its CSR pattern exactly, its values to 1e-14
    PCA start     both sides of the tensor-core Gram switch (n >= 4096), d from 1 to 1024, planted spectra, offsets and
                  column scales
    gradient      angle 0 against the exact sum on small, duplicated, collinear and coincident positions; angles 0.2,
                  0.5 and 1 against bh_gradient, sklearn's tree restated cell by cell, on the goldens' positions and on
                  seeded positions with duplicates; a tree deeper than the 32 levels of the cell keys
    plumbing      the d > 1024 refusal, determinism, device-block ownership"""
import numpy as np
import pytest
import scipy.sparse as sp

from tsne_golden import CASES, load, to

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24       # fp32 unit roundoff


def perplexity_for(k):
    """A perplexity whose neighbour count min(n - 1, int(3 perplexity + 1)) is k (for n > k)."""
    return (k - 0.5) / 3.0


def affinities(ctx, X, perplexity):
    from gem_b200 import _native
    return _native.tsne_affinities(ctx, np.ascontiguousarray(X, np.float32), perplexity)


def assert_rows_ascending(a):
    d, i = a['knn_d2'], a['knn_idx']
    assert np.all((d[:, 1:] > d[:, :-1]) | ((d[:, 1:] == d[:, :-1]) & (i[:, 1:] > i[:, :-1])))


# ------------------------------------------------------------------------------------------------------------- kNN
# (n, d, k): n about the 64-row query block and the 128-column tile, d about the 32-dimension stage, k up to 320
KNN_SHAPES = [(2, 1, 1), (3, 3, 2), (3, 32, 2), (63, 31, 16), (64, 33, 16), (65, 32, 16), (127, 65, 91), (128, 1, 91),
              (129, 100, 91), (129, 1000, 16), (400, 257, 319), (400, 33, 320), (4097, 3, 16), (4097, 65, 320)]


@pytest.mark.parametrize('n,d,k', KNN_SHAPES)
def test_knn_exact_on_integer_data(gpu_ctx, n, d, k):
    """Small integers give exact fp32 d^2 (every partial sum an integer below 2^24), so the selection has no rounding:
    the (d^2, index) lists must equal the oracle's exactly, with the many exact ties broken by the lower index."""
    X = np.random.RandomState(n * 1000 + d).randint(-3, 4, (n, d)).astype(np.float32)
    a = affinities(gpu_ctx, X, perplexity_for(k))
    idx, d2 = to.knn(X, k)
    assert a['knn_idx'].shape == (n, k)
    assert np.array_equal(a['knn_idx'], idx)
    assert np.array_equal(a['knn_d2'].astype(np.float64), d2)


@pytest.mark.parametrize('n,d,k', KNN_SHAPES)
def test_knn_real_data(gpu_ctx, n, d, k):
    """Real X.  The kernel selects by s = sum_c (x_c - y_c)^2 in fp32 (one rounding for the difference, one for each
    fused multiply-add): |s - d^2| <= (d + 2) u d^2 with u = 2^-24 (the standard recursive-sum bound, to first order).
    A neighbour set can therefore differ from the exact one only by indices whose exact d^2 lie within 2 (d + 2) u d^2_k
    of the k-th; the d^2 the oracle keeps for an index it did not select is the GPU's returned one, one more rounding:
    bar (2 d + 6) u of the k-th d^2.  The returned d^2 are fp64 sums rounded to fp32: within 1 ulp of fp32(fp64 d^2)."""
    rng = np.random.RandomState(n * 1000 + d + 7)
    X = (rng.randn(n, d) * rng.uniform(0.5, 2.0, d)).astype(np.float32)
    a = affinities(gpu_ctx, X, perplexity_for(k))
    idx, d2 = to.knn(X, k)
    bad = to.neighbour_mismatches(a['knn_idx'], a['knn_d2'], idx, d2, rel=(2 * d + 6) * U32)
    swapped = sum(set(a['knn_idx'][i].tolist()) != set(idx[i].tolist()) for i in range(n))
    print('n %d d %d k %d: %d rows with swaps at the k-th distance' % (n, d, k, swapped))
    assert not bad
    rows = np.repeat(np.arange(n), k)
    exact = ((X[rows].astype(np.float64) - X[a['knn_idx'].ravel()].astype(np.float64)) ** 2).sum(1)
    e32 = exact.astype(np.float32)
    got = a['knn_d2'].ravel()
    assert np.all(np.abs(got.astype(np.float64) - e32) <= np.spacing(e32))
    assert np.all(a['knn_idx'] != np.arange(n)[:, None])
    assert_rows_ascending(a)


def test_knn_k321_refused(gpu_ctx):
    """k = 321 does not fit the kernel's shared-memory lists: refused before any launch, by both entry points."""
    from gem_b200 import _native
    X = np.random.RandomState(3).randn(400, 8).astype(np.float32)
    for call in (lambda: affinities(gpu_ctx, X, perplexity_for(321)),
                 lambda: _native.tsne(gpu_ctx, X, perplexity_for(321), 12.0, 50.0, 0, 300, 1e-7, 0.5)):
        n0 = _native.lib().gemb_launch_count()
        with pytest.raises(RuntimeError):
            call()
        assert _native.lib().gemb_launch_count() == n0
    assert affinities(gpu_ctx, X, perplexity_for(320))['knn_idx'].shape == (400, 320)


# ----------------------------------------------------------------------------------------------------- calibration
def _calibration_inputs():
    rng = np.random.RandomState(11)
    X = rng.randn(500, 8)
    dup = X.copy()
    dup[:120] = dup[0]                  # 120 identical rows > k + 1 = 92: their lists are all d^2 = 0
    # 8 clusters of ~62 rows 1e3 apart: a row's perplexity is reached inside its own cluster (d^2 ~ 16), and
    # exp(-beta d^2) of the other clusters' rows among its 91 neighbours (d^2 ~ 1e7) underflows to exactly 0
    far = rng.randn(8, 8)[np.arange(500) % 8] * 1e3 + X
    return {'small': X * 1e-4, 'large': far, 'dup_block': dup}


@pytest.fixture(scope='module')
def calibrated(gpu_ctx):
    return {name: (X.astype(np.float32), affinities(gpu_ctx, X, 30.0)) for name, X in _calibration_inputs().items()}


@pytest.mark.parametrize('name', ['small', 'large', 'dup_block'])
def test_calibration(calibrated, name):
    """p_cond against the oracle's bisection on the GPU's own d^2.  The two run the same steps in fp64 with sums in
    different orders, so a row agrees to ~1e-12 unless |H - log perplexity| sits at the 1e-5 tolerance and the two
    stopped one step apart: such rows must both be calibrated.  'large' underflows exp (p exactly 0),
    'small' doubles beta many times, 'dup_block' has rows of equal d^2 (no beta reaches the target: 100 steps)."""
    X, a = calibrated[name]
    ref = to.calibrate(a['knn_d2'], 30.0)
    P = a['p_cond']
    err = np.abs(P - ref).max(1) / ref.max(1)
    apart = np.flatnonzero(err > 1e-12)
    target = np.log(30.0)
    for i in apart:
        Hg = to.entropy(None, P[i:i + 1])[0]
        Ho = to.entropy(None, ref[i:i + 1])[0]
        assert abs(Hg - target) <= 1e-5 + 1e-9 and abs(Ho - target) <= 1e-5 + 1e-9, (i, Hg, Ho)
    print('%s: %d rows stopped a step apart; worst other row %.2e; %d exact zeros'
          % (name, apart.size, np.delete(err, apart).max(), int((P == 0).sum())))
    assert apart.size <= 0.02 * P.shape[0]
    if name == 'large':
        assert (P == 0).any()
    if name == 'dup_block':
        assert np.all(P[:120] == 1.0 / P.shape[1])


@pytest.mark.parametrize('name', ['small', 'large', 'dup_block'])
def test_joint(calibrated, name):
    """The joint P of the GPU's own neighbours and p_cond: the CSR pattern (zeros dropped) exactly, values to 1e-14."""
    X, a = calibrated[name]
    n = X.shape[0]
    R = to.joint(a['knn_idx'], a['p_cond'], n)
    assert np.array_equal(a['p_indptr'], R.indptr) and np.array_equal(a['p_indices'], R.indices)
    assert np.all(np.abs(a['p_val'] - R.data) <= 1e-14 * R.data)
    assert abs(a['p_val'].sum() - 1.0) <= 1e-13
    assert np.all(a['p_val'] > 0)


# ------------------------------------------------------------------------------------------------------- PCA start
def _planted(n, d, rng, offset=0.0, col_scales=False):
    """Rows with singular values 40, 20 and then at most 5 (a clear gap after the second), or, with col_scales,
    independent columns scaled over 1e-3 .. 1e3 (the two widest 1e3 and 3e2, the rest at most 10)."""
    if col_scales:
        s = 10.0 ** rng.uniform(-3, 1, d)
        s[rng.permutation(d)[:2]] = [1e3, 3e2][:d]
        X = rng.randn(n, d) * s
    else:
        r = min(d, 8)
        sv = np.array([40.0, 20.0, 5.0, 4.0, 3.0, 2.0, 1.0, 0.5])[:r]
        U = np.linalg.qr(rng.randn(n, r))[0] * np.sqrt(n)
        V = np.linalg.qr(rng.randn(d, r))[0]
        X = (U * sv) @ V.T
    return X + offset


PCA_CASES = [(34, 1, 0.0, False), (34, 2, 1e3, False), (34, 3, 0.0, True), (4095, 3, 1e3, False),
             (4096, 3, 0.0, False), (4095, 129, 0.0, True), (4096, 257, 1e3, False), (4096, 1024, 0.0, False),
             (20000, 2, 0.0, True), (20000, 129, 1e3, False)]


@pytest.mark.parametrize('n,d,offset,col_scales', PCA_CASES)
def test_pca_start(gpu_ctx, n, d, offset, col_scales):
    """The start of a max_iter = 0 run against the fp64 PCA scores of the same fp32 X."""
    from gem_b200 import _native
    rng = np.random.RandomState(n + d)
    X = _planted(n, d, rng, offset, col_scales).astype(np.float32)
    Y, st = _native.tsne(gpu_ctx, X, 5.0, 12.0, 50.0, 0, 300, 1e-7, 0.5)
    ref = to.pca_start(X)
    err = np.abs(Y - ref).max(0) / np.abs(ref).max(0).clip(1e-300)
    print('n %d d %d offset %g col_scales %s: max error per column / column max %s' % (n, d, offset, col_scales, err))
    assert st['n_iter'] == -1
    assert err[0] <= 1e-4
    if d == 1:
        assert np.all(Y[:, 1] == 0.0)
    else:
        assert err[1] <= 1e-4


# ------------------------------------------------------------------------------------------------------- gradients
def _joint_for(n, seed):
    """A joint P for n points: the oracle's chain on seeded 5-D rows (k = min(n - 1, 31))."""
    X = np.random.RandomState(seed).randn(n, 5)
    k = min(n - 1, 31)
    idx, d2 = to.knn(X, k)
    return to.joint(idx, to.calibrate(d2.astype(np.float32), min(10.0, (n - 1) / 3.0 + 0.1) if n > 2 else 0.5), n)


def _grad_scale(Y, P):
    """Per point, 4 (sum_j p_ij q_ij |y_i - y_j| + sum_j q_ij^2 |y_i - y_j| / Z): the magnitude the fp32 sums cancel
    down from.  Each term is rounded a few times and added into an fp32 total, so the error of a point's gradient is a
    small multiple of u times this (the sum's length enters only through the summation order)."""
    Y = np.asarray(Y, np.float64)
    D = np.sqrt(to.sqdist(Y, Y))
    W = 1.0 / (1.0 + D * D)
    np.fill_diagonal(W, 0.0)
    Pd = P.toarray()
    Z = max(W.sum(), 1e-300)
    return 4.0 * ((Pd * W * D).sum(1) + (W * W * D).sum(1) / Z)


def _check_close(g, ref, scale, rel, what):
    e = np.abs(np.asarray(g, np.float64) - ref).max(1) / np.maximum(scale, 1e-300)
    worst = int(np.argmax(e))
    print('%s: worst |g - ref| / scale %.2e at point %d (bar %.0e)' % (what, e[worst], worst, rel))
    assert np.all(np.isfinite(g))
    assert e[worst] <= rel, (worst, g[worst], ref[worst])


def _positions(n, kind, rng):
    if kind == 'pca':
        # the PCA start's scale (standard deviation ~1e-4) on a jittered grid: no two points within 1e-6, where
        # sklearn's leaf rule and the pairwise rule of the exact sum could differ (random normal points would have some)
        m = int(np.ceil(np.sqrt(n)))
        h = 4e-4 / m
        cell = rng.permutation(m * m)[:n]
        Y = np.stack([cell % m, cell // m], 1) * h + rng.uniform(-h / 4, h / 4, (n, 2))
        return (Y - Y.mean(0)).astype(np.float32)
    if kind == 'run':
        return (rng.randn(n, 2) * 50).astype(np.float32)
    if kind == 'dups':
        Y = rng.randn(n, 2) * 50
        m = max(1, n // 10)
        Y[-m:] = Y[rng.choice(n - m, m)]                                              # exact duplicates
        if n >= 20:
            Y[-2 * m:-m] = Y[rng.choice(n - 2 * m, m)] + rng.uniform(-1e-7, 1e-7, (m, 2))    # clusters inside 2e-7
        return Y.astype(np.float32)
    if kind == 'collinear':
        Y = rng.randn(n, 2) * 50
        Y[:, 1] = 3.0
        return Y.astype(np.float32)
    if kind == 'coincident':
        return np.full((n, 2), 2.5, np.float32)
    raise ValueError(kind)


ANGLE0 = [(n, kind) for n in (2, 3, 255, 256, 257, 5000) for kind in ('pca', 'run', 'dups', 'collinear', 'coincident')
          if not (n < 20 and kind == 'dups')]


@pytest.mark.parametrize('n,kind', ANGLE0)
def test_gradient_angle0_exact(gpu_ctx, n, kind):
    """Angle 0 opens every cell down to sklearn's leaves: the exact sum over the pairs the tree counts (points within
    1e-6 of each other on both axes leave each other out).  Per point within 2e-5 of the magnitude of its terms
    (measured up to 3.5e-6, at n = 5000 with duplicates); the
    KL to 1e-5 (its p and q are float32, as sklearn's are).  Coincident points repel nothing: sum_Q is floored at the fp64 epsilon as sklearn floors it, and the
    gradient is the attraction alone (zero here)."""
    from gem_b200 import _native
    rng = np.random.RandomState(n * 10 + len(kind))
    Y = _positions(n, kind, rng)
    P = _joint_for(n, n)
    g, kl = _native.tsne_gradient(gpu_ctx, Y, P.indptr, P.indices, P.data, 0.0)
    ge, kle = to.exact_gradient(Y, P, tree_pairs=True)
    if kind == 'coincident':
        assert np.all(g == 0.0) and np.abs(ge).max() <= 1e-12
    else:
        _check_close(g, ge, _grad_scale(Y, P), 2e-5, 'n %d %s' % (n, kind))
    print('KL %.10f vs %.10f' % (kl, kle))
    assert abs(kl - kle) <= 1e-5 * max(abs(kle), 1e-3)


def _flips(Y, P, angle):
    """Points whose gradient changes beyond fp32 rounding when the oracle's barycentres are sklearn's running float32
    means instead of fp64 sums: opening decisions the barycentre rounding flips."""
    a, _ = to.bh_gradient(Y, P, angle, barycentre='sklearn')
    b, _ = to.bh_gradient(Y, P, angle, barycentre='sum')
    return int(np.sum(np.abs(a - b).max(1) > 1e-4 * np.abs(b).max()))


def _seeded_bh_positions(n, seed):
    rng = np.random.RandomState(seed)
    Y = rng.randn(n, 2) * 30
    Y[: n // 3] = Y[: n // 3] * 0.1 + 20            # a dense cluster: deep cells
    m = n // 20
    Y[-m:] = Y[rng.choice(n - 2 * m, m)]                                              # exact duplicates
    Y[-2 * m:-m] = Y[rng.choice(n - 2 * m, m)] + rng.uniform(-1e-7, 1e-7, (m, 2))     # clusters inside 2e-7
    return Y.astype(np.float32)


BH_CASES = [(name, pos) for name in CASES for pos in ('Y0', 'Y250', 'Y1000')] + [('seeded', 600), ('seeded', 3000)]


@pytest.mark.parametrize('angle', [0.2, 0.5, 1.0])
@pytest.mark.parametrize('case', BH_CASES, ids=['%s-%s' % c for c in BH_CASES])
def test_gradient_bh(gpu_ctx, case, angle):
    """Angle > 0 against bh_gradient, sklearn's quadtree and walk restated float op by float op (pinned bit for bit to
    sklearn's stored gradients in tests/test_oracle_tsne.py), with the barycentres formed as the GPU forms them (fp64
    sums).  The same opening decisions leave only fp32 rounding: per point within 1e-6 of the magnitude of its terms
    (measured up to 1.8e-7), KL to 1e-6.  One flipped decision moves a point by a cell's whole approximation error, far
    above that.  Positions with pairs 2.5e-7 to 1e-6 apart (the goldens' PCA starts hold 200 to 1500 such pairs)
    get 3e-5 (measured up to 1.7e-5) and the KL 1e-5 (measured 2.5e-6): sklearn's leaves depend on the insertion
    path there (a point within 1e-6 of a leaf's first point across a cell boundary becomes its own leaf), while the
    GPU's leaf is the node whose points all lie within 1e-6 of its lowest-index point, so the two place such a pair's
    mass up to 1e-6 apart."""
    from gem_b200 import _native
    name, pos = case
    if name == 'seeded':
        Y = _seeded_bh_positions(pos, pos)
        P = _joint_for(pos, pos + 1)
    else:
        z = load(name)
        Y, P = z[pos], z['P']
    g, kl = _native.tsne_gradient(gpu_ctx, Y, P.indptr, P.indices, P.data, angle)
    ref, klr = to.bh_gradient(Y, P, angle, barycentre='sum')
    print('%s %s angle %.1f: %d points change with sklearn\'s float32 barycentres' % (name, pos, angle, _flips(Y, P, angle)))
    Y64 = Y.astype(np.float64)
    D = np.abs(Y64[:, None, :] - Y64[None, :, :]).max(-1)
    near = bool(np.any((D <= 1e-6) & (D > 2.5e-7)))
    _check_close(g, ref, _grad_scale(Y, P), 3e-5 if near else 1e-6, '%s %s angle %.1f' % (name, pos, angle))
    assert abs(kl - klr) <= (1e-5 if near else 1e-6) * max(abs(klr), 1e-3)


def _deep_positions():
    """~200 points over +-6000 and pairs 1.5e-6 .. 3e-6 apart near the origin: the root cell is ~12000 wide, so a depth-32
    cell is ~2.8e-6 wide and some pairs share all 32 levels of their cell path without being duplicates (1e-6)."""
    rng = np.random.RandomState(32)
    Y = rng.uniform(-6000, 6000, (200, 2))
    Y[0], Y[1] = (-6000, -6000), (6000, 6000)
    base = rng.uniform(-2e-5, 2e-5, (12, 2))
    sep = np.linspace(1.5e-6, 3e-6, 12)
    pairs = np.concatenate([base, base + np.stack([sep, np.zeros(12)], 1)])
    return np.concatenate([Y, pairs]).astype(np.float32)


def _cell_keys(Y):
    """The 64-bit cell paths of tsne_morton_kernel (fp32 halving of the widened root), for the test's precondition."""
    f = np.float32
    lo = Y.min(0)
    hi = to._widen(Y.max(0))
    keys = []
    for x, y in Y:
        lx, ly, hx, hy = lo[0], lo[1], hi[0], hi[1]
        k = 0
        for _ in range(32):
            cx, cy = f(f(lx + hx) * f(0.5)), f(f(ly + hy) * f(0.5))
            bx, by = int(x >= cx), int(y >= cy)
            lx, hx = (cx, hx) if bx else (lx, cx)
            ly, hy = (cy, hy) if by else (ly, cy)
            k = k << 2 | (bx << 1 | by)
        keys.append(k)
    return keys


def test_gradient_deeper_than_cell_keys(gpu_ctx):
    """Points that share all 32 levels of their cell path but are not duplicates: sklearn's tree keeps splitting until
    they separate, so each sees the other.  At angle 0 the exact sum and bh_gradient; at 0.5 bh_gradient."""
    from gem_b200 import _native
    Y = _deep_positions()
    keys = _cell_keys(Y)
    shared = [(i, j) for i in range(len(Y)) for j in range(i + 1, len(Y)) if keys[i] == keys[j]
              and np.abs(Y[i].astype(np.float64) - Y[j]).max() > 1e-6]
    print('%d non-duplicate pairs share a 64-bit cell path' % len(shared))
    assert shared
    P = _joint_for(len(Y), 5)
    scale = _grad_scale(Y, P)
    g, kl = _native.tsne_gradient(gpu_ctx, Y, P.indptr, P.indices, P.data, 0.0)
    ge, kle = to.exact_gradient(Y, P, tree_pairs=True)
    _check_close(g, ge, scale, 1e-5, 'angle 0 vs exact')
    ref, _ = to.bh_gradient(Y, P, 0.0)
    _check_close(g, ref, scale, 1e-5, 'angle 0 vs bh_gradient')
    g5, kl5 = _native.tsne_gradient(gpu_ctx, Y, P.indptr, P.indices, P.data, 0.5)
    ref5, klr5 = to.bh_gradient(Y, P, 0.5, barycentre='sum')
    _check_close(g5, ref5, scale, 1e-5, 'angle 0.5 vs bh_gradient')
    assert abs(kl - kle) <= 1e-5 * abs(kle) and abs(kl5 - klr5) <= 1e-6 * abs(klr5)


# ------------------------------------------------------------------------------------------------------- plumbing
def test_d1025_refused_before_any_launch(gpu_ctx):
    """The PCA start's Jacobi eigensolver takes at most 1024 columns: gemb_tsne refuses d = 1025 before any device work
    (the kNN would otherwise run first), and tsne() before creating a context."""
    from gem_b200 import _native
    from gem_b200.evaluation.visualize_embedding import tsne
    X = np.random.RandomState(0).randn(100, 1025).astype(np.float32)
    n0 = _native.lib().gemb_launch_count()
    with pytest.raises(RuntimeError, match='1024'):
        _native.tsne(gpu_ctx, X, 30.0, 12.0, 50.0, 0, 300, 1e-7, 0.5)
    assert _native.lib().gemb_launch_count() == n0
    with pytest.raises(ValueError, match='1024'):
        tsne(X)
    assert _native.lib().gemb_launch_count() == n0


def test_deterministic_and_owned(gpu_ctx):
    """Two calls give the same bits (kNN at k = 320 over several tiles; the gradient on duplicates at angle 0.5), and
    no device block outlives its call."""
    from gem_b200 import _native
    X = np.random.RandomState(9).randn(4097, 65).astype(np.float32)
    Y = _seeded_bh_positions(3000, 3000)
    P = _joint_for(3000, 3001)
    calls = [lambda: affinities(gpu_ctx, X, perplexity_for(320)),
             lambda: _native.tsne_gradient(gpu_ctx, Y, P.indptr, P.indices, P.data, 0.5)]
    first = [c() for c in calls]
    before = _native.mem_live_blocks()
    second = [c() for c in calls]
    assert _native.mem_live_blocks() == before
    for k in first[0]:
        assert first[0][k].tobytes() == second[0][k].tobytes(), k
    assert first[1][0].tobytes() == second[1][0].tobytes() and first[1][1] == second[1][1]
