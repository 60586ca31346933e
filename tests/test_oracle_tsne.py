"""The fp64 t-SNE oracle (oracle/tsne_oracle.py) pinned to sklearn's goldens (tests/golden/make_golden_tsne.py): kNN,
calibration, symmetrisation, PCA start, the exact gradient and KL, and trustworthiness.  CPU only."""
import numpy as np
import pytest

from tsne_golden import CASES, load, to


@pytest.mark.parametrize('name', CASES)
def test_knn_and_calibration(name):
    z = load(name)
    k = z['knn_idx'].shape[1]
    idx, d2 = to.knn(z['X'], k)
    assert not to.neighbour_mismatches(idx, d2, z['knn_idx'], z['knn_d2'])
    # sklearn's calibrated rows (stored as float32) against the oracle's on the same neighbour sets
    P = z['p_cond_oracle'][z['p_rows']]
    assert np.all(np.abs(P - z['p_cond']) <= 1e-6 * z['p_cond'] + 1e-12)
    H = to.entropy(z['knn_d2'], z['p_cond_oracle'])
    assert np.all(np.abs(H - np.log(float(z['perplexity']))) <= 1e-5 + 1e-9)


@pytest.mark.parametrize('name', CASES)
def test_joint_probabilities(name):
    P = load(name)['P']
    assert P.nnz == int(load(name)['nnz_P'])
    assert abs(P.sum() - 1.0) < 1e-12 and abs(P - P.T).max() <= 1e-18


@pytest.mark.parametrize('name', CASES)
def test_pca_start(name):
    z = load(name)
    Y = to.pca_start(z['X'])
    tol = 1e-3 if str(z['pca_solver']) == 'randomized' else 1e-5
    assert np.linalg.norm(Y - z['Y0']) <= tol * np.linalg.norm(z['Y0'])


@pytest.mark.parametrize('name', CASES)
@pytest.mark.parametrize('pos', ['Y0', 'Y250', 'Y1000'])
def test_exact_gradient(name, pos):
    z = load(name)
    g, kl = to.exact_gradient(z[pos], z['P'])
    ref = z['grad_exact_' + pos]
    assert np.linalg.norm(g - ref) <= 1e-6 * np.linalg.norm(ref)
    assert abs(kl - float(z['kl_exact_' + pos])) <= 1e-6 * max(1.0, abs(kl))


@pytest.mark.parametrize('name', CASES)
def test_descend_matches_sklearn_update(name):
    """One step from the start equals sklearn's first update: gains 1 -> 0.8 (update 0), Y - lr * 0.8 * grad."""
    z = load(name)
    n = z['X'].shape[0]
    P = z['P']
    lr = max(n / 12.0 / 4.0, 50.0)
    g, _ = to.exact_gradient(z['Y0'], P, 12.0)
    Y1 = to.descend(z['Y0'], P, 1, 12.0, 0.5, lr)
    assert np.allclose(Y1, z['Y0'] - lr * 0.8 * g, rtol=1e-12, atol=1e-18)


@pytest.mark.parametrize('name', CASES)
def test_trustworthiness(name):
    """Karate's HOPE rows repeat (equal input distances), and the input ranks of tied rows are sklearn's argsort
    order there: a few ranks differ."""
    z = load(name)
    tol = 5e-3 if name == 'tsne_karate_d4' else 1e-6
    assert abs(to.trustworthiness(z['X'].astype(np.float64), z['Y1000'].astype(np.float64), 12) - float(z['trust12'])) < tol


@pytest.mark.parametrize('name', CASES)
@pytest.mark.parametrize('pos', ['Y0', 'Y250', 'Y1000'])
def test_bh_gradient_is_sklearns(name, pos):
    """bh_gradient against sklearn's own _kl_divergence_bh at angle 0 and 0.5, bit for bit: the quadtree, the opening
    decisions and every float32 step are restated operation by operation (and the KL summed in float32 in CSR order as
    sklearn sums it), so there is no rounding left to allow for, and none is allowed.  Measured: equal at all 24
    (case, position, angle) triples.  For scale, sklearn's own Barnes-Hut error at angle 0.5 is 1.5e-7 to 0.89 of
    |g_exact| on these positions, so a bar at its size could not tell a wrong tree from a right one."""
    z = load(name)
    for angle, tag in ((0.0, '0'), (0.5, '05')):
        g, kl = to.bh_gradient(z[pos], z['P'], angle, kl_float32=True)
        assert g.dtype == np.float32 and np.array_equal(g, z['grad_bh%s_%s' % (tag, pos)]), angle
        assert kl == float(z['kl_bh%s_%s' % (tag, pos)]), angle


@pytest.mark.parametrize('name', ['tsne_karate_d4', 'tsne_mix2000_d64'])
def test_bh_gradient_angle0_is_the_tree_pairs_sum(name):
    """At angle 0 every cell is opened to sklearn's leaves: bh_gradient is the fp64 exact sum over the pairs the tree
    counts, up to float32 rounding: measured at most 5.7e-5 of |g| (bar 2e-4) and 2.2e-6 of the KL (bar 1e-5)."""
    z = load(name)
    for pos in ('Y0', 'Y1000'):
        g, kl = to.bh_gradient(z[pos], z['P'], 0.0)
        ge, kle = to.exact_gradient(z[pos], z['P'], tree_pairs=True)
        assert np.linalg.norm(g - ge) <= 2e-4 * np.linalg.norm(ge)
        assert abs(kl - kle) <= 1e-5 * abs(kle)


def test_knn_blocks_do_not_change_results(monkeypatch):
    """knn and sqdist work in row blocks: the results are the same bits whatever the block size."""
    X = np.random.RandomState(4).randn(300, 7)
    idx, d2 = to.knn(X, 20)
    D = to.sqdist(X, X)
    monkeypatch.setattr(to, '_BLOCK_ELEMS', 1000)
    idx2, d22 = to.knn(X, 20)
    assert np.array_equal(idx, idx2) and np.array_equal(d2, d22)
    assert np.array_equal(D, to.sqdist(X, X))
