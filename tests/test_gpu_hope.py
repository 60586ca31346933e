"""HOPE parity on the GPU, through the reference-facing plugin class (gem_b200.embedding.hope.HOPE ->
ctypes -> libgemb200.so).  Compared with
  * the reference's own goldens (tests/golden/karate_HOPE.txt, sbm1024.npz:hope_golden) and the
    reference-class outputs in tests/golden/ref_hope_*.npz,
  * the fp64 oracle (oracle/hope_oracle.py) on the same inputs.
Tolerances (fp32 arithmetic vs the reference's fp64; SURVEY H2): sigma 2e-5 relative, reconstruction
||X1 X2^T - ref||_F/||ref||_F 2e-4, principal angle of the well separated part of the subspace 0.05 deg,
|mean(target - X)| < 1e-3 (the reference's own bar, tests/test_sbm.py:94)."""
import numpy as np
import pytest

from conftest import golden_path, load_karate_nx, load_sbm1024_nx, nx_from_npz

pytestmark = pytest.mark.gpu

SIG_RTOL = 2e-5
RECON_TOL = 2e-4


def _fresh_hope(**kw):
    from gem_b200.embedding.hope import HOPE
    HOPE.hyper_params.clear()
    HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
    return HOPE(**kw)


def _printed_svd_error(out):
    """The value of hope.py:38-40's line in captured stdout."""
    lines = [ln for ln in out.splitlines() if ln.startswith('SVD error (low rank): ')]
    assert len(lines) == 1, out
    return float(lines[0].split(': ', 1)[1])


def test_karate_golden(gpu_ctx, hope_oracle, capsys):
    ho = hope_oracle
    G = load_karate_nx()
    gold = np.loadtxt(golden_path('karate_HOPE.txt'))
    m = _fresh_hope(d=4, beta=0.01, oversample=32, tol=1e-9, max_iters=60, compute_residual=1)
    X = m.learn_embedding(graph=G, is_weighted=True, no_python=True)
    assert X.shape == (34, 4) and m.get_embedding() is X
    Xa = ho.align_pair_signs(X, gold)
    assert np.allclose(Xa, gold, atol=2e-6), np.abs(Xa - gold).max()     # reference: np.allclose
    sig = ho.sigma_from_embedding(gold)
    assert np.allclose(m._sigma, sig, rtol=SIG_RTOL)
    assert np.all(np.diff(m._sigma) >= 0)
    assert m.stats['resid_max'] < 1e-4
    # get_edge_weight / get_reconstructed_adj follow the reference (hope.py:43-44)
    A = m.get_reconstructed_adj()
    assert abs(A[3, 5] - np.dot(X[3, :2], X[5, 2:])) < 1e-7 and A[4, 4] == 0
    # the reference prints 0.053622; X is within 2e-6 of the optimum, whose error is stationary (Eckart-Young)
    assert abs(_printed_svd_error(capsys.readouterr().out) - 0.053622) <= 2e-6


def test_karate_svd_error_above_the_norm_bound(gpu_ctx, hope_oracle, capsys):
    """Karate as the reference loads it is strictly upper triangular: rho(A) = 0 while beta ||A||_2 = 1.52 at
    beta = 0.3.  The series is finite, the solver accepts it, and the reference prints 1.541227 for d = 4; so must
    the plugin, rather than 'unavailable'."""
    ho = hope_oracle
    G = load_karate_nx()
    m = _fresh_hope(d=4, beta=0.3, oversample=32, tol=1e-9, max_iters=60)
    X = m.learn_embedding(graph=G)
    Xo, so = ho.hope_dense_lapack(ho.adjacency_from_nx(G), 4, 0.3)
    assert np.allclose(m._sigma, so, rtol=SIG_RTOL)
    assert ho.recon_rel_err(X, Xo) < RECON_TOL
    e = _printed_svd_error(capsys.readouterr().out)
    assert abs(e - 1.541227) <= 1e-5 * 1.541227, e


@pytest.mark.parametrize('algorithm', [1, 2])
def test_sbm1024_golden(gpu_ctx, hope_oracle, algorithm):
    """algorithm 1 = subspace iteration on S^T S (Katz sweeps); 2 = Chebyshev filter on A (S = f(A), symmetric A)."""
    ho = hope_oracle
    G, z = load_sbm1024_nx()
    gold = z['hope_golden']
    m = _fresh_hope(d=256, beta=0.01, oversample=128, tol=1e-9, max_iters=400, min_iters=8, algorithm=algorithm)
    X = m.learn_embedding(graph=G, is_weighted=True, no_python=True)
    assert m.stats['algorithm'] == algorithm
    assert abs(np.mean(gold - X)) < 1e-3                                   # tests/test_sbm.py:94
    sg, sx = ho.sigma_from_embedding(gold), np.asarray(m._sigma, dtype=np.float64)
    assert np.allclose(sx, sg, rtol=1e-4), np.abs(sx / sg - 1).max()
    # top of the spectrum is well separated (3 communities): tight subspace check there
    k = 128
    U, Ug = X[:, :k], gold[:, :k]
    assert ho.principal_angles_deg(U[:, -3:], Ug[:, -3:])[0] < 0.05
    assert ho.recon_rel_err(X, gold) < 5e-2      # bulk singular values are nearly degenerate at the cut


@pytest.mark.parametrize('name,recon_tol,algorithm', [('karate_d16', RECON_TOL, 0), ('sbm1024_d16', 2e-3, 1),
                                                      ('sbm1024_d16', 2e-3, 2), ('randw200_d32', RECON_TOL, 0)])
def test_against_reference_class_outputs(gpu_ctx, hope_oracle, name, recon_tol, algorithm):
    ho = hope_oracle
    z = np.load(golden_path('ref_hope_%s.npz' % name))
    G = nx_from_npz(z)
    d, beta, Xref = int(z['d']), float(z['beta']), z['X']
    m = _fresh_hope(d=d, beta=beta, oversample=64, tol=1e-10, max_iters=300, min_iters=6, compute_residual=1,
                    algorithm=algorithm)
    X = m.learn_embedding(graph=G)
    assert m.stats['algorithm'] == (algorithm or 1)          # directed inputs take the general solver
    assert np.allclose(m._sigma, ho.sigma_from_embedding(Xref), rtol=SIG_RTOL, atol=1e-9)
    assert ho.recon_rel_err(X, Xref) < recon_tol, ho.recon_rel_err(X, Xref)
    assert m.stats['resid_max'] < 1e-3


@pytest.mark.parametrize('algorithm', [1, 2])
def test_repeated_singular_values_cliques(gpu_ctx, hope_oracle, algorithm):
    """Ring of cliques: exactly repeated sigma (and negative eigenvalues of A) -> vectors are not unique;
    sigma and residuals are."""
    ho = hope_oracle
    z = np.load(golden_path('ref_hope_cliques_d24.npz'))
    G = nx_from_npz(z)
    m = _fresh_hope(d=24, beta=0.05, oversample=40, tol=1e-10, max_iters=200, compute_residual=1, algorithm=algorithm)
    X = m.learn_embedding(graph=G)
    assert np.allclose(m._sigma, ho.sigma_from_embedding(z['X']), rtol=SIG_RTOL)
    A = ho.adjacency_from_nx(G)
    r1, r2, _, _ = ho.svd_residuals(A, 0.05, X, ho.katz_terms_needed(A, 0.05, 1e-14))
    assert max(r1.max(), r2.max()) < 2e-5


def test_symmetric_solver_refuses_directed_input(gpu_ctx):
    m = _fresh_hope(d=4, beta=0.01, algorithm=2)
    with pytest.raises(RuntimeError, match='symmetric'):
        m.learn_embedding(graph=load_karate_nx())


def test_bipartite_negative_spectrum(gpu_ctx, hope_oracle):
    """Bipartite graph: spectrum symmetric about 0, so |f(l)| ranks +l above -l but both ends matter."""
    import networkx as nx
    ho = hope_oracle
    B = nx.DiGraph(nx.complete_bipartite_graph(9, 14))
    B.add_edges_from([(0, 1), (1, 0), (10, 11), (11, 10)])      # break exact bipartiteness a little
    A = ho.adjacency_from_nx(B)
    Xo, so = ho.hope_dense_lapack(A, 8, 0.05)
    for algorithm in (1, 2):
        m = _fresh_hope(d=8, beta=0.05, oversample=19, tol=1e-10, max_iters=200, compute_residual=1, algorithm=algorithm)
        X = m.learn_embedding(graph=B)
        assert np.allclose(m._sigma, so, rtol=SIG_RTOL), (algorithm, m._sigma, so)
        assert ho.recon_rel_err(X, Xo) < RECON_TOL
        assert m.stats['resid_max'] < 1e-4


def test_divergent_beta_fails_loudly(gpu_ctx):
    G, _ = load_sbm1024_nx()
    m = _fresh_hope(d=8, beta=0.5)
    with pytest.raises(RuntimeError, match='Katz series'):
        m.learn_embedding(graph=G)


@pytest.mark.parametrize('algorithm', [1, 2])
def test_large_sparse_input_properties(gpu_ctx, hope_oracle, algorithm):
    """SBM at 100k nodes through the CSR entry of the plugin; checked with size-independent properties:
    ascending sigma, orthonormal U and V, SVD residuals of the fp64 matrix-free operator, and sigma
    against the CPU sparse oracle (scipy svds on the same Katz operator)."""
    from gem_b200 import synth
    ho = hope_oracle
    csr = synth.sbm(n=100_000, block=1000, seed=11)
    m = _fresh_hope(d=16, beta=0.01, tol=1e-8, max_iters=100, min_iters=4, compute_residual=1, algorithm=algorithm)
    X = m.learn_embedding(graph=csr)
    assert m.stats['algorithm'] == algorithm
    sig = np.asarray(m._sigma, dtype=np.float64)
    assert np.all(np.diff(sig) >= 0)
    A = csr.to_scipy()
    J = ho.katz_terms_needed(A, 0.01, 1e-12)
    r1, r2, U, V = ho.svd_residuals(A, 0.01, X, J, sigma=sig)
    assert np.abs(U.T @ U - np.eye(8)).max() < 1e-4 and np.abs(V.T @ V - np.eye(8)).max() < 1e-4
    assert r1.max() < 5e-3 and r2.max() < 5e-3, (r1.max(), r2.max())
    assert m.stats['resid_max'] < 5e-3
    Xo, so, _ = ho.hope_sparse(A, 16, 0.01, tol=1e-6)
    assert np.allclose(sig[-1], so[-1], rtol=1e-5)               # isolated top value
    assert np.allclose(sig, so, rtol=2e-3)                       # clustered community values


def test_work_buffers_are_reused_between_calls(gpu_ctx):
    """Two learn_embedding calls on the same shape: the second is served from the device block cache
    (gemb_mem_cached_bytes > 0 between the calls), gives bit-identical output although its buffers hold the
    previous call's data, and gemb_mem_trim empties the cache."""
    from gem_b200 import _native, synth
    csr = synth.sbm(n=120_000, block=1000, seed=3)
    m = _fresh_hope(d=32, beta=0.01, tol=1e-6, max_iters=40)
    X1 = m.learn_embedding(graph=csr).copy()
    cached = _native.mem_cached_bytes()
    assert cached >= 5 * 120_000 * 32 * 4            # at least the five n x b work blocks
    X2 = m.learn_embedding(graph=csr)
    assert np.array_equal(X1, X2)
    assert _native.mem_cached_bytes() == cached      # nothing new was allocated for the second call
    _native.mem_trim()
    assert _native.mem_cached_bytes() == 0
    X3 = m.learn_embedding(graph=csr)
    assert np.array_equal(X1, X3)


@pytest.mark.parametrize('algorithm', [1, 2, 3])
def test_power_law_graph_skewed_spectrum(gpu_ctx, hope_oracle, algorithm):
    """R-MAT (BASELINE configs[3] at scale 12): hubs (heavy-row SpMM path), half the nodes isolated, and with
    beta = 0.5 / rho(A) a spectrum whose k-th singular value is ~1e-2 of the first -- the convergence test must
    resolve every sigma_j relative to ITSELF.  sigma vs scipy svds on the same Katz operator, reconstruction
    vs the oracle's."""
    import scipy.sparse.linalg as sla
    from gem_b200 import synth
    ho = hope_oracle
    csr = synth.rmat(scale=12, edge_factor=8, seed=3)
    A = csr.to_scipy().astype(np.float64)
    rho = float(abs(sla.eigsh(A, k=1, which='LA', return_eigenvectors=False)[0]))
    beta = 0.5 / rho
    m = _fresh_hope(d=16, beta=beta, tol=1e-6, max_iters=200, min_iters=4, algorithm=algorithm)
    X = m.learn_embedding(graph=csr)
    assert m.stats['algorithm'] == algorithm and m.stats['converged'] == 1
    sig = np.asarray(m._sigma, dtype=np.float64)
    Xo, so, _ = ho.hope_sparse(A, 16, beta, tol=1e-10)
    assert so[0] < 0.1 * so[-1]                                  # the spectrum IS skewed
    assert np.allclose(sig, so, rtol=2e-4), np.abs(sig / so - 1).max()
    k = 8
    rec = X[:, :k].astype(np.float64) @ X[:, k:].astype(np.float64).T
    reco = Xo[:, :k] @ Xo[:, k:].T
    assert np.linalg.norm(rec - reco) <= 5e-3 * np.linalg.norm(reco)      # fp32 vectors of the small-sigma end


def test_bench_solver_setting_against_fp64_oracle(gpu_ctx, hope_oracle):
    """VERDICT r1 item 1: the solver setting bench.py TIMES (bench.HOPE_SOLVER) compared with the fp64 oracle at a size
    the oracle finishes (SBM n = 100k, same generator / density / d / beta as BASELINE configs[1]).  Tolerances are the
    ones DESIGN.md section 6 states for the headline: the spectrum is one isolated value + a cluster of ~99 values within
    a few percent, and k = 64 cuts inside the cluster, so individual cluster vectors are not comparable -- what is:
      sigma        every one of the k values within the solver's own stopping tolerance (bench.HOPE_SOLVER['tol'] = 4e-3,
                   a bound on the Ritz residual relative to sigma_max, hence by Weyl on every sigma error) of scipy
                   svds(tol=1e-8), relative to the value itself; the isolated top value to 1e-5,
      top-1 angle  the isolated top pair within 0.05 degrees of the oracle's,
      residuals    max_j ||S v_j - sigma_j u_j||, ||S^T u_j - sigma_j v_j|| <= 1e-2 sigma_max against the fp64 operator
                   (the oracle itself run at ARPACK tol=1e-3, the CPU arm's setting, is measured beside it),
      orthonormal  |U^T U - I|, |V^T V - I| <= 1e-4."""
    import os
    import sys
    from gem_b200 import synth
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    ho = hope_oracle
    csr = synth.sbm(n=100_000, block=1000, seed=42)
    d, beta = 128, 0.01
    k = d // 2
    m = _fresh_hope(d=d, beta=beta, compute_residual=1, **bench.HOPE_SOLVER)
    X = m.learn_embedding(graph=csr)
    sig = np.asarray(m._sigma, dtype=np.float64)
    A = csr.to_scipy()
    nthreads = min(32, os.cpu_count() or 1)
    Xo, so, _ = ho.hope_sparse(A, d, beta, katz_tol=1e-12, tol=1e-8, threads=nthreads)
    J = ho.katz_terms_needed(A, beta, 1e-12)
    r1, r2, U, V = ho.svd_residuals(A, beta, X, J, sigma=sig)
    ang = ho.principal_angles_deg(X[:, k - 1:k], Xo[:, k - 1:k])[0]
    orth = max(np.abs(U.T @ U - np.eye(k)).max(), np.abs(V.T @ V - np.eye(k)).max())
    # the CPU arm's own accuracy at its bench setting (ARPACK tol = 1e-3), for the record in the test log
    Xc, sc, _ = ho.hope_sparse(A, d, beta, katz_tol=1e-7, tol=bench.CPU_ARPACK_TOL, threads=nthreads)
    c1, c2, _, _ = ho.svd_residuals(A, beta, Xc, J, sigma=sc)
    print('bench-setting parity: sigma rel err max %.3g (top %.3g), top-1 angle %.3g deg, residual %.3g (GPU reports %.3g), '
          'orth %.3g, iters %d, converged %d | scipy svds(tol=%g): sigma rel err %.3g, residual %.3g'
          % (np.abs(sig / so - 1).max(), abs(sig[-1] / so[-1] - 1), ang, max(r1.max(), r2.max()), m.stats['resid_max'], orth,
             m.stats['iters'], m.stats['converged'], bench.CPU_ARPACK_TOL, np.abs(sc / so - 1).max(), max(c1.max(), c2.max())))
    assert np.all(np.diff(sig) >= 0)
    assert np.allclose(sig, so, rtol=bench.HOPE_SOLVER['tol']), np.abs(sig / so - 1).max()
    assert abs(sig[-1] / so[-1] - 1) < 1e-5
    assert ang < 0.05
    assert max(r1.max(), r2.max()) < 1e-2
    assert orth < 1e-4
    assert abs(m.stats['resid_max'] - max(r2.max(), 0)) < 2e-3          # the library's own fp32 residual tells the truth


def test_lanczos_on_rmat_scale16_converges_and_matches_oracle(gpu_ctx, hope_oracle):
    """BASELINE configs[3] in small (R-MAT scale 16, 65k nodes, beta = 0.5 / rho, d = 128): the thick-restart block
    Lanczos solver (algorithm 3; chosen automatically on such a spectrum) must CONVERGE -- round 1's filtered subspace
    iteration ran to max_iters here -- and agree with scipy svds on the same Katz operator: every sigma to 1e-4, the
    span of the 8 leading pairs to 0.1 degrees, fp64 residuals below 1e-3 sigma_max."""
    import os
    import scipy.sparse.linalg as sla
    from gem_b200 import synth
    ho = hope_oracle
    csr = synth.rmat(scale=16, edge_factor=8, seed=42)
    A = csr.to_scipy().astype(np.float64)
    rho = float(abs(sla.eigsh(A, k=1, which='LA', return_eigenvectors=False)[0]))
    beta = 0.5 / rho
    d, k = 128, 64
    m = _fresh_hope(d=d, beta=beta, tol=1e-5, max_iters=60)          # algorithm = 0: auto
    X = m.learn_embedding(graph=csr)
    assert m.stats['algorithm'] == 3 and m.stats['converged'] == 1, m.stats
    sig = np.asarray(m._sigma, dtype=np.float64)
    nthreads = min(32, os.cpu_count() or 1)
    Xo, so, _ = ho.hope_sparse(A, d, beta, katz_tol=1e-12, tol=1e-10, threads=nthreads)
    assert so[0] < 0.1 * so[-1]
    assert np.allclose(sig, so, rtol=1e-4), np.abs(sig / so - 1).max()
    assert ho.principal_angles_deg(X[:, k - 8:k], Xo[:, k - 8:k])[0] < 0.1
    J = ho.katz_terms_needed(A, beta, 1e-12)
    r1, r2, U, V = ho.svd_residuals(A, beta, X, J, sigma=sig)
    assert max(r1.max(), r2.max()) < 1e-3, (r1.max(), r2.max())
    assert np.abs(U.T @ U - np.eye(k)).max() < 1e-4


def test_lanczos_on_the_clustered_sbm_spectrum(gpu_ctx, hope_oracle):
    """algorithm 3 asked for explicitly on the SBM (one isolated value + a cluster): converges to a residual far below
    what the filtered subspace iteration stops at; sigma vs scipy svds."""
    from gem_b200 import synth
    ho = hope_oracle
    csr = synth.sbm(n=100_000, block=1000, seed=42)
    m = _fresh_hope(d=128, beta=0.01, tol=1e-4, max_iters=60, algorithm=3)
    X = m.learn_embedding(graph=csr)
    assert m.stats['algorithm'] == 3 and m.stats['converged'] == 1
    sig = np.asarray(m._sigma, dtype=np.float64)
    A = csr.to_scipy()
    Xo, so, _ = ho.hope_sparse(A, 128, 0.01, katz_tol=1e-12, tol=1e-8, threads=min(32, __import__('os').cpu_count() or 1))
    assert np.allclose(sig, so, rtol=2e-4), np.abs(sig / so - 1).max()
    J = ho.katz_terms_needed(A, 0.01, 1e-12)
    r1, r2, _, _ = ho.svd_residuals(A, 0.01, X, J, sigma=sig)
    assert max(r1.max(), r2.max()) < 5e-4
