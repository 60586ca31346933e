"""The stop measures of the HOPE and Laplacian solvers against fp64 recomputations at the vectors they return.

Each iterative solver ends on one number and reports it: `resid_est` (stop_rule 1; algorithm 3 always), `ritz_change`
(the change rule), `resid_max` (compute_residual) and `converged`.  Here every one is recomputed in fp64 from the returned
embedding with oracle/hope_oracle.py (katz_stop_residual, mode1_stop_residual, general_stop_residual, value_change,
svd_residuals), on the weights the device holds (fp32-rounded), and printed beside its bar (pytest -s).

A  estimate fidelity    |resid_est - ref| <= 0.1 ref + floor, ref the fp64 value of the documented quantity.
B  the converged contract  converged == 1 => every wanted pair's fp64 Katz residual ||S v - sigma u|| / sigma_max is at most
                        kappa_q (tol + floor) 1.05, kappa_q = (1 - beta l_q) / (1 - beta lambda_max) (hope_oracle.katz_kappa);
                        mode 1 and algorithm 1: (tol + floor) on their own residual; algorithm 1: ||S v - sigma u|| at the floor.
C  ritz_change fidelity    solves are bit-reproducible, so max_iters = m - 1 returns round m - 1's values: the ritz_change of
                        the max_iters = m run equals value_change of the two runs' sigma within 1e-3 ref + 2e-7.
D  resid_max            = fp64 max ||S^T u - sigma v|| / sigma_max within 0.05 ref + 1e-5.
E  Katz terms           power iteration ran: 0.98 ||A||_2 <= norm2_A <= (1 + 1e-5) ||A||_2 (the margin series_terms
                        assumes); it did not: norm2_A = ||A||_inf; algorithm 1: (beta ||A||_2)^J <= 1.5 katz_tol.

Floors, from the fp32 error model (u = 2^-24 = 6.0e-8, the unit roundoff of the stored blocks):
  Gram-difference estimators (algorithm 2: z^T (AV)^T (AV) z - l^2; algorithm 1: (Wk^T Wk)_jj - theta_j).  The estimate
  is r^2 = q - l^2 with q ~ l^2 ~ l_max^2, so an error delta l_max^2 in the difference is an error sqrt(delta) l_max in r,
  whatever r is.  delta has two parts.  (a) 2u: the identity ||A V z - l V z||^2 = z^T H z - l^2 assumes ||V z|| = 1 and
  V^T A V z = l z, which the CholeskyQR2-orthonormalised fp32 V and the fp32-rounded AV satisfy to ~u each.  (b) 4u: the
  Gram's 3xTF32 products (gram_tc.cu) drop lo*lo and the remainder x - hi - lo, each up to 2^-22 = 4u of the product;
  in a sum of squares (q = ||A V z||^2, (Wk^T Wk)_jj) the dropped lo*lo terms all have one sign, so they add up instead
  of averaging out.  delta = 6u = 3.6e-7, sqrt(delta) = 6.0e-4 of l_max.  (The 4e-6 test_gpu_dense.py pins on single
  Gram entries is the same model's bound with every term at its worst.)  Mapped to the reported measure:
  x slope(l) l_max / sigma_max = 1 / (1 - beta l_max) for HOPE, 1 in mode 1: floor2 = 6.0e-4 / (1 - beta lambda_max), the
  "~3e-4" lap.py states within 2x.  Algorithm 1: the Gram is of Wk = S^T T1, ||Wk_j||^2 = theta_j <= sigma_max^2, so
  floor1 = sqrt(delta) = 6.0e-4 relative to sigma_max.  A tol below the floor cannot be certified: the solve runs to
  max_iters (the tol 2e-4 cases).
  Lanczos (algorithm 3): ||R Y_last|| is formed from fp64 small matrices, so its error is that of the Krylov relation the
  fp32 basis satisfies plus the rounding of the returned vectors, ~ c u ||A|| per pair; with c = 16 (the basis width 160
  and the fp32 store of X) floor3 = 16 u ||A||_2 max_q slope(l_q) / sigma_max, about 2e-6 on R-MAT at beta = 0.5 / rho.
"""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as sla

from conftest import REPO

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings('ignore::RuntimeWarning')]
sys.path.insert(0, os.path.join(REPO, 'oracle'))
sys.path.insert(0, REPO)

U32 = 2.0 ** -24
_FAILED = []        # every check of a test runs and prints; the test then fails on the first that missed its bar
SQRT_DELTA = float(np.sqrt(6 * U32))          # 6.0e-4: Gram-difference estimators, per unit of l_max


def _device_matrix(csr):
    """The matrix the device multiplies by: the CSR with its weights rounded to fp32, in fp64."""
    A = csr.to_scipy().astype(np.float64)
    A.data = A.data.astype(np.float32).astype(np.float64)
    return A


def _solve(ctx, csr, d, beta, directed=False, **opts):
    from gem_b200 import _native
    args = [ctx, csr.n, csr.indptr, csr.indices, csr.data_f32()]
    if directed:
        t = csr.transpose()
        args += [t.indptr, t.indices, t.data_f32()]
    with _native.DeviceGraph(*args) as g:
        X, sig, st = g.hope(d, beta, **opts)
    return X.astype(np.float64), np.asarray(sig, dtype=np.float64), st


def _lambda_max(A):
    return float(sla.eigsh(A, k=1, which='LA', return_eigenvectors=False, tol=1e-12)[0])


def _norm2(A):
    return float(sla.svds(A, k=1, return_singular_vectors=False, tol=1e-12)[0])


@pytest.fixture(autouse=True)
def _checks():
    _FAILED.clear()
    yield
    assert not _FAILED, _FAILED


def _expect(ok, *what):
    if not ok:
        _FAILED.append(what)


def check_A(name, est, ref, floor):
    bar = 0.1 * ref + floor
    print('[A] %-34s resid_est %.4g  fp64 %.4g  |diff| %.3g  bar %.3g (floor %.3g)' % (name, est, ref, abs(est - ref), bar, floor))
    _expect(abs(est - ref) <= bar, 'A', name, est, ref, floor)


def check_B(name, st, tol, floor, resid, kappa=None):
    """resid: the per-pair fp64 residuals the contract bounds; kappa: their per-pair factors (None: 1)."""
    kappa = np.ones_like(resid) if kappa is None else np.asarray(kappa)
    bar = kappa * (tol + floor) * 1.05
    print('[B] %-34s converged %d  iters %d  max resid %.4g  worst resid/bar %.3f' % (name, st['converged'], st['iters'],
                                                                                  resid.max(), (resid / bar).max()))
    if st['converged'] == 1:
        _expect(np.all(resid <= bar), 'B', name, resid.max(), (resid / bar).max())


def check_C(name, change, s_m, s_prev):
    import hope_oracle as ho
    ref = ho.value_change(s_m, s_prev)
    bar = 1e-3 * ref + 2e-7
    print('[C] %-34s ritz_change %.6g  recomputed %.6g  |diff| %.3g  bar %.3g' % (name, change, ref, abs(change - ref), bar))
    _expect(abs(change - ref) <= bar, 'C', name, change, ref)


def check_D(name, resid_max, ref):
    bar = 0.05 * ref + 1e-5
    print('[D] %-34s resid_max %.4g  fp64 %.4g  |diff| %.3g  bar %.3g' % (name, resid_max, ref, abs(resid_max - ref), bar))
    _expect(abs(resid_max - ref) <= bar, 'D', name, resid_max, ref)


def check_C_runs(ctx, name, csr, d, beta, m, **opts):
    """Two solves with max_iters m - 1 and m at tol 1e-12 (neither stops early): C on the second's ritz_change."""
    opts = dict(opts, tol=1e-12, stop_rule=0)
    _, s1, st1 = _solve(ctx, csr, d, beta, max_iters=m - 1, **opts)
    _, s2, st2 = _solve(ctx, csr, d, beta, max_iters=m, **opts)
    assert (st1['iters'], st2['iters'], st2['converged']) == (m - 1, m, 0)
    # sigma_out: HOPE ascending (largest last), mode 1 descending; the change pairs values of equal rank
    check_C('%s m=%d' % (name, m), st2['ritz_change'], s2, s1)


def katz_case(name, A, beta, X, sig, st, tol, floor, lmax, svd_J=None):
    """A and B for a HOPE embedding of the symmetric solvers; returns the fp64 svd_residuals for D."""
    import hope_oracle as ho
    ref, t = ho.katz_stop_residual(A, beta, X, sig)
    print('    %s: |v| - 1 up to %.2g, %d negative f, kappa max %.3f' % (name, t['norm_dev'].max(), int((t['sign'] < 0).sum()),
                                                                      ho.katz_kappa(beta, t['l'], lmax).max()))
    check_A(name, float(st['resid_est']), ref, floor)
    J = svd_J or ho.katz_terms_needed(A, beta, 1e-13)
    r1, r2, _, _ = ho.svd_residuals(A, beta, X, J, sigma=sig)
    check_B(name, st, tol, floor, r1, ho.katz_kappa(beta, t['l'], lmax))
    return r1, r2


# ------------------------------------------------------------------------------------------------- algorithm 2 (Katz)
@pytest.fixture(scope='module')
def sbm100k():
    from gem_b200 import synth
    csr = synth.sbm(n=100_000, block=1000, seed=42)
    A = _device_matrix(csr)
    return csr, A, _lambda_max(A)


def test_bench_setting_sbm100k(gpu_ctx, sbm100k):
    """bench.HOPE_SOLVER on the SBM the benchmark scales up (auto picks algorithm 2): A, B, D, and E's ||A||_inf."""
    import bench
    csr, A, lmax = sbm100k
    beta, tol = 0.01, bench.HOPE_SOLVER['tol']
    X, sig, st = _solve(gpu_ctx, csr, 128, beta, compute_residual=1, **bench.HOPE_SOLVER)
    assert st['algorithm'] == 2
    floor = SQRT_DELTA / (1 - beta * lmax)
    r1, r2 = katz_case('bench sbm100k d128', A, beta, X, sig, st, tol, floor, lmax)
    check_D('bench sbm100k d128', float(st['resid_max']), float(r2.max()))
    ninf = float(abs(A).sum(axis=1).max())
    print('[E] ||A||_inf %.6g, norm2_A %.6g (no power iteration: non-negative weights)' % (ninf, st['norm2_A']))
    _expect(st['norm2_A'] == np.float32(ninf), 'E', ninf, st['norm2_A'])
    print('    bench tol %.3g vs estimator floor %.3g: %.1fx' % (tol, floor, tol / floor))


@pytest.fixture(scope='module')
def sbm20k():
    from gem_b200 import synth
    csr = synth.sbm(n=20_000, block=100, seed=7)
    A = _device_matrix(csr)
    return csr, A, _lambda_max(A)


@pytest.mark.parametrize('tol', [1e-3, 2e-4])
def test_sbm20k_residual_rule(gpu_ctx, sbm20k, tol):
    csr, A, lmax = sbm20k
    beta = 0.01
    X, sig, st = _solve(gpu_ctx, csr, 64, beta, algorithm=2, stop_rule=1, tol=tol, max_iters=60)
    floor = SQRT_DELTA / (1 - beta * lmax)
    katz_case('sbm20k d64 tol %g' % tol, A, beta, X, sig, st, tol, floor, lmax)


@pytest.mark.parametrize('m', [4, 9])
def test_sbm20k_change_rule(gpu_ctx, sbm20k, m):
    csr, _, _ = sbm20k
    check_C_runs(gpu_ctx, 'sbm20k d64 alg2', csr, 64, 0.01, m, algorithm=2)


def test_signed_symmetric_sbm(gpu_ctx):
    """Weights -U[0.5, 1.5] inside the communities, +-U[0.5, 1.5] between them, w_ij = w_ji: rowsum_bound sees negative
    weights, so the power-iteration bound runs instead of the Ritz bound; the dominant eigenvalue is negative, so wanted
    columns have f < 0 (the negated left half of X)."""
    from gem_b200 import graph as hg
    from gem_b200 import synth
    base = synth.sbm(n=20_000, block=100, seed=5).to_scipy()
    up = sp.triu(base, 1).tocoo()
    rng = np.random.default_rng(5)
    mag = rng.uniform(0.5, 1.5, up.nnz)
    same = (up.row // 100) == (up.col // 100)
    w = np.where(same, -mag, mag * rng.choice([-1.0, 1.0], up.nnz))
    A0 = sp.coo_matrix((w, (up.row, up.col)), shape=base.shape)
    csr = hg.from_scipy((A0 + A0.T).tocsr())
    A = _device_matrix(csr)
    nrm = float(abs(sla.eigsh(A, k=1, which='LM', return_eigenvectors=False, tol=1e-12)[0]))
    lmin = float(sla.eigsh(A, k=1, which='SA', return_eigenvectors=False, tol=1e-12)[0])
    lmax = _lambda_max(A)
    assert -lmin > lmax and abs(nrm + lmin) < 1e-9 * nrm          # the dominant eigenvalue is negative
    beta, tol = 0.5 / nrm, 1e-3
    X, sig, st = _solve(gpu_ctx, csr, 64, beta, algorithm=2, stop_rule=1, tol=tol, max_iters=80, compute_residual=1)
    floor = SQRT_DELTA / (1 - beta * lmax)
    r1, r2 = katz_case('signed sbm20k d64', A, beta, X, sig, st, tol, floor, lmax)
    check_D('signed sbm20k d64', float(st['resid_max']), float(r2.max()))
    print('[E] ||A||_2 %.7g, norm2_A %.7g (power iteration), ratio %.6f' % (nrm, st['norm2_A'], st['norm2_A'] / nrm))
    _expect(0.98 * nrm <= st['norm2_A'] <= (1 + 1e-5) * nrm, 'E', nrm, st['norm2_A'])


# ------------------------------------------------------------------------------------------------- algorithm 3
@pytest.fixture(scope='module')
def rmat16():
    from gem_b200 import synth
    csr = synth.rmat(scale=16, edge_factor=8, seed=42)
    A = _device_matrix(csr)
    return csr, A, _lambda_max(A)


@pytest.mark.parametrize('tol', [1e-3, 1e-5])
def test_lanczos_rmat16(gpu_ctx, rmat16, tol):
    import hope_oracle as ho
    csr, A, lmax = rmat16
    beta = 0.5 / lmax
    X, sig, st = _solve(gpu_ctx, csr, 128, beta, tol=tol, max_iters=60)
    assert st['algorithm'] == 3
    assert st['ritz_change'] == st['resid_est']
    _, t = ho.katz_stop_residual(A, beta, X, sig)
    floor = 16 * U32 * lmax * float(ho.katz_slope(beta, t['l']).max()) / sig.max()
    katz_case('rmat16 d128 tol %g' % tol, A, beta, X, sig, st, tol, floor, lmax)


def test_lanczos_sbm100k(gpu_ctx, sbm100k):
    import hope_oracle as ho
    csr, A, lmax = sbm100k
    beta, tol = 0.01, 1e-4
    X, sig, st = _solve(gpu_ctx, csr, 128, beta, tol=tol, max_iters=60, algorithm=3)
    assert st['algorithm'] == 3 and st['ritz_change'] == st['resid_est']
    _, t = ho.katz_stop_residual(A, beta, X, sig)
    floor = 16 * U32 * lmax * float(ho.katz_slope(beta, t['l']).max()) / sig.max()
    katz_case('sbm100k d128 alg3 tol %g' % tol, A, beta, X, sig, st, tol, floor, lmax)


# ------------------------------------------------------------------------------------------------- algorithm 1
@pytest.fixture(scope='module')
def directed6k():
    """A directed weighted graph above the tensor-core threshold (4096 rows): 6000 nodes, ~10 out-edges each,
    weights U[0.5, 1.5]."""
    from gem_b200 import graph as hg
    rng = np.random.default_rng(13)
    n, m = 6000, 60_000
    A0 = sp.coo_matrix((rng.uniform(0.5, 1.5, m), (rng.integers(0, n, m), rng.integers(0, n, m))), shape=(n, n)).tocsr()
    csr = hg.from_scipy(A0)
    assert not csr.is_symmetric()
    A = _device_matrix(csr)
    return csr, A, _norm2(A)


@pytest.mark.parametrize('stop_rule,tol', [(0, 1e-6), (1, 1e-3), (1, 2e-4)])
def test_general_solver(gpu_ctx, directed6k, stop_rule, tol):
    import hope_oracle as ho
    csr, A, nrm = directed6k
    beta, katz_tol = 0.5 / nrm, 1e-7
    X, sig, st = _solve(gpu_ctx, csr, 32, beta, directed=True, stop_rule=stop_rule, tol=tol, max_iters=80,
                        compute_residual=1, katz_tol=katz_tol)
    name = 'directed6k d32 rule %d tol %g' % (stop_rule, tol)
    assert st['algorithm'] == 1
    J = ho.katz_terms_needed(A, beta, 1e-13)
    r1, r2, _, _ = ho.svd_residuals(A, beta, X, J, sigma=sig)
    if stop_rule == 1:
        check_A(name, float(st['resid_est']), float(r2.max()), SQRT_DELTA)
        check_B(name, st, tol, SQRT_DELTA, r2)
    else:
        assert st['resid_est'] == -1.0                 # the change rule computes no residual estimate
    print('    ||S v - sigma u|| / sigma_max %.3g (0 by construction)' % r1.max())
    _expect(r1.max() <= SQRT_DELTA, 'B', name, 'S v - sigma u', r1.max())
    check_D(name, float(st['resid_max']), float(r2.max()))
    print('[E] ||A||_2 %.7g, norm2_A %.7g, ratio %.6f; J %d, (beta ||A||_2)^J %.3g vs katz_tol %g'
          % (nrm, st['norm2_A'], st['norm2_A'] / nrm, st['katz_terms'], (beta * nrm) ** st['katz_terms'], katz_tol))
    _expect(0.98 * nrm <= st['norm2_A'] <= (1 + 1e-5) * nrm, 'E', nrm, st['norm2_A'])
    _expect((beta * nrm) ** st['katz_terms'] <= 1.5 * katz_tol, 'E', 'J', st['katz_terms'])


def test_general_solver_change_rule(gpu_ctx, directed6k):
    csr, _, nrm = directed6k
    check_C_runs(gpu_ctx, 'directed6k d32 alg1', csr, 32, 0.5 / nrm, 6, directed=True, algorithm=1)


# ------------------------------------------------------------------------------------------------- spectral_mode 1
@pytest.fixture(scope='module')
def le20k():
    from gem_b200 import synth
    from gem_b200.embedding import lap
    op, _ = lap.undirected_normalised(synth.sbm(n=20_000, block=100, seed=7))
    return op, _device_matrix(op)


def test_le_residual_rule(gpu_ctx, le20k):
    import hope_oracle as ho
    op, A = le20k
    tol = 1e-3
    X, lam, st = _solve(gpu_ctx, op, 17, 0.0, spectral_mode=1, stop_rule=1, tol=tol, max_iters=300)
    ref, r = ho.mode1_stop_residual(A, X, lam)
    check_A('LE sbm20k d16 tol %g' % tol, float(st['resid_est']), ref, SQRT_DELTA)
    check_B('LE sbm20k d16 tol %g' % tol, st, tol, SQRT_DELTA, r / np.abs(lam).max())


@pytest.mark.parametrize('m', [5, 12])
def test_le_change_rule(gpu_ctx, le20k, m):
    op, _ = le20k
    check_C_runs(gpu_ctx, 'LE sbm20k d16', op, 17, 0.0, m, spectral_mode=1)


@pytest.mark.parametrize('m', [5, 12])
def test_lle_change_rule(gpu_ctx, m):
    from gem_b200 import synth
    from gem_b200.embedding import lle
    op, _ = lle.lle_operator(synth.sbm(n=5_000, block=100, seed=3))
    check_C_runs(gpu_ctx, 'LLE sbm5k d8', op, 9, 0.0, m, spectral_mode=1)
