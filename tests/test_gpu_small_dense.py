"""The b x b fp64 factorizations of the HOPE solvers through their C ABI test hooks, against NumPy fp64.

  gemb_chol_inverse -> chol_inverse_launch: Minv = R^-1 of CholeskyQR (G = R^T R) with the scale-free rank test
  gemb_eigh         -> eigh_launch: cyclic Jacobi, w ascending, Z column j <-> w[j]

Both launchers choose where the kernel keeps its matrices by b; the sizes below sit on each side of every switch, and
b = 1024 is the widest block the solvers use:
  chol_inverse_kernel<true>             b <= 168         (matrix in shared memory; 168 on H100, 227 KB per block)
  chol_inverse_kernel<false>            b >= 169         (matrix in global memory)
  eigh_jacobi_kernel<JAC_SHARED>        b <= 117         (matrix and eigenvectors in shared memory)
  eigh_jacobi_kernel<JAC_ZT_GLOBAL>     118 <= b <= 167  (eigenvectors in global memory)
  eigh_jacobi_kernel<JAC_GLOBAL>        b >= 168         (matrix and eigenvectors in global memory)
Odd b gives the round-robin Jacobi ordering a dummy player."""
import numpy as np
import pytest
from scipy.linalg import solve_triangular

PIV_EPS = 1e-5                   # GEMB_PIV_EPS of dense.cu
CHOL_SIZES = [1, 2, 16, 80, 127, 128, 129, 144, 166, 167, 168, 169, 200, 256, 1024]
EIGH_SIZES = [1, 2, 3, 80, 117, 118, 144, 167, 168, 192, 256, 400, 1024]


def chol_inverse_ref(G):
    """The kernel's algorithm in NumPy fp64: scale to unit diagonal (A = D^-1/2 G D^-1/2), right-looking Cholesky in
    which a pivot <= PIV_EPS drops its column, Minv = D^-1/2 L^-T over the kept columns (dropped ones are 0).
    Returns (Minv, keep, L, dscale) with dscale = diag(D^-1/2) (0 where G_jj <= 0)."""
    G = np.asarray(G, dtype=np.float64)
    b = G.shape[0]
    d = np.diag(G)
    ds = np.zeros(b)
    ds[d > 0] = 1.0 / np.sqrt(d[d > 0])
    A = G * ds[:, None] * ds[None, :]
    L = np.zeros((b, b))
    keep = np.zeros(b, dtype=bool)
    for j in range(b):
        if A[j, j] > PIV_EPS:
            keep[j] = True
            L[j, j] = np.sqrt(A[j, j])
            L[j + 1:, j] = A[j + 1:, j] / L[j, j]
            A[j + 1:, j + 1:] -= np.outer(L[j + 1:, j], L[j + 1:, j])
    k = np.flatnonzero(keep)
    X = np.zeros((b, b))                      # L^-1 on the kept rows and columns
    if k.size:
        X[np.ix_(k, k)] = solve_triangular(L[np.ix_(k, k)], np.eye(k.size), lower=True)
    return ds[:, None] * X.T, keep, L, ds


def _sym(G):
    return (G + G.T) / 2                      # exactly symmetric: the kernels read one triangle or both


def _gram(P):
    return _sym(P.T @ P)


def _near_dependent(b, pivot, rng, scales=(1e3, 1e-3)):
    """G = P^T P in which column j2 (scale scales[1]) has correlation c with column j1 (scale scales[0]) and is
    otherwise orthogonal to every column, so that its pivot of the scaled Cholesky is exactly 1 - c^2 = pivot."""
    P = rng.standard_normal((4 * b + 8, b))
    j1 = b // 3
    j2 = max(j1 + 1, 2 * b // 3)
    others = np.delete(P, j2, axis=1)
    Q, _ = np.linalg.qr(others)
    v = rng.standard_normal(P.shape[0])
    v -= Q @ (Q.T @ v)
    v /= np.linalg.norm(v)
    u = P[:, j1] / np.linalg.norm(P[:, j1])
    P[:, j1] = scales[0] * u
    P[:, j2] = scales[1] * (np.sqrt(1.0 - pivot) * u + np.sqrt(pivot) * v)
    return _gram(P), j2


def _chol_input(kind, b, rng):
    """(G, the columns the rank test must drop)"""
    P = rng.standard_normal((4 * b + 8, b))
    if kind == 'well':
        return _gram(P), []
    if kind == 'scaled':                      # column scales over 1e-6 .. 1e6: the rank test is scale free
        return _gram(P * np.logspace(-6, 6, b)[rng.permutation(b)]), []
    if kind == 'dup_zero':                    # the last column duplicates column j1; column z is zero (G_zz = 0)
        j1, z, drop = (b - 1) // 4, b // 2, set()
        if b >= 2:
            P[:, b - 1] = P[:, j1]
            drop.add(b - 1)
        if z not in drop:
            P[:, z] = 0.0
            drop.add(z)
        return _gram(P), sorted(drop)
    if kind in ('pivot_kept', 'pivot_dropped'):   # second pivot 2x above / below PIV_EPS
        G, j2 = _near_dependent(b, 2 * PIV_EPS if kind == 'pivot_kept' else PIV_EPS / 2, rng)
        return G, ([] if kind == 'pivot_kept' else [j2])
    raise ValueError(kind)


CHOL_KINDS = ['well', 'scaled', 'dup_zero', 'pivot_kept', 'pivot_dropped']


def test_chol_reference_matches_numpy():
    """The reference itself: on full-rank input it is numpy's Cholesky (also with wide column scales), and it drops
    exactly the columns the inputs are built to lose."""
    rng = np.random.default_rng(0)
    for b in (1, 2, 7, 40):
        for kind in ('well', 'scaled'):
            G, _ = _chol_input(kind, b, rng)
            M, keep, L, ds = chol_inverse_ref(G)
            assert keep.all()
            Lnp = np.linalg.cholesky(G)
            assert np.all(np.abs(L / ds[:, None] - Lnp) <= 1e-12 * np.abs(Lnp).max(axis=1, keepdims=True))
            Rinv = solve_triangular(Lnp.T, np.eye(b), lower=False)          # R = Lnp^T
            assert np.all(np.abs(M - Rinv) <= 1e-12 * np.abs(Rinv).max(axis=1, keepdims=True))
    for b in (1, 2, 3, 12):
        for kind in ('dup_zero', 'pivot_kept', 'pivot_dropped'):
            if b == 1 and kind != 'dup_zero':
                continue
            G, drop = _chol_input(kind, b, rng)
            M, keep, _, _ = chol_inverse_ref(G)
            assert np.array_equal(np.flatnonzero(~keep), drop), (b, kind)
            k = np.flatnonzero(keep)
            assert np.all(M[:, ~keep] == 0) and np.all(M[~keep] == 0)
            E = M[:, k].T @ G @ M[:, k]
            assert np.all(np.abs(E - np.eye(k.size)) < 1e-6)


def _check_chol(ctx, G, drop):
    b = G.shape[0]
    M64, M32, rank = ctx.chol_inverse(G)
    ref, keep, _, ds = chol_inverse_ref(G)
    assert np.array_equal(np.flatnonzero(~keep), drop)          # the inputs are built to lose exactly these
    assert rank == keep.sum()
    assert np.array_equal(np.diag(M64) > 0, keep)               # the same columns are dropped
    assert np.all(M64[:, ~keep] == 0) and np.all(M64[~keep] == 0)
    assert np.all(np.tril(M64, -1) == 0)
    assert np.array_equal(M32, M64.astype(np.float32))
    k = np.flatnonzero(keep)
    if not k.size:
        return
    kappa = np.linalg.cond((G * ds[:, None] * ds[None, :])[np.ix_(k, k)])
    # rows of Minv carry the column scale D^-1/2: compare L^-T (scale free), bound ~ b eps kappa with a wide margin
    X, Xr = M64[k] / ds[k, None], ref[k] / ds[k, None]
    err = np.abs(X - Xr).max() / np.abs(Xr).max()
    assert err <= 1e-12 * kappa, (b, err, kappa)
    E = M64[:, k].T @ G @ M64[:, k]
    assert np.abs(E - np.eye(k.size)).max() <= 1e-12 * kappa, (b, np.abs(E - np.eye(k.size)).max(), kappa)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', CHOL_KINDS)
@pytest.mark.parametrize('b', CHOL_SIZES)
def test_chol_inverse(gpu_ctx, b, kind):
    if b == 1 and kind.startswith('pivot'):
        pytest.skip('needs two columns')
    G, drop = _chol_input(kind, b, np.random.default_rng(1000 + b))
    _check_chol(gpu_ctx, G, drop)


@pytest.mark.gpu
@pytest.mark.parametrize('b', [80, 144, 256])
def test_chol_inverse_is_reproducible(gpu_ctx, b):
    G, _ = _chol_input('pivot_kept', b, np.random.default_rng(b))
    a = gpu_ctx.chol_inverse(G)
    c = gpu_ctx.chol_inverse(G)
    assert np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]) and a[2] == c[2]


def _orthogonal(b, rng):
    Q, R = np.linalg.qr(rng.standard_normal((b, b)))
    return Q * np.sign(np.diag(R))


def _block_tridiagonal(b, rng, p=16):
    """Indefinite block tridiagonal matrix shaped like the thick-restart Lanczos T (blocks of p, B_j upper triangular)."""
    T = np.zeros((b, b))
    for s in range(0, b, p):
        e = min(s + p, b)
        T[s:e, s:e] = _sym(rng.standard_normal((e - s, e - s)))
        if e < b:
            e2 = min(e + p, b)
            B = np.triu(rng.standard_normal((e2 - e, e - s)))
            T[e:e2, s:e] = B
            T[s:e, e:e2] = B.T
    return T


def _eigh_input(kind, b, rng):
    """(G, clusters): clusters = index groups (into the ascending order) whose eigenvalues are equal or close and
    are compared through the projector onto their span."""
    if kind == 'random':
        return _sym(rng.standard_normal((b, b))), []
    if kind == 'lanczos':
        return _block_tridiagonal(b, rng), []
    if kind == 'sbm':                          # one isolated value + a cluster within 3 %
        lam = np.concatenate((0.25 * (1 + 0.03 * rng.random(b - 1)), [1.0]))
        clusters = [np.arange(b - 1), np.array([b - 1])] if b > 1 else []
    elif kind == 'repeated':                   # exactly repeated eigenvalues (disjoint cliques)
        counts = [b // 3, b // 3, b - 2 * (b // 3)]
        lam = np.repeat([-1.0, 0.5, 2.0], counts)
        bounds = np.cumsum([0] + counts)
        clusters = [np.arange(bounds[i], bounds[i + 1]) for i in range(3) if counts[i]]
    elif kind == 'graded':                     # theta = sigma^2 of a skewed spectrum: 1 down to 1e-12
        lam, clusters = np.logspace(0, -12, b), []
    else:
        raise ValueError(kind)
    Q = _orthogonal(b, rng)
    return _sym((Q * lam) @ Q.T), clusters


EIGH_KINDS = ['random', 'lanczos', 'sbm', 'repeated', 'graded']


@pytest.mark.gpu
@pytest.mark.parametrize('kind', EIGH_KINDS)
@pytest.mark.parametrize('b', EIGH_SIZES)
def test_eigh(gpu_ctx, b, kind):
    """rel_tol = 1e-13: eigenvalues, orthogonality and residual at roundoff level.  The residual also shows that the
    Jacobi sweeps converged before their cap of 30 (eigh_launch does not report it)."""
    G, clusters = _eigh_input(kind, b, np.random.default_rng(2000 + b))
    w, Z = gpu_ctx.eigh(G, rel_tol=1e-13)
    wr, Zr = np.linalg.eigh(G)
    nrm2, nrmF = np.abs(wr).max(), np.linalg.norm(G)
    assert np.all(np.diff(w) >= 0)
    assert np.abs(w - wr).max() <= 1e-11 * nrm2, np.abs(w - wr).max() / nrm2
    assert np.linalg.norm(Z.T @ Z - np.eye(b)) <= 1e-11, np.linalg.norm(Z.T @ Z - np.eye(b))
    res = np.linalg.norm(G @ Z - Z * w) / nrmF
    assert res <= 1e-11, res
    for c in clusters:
        P, Pr = Z[:, c] @ Z[:, c].T, Zr[:, c] @ Zr[:, c].T
        assert np.linalg.norm(P - Pr) <= 1e-10, (c.size, np.linalg.norm(P - Pr))


@pytest.mark.gpu
@pytest.mark.parametrize('b', EIGH_SIZES)
def test_eigh_diagonal_and_zero(gpu_ctx, b):
    """No rotation to do: the ascending sort alone must permute (ties keep their index order); the zero matrix gives
    w = 0, Z = I."""
    rng = np.random.default_rng(3000 + b)
    d = rng.integers(-3, 4, b).astype(np.float64)       # unsorted, with ties
    w, Z = gpu_ctx.eigh(np.diag(d), rel_tol=1e-13)
    order = np.argsort(d, kind='stable')
    assert np.array_equal(w, d[order])
    assert np.array_equal(Z, np.eye(b)[:, order])
    w, Z = gpu_ctx.eigh(np.zeros((b, b)), rel_tol=1e-13)
    assert np.array_equal(w, np.zeros(b)) and np.array_equal(Z, np.eye(b))


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['random', 'sbm', 'graded'])
@pytest.mark.parametrize('b', EIGH_SIZES)
def test_eigh_solver_tolerance(gpu_ctx, b, kind):
    """rel_tol = 1e-5 (what the solvers pass at the bench tolerance): the sweeps stop once ||offdiag(Z^T G Z)||_F
    <= rel_tol ||G||_F, w is the diagonal of Z^T G Z in ascending order, and Z stays orthogonal."""
    G, _ = _eigh_input(kind, b, np.random.default_rng(4000 + b))
    w, Z = gpu_ctx.eigh(G, rel_tol=1e-5)
    nrmF = np.linalg.norm(G)
    T = Z.T @ G @ Z
    off = np.linalg.norm(T - np.diag(np.diag(T)))
    assert off <= 1e-5 * nrmF * (1 + 1e-6), off / nrmF
    assert np.all(np.diff(w) >= 0)
    assert np.abs(w - np.diag(T)).max() <= 1e-12 * nrmF
    assert np.linalg.norm(Z.T @ Z - np.eye(b)) <= 1e-11


@pytest.mark.gpu
@pytest.mark.parametrize('b', [80, 144, 256])
def test_eigh_is_reproducible(gpu_ctx, b):
    G, _ = _eigh_input('random', b, np.random.default_rng(b))
    w1, Z1 = gpu_ctx.eigh(G, rel_tol=1e-13)
    w2, Z2 = gpu_ctx.eigh(G, rel_tol=1e-13)
    assert np.array_equal(w1, w2) and np.array_equal(Z1, Z2)
