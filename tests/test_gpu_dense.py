"""The tall-skinny Gram contraction G = P^T Q (the one dense contraction of the HOPE solver) through the C ABI
test hook gemb_gram: wgmma kernel (3xTF32, register accumulators) and CUDA-core kernel vs NumPy fp64.
Tolerance: |G - Gref|_ij <= 4e-6 * ||P_i|| ||Q_j||  (fp32-class accuracy; plain TF32 would be ~5e-4)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _check(ctx, n, b1, b2, cross, tc, seed=0, scale_cols=False):
    rng = np.random.default_rng(seed)
    P = rng.standard_normal((n, b1)).astype(np.float32)
    if scale_cols:                                   # wide dynamic range between columns (filter gains)
        P *= np.logspace(0, 4, b1, dtype=np.float32)[None, :]
    Q = rng.standard_normal((n, b2)).astype(np.float32) + 0.3 * P[:, :b2] if cross and b2 <= b1 else \
        (rng.standard_normal((n, b2)).astype(np.float32) if cross else None)
    try:
        G = ctx.gram(P, Q, tensor_cores=tc)
    except RuntimeError as e:
        if tc and 'not supported by the tensor-core kernel' in str(e):
            pytest.skip('shape outside the tensor-core kernel (falls back to the CUDA-core kernel in gram_launch)')
        raise
    Qr = P if Q is None else Q
    ref = P.astype(np.float64).T @ Qr.astype(np.float64)
    bound = np.outer(np.linalg.norm(P.astype(np.float64), axis=0), np.linalg.norm(Qr.astype(np.float64), axis=0))
    err = np.abs(G - ref) / bound
    assert err.max() < 4e-6, (n, b1, b2, cross, tc, err.max())
    if Q is None:
        assert np.abs(G - G.T).max() <= 1e-5 * np.abs(G).max()


@pytest.mark.parametrize('tc', [True, False])
@pytest.mark.parametrize('n,b1,b2,cross', [(5000, 80, 80, False), (70001, 80, 80, False), (20000, 144, 144, False),
                                            (30000, 80, 80, True), (4097, 96, 96, False), (9000, 20, 20, False),
                                            (12345, 256, 256, False), (8192, 128, 64, True), (100, 80, 80, False)])
def test_gram_kernels(gpu_ctx, n, b1, b2, cross, tc):
    _check(gpu_ctx, n, b1, b2, cross, tc)


def test_gram_tc_dynamic_range(gpu_ctx):
    _check(gpu_ctx, 50000, 80, 80, False, True, scale_cols=True)


def test_gram_tc_large_streaming(gpu_ctx):
    """1M x 80 (the bench shape): every CTA streams ~100 stages through the two-stage ring."""
    rng = np.random.default_rng(1)
    P = rng.standard_normal((1_000_000, 80)).astype(np.float32)
    G = gpu_ctx.gram(P, None, tensor_cores=True)
    G32 = gpu_ctx.gram(P, None, tensor_cores=False)
    d = np.sqrt(np.diag(G32))
    assert np.abs(G - G32).max() / (d.max() ** 2) < 4e-6
    assert np.allclose(np.diag(G), (P.astype(np.float64) ** 2).sum(axis=0), rtol=2e-6)


@pytest.mark.parametrize('tc', [True, False])
@pytest.mark.parametrize('n,b1,b2', [(5000, 80, 80), (70001, 80, 80), (1_000_000, 80, 80), (33000, 96, 64),
                                     (4100, 128, 128), (9000, 24, 24), (300, 80, 80)])
def test_apply_kernels(gpu_ctx, n, b1, b2, tc):
    """Out = Q M (CholeskyQR's Q R^-1, Ritz rotations): wgmma 3xTF32 kernel and CUDA-core kernel vs NumPy fp64;
    |Out - ref|_ij <= 4e-6 * ||Q_i|| ||M_j||."""
    rng = np.random.default_rng(n + b1)
    Q = rng.standard_normal((n, b1)).astype(np.float32)
    M = np.triu(rng.standard_normal((b1, b2))).astype(np.float32)
    try:
        out = gpu_ctx.apply(Q, M, tensor_cores=tc)
    except RuntimeError as e:
        if tc and 'not supported by the tensor-core kernel' in str(e):
            pytest.skip('shape outside the tensor-core kernel')
        raise
    ref = Q.astype(np.float64) @ M.astype(np.float64)
    bound = np.outer(np.linalg.norm(Q.astype(np.float64), axis=1), np.linalg.norm(M.astype(np.float64), axis=0)) + 1e-30
    err = np.abs(out - ref) / bound
    assert err.max() < 4e-6, (n, b1, b2, tc, err.max())


@pytest.mark.parametrize('tc', [True, False])
def test_gram_is_reproducible(gpu_ctx, tc):
    """The partial sums of the CTAs are added in a fixed order: the same input gives the same bits on every call
    (the solvers' iterates, and so the embeddings, are then reproducible)."""
    rng = np.random.default_rng(7)
    P = rng.standard_normal((300_000, 72)).astype(np.float32)
    Q = rng.standard_normal((300_000, 200)).astype(np.float32)
    for a, b in ((P, None), (Q, None), (P, Q[:, :64])):
        G1 = gpu_ctx.gram(a, b, tensor_cores=tc)
        G2 = gpu_ctx.gram(a, b, tensor_cores=tc)
        assert np.array_equal(G1, G2)
