"""oracle/lle_composite_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The composite-operator form of oracle/lle_oracle.py (fp64, NumPy / SciPy): the d + 1 smallest singular values of
M = I - D^-1 W and their right singular vectors as the d + 1 largest algebraic eigenpairs of -M^T M, with M^T M never formed
(scipy LinearOperator + eigsh(which='LA'); dense eigh at small n), and the matrix-free fp64 residual of returned pairs.
Pinned on the CPU (tests/test_oracle_lle_composite.py) against lle_oracle.lle_dense, the reference class outputs
tests/golden/ref_lle_*.npz and the reference's Karate golden.
"""
import numpy as np
import scipy.sparse as sp

from lle_oracle import lle_matrix


def lle_composite(A, d, dense_max=2000, tol=1e-12, seed=0):
    """The composite-operator form of lle_dense: the d + 1 largest algebraic eigenpairs of -M^T M, M = lle_matrix(A), never
    forming M^T M -- scipy eigsh(which='LA') on a LinearOperator of two sparse products (dense eigh of M^T M at
    n <= dense_max).  -> (X n x d, sigma ascending (d+1), V n x (d+1)), as lle_dense.  On a repeated sigma any basis of
    its eigenspace is an answer: compare subspaces there, not vectors."""
    from scipy.sparse.linalg import LinearOperator, eigsh
    M = sp.csr_matrix(lle_matrix(A))
    n = M.shape[0]
    if n <= dense_max:
        Md = M.toarray()
        w, V = np.linalg.eigh(-(Md.T @ Md))
        idx = np.argsort(-w, kind='stable')[:d + 1]
    else:
        MT = sp.csr_matrix(M.T)
        op = LinearOperator((n, n), matvec=lambda x: -(MT @ (M @ x)), dtype=np.float64)
        v0 = np.random.default_rng(seed).standard_normal(n)
        w, V = eigsh(op, k=d + 1, which='LA', tol=tol, v0=v0)
        idx = np.argsort(-w, kind='stable')
    w, V = w[idx], V[:, idx]
    s = np.sqrt(np.maximum(-w, 0.0))
    return V[:, 1:], s, V


def composite_residuals(A, X, s, seed=0):
    """max over the columns j of ||M^T M x_j - s_j^2 x_j|| / (||x_j|| ||M||_2^2), matrix-free in fp64 (M^T M is never
    formed; ||M||_2^2 by eigsh on the same products, from a seeded Gaussian start: the ones vector lies in M's null space).
    X: n x m, s: m values."""
    from scipy.sparse.linalg import LinearOperator, eigsh
    M = sp.csr_matrix(lle_matrix(A))
    MT = sp.csr_matrix(M.T)
    n = M.shape[0]
    X = np.asarray(X, dtype=np.float64)
    R = MT @ (M @ X) - X * (np.asarray(s, dtype=np.float64) ** 2)
    op = LinearOperator((n, n), matvec=lambda x: MT @ (M @ x), dtype=np.float64)
    nrm = float(eigsh(op, k=1, which='LA', tol=1e-6, v0=np.random.default_rng(seed).standard_normal(n),
                           return_eigenvectors=False)[0]) if n > 2 else \
        float(np.linalg.norm(M.toarray(), 2) ** 2)
    return np.linalg.norm(R, axis=0) / np.linalg.norm(X, axis=0) / nrm, nrm
