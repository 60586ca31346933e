"""oracle/eval_gauss_oracle.py -- TEST INFRASTRUCTURE ONLY (not shipped, never imported by gem_b200/).

The reconstruction of LaplacianEigenmaps and LocallyLinearEmbedding for the evaluation oracle (eval_oracle.py):

    reconstruct_gaussian()   static_graph_embedding.py:48-65 with get_edge_weight of lap.py:39-42 / lle.py:37-40,
                             A_hat[i, j] = exp(-|x_i - x_j|^2), diagonal 0

eval_oracle.evaluate() then runs the reference's metrics on that matrix.
Pinned: yes -- tests/test_oracle_eval_gauss.py compares with goldens made by the reference's own functions
(tests/golden/make_golden_eval_gauss.py -> eval_*_lap / _lle / _gauss .npz).
"""
import numpy as np


def reconstruct_gaussian(X, exact=True):
    """exact=True: the reference's statements per (i, j) (np.linalg.norm, np.power, np.exp; small n);
    exact=False: the same in fp64, vectorised by rows (large n; may differ from exact=True in the last bit)."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    A = np.zeros((n, n))
    if exact:
        for v_i in range(n):
            for v_j in range(n):
                if v_i == v_j:
                    continue
                A[v_i, v_j] = np.exp(-np.power(np.linalg.norm(X[v_i, :] - X[v_j, :]), 2))
    else:
        for i in range(n):
            D = X[i] - X
            A[i] = np.exp(-np.einsum('jk,jk->j', D, D))
    np.fill_diagonal(A, 0.0)
    return A
