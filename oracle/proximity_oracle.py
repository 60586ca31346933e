"""oracle/proximity_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

fp64 restatement of the HOPE proximities other than Katz (Ou et al., KDD 2016, Table 1), as gem_b200's HOPE(proximity=...)
defines them on the weighted adjacency A (rows and columns in list(graph.nodes) order):

    'common_neighbors'   S = A A
    'adamic_adar'        S = A D A,  D_ii = 1 / sum_j (A_ij + A_ji), 0 where that sum is 0
    'rooted_pagerank'    S = (1 - alpha) (I - alpha P)^-1,  P = D_out^-1 A (rows with out-degree 0 stay 0);
                         truncated: (1 - alpha) sum_{j=0..J} (alpha P)^j

Routes: dense S (small n), a matrix-free S / S^T as a scipy LinearOperator, the top-k SVD in GEM's layout
X = [U sqrt(Sigma) | V sqrt(Sigma)], sigma ascending, and the residuals of an embedding's triplets.
Only tests/ and scripts/ import this module; gem_b200/ never does.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

PROXIMITIES = ('common_neighbors', 'adamic_adar', 'rooted_pagerank')


def random_digraph(n=200, seed=3, p=0.04):
    """A seeded directed weighted test graph (CSR, weights in [0.2, 3)) with an isolated node (7) and a row without
    out-edges (11)."""
    rng = np.random.default_rng(seed)
    M = (rng.random((n, n)) < p) * rng.uniform(0.2, 3.0, (n, n))
    np.fill_diagonal(M, 0.0)
    M[7, :] = 0.0
    M[:, 7] = 0.0
    M[11, :] = 0.0
    return sp.csr_matrix(M)


def inv_degree(A):
    """D_ii = 1 / (row sum + column sum) of A, 0 where that sum is 0 (Adamic-Adar's weight of a common neighbour)."""
    A = sp.csr_matrix(A, dtype=np.float64)
    s = np.asarray(A.sum(axis=1)).ravel() + np.asarray(A.sum(axis=0)).ravel()
    return np.where(s > 0, 1.0 / np.where(s > 0, s, 1.0), 0.0)


def transition(A):
    """P = D_out^-1 A: each row over its weighted out-degree; a row with out-degree 0 stays zero."""
    A = sp.csr_matrix(A, dtype=np.float64)
    out = np.asarray(A.sum(axis=1)).ravel()
    return sp.csr_matrix(sp.diags(np.where(out > 0, 1.0 / np.where(out > 0, out, 1.0), 0.0)) @ A)


def rooted_pagerank_terms(alpha, katz_tol):
    """J = ceil(log(katz_tol) / log(alpha)): ||alpha P||_inf <= alpha, so the series' tail after J is at most alpha^(J+1)."""
    return int(max(1, np.ceil(np.log(katz_tol) / np.log(alpha))))


def proximity_dense(A, proximity, alpha=None, terms=None):
    """S as a dense fp64 matrix.  Rooted PageRank: the inverse, or the series truncated after `terms` when given."""
    A = sp.csr_matrix(A, dtype=np.float64)
    if proximity == 'common_neighbors':
        return (A @ A).toarray()
    if proximity == 'adamic_adar':
        return (A @ sp.diags(inv_degree(A)) @ A).toarray()
    if proximity == 'rooted_pagerank':
        P = transition(A).toarray()
        n = P.shape[0]
        if terms is None:
            return (1.0 - alpha) * np.linalg.inv(np.eye(n) - alpha * P)
        S, T = np.eye(n), np.eye(n)
        for _ in range(terms):
            T = alpha * (P @ T)
            S += T
        return (1.0 - alpha) * S
    raise ValueError(proximity)


def proximity_operator(A, proximity, alpha=None, terms=None):
    """S as a LinearOperator (S x and S^T x by sparse products, never formed).  Rooted PageRank applies the series by
    Horner, truncated after `terms` (default: where alpha^J <= 1e-16)."""
    A = sp.csr_matrix(A, dtype=np.float64)
    AT = sp.csr_matrix(A.T)
    n = A.shape[0]
    if proximity in ('common_neighbors', 'adamic_adar'):
        dv = inv_degree(A) if proximity == 'adamic_adar' else np.ones(n)

        def mv(X, M):
            X = np.asarray(X, dtype=np.float64)
            Y = M @ X
            Y = Y * (dv[:, None] if Y.ndim == 2 else dv)
            return M @ Y
    elif proximity == 'rooted_pagerank':
        P = transition(A)
        PT = sp.csr_matrix(P.T)
        J = rooted_pagerank_terms(alpha, 1e-16) if terms is None else terms

        def mv(X, M):
            X = np.asarray(X, dtype=np.float64)
            W = X
            for _ in range(J):
                W = X + alpha * (M @ W)
            return (1.0 - alpha) * W
        A, AT = P, PT
    else:
        raise ValueError(proximity)
    return spla.LinearOperator((n, n), matvec=lambda x: mv(x, A), rmatvec=lambda x: mv(x, AT),
                               matmat=lambda X: mv(X, A), rmatmat=lambda X: mv(X, AT), dtype=np.float64)


def embedding(A, proximity, d, alpha=None, dense_max=3000, tol=1e-12, seed=0, terms=None):
    """(X, sigma): the top k = d/2 singular triplets of S in GEM's layout, X = [U sqrt(Sigma) | V sqrt(Sigma)], sigma
    ascending.  Dense LAPACK SVD up to dense_max nodes, else svds on proximity_operator (terms: as there)."""
    n = A.shape[0]
    k = d // 2
    if n <= dense_max:
        u, s, vt = np.linalg.svd(proximity_dense(A, proximity, alpha, terms), full_matrices=False)
        u, s, vt = u[:, :k], s[:k], vt[:k]
    else:
        v0 = np.random.default_rng(seed).standard_normal(n)
        u, s, vt = spla.svds(proximity_operator(A, proximity, alpha, terms), k=k, tol=tol, v0=v0)
    order = np.argsort(s)
    u, s, vt = u[:, order], s[order], vt[order]
    return np.concatenate((u * np.sqrt(s)[None, :], vt.T * np.sqrt(s)[None, :]), axis=1), s


def residuals(A, proximity, X, sigma, alpha=None, S=None):
    """Per triplet of an embedding X = [U sqrt(sigma) | V sqrt(sigma)]: ||S v - sigma u|| / sigma_max and
    ||S^T u - sigma v|| / sigma_max, in fp64 with u = X1_j / sqrt(sigma_j), v = X2_j / sqrt(sigma_j).  S: a matrix or
    operator already made (default: proximity_operator)."""
    X = np.asarray(X, dtype=np.float64)
    k = X.shape[1] // 2
    sig = np.asarray(sigma, dtype=np.float64)
    rs = np.sqrt(np.maximum(sig, 1e-300))
    U, V = X[:, :k] / rs[None, :], X[:, k:] / rs[None, :]
    S = proximity_operator(A, proximity, alpha) if S is None else S
    smax = max(sig.max(), 1e-300)
    r1 = np.linalg.norm(S @ V - U * sig[None, :], axis=0) / smax
    r2 = np.linalg.norm(S.T @ U - V * sig[None, :], axis=0) / smax
    return r1, r2
