"""oracle/hope_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement (NumPy / SciPy, fp64) of the reference's HOPE path,
`gem/embedding/hope.py:23-41`:

    A = nx.to_numpy_matrix(graph)                 hope.py:28
    m_g = I - beta*A ; m_l = beta*A               hope.py:29-30
    S = inv(m_g) @ m_l                            hope.py:31
    u, s, vt = scipy.sparse.linalg.svds(S, k=d//2) hope.py:33   (third party, SciPy>=0.19;
                                                   1.18.1 in this image; ascending sigma)
    X = [u*sqrt(s) | vt.T*sqrt(s)]                hope.py:34-36

Three routes, all returning (X, sigma) with sigma ASCENDING like svds:

  * hope_dense_svds   -- the reference recipe verbatim (dense inverse + SciPy svds/ARPACK).
  * hope_dense_lapack -- same S, but a full LAPACK SVD truncated to the top k.  Deterministic
                         (no random v0), used as the tight numerical oracle for small n.
  * hope_sparse       -- matrix-free: S.x evaluated by the Katz/Neumann series
                         sum_{j=1..J} (beta*A)^j x over a scipy.sparse CSR, fed to the same
                         SciPy svds.  This is the only route that scales to BASELINE's 1M-node
                         configuration (the dense one needs 8 TB) and is what bench.py's
                         cpu_baseline / --impl reference time.

Pinned against the reference's own goldens (tests/karate_res/HOPE.txt, tests/smb_res/HOPE.txt,
copied to tests/golden/ by tests/golden/make_golden.py) in tests/test_oracle_hope.py.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  gem_b200/ never does.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


# --------------------------------------------------------------------------- graph -> matrix
def adjacency_from_nx(graph):
    """Rows/cols follow list(graph.nodes) (insertion order), weight attr 'weight', missing -> 1:
    exactly what nx.to_numpy_matrix(graph) gave the reference (hope.py:28, SURVEY F6)."""
    import networkx as nx
    return nx.to_scipy_sparse_array(graph, nodelist=list(graph.nodes), weight='weight',
                                    dtype=np.float64, format='csr')


# --------------------------------------------------------------------------- Katz proximity
def katz_dense(A, beta):
    """S = (I - beta A)^-1 (beta A), hope.py:29-31."""
    A = np.asarray(A.todense() if sp.issparse(A) else A, dtype=np.float64)
    n = A.shape[0]
    m_g = np.eye(n) - beta * A
    m_l = beta * A
    return np.dot(np.linalg.inv(m_g), m_l)


def katz_terms_needed(A, beta, tol=1e-12, max_terms=2000):
    """Number J of Neumann terms so that (beta*||A||_2)^J <= tol (||A||_2 by svds)."""
    A = sp.csr_matrix(A)
    if A.nnz == 0:
        return 1
    smax = spla.svds(A.astype(np.float64), k=1, return_singular_vectors=False)[0] \
        if min(A.shape) > 2 else np.linalg.norm(A.toarray(), 2)
    x = beta * float(smax)
    if x >= 1.0:
        raise ValueError('beta*||A||_2 = %.4g >= 1: Katz series diverges' % x)
    if x <= 0:
        return 1
    return int(min(max_terms, max(1, np.ceil(np.log(tol) / np.log(x)))))


def katz_apply(A, beta, X, terms, transpose=False):
    """sum_{j=1..terms} (beta*A)^j X by Horner:  W <- X + beta*A*W ... ; Y = beta*A*W."""
    M = A.T.tocsr() if transpose else A
    W = X
    for _ in range(terms - 1):
        W = X + beta * (M @ W)
    return beta * (M @ W)


# --------------------------------------------------------------------------- embeddings
def _embed_from_svd(u, s, vt):
    """hope.py:34-36."""
    X1 = u * np.sqrt(s)[None, :]
    X2 = vt.T * np.sqrt(s)[None, :]
    return np.concatenate((X1, X2), axis=1)


def hope_dense_svds(A, d, beta, rng=None):
    S = katz_dense(A, beta)
    kw = {}
    if rng is not None:
        kw['v0'] = np.random.default_rng(rng).standard_normal(S.shape[0])
    u, s, vt = spla.svds(S, k=d // 2, **kw)
    return _embed_from_svd(u, s, vt), s


def hope_dense_lapack(A, d, beta):
    S = katz_dense(A, beta)
    k = d // 2
    u, s, vt = np.linalg.svd(S, full_matrices=False)
    u, s, vt = u[:, :k][:, ::-1], s[:k][::-1], vt[:k][::-1]
    return _embed_from_svd(u, s, vt), s


_katz_lib = None


def katz_omp_lib():
    """oracle/build/libkatz_omp.so (OpenMP Katz operator, same arithmetic as katz_apply), built on demand."""
    global _katz_lib
    if _katz_lib is None:
        import ctypes
        import os
        import subprocess
        here = os.path.dirname(os.path.abspath(__file__))
        so = os.path.join(here, 'build', 'libkatz_omp.so')
        src = os.path.join(here, 'katz_omp.c')
        if not os.path.exists(so) or (os.path.exists(src) and os.path.getmtime(so) < os.path.getmtime(src)):
            subprocess.check_call(['make', '-C', here, 'build/libkatz_omp.so'], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(so)
        i64p = np.ctypeslib.ndpointer(np.int64, flags='C')
        i32p = np.ctypeslib.ndpointer(np.int32, flags='C')
        f64p = np.ctypeslib.ndpointer(np.float64, flags='C')
        L.katz_apply_omp.argtypes = [ctypes.c_int64, i64p, i32p, ctypes.c_void_p, ctypes.c_double, ctypes.c_int,
                                     ctypes.c_int, f64p, f64p, f64p, f64p]
        L.katz_omp_threads.restype = ctypes.c_int
        _katz_lib = L
    return _katz_lib


class KatzOMP:
    """x -> sum_{j=1..J} (beta M)^j x for a fixed CSR M (fp64), rows spread over the host cores."""

    def __init__(self, M, beta, J):
        M = sp.csr_matrix(M, dtype=np.float64)
        M.sort_indices()
        self.n = M.shape[0]
        self.indptr = np.ascontiguousarray(M.indptr, dtype=np.int64)
        self.idx = np.ascontiguousarray(M.indices, dtype=np.int32)
        self.w = None if np.all(M.data == 1.0) else np.ascontiguousarray(M.data, dtype=np.float64)
        self.beta, self.J = float(beta), int(J)
        self.L = katz_omp_lib()
        self._scratch = {}

    def __call__(self, x):
        x = np.asarray(x, dtype=np.float64)
        shape = x.shape
        x2 = np.ascontiguousarray(x.reshape(self.n, -1))
        m = x2.shape[1]
        if m not in self._scratch:
            self._scratch[m] = (np.empty((self.n, m)), np.empty((self.n, m)))
        t1, t2 = self._scratch[m]
        y = np.empty((self.n, m))
        wp = None if self.w is None else self.w.ctypes.data
        self.L.katz_apply_omp(self.n, self.indptr, self.idx, wp, self.beta, self.J, m, x2, y, t1, t2)
        return y.reshape(shape)


def hope_sparse(A, d, beta, katz_tol=1e-12, terms=None, tol=0, maxiter=None, rng=0, ncv=None, threads=False):
    # threads: False = scipy.sparse products on one core; True = oracle/katz_omp.c on the OpenMP default; int = that many
    """threads=True: the Katz operator runs in oracle/katz_omp.c on all host cores (same arithmetic; for the
    million-node reference arm of bench.py) instead of scipy.sparse products on one."""
    A = sp.csr_matrix(A, dtype=np.float64)
    AT = A.T.tocsr()
    n = A.shape[0]
    J = terms if terms is not None else katz_terms_needed(A, beta, katz_tol)
    counter = {'spmv': 0}
    if threads:
        if threads is not True:
            katz_omp_lib().katz_omp_set_threads(int(threads))
        kA, kAT = KatzOMP(A, beta, J), KatzOMP(AT, beta, J)

    def mv(x):
        counter['spmv'] += J
        return kA(x) if threads else katz_apply(A, beta, x, J)

    def rmv(x):
        counter['spmv'] += J
        return kAT(x) if threads else katz_apply(AT, beta, x, J)

    S = spla.LinearOperator((n, n), matvec=mv, rmatvec=rmv, matmat=mv, rmatmat=rmv, dtype=np.float64)
    v0 = np.random.default_rng(rng).standard_normal(n)
    u, s, vt = spla.svds(S, k=d // 2, tol=tol, maxiter=maxiter, v0=v0, ncv=ncv)
    X = _embed_from_svd(u, s, vt)
    return X, s, dict(katz_terms=J, spmv=counter['spmv'])


# --------------------------------------------------------------------------- comparators (SURVEY C.3)
def split_halves(X):
    k = X.shape[1] // 2
    return X[:, :k], X[:, k:]


def sigma_from_embedding(X):
    """X1 = U sqrt(Sigma)  =>  sigma_j = ||X1[:, j]||^2."""
    X1, _ = split_halves(X)
    return np.sum(np.asarray(X1, dtype=np.float64) ** 2, axis=0)


def align_pair_signs(X, Xref):
    """(u_j, v_j) is defined up to a joint sign: flip columns j and k+j together (SURVEY F5)."""
    X = np.array(X, dtype=np.float64, copy=True)
    k = X.shape[1] // 2
    for j in range(k):
        sgn = np.sign(np.dot(X[:, j], Xref[:, j]) + np.dot(X[:, k + j], Xref[:, k + j]))
        if sgn < 0:
            X[:, j] *= -1
            X[:, k + j] *= -1
    return X


def principal_angles_deg(Qa, Qb):
    """Principal angles (degrees, descending) between span(Qa) and span(Qb) (same dimension).
    cosines from svd(qa^T qb), sines from svd((I - qa qa^T) qb); atan2 keeps accuracy at both ends."""
    qa, _ = np.linalg.qr(np.asarray(Qa, dtype=np.float64))
    qb, _ = np.linalg.qr(np.asarray(Qb, dtype=np.float64))
    c = np.clip(np.linalg.svd(qa.T @ qb, compute_uv=False), 0.0, 1.0)          # descending cos
    sn = np.clip(np.linalg.svd(qb - qa @ (qa.T @ qb), compute_uv=False), 0.0, 1.0)  # descending sin
    m = min(len(c), len(sn))
    ang = np.arctan2(sn[:m], np.sort(c)[:m])   # largest sine pairs with smallest cosine
    return np.degrees(ang)


def recon_rel_err(X, Xref):
    """|| X1 X2^T - X1r X2r^T ||_F / || X1r X2r^T ||_F  (sign- and rotation-invariant)."""
    X1, X2 = split_halves(np.asarray(X, dtype=np.float64))
    R1, R2 = split_halves(np.asarray(Xref, dtype=np.float64))
    ref = R1 @ R2.T
    return np.linalg.norm(X1 @ X2.T - ref) / max(np.linalg.norm(ref), 1e-300)


def svd_error(A, beta, X, S=None):
    """hope.py:38-40, 'SVD error (low rank)': || X1 X2^T - S ||_F with S = katz_dense(A, beta) (the reference writes
    u diag(s) vt for X1 X2^T; the two are equal for its own embedding).  S: katz_dense(A, beta) computed already."""
    X1, X2 = split_halves(np.asarray(X, dtype=np.float64))
    S = katz_dense(A, beta) if S is None else S
    return float(np.linalg.norm(X1 @ X2.T - S))


def rademacher_probes(n, cols, seed, p0=0):
    """n x cols matrix of +-1: column c is probe p0 + c of gemb_hope_svd_error's probe_block_kernel (the same 64-bit
    hash of (seed, row, probe), in uint64 arithmetic that wraps as the kernel's does)."""
    r = np.arange(n, dtype=np.uint64)[:, None]
    p = (np.uint64(p0) + np.arange(cols, dtype=np.uint64))[None, :]
    with np.errstate(over='ignore'):
        h = np.uint64(seed) ^ (r * np.uint64(0x9E3779B97F4A7C15)) ^ (p * np.uint64(0xBF58476D1CE4E5B9))
        h ^= h >> np.uint64(31)
        h *= np.uint64(0x94D049BB133111EB)
        h ^= h >> np.uint64(29)
    return np.where((h & np.uint64(1)) != 0, 1.0, -1.0)


def svd_error_probes(A, beta, X, n_probe, seed, S=None):
    """The Hutchinson estimate of svd_error: sqrt(mean_j || E z_j ||^2), E = X1 X2^T - S, over the probes z_j of
    rademacher_probes(n, n_probe, seed)."""
    X1, X2 = split_halves(np.asarray(X, dtype=np.float64))
    Z = rademacher_probes(X1.shape[0], n_probe, seed)
    S = katz_dense(A, beta) if S is None else S
    EZ = X1 @ (X2.T @ Z) - S @ Z
    return float(np.sqrt(np.sum(EZ * EZ) / n_probe))


def katz_pairs(beta, X, sigma):
    """The eigenpairs of a symmetric A behind an embedding of the symmetric solvers (algorithms 2 and 3), whose columns are
    X = [v sign(f) sqrt(sigma) | v sqrt(sigma)] with f = f(l) = beta l / (1 - beta l):
        v_q = X[:, k+q] / sqrt(sigma_q), normalised (norm_dev_q = | ||v_q|| - 1 | before that),
        s_q = sign(X[:, q] . X[:, k+q]),  f_q = s_q sigma_q,  l_q = f_q / (beta (1 + f_q)).
    Returns (V n x k, l, s, norm_dev), all fp64."""
    X = np.asarray(X, dtype=np.float64)
    k = X.shape[1] // 2
    sig = np.asarray(sigma, dtype=np.float64)
    V = X[:, k:] / np.sqrt(np.maximum(sig, 1e-300))[None, :]
    nrm = np.linalg.norm(V, axis=0)
    s = np.sign(np.sum(X[:, :k] * X[:, k:], axis=0))
    s[s == 0] = 1.0
    f = s * sig
    return V / nrm[None, :], f / (beta * (1.0 + f)), s, np.abs(nrm - 1.0)


def eig_residuals(A, V, l):
    """||A v_q - l_q v_q|| per column, fp64."""
    V = np.asarray(V, dtype=np.float64)
    return np.linalg.norm(A @ V - V * np.asarray(l, dtype=np.float64)[None, :], axis=0)


def katz_slope(beta, l):
    """|f'(l)| = beta / (1 - beta l)^2: maps an eigen-residual of A to the residual of the Katz triplet."""
    return beta / (1.0 - beta * np.asarray(l, dtype=np.float64)) ** 2


def katz_kappa(beta, l, lmax):
    """kappa_q = (1 - beta l_q) / (1 - beta lambda_max): with f(lam) - f(l) = beta (lam - l) / ((1 - beta lam)(1 - beta l)),
    ||S v - f(l) v|| <= kappa_q slope(l_q) ||A v - l_q v||, with equality when v mixes only x(l_q) and x(lambda_max)."""
    return (1.0 - beta * np.asarray(l, dtype=np.float64)) / (1.0 - beta * lmax)


def katz_stop_residual(A, beta, X, sigma):
    """What the symmetric solvers' stop_rule 1 documents, recomputed in fp64 at the returned vectors:
    max_q slope(l_q) ||A v_q - l_q v_q|| / max sigma.  Returns (value, dict of the per-pair terms)."""
    V, l, s, norm_dev = katz_pairs(beta, X, sigma)
    r = eig_residuals(A, V, l)
    sig = np.asarray(sigma, dtype=np.float64)
    terms = katz_slope(beta, l) * r / max(sig.max(), 1e-300)
    return float(terms.max()), dict(V=V, l=l, sign=s, norm_dev=norm_dev, r=r, terms=terms)


def mode1_stop_residual(A, X, lam):
    """spectral_mode 1 (Laplacian Eigenmaps / LLE): v_q = X[:, q], l_q = lam_q;  max_q ||A v_q - l_q v_q|| / max_q |l_q|.
    Returns (value, per-pair residuals)."""
    lam = np.asarray(lam, dtype=np.float64)
    r = eig_residuals(A, np.asarray(X, dtype=np.float64), lam)
    return float(r.max() / max(np.abs(lam).max(), 1e-300)), r


def general_stop_residual(A, beta, X, terms, sigma):
    """The general solver's (algorithm 1) stop_rule 1: max_q ||S^T u_q - sigma_q v_q|| / sigma_max (the second residual of
    svd_residuals); also returns the first, max_q ||S v_q - sigma_q u_q|| / sigma_max, which is 0 by construction there."""
    r1, r2, _, _ = svd_residuals(A, beta, X, terms, sigma=sigma)
    return float(r2.max()), float(r1.max())


def value_change(s, s_prev):
    """The change measure of the solvers between two rounds' values: max_j |s_j - s_j'| / max(|s_j|, 1e-3 max|s|)."""
    s, s_prev = np.asarray(s, dtype=np.float64), np.asarray(s_prev, dtype=np.float64)
    return float(np.max(np.abs(s - s_prev) / np.maximum(np.abs(s), 1e-3 * np.abs(s).max())))


def svd_residuals(A, beta, X, terms, sigma=None):
    """Size-independent property: for each triplet  ||S v - sigma u|| / sigma_max and
    ||S^T u - sigma v|| / sigma_max, with S applied matrix-free (fp64)."""
    A = sp.csr_matrix(A, dtype=np.float64)
    X = np.asarray(X, dtype=np.float64)
    X1, X2 = split_halves(X)
    sig = sigma_from_embedding(X) if sigma is None else np.asarray(sigma, dtype=np.float64)
    rs = np.sqrt(np.maximum(sig, 1e-300))
    U, V = X1 / rs[None, :], X2 / rs[None, :]
    SV = katz_apply(A, beta, V, terms)
    STU = katz_apply(A, beta, U, terms, transpose=True)
    smax = max(sig.max(), 1e-300)
    r1 = np.linalg.norm(SV - U * sig[None, :], axis=0) / smax
    r2 = np.linalg.norm(STU - V * sig[None, :], axis=0) / smax
    return r1, r2, U, V
