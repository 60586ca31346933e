"""The 'SVD error (low rank)' diagnostic of hope.py:38-40 on the GPU (gemb_hope_svd_error, through
DeviceGraph.hope_svd_error) against the fp64 Katz matrix S = (I - beta A)^-1 beta A of oracle/hope_oracle.py.

Inputs are exact in both: weights and beta are rounded to fp32 before the oracle sees them, and X is fp32.

Tolerance, from the fp32 error model.  The device forms S Z by J fp32 Horner sweeps W <- Z + beta A W, and X1 (X2^T Z)
by an fp64 Gram rounded to fp32 followed by an fp32 product (3xTF32 on the tensor cores).  Every rounding is relative to
the quantity rounded, and those quantities are bounded entrywise by P |Z| and Q |Z|, where P = sum_{j>=1} (beta |A|)^j
and Q = |X1| |X2|^T.  So E Z = (X1 X2^T - S) Z is off by at most c u (P + Q) |Z| entrywise, with u = 2^-24 and c a small
constant: the length of the sums and the amplification of earlier sweeps' rounding by the later ones.  Because
|e_gpu - e_ref| <= || (E_gpu - E_ref) Z ||, this gives
    exact    (Z = I):         |e_gpu - e_ref| <= c u (||P||_F + ||Q||_F)
    estimate (|z_j| = 1):     |e_gpu - e_ref| <= c u (||P 1|| + ||Q 1||)     (the root of the mean over the probes)
with c = 64.  Every graph here has nonnegative weights, so P = S, and the |A| series converges wherever S does.  Each
test prints the largest measured |e_gpu - e_ref| / (u (...)) (pytest -s).  Measured on an H100 80GB HBM3 (700 W): 38.5
on the cliques at beta ||A||_2 = 0.97, where about 2000 sweeps each add rounding that the later ones amplify up to
1 / (1 - 0.97) times; at most 1.4 everywhere else.

Directed graphs go up with their transpose, as the HOPE class uploads them: without it the device takes A^T = A."""
import numpy as np
import pytest

from conftest import golden_path, load_karate_nx, load_sbm1024_nx, nx_from_npz

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
C = 64


def _f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def _random_directed(n, deg, seed):
    """Each node points to `deg` random nodes (weights in [0.5, 1.5)), and the last four columns get in-edges, so that
    S is nonzero there: at n = 4100 they are the four live columns of the last 64-column panel."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    src = np.concatenate((np.repeat(np.arange(n), deg), rng.integers(0, n, 4)))
    dst = np.concatenate((rng.integers(0, n, n * deg), np.arange(n - 4, n)))
    A = sp.csr_matrix((rng.uniform(0.5, 1.5, src.size), (src, dst)), shape=(n, n))
    A.sum_duplicates()
    return A


def _tiny(n):
    import scipy.sparse as sp
    if n == 1:
        return sp.csr_matrix(np.array([[0.75]]))                 # a self-loop: S = b a / (1 - b a)
    rng = np.random.default_rng(n)
    M = rng.uniform(0.1, 0.5, (n, n)) * (rng.random((n, n)) < 0.6)
    M[0, n - 1] = 0.45                                          # not symmetric
    return sp.csr_matrix(M)


def _build(name):
    import scipy.sparse as sp
    from gem_b200 import synth
    from gem_b200.graph import from_networkx
    if name == 'karate':
        return from_networkx(load_karate_nx()).to_scipy()
    if name in ('randw200', 'cliques'):
        z = np.load(golden_path('ref_hope_%s.npz' % {'randw200': 'randw200_d32', 'cliques': 'cliques_d24'}[name]))
        return from_networkx(nx_from_npz(z)).to_scipy()
    if name == 'sbm1024':
        return from_networkx(load_sbm1024_nx()[0]).to_scipy()
    if name.startswith('rand'):
        n = int(name[4:])
        return _random_directed(n, 6, n)
    if name.startswith('tiny'):
        return _tiny(int(name[4:]))
    if name == 'empty6':
        return sp.csr_matrix((6, 6))
    if name == 'rmat12':
        return synth.rmat(scale=12, edge_factor=8, seed=3).to_scipy()      # hubs, isolated nodes
    raise KeyError(name)


_GRAPHS = {}
_KATZ = {}


def _graph(name):
    """The adjacency (fp64 holding fp32 values) of one test graph, built once per session."""
    if name not in _GRAPHS:
        A = _build(name).tocsr().astype(np.float64)
        A.data = _f32(A.data)
        A.sort_indices()
        assert np.all(A.data >= 0)                               # P = S (see the module docstring)
        _GRAPHS[name] = A
    return _GRAPHS[name]


def _katz(ho, name, beta):
    if (name, beta) not in _KATZ:
        _KATZ[(name, beta)] = ho.katz_dense(_graph(name), beta)
    return _KATZ[(name, beta)]


def _beta(name, beta):
    """beta as the device receives it (fp32); 'r0.97' = 0.97 / ||A||_2, 'h0.5' = 0.5 / rho(A)."""
    if isinstance(beta, str):
        A = _graph(name)
        if beta[0] == 'r':
            beta = float(beta[1:]) / np.linalg.norm(A.toarray(), 2)
        else:
            import scipy.sparse.linalg as sla
            beta = float(beta[1:]) / float(abs(sla.eigsh(A, k=1, which='LA', return_eigenvectors=False)[0]))
    return float(np.float32(beta))


def _upload(ctx, A):
    from gem_b200 import _native
    from gem_b200.graph import from_scipy
    csr = from_scipy(A)
    if csr.is_symmetric():
        return _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, csr.data_f32())
    t = csr.transpose()
    return _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, csr.data_f32(), t.indptr, t.indices, t.data_f32())


def _embedding(ho, g, A, S, d, beta, kind, seed, usv=None):
    """(a) the solver's own X; (b) the fp64 LAPACK embedding rounded to fp32 (error ~ the Eckart-Young tail);
    (c) random X scaled to ||X1 X2^T||_F ~ ||S||_F (error of the order of ||S||: a dropped, duplicated or transposed
    piece of S or of X1 X2^T moves it far beyond the tolerance); (d) X = 0 (error = ||S||_F, the Katz chain alone)."""
    n, k = A.shape[0], d // 2
    if kind == 'a':
        return g.hope(d, beta, oversample=32, tol=1e-8, max_iters=200, seed=seed)[0]
    if kind == 'b':
        u, s, vt = usv
        X1, X2 = u[:, :k] * np.sqrt(s[:k]), vt[:k].T * np.sqrt(s[:k])
        return np.concatenate((X1, X2), axis=1).astype(np.float32)
    if kind == 'c':
        rng = np.random.default_rng(seed)
        X1, X2 = rng.standard_normal((n, k)), rng.standard_normal((n, k))
        rec = np.sqrt(max(np.sum((X1.T @ X1) * (X2.T @ X2)), 1e-300))        # ||X1 X2^T||_F
        sc = np.sqrt((np.linalg.norm(S) or 1.0) / rec)
        return np.concatenate((X1 * sc, X2 * sc), axis=1).astype(np.float32)
    return np.zeros((n, d), np.float32)


def _bound_exact(S, X):
    X1, X2 = np.abs(_f32(X[:, :X.shape[1] // 2])), np.abs(_f32(X[:, X.shape[1] // 2:]))
    return U32 * (np.linalg.norm(S) + np.linalg.norm(X1 @ X2.T))


def _bound_probes(S, X):
    X1, X2 = np.abs(_f32(X[:, :X.shape[1] // 2])), np.abs(_f32(X[:, X.shape[1] // 2:]))
    return U32 * (np.linalg.norm(S.sum(axis=1)) + np.linalg.norm(X1 @ X2.sum(axis=0)))


# graph, beta, [(d, kinds)]: odd k (d = 2, 6), k not a multiple of 4 (d = 4, 6), the tensor cores at n >= 4096 with
# k = 8, 64, and k = 132 (gram_tc's second row block of 4 columns); panel widths 4 (n <= 4), 8, 36 (karate: 252-thread
# column sums), 64 with a full, a 63-column and a 4-column last panel (n = 4096, 4095, 4100)
SMALL = [(2, 'bcd'), (4, 'abcd'), (6, 'bcd'), (8, 'acd'), (16, 'bcd')]
EXACT_CASES = [
    ('karate', 0.01, SMALL),
    ('karate', 0.3, SMALL),                       # beta ||A||_2 = 1.52 > 1, nilpotent A: the series is finite
    ('randw200', 0.01, SMALL + [(128, 'bcd')]),
    ('randw200', 0.075, SMALL + [(128, 'bcd')]),  # beta ||A||_2 = 1.05, beta rho(A) = 0.88
    ('cliques', 0.01, SMALL),
    ('cliques', 'r0.97', SMALL),                  # symmetric, near the radius: ~2000 Horner sweeps
    ('sbm1024', 0.01, [(6, 'cd'), (16, 'abcd'), (128, 'cd'), (264, 'cd')]),
    ('rand4095', 0.01, [(6, 'cd'), (128, 'cd')]),
    ('rand4096', 0.01, [(8, 'cd'), (16, 'acd'), (128, 'cd'), (264, 'cd')]),
    ('rand4100', 0.01, [(2, 'cd'), (16, 'cd'), (128, 'cd'), (264, 'cd')]),
    ('tiny1', 0.3, [(2, 'bcd'), (6, 'cd')]),
    ('tiny2', 0.3, [(2, 'bcd'), (4, 'bcd'), (6, 'cd')]),
    ('tiny5', 0.3, [(2, 'bcd'), (6, 'bcd'), (8, 'cd')]),
    ('empty6', 0.01, [(2, 'cd'), (6, 'cd')]),
    ('rmat12', 'h0.5', [(16, 'acd'), (128, 'cd')]),
]


@pytest.mark.parametrize('name,beta,cases', EXACT_CASES, ids=['%s-%s' % (c[0], c[1]) for c in EXACT_CASES])
def test_exact_error_matches_the_fp64_katz_matrix(gpu_ctx, hope_oracle, name, beta, cases):
    ho = hope_oracle
    A = _graph(name)
    beta = _beta(name, beta)
    S = _katz(ho, name, beta)
    if name == 'rand4100':
        assert np.all(np.abs(S[:, -4:]).sum(axis=0) > 0)
    usv = np.linalg.svd(S) if any('b' in kinds for _, kinds in cases) else None
    worst = 0.0
    with _upload(gpu_ctx, A) as g:
        for d, kinds in cases:
            for kind in kinds:
                X = _embedding(ho, g, A, S, d, beta, kind, seed=d + 1, usv=usv)
                e = g.hope_svd_error(d, beta, X)
                ref = ho.svd_error(A, beta, _f32(X), S=S)
                bound = _bound_exact(S, X)
                worst = max(worst, abs(e - ref) / bound if bound > 0 else abs(e - ref) * np.inf)
                assert abs(e - ref) <= C * bound, (d, kind, e, ref, bound)
                if kind == 'b':                  # the optimum: the Eckart-Young tail
                    assert abs(e - np.sqrt(np.sum(usv[1][d // 2:] ** 2))) <= C * bound
                if kind == 'd':
                    assert abs(ref - np.linalg.norm(S)) <= 1e-12 * ref
    print('svd_error exact %s beta=%.6g: max |e - ref| / (u (||P|| + ||Q||)) = %.3g' % (name, beta, worst))


PROBE_GRAPHS = [('karate', 0.3), ('randw200', 0.075), ('rand4100', 0.01)]


@pytest.mark.parametrize('name,beta', PROBE_GRAPHS)
def test_probe_estimate_matches_the_oracle_on_the_same_probes(gpu_ctx, hope_oracle, name, beta):
    """The Hutchinson estimate is a deterministic function of the probes: equal to the oracle's svd_error_probes on the
    same Rademacher vectors, for probe counts that fill no panel, part of one, exactly one and parts of several; the
    same seed twice agrees to 1e-12 (the fp64 atomics of the column sums may reorder)."""
    ho = hope_oracle
    A = _graph(name)
    beta = _beta(name, beta)
    S = _katz(ho, name, beta)
    worst = 0.0
    with _upload(gpu_ctx, A) as g:
        for d in (6, 16):
            X = _embedding(ho, g, A, S, d, beta, 'c', seed=d)
            bound = _bound_probes(S, X)
            for seed in (0, 1, 2 ** 63 + 5):
                vals = []
                for n_probe in (1, 3, 4, 64, 65, 130):
                    e = g.hope_svd_error(d, beta, X, n_probe=n_probe, seed=seed)
                    ref = ho.svd_error_probes(A, beta, _f32(X), n_probe, seed, S=S)
                    worst = max(worst, abs(e - ref) / bound)
                    assert abs(e - ref) <= C * bound, (d, seed, n_probe, e, ref, abs(e - ref) / bound)
                    vals.append(e)
                again = g.hope_svd_error(d, beta, X, n_probe=130, seed=seed)
                assert abs(again - vals[-1]) <= 1e-12 * vals[-1]
                assert len(set(vals)) == len(vals)
    print('svd_error probes %s beta=%.6g: max |e - ref| / (u (||P 1|| + ||Q 1||)) = %.3g' % (name, beta, worst))


def test_odd_d_is_refused(gpu_ctx):
    with _upload(gpu_ctx, _graph('karate')) as g:
        with pytest.raises(RuntimeError, match='bad argument'):
            g.hope_svd_error(5, 0.01, np.zeros((34, 5), np.float32))


@pytest.mark.parametrize('name,beta', [('sbm1024', 0.05), ('cycle', 1.5)])
def test_divergent_series_is_refused(gpu_ctx, name, beta):
    """beta rho(A) > 1: symmetric (sbm1024, rho = ||A||_2 = 42.5) and a directed cycle (rho = ||A||_2 = 1)."""
    import scipy.sparse as sp
    A = _graph(name) if name != 'cycle' else sp.csr_matrix((np.ones(7), (np.arange(7), (np.arange(7) + 1) % 7)), (7, 7))
    with _upload(gpu_ctx, A) as g:
        with pytest.raises(RuntimeError, match='does not converge'):
            g.hope_svd_error(4, beta, np.zeros((A.shape[0], 4), np.float32))
