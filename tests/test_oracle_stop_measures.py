"""The fp64 recomputations of the HOPE / Laplacian solvers' stop measures (oracle/hope_oracle.py: katz_pairs,
katz_stop_residual, katz_kappa, mode1_stop_residual, general_stop_residual, value_change), pinned on small dense matrices
whose eigenpairs are known exactly: exact pairs give residual 0, perturbed pairs give the analytic residual, and the
bound ||S v - f(l) v|| <= kappa slope(l) ||A v - l v|| holds and is attained.  No GPU."""
import numpy as np
import pytest
import scipy.sparse as sp


@pytest.fixture(scope='module')
def ho(hope_oracle):
    return hope_oracle


def _sym(n, seed, signed=False):
    """Symmetric A with known eigenpairs (lam ascending, x orthonormal) and a dominant positive eigenvalue."""
    rng = np.random.default_rng(seed)
    x, _ = np.linalg.qr(rng.standard_normal((n, n)))
    lam = np.sort(rng.uniform(-1.0 if signed else 0.0, 1.0, n) * 4.0)
    lam[-1] = 9.0
    if signed:
        lam[0] = -6.0
    return sp.csr_matrix((x * lam) @ x.T), lam, x


def _katz_embedding(beta, lam, vecs):
    """X = [v sign(f) sqrt(|f|) | v sqrt(|f|)] and sigma = |f(l)|, sigma ascending, for the given (l, v) pairs."""
    f = beta * lam / (1.0 - beta * lam)
    order = np.argsort(np.abs(f))
    f, V = f[order], vecs[:, order]
    rs = np.sqrt(np.abs(f))
    return np.concatenate((V * (np.sign(f) * rs), V * rs), axis=1), np.abs(f), lam[order], V


@pytest.mark.parametrize('signed', [False, True])
def test_katz_pairs_recover_exact_eigenpairs(ho, signed):
    A, lam, x = _sym(40, 3, signed)
    beta = 0.5 / 9.0
    f = np.abs(beta * lam / (1 - beta * lam))
    top = np.argsort(f)[-6:]
    X, sig, l_exp, V_exp = _katz_embedding(beta, lam[top], x[:, top])
    V, l, s, norm_dev = ho.katz_pairs(beta, X, sig)
    assert np.allclose(l, l_exp, rtol=0, atol=1e-13)
    assert np.array_equal(s, np.sign(beta * l_exp / (1 - beta * l_exp)))
    assert norm_dev.max() < 1e-14
    assert np.abs(np.abs(np.sum(V * V_exp, axis=0)) - 1).max() < 1e-14
    if signed:
        assert (s < 0).any()                      # the dominant negative eigenvalue is among the wanted
    est, _ = ho.katz_stop_residual(A, beta, X, sig)
    assert est < 1e-14


def test_katz_residual_of_perturbed_pairs_is_analytic(ho):
    """v = (x_q + eps w) / ||.||, w random: ||A v - l_q v||^2 = sum_i c_i^2 (lam_i - l_q)^2 with c = x^T v; and the
    documented estimate max_q beta / (1 - beta l_q)^2 r_q / max sigma.  The X columns are built with the exact
    sigma_q = |f(l_q)|, so the l the helper recovers is l_q itself; a scaled column is reported as norm_dev."""
    A, lam, x = _sym(50, 5)
    beta = 0.9 / 9.0
    rng = np.random.default_rng(1)
    q = np.array([44, 47, 49])
    Vp = x[:, q] + 1e-3 * rng.standard_normal((50, 3))
    Vp /= np.linalg.norm(Vp, axis=0)
    X, sig, lq, Vs = _katz_embedding(beta, lam[q], Vp)
    c = x.T @ Vs
    r_exact = np.sqrt(np.sum(c ** 2 * (lam[:, None] - lq[None, :]) ** 2, axis=0))
    V, l, _, norm_dev = ho.katz_pairs(beta, X * 1.0, sig)
    assert np.allclose(l, lq, rtol=0, atol=1e-13)
    r = ho.eig_residuals(A, V, l)
    assert np.allclose(r, r_exact, rtol=1e-10, atol=0)
    est, t = ho.katz_stop_residual(A, beta, X, sig)
    want = np.max(beta / (1 - beta * lq) ** 2 * r_exact) / sig.max()
    assert abs(est - want) <= 1e-10 * want
    # a column of v stored 1 % long: recovered as a unit vector, the deviation reported
    X2 = X.copy()
    X2[:, 3 + 1] *= 1.01
    _, _, _, nd = ho.katz_pairs(beta, X2, sig)
    assert abs(nd[1] - 0.01) < 1e-12 and nd[0] < 1e-14


def test_kappa_bound_holds_and_is_attained(ho):
    """S = (I - beta A)^-1 beta A.  For v = cos t x_q + sin t x_max (x_max: the eigenvector of lambda_max) and l = lam_q:
    ||S v - f(l) v|| = kappa_q slope(l_q) ||A v - l v|| exactly; for any other mix it is at most that.  Checked through
    svd_residuals (Katz series, fp64) on the embedding built from (v, |f(l)|)."""
    A, lam, x = _sym(40, 7)
    beta = 0.8 / 9.0
    J = ho.katz_terms_needed(A, beta, 1e-15)
    S = ho.katz_dense(A, beta)
    rng = np.random.default_rng(2)
    for q in (30, 36, 38):
        l = lam[q]
        f = beta * l / (1 - beta * l)
        bound_factor = ho.katz_kappa(beta, l, lam[-1]) * ho.katz_slope(beta, l)
        assert ho.katz_kappa(beta, l, lam[-1]) >= 1.0
        t = 2e-3
        v = np.cos(t) * x[:, q] + np.sin(t) * x[:, -1]
        r = np.linalg.norm(A @ v - l * v)
        lhs = np.linalg.norm(S @ v - f * v)
        assert abs(lhs - bound_factor * r) <= 1e-9 * lhs                     # attained
        X = np.concatenate((v[:, None] * np.sqrt(abs(f)) * np.sign(f), v[:, None] * np.sqrt(abs(f))), axis=1)
        r1, r2, _, _ = ho.svd_residuals(A, beta, X, J, sigma=[abs(f)])
        assert abs(r1[0] * abs(f) - bound_factor * r) <= 1e-9 * lhs          # svd_residuals divides by sigma_max = |f|
        for _ in range(5):                                                    # any other perturbation: below the bound
            w = x[:, q] + 1e-2 * rng.standard_normal(40)
            w /= np.linalg.norm(w)
            lhs = np.linalg.norm(S @ w - f * w)
            assert lhs <= bound_factor * np.linalg.norm(A @ w - l * w) * (1 + 1e-12)


def test_mode1_residual(ho):
    A, lam, x = _sym(30, 11, signed=True)
    idx = np.arange(29, 21, -1)                                               # the 8 largest, descending (mode 1 order)
    est, r = ho.mode1_stop_residual(A, x[:, idx], lam[idx])
    assert est < 1e-14
    rng = np.random.default_rng(4)
    Vp = x[:, idx] + 1e-4 * rng.standard_normal((30, 8))
    Vp /= np.linalg.norm(Vp, axis=0)
    c = x.T @ Vp
    r_exact = np.sqrt(np.sum(c ** 2 * (lam[:, None] - lam[idx][None, :]) ** 2, axis=0))
    est, r = ho.mode1_stop_residual(A, Vp, lam[idx])
    assert np.allclose(r, r_exact, rtol=1e-10, atol=0)
    assert abs(est - r_exact.max() / 9.0) <= 1e-10 * est                      # max |l| over the wanted = 9


def test_general_residual(ho):
    """Directed A: exact singular triplets of S give 0; v_q turned towards another right singular vector (u_q kept) gives
    ||S^T u_q - sigma_q v|| = sigma_q ||v - v_q|| exactly, and ||S v - sigma_q u_q|| as the dense product gives it."""
    rng = np.random.default_rng(9)
    n = 40
    A = sp.random(n, n, density=0.15, random_state=np.random.RandomState(3), format='csr')
    beta = 0.3 / np.linalg.norm(A.toarray(), 2)
    S = ho.katz_dense(A, beta)
    U, s, Vt = np.linalg.svd(S)
    k = 4
    u, sg, v = U[:, :k][:, ::-1], s[:k][::-1], Vt[:k][::-1].T
    X = np.concatenate((u * np.sqrt(sg), v * np.sqrt(sg)), axis=1)
    J = ho.katz_terms_needed(A, beta, 1e-15)
    r_t, r_n = ho.general_stop_residual(A, beta, X, J, sg)
    assert r_t < 1e-12 and r_n < 1e-12
    t = 1e-3
    v2 = v.copy()
    v2[:, 0] = np.cos(t) * v[:, 0] + np.sin(t) * Vt[k + 1]                   # S^T u_0 = sg_0 v_0
    X2 = np.concatenate((u * np.sqrt(sg), v2 * np.sqrt(sg)), axis=1)
    r_t, r_n = ho.general_stop_residual(A, beta, X2, J, sg)
    want_t = sg[0] * np.linalg.norm(v2[:, 0] - v[:, 0]) / sg.max()
    want_n = np.linalg.norm(S @ v2[:, 0] - sg[0] * u[:, 0]) / sg.max()
    assert abs(r_t - want_t) <= 1e-9 * want_t
    assert abs(r_n - want_n) <= 1e-9 * want_n and r_n > 0


def test_value_change(ho):
    s_prev = np.array([10.5, 2.0, 1e-3, -1.0])
    s = np.array([10.0, 2.0, 2e-3, -1.1])
    # per value: 0.5/10, 0, 1e-3 / max(2e-3, 1e-3 * 10) = 0.1, 0.1/1.1
    assert ho.value_change(s, s_prev) == pytest.approx(0.1, rel=1e-12)
    assert ho.value_change(s[:2], s_prev[:2]) == pytest.approx(0.05, rel=1e-12)
    assert ho.value_change(s, s) == 0.0
