"""LocallyLinearEmbedding's composite operator on the GPU (gemb_hope spectral_mode 2: -M^T M, M = I - D^-1 W, applied as a
sweep of P = D^-1 W and a sweep of P^T, never formed).

- the four-operand SpMM epilogue of the Chebyshev step (gemb_spmm4) against an fp64 product, on both SpMM paths;
- parity with the explicit form, the reference goldens and the fp64 oracle on the fixtures of tests/test_gpu_lle.py, with
  its bars;
- a power-law graph (the largest component of host R-MAT scale 14) against the fp64 composite oracle, beside the explicit form;
- the largest component of device R-MAT scale 20 at d = 128 through operator='auto';
- kept behaviour: 'auto' = 'explicit' bit for bit on the fixtures, the documented refusals, no leaked device blocks, and
  bit-identical repeated runs.

M has one zero singular value per non-singleton component, so the power-law cases run on a largest component and compare
subspaces wherever sigma is repeated."""
import os
import sys
import time
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import REPO, golden_path, load_karate_nx, load_sbm1024_nx

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings('ignore::RuntimeWarning')]   # tol = 1e-9 runs to max_iters on purpose
sys.path.insert(0, os.path.join(REPO, 'oracle'))


def _fresh(**kw):
    from gem_b200.embedding.lle import LocallyLinearEmbedding
    LocallyLinearEmbedding.hyper_params.clear()
    LocallyLinearEmbedding.hyper_params.update({'method_name': 'lle_svd'})
    return LocallyLinearEmbedding(**kw)


def _adj(name, d):
    z = np.load(golden_path('ref_lle_%s_d%d.npz' % (name, d)))
    e, n = z['edges'], int(z['n'])
    return sp.csr_matrix((e[:, 2], (e[:, 0].astype(int), e[:, 1].astype(int))), shape=(n, n)), z


def _bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


# ---------------------------------------------------------------------------------------------------- kernel
def _kernel_graph(seed=5, n=3000):
    """Weighted, non-symmetric, with rows of 700 and 300 nonzeros (the heavy-row path: > 128) and empty rows."""
    rng = np.random.default_rng(seed)
    m = 12 * n
    r = rng.integers(0, n, m)
    c = rng.integers(0, n, m)
    r = np.concatenate((r, np.zeros(700, dtype=np.int64), np.ones(300, dtype=np.int64)))
    c = np.concatenate((c, rng.choice(n, 700, replace=False), rng.choice(n, 300, replace=False)))
    A = sp.csr_matrix((rng.uniform(0.1, 2.0, r.size), (r, c)), shape=(n, n))
    A.sum_duplicates()
    keep = np.ones(n, dtype=bool)
    keep[[5, 17, 2999]] = False                              # zero-degree rows
    A = sp.csr_matrix(sp.diags(keep.astype(float)) @ A)
    A.eliminate_zeros()
    A.sort_indices()
    return A


@pytest.mark.parametrize('b', [4, 64, 132, 148])
@pytest.mark.parametrize('transpose', [False, True])
def test_four_operand_epilogue(gpu_ctx, b, transpose):
    from gem_b200 import _native
    A = _kernel_graph()
    n = A.shape[0]
    assert np.diff(A.indptr).max() > 128 and (np.diff(A.indptr) == 0).sum() >= 3
    AT = sp.csr_matrix(A.T)
    AT.sort_indices()
    rng = np.random.default_rng(b)
    X, S, X0, X1 = (rng.standard_normal((n, b)).astype(np.float32) for _ in range(4))
    al, ga, de, ep = 0.37, -1.25, 0.5, -0.8125
    with _native.DeviceGraph(gpu_ctx, n, A.indptr, A.indices, A.data, AT.indptr, AT.indices, AT.data) as g:
        Y = g.spmm4(X, al, ga, S, de, X0, ep, X1, transpose=transpose)
        Y2 = g.spmm4(X, al, ga, S, de, X0, ep, X1, transpose=transpose)
        Y3 = g.spmm(X, alpha=al, X0=X0, transpose=transpose, gamma=ga, Xself=S, delta=de)
    Op = (AT if transpose else A).astype(np.float32).astype(np.float64)
    ref = al * (Op @ X.astype(np.float64)) + ga * S.astype(np.float64) + de * X0.astype(np.float64) + ep * X1.astype(np.float64)
    scale = np.abs(al) * (abs(Op) @ np.abs(X.astype(np.float64))) + np.abs(S) + np.abs(X0) + np.abs(X1)
    err = (np.abs(Y - ref) / scale).max()
    print('b=%d transpose=%d  max |Y - fp64| / (|alpha||A||X| + |terms|) = %.2e (bar 1e-6)' % (b, transpose, err))
    assert err < 1e-6
    assert _bits(Y, Y2)                                      # no atomics: the same bits every call
    assert np.abs(Y - (Y3 + np.float32(ep) * X1)).max() < 1e-5 * scale.max()   # the three-operand form plus eps X1


def test_spmm4_refuses_a_fourth_operand_alone(gpu_ctx):
    from gem_b200 import _native
    A = _kernel_graph()
    n, b = A.shape[0], 8
    X = np.ones((n, b), dtype=np.float32)
    with _native.DeviceGraph(gpu_ctx, n, A.indptr, A.indices, A.data) as g:
        with pytest.raises(RuntimeError, match='X1 needs Xself and X0'):
            _native.check(_native.lib().gemb_spmm4(g._h, 0, b, 1.0, _native._ptr(X), 0.0, None, 0.0, None, 1.0,
                                                   _native._ptr(X), _native._ptr(X)))


# ---------------------------------------------------------------------------------------------------- parity
def test_karate_golden_composite(native_lib):
    import lap_oracle as lo
    G = load_karate_nx()
    m = _fresh(d=2, tol=1e-9, oversample=16, max_iters=120, operator='composite')
    X = m.learn_embedding(graph=G, is_weighted=True, no_python=True)
    assert m.stats['operator'] == 'composite' and m.stats['algorithm'] == 2
    gold = np.loadtxt(golden_path('karate_LocallyLinearEmbedding.txt'))
    assert X.shape == gold.shape
    d = np.abs(lo.align_signs(X.astype(np.float64), gold) - gold).max()
    print('karate d=2 composite: max |X - golden| = %.2e (bar 1e-4), sigma_0 = %.2e' % (d, m._s[0]))
    assert d < 1e-4
    assert m._s[0] < 2e-3


@pytest.mark.parametrize('name,d', [('karate', 4), ('sbm1024', 16), ('randw120', 8)])
def test_reference_class_outputs_composite(native_lib, name, d):
    import lle_oracle as le
    from gem_b200 import graph as hg
    A, z = _adj(name, d)
    m = _fresh(d=d, tol=1e-9, oversample=24, max_iters=150, operator='composite')
    X = m.learn_embedding(graph=hg.from_scipy(A)).astype(np.float64)
    me = _fresh(d=d, tol=1e-9, oversample=24, max_iters=150, operator='explicit')
    me.learn_embedding(graph=hg.from_scipy(A))
    assert m.stats['operator'] == 'composite' and me.stats['operator'] == 'explicit'
    ref = np.real(z['X'])
    Xo, s, V = le.lle_dense(A, d)
    e_or = np.abs(m._s[1:] ** 2 - s[1:] ** 2).max()
    e_ex = np.abs(m._s ** 2 - me._s ** 2).max()
    print('%s d=%d: |s^2 - oracle| %.2e (explicit run %.2e), |s^2 - explicit run| %.2e, sweeps %d'
          % (name, d, e_or, np.abs(me._s[1:] ** 2 - s[1:] ** 2).max(), e_ex, m.stats['spmm_count']))
    assert e_or < 2e-5 and e_ex < 2e-5
    for j in range(d):
        lo_gap = s[j + 1] ** 2 - s[j] ** 2
        hi_gap = (s[j + 2] ** 2 - s[j + 1] ** 2) if j + 2 < len(s) else 1.0
        if min(lo_gap, hi_gap) > 1e-3:
            sg = np.sign(X[:, j] @ ref[:, j]) or 1.0
            assert np.abs(sg * X[:, j] - ref[:, j]).max() < 2e-4, (j, np.abs(sg * X[:, j] - ref[:, j]).max())
    Qr = np.linalg.qr(ref)[0]
    Xh = X[:, :max(1, d // 2)]
    assert np.linalg.norm(Xh - Qr @ (Qr.T @ Xh), 2) < 2e-3


def test_sbm1024_golden_d128_composite(native_lib):
    import lle_oracle as le
    import networkx as nx
    S, _ = load_sbm1024_nx()
    m = _fresh(d=128, tol=1e-8, oversample=32, max_iters=150, operator='composite')
    X = m.learn_embedding(graph=S).astype(np.float64)
    gold = np.load(golden_path('sbm1024_LocallyLinearEmbedding.npy')).astype(np.float64)
    assert X.shape == gold.shape
    assert abs(np.mean(gold - X)) < 1e-3                                    # the reference's tests/test_sbm.py:94
    A = nx.to_scipy_sparse_array(S, nodelist=list(S.nodes), weight='weight', format='csr')
    Xo, s, V = le.lle_dense(A, 128)
    assert np.allclose(m._s[1:] ** 2, s[1:] ** 2, atol=5e-5), np.abs(m._s ** 2 - s ** 2).max()
    M = le.lle_matrix(A)
    R = M.T @ (M @ X) - X * (m._s[1:] ** 2)
    assert np.linalg.norm(R, axis=0).max() < 2e-4


# ---------------------------------------------------------------------------------------------------- power law
def _principal_sines(X, Y):
    Qx, Qy = np.linalg.qr(X)[0], np.linalg.qr(Y)[0]
    return np.linalg.norm(Qx - Qy @ (Qy.T @ Qx), 2)


RESID_BAR = 1e-4       # ||M^T M v - sigma^2 v|| / ||M||_2^2 of an fp32 vector, fp64 on the host


def test_rmat14_lcc_against_fp64_oracle(native_lib):
    """The vectors are checked by Davis-Kahan against the fp64 oracle's: a unit x with Ritz value t and residual
    r = ||M^T M x - t x|| lies within sin(angle) <= r / gap of the eigenvector whose eigenvalue is nearest t, gap = the
    distance from t to every other eigenvalue; the span of [1, X] (d + 1 vectors) likewise within ||R|| / gap of the
    oracle's d + 1 leading vectors, gap = sigma_{d+1}^2 - max Ritz value.  stop_rule 1 stops on the residual itself."""
    import lle_composite_oracle as lc
    import lle_oracle as le
    from gem_b200 import synth
    from gem_b200.utils.graph_util import get_lcc
    csr, _ = get_lcc(synth.rmat(scale=14, seed=7))
    A = csr.to_scipy()
    d = 16
    m = _fresh(d=d, stop_rule=1, tol=1e-6, max_iters=400, operator='composite')
    with warnings.catch_warnings():
        warnings.simplefilter('error')                       # converged: no warning
        X = m.learn_embedding(graph=csr).astype(np.float64)
    Xo, s, V = lc.lle_composite(A, d + 1, tol=1e-12)         # d + 2 pairs: sigma_{d+1} bounds the gap after the block
    res, nrm = lc.composite_residuals(A, X, m._s[1:])
    err_c = np.abs(m._s ** 2 - s[:d + 1] ** 2).max() / nrm
    me = _fresh(d=d, stop_rule=1, tol=1e-6, max_iters=400, operator='explicit')
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        me.learn_embedding(graph=csr)
    err_e = np.abs(me._s ** 2 - s[:d + 1] ** 2).max() / nrm
    print('R-MAT 14 LCC n=%d nnz=%d ||M||^2=%.4g: composite resid max %.2e (bar %.0e), |s^2 - fp64| / ||M||^2 %.2e; '
          'explicit |s^2 - fp64| / ||M||^2 %.2e; iters %d sweeps %d'
          % (csr.n, csr.nnz, nrm, res.max(), RESID_BAR, err_c, err_e, m.stats['iters'], m.stats['spmm_count']))
    print('sigma^2 fp64   ', s[1:d + 1] ** 2)
    print('sigma^2 compos.', m._s[1:] ** 2)
    print('sigma^2 explic.', me._s[1:] ** 2)
    assert res.max() < RESID_BAR
    assert err_c < 1e-6
    M = le.lle_matrix(A)
    MT = sp.csr_matrix(M.T)
    B = lambda Y: MT @ (M @ Y)
    s2, th = s ** 2, m._s[1:] ** 2
    Xn = X / np.linalg.norm(X, axis=0)
    r = np.linalg.norm(B(Xn) - Xn * th, axis=0)
    checked = 0
    for j in range(d):
        gap = np.abs(np.delete(s2, j + 1) - th[j]).min()
        bound = r[j] / gap
        sine = _principal_sines(Xn[:, j:j + 1], V[:, j + 1:j + 2])
        print('pair %2d: sin %.2e  Davis-Kahan bound %.2e' % (j + 1, sine, bound))
        if bound < 0.5:
            assert sine <= bound + 1e-6, (j, sine, bound)
            checked += 1
    assert checked >= d - 2, checked                          # the bound is informative for (nearly) every pair
    Y = np.linalg.qr(np.concatenate((np.full((csr.n, 1), 1.0 / np.sqrt(csr.n)), X), axis=1))[0]
    H = Y.T @ B(Y)
    gap = s2[d + 1] - np.linalg.eigvalsh(0.5 * (H + H.T)).max()
    bound = np.linalg.norm(B(Y) - Y @ H, 2) / gap
    sine = _principal_sines(Y, V[:, :d + 1])
    print('span of the d + 1 vectors: sin %.2e  Davis-Kahan bound %.2e (gap %.3g)' % (sine, bound, gap))
    assert bound < 0.1 and sine <= bound + 1e-6


def test_rmat20_lcc_d128_auto(native_lib):
    import lle_composite_oracle as lc
    from gem_b200 import _native
    from gem_b200.graph import HostCSR
    from gem_b200.utils.graph_util import get_lcc
    with _native.Context(0) as ctx:
        indptr, indices, _ = _native.synth_rmat(ctx, 20, permute=True)
    csr, _ = get_lcc(HostCSR(1 << 20, indptr, indices, symmetric=True))
    from gem_b200.embedding.lle import choose_operator
    assert choose_operator(csr) == 'composite'
    m = _fresh(d=128)                     # operator='auto', the default solver options
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        X = m.learn_embedding(graph=csr)
    wall = time.perf_counter() - t0
    assert m.stats['operator'] == 'composite' and m.stats['converged'] == 1
    res, nrm = lc.composite_residuals(csr.to_scipy(), X, m._s[1:])
    print('R-MAT 20 LCC n=%d nnz=%d d=128: wall %.1f s (budget 120 s), iters %d, sweeps %d, solve device %.0f ms, '
          'resid max %.2e (bar %.0e), ||M||^2 %.4g, sigma^2[1:4] %s' % (csr.n, csr.nnz, wall, m.stats['iters'],
                                                       m.stats['spmm_count'], m.stats['total_ms'], res.max(), RESID_BAR,
                                                       nrm, m._s[1:4] ** 2))
    assert res.max() < RESID_BAR
    assert wall < 120.0


# ---------------------------------------------------------------------------------------------------- kept behaviour
@pytest.mark.parametrize('name,d', [('karate', 2), ('karate', 4), ('sbm1024', 16), ('randw120', 8)])
def test_auto_is_explicit_bit_for_bit(native_lib, name, d):
    from gem_b200 import graph as hg
    A, _ = _adj(name, d)
    Xa = _fresh(d=d, tol=1e-9, max_iters=60).learn_embedding(graph=hg.from_scipy(A))
    me = _fresh(d=d, tol=1e-9, max_iters=60, operator='explicit')
    Xe = me.learn_embedding(graph=hg.from_scipy(A))
    assert _bits(Xa, Xe)


def test_composite_runs_are_bit_identical_and_release_their_blocks(native_lib):
    from gem_b200 import _native
    from gem_b200 import graph as hg
    A, _ = _adj('sbm1024', 16)

    def run():
        m = _fresh(d=16, tol=1e-9, max_iters=40, operator='composite')
        return m.learn_embedding(graph=hg.from_scipy(A)), m._s

    X1, s1 = run()
    before = _native.mem_live_blocks()
    X2, s2 = run()
    if os.environ.get('GEMB_CACHE_MB', '').strip() != '0':
        assert _native.mem_live_blocks() == before
    assert _bits(X1, X2) and _bits(s1, s2)


def test_mode2_refusals_and_blocks(gpu_ctx):
    from gem_b200 import _native, graph as hg
    from gem_b200.embedding.lle import lle_composite_operator
    A, _ = _adj('randw120', 8)
    P, PT = lle_composite_operator(hg.from_scipy(A))
    with _native.DeviceGraph(gpu_ctx, P.n, P.indptr, P.indices, P.data_f32()) as g:          # no transpose
        with pytest.raises(RuntimeError, match='spectral_mode 2 needs A = D\\^-1 W uploaded together with its transpose'):
            g.hope(9, 0.0, spectral_mode=2)
    with _native.DeviceGraph(gpu_ctx, P.n, P.indptr, P.indices, P.data_f32(), PT.indptr, PT.indices, PT.data_f32()) as g:
        with pytest.raises(RuntimeError, match='spectral_mode 2 runs on the Chebyshev'):
            g.hope(9, 0.0, spectral_mode=2, algorithm=3)
        X, lam, st = g.hope(9, 0.0, spectral_mode=2, tol=1e-9, max_iters=50)   # warm-up: grows the context's scratch
        assert lam.shape == (9,) and np.all(np.diff(lam) <= 0) and lam[0] <= 0.0
        assert st['spmm_count'] % 2 == 0                     # one application = two sweeps
        before = _native.mem_live_blocks()
        X2, lam2, _ = g.hope(9, 0.0, spectral_mode=2, tol=1e-9, max_iters=50)
        if os.environ.get('GEMB_CACHE_MB', '').strip() != '0':
            assert _native.mem_live_blocks() == before
        assert _bits(X, X2) and _bits(lam, lam2)


def test_mode2_refused_on_a_multi_gpu_communicator(native_lib):
    """Needs >= 2 GPUs (skipped on one): scripts/mgpu_lle_check.py, launched with torchrun as tests/test_gpu_multi.py does."""
    import json
    import socket
    import subprocess
    if native_lib.gemb_device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    sck = socket.socket(); sck.bind(('127.0.0.1', 0)); port = sck.getsockname()[1]; sck.close()
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
           '127.0.0.1', '--master-port', str(port), os.path.join(REPO, 'scripts/mgpu_lle_check.py')]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    line = [l for l in p.stdout.splitlines() if l.startswith('{')]
    assert p.returncode == 0 and line, p.stdout[-2000:] + p.stderr[-2000:]
    assert json.loads(line[-1])['ok']
