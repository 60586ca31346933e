"""One application of each operator gemb_hope solves for (gemb_hope_apply), and the row-scaled SpMM sweep
(gemb_spmm_scaled), against fp64 entry by entry (oracle/proximity_oracle.py: operator_apply, operator_abs).

The solver tests (test_gpu_hope_proximity.py) see S only through converged triplets, at bars an operator error that is
small against sigma_max, or that lies outside the top subspace, passes.  Here every entry of Y = S X (S^T X) is held to
    |Y - S X| <= c * 2e-6 * (|S| |X|)     c = SpMM sweeps per application: J (modes 0 and 5), 1 (mode 1), 2 (modes 2-4),
2e-6 being test_gpu_spmm.py's per-sweep bar and |S| |X| (operator_abs: the same products on |A|, |D|, |X|) the scale of
the forward error of any summation order; an entry whose scale is 0 must be exactly 0.  Data whose every partial sum
is exact in fp32 (integers, powers of two) must give the fp64 result bit for bit.

Graphs: undirected Karate (symmetric upload), po.random_digraph (an isolated node, a row without out-edges), R-MAT
scale 12 and 15 (hub rows on the chunked heavy-row kernels) unweighted, weighted and randomly oriented (A and A^T then
have different hub rows), test_gpu_spmm.py's heavy-threshold graph (degrees 128/129/512/513/1025 at tile edges) and a
graph without edges.  Modes 2 and 5 take P = D_out^-1 A uploaded with its transpose, as their callers upload it."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import REPO, load_karate_nx
from test_gpu_spmm import _capacity_graph, _eighths, _hub_graph, _threshold_graph

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(REPO, 'oracle'))
import hope_oracle as ho
import proximity_oracle as po

EPS = 2e-6                 # test_gpu_spmm.py's bar for one sweep, relative to the sweep's |alpha| |A| |X| + epilogue terms
ALPHA = 0.5                # rooted PageRank
KATZ_TERMS = 5
WIDTHS = [4, 12, 80, 132, 1024]
MARGINS = {}               # worst err / bar per check: printed at the end of the module (1.0 = at the bar)


@pytest.fixture(scope='module', autouse=True)
def _report_margins():
    yield
    for k in sorted(MARGINS, key=str):
        print('worst err / bar %-28s %.3g' % (k, MARGINS[k]))


def _f32(A):
    """A as a CSR of fp32-representable fp64 values, sorted indices: what the device holds, in fp64."""
    A = sp.csr_matrix(A, dtype=np.float32).astype(np.float64)
    A.sort_indices()
    return A


def _oriented(A, seed):
    """Every undirected edge of the symmetric A kept in one random direction, with weights in [0.1, 2)."""
    U = sp.triu(A, k=1).tocoo()
    rng = np.random.default_rng(seed)
    flip = rng.random(U.nnz) < 0.5
    r, c = np.where(flip, U.col, U.row), np.where(flip, U.row, U.col)
    return _f32(sp.csr_matrix((rng.uniform(0.1, 2.0, U.nnz), (r, c)), shape=A.shape))


def _sym_weighted(A, seed):
    U = sp.triu(A, k=1).tocsr()
    U.data = np.random.default_rng(seed).uniform(0.1, 2.0, U.nnz)
    return _f32(U + U.T)


_GRAPHS = {}


def _graph(name):
    """(A in fp64, symmetric upload?, weighted?) -- cached: the R-MAT generators and the oracle inputs are reused."""
    if name in _GRAPHS:
        return _GRAPHS[name]
    import networkx as nx
    from gem_b200 import synth
    if name == 'karate':
        G = nx.Graph(load_karate_nx().to_undirected())
        A = _f32(ho.adjacency_from_nx(G))
        out = (A, True, bool(np.any(A.data != 1.0)))
    elif name == 'randw200':
        out = (_f32(po.random_digraph()), False, True)
    elif name.startswith('rmat'):
        scale = int(name[4:6])
        A = _f32(synth.rmat(scale=scale, edge_factor=8, seed=3 if scale == 12 else 4).to_scipy())
        kind = name[6:]
        if kind == '':
            out = (A, True, False)
        elif kind == 'w':
            out = (_sym_weighted(A, scale), True, True)
        else:
            out = (_oriented(A, scale), False, True)
    elif name == 'threshold':
        out = (_f32(_threshold_graph(np.random.default_rng(21)).to_scipy()), False, False)
    elif name == 'empty':
        out = (sp.csr_matrix((300, 300)), True, False)
    else:
        raise ValueError(name)
    _GRAPHS[name] = out
    return out


GRAPHS = ['karate', 'randw200', 'rmat12', 'rmat12w', 'rmat12o', 'rmat15', 'rmat15w', 'rmat15o', 'threshold', 'empty']


def _upload(ctx, A, symmetric, weighted):
    from gem_b200 import _native
    A = sp.csr_matrix(A)
    data = A.data.astype(np.float32) if weighted and A.nnz else None
    if symmetric:
        return _native.DeviceGraph(ctx, A.shape[0], A.indptr, A.indices, data)
    T = A.T.tocsr()
    T.sort_indices()
    tdata = T.data.astype(np.float32) if data is not None else None
    return _native.DeviceGraph(ctx, A.shape[0], A.indptr, A.indices, data, T.indptr, T.indices, tdata)


def _operand(name, mode):
    """(uploaded matrix in fp64, symmetric, weighted, coefficient, opts) for spectral_mode `mode` on graph `name`."""
    A, sym, w = _graph(name)
    if mode in (2, 5):
        P = _f32(po.transition(A))
        assert np.all(np.asarray(abs(P).sum(axis=1)).ravel() <= 1.0 + 1e-6)
        return P, False, P.nnz > 0, (ALPHA if mode == 5 else 0.0), {}
    if mode == 0:
        rs = np.asarray(abs(A).sum(axis=1)).ravel()
        return A, sym, w, 0.5 / max(1.0, rs.max() if rs.size else 1.0), {'katz_terms': KATZ_TERMS}
    return A, sym, w, 0.0, {}


def _sweeps(mode, J):
    return {0: J, 1: 1, 2: 2, 3: 2, 4: 2, 5: J}[mode]


def _check_bar(Y, ref, bound, sweeps, key):
    err = np.abs(Y.astype(np.float64) - ref)
    zero = bound == 0
    assert not np.any(err[zero]), 'an entry whose |S| |X| is 0 is %g' % err[zero].max()
    ratio = float((err[~zero] / (sweeps * EPS * bound[~zero])).max()) if (~zero).any() else 0.0
    MARGINS[key] = max(MARGINS.get(key, 0.0), ratio)
    assert ratio <= 1.0, '%s: err / bar = %.3g' % (key, ratio)
    return ratio


def _apply_and_check(ctx, name, mode, b, transposes=(False, True), seed=0, key=None):
    A, sym, w, coef, opts = _operand(name, mode)
    coef32 = float(np.float32(coef))                          # what the kernels compute with
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((A.shape[0], b)).astype(np.float32)
    worst = 0.0
    with _upload(ctx, A, sym, w) as g:
        for tr in transposes:
            Y, J = g.hope_apply(X, coef, transpose=tr, spectral_mode=mode, **opts)
            if mode == 5:
                assert J == po.rooted_pagerank_terms(coef32, float(np.float32(1e-7)))
            elif mode == 0:
                assert J == KATZ_TERMS
            else:
                assert J == 0
            terms = J if mode in (0, 5) else None
            ref = po.operator_apply(A, mode, X, tr, coef32, terms)
            bound = po.operator_abs(A, mode, X, tr, coef32, terms)
            worst = max(worst, _check_bar(Y, ref, bound, _sweeps(mode, J), key or ('grid', mode)))
    return worst


def _modes(name):
    return [m for m in range(6) if m != 1 or _graph(name)[1]]     # mode 1 needs a symmetric upload


@pytest.mark.parametrize('name', GRAPHS)
def test_every_operator_against_fp64(gpu_ctx, name):
    """S X and S^T X for every spectral_mode (mode 1 on the symmetric uploads) at b = 12 and 80."""
    for mode in _modes(name):
        for b in (12, 80):
            r = _apply_and_check(gpu_ctx, name, mode, b, seed=mode * 7 + b)
            print('%-9s mode %d b %4d: worst |Y - SX| / (c 2e-6 |S||X|) = %.3g' % (name, mode, b, r))


@pytest.mark.parametrize('b', WIDTHS)
def test_block_widths(gpu_ctx, b):
    """b = 4 (one thread per row), 12 (3-thread groups that do not divide 256), 80, 132 (33-thread groups, 7 rows per
    CTA pass), 1024 (one row per pass) on the oriented weighted R-MAT scale 12 graph (mode 1: its weighted undirected
    form)."""
    for mode in range(6):
        name = 'rmat12w' if mode == 1 else 'rmat12o'
        r = _apply_and_check(gpu_ctx, name, mode, b, seed=b + mode, key=('widths', mode))
        print('b %4d mode %d on %s: worst err / bar = %.3g' % (b, mode, name, r))


def test_graph_without_edges_is_exact(gpu_ctx):
    """No edges: S = 0 for modes 0, 1, 3 and 4 (D = 0: no 1/0 reaches Y), -I for mode 2 (P = 0, M = I), and rooted
    PageRank gives exactly (1 - alpha) X, (1 - alpha) rounded to fp32 once, as the last sweep's epilogue does."""
    n, b = 300, 80
    X = np.random.default_rng(5).standard_normal((n, b)).astype(np.float32)
    E = sp.csr_matrix((n, n))
    with _upload(gpu_ctx, E, True, False) as gs, _upload(gpu_ctx, E, False, False) as gt:
        for tr in (False, True):
            for mode, coef, kw in ((0, 0.3, {'katz_terms': 4}), (3, 0.0, {}), (4, 0.0, {})):
                for g in (gs, gt):
                    Y, _ = g.hope_apply(X, coef, transpose=tr, spectral_mode=mode, **kw)
                    assert np.array_equal(Y, np.zeros_like(X))
            Y, _ = gs.hope_apply(X, 0.0, spectral_mode=1)
            assert np.array_equal(Y, np.zeros_like(X))
            Y, _ = gt.hope_apply(X, 0.0, spectral_mode=2)
            assert np.array_equal(Y, -X)
            for alpha in (0.3, 0.5, 0.99):
                Y, J = gt.hope_apply(X, alpha, transpose=tr, spectral_mode=5)
                a = float(np.float32(alpha))
                assert J == po.rooted_pagerank_terms(a, float(np.float32(1e-7)))
                assert np.array_equal(Y, np.float32(1.0 - a) * X)


# ------------------------------------------------------------------------------------------------ exact arithmetic
def _circulant(n, k):
    """The k-regular circulant graph (offsets +-1 .. +-k/2), unweighted: D = 1 / (2k) for every row."""
    offs = np.concatenate([np.arange(1, k // 2 + 1), -np.arange(1, k // 2 + 1)])
    rows = np.repeat(np.arange(n), k)
    cols = (rows + np.tile(offs, n)) % n
    return _f32(sp.csr_matrix((np.ones(rows.size), (rows, cols)), shape=(n, n)))


def _star(leaves, hub):
    """A star whose hub (row `hub`) has `leaves` neighbours and weighted degree 1024: unit weights for 1024 leaves; for
    1025, two leaves of weight 1/2.  D: 1/2048 at the hub, 1/2 or 1 at the leaves.  The hub row takes 2 (1024) or 3
    (1025) heavy-row chunks of 512."""
    n = leaves + 1
    others = np.array([i for i in range(n) if i != hub])
    w = np.ones(leaves)
    if leaves == 1025:
        w[[3, 700]] = 0.5
    assert w.sum() == 1024
    r = np.concatenate([np.full(leaves, hub), others])
    c = np.concatenate([others, np.full(leaves, hub)])
    return _f32(sp.csr_matrix((np.concatenate([w, w]), (r, c)), shape=(n, n)))


@pytest.mark.parametrize('graph', ['regular16', 'regular256', 'star1024', 'star1025'])
def test_common_neighbours_and_adamic_adar_exact(gpu_ctx, graph):
    """Powers of two in D and X in {-4..4}: every partial sum of both sweeps is exact in fp32, so S X and S^T X equal
    fp64 bit for bit -- for a symmetric upload (inv_degree_kernel reads A twice) and one with A^T (it reads both)."""
    if graph.startswith('regular'):
        k = int(graph[7:])
        A = _circulant(8 * k if k > 16 else 4096, k)
    else:
        A = _star(int(graph[4:]), hub=517)
    d = po.inv_degree(A)
    assert np.all(d == 2.0 ** np.round(np.log2(d)))                  # powers of two
    weighted = bool(np.any(A.data != 1.0))
    rng = np.random.default_rng(len(graph))
    for b in (4, 80):
        X = rng.integers(-4, 5, (A.shape[0], b)).astype(np.float32)
        for sym in (True, False):
            with _upload(gpu_ctx, A, sym, weighted) as g:
                for mode in (3, 4):
                    for tr in (False, True):
                        Y, _ = g.hope_apply(X, 0.0, transpose=tr, spectral_mode=mode)
                        ref = po.operator_apply(A, mode, X, tr)
                        assert np.array_equal(Y.astype(np.float64), ref), (mode, tr, sym, b,
                                                                           np.abs(Y - ref).max())


def _pow2_scales(rng, n):
    return rng.choice([-4.0, -2.0, -1.0, -0.5, -0.25, 0.0, 0.25, 0.5, 1.0, 2.0, 4.0], n).astype(np.float32)


def _scaled_ref(csr, X, rscale, alpha, transpose):
    A = csr.to_scipy().astype(np.float64)
    if transpose:
        A = A.T.tocsr()
    return alpha * rscale.astype(np.float64)[:, None] * (A @ X.astype(np.float64)), \
        abs(alpha) * np.abs(rscale.astype(np.float64))[:, None] * (abs(A) @ np.abs(X.astype(np.float64)))


def _scaled_run(ctx, csr, b, alpha, rscale, rng, exact, transposes=(False, True)):
    from gem_b200 import _native
    t = csr.transpose()
    worst = 0.0
    with _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, csr.data_f32(), t.indptr, t.indices,
                             t.data_f32()) as g:
        for tr in transposes:
            if exact:
                X = rng.integers(-4, 5, (csr.n, b)).astype(np.float32)
            else:
                X = rng.standard_normal((csr.n, b)).astype(np.float32)
            Y = g.spmm_scaled(X, rscale, alpha=alpha, transpose=tr)
            ref, bound = _scaled_ref(csr, X, rscale, float(np.float32(alpha)), tr)
            if exact:
                assert np.array_equal(Y.astype(np.float64), ref), np.abs(Y - ref).max()
            else:
                worst = max(worst, _check_bar(Y, ref, bound, 1, ('spmm_scaled', b)))
    return worst


def test_spmm_scaled_exact(gpu_ctx):
    """Signed power-of-two and zero row scales, multiples of 1/8 as weights, X in {-4..4}: exact on the R-MAT hub graph
    (heavy rows: the scale in the finish kernel), the heavy-threshold graph, the staging-capacity graph and a graph
    without edges (Y = 0)."""
    from gem_b200 import graph as hg
    rng = np.random.default_rng(61)
    hub = _hub_graph('eighths')
    thr = _threshold_graph(np.random.default_rng(21))
    thr.data = _eighths(rng, thr.nnz)
    cap = _capacity_graph(np.random.default_rng(31))
    cap.data = _eighths(rng, cap.nnz)
    empty = hg.HostCSR(5000, np.zeros(5001, np.int64), np.zeros(0, np.int32))
    for csr, widths in ((hub, (4, 12, 80, 1024)), (thr, (4, 12, 80)), (cap, (80,)), (empty, (80,))):
        for b in widths:
            for alpha in (1.0, -0.5, 4.0):
                _scaled_run(gpu_ctx, csr, b, alpha, _pow2_scales(rng, csr.n), rng, exact=True)
    X = rng.standard_normal((5000, 80)).astype(np.float32)
    from gem_b200 import _native
    with _native.DeviceGraph(gpu_ctx, 5000, empty.indptr, empty.indices, None) as g:
        assert np.array_equal(g.spmm_scaled(X, np.ones(5000, np.float32)), np.zeros_like(X))


@pytest.mark.parametrize('b', WIDTHS)
def test_spmm_scaled_real(gpu_ctx, b):
    """Real weights and scales (a tenth of them 0) at every block width: the per-sweep bar, A and A^T."""
    rng = np.random.default_rng(b)
    csr = _hub_graph('real')
    s = rng.uniform(-2.0, 2.0, csr.n).astype(np.float32)
    s[rng.random(csr.n) < 0.1] = 0.0
    r = _scaled_run(gpu_ctx, csr, b, 0.7, s, rng, exact=False)
    print('spmm_scaled b %d: worst err / bar = %.3g' % (b, r))


def test_spmm_scaled_refusals(gpu_ctx):
    from gem_b200 import _native
    lib = _native.lib()
    A, _, _ = _graph('karate')
    with _upload(gpu_ctx, A, True, False) as g:
        n0 = lib.gemb_launch_count()
        for b in (6, 1028):
            with pytest.raises(RuntimeError, match='bad argument'):
                g.spmm_scaled(np.ones((A.shape[0], b), np.float32), np.ones(A.shape[0], np.float32))
        assert lib.gemb_launch_count() == n0


# ------------------------------------------------------------------------------------------- rooted PageRank series
def _digraph_P():
    return _f32(po.transition(po.random_digraph()))


@pytest.mark.parametrize('katz_tol', [1e-3, 1e-7])
@pytest.mark.parametrize('alpha', [0.05, 0.5, 0.9, 0.99])
def test_rooted_pagerank_terms_and_tail(gpu_ctx, alpha, katz_tol):
    """J_out = ceil(log katz_tol / log alpha) of the fp32 arguments; Y = (1 - alpha) sum_{j<=J} (alpha P)^j X at the
    J-sweep bar; and, as the header says, ||(S_J - S_inf) X||_inf <= alpha^(J+1) ||X||_inf against the fp64 inverse
    (for S: ||alpha P||_inf <= alpha; S^T has no such bound and is held to the series only)."""
    P = _digraph_P()
    n = P.shape[0]
    a, t = float(np.float32(alpha)), float(np.float32(katz_tol))
    X = np.random.default_rng(7).standard_normal((n, 8)).astype(np.float32)
    Sinf = (1.0 - a) * np.linalg.inv(np.eye(n) - a * P.toarray())
    with _upload(gpu_ctx, P, False, True) as g:
        for tr in (False, True):
            Y, J = g.hope_apply(X, alpha, transpose=tr, spectral_mode=5, katz_tol=katz_tol)
            assert J == po.rooted_pagerank_terms(a, t)
            ref = po.operator_apply(P, 5, X, tr, a, J)
            bound = po.operator_abs(P, 5, X, tr, a, J)
            r = _check_bar(Y, ref, bound, J, ('rpr_series', alpha))
            if not tr:
                xm = np.abs(X).max()
                tail = np.abs(ref - Sinf @ X).max()
                assert tail <= a ** (J + 1) * xm * (1 + 1e-6)
                assert np.abs(Y - Sinf @ X).max() <= a ** (J + 1) * xm * (1 + 1e-6) + J * EPS * bound.max()
                print('alpha %.2f tol %.0e: J %d, fp64 tail %.3g <= alpha^(J+1) |X| = %.3g; err / bar %.3g'
                      % (alpha, katz_tol, J, tail, a ** (J + 1) * xm, r))
        for terms in (1, 2, 3):
            Y, J = g.hope_apply(X, alpha, spectral_mode=5, katz_tol=katz_tol, katz_terms=terms)
            assert J == terms                                        # katz_terms overrides katz_tol
            _check_bar(Y, po.operator_apply(P, 5, X, False, a, terms), po.operator_abs(P, 5, X, False, a, terms),
                       terms, ('rpr_terms', terms))


# ----------------------------------------------------------------------------------------------------- refusals
def _rescale_row(P, r, factor):
    """P with row r multiplied by `factor` in fp32; returns (P', its row sum in fp64 over the fp32 values)."""
    Q = P.copy()
    s, e = Q.indptr[r], Q.indptr[r + 1]
    assert e > s
    Q.data[s:e] = (Q.data[s:e].astype(np.float32) * np.float32(factor)).astype(np.float64)
    return Q, float(Q.data[s:e].sum())


def test_row_sum_refusal_at_the_boundary(gpu_ctx):
    """A P row summing to 1 + 2e-5 is refused ('row sum <= 1'), one summing to 1 + 5e-6 accepted, wherever the row is:
    the R-MAT hub row (heavy), the last row, a row whose index is not a multiple of 32.  The refusal costs exactly the
    one pass over the CSR that finds it -- no SpMM runs -- and leaks no block."""
    from gem_b200 import _native
    lib = _native.lib()
    cases = []
    Ph = _f32(po.transition(_graph('rmat12')[0]))
    cases.append(('hub', Ph, int(np.argmax(np.diff(Ph.indptr)))))
    Pd = _digraph_P()
    assert Pd.indptr[-1] > Pd.indptr[-2]
    cases.append(('last', Pd, Pd.shape[0] - 1))
    r = next(i for i in range(33, Pd.shape[0]) if i % 32 and Pd.indptr[i + 1] > Pd.indptr[i])
    cases.append(('row %d' % r, Pd, r))
    for label, P, row in cases:
        X = np.random.default_rng(row).standard_normal((P.shape[0], 8)).astype(np.float32)
        for factor, ok in ((1 + 2e-5, False), (1 + 5e-6, True)):
            Q, rs = _rescale_row(P, row, factor)
            assert (rs > 1 + 1e-5) != ok, (label, rs)
            with _upload(gpu_ctx, Q, False, True) as g:
                blocks, n0 = _native.mem_live_blocks(), lib.gemb_launch_count()
                if ok:
                    Y, J = g.hope_apply(X, ALPHA, spectral_mode=5)
                    ref = po.operator_apply(Q, 5, X, False, ALPHA, J)
                    _check_bar(Y, ref, po.operator_abs(Q, 5, X, False, ALPHA, J), J, ('rowsum', label))
                else:
                    with pytest.raises(RuntimeError, match='row sum <= 1'):
                        g.hope_apply(X, ALPHA, spectral_mode=5)
                    assert lib.gemb_launch_count() == n0 + 1            # csr_rowsum_kernel, nothing else
                    with pytest.raises(RuntimeError, match='row sum <= 1'):
                        g.hope(8, ALPHA, spectral_mode=5)             # the solver takes the same path
                    if os.environ.get('GEMB_CACHE_MB', '').strip() != '0':
                        assert _native.mem_live_blocks() == blocks
                print('%s: row sum - 1 = %.3g -> %s' % (label, rs - 1, 'accepted' if ok else 'refused'))


def test_negative_weight_refusal(gpu_ctx):
    """One -1e-30 weight as the very last nonzero: refused by modes 4 and 5 (after the one pass that finds it), taken
    by mode 3.  -0.0 is not negative, for the device as for hope.check_proximity."""
    from gem_b200 import _native
    from gem_b200 import graph as hg
    from gem_b200.embedding.hope import check_proximity
    lib = _native.lib()
    A = _graph('randw200')[0]
    P = _digraph_P()
    X = np.random.default_rng(9).standard_normal((A.shape[0], 8)).astype(np.float32)
    for tiny in (np.float32(-1e-30), np.float32(-0.0)):
        An, Pn = A.copy(), P.copy()
        An.data[-1] = tiny
        Pn.data[-1] = tiny
        refused = bool(tiny < 0)
        for mode, M in ((3, An), (4, An), (5, Pn)):
            coef = ALPHA if mode == 5 else 0.0
            proximity = {3: 'common_neighbors', 4: 'adamic_adar', 5: 'rooted_pagerank'}[mode]
            host_refuses = False
            try:
                check_proximity(proximity, ALPHA if mode == 5 else None, csr=hg.from_scipy(M))
            except ValueError:
                host_refuses = True
            with _upload(gpu_ctx, M, False, True) as g:
                n0 = lib.gemb_launch_count()
                if refused and mode >= 4:
                    assert host_refuses
                    with pytest.raises(RuntimeError, match='non-negative weights'):
                        g.hope_apply(X, coef, spectral_mode=mode)
                    assert lib.gemb_launch_count() == n0 + 1
                else:
                    assert not host_refuses
                    Y, J = g.hope_apply(X, coef, spectral_mode=mode)
                    terms = J if mode == 5 else None
                    _check_bar(Y, po.operator_apply(M, mode, X, False, coef, terms),
                               po.operator_abs(M, mode, X, False, coef, terms), _sweeps(mode, J), ('negzero', mode))


def test_argument_refusals_launch_nothing(gpu_ctx):
    from gem_b200 import _native
    lib = _native.lib()
    A = _graph('randw200')[0]
    K, _, _ = _graph('karate')
    X = np.ones((A.shape[0], 8), np.float32)
    XK = np.ones((K.shape[0], 8), np.float32)
    with _upload(gpu_ctx, A, False, True) as g, _upload(gpu_ctx, K, True, False) as gk:
        blocks = _native.mem_live_blocks()
        for call, match in (
                (lambda: g.hope_apply(X, 0.1, spectral_mode=0), 'katz_terms > 0'),
                (lambda: g.hope_apply(X, -0.5, spectral_mode=0, katz_terms=3), 'katz_terms > 0'),
                (lambda: g.hope_apply(np.ones((A.shape[0], 6), np.float32), 0.0, spectral_mode=3), 'multiple of 4'),
                (lambda: g.hope_apply(np.ones((A.shape[0], 1028), np.float32), 0.0, spectral_mode=3), 'multiple of 4'),
                (lambda: g.hope_apply(X, 0.0, spectral_mode=3, algorithm=2), 'general solver'),
                (lambda: g.hope_apply(X, 1.0, spectral_mode=5), '0 < alpha < 1'),
                (lambda: g.hope_apply(X, 0.0, spectral_mode=1), 'symmetric upload'),
                (lambda: gk.hope_apply(XK, 0.0, spectral_mode=2), 'transpose'),
                (lambda: g.hope_apply(X, 0.0, spectral_mode=6), 'spectral_mode')):
            n0 = lib.gemb_launch_count()
            with pytest.raises(RuntimeError, match=match):
                call()
            assert lib.gemb_launch_count() == n0, match
        if os.environ.get('GEMB_CACHE_MB', '').strip() != '0':
            assert _native.mem_live_blocks() == blocks


# ---------------------------------------------------------------------------------------- repeatability, memory
def test_repeated_applications_are_bit_identical(gpu_ctx):
    """Every mode on the oriented R-MAT scale 15 graph (heavy rows in A and A^T; mode 1 on its undirected weighted
    form): the same bits on every call, and no device block kept by a call (counted after the first, which may grow
    the context's heavy-row scratch)."""
    from gem_b200 import _native
    for mode in range(6):
        A, sym, w, coef, opts = _operand('rmat15w' if mode == 1 else 'rmat15o', mode)
        X = np.random.default_rng(mode).standard_normal((A.shape[0], 80)).astype(np.float32)
        with _upload(gpu_ctx, A, sym, w) as g:
            for tr in (False, True):
                Y1, J1 = g.hope_apply(X, coef, transpose=tr, spectral_mode=mode, **opts)
                before = _native.mem_live_blocks()
                Y2, J2 = g.hope_apply(X, coef, transpose=tr, spectral_mode=mode, **opts)
                if os.environ.get('GEMB_CACHE_MB', '').strip() != '0':
                    assert _native.mem_live_blocks() == before
                assert J1 == J2 and Y1.tobytes() == Y2.tobytes()

