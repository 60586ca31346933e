"""node2vec's SGNS kernel and Graph Factorization's edge-SGD kernels at every embedding width they are built for, against the fp64
oracles (oracle/n2v_oracle.c, pinned to the reference binary by tests/test_oracle_n2v.py; oracle/gf_oracle.py, pinned to the
reference class by tests/test_oracle_gf.py).

sgns_kernel<NV, VEC> (n2v.cu, dispatch_sgns) keeps NV values of a row per lane: the scalar layout (value v of a lane is dimension
32 v + lane, NV = 1, 2, 4, 8, 16, the last value masked when d % 32 != 0) or, when d % 128 == 0, the float4 layout (dimension
(v / 4) 128 + 4 lane + v % 4, NV = 4, 8, 12, 16).  A pair's five negatives are updated together from registers, or one by one
through memory when one of them repeats (small vocabularies).  Both are covered here at every NV:
  * sequential mode (one warp on the binary's single stream) against the oracle on the same walks;
  * Hogwild mode with ONE walk per epoch: one warp, so the result is a deterministic function of the per-walk stream, which the
    oracle reproduces with walk_streams=True;
  * the pair count of a full Hogwild run, which the races cannot change, against a restatement of the window draws.
gf_sequential_kernel<NV> / gf_rows_kernel<NV> (gf.cu) keep NV = 1 ... 32 values per lane (d <= 1024): both schedules against the
oracle's sweep at every NV, and bit-identical to each other.

Bars, the same at every width: node2vec 2e-3 max|Xo| with correlation above 0.99999 (tests/test_gpu_n2v.py at d <= 16), GF 2e-4
max|Xo| (tests/test_gpu_gf.py).  Every comparison prints its measured error (pytest -s)."""
import os
import sys

import numpy as np
import pytest

from conftest import REPO, golden_path, load_sbm1024_nx, nx_from_npz

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(REPO, 'oracle'))

M31 = 2147483647
NEG = 5                      # negatives per pair (SG_NEG)
# node2vec d -> sgns_kernel<NV, VEC>: scalar NV = 1 (1), 2 (40, 64), 4 (100), 8 (200), 16 (300); float4 NV = 4, 8, 12, 16
WIDTHS = [1, 40, 64, 100, 128, 200, 256, 300, 384, 512]
# gf.cu NV = 2 (33, 64), 4 (100, 128), 8 (256), 16 (512), 32 (1000, 1024)
GF_WIDTHS = [33, 64, 100, 128, 256, 512, 1000, 1024]


def _inputs(G):
    from gem_b200 import graph as hg
    return hg.n2v_inputs_from_networkx(G)


def _dev(ctx, csr):
    from gem_b200 import _native
    return _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)


def _launches():
    from gem_b200 import _native
    return int(_native.lib().gemb_launch_count())


def _smem_optin():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


# ---------------------------------------------------------------------------------------------- restated window draws
def _walk_pairs(st, L, win):
    """Pairs of one walk trained from stream state st, and the state after it: per word one draw picks the window
    (offset = draw % win, pairs with the 2 (win - offset) neighbours inside the walk), and every pair then takes ten draws
    (two per negative, also for a negative that is skipped because it equals the word)."""
    a10 = [pow(16807, 10 * k, M31) for k in range(2 * win + 1)]
    pairs = 0
    for pos in range(L):
        st = st * 16807 % M31
        off = st % win
        n = min(pos + win - off, L - 1) - max(pos - win + off, 0)
        pairs += n
        st = st * a10[n] % M31
    return pairs, st


def _pairs_sequential(seed, V, d, n_walks, L, win, iters):
    """Sequential mode: one stream, after the V d draws of the initial embedding."""
    st, pairs = pow(16807, V * d, M31) * seed % M31, 0
    for _ in range(iters * n_walks):
        p, st = _walk_pairs(st, L, win)
        pairs += p
    return pairs


def _pairs_hogwild(seed, n_walks, L, win, iters):
    """Hogwild mode: walk w of epoch e starts at 2^30 + (e n_walks + w) L (1 + 20 win) (n2v.cu, sgns_kernel)."""
    stride = L * (1 + 2 * win * NEG * 2)
    return sum(_walk_pairs(pow(16807, 2 ** 30 + (e * n_walks + w) * stride, M31) * seed % M31, L, win)[0]
               for e in range(iters) for w in range(n_walks))


def test_pair_restatement_matches_a_direct_count():
    """_walk_pairs' closed-form window size against the loop of TrainModel (a from offset to 2 win - offset, a != win)."""
    for L, win, st in [(1, 3, 5), (7, 3, 99), (40, 5, 123456), (9, 10, 777)]:
        s, direct = st, 0
        for pos in range(L):
            s = s * 16807 % M31
            off = s % win
            n = sum(1 for a in range(off, 2 * win + 1 - off) if a != win and 0 <= pos - win + a < L)
            direct += n
            s = s * pow(16807, 10 * n, M31) % M31
        assert _walk_pairs(st, L, win) == (direct, s)


# ---------------------------------------------------------------------------------------------- graphs and oracle walks
def _report(what, err, bar):
    print('\n[widths] %-44s max|X - Xo| / max|Xo| = %.2e  (bar %.0e)' % (what, err, bar))


def _compare(X, Xo, what, bar=2e-3):
    err = float(np.abs(X - Xo).max() / np.abs(Xo).max())
    _report(what, err, bar)
    assert np.isfinite(X).all()
    assert err < bar, err
    assert np.corrcoef(X.ravel(), Xo.ravel())[0, 1] > 0.99999


@pytest.fixture(scope='module')
def seq_graphs(n2v_oracle):
    """name -> (csr, nids, hp, oracle mode-1 walks).  symw60: 60 tokens, so negatives repeat inside a pair's group of five
    and most pairs take the one-by-one path; sbm1024: 1024 tokens, mostly the batched five-row path."""
    z = np.load(golden_path('n2v_bin_symw60.npz'))
    G, _ = load_sbm1024_nx()
    out = {}
    for name, graph, hp in [('symw60', nx_from_npz(z), dict(walk_len=15, num_walks=3, con_size=4, seed=4242)),
                            ('sbm1024', G, dict(walk_len=40, num_walks=2, con_size=5, seed=5))]:
        csr, nids = _inputs(graph)
        Wo = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, nids, hp['walk_len'], hp['num_walks'], seed=hp['seed'],
                              mode=1)
        out[name] = (csr, nids, hp, Wo)
    return out


# ---------------------------------------------------------------------------------------------- SGNS, sequential mode
@pytest.mark.parametrize('graph', ['symw60', 'sbm1024'])
@pytest.mark.parametrize('d', WIDTHS)
def test_sgns_sequential_every_width_follows_oracle(gpu_ctx, n2v_oracle, seq_graphs, d, graph):
    csr, nids, hp, Wo = seq_graphs[graph]
    g = _dev(gpu_ctx, csr)
    X, st = g.node2vec(nids, d, hp['walk_len'], hp['num_walks'], hp['con_size'], 1, seed=hp['seed'], sequential=True,
                       weights64=csr.data)
    g.free()
    Xo, tok = n2v_oracle.learn(Wo, csr.n, d, hp['con_size'], 1, hp['seed'])
    assert st['n_tokens'] == len(tok)
    assert st['pairs'] == _pairs_sequential(hp['seed'], len(tok), d, Wo.shape[0], hp['walk_len'], hp['con_size'], 1)
    _compare(X, Xo, 'sequential %s d=%d' % (graph, d))


@pytest.mark.parametrize('case', ['sbm128_d100', 'sbm128_d128', 'symw60_pq_d256', 'offset40_d128'])
def test_sgns_sequential_wide_goldens_follow_oracle_and_binary(gpu_ctx, n2v_oracle, case):
    """The reference binary's own output at wide d (tests/golden/n2v_bin_*_d*.npz).  sbm128 and symw60 are symmetric (no dead
    ends), so the GPU's walks are the binary's and its embedding must follow the binary's printed one too; offset40 has dead
    ends and an id offset, so its walks pad with the phantom node 0 (compared with the oracle on the GPU's walks)."""
    z = np.load(golden_path('n2v_bin_%s.npz' % case))
    csr, nids = _inputs(nx_from_npz(z))
    hp = {k: z[k].item() for k in ('d', 'walk_len', 'num_walks', 'con_size', 'max_iter', 'seed', 'p', 'q')}
    g = _dev(gpu_ctx, csr)
    X, st = g.node2vec(nids, hp['d'], hp['walk_len'], hp['num_walks'], hp['con_size'], hp['max_iter'], p=hp['p'], q=hp['q'],
                       seed=hp['seed'], sequential=True, weights64=csr.data)
    g.free()
    Wo = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, nids, hp['walk_len'], hp['num_walks'], p=hp['p'], q=hp['q'],
                          seed=hp['seed'], mode=1)
    Xo, tok = n2v_oracle.learn(Wo, csr.n, hp['d'], hp['con_size'], hp['max_iter'], hp['seed'])
    assert st['n_tokens'] == len(tok)
    _compare(X, Xo, 'golden %s (oracle)' % case)
    ids, emb = z['ids'], z['emb'].astype(np.float64)
    if case.startswith('offset40'):
        assert 0 in tok.tolist() and 0 in ids.tolist()
    else:
        err = float(np.abs(X[ids] - emb).max() / np.abs(emb).max())
        _report('golden %s (binary)' % case, err, 2e-3)
        assert err < 2e-3


# ---------------------------------------------------------------------------------------------- SGNS, Hogwild mode
@pytest.mark.parametrize('walk_len', [40, 2000])
@pytest.mark.parametrize('d', [16, 128, 512])
def test_hogwild_one_walk_follows_oracle_per_walk_streams(gpu_ctx, n2v_oracle, d, walk_len):
    """One start node, num_walks = 1: one walk per epoch, trained by one warp from its own stream offset, three epochs.  The short
    walk has a vocabulary of a few dozen tokens (repeated negatives), the long one most of SBM-1024 (the batched path)."""
    G, _ = load_sbm1024_nx()
    csr, nids = _inputs(G)
    start, seed, win, iters = nids[:1].copy(), 21, 5, 3
    g = _dev(gpu_ctx, csr)
    X, st = g.node2vec(start, d, walk_len, 1, win, iters, seed=seed, sequential=False)
    g.free()
    Wo = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, start, walk_len, 1, seed=seed, mode=1)
    Xo, tok = n2v_oracle.learn(Wo, csr.n, d, win, iters, seed, walk_streams=True)
    assert st['n_tokens'] == len(tok)
    assert st['pairs'] == _pairs_hogwild(seed, 1, walk_len, win, iters)
    _compare(X, Xo, 'hogwild one walk L=%d d=%d' % (walk_len, d))


def test_hogwild_pair_count_of_a_full_run(gpu_ctx):
    """All 2048 walks of SBM-1024 on many warps for two epochs: the embedding races, the pair count does not -- it depends on
    every walk's stream offset, epoch and walk-index terms included."""
    G, _ = load_sbm1024_nx()
    csr, nids = _inputs(G)
    walk_len, num_walks, win, iters, seed = 40, 2, 5, 2, 13
    g = _dev(gpu_ctx, csr)
    X, st = g.node2vec(nids, 64, walk_len, num_walks, win, iters, seed=seed, sequential=False)
    g.free()
    assert st['n_tokens'] == 1024 and np.isfinite(X).all()
    assert st['pairs'] == _pairs_hogwild(seed, len(nids) * num_walks, walk_len, win, iters)


# ---------------------------------------------------------------------------------------------- node2vec limits
def test_d_above_512_is_refused_before_any_work(gpu_ctx):
    z = np.load(golden_path('n2v_bin_symw60.npz'))
    csr, nids = _inputs(nx_from_npz(z))
    g = _dev(gpu_ctx, csr)
    try:
        n0 = _launches()
        for sequential in (True, False):
            with pytest.raises(RuntimeError, match=r'd = 513 is not supported \(d <= 512\)'):
                g.node2vec(nids, 513, 10, 1, 3, 1, seed=3, sequential=sequential)
        assert _launches() == n0
    finally:
        g.free()


@pytest.mark.parametrize('sequential', [True, False])
def test_walk_len_at_the_shared_memory_limit(gpu_ctx, n2v_oracle, sequential):
    """Every warp keeps its walk in shared memory: walk_len <= opt-in bytes / (4 warps per block), 1 warp in sequential mode and
    4 in Hogwild mode.  At the limit (above the default 48 KB for both) the kernel runs -- sequential against the oracle,
    Hogwild by its pair count; one more is refused up front, without a launch."""
    z = np.load(golden_path('n2v_bin_symw60.npz'))
    csr, nids = _inputs(nx_from_npz(z))
    warps = 1 if sequential else 4
    L = _smem_optin() // (4 * warps)
    assert 4 * warps * L > 48 * 1024
    start, d, win, seed = nids[:1].copy(), 8, 3, 17
    g = _dev(gpu_ctx, csr)
    try:
        X, st = g.node2vec(start, d, L, 1, win, 1, seed=seed, sequential=sequential, weights64=csr.data)
        Wo = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, start, L, 1, seed=seed, mode=1)
        Xo, tok = n2v_oracle.learn(Wo, csr.n, d, win, 1, seed, walk_streams=not sequential)
        assert st['n_tokens'] == len(tok)
        if sequential:
            assert st['pairs'] == _pairs_sequential(seed, len(tok), d, 1, L, win, 1)
            _compare(X, Xo, 'sequential walk_len=%d' % L)
        else:
            assert st['pairs'] == _pairs_hogwild(seed, 1, L, win, 1)
        n0 = _launches()
        mode = 'sequential' if sequential else 'Hogwild'
        with pytest.raises(RuntimeError, match=r'walk_len = %d is not supported in %s mode \(walk_len <= %d' % (L + 1, mode, L)):
            g.node2vec(start, d, L + 1, 1, win, 1, seed=seed, sequential=sequential, weights64=csr.data)
        assert _launches() == n0
    finally:
        g.free()


# ---------------------------------------------------------------------------------------------- Graph Factorization
def _gf_case(d):
    """randw60 (edges grouped by ascending source, so both schedules apply) with a seeded start of width d."""
    z = np.load(golden_path('ref_gf_randw60_d8_it60.npz'))
    e = z['edges']
    n = int(z['n'])
    X0 = (0.01 * np.random.RandomState(9).randn(n, d)).astype(np.float32)
    kw = dict(eta=float(z['eta']), regu=float(z['regu']), max_iter=int(z['max_iter']))
    return n, e[:, 0].astype(np.int32), e[:, 1].astype(np.int32), e[:, 2].astype(np.float32), X0, kw


@pytest.mark.parametrize('d', GF_WIDTHS)
def test_gf_every_width_both_schedules_follow_oracle(gpu_ctx, d):
    import gf_oracle as go
    from gem_b200 import _native
    n, src, dst, w, X0, kw = _gf_case(d)
    X0s, _ = _native.graph_factorization(gpu_ctx, n, src, dst, w, d=d, X0=X0, mode=0, **kw)
    X1s, _ = _native.graph_factorization(gpu_ctx, n, src, dst, w, d=d, X0=X0, mode=1, **kw)
    assert np.array_equal(X0s, X1s)                  # the same arithmetic in the same order (tests/test_gpu_gf.py)
    Xo = go.gf_sequential(n, src, dst, w, d, kw['eta'], kw['regu'], kw['max_iter'], X0)
    err = float(np.abs(X0s - Xo).max() / np.abs(Xo).max())
    _report('gf d=%d' % d, err, 2e-4)
    assert err < 2e-4, err
    assert np.abs(Xo - X0).max() > 0.1 * np.abs(X0).max()  # the sweep did move the start


def test_gf_d_above_1024_is_refused_before_any_work(gpu_ctx):
    from gem_b200 import _native
    n, src, dst, w, X0, kw = _gf_case(1025)
    n0 = _launches()
    for mode in (0, 1):
        with pytest.raises(RuntimeError, match=r'd must be in 1\.\.1024'):
            _native.graph_factorization(gpu_ctx, n, src, dst, w, d=1025, X0=X0, mode=mode, **kw)
    assert _launches() == n0
