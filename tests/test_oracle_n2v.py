"""Pins oracle/n2v_oracle.c against the UNMODIFIED reference binary gem/c_exe/node2vec: the goldens in
tests/golden/n2v_bin_*.npz were produced by that binary with time() interposed (seed = N2V_FAKE_TIME)
and OMP_NUM_THREADS=1 (tests/golden/make_golden.py).  The oracle must reproduce every embedding to the
6 significant digits the binary prints -- which it can only do if its alias tables, shuffles, walks,
vocabulary, negative sampler and SGD updates are all identical.  CPU only."""
import glob
import os

import numpy as np
import pytest

from conftest import golden_path, load_karate_nx, nx_from_npz

CASES = sorted(os.path.basename(p)[8:-4] for p in glob.glob(golden_path('n2v_bin_*.npz')))


def oracle_inputs(G):
    from gem_b200 import graph as hg
    csr, nids = hg.n2v_inputs_from_networkx(G)
    return csr, nids


@pytest.mark.parametrize('name', CASES)
def test_oracle_reproduces_reference_binary(n2v_oracle, name):
    z = np.load(golden_path('n2v_bin_%s.npz' % name))
    G = nx_from_npz(z)
    csr, nids = oracle_inputs(G)
    hp = {k: z[k].item() for k in ('d', 'walk_len', 'num_walks', 'con_size', 'max_iter', 'p', 'q', 'seed')}
    X, tok, wm = n2v_oracle.node2vec(csr.indptr, csr.indices, csr.data, nids, hp['d'], hp['walk_len'],
                                     hp['num_walks'], hp['con_size'], hp['max_iter'], hp['p'], hp['q'],
                                     hp['seed'], mode=0)
    ids, emb = z['ids'], z['emb']
    assert sorted(ids.tolist()) == sorted(tok.tolist())        # same vocabulary (incl. phantom 0, SURVEY F10)
    rel = np.abs(X[ids] - emb) / (np.abs(emb) + 1e-12)
    assert rel.max() < 6e-6, rel.max()                          # printing precision of the binary


def test_strided_mode_equals_sequential_without_dead_ends(n2v_oracle):
    z = np.load(golden_path('n2v_bin_symw60.npz'))              # symmetric: no dead ends
    csr, nids = oracle_inputs(nx_from_npz(z))
    a = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, nids, 15, 3, seed=4242, mode=0)
    b = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, nids, 15, 3, seed=4242, mode=1)
    assert np.array_equal(a, b)
    # with dead ends (directed Karate) the two modes must differ only AFTER the first early stop
    csr, nids = oracle_inputs(load_karate_nx())
    a = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, nids, 10, 2, seed=7, mode=0)
    b = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, nids, 10, 2, seed=7, mode=1)
    assert a.shape == b.shape and not np.array_equal(a, b)
    assert np.array_equal(a[0], b[0])


def test_rng_skip_matches_stepping(n2v_oracle):
    s = 12345
    for k in (0, 1, 2, 1000, 123457):
        x = s
        for _ in range(min(k, 2000)):
            x = (16807 * x) % 2147483647
        if k <= 2000:
            assert n2v_oracle.rng_skip(s, k) == x
    assert n2v_oracle.rng_skip(s, 123457) == pow(16807, 123457, 2147483647) * s % 2147483647


def test_walk_edge_cases(n2v_oracle):
    # chain 5->6->7->8: dead end pads with 0 and creates the phantom token 0 (SURVEY F10)
    import networkx as nx
    G = nx.DiGraph([(5, 6), (6, 7), (7, 8)])
    csr, nids = oracle_inputs(G)
    assert nids.tolist() == [5, 6, 7, 8]
    wm = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, nids, 6, 1, seed=3, mode=1)
    for row in wm:
        nz = row[row != 0]
        assert np.all(np.diff(nz) == 1) and nz[-1] == 8 and np.all(row[len(nz):] == 0)
    X, tok = n2v_oracle.learn(wm, 9, 4, 2, 1, 3)
    assert sorted(tok.tolist()) == [0, 5, 6, 7, 8]
    # walk_len = 1
    wm1 = n2v_oracle.walks(csr.indptr, csr.indices, csr.data, nids, 1, 2, seed=3, mode=1)
    assert wm1.shape == (8, 1) and sorted(wm1[:4, 0].tolist()) == [5, 6, 7, 8]


def _learn_restated(walks, d, win, iters, seed, walk_streams):
    """TrainModel statement by statement in plain Python fp64 (the C file's order, no FMA): the check of the oracle's
    stream layouts.  walk_streams: walk wi of epoch it starts at 2^30 + (it*n_walks + wi) * L * (1 + 20*win)."""
    import math
    M = 2147483647
    tok, rows = {}, []
    for row in walks:
        rows.append([tok.setdefault(int(x), len(tok)) for x in row])
    V, L = len(tok), len(rows[0])
    vocab = [0] * V
    for row in rows:
        for t in row:
            vocab[t] += 1
    st = [seed]

    def uni():
        st[0] = st[0] * 16807 % M
        return st[0] / 2147483647.0
    sp = [[(uni() - 0.5) / d for _ in range(d)] for _ in range(V)]
    sn = [[0.0] * d for _ in range(V)]
    prob = [math.exp(math.log(c) * 0.75) for c in vocab]
    tw = 0.0
    for x in prob:
        tw += x
    U = [x / tw * V for x in prob]
    K = [0] * V
    under = [i for i in range(V) if U[i] < 1]
    over = [i for i in range(V) if U[i] >= 1]
    while under and over:
        small, large = under.pop(), over.pop()
        K[small] = large
        U[large] = U[large] + U[small] - 1
        (under if U[large] < 1 else over).append(large)
    for i in under + over:
        U[i] = 1.0
    alpha, word_cnt, tot = 0.025, 0, len(rows) * L
    for it in range(iters):
        for wi, wk in enumerate(rows):
            if walk_streams:
                st[0] = pow(16807, 2 ** 30 + (it * len(rows) + wi) * L * (1 + 20 * win), M) * seed % M
            for pos in range(L):
                if word_cnt % 10000 == 0:
                    alpha = max(0.025 * (1 - word_cnt / float(iters * tot + 1)), 0.025 * 0.0001)
                word = wk[pos]
                uni()
                offset = st[0] % win
                for a in range(offset, 2 * win + 1 - offset):
                    c = pos - win + a
                    if a == win or c < 0 or c >= L:
                        continue
                    p, neu = sp[wk[c]], [0.0] * d
                    for j in range(6):
                        if j == 0:
                            target, label = word, 1
                        else:
                            X = K[int(uni() * V)]
                            target = X if uni() < U[X] else K[X]
                            if target == word:
                                continue
                            label = 0
                        q = sn[target]
                        f = 0.0
                        for i in range(d):
                            f += p[i] * q[i]
                        if f > 6:
                            g = (label - 1) * alpha
                        elif f < -6:
                            g = label * alpha
                        else:
                            e = math.exp(math.log(2.718281828459045) * (-6.0 + (int(f * 10000) + 60000) / 10000.0))
                            g = (label - 1 + 1 / (1 + e)) * alpha
                        for i in range(d):
                            neu[i] += g * q[i]
                            q[i] += g * p[i]
                    for i in range(d):
                        p[i] += neu[i]
                word_cnt += 1
    return np.array(sp), [node for node, _ in sorted(tok.items(), key=lambda kv: kv[1])]


@pytest.mark.parametrize('walk_streams', [False, True])
def test_learn_stream_layouts_against_plain_restatement(n2v_oracle, walk_streams):
    """Both stream layouts of the oracle's word2vec phase: the binary's single stream, and the per-walk streams the GPU's
    Hogwild mode draws from (tests/test_gpu_n2v_widths.py compares the GPU with the latter).  Small vocabulary, so
    negatives hit the centre word and get skipped; two epochs, so the epoch term of the stream offset is exercised."""
    rng = np.random.default_rng(8)
    walks = rng.integers(3, 12, size=(3, 9)).astype(np.int32)
    X, tok = n2v_oracle.learn(walks, 12, 5, 3, 2, 777, walk_streams=walk_streams)
    Xr, tok_r = _learn_restated(walks, 5, 3, 2, 777, walk_streams)
    assert tok.tolist() == tok_r
    assert np.allclose(X[tok], Xr, rtol=1e-12, atol=1e-15)
    other, _ = n2v_oracle.learn(walks, 12, 5, 3, 2, 777, walk_streams=not walk_streams)
    assert not np.allclose(X, other)                             # the two layouts really are different streams
