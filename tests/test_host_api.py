"""Host-side mirror of the reference plugin API (reference tests/test_embedding_classes.py:37-48 style)
and of the graph ingestion.  CPU only."""
import numpy as np
import pytest

from conftest import load_karate_nx


def test_embedding_class_contract():
    # reference tests/test_embedding_classes.py:37-48
    from gem_b200.embedding.hope import HOPE
    from gem_b200.embedding.node2vec import node2vec
    for cls, name in ((HOPE, 'hope_gsvd'), (node2vec, 'node2vec_rw')):
        model = cls()
        with pytest.raises(ValueError, match='graph needed'):
            model.learn_embedding()
        assert model.hyper_params['method_name'] == model.get_method_name() == name
        with pytest.raises(ValueError, match='Embedding not learned yet'):
            model.get_embedding()
    import networkx as nx
    with pytest.raises(ValueError, match='graph needed'):
        HOPE(d=4, beta=0.01).learn_embedding(graph=nx.DiGraph())      # empty graph is falsy (hope.py:25)
    m = HOPE(d=4, beta=0.01)
    assert m.get_method_summary() == 'hope_gsvd_4'
    m2 = node2vec(d=2, max_iter=1, walk_len=80, num_walks=10, con_size=10, ret_p=1, inout_p=1, data_set='sbm')
    assert m2._walk_len == 80 and m2._data_set == 'sbm' and m2.get_method_summary() == 'node2vec_rw_2'


def test_hyper_params_class_dict_semantics():
    # SURVEY F13: kwargs update the CLASS dict, later instances inherit them (kept on purpose)
    from gem_b200.embedding.hope import HOPE
    saved = dict(HOPE.hyper_params)
    try:
        HOPE(d=6, beta=0.5)
        assert HOPE()._d == 6
    finally:
        HOPE.hyper_params.clear()
        HOPE.hyper_params.update(saved)


def test_reconstructed_adj_has_no_cpu_path():
    """get_reconstructed_adj runs on the GPU (tests/test_gpu_recon.py); here: it keeps the reference's side effect
    (self._X = X, static_graph_embedding.py:56) and fails loudly without a device instead of falling back."""
    from gem_b200 import _native
    from gem_b200.embedding.hope import HOPE
    if _native.lib().gemb_device_count() > 0:
        pytest.skip('a GPU is visible')
    X = np.random.default_rng(0).standard_normal((7, 6))
    m = HOPE(d=6, beta=0.1)
    with pytest.raises(RuntimeError, match='no CUDA device|CUDA'):
        m.get_reconstructed_adj(X=X)
    assert m.get_embedding() is X


def test_csr_from_networkx_matches_to_numpy_array():
    import networkx as nx
    from gem_b200 import graph as hg
    G = load_karate_nx()
    csr = hg.from_networkx(G)
    dense = nx.to_numpy_array(G, nodelist=list(G.nodes))
    assert np.array_equal(csr.to_scipy().toarray(), dense)
    assert csr.nodes == list(G.nodes) and csr.data is None     # unit weights are dropped
    assert not csr.is_symmetric()
    t = csr.transpose()
    assert np.array_equal(t.to_scipy().toarray(), dense.T)
    H = nx.DiGraph()
    H.add_weighted_edges_from([(0, 1, 0.5), (1, 0, 0.5), (1, 2, 2.0), (2, 1, 2.0)])
    c2 = hg.from_networkx(H)
    assert c2.is_symmetric() and c2.data is not None


def test_n2v_inputs_order_and_weights():
    import networkx as nx
    from gem_b200 import graph as hg
    G = nx.DiGraph()
    G.add_weighted_edges_from([(5, 2, 0.1234567), (2, 7, 1.0), (5, 7, 3.0)])
    csr, nids = hg.n2v_inputs_from_networkx(G)
    assert nids.tolist() == [5, 2, 7]                           # first appearance in the edge list
    assert csr.n == 8 and csr.indices[csr.indptr[5]:csr.indptr[6]].tolist() == [2, 7]
    assert csr.data[csr.indptr[5]] == float('%f' % 0.1234567)   # graph_util.py:140 writes %f
    sh = csr.row_shard(1, 2)
    assert sh[0] == 4 and sh[1][0] == 0


def test_wire_formats_roundtrip(tmp_path):
    from gem_b200.utils import graph_util
    G = load_karate_nx()
    f = str(tmp_path / 'g.txt')
    graph_util.saveGraphToEdgeListTxtn2v(G, f)
    lines = open(f).read().splitlines()
    assert lines[0] == '0 31 1.000000' and len(lines) == G.number_of_edges()
    G2 = graph_util.loadGraphFromEdgeListTxt(f, directed=True)
    assert sorted(G2.edges()) == sorted(G.edges())
    X = np.arange(12, dtype=np.float64).reshape(4, 3) / 7
    e = str(tmp_path / 'x.emb')
    graph_util.saveEmbedding(X, e, ids=[2, 0, 3, 1])
    assert np.allclose(graph_util.loadEmbedding(e), X, rtol=1e-5)


def test_from_networkx_fast_and_fallback_paths_match_to_numpy_array():
    """Integer-labelled graphs take the vectorised adjacency walk, everything else the per-edge loop; both must equal
    nx.to_numpy_array(graph, nodelist=list(graph.nodes)) (= the reference's nx.to_numpy_matrix, hope.py:28),
    including undirected graphs (both directions), self loops, missing weights and shifted / unordered labels."""
    import networkx as nx
    from gem_b200 import graph as hg
    rng = np.random.default_rng(0)

    def check(G, by_label=False):
        c = hg.from_networkx(G, by_label=by_label)
        if by_label:
            n = max(G.nodes) + 1
            dense = np.zeros((n, n))
            for u, v, w in G.edges(data='weight', default=1):
                dense[u, v] = w
                if not G.is_directed():
                    dense[v, u] = w
        else:
            dense = nx.to_numpy_array(G, nodelist=list(G.nodes))
            assert c.nodes == list(G.nodes)
        assert np.array_equal(c.to_scipy().toarray(), dense)

    G = nx.DiGraph()
    for _ in range(500):
        u, v = (int(x) for x in rng.integers(0, 60, 2))
        G.add_edge(u * 3 + 5, v * 3 + 5, weight=float(rng.uniform(0.1, 2)))
    G.add_edge(7, 8)                                          # no weight attribute -> 1
    check(G); check(G, True)
    H = nx.Graph()
    for _ in range(300):
        u, v = (int(x) for x in rng.integers(0, 50, 2))
        H.add_edge(u, v, weight=float(rng.integers(1, 4)))
    H.add_edge(3, 3)
    check(H); check(H, True)
    S = nx.DiGraph(); S.add_edge('a', 'b', weight=2.0); S.add_edge('b', 'c')
    check(S)
    U = nx.Graph(); U.add_edge('x', 'y'); U.add_edge('y', 'y')
    check(U)
    E = nx.DiGraph(); E.add_nodes_from([0, 1, 2])
    check(E)


def test_synthetic_generators_match_the_survey_configs():
    """SURVEY 8(d): SBM with ~16 intra + ~4 inter neighbours per node, symmetric, no loops, deterministic in the seed;
    Graph500 R-MAT symmetrised, deduplicated, hubs and isolated nodes, vertex labels permuted so that contiguous
    equal-row shards carry similar numbers of edges."""
    from gem_b200 import synth
    a = synth.sbm(n=20_000, block=1000, seed=42)
    b = synth.sbm(n=20_000, block=1000, seed=42)
    assert np.array_equal(a.indptr, b.indptr) and np.array_equal(a.indices, b.indices) and a.data is None
    assert a.is_symmetric() and abs(a.nnz / a.n - 20.0) < 0.3
    rows = np.repeat(np.arange(a.n), np.diff(a.indptr))
    assert not np.any(rows == a.indices)                                     # no self loops
    intra = (rows // 1000) == (a.indices // 1000)
    assert abs(intra.mean() - 0.8) < 0.02                                    # 16 of 20 neighbours inside the block
    t = a.transpose()
    assert np.array_equal(t.indptr, a.indptr) and np.array_equal(t.indices, a.indices)
    r = synth.rmat(scale=13, edge_factor=8, seed=42)
    assert r.n == 8192 and r.is_symmetric() and r.nnz <= 2 * 8 * 8192
    deg = np.diff(r.indptr)
    assert deg.max() > 100 * max(1.0, np.median(deg)) and (deg == 0).sum() > 0.2 * r.n
    per = r.n // 8
    shard_nnz = np.array([r.indptr[(p + 1) * per] - r.indptr[p * per] for p in range(8)])
    assert shard_nnz.max() < 1.6 * shard_nnz.mean()                          # permuted labels: balanced shards
    u = synth.rmat(scale=13, edge_factor=8, seed=42, permute=False)
    per_u = np.array([u.indptr[(p + 1) * per] - u.indptr[p * per] for p in range(8)])
    assert per_u.max() > 2.0 * per_u.mean()                                  # without it rank 0 owns the hubs
    assert np.array_equal(np.sort(np.diff(u.indptr)), np.sort(deg))          # same graph up to relabelling


def test_scipy_inputs_get_past_the_empty_graph_guard():
    """ADVICE r1: scipy sparse matrices AND arrays raise TypeError from len(); the guard must look at .shape first."""
    import scipy.sparse as sp
    from gem_b200.embedding.hope import HOPE
    from gem_b200.embedding.static_graph_embedding import _graph_is_empty
    from gem_b200.graph import HostCSR
    A = sp.random(12, 12, 0.3, format='csr', random_state=0)
    for M in (A, sp.csr_array(A), sp.coo_matrix(A)):
        assert not _graph_is_empty(M)
        csr = HOPE(d=4, beta=0.01)._to_csr(M)
        assert isinstance(csr, HostCSR) and csr.n == 12 and csr.nnz == A.nnz
    assert _graph_is_empty(sp.csr_matrix((0, 0))) and _graph_is_empty(None)
    import networkx as nx
    assert _graph_is_empty(nx.DiGraph()) and not _graph_is_empty(nx.path_graph(3))
    with pytest.raises(ValueError, match='graph needed'):
        HOPE(d=4, beta=0.01).learn_embedding(graph=sp.csr_matrix((0, 0)))


def test_multigraph_parallel_edges_are_summed_like_to_numpy_matrix():
    import networkx as nx
    from gem_b200 import graph as hg
    M = nx.MultiDiGraph()
    M.add_edge(0, 1, weight=2.0); M.add_edge(0, 1, weight=3.0); M.add_edge(1, 2); M.add_edge(1, 2); M.add_edge(2, 0)
    assert np.array_equal(hg.from_networkx(M).to_scipy().toarray(), nx.to_numpy_array(M))


def test_device_graph_refuses_offsets_beyond_int32():
    from gem_b200 import _native

    class FakeCtx:
        _h = None
    ip = np.array([0, 2 ** 31], dtype=np.int64)
    with pytest.raises(ValueError, match='int32 offsets'):
        _native.DeviceGraph(FakeCtx(), 1, ip, np.zeros(1, np.int32))


def test_bench_reference_arm_contract(tmp_path):
    """`bench.py --impl reference` (the CPU arm the driver runs first): one JSON line with the contract's keys, on a tiny sample."""
    import json
    import os
    import subprocess
    import sys
    from conftest import REPO
    env = dict(os.environ, OMP_NUM_THREADS='2')
    p = subprocess.run([sys.executable, os.path.join(REPO, 'bench.py'), '--impl', 'reference', '--cpu-sample', '3000', '--steps', '1',
                        '--warmup', '0'], capture_output=True, text=True, timeout=600, env=env, cwd=str(tmp_path))
    assert p.returncode == 0, p.stderr[-2000:]
    line = json.loads([l for l in p.stdout.splitlines() if l.startswith('{')][-1])
    assert line['impl'] == 'reference' and line['metric'].startswith('nodes/sec embedded') and line['unit'] == 'nodes/s'
    assert line['value'] > 0 and line['higher_is_better'] is True and line['n_gpus'] == 1
    assert line['cpu_baseline']['kind'] == 'port' and line['cpu_baseline']['cores'] >= 1
    assert line['e2e']['value'] == line['value'] and line['e2e']['h2d_bytes_per_step'] == 0
    # under torchrun every rank but 0 prints nothing and exits 0
    p1 = subprocess.run([sys.executable, os.path.join(REPO, 'bench.py'), '--impl', 'reference', '--cpu-sample', '3000'],
                        capture_output=True, text=True, timeout=60, env=dict(env, RANK='1', WORLD_SIZE='2'), cwd=str(tmp_path))
    assert p1.returncode == 0 and p1.stdout.strip() == ''
