"""tests/golden/make_golden.py -- regenerates the committed fixtures in tests/golden/.

Runs ONLY in the build container (needs /root/reference, which does not exist on the GPU box).
Nothing in tests/, bench.py or __graft_entry__.py imports this file; they read the .npz/.txt
fixtures it wrote.

What it writes
  karate.edgelist, karate_HOPE.txt, karate_node2vec.txt
        the reference's own test fixture + goldens   (/root/reference/tests/data, tests/karate_res)
  sbm1024.npz
        the reference's SBM fixture (tests/data/sbm.gpickle, a networkx-1.x pickle) rebuilt the way
        tests/test_sbm.py:33-40 does it: node order, directed edge list (weights dropped), labels;
        plus the reference goldens tests/smb_res/HOPE.txt (fp64) and node2vec.txt (fp32)
  ref_hope_*.npz
        outputs of the UNMODIFIED reference class gem.embedding.hope.HOPE (imported from
        /root/reference with the harness-side networkx shim, SURVEY F4/C.2) on karate, sbm1024 and
        two extra graphs (weighted directed random; symmetric ring-of-cliques)
  n2v_bin_*.npz
        outputs of the UNMODIFIED reference binary gem/c_exe/node2vec, made deterministic with
        oracle/_ref/libfaketime_shim.so (N2V_FAKE_TIME = seed) and OMP_NUM_THREADS=1, on several
        graphs (karate directed with dead ends; weighted symmetric; second-order p,q; id offset
        -> phantom node 0).  tests/test_oracle_n2v.py requires oracle/n2v_oracle.c to reproduce
        them to the 6 significant digits the binary prints.  The `*_d<d>` cases repeat a graph at a
        wide embedding (d = 100 ... 256: the multi-value-per-lane SGNS kernels); they store the
        printed embedding as float32, which holds its 6 digits, to keep the fixtures small.

`python make_golden.py NAME ...` rewrites only the named fixtures (file names without .npz), so
that adding a case leaves the bytes of the others alone.
"""
import os
import pickle
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get('GEM_REFERENCE', '/root/reference')
sys.dont_write_bytecode = True


def load_karate_nx():
    import networkx as nx
    G = nx.DiGraph()
    with open(os.path.join(REF, 'tests/data/karate.edgelist')) as f:
        for line in f:
            e = line.split()
            G.add_edge(int(e[0]), int(e[1]), weight=float(e[2]) if len(e) == 3 else 1.0)
    return G


def load_sbm_nx():
    """tests/test_sbm.py:33-40 with plain pickle (nx.read_gpickle is gone in networkx 3)."""
    import networkx as nx
    with open(os.path.join(REF, 'tests/data/sbm.gpickle'), 'rb') as f:
        G = pickle.load(f, encoding='latin1')
    H = nx.DiGraph()
    H.add_nodes_from(G.node)
    for s in G.edge.keys():
        for t in G.edge[s].keys():
            H.add_edge(s, t)
    return H


def ref_hope(G, d, beta):
    """The reference class itself (hope.py:8-44), with the harness-side shim for networkx 3."""
    import networkx as nx
    if not hasattr(nx, 'to_numpy_matrix'):
        nx.to_numpy_matrix = lambda g, **k: np.asmatrix(nx.to_numpy_array(g, **k))
    sys.path.insert(0, REF)
    try:
        from gem.embedding.hope import HOPE
    finally:
        sys.path.remove(REF)
    HOPE.hyper_params = {'method_name': 'hope_gsvd'}   # undo class-dict leakage (SURVEY F13)
    m = HOPE(d=d, beta=beta)
    X = np.asarray(m.learn_embedding(graph=G, is_weighted=True, no_python=True))
    return X


def edges_of(G):
    """(nodes in list(G.nodes) order, edges in G.edges(data='weight', default=1) order):
    the order graph_util.saveGraphToEdgeListTxtn2v writes them (graph_util.py:137-140)."""
    nodes = np.array(list(G.nodes), dtype=np.int64)
    e = [(int(i), int(j), float(w)) for i, j, w in G.edges(data='weight', default=1)]
    src = np.array([x[0] for x in e], dtype=np.int64)
    dst = np.array([x[1] for x in e], dtype=np.int64)
    w = np.array([x[2] for x in e], dtype=np.float64)
    return nodes, src, dst, w


def run_n2v_binary(src, dst, w, d, walk_len, num_walks, con_size, max_iter, p, q, seed):
    exe = os.path.join(REPO, 'oracle/_ref/node2vec')
    shim = os.path.join(REPO, 'oracle/_ref/libfaketime_shim.so')
    with tempfile.TemporaryDirectory() as td:
        with open(os.path.join(td, 'g.graph'), 'w') as f:
            for i, j, ww in zip(src, dst, w):
                f.write('%d %d %f\n' % (i, j, ww))          # graph_util.py:137-140
        env = dict(os.environ, N2V_FAKE_TIME=str(seed), OMP_NUM_THREADS='1', LD_PRELOAD=shim)
        args = [exe, '-i:g.graph', '-o:g.emb', '-d:%d' % d, '-l:%d' % walk_len, '-r:%d' % num_walks,
                '-k:%d' % con_size, '-e:%d' % max_iter, '-p:%f' % p, '-q:%f' % q, '-v', '-dr', '-w']
        subprocess.check_call(args, cwd=td, env=env, stdout=subprocess.DEVNULL)   # node2vec.py:35-48
        ids, rows = [], []
        with open(os.path.join(td, 'g.emb')) as f:
            V, dd = map(int, f.readline().split())
            for line in f:
                t = line.split()
                ids.append(int(t[0]))
                rows.append([float(x) for x in t[1:]])
    return np.array(ids, dtype=np.int64), np.array(rows, dtype=np.float64)


def rand_graph(rng, n, m, sym, weighted, offset=0):
    import networkx as nx
    G = nx.DiGraph()
    while G.number_of_edges() < m:
        u, v = (int(x) for x in rng.integers(0, n, 2))
        if u == v:
            continue
        wt = float(np.round(rng.uniform(0.1, 3.0), 6)) if weighted else 1.0
        G.add_edge(u + offset, v + offset, weight=wt)
        if sym:
            G.add_edge(v + offset, u + offset, weight=wt)
    return G


def main(only=()):
    import networkx as nx
    want = lambda name: not only or name in only
    subprocess.check_call(['make', '-C', os.path.join(REPO, 'oracle'), 'all', 'ref'])
    for a, b in [('tests/data/karate.edgelist', 'karate.edgelist'),
                 ('tests/karate_res/HOPE.txt', 'karate_HOPE.txt'),
                 ('tests/karate_res/node2vec.txt', 'karate_node2vec.txt')]:
        if want(b.rsplit('.', 1)[0]):
            shutil.copyfile(os.path.join(REF, a), os.path.join(HERE, b))

    # --- SBM-1024 fixture + reference goldens
    Gs = load_sbm_nx()
    nodes, src, dst, w = edges_of(Gs)
    with open(os.path.join(REF, 'tests/data/sbm_node_labels.pickle'), 'rb') as f:
        lab = pickle.load(f, encoding='latin1')
    labels = np.asarray(lab.argmax(axis=1)).ravel().astype(np.int16)
    hope_gold = np.loadtxt(os.path.join(REF, 'tests/smb_res/HOPE.txt'))
    n2v_gold = np.loadtxt(os.path.join(REF, 'tests/smb_res/node2vec.txt')).astype(np.float32)
    if want('sbm1024'):
        np.savez_compressed(os.path.join(HERE, 'sbm1024.npz'), nodes=nodes.astype(np.int32),
                            src=src.astype(np.int32), dst=dst.astype(np.int32), labels=labels,
                            hope_golden=hope_gold, node2vec_golden=n2v_gold)

    # --- reference HOPE class outputs
    rng = np.random.default_rng(2024)
    Gk = load_karate_nx()
    Gw = rand_graph(rng, 200, 1500, sym=False, weighted=True)
    Gc = nx.DiGraph(nx.ring_of_cliques(12, 9))           # symmetric, well separated spectrum
    cases = {'karate_d4': (Gk, 4, 0.01), 'karate_d16': (Gk, 16, 0.05), 'sbm1024_d256': (Gs, 256, 0.01),
             'sbm1024_d16': (Gs, 16, 0.01), 'randw200_d32': (Gw, 32, 0.02), 'cliques_d24': (Gc, 24, 0.05)}
    for name, (G, d, beta) in cases.items():
        if not want('ref_hope_' + name):
            continue
        X = ref_hope(G, d, beta)
        nd, s, t, ww = edges_of(G)
        np.savez_compressed(os.path.join(HERE, 'ref_hope_%s.npz' % name), nodes=nd.astype(np.int32),
                            src=s.astype(np.int32), dst=t.astype(np.int32), w=ww, d=d, beta=beta, X=X)
        print('ref_hope', name, X.shape)

    # --- reference node2vec binary outputs (deterministic via time shim)
    Gsym = rand_graph(rng, 60, 300, sym=True, weighted=True)
    Gdir = rand_graph(rng, 50, 200, sym=False, weighted=True)
    Goff = rand_graph(rng, 40, 100, sym=False, weighted=False, offset=3)
    Gsb = nx.DiGraph()
    Gsb.add_edges_from((int(a), int(b)) for a, b in zip(src[:], dst[:]) if a < 128 and b < 128)
    n2v_cases = {
        'karate_a': (Gk, dict(d=2, walk_len=80, num_walks=10, con_size=10, max_iter=1, p=1.0, q=1.0, seed=1234)),
        'karate_b': (Gk, dict(d=8, walk_len=20, num_walks=3, con_size=5, max_iter=2, p=1.0, q=1.0, seed=99)),
        'symw60': (Gsym, dict(d=6, walk_len=15, num_walks=3, con_size=4, max_iter=1, p=1.0, q=1.0, seed=4242)),
        'symw60_pq': (Gsym, dict(d=6, walk_len=15, num_walks=3, con_size=4, max_iter=1, p=0.5, q=2.0, seed=4242)),
        'dirw50_pq': (Gdir, dict(d=6, walk_len=15, num_walks=3, con_size=4, max_iter=1, p=4.0, q=0.25, seed=7)),
        'offset40': (Goff, dict(d=6, walk_len=15, num_walks=3, con_size=4, max_iter=1, p=1.0, q=1.0, seed=31337)),
        'sbm128': (Gsb, dict(d=16, walk_len=40, num_walks=4, con_size=5, max_iter=1, p=1.0, q=1.0, seed=5)),
        # wide d: scalar layout with a partial last value (100), float4 layouts (128, 256)
        'sbm128_d100': (Gsb, dict(d=100, walk_len=40, num_walks=4, con_size=5, max_iter=1, p=1.0, q=1.0, seed=5)),
        'sbm128_d128': (Gsb, dict(d=128, walk_len=40, num_walks=4, con_size=5, max_iter=1, p=1.0, q=1.0, seed=5)),
        'symw60_pq_d256': (Gsym, dict(d=256, walk_len=15, num_walks=3, con_size=4, max_iter=1, p=0.5, q=2.0, seed=4242)),
        'offset40_d128': (Goff, dict(d=128, walk_len=15, num_walks=3, con_size=4, max_iter=1, p=1.0, q=1.0, seed=31337)),
    }
    for name, (G, hp) in n2v_cases.items():
        if not want('n2v_bin_' + name):
            continue
        nd, s, t, ww = edges_of(G)
        ids, emb = run_n2v_binary(s, t, ww, **hp)
        if hp['d'] >= 100:
            emb = emb.astype(np.float32)
        np.savez_compressed(os.path.join(HERE, 'n2v_bin_%s.npz' % name), nodes=nd.astype(np.int32),
                            src=s.astype(np.int32), dst=t.astype(np.int32), w=ww, ids=ids, emb=emb,
                            **{k: np.array(v) for k, v in hp.items()})
        print('n2v_bin', name, emb.shape)


if __name__ == '__main__':
    main(set(sys.argv[1:]))
