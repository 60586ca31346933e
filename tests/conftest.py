import os
import subprocess
import sys

# BLAS / OpenMP pools of 64+ threads per process (and two such processes in the gloo tests) thrash on a shared or
# CPU-limited box: the CPU suite went from 30 s to 5 minutes under load.  Nothing here needs more than a few threads.
for _v in ('OMP_NUM_THREADS', 'OPENBLAS_NUM_THREADS', 'MKL_NUM_THREADS'):
    os.environ.setdefault(_v, '4')

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)
GOLDEN = os.path.join(REPO, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100; select with -m gpu)')


@pytest.fixture(scope='session')
def native_lib():
    """libgemb200.so, built in-tree if missing (nvcc cross-compiles without a GPU)."""
    from gem_b200 import _native, build
    if not os.path.exists(_native.LIB_PATH):
        build.build()
    return _native.lib()


@pytest.fixture(scope='session')
def n2v_oracle():
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import n2v_oracle_py
    return n2v_oracle_py


@pytest.fixture(scope='session')
def hope_oracle():
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import hope_oracle as ho
    return ho


@pytest.fixture(scope='session')
def eval_oracle():
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import eval_oracle as eo
    return eo


def eval_golden(name):
    """One eval_*.npz golden -> (z, n, CSR (indptr, indices, weights) of the true graph in id order)."""
    z = np.load(golden_path(name + '.npz'))
    n = int(z['n'])
    e = z['edges']
    src, dst, w = e[:, 0].astype(np.int64), e[:, 1].astype(np.int64), e[:, 2]
    order = np.lexsort((dst, src))
    src, dst, w = src[order], dst[order], w[order]
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, src + 1, 1)
    return z, n, (np.cumsum(indptr), dst, w)


def golden_path(name):
    return os.path.join(GOLDEN, name)


def load_karate_nx():
    """The reference's Karate fixture exactly as tests/test_karate.py:31-35 loads it (directed)."""
    import networkx as nx
    G = nx.DiGraph()
    with open(golden_path('karate.edgelist')) as f:
        for line in f:
            e = line.split()
            G.add_edge(int(e[0]), int(e[1]), weight=float(e[2]) if len(e) == 3 else 1.0)
    return G


def load_sbm1024_nx():
    """The reference's SBM fixture rebuilt as tests/test_sbm.py:33-40 (weights dropped)."""
    import networkx as nx
    z = np.load(golden_path('sbm1024.npz'))
    H = nx.DiGraph()
    H.add_nodes_from(int(x) for x in z['nodes'])
    H.add_edges_from(zip(z['src'].tolist(), z['dst'].tolist()))
    return H, z


def nx_from_npz(z):
    import networkx as nx
    G = nx.DiGraph()
    G.add_nodes_from(int(x) for x in z['nodes'])
    if 'w' in z.files:
        G.add_weighted_edges_from(zip(z['src'].tolist(), z['dst'].tolist(), z['w'].tolist()))
    else:
        G.add_edges_from(zip(z['src'].tolist(), z['dst'].tolist()))
    return G


@pytest.fixture(scope='session')
def gpu_ctx(native_lib):
    from gem_b200 import _native
    ctx = _native.Context(0)
    yield ctx
    ctx.close()
