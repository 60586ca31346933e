"""Records tests/golden/hope_rounds.npz: the exact output of the Chebyshev HOPE solve (algorithm 2) on two seeded graphs,
for tests/test_gpu_hope_rounds.py.  Needs an H100; the file in the repository was recorded on an H100 80GB HBM3 from the
build that ran the Rayleigh-Ritz stop rule on the host and extracted X with two apply launches.

    python tests/golden/make_golden_hope_rounds.py [OUT.npz]
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

SBM = dict(n=20_000, block=100, seed=7)      # 200 communities: the 64 wanted values lie inside the cluster, as at bench size
SBM_ROWS, SBM_ROWS_SEED = 1024, 11
KARATE_SOLVER = dict(tol=1e-6, stop_rule=1, cheb_degree=16, cheb_range_log2=14, max_iters=30, min_iters=2, oversample=32,
                     seed=1234, algorithm=2)


def sbm_case(ctx):
    import bench
    from gem_b200 import _native, synth
    csr = synth.sbm(**SBM)
    g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)
    X, sig, st = g.hope(128, 0.01, algorithm=2, **bench.HOPE_SOLVER)
    g.free()
    rows = np.sort(np.random.default_rng(SBM_ROWS_SEED).choice(csr.n, SBM_ROWS, replace=False))
    return rows, X[rows], sig, st


def karate_case(ctx):
    """The Karate graph made undirected: 34 nodes, block width 36 > n, so every orthonormalisation drops columns and the
    solver refills them."""
    from gem_b200 import _native
    from gem_b200 import graph as hg
    e = np.loadtxt(os.path.join(HERE, 'karate.edgelist'))[:, :2].astype(np.int64)
    csr = hg.from_edges(34, np.concatenate((e[:, 0], e[:, 1])), np.concatenate((e[:, 1], e[:, 0])))
    g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)
    X, sig, st = g.hope(4, 0.01, **KARATE_SOLVER)
    g.free()
    return X, sig, st


def main():
    from gem_b200 import _native
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, 'hope_rounds.npz')
    ctx = _native.Context(0)
    rows, Xs, sig, st = sbm_case(ctx)
    Xk, sigk, stk = karate_case(ctx)
    ctx.close()
    np.savez_compressed(out, sbm_rows=rows, sbm_X=Xs, sbm_sigma=sig, sbm_iters=st['iters'], sbm_spmm=st['spmm_count'],
                        sbm_resid_est=np.float32(st['resid_est']), sbm_ritz_change=np.float32(st['ritz_change']),
                        karate_X=Xk, karate_sigma=sigk, karate_iters=stk['iters'],
                        karate_resid_est=np.float32(stk['resid_est']), karate_ritz_change=np.float32(stk['ritz_change']))
    print('wrote %s: sbm %d rounds / %d sweeps, karate %d rounds' % (out, st['iters'], st['spmm_count'], stk['iters']))


if __name__ == '__main__':
    main()
