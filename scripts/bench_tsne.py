"""scripts/bench_tsne.py -- t-SNE (gem_b200.evaluation.visualize_embedding.tsne, sklearn's defaults) on the HOPE d = 128
embedding of bench.py's SBM (1000-node blocks, seed 42, beta 0.01, bench.py's solver settings), per stage.

    python scripts/bench_tsne.py [--n 100000 1000000] [--sample 10000]

One JSON line per n: the card and its power limit, the stage times (host clock, each stage ending in a device
synchronise), the kNN time against the FP32 bound 2 n^2 d / 67 TFLOP/s (H100 SXM data sheet), the quadtree and gradient
milliseconds per iteration (device events), the final KL and the trustworthiness(12) of a random sample of rows.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FP32_PEAK = 67e12          # H100 SXM data sheet, dense FP32 (a 700 W card)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001 -- the numbers are still reported, without the card
        return dict(gpu='unknown (%s)' % e)


def trustworthiness(X, Y, k):
    """sklearn.manifold.trustworthiness (euclidean) with Gram-form distances, for samples of ~10^4 rows."""
    def sq(A):
        A = np.asarray(A, np.float64)
        s = (A * A).sum(1)
        D = s[:, None] + s[None, :] - 2.0 * (A @ A.T)
        np.fill_diagonal(D, np.inf)
        return D
    n = X.shape[0]
    order = np.argsort(sq(X), axis=1, kind='stable')
    rank = np.empty((n, n), np.int32)
    rank[np.arange(n)[:, None], order] = np.arange(n, dtype=np.int32)[None, :]
    nbr = np.argsort(sq(Y), axis=1, kind='stable')[:, :k]
    r = rank[np.arange(n)[:, None], nbr].astype(np.int64) + 1 - k
    return 1.0 - np.sum(r[r > 0]) * (2.0 / (n * k * (2.0 * n - 3.0 * k - 1.0)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, nargs='+', default=[100_000, 1_000_000])
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--sample', type=int, default=10_000)
    args = ap.parse_args()
    from gem_b200 import _native, synth
    from gem_b200.evaluation.visualize_embedding import tsne
    info = card()
    for n in args.n:
        ctx = _native.Context(0)
        csr = synth.sbm(n=n, block=1000, seed=42)
        g = _native.DeviceGraph(ctx, csr.n, csr.indptr, csr.indices, None)
        X, _, _ = g.hope(args.d, 0.01, tol=4e-3, stop_rule=1, cheb_degree=16, cheb_range_log2=14, max_iters=30,
                         min_iters=2, oversample=8, seed=1234)
        g.free()
        ctx.close()
        st = {}
        t0 = time.perf_counter()
        Y = tsne(X, stats=st)
        wall = time.perf_counter() - t0
        iters = st['n_iter'] + 1
        flop = 2.0 * n * n * args.d
        rng = np.random.RandomState(0)
        s = rng.choice(n, min(args.sample, n), replace=False)
        out = dict(info, workload='t-SNE of HOPE d=%d on SBM n=%d' % (args.d, n), n=n, d=args.d,
                   knn_ms=st['knn_ms'], knn_fp32_bound_ms=flop / FP32_PEAK * 1e3,
                   knn_share_of_fp32_peak=flop / FP32_PEAK * 1e3 / st['knn_ms'],
                   calib_ms=st['calib_ms'], sym_ms=st['sym_ms'], pca_ms=st['pca_ms'], opt_ms=st['opt_ms'],
                   tree_ms_per_iter=st['tree_ms'] / iters, grad_ms_per_iter=st['grad_ms'] / iters, iterations=iters,
                   total_ms=st['total_ms'], wall_s=wall, kl_divergence=st['kl_divergence'], nnz_P=st['nnz_P'],
                   finite=bool(np.all(np.isfinite(Y))),
                   trustworthiness12_sample=trustworthiness(X[s], Y[s], 12), sample=int(s.size))
        print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
