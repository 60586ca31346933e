"""scripts/bench_nc.py -- node classification at scale on one GPU.

    python scripts/bench_nc.py --out DIR [--n 1000000] [--d 128] [--cpu-classes 2] [--profile]

Workload: the BASELINE SBM (1M nodes, 1000 blocks of 1000 consecutive ids, seed 42), a HOPE d = 128 embedding
(bench.HOPE_SOLVER), label = node // 1000 (1000 one-hot labels), test_ratio 0.5, seed 42.  The evaluation runs twice.
Reported: the card's name and power limit (read in the same run); split (host), fit and top-k times (host clock around
calls that end in a device synchronise, uploads included); iterations per label (min / median / max); evaluations,
compulsory bytes of the fit's launches (include/gemb200.h, gemb_nc_stats.eval_bytes) and of top-k (X_test in,
decision values out and back in, predictions out) with the achieved GB/s over the fit's device time / the top-k time;
micro / macro F1 with their bits, equal across the two runs.  CPU arm: the fp64 oracle (scipy L-BFGS-B, tight) on
--cpu-classes labels over the same training rows, given per label.  --profile: a third run under torch.profiler,
kernel totals written to DIR/bench_nc_profile.txt.  Writes DIR/bench_nc.json and prints it as one line.
Needs a GPU; nothing falls back.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'scripts'))
from bench_linkpred import card  # noqa: E402


def run(X, Y, args):
    from gem_b200.evaluation.evaluate_node_classification import evaluateNodeClassification
    st = {}
    mi, ma = evaluateNodeClassification(X, Y, 0.5, seed=args.seed, stats=st)
    fs = st['fit_stats']
    it = st['iters'][st['status'] != 2]
    m = st['test_idx'].size
    L, d = Y.shape[1], X.shape[1]
    k_tot = int(st['pred_indptr'][-1])
    topk_bytes = 4.0 * m * d + 8.0 * m * L + 4.0 * k_tot
    r = {'split_ms': st['split_ms'], 'fit_ms': st['fit_ms'], 'topk_ms': st['topk_ms'],
         'fit_device_ms': fs['total_ms'], 'evaluations': fs['evaluations'], 'panels': fs['panels'],
         'iters_min': int(it.min()), 'iters_median': float(np.median(it)), 'iters_max': int(it.max()),
         'unconverged': int(fs['unconverged']), 'fit_bytes': fs['eval_bytes'],
         'fit_GBps': fs['eval_bytes'] / (fs['total_ms'] * 1e-3) / 1e9, 'topk_bytes': topk_bytes,
         'topk_GBps': topk_bytes / (st['topk_ms'] * 1e-3) / 1e9,
         'micro_f1': mi, 'macro_f1': ma, 'micro_hex': float(mi).hex(), 'macro_hex': float(ma).hex()}
    return r, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--n', type=int, default=1_000_000)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--beta', type=float, default=0.01)
    ap.add_argument('--seed', type=int, default=42)
    ap.add_argument('--cpu-classes', type=int, default=2)
    ap.add_argument('--profile', action='store_true')
    args = ap.parse_args()
    from bench import HOPE_SOLVER
    from gem_b200 import synth
    from gem_b200.embedding.hope import HOPE
    os.makedirs(args.out, exist_ok=True)
    res = {'metric': 'node_classification', 'card': card(), 'n': args.n, 'd': args.d, 'test_ratio': 0.5}
    csr = synth.sbm(n=args.n, block=1000, seed=42)
    HOPE.hyper_params.clear(); HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
    t0 = time.perf_counter()
    X = HOPE(d=args.d, beta=args.beta, **HOPE_SOLVER).learn_embedding(graph=csr)
    res['hope_s'] = time.perf_counter() - t0
    del csr
    import scipy.sparse as sp
    L = (args.n + 999) // 1000
    Y = sp.csr_matrix((np.ones(args.n, dtype=np.int8), np.arange(args.n) // 1000, np.arange(args.n + 1)),
                      shape=(args.n, L))
    res['labels'] = L
    runs = []
    for _ in range(2):
        r, st = run(X, Y, args)
        runs.append(r)
    res['runs'] = runs
    res['f1_bits_equal'] = runs[0]['micro_hex'] == runs[1]['micro_hex'] and runs[0]['macro_hex'] == runs[1]['macro_hex']
    # CPU arm: the fp64 oracle on the first --cpu-classes labels, same training rows
    sys.path.insert(0, os.path.join(REPO, 'oracle'))
    import nc_oracle as no
    tr = st['train_idx']
    Xtr = np.asarray(X[tr], dtype=np.float64)
    Ytr = Y[tr][:, :args.cpu_classes].toarray()
    t0 = time.perf_counter()
    Wc = no.fit(Xtr, Ytr)
    cpu_s = time.perf_counter() - t0
    res['cpu_oracle'] = {'classes': args.cpu_classes, 'rows': int(tr.size), 'total_s': cpu_s,
                         'per_class_s': cpu_s / args.cpu_classes, 'threads': os.environ.get('OMP_NUM_THREADS'),
                         'note': 'scipy L-BFGS-B to gtol 1e-13 on the listed labels only; not extrapolated'}
    cert = no.certificate(Xtr, Ytr, 1.0, st['W'][:args.cpu_classes])
    res['gpu_certificate_first_classes'] = [float(c) for c in cert]
    res['gpu_vs_cpu_max_rel_w'] = float(np.abs(st['W'][:args.cpu_classes] - Wc).max() / np.abs(Wc).max())
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(X, Y, args)
        with open(os.path.join(args.out, 'bench_nc_profile.txt'), 'w') as f:
            f.write(prof.key_averages().table(sort_by='cuda_time_total', row_limit=30))
        del torch
    with open(os.path.join(args.out, 'bench_nc.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
