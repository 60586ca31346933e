"""scripts/bench_linkpred.py -- link prediction at scale on one GPU.

    python scripts/bench_linkpred.py --out DIR [--n 1000000] [--sample 32768] [--full-n 32768] [--max-k 1000]

Two workloads, each: split the graph at 0.8 (HostCSR, undirected, np.random.RandomState(seed)), train HOPE d = 128
(bench.HOPE_SOLVER) on the training graph, then evaluate with the training edges excluded on the device.
  sampled  the BASELINE SBM (1M nodes, 1000-node blocks, seed 42), n_sample_nodes = --sample, max_k = --max-k
  full     a --full-n node SBM (1024-node blocks, seed 42) evaluated on every node, max_k = --max-k
Reported per workload: host split (and sample) time, learn time, and the time of gemb_recon_create / _exclude /
_ranks / _top (host clock around calls that end in a device synchronise, so uploads of the CSRs are included) with
node pairs per second (n_eval^2 / time); MAP (with its bits) and the curve's precision at 100 and max_k; the card's
name and power limit.  Writes DIR/bench_linkpred.json and prints it as one line.  Needs a GPU; nothing falls back.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit',
                                       '--format=csv,noheader,nounits'], text=True).strip().splitlines()[0]
        name, plim = [x.strip() for x in out.split(',')]
        return {'gpu': name, 'power_limit_w': plim}
    except Exception as exc:
        return {'gpu': 'unknown (%s)' % exc, 'power_limit_w': None}


def workload(csr, n_sample, max_k, d, beta, seed):
    from bench import HOPE_SOLVER
    from gem_b200 import _native
    from gem_b200.embedding.hope import HOPE
    from gem_b200.evaluation import metrics
    from gem_b200.evaluation.evaluate_graph_reconstruction import _true_csr
    from gem_b200.evaluation.evaluate_link_prediction import split_and_sample
    r = {'n': csr.n, 'nnz': csr.nnz, 'n_sample_nodes': n_sample, 'max_k': max_k}
    t0 = time.perf_counter()
    train, test_s, train_s, node_l = split_and_sample(csr, 0.8, n_sample, True, np.random.RandomState(seed))
    r['split_sample_s'] = time.perf_counter() - t0
    r['train_nnz'], r['test_nnz_eval'], r['train_nnz_eval'] = train.nnz, test_s.nnz, train_s.nnz
    HOPE.hyper_params.clear(); HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
    model = HOPE(d=d, beta=beta, **HOPE_SOLVER)
    t0 = time.perf_counter()
    X = model.learn_embedding(graph=train)
    r['learn_s'] = time.perf_counter() - t0
    Xs = np.ascontiguousarray(X[node_l])
    n = node_l.size
    te_p, te_i = _true_csr(test_s, n)
    tr_p, tr_i = _true_csr(train_s, n)
    pairs = float(n) * n
    with _native.Context(0) as ctx:
        t0 = time.perf_counter()
        rec = _native.Reconstruction(ctx, Xs, True)
        t1 = time.perf_counter()
        rec.exclude(tr_p, tr_i)
        t2 = time.perf_counter()
        ranks, _ = rec.ranks(te_p, te_i, True)
        t3 = time.perf_counter()
        ti, tj, tw = rec.top(True, max_k)
        t4 = time.perf_counter()
        rec.free()
    MAP, _, count = metrics.map_from_ranks(n, te_p, ranks, False)
    prec, _ = metrics.precision_curve_from_top(ti, tj, tw, metrics.csr_has_edge(n, te_p, te_i), max_k)
    for k, a, b in (('create', t0, t1), ('exclude', t1, t2), ('ranks', t2, t3), ('top', t3, t4)):
        r[k + '_ms'] = (b - a) * 1e3
    for k in ('create', 'ranks', 'top'):
        r[k + '_pairs_per_s'] = pairs / (r[k + '_ms'] * 1e-3)
    r.update(MAP=MAP, MAP_hex=float(MAP).hex(), nodes_counted=count, n_top=int(ti.size),
             prec_at_100=prec[99] if len(prec) >= 100 else None, prec_at_max_k=prec[-1] if prec else None)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--n', type=int, default=1_000_000)
    ap.add_argument('--sample', type=int, default=32768)
    ap.add_argument('--full-n', type=int, default=32768)
    ap.add_argument('--max-k', type=int, default=1000)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--beta', type=float, default=0.01)
    ap.add_argument('--seed', type=int, default=42, help='seed of the split and the node sample')
    args = ap.parse_args()
    from gem_b200 import synth
    os.makedirs(args.out, exist_ok=True)
    res = {'metric': 'link_prediction', 'card': card()}
    csr = synth.sbm(n=args.n, block=1000, seed=42)
    res['sampled'] = workload(csr, args.sample, args.max_k, args.d, args.beta, args.seed)
    del csr
    csr = synth.sbm(n=args.full_n, block=1024 if args.full_n % 1024 == 0 else 1000, seed=42)
    res['full'] = workload(csr, None, args.max_k, args.d, args.beta, args.seed)
    with open(os.path.join(args.out, 'bench_linkpred.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
