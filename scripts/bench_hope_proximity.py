"""scripts/bench_hope_proximity.py -- HOPE on its four proximities on one GPU, the general solver (algorithm 1) throughout.

    python scripts/bench_hope_proximity.py [--out DIR] [--d 128] [--alpha 0.5] [--skip-rmat]

Graphs:
  sbm1M      the 1M-node SBM of bench.py (synth.sbm, 1000-node blocks, seed 42); Katz at beta = 0.01, as bench.py
  rmat20lcc  the largest component (get_lcc) of device R-MAT scale 20 (Graph500 parameters, permuted, seed 42); Katz at
             beta = 0.5 / ||A||_2 (beta_over_rho = 0.5), since beta = 0.01 lies outside its convergence radius
Proximities: katz (the same-solver baseline), common_neighbors, adamic_adar, rooted_pagerank (alpha, default 0.5; J from
the default katz_tol 1e-7).  Solver: bench.HOPE_SOLVER (residual stop rule at tol 4e-3, at most 30 rounds) with
algorithm = 1, at d (default 128).
Per run:
  solve_ms      device time of the gemb_hope call (CUDA events); iters; sweeps (block-width SpMM sweeps); spmm_ms
  sweep_GBps    spmm_bytes * sweeps / spmm_ms: the compulsory bytes of the sweeps over their time
  converged
  resid_max     max_j max(||S v_j - sigma_j u_j||, ||S^T u_j - sigma_j v_j||) / sigma_max, fp64 on the host, S applied
                matrix-free (scipy products) with the solver's own J for the two series
The card's name and power limit are read in the same run.  Prints one JSON line per run and one for the whole (and writes
DIR/bench_hope_proximity.json when --out is given).
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
sys.path.insert(0, os.path.join(REPO, 'oracle'))

PROXIMITIES = ('katz', 'common_neighbors', 'adamic_adar', 'rooted_pagerank')


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit',
                                       '--format=csv,noheader,nounits'], text=True).strip().splitlines()[0]
        name, plim = [x.strip() for x in out.split(',')]
        return {'gpu': name, 'power_limit_w': plim}
    except Exception as exc:
        return {'gpu': 'unknown (%s)' % exc, 'power_limit_w': None}


def run(name, csr, A, d, proximity, alpha, katz_kw):
    import warnings
    import bench
    import hope_oracle as ho
    import proximity_oracle as po
    from gem_b200.embedding.hope import HOPE
    HOPE.hyper_params.clear()
    HOPE.hyper_params.update({'method_name': 'hope_gsvd'})
    kw = dict(bench.HOPE_SOLVER, algorithm=1, svd_error_probes=False)
    if proximity == 'katz':
        kw.update(katz_kw)
    else:
        kw.update(beta=0.01, proximity=proximity, alpha=alpha if proximity == 'rooted_pagerank' else None)
    m = HOPE(d=d, **kw)
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        X = m.learn_embedding(graph=csr)
    wall = time.perf_counter() - t0
    st = m.stats
    sig = np.asarray(m._sigma, dtype=np.float64)
    r = {'graph': name, 'n': csr.n, 'nnz': csr.nnz, 'proximity': proximity, 'd': d,
         'solve_ms': st['total_ms'], 'wall_s': wall, 'iters': st['iters'], 'sweeps': st['spmm_count'],
         'spmm_ms': st['spmm_ms'], 'spmm_bytes': st['spmm_bytes'],
         'sweep_GBps': st['spmm_bytes'] * st['spmm_count'] / (st['spmm_ms'] * 1e-3) / 1e9 if st['spmm_ms'] > 0 else None,
         'converged': st['converged'], 'resid_est': st['resid_est'], 'katz_terms': st['katz_terms'],
         'beta_used': st['beta_used'], 'sigma_top': float(sig[-1]), 'sigma_k': float(sig[0])}
    t0 = time.perf_counter()
    if proximity == 'katz':
        r1, r2, _, _ = ho.svd_residuals(A, st['beta_used'], X, st['katz_terms'], sigma=sig)
    else:
        op = po.proximity_operator(A, proximity, alpha=alpha, terms=st['katz_terms'] or None)
        r1, r2 = po.residuals(A, proximity, X, sig, S=op)
    r.update(resid_max=float(max(r1.max(), r2.max())), resid_host_s=time.perf_counter() - t0)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--alpha', type=float, default=0.5)
    ap.add_argument('--skip-rmat', action='store_true')
    a = ap.parse_args()
    from gem_b200 import _native, synth
    from gem_b200.graph import HostCSR
    from gem_b200.utils.graph_util import get_lcc
    out = {'card': card(), 'alpha': a.alpha, 'runs': []}
    graphs = [('sbm1M', lambda: synth.sbm(n=1_000_000, block=1000, seed=42), {'beta': 0.01})]
    if not a.skip_rmat:
        def rmat():
            with _native.Context(0) as ctx:
                indptr, indices, _ = _native.synth_rmat(ctx, 20, permute=True)
            return get_lcc(HostCSR(1 << 20, indptr, indices, symmetric=True))[0]
        graphs.append(('rmat20lcc', rmat, {'beta': 0.01, 'beta_over_rho': 0.5}))
    for name, make, katz_kw in graphs:
        csr = make()
        A = csr.to_scipy().astype(np.float64)
        for p in PROXIMITIES:
            out['runs'].append(run(name, csr, A, a.d, p, a.alpha, katz_kw))
        del csr, A
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_hope_proximity.json'), 'w') as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
