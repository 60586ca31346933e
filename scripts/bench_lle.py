"""scripts/bench_lle.py -- LocallyLinearEmbedding's two operator forms on one GPU.

    python scripts/bench_lle.py [--out DIR] [--d 128] [--skip-explicit] [--skip-rmat]

Runs:
  sbm1M      the 1M-node SBM of BASELINE config 2 (synth.sbm, 1000-node blocks, seed 42), explicit and composite
  rmat20lcc  the largest component (get_lcc) of device R-MAT scale 20 (gemb_synth_rmat, Graph500 parameters, permuted,
             seed 42), composite only (the explicit C would hold ~2.1e10 entries)
Per run, at d (default 128), LLE's default solver options (tol 1e-6):
  host_op_s  forming the operator on the host: C = c I - M^T M (explicit), or P = D^-1 W and P^T (composite)
  upload_s   gemb_graph_upload of it, host clock around the DeviceGraph constructor
  solve_ms   device time of the gemb_hope call (CUDA events); iters, sweeps (block-width SpMM sweeps; a composite
             application counts two), spmm_ms, converged
  resid_max  max_j ||M^T M x_j - sigma_j^2 x_j|| / (||x_j|| ||M||_2^2), fp64 on the host, matrix-free (scipy products)
The card's name and power limit are read in the same run.  Prints one JSON line per run and one for the whole (and writes
DIR/bench_lle.json when --out is given).
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


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit',
                                       '--format=csv,noheader,nounits'], text=True).strip().splitlines()[0]
        name, plim = [x.strip() for x in out.split(',')]
        return {'gpu': name, 'power_limit_w': plim}
    except Exception as exc:
        return {'gpu': 'unknown (%s)' % exc, 'power_limit_w': None}


def run(name, csr, d, operator):
    import lle_composite_oracle as lc
    from gem_b200 import _native
    from gem_b200.embedding.lle import lle_composite_operator, lle_operator
    r = {'graph': name, 'n': csr.n, 'nnz_W': csr.nnz, 'operator': operator, 'd': d}
    t0 = time.perf_counter()
    if operator == 'explicit':
        op, c = lle_operator(csr)
        tr = {}
        mode = 1
        r['c'] = c
    else:
        op, op_t = lle_composite_operator(csr)
        tr = {'indptr_t': op_t.indptr, 'indices_t': op_t.indices, 'data_t': op_t.data_f32()}
        mode = 2
    r['host_op_s'] = time.perf_counter() - t0
    r['nnz_uploaded'] = op.nnz * (1 if mode == 1 else 2)
    with _native.Context(0) as ctx:
        t0 = time.perf_counter()
        g = _native.DeviceGraph(ctx, op.n, op.indptr, op.indices, op.data_f32(), **tr)
        r['upload_s'] = time.perf_counter() - t0
        with g:
            V, lam, st = g.hope(d + 1, 0.0, spectral_mode=mode, tol=1e-6, max_iters=300)
    lam = np.asarray(lam, dtype=np.float64)
    s = np.sqrt(np.maximum((c - lam) if mode == 1 else -lam, 0.0))
    r.update(solve_ms=st['total_ms'], iters=st['iters'], sweeps=st['spmm_count'], spmm_ms=st['spmm_ms'],
             converged=st['converged'], norm2_A=st['norm2_A'])
    t0 = time.perf_counter()
    res, nrm = lc.composite_residuals(csr.to_scipy(), V[:, 1:], s[1:])
    r.update(resid_max=float(res.max()), norm_M2=nrm, sigma2_head=(s[:4] ** 2).tolist(), resid_host_s=time.perf_counter() - t0)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--skip-explicit', action='store_true')
    ap.add_argument('--skip-rmat', action='store_true')
    a = ap.parse_args()
    from gem_b200 import _native, synth
    from gem_b200.graph import HostCSR
    from gem_b200.utils.graph_util import get_lcc
    out = {'card': card(), 'runs': []}
    sbm = synth.sbm(n=1_000_000, block=1000, seed=42)
    for op in (() if a.skip_explicit else ('explicit',)) + ('composite',):
        out['runs'].append(run('sbm1M', sbm, a.d, op))
    del sbm
    if not a.skip_rmat:
        with _native.Context(0) as ctx:
            indptr, indices, _ = _native.synth_rmat(ctx, 20, permute=True)
        lcc, _ = get_lcc(HostCSR(1 << 20, indptr, indices, symmetric=True))
        out['runs'].append(run('rmat20lcc', lcc, a.d, 'composite'))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_lle.json'), 'w') as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
