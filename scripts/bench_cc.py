"""scripts/bench_cc.py -- weakly connected components and largest-component extraction on one GPU.

    python scripts/bench_cc.py [--out DIR] [--scales 20 24] [--repeats 5] [--no-host]

Graphs: device R-MAT (gemb_synth_rmat, Graph500 parameters, permuted, seed 42) at each --scales value, and the
1M-node SBM of BASELINE config 2 (synth.sbm, 1000-node blocks, seed 42).  Per graph, after one warm-up call:
  label    gemb_cc_create's labelling: device time from CUDA events around its kernels (uploads outside), stored
           edges per second, and compulsory bytes (read indptr 8 (n + 1) and indices 4 nnz, write 4 n labels) over that
           time against the 3.35 TB/s of the H100 SXM data sheet
  extract  gemb_cc_lcc's extraction of the largest component, the same three figures (compulsory: read 4 n labels,
           8 (n + 1) indptr and the 4 m kept indices; write 8 k node_l, 8 (k + 1) indptr and 4 m indices)
  e2e      get_lcc(HostCSR) on the host clock: context, upload, labelling, extraction and copies back
  host     scipy connected_components(connection='weak') + the NumPy induced graph (graph_util.induced_graph) on the
           same CSR, on the host clock (--no-host skips it)
The card's name and power limit are read in the same run.  Prints one JSON line (and writes DIR/bench_cc.json).
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

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit',
                                       '--format=csv,noheader,nounits'], text=True).strip().splitlines()[0]
        name, plim = [x.strip() for x in out.split(',')]
        return {'gpu': name, 'power_limit_w': plim}
    except Exception as exc:
        return {'gpu': 'unknown (%s)' % exc, 'power_limit_w': None}


def _rate(ms, items, nbytes):
    s = ms * 1e-3
    return {'ms': ms, 'edges_per_s': items / s, 'bytes': nbytes, 'hbm_share': nbytes / s / HBM_BYTES_PER_S}


def workload(ctx, name, n, indptr, indices, repeats, host):
    from gem_b200 import _native
    from gem_b200.graph import HostCSR
    from gem_b200.utils.graph_util import get_lcc, induced_graph
    nnz = int(indptr[-1])
    r = {'graph': name, 'n': n, 'nnz': nnz}
    label, extract = [], []
    for it in range(repeats + 1):
        with _native.Components(ctx, n, indptr, indices) as cc:
            node_l, _, _, _ = cc.lcc()
            lm, em = cc.times()
            info = (cc.n_comp, cc.lcc_root, cc.lcc_size, cc.lcc_nnz)
        if it:                                            # the first call warms up
            label.append(lm)
            extract.append(em)
    n_comp, root, k, m = info
    r.update(components=n_comp, lcc_root=root, lcc_size=k, lcc_nnz=m)
    r['label'] = _rate(float(np.median(label)), nnz, 8.0 * (n + 1) + 4.0 * nnz + 4.0 * n)
    r['extract'] = _rate(float(np.median(extract)), m, 4.0 * n + 8.0 * (n + 1) + 4.0 * m + 8.0 * k + 8.0 * (k + 1) + 4.0 * m)
    r['label_ms_all'], r['extract_ms_all'] = label, extract
    csr = HostCSR(n, indptr, indices)
    get_lcc(csr)
    t0 = time.perf_counter()
    H, node_l2 = get_lcc(csr)
    r['e2e_ms'] = (time.perf_counter() - t0) * 1e3
    assert np.array_equal(node_l, node_l2) and H.nnz == m
    if host:
        import scipy.sparse as sp
        from scipy.sparse.csgraph import connected_components
        t0 = time.perf_counter()
        A = sp.csr_matrix((np.ones(nnz, dtype=np.int8), indices, indptr), shape=(n, n))
        nc, lab = connected_components(A, directed=True, connection='weak')
        t1 = time.perf_counter()
        sizes = np.bincount(lab)
        big = lab == int(np.argmax(sizes))
        Hh = induced_graph(csr, np.flatnonzero(big))
        t2 = time.perf_counter()
        assert nc == n_comp and Hh.nnz == m and int(big.sum()) == k
        r['host'] = {'scipy_cc_ms': (t1 - t0) * 1e3, 'numpy_induced_ms': (t2 - t1) * 1e3, 'total_ms': (t2 - t0) * 1e3}
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--scales', type=int, nargs='+', default=[20, 24])
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--no-host', action='store_true')
    args = ap.parse_args()
    from gem_b200 import _native, synth
    res = {'metric': 'weakly_connected_components', 'card': card(), 'results': []}
    with _native.Context(0) as ctx:
        for s in args.scales:
            indptr, indices, _ = _native.synth_rmat(ctx, s, permute=True)
            res['results'].append(workload(ctx, 'rmat%d' % s, 1 << s, indptr, indices, args.repeats, not args.no_host))
            del indptr, indices
        csr = synth.sbm(n=1_000_000, block=1000, seed=42)
        res['results'].append(workload(ctx, 'sbm1m', csr.n, csr.indptr, csr.indices, args.repeats, not args.no_host))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_cc.json'), 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
